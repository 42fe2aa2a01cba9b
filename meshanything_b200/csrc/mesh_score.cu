// mesh_score.cu -- Chamfer distance and normal consistency of candidate meshes against the point cloud they were made
// from, for best-of-N sampling (DESIGN.md section 1, row f6, gives the metric).
//
// S shapes x N candidates per call.  A candidate is a face soup [F][3][3] as MeshAnything.forward returns it (a face is
// valid iff its first coordinate is not NaN); its cloud is [P][6] (xyz | normal), already in the output frame.
//   mesh_score_p2m_kernel   one thread per cloud point: nearest valid face by the fixed fp32 formula of tri_dist.cuh
//                           (strict < over ascending faces: lowest index on ties), faces staged through shared memory
//                           with their per-face terms computed once; |n_p . unit normal of that face|.
//   mesh_score_m2p_kernel   one thread per quadrature point (16 sub-triangle centroids per face): nearest cloud point
//                           by d^2 = (dx dx + dy dy) + dz dz (lowest index on ties), cloud xyz staged through shared
//                           memory; weight = face area / 16 in double; |unit face normal . n_q|.
//   mesh_score_reduce_kernel  per candidate, the per-tile fp64 partials of both kernels in tile order.
// Every fp32 step is an explicit round-to-nearest intrinsic and every fp64 sum runs in a fixed order with no atomics, so
// a call is bit-deterministic and tests/mesh_score_oracle.py restates the per-point results bit for bit.
#include "canon.cuh"
#include "tri_dist.cuh"
#include "workspace.h"

namespace ma {

constexpr int kMsThreads = 256;
constexpr int kMsFaceChunk = 64;     // faces per shared-memory stage of the p2m kernel (64 x 88 B)
constexpr int kMsCloudChunk = 1024;  // cloud points per shared-memory stage of the m2p kernel (1024 x 16 B)
constexpr int kMsQuad = 16;          // quadrature points per face: s^2 sub-triangles, s = 4

// barycentric numerators (over 3s = 12) of the 16 sub-triangle centroids: the 10 upward ones (i, j), i + j <= 3, at
// ((3i+1)/12, (3j+1)/12), then the 6 downward ones, i + j <= 2, at ((3i+2)/12, (3j+2)/12); i outer, j inner
__constant__ unsigned char kMsQuadU[kMsQuad] = {1, 1, 1, 1, 4, 4, 4, 7, 7, 10, 2, 2, 2, 5, 5, 8};
__constant__ unsigned char kMsQuadV[kMsQuad] = {1, 4, 7, 10, 1, 4, 7, 1, 4, 1, 2, 5, 8, 2, 5, 2};

__device__ __forceinline__ wt_v3 ms_load(const float* m) { return {m[0], m[1], m[2]}; }

// cross(b - a, c - a) / sqrt(its squared length) in fixed fp32 order; the zero vector when that length is zero
__device__ __forceinline__ wt_v3 ms_unit_normal(wt_v3 a, wt_v3 b, wt_v3 c) {
  const wt_v3 n = wt_cross(wt_sub(b, a), wt_sub(c, a));
  const float nn = wt_dot(n, n);
  if (!(nn > 0.0f)) return {0.0f, 0.0f, 0.0f};
  const float l = __fsqrt_rn(nn);
  return {__fdiv_rn(n.x, l), __fdiv_rn(n.y, l), __fdiv_rn(n.z, l)};
}

// face area in double from the fp32 vertex differences (surface_area_kernel's formula, without contraction)
__device__ __forceinline__ double ms_area(wt_v3 a, wt_v3 b, wt_v3 c) {
  const double ux = __dsub_rn(b.x, a.x), uy = __dsub_rn(b.y, a.y), uz = __dsub_rn(b.z, a.z);
  const double wx = __dsub_rn(c.x, a.x), wy = __dsub_rn(c.y, a.y), wz = __dsub_rn(c.z, a.z);
  const double nx = __dsub_rn(__dmul_rn(uy, wz), __dmul_rn(uz, wy));
  const double ny = __dsub_rn(__dmul_rn(uz, wx), __dmul_rn(ux, wz));
  const double nz = __dsub_rn(__dmul_rn(ux, wy), __dmul_rn(uy, wx));
  return __dmul_rn(0.5, __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(nx, nx), __dmul_rn(ny, ny)), __dmul_rn(nz, nz))));
}

// out[k] = sum of v[k] over the CTA, in a fixed order (shuffle tree per warp, then the warps in order); thread 0 writes
template <int NV>
__device__ __forceinline__ void ms_block_sum(double (&v)[NV], double* __restrict__ out) {
  __shared__ double red[kMsThreads / 32][NV];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < NV; k++)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[k] = __dadd_rn(v[k], __shfl_down_sync(0xffffffffu, v[k], o));
  if (lane == 0)
#pragma unroll
    for (int k = 0; k < NV; k++) red[warp][k] = v[k];
  __syncthreads();
  if (threadIdx.x == 0)
#pragma unroll
    for (int k = 0; k < NV; k++) {
      double s = 0.0;
#pragma unroll
      for (int w = 0; w < kMsThreads / 32; w++) s = __dadd_rn(s, red[w][k]);
      out[k] = s;
    }
}

// grid (ceil(P / 256), S N); part [S N][tiles][2] = {sum of distances, sum of |n_p . n_f|} of the tile's points
__global__ void __launch_bounds__(kMsThreads) mesh_score_p2m_kernel(const float* __restrict__ meshes,
                                                                    const float* __restrict__ clouds, int N, int F,
                                                                    int P, double* __restrict__ part,
                                                                    float* __restrict__ point_dist,
                                                                    int32_t* __restrict__ point_face) {
  __shared__ wt_tri tri[kMsFaceChunk];
  __shared__ int ok[kMsFaceChunk];
  const int sn = blockIdx.y, s = sn / N;
  const float* mesh = meshes + (size_t)sn * F * 9;
  const int i = blockIdx.x * kMsThreads + threadIdx.x;
  const bool active = i < P;
  wt_v3 p = {0.0f, 0.0f, 0.0f}, np = {0.0f, 0.0f, 0.0f};
  if (active) {
    const float* c = clouds + ((size_t)s * P + i) * 6;
    p = ms_load(c);
    np = ms_load(c + 3);
  }
  float best = INFINITY;
  int bf = -1;
  for (int f0 = 0; f0 < F; f0 += kMsFaceChunk) {
    const int nf = min(kMsFaceChunk, F - f0);
    __syncthreads();
    if (threadIdx.x < nf) {
      const float* m = mesh + (size_t)(f0 + threadIdx.x) * 9;
      const bool valid = !isnan(m[0]);
      ok[threadIdx.x] = valid;
      if (valid) tri[threadIdx.x] = wt_tri_prep(ms_load(m), ms_load(m + 3), ms_load(m + 6));
    }
    __syncthreads();
    if (active)
      for (int t = 0; t < nf; t++) {
        if (!ok[t]) continue;
        const float d = wt_tri_dist(p, tri[t]);
        if (d < best) { best = d; bf = f0 + t; }
      }
  }
  double v[2] = {0.0, 0.0};
  if (active && bf >= 0) {
    const float* m = mesh + (size_t)bf * 9;
    const wt_v3 n = ms_unit_normal(ms_load(m), ms_load(m + 3), ms_load(m + 6));
    v[0] = (double)best;
    v[1] = (double)fabsf(wt_dot(np, n));
  }
  if (active && point_dist) {
    point_dist[(size_t)sn * P + i] = best;
    point_face[(size_t)sn * P + i] = bf;
  }
  ms_block_sum<2>(v, part + ((size_t)sn * gridDim.x + blockIdx.x) * 2);
}

// grid (ceil(16 F / 256), S N); part [S N][tiles][4] = {sum w d, sum w |n_f . n_q|, sum w, valid faces} of the tile
__global__ void __launch_bounds__(kMsThreads) mesh_score_m2p_kernel(const float* __restrict__ meshes,
                                                                    const float* __restrict__ clouds, int N, int F,
                                                                    int P, double* __restrict__ part,
                                                                    float* __restrict__ quad_dist,
                                                                    int32_t* __restrict__ quad_point) {
  __shared__ float4 cxyz[kMsCloudChunk];
  const int sn = blockIdx.y, s = sn / N;
  const int q = blockIdx.x * kMsThreads + threadIdx.x, f = q / kMsQuad, k = q % kMsQuad;
  const float* cloud = clouds + (size_t)s * P * 6;
  const float* m = meshes + ((size_t)sn * F + f) * 9;
  const bool valid = f < F && !isnan(m[0]);
  wt_v3 a = {0.0f, 0.0f, 0.0f}, b = a, c = a, x = a;
  if (valid) {
    a = ms_load(m); b = ms_load(m + 3); c = ms_load(m + 6);
    const wt_v3 ab = wt_sub(b, a), ac = wt_sub(c, a);
    const float u = __fdiv_rn((float)kMsQuadU[k], 12.0f), w = __fdiv_rn((float)kMsQuadV[k], 12.0f);
    x = {__fadd_rn(__fadd_rn(a.x, __fmul_rn(u, ab.x)), __fmul_rn(w, ac.x)),
         __fadd_rn(__fadd_rn(a.y, __fmul_rn(u, ab.y)), __fmul_rn(w, ac.y)),
         __fadd_rn(__fadd_rn(a.z, __fmul_rn(u, ab.z)), __fmul_rn(w, ac.z))};
  }
  float best = INFINITY;
  int bj = -1;
  for (int j0 = 0; j0 < P; j0 += kMsCloudChunk) {
    const int nj = min(kMsCloudChunk, P - j0);
    __syncthreads();
    for (int t = threadIdx.x; t < nj; t += kMsThreads) {
      const float* y = cloud + (size_t)(j0 + t) * 6;
      cxyz[t] = make_float4(y[0], y[1], y[2], 0.0f);
    }
    __syncthreads();
    if (valid) {
#pragma unroll 4
      for (int t = 0; t < nj; t++) {
        const float4 y = cxyz[t];
        const float dx = __fsub_rn(x.x, y.x), dy = __fsub_rn(x.y, y.y), dz = __fsub_rn(x.z, y.z);
        const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
        if (d2 < best) { best = d2; bj = j0 + t; }
      }
    }
  }
  double v[4] = {0.0, 0.0, 0.0, 0.0};
  if (valid) {
    const float d = __fsqrt_rn(best);
    const wt_v3 n = ms_unit_normal(a, b, c);
    const float nc = fabsf(wt_dot(ms_load(cloud + (size_t)bj * 6 + 3), n));
    const double w = __dmul_rn(ms_area(a, b, c), 1.0 / kMsQuad);
    v[0] = __dmul_rn(w, (double)d);
    v[1] = __dmul_rn(w, (double)nc);
    v[2] = w;
    v[3] = k == 0 ? 1.0 : 0.0;
  }
  if (f < F && quad_dist) {
    quad_dist[(size_t)sn * F * kMsQuad + q] = valid ? __fsqrt_rn(best) : INFINITY;
    quad_point[(size_t)sn * F * kMsQuad + q] = valid ? bj : -1;
  }
  ms_block_sum<4>(v, part + ((size_t)sn * gridDim.x + blockIdx.x) * 4);
}

// one thread per candidate: the tiles' partials in tile order -> {p2m, m2p, nc_p, nc_m}, valid-face count
__global__ void mesh_score_reduce_kernel(const double* __restrict__ part_p, int tiles_p, const double* __restrict__ part_q,
                                         int tiles_q, int SN, int P, double* __restrict__ out,
                                         int32_t* __restrict__ out_faces) {
  const int sn = blockIdx.x * blockDim.x + threadIdx.x;
  if (sn >= SN) return;
  double d = 0.0, ncp = 0.0;
  for (int t = 0; t < tiles_p; t++) {
    d = __dadd_rn(d, part_p[((size_t)sn * tiles_p + t) * 2]);
    ncp = __dadd_rn(ncp, part_p[((size_t)sn * tiles_p + t) * 2 + 1]);
  }
  double wd = 0.0, wnc = 0.0, w = 0.0, cnt = 0.0;
  for (int t = 0; t < tiles_q; t++) {
    const double* r = part_q + ((size_t)sn * tiles_q + t) * 4;
    wd = __dadd_rn(wd, r[0]);
    wnc = __dadd_rn(wnc, r[1]);
    w = __dadd_rn(w, r[2]);
    cnt = __dadd_rn(cnt, r[3]);
  }
  const bool any = cnt > 0.0, area = w > 0.0;
  out[(size_t)sn * 4 + 0] = any ? __ddiv_rn(d, (double)P) : INFINITY;
  out[(size_t)sn * 4 + 1] = area ? __ddiv_rn(wd, w) : INFINITY;
  out[(size_t)sn * 4 + 2] = any ? __ddiv_rn(ncp, (double)P) : 0.0;
  out[(size_t)sn * 4 + 3] = area ? __ddiv_rn(wnc, w) : 0.0;
  out_faces[sn] = (int32_t)cnt;
}

static int ms_tiles_p(int P) { return (P + kMsThreads - 1) / kMsThreads; }
static int ms_tiles_q(int F) { return (int)(((long long)F * kMsQuad + kMsThreads - 1) / kMsThreads); }
static bool ms_shape_ok(int S, int N, int F, int P) {
  return S >= 1 && N >= 1 && F >= 1 && P >= 1 && (long long)S * N <= 65535 && F <= (1 << 26) && P <= (1 << 26);
}

// the per-tile partials of both directions
struct MsBuffers {
  double *part_p, *part_q;
  size_t total;
};

static MsBuffers ms_buffers(int S, int N, int F, int P, void* ws) {
  const size_t sn = (size_t)S * N;
  Carver c(ws);
  MsBuffers b;
  b.part_p = c.take<double>(sn * ms_tiles_p(P) * 2);
  b.part_q = c.take<double>(sn * ms_tiles_q(F) * 4);
  b.total = c.total;
  return b;
}

}  // namespace ma

using namespace ma;

extern "C" {

size_t ma_mesh_score_workspace_bytes(int S, int N, int F, int P) {
  if (!ms_shape_ok(S, N, F, P)) return 0;
  return ms_buffers(S, N, F, P, nullptr).total;
}

int ma_mesh_score(const float* meshes, const float* clouds, int S, int N, int F, int P, double* out,
                  int32_t* out_faces, float* point_dist, int32_t* point_face, float* quad_dist, int32_t* quad_point,
                  void* ws, void* stream) {
  if (!meshes || !clouds || !out || !out_faces || !ws || !ms_shape_ok(S, N, F, P) || (!point_dist != !point_face) ||
      (!quad_dist != !quad_point)) {
    set_error("ma_mesh_score: bad arguments");
    return 1;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const int sn = S * N, tiles_p = ms_tiles_p(P), tiles_q = ms_tiles_q(F);
  const MsBuffers b = ms_buffers(S, N, F, P, ws);
  mesh_score_p2m_kernel<<<dim3(tiles_p, sn), kMsThreads, 0, st>>>(meshes, clouds, N, F, P, b.part_p, point_dist,
                                                                   point_face);
  mesh_score_m2p_kernel<<<dim3(tiles_q, sn), kMsThreads, 0, st>>>(meshes, clouds, N, F, P, b.part_q, quad_dist,
                                                                   quad_point);
  mesh_score_reduce_kernel<<<(sn + 63) / 64, 64, 0, st>>>(b.part_p, tiles_p, b.part_q, tiles_q, sn, P, out, out_faces);
  count_launch(3);
  return check_launch("ma_mesh_score") ? 0 : 1;
}

}  // extern "C"
