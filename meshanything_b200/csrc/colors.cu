// colors.cu -- the colours of a scan carried onto the mesh made from it, for `--transfer_colors` (DESIGN.md section 1.9
// defines it).
//
// The vertices and the points arrive already in the points' frame ((x - c) / L, colors.py), fp32 [V][3] and [N][3].
//   (a) assign     colors_assign_kernel, one thread per point: the nearest face by wt_tri_dist (strict < over
//                  ascending faces: the lowest index on ties, as mesh_score_p2m_kernel picks), faces staged through
//                  shared memory with their per-face terms computed once; the barycentric weights of the nearest point
//                  on that face (wt_tri_bary).  A point farther than r from every face is unused.
//   (b) accumulate colors_accum_kernel, a grid-stride loop over the points: W[v] += llrint(w_k 2^24) and
//                  C[v][ch] += llrint(fl32(w_k c_ch) 2^24) at the three corners of each used point's face, unsigned 64-bit
//                  sums in shared memory while V fits (kClSharedMaxV), added to the global sums once per CTA.
//   (c) fallback   colors_list_kernel lists the vertices with W = 0; colors_nearest_kernel finds each one's nearest point
//                  by d^2 = (dx dx + dy dy) + dz dz, lowest index on ties, as an atomicMin over the 64-bit key
//                  (fp32 bits of d^2, index).  Its fixed grid reads the list's length on the device, so a call with no
//                  such vertex costs one launch of CTAs that return at once and needs no read-back.
//   (d) finish     colors_finish_kernel: fl32(C / W) in fp64 per channel, or the colour of the nearest point.
// Every sum is an integer sum and every fp32 step an explicit round-to-nearest intrinsic, so a call is bit-deterministic
// and tests/colors_oracle.py restates the faces, the weights, the sums, the colours and the stats bit for bit.
#include <stdint.h>

#include "tri_dist.cuh"
#include "workspace.h"

namespace ma {

constexpr int kClThreads = 256;
constexpr int kClAccThreads = 1024;        // accumulation: one CTA per SM, so each SM adds its shared sums once
constexpr int kClFaceChunk = 64;           // faces per shared-memory stage of the assignment (64 x 88 B)
constexpr int kClPointChunk = 1024;        // points per shared-memory stage of the fallback search (1024 x 16 B)
constexpr int kClTile = 16384;             // points one fallback work item scans
constexpr int kClMaxN = 1 << 24;           // the cap shared by every point-cloud stage; keeps every sum below 2^50
constexpr int kClMaxF = 1 << 16;           // one thread per point scans every face: beyond this a search structure pays
constexpr int kClMaxV = 3 * kClMaxF;       // an unmerged soup of kClMaxF faces
constexpr int kClSharedMaxV = 4096;        // 4096 x 32 B = 128 KB of shared sums per CTA
constexpr float kClScale = 16777216.0f;    // 2^24: the fixed point of the sums

__device__ __forceinline__ wt_v3 cl_load(const float* m) { return {m[0], m[1], m[2]}; }

__device__ __forceinline__ unsigned long long cl_fix(float x) {
  return (unsigned long long)__float2ll_rn(__fmul_rn(x, kClScale));
}

// grid ceil(N / 256); face[i], dist[i], weight[i][3] of every point; stats[0] += used points, stats[1] += beyond r
__global__ void __launch_bounds__(kClThreads) colors_assign_kernel(const float* __restrict__ verts,
                                                                  const int32_t* __restrict__ faces, int F,
                                                                  const float* __restrict__ points, int N, float r,
                                                                  int32_t* __restrict__ face_out,
                                                                  float* __restrict__ dist_out,
                                                                  float* __restrict__ weight_out,
                                                                  unsigned long long* __restrict__ stats) {
  __shared__ wt_tri tri[kClFaceChunk];
  const int i = blockIdx.x * kClThreads + threadIdx.x;
  const bool active = i < N;
  const wt_v3 p = active ? cl_load(points + 3 * (size_t)i) : wt_v3{0.0f, 0.0f, 0.0f};
  float best = INFINITY;
  int bf = 0;
  for (int f0 = 0; f0 < F; f0 += kClFaceChunk) {
    const int nf = min(kClFaceChunk, F - f0);
    __syncthreads();
    if (threadIdx.x < nf) {
      const int32_t* f = faces + 3 * (size_t)(f0 + threadIdx.x);
      tri[threadIdx.x] = wt_tri_prep(cl_load(verts + 3 * (size_t)f[0]), cl_load(verts + 3 * (size_t)f[1]),
                                     cl_load(verts + 3 * (size_t)f[2]));
    }
    __syncthreads();
    if (active)
      for (int t = 0; t < nf; t++) {
        const float d = wt_tri_dist(p, tri[t]);
        if (d < best) { best = d; bf = f0 + t; }
      }
  }
  bool used = false;
  if (active) {
    const int32_t* f = faces + 3 * (size_t)bf;
    const wt_tri t = wt_tri_prep(cl_load(verts + 3 * (size_t)f[0]), cl_load(verts + 3 * (size_t)f[1]),
                                 cl_load(verts + 3 * (size_t)f[2]));
    float w[3];
    wt_tri_bary(p, t, w);
    used = best <= r;
    face_out[i] = bf;
    dist_out[i] = best;
    weight_out[3 * (size_t)i] = w[0];
    weight_out[3 * (size_t)i + 1] = w[1];
    weight_out[3 * (size_t)i + 2] = w[2];
  }
  const unsigned mu = __ballot_sync(0xffffffffu, active && used), mb = __ballot_sync(0xffffffffu, active && !used);
  if ((threadIdx.x & 31) == 0) {
    if (mu) atomicAdd(stats, (unsigned long long)__popc(mu));
    if (mb) atomicAdd(stats + 1, (unsigned long long)__popc(mb));
  }
}

// grid-stride over the points; sums [V][4] = (W, C_r, C_g, C_b), in shared memory (dynamic, V x 32 B) with kShared
template <bool kShared>
__global__ void __launch_bounds__(kClAccThreads) colors_accum_kernel(const int32_t* __restrict__ faces,
                                                                 const float* __restrict__ colors, int N, int V,
                                                                 float r, const int32_t* __restrict__ face,
                                                                 const float* __restrict__ dist,
                                                                 const float* __restrict__ weight,
                                                                 unsigned long long* __restrict__ sums) {
  extern __shared__ unsigned long long cl_shared[];
  unsigned long long* acc = kShared ? cl_shared : sums;
  if (kShared) {
    for (int k = threadIdx.x; k < 4 * V; k += kClAccThreads) acc[k] = 0ull;
    __syncthreads();
  }
  for (int i = blockIdx.x * kClAccThreads + threadIdx.x; i < N; i += gridDim.x * kClAccThreads) {
    if (!(dist[i] <= r)) continue;
    const int32_t* f = faces + 3 * (size_t)face[i];
    const float c0 = colors[3 * (size_t)i], c1 = colors[3 * (size_t)i + 1], c2 = colors[3 * (size_t)i + 2];
#pragma unroll
    for (int k = 0; k < 3; k++) {
      const float w = weight[3 * (size_t)i + k];
      unsigned long long* a = acc + 4 * (size_t)f[k];
      atomicAdd(a, cl_fix(w));
      atomicAdd(a + 1, cl_fix(__fmul_rn(w, c0)));
      atomicAdd(a + 2, cl_fix(__fmul_rn(w, c1)));
      atomicAdd(a + 3, cl_fix(__fmul_rn(w, c2)));
    }
  }
  if (kShared) {
    __syncthreads();
    for (int k = threadIdx.x; k < 4 * V; k += kClAccThreads)
      if (acc[k]) atomicAdd(sums + k, acc[k]);
  }
}

// one thread per vertex: list[count++] = v for every vertex with W = 0 (the list's order does not matter: each listed
// vertex gets its own nearest point)
__global__ void colors_list_kernel(const unsigned long long* __restrict__ sums, int V, int32_t* __restrict__ list,
                                   unsigned int* __restrict__ count) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v < V && sums[4 * (size_t)v] == 0ull) list[atomicAdd(count, 1u)] = v;
}

// fixed grid; work item = (tile of kClTile points, group of 256 listed vertices), tile-major; each thread scans the tile
// for its vertex through 1024-point chunks in shared memory and folds its best key into key[v] with one atomicMin
__global__ void __launch_bounds__(kClThreads) colors_nearest_kernel(const float* __restrict__ verts,
                                                                   const float* __restrict__ points, int N,
                                                                   const int32_t* __restrict__ list,
                                                                   const unsigned int* __restrict__ count,
                                                                   unsigned long long* __restrict__ key) {
  __shared__ float4 pts[kClPointChunk];
  const int n_fb = (int)*count;
  if (n_fb == 0) return;
  const int tiles = (N + kClTile - 1) / kClTile, groups = (n_fb + kClThreads - 1) / kClThreads;
  for (long long w = blockIdx.x; w < (long long)tiles * groups; w += gridDim.x) {
    const int tile = (int)(w % tiles), g = (int)(w / tiles);
    const int slot = g * kClThreads + threadIdx.x;
    const bool active = slot < n_fb;
    const int v = active ? list[slot] : 0;
    const wt_v3 x = active ? cl_load(verts + 3 * (size_t)v) : wt_v3{0.0f, 0.0f, 0.0f};
    float best = INFINITY;
    int bj = 0;
    const int j_end = min(N, (tile + 1) * kClTile);
    for (int j0 = tile * kClTile; j0 < j_end; j0 += kClPointChunk) {
      const int nj = min(kClPointChunk, j_end - j0);
      __syncthreads();
      for (int t = threadIdx.x; t < nj; t += kClThreads) {
        const float* y = points + 3 * (size_t)(j0 + t);
        pts[t] = make_float4(y[0], y[1], y[2], 0.0f);
      }
      __syncthreads();
      if (active) {
#pragma unroll 4
        for (int t = 0; t < nj; t++) {
          const float4 y = pts[t];
          const float dx = __fsub_rn(x.x, y.x), dy = __fsub_rn(x.y, y.y), dz = __fsub_rn(x.z, y.z);
          const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
          if (d2 < best) { best = d2; bj = j0 + t; }
        }
      }
    }
    // d^2 >= 0 (or +inf), so its bits order as its values; the index breaks ties toward the lowest
    if (active) atomicMin(key + v, ((unsigned long long)__float_as_uint(best) << 32) | (unsigned)bj);
  }
}

// one thread per vertex: the colour, the fallback flag; stats[2] = listed vertices
__global__ void colors_finish_kernel(const unsigned long long* __restrict__ sums,
                                     const unsigned long long* __restrict__ key, const float* __restrict__ colors,
                                     int V, const unsigned int* __restrict__ count, float* __restrict__ out,
                                     uint8_t* __restrict__ flag_out, unsigned long long* __restrict__ stats) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v == 0) stats[2] = *count;
  if (v >= V) return;
  const unsigned long long* s = sums + 4 * (size_t)v;
  const bool fb = s[0] == 0ull;
  if (fb) {
    const size_t j = (size_t)(key[v] & 0xffffffffull);
#pragma unroll
    for (int ch = 0; ch < 3; ch++) out[3 * (size_t)v + ch] = colors[3 * j + ch];
  } else {
    const double W = (double)s[0];
#pragma unroll
    for (int ch = 0; ch < 3; ch++) out[3 * (size_t)v + ch] = __double2float_rn(__ddiv_rn((double)s[1 + ch], W));
  }
  if (flag_out) flag_out[v] = fb ? 1 : 0;
}

// ---------------------------------------------------------------- workspace

static bool cl_shape_ok(int V, int F, int N) {
  return V >= 1 && V <= kClMaxV && F >= 1 && F <= kClMaxF && N >= 1 && N <= kClMaxN;
}

struct ClBuffers {
  int32_t* face;
  float *dist, *weight;
  unsigned long long *sums, *key;
  int32_t* list;
  unsigned int* count;
  size_t total;
};

static ClBuffers cl_buffers(int V, int N, void* ws) {
  Carver c(ws);
  ClBuffers b;
  b.face = c.take<int32_t>(N);
  b.dist = c.take<float>(N);
  b.weight = c.take<float>(3 * (size_t)N);
  b.sums = c.take<unsigned long long>(4 * (size_t)V);
  b.key = c.take<unsigned long long>(V);
  b.list = c.take<int32_t>(V);
  b.count = c.take<unsigned int>(1);
  b.total = c.total;
  return b;
}

static StageEvents<4> cl_events;

}  // namespace ma

using namespace ma;

extern "C" {

size_t ma_transfer_colors_workspace_bytes(int V, int F, int N) {
  if (!cl_shape_ok(V, F, N)) return 0;
  return cl_buffers(V, N, nullptr).total;
}

void ma_transfer_colors_set_events(void* const* events) { cl_events.set(events); }

int ma_transfer_colors(const float* vertices, int V, const int32_t* faces, int F, const float* points,
                       const float* colors, int N, float r, float* out_colors, int64_t* stats_out, int32_t* point_face,
                       float* point_dist, float* point_weights, uint64_t* sums_out, uint8_t* fallback_out, void* ws,
                       void* stream) {
  if (!vertices || !faces || !points || !colors || !out_colors || !stats_out || !ws || !cl_shape_ok(V, F, N) ||
      !(r > 0.0f && r < INFINITY)) {
    set_error("ma_transfer_colors: bad arguments (1 <= V <= %d, 1 <= F <= %d, 1 <= N <= 2^24, 0 < r finite)", kClMaxV,
              kClMaxF);
    return 1;
  }
  const char* what = "ma_transfer_colors";
  cudaStream_t st = (cudaStream_t)stream;
  ClBuffers b = cl_buffers(V, N, ws);
  if (point_face) b.face = point_face;
  if (point_dist) b.dist = point_dist;
  if (point_weights) b.weight = point_weights;
  if (sums_out) b.sums = reinterpret_cast<unsigned long long*>(sums_out);
  unsigned long long* stats = reinterpret_cast<unsigned long long*>(stats_out);

  cl_events.mark(0, st);
  cudaError_t e = cudaMemsetAsync(stats, 0, 3 * sizeof(int64_t), st);
  if (e == cudaSuccess) e = cudaMemsetAsync(b.sums, 0, 4 * (size_t)V * sizeof(unsigned long long), st);
  if (e == cudaSuccess) e = cudaMemsetAsync(b.key, 0xff, (size_t)V * sizeof(unsigned long long), st);
  if (e == cudaSuccess) e = cudaMemsetAsync(b.count, 0, sizeof(unsigned int), st);
  const bool shared = V <= kClSharedMaxV;
  const size_t smem = shared ? 4 * (size_t)V * sizeof(unsigned long long) : 0;
  if (e == cudaSuccess && shared)
    e = cudaFuncSetAttribute(colors_accum_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return stage_status(what, e);
  colors_assign_kernel<<<blocks(N, kClThreads), kClThreads, 0, st>>>(vertices, faces, F, points, N, r, b.face, b.dist,
                                                                      b.weight, stats);
  cl_events.mark(1, st);
  const int acc_blocks = min(blocks(N, kClAccThreads), sm_count());
  if (shared)
    colors_accum_kernel<true><<<acc_blocks, kClAccThreads, smem, st>>>(faces, colors, N, V, r, b.face, b.dist,
                                                                       b.weight, b.sums);
  else
    colors_accum_kernel<false><<<acc_blocks, kClAccThreads, 0, st>>>(faces, colors, N, V, r, b.face, b.dist,
                                                                     b.weight, b.sums);
  cl_events.mark(2, st);
  colors_list_kernel<<<blocks(V, kClThreads), kClThreads, 0, st>>>(b.sums, V, b.list, b.count);
  colors_nearest_kernel<<<4 * sm_count(), kClThreads, 0, st>>>(vertices, points, N, b.list, b.count, b.key);
  colors_finish_kernel<<<blocks(V, kClThreads), kClThreads, 0, st>>>(b.sums, b.key, colors, V, b.count, out_colors,
                                                                      fallback_out, stats);
  count_launch(5);
  cl_events.mark(3, st);
  return stage_status(what, cudaSuccess);
}

}  // extern "C"
