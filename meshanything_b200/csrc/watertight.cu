// watertight.cu -- watertight remesh of `--mc` on the GPU: narrow-band unsigned distance field + marching cubes.
//
// Replaces mesh2sdf.core.compute + skimage.measure.marching_cubes(|sdf|, 2/size) of the reference's pre-processing
// (/root/reference/mesh_to_pc.py:13-40).
//
// (a) ma_udf_grid: field[i][j][k] = min(band, distance from the grid point (-1 + i dx, -1 + j dx, -1 + k dx), dx = 2/n,
//     to the nearest face).  One CTA per face walks the grid points of the face's bounding box grown by the band, skips
//     the points outside the face's slab, and combines with atomicMin on the fp32 bit pattern (the values are
//     non-negative, so unsigned order is float order).  The distance is one fixed fp32 formula written with explicit
//     round-to-nearest intrinsics (nvcc cannot contract it) and a minimum does not depend on order, so the field is
//     bit-deterministic and restated bit for bit by tests/watertight_oracle.py.  Culling is conservative: a
//     (point, face) pair is skipped only when its distance exceeds the band by a margin far above fp32 rounding.
// (b) ma_marching_cubes_count / _emit: cells in linear order, triangles from the generated table of mc_table.h, one
//     vertex per crossed grid edge (owned by the edge's lower grid point, shared by every face that uses it) at
//     a + t (b - a), t = (level - f_a) / (f_b - f_a), in index space.  Classify -> CUB exclusive scan of packed
//     (triangles << 32 | vertices) counts -> one 8-byte read-back -> emit.
#include <cub/device/device_scan.cuh>

#include "canon.cuh"
#include "mc_table.h"
#include "tri_dist.cuh"
#include "workspace.h"

namespace ma {

// ---------------------------------------------------------------- (a) distance field (wt_tri_dist: tri_dist.cuh)

__global__ void udf_fill_kernel(float* __restrict__ field, size_t count, float band) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < count; i += (size_t)gridDim.x * blockDim.x)
    field[i] = band;
}

// grid index range [lo, hi] of the points with coordinate in [x0, x1] (one index of slack on each side)
__device__ __forceinline__ void udf_range(float x0, float x1, float dx, int n, int* lo, int* hi) {
  const float a = fminf(fmaxf((x0 + 1.0f) / dx, -1.0f), (float)n), b = fminf(fmaxf((x1 + 1.0f) / dx, -1.0f), (float)n);
  *lo = max(0, (int)floorf(a) - 1);
  *hi = min(n - 1, (int)ceilf(b) + 1);
}

__global__ void __launch_bounds__(128) udf_face_kernel(const float* __restrict__ v, const int32_t* __restrict__ faces,
                                                       int n, float band, float* __restrict__ field) {
  const int f = blockIdx.x;
  const int32_t* fi = faces + 3 * (size_t)f;
  const wt_v3 a = {v[3 * (size_t)fi[0]], v[3 * (size_t)fi[0] + 1], v[3 * (size_t)fi[0] + 2]};
  const wt_v3 b = {v[3 * (size_t)fi[1]], v[3 * (size_t)fi[1] + 1], v[3 * (size_t)fi[1] + 2]};
  const wt_v3 c = {v[3 * (size_t)fi[2]], v[3 * (size_t)fi[2] + 1], v[3 * (size_t)fi[2] + 2]};
  const float dx = __fdiv_rn(2.0f, (float)n);
  // culling margin: far above the rounding of the fp32 distance formula for coordinates of this size
  const float scale = fmaxf(1.0f, fmaxf(fmaxf(fmaxf(fabsf(a.x), fabsf(a.y)), fmaxf(fabsf(a.z), fabsf(b.x))),
                                        fmaxf(fmaxf(fabsf(b.y), fabsf(b.z)), fmaxf(fmaxf(fabsf(c.x), fabsf(c.y)), fabsf(c.z)))));
  const float reach = band * 1.001f + 1e-5f * scale;
  int i0, i1, j0, j1, k0, k1;
  udf_range(fminf(fminf(a.x, b.x), c.x) - reach, fmaxf(fmaxf(a.x, b.x), c.x) + reach, dx, n, &i0, &i1);
  udf_range(fminf(fminf(a.y, b.y), c.y) - reach, fmaxf(fmaxf(a.y, b.y), c.y) + reach, dx, n, &j0, &j1);
  udf_range(fminf(fminf(a.z, b.z), c.z) - reach, fmaxf(fmaxf(a.z, b.z), c.z) + reach, dx, n, &k0, &k1);
  if (i0 > i1 || j0 > j1 || k0 > k1) return;
  const int nj = j1 - j0 + 1, nk = k1 - k0 + 1;
  const long long total = (long long)(i1 - i0 + 1) * nj * nk;
  // slab of the face's plane: |(p - a).n| > reach |n| -> farther than the band.  The normal is taken in double (fp32
  // products are exact there), so that a sliver's normal still points the right way; zero normal -> no slab test.
  const double ux = (double)b.x - a.x, uy = (double)b.y - a.y, uz = (double)b.z - a.z;
  const double wx = (double)c.x - a.x, wy = (double)c.y - a.y, wz = (double)c.z - a.z;
  const double nx = uy * wz - uz * wy, ny = uz * wx - ux * wz, nz = ux * wy - uy * wx;
  const double slab = reach * sqrt(nx * nx + ny * ny + nz * nz);
  for (long long t = threadIdx.x; t < total; t += blockDim.x) {
    const int k = k0 + (int)(t % nk), j = j0 + (int)((t / nk) % nj), i = i0 + (int)(t / ((long long)nk * nj));
    const wt_v3 p = {__fadd_rn(-1.0f, __fmul_rn((float)i, dx)), __fadd_rn(-1.0f, __fmul_rn((float)j, dx)),
                     __fadd_rn(-1.0f, __fmul_rn((float)k, dx))};
    if (slab > 0.0 && fabs(((double)p.x - a.x) * nx + ((double)p.y - a.y) * ny + ((double)p.z - a.z) * nz) > slab) continue;
    const float d = wt_tri_dist(p, a, b, c);
    if (d < band) atomicMin(reinterpret_cast<unsigned int*>(field) + ((size_t)i * n + j) * n + k, __float_as_uint(d));
  }
}

// ---------------------------------------------------------------- (b) marching cubes

// info[p] = (case << 3) | crossed-edge mask of the grid point's +x/+y/+z edges; cnt[p] = triangles << 32 | vertices
__global__ void mc_classify_kernel(const float* __restrict__ field, int n, float level, uint16_t* __restrict__ info,
                                   unsigned long long* __restrict__ cnt) {
  const size_t N = (size_t)n * n * n;
  for (size_t p = blockIdx.x * (size_t)blockDim.x + threadIdx.x; p < N; p += (size_t)gridDim.x * blockDim.x) {
    const int k = (int)(p % n), j = (int)((p / n) % n), i = (int)(p / ((size_t)n * n));
    const size_t sx = (size_t)n * n, sy = n;
    const bool in0 = field[p] < level;
    unsigned mask = 0;
    if (i < n - 1 && (field[p + sx] < level) != in0) mask |= 1u;
    if (j < n - 1 && (field[p + sy] < level) != in0) mask |= 2u;
    if (k < n - 1 && (field[p + 1] < level) != in0) mask |= 4u;
    unsigned cs = 0, tris = 0;
    if (i < n - 1 && j < n - 1 && k < n - 1) {
#pragma unroll
      for (int c = 0; c < 8; c++)
        if (field[p + (c & 1) * sx + ((c >> 1) & 1) * sy + ((c >> 2) & 1)] < level) cs |= 1u << c;
      tris = kMcTriCount[cs];
    }
    info[p] = (uint16_t)((cs << 3) | mask);
    cnt[p] = ((unsigned long long)tris << 32) | (unsigned long long)__popc(mask);
  }
}

__global__ void mc_emit_kernel(const float* __restrict__ field, int n, float level, const uint16_t* __restrict__ info,
                               const unsigned long long* __restrict__ off, float* __restrict__ out_v,
                               int32_t* __restrict__ out_f) {
  const size_t N = (size_t)n * n * n;
  const size_t sx = (size_t)n * n, sy = n;
  for (size_t p = blockIdx.x * (size_t)blockDim.x + threadIdx.x; p < N; p += (size_t)gridDim.x * blockDim.x) {
    const unsigned inf = info[p];
    const unsigned mask = inf & 7u, cs = inf >> 3;
    if (mask == 0 && cs == 0) continue;
    const int k = (int)(p % n), j = (int)((p / n) % n), i = (int)(p / sx);
    const unsigned long long base = off[p];
    unsigned vid = (unsigned)base;
    const float fa = field[p];
#pragma unroll
    for (int axis = 0; axis < 3; axis++) {
      if (!(mask >> axis & 1u)) continue;
      const float fb = field[p + (axis == 0 ? sx : axis == 1 ? sy : 1)];
      const float t = __fdiv_rn(__fsub_rn(level, fa), __fsub_rn(fb, fa));
      float x = (float)i, y = (float)j, z = (float)k;
      if (axis == 0) x = __fadd_rn(x, t); else if (axis == 1) y = __fadd_rn(y, t); else z = __fadd_rn(z, t);
      out_v[3 * (size_t)vid] = x; out_v[3 * (size_t)vid + 1] = y; out_v[3 * (size_t)vid + 2] = z;
      vid++;
    }
    const unsigned nt = kMcTriCount[cs];
    const unsigned tbase = (unsigned)(base >> 32);
    for (unsigned t = 0; t < nt; t++) {
#pragma unroll
      for (int s = 0; s < 3; s++) {
        const int e = kMcTris[cs][3 * t + s], axis = e >> 2, m = e & 3;
        // lower corner of edge e (mc_table.py: the two other axes, lower axis first, take the bits of m)
        const int c0 = axis == 0 ? (m << 1) : axis == 1 ? ((m & 1) | ((m >> 1) << 2)) : m;
        const size_t q = p + (c0 & 1) * sx + ((c0 >> 1) & 1) * sy + ((c0 >> 2) & 1);
        out_f[3 * ((size_t)tbase + t) + s] = (int32_t)((unsigned)off[q] + __popc(info[q] & 7u & ((1u << axis) - 1u)));
      }
    }
  }
}

static size_t mc_scan_bytes(int n) {
  size_t bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, bytes, (unsigned long long*)nullptr, (int)((size_t)n * n * n));
  return bytes;
}

static int grid_blocks(size_t count) { return (int)std::min<size_t>((count + 255) / 256, (size_t)132 * 32); }

}  // namespace ma

using namespace ma;

extern "C" {

int ma_udf_grid(const float* vertices, const int32_t* faces, int n_faces, int n, float band, float* out_field,
                void* stream) {
  if (!vertices || !faces || !out_field || n_faces < 0 || n < 2 || n > 1024 || !(band > 0.0f) || !isfinite(band)) {
    set_error("ma_udf_grid: bad arguments");
    return 1;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const size_t N = (size_t)n * n * n;
  udf_fill_kernel<<<grid_blocks(N), 256, 0, st>>>(out_field, N, band);
  count_launch();
  if (n_faces > 0) {
    udf_face_kernel<<<n_faces, 128, 0, st>>>(vertices, faces, n, band, out_field);
    count_launch();
  }
  return check_launch("ma_udf_grid") ? 0 : 1;
}

size_t ma_marching_cubes_workspace_bytes(int n) {
  if (n < 2 || n > 1024) return 0;
  const size_t N = (size_t)n * n * n;
  return ws_align(N * sizeof(unsigned long long)) + ws_align(N * sizeof(uint16_t)) + ws_align(mc_scan_bytes(n));
}

int ma_marching_cubes_count(const float* field, int n, float level, void* ws, int64_t* counts_host, void* stream) {
  if (!field || !ws || !counts_host || n < 2 || n > 1024 || !isfinite(level)) {
    set_error("ma_marching_cubes_count: bad arguments");
    return 1;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const size_t N = (size_t)n * n * n;
  char* w = reinterpret_cast<char*>(ws);
  auto* cnt = reinterpret_cast<unsigned long long*>(w);
  auto* info = reinterpret_cast<uint16_t*>(w + ws_align(N * sizeof(unsigned long long)));
  void* tmp = w + ws_align(N * sizeof(unsigned long long)) + ws_align(N * sizeof(uint16_t));
  size_t tmp_bytes = mc_scan_bytes(n);
  mc_classify_kernel<<<grid_blocks(N), 256, 0, st>>>(field, n, level, info, cnt);
  count_launch();
  if (!check_launch("ma_marching_cubes_count")) return 1;
  cudaError_t e = cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, cnt, (int)N, st);
  count_launch();
  // the last grid point owns no edge and is no cell: its exclusive prefix is the total
  unsigned long long total = 0;
  if (e == cudaSuccess) e = cudaMemcpyAsync(&total, cnt + (N - 1), sizeof(total), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (e != cudaSuccess) {
    set_error("ma_marching_cubes_count: %s", cudaGetErrorString(e));
    cudaGetLastError();
    return 1;
  }
  const unsigned long long nv = total & 0xffffffffull, nt = total >> 32;
  if (nv > 0x7fffffffull || nt > 0x7fffffffull) {
    set_error("ma_marching_cubes_count: %llu vertices / %llu triangles exceed int32 indexing", nv, nt);
    return 1;
  }
  counts_host[0] = (int64_t)nv;
  counts_host[1] = (int64_t)nt;
  return 0;
}

int ma_marching_cubes_emit(const float* field, int n, float level, const void* ws, float* out_vertices,
                           int32_t* out_faces, void* stream) {
  if (!field || !ws || n < 2 || n > 1024 || !isfinite(level)) {
    set_error("ma_marching_cubes_emit: bad arguments");
    return 1;
  }
  const size_t N = (size_t)n * n * n;
  const char* w = reinterpret_cast<const char*>(ws);
  const auto* off = reinterpret_cast<const unsigned long long*>(w);
  const auto* info = reinterpret_cast<const uint16_t*>(w + ws_align(N * sizeof(unsigned long long)));
  mc_emit_kernel<<<grid_blocks(N), 256, 0, (cudaStream_t)stream>>>(field, n, level, info, off, out_vertices, out_faces);
  count_launch();
  return check_launch("ma_marching_cubes_emit") ? 0 : 1;
}

}  // extern "C"
