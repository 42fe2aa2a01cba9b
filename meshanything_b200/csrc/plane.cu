// plane.cu -- removal of the dominant plane of a point cloud (the table, turntable or floor a scanned object stands
// on) by RANSAC and a least-squares refit (DESIGN.md section 1.6 defines it).
//
// The points arrive already in the output frame (p' = (p - c) / L, metrics.to_output_frame), fp32 [N][3].
//   (a) hypotheses  one thread per hypothesis h: three indices from Philox4x32-10 (philox.cuh) with the stream tag
//                   "PLAN", the fp32 plane through them as float4 (n, d); an invalid hypothesis (a zero or non-finite
//                   cross product) is stored as (0, 0, 0, +inf), which no point is on.
//   (b) scoring     the hot path: every thread holds kPlPerThread planes in registers, the CTA streams the points
//                   through shared memory in stages of kPlPoints; per (point, plane) pair 3 FMUL + 3 FADD and |s| <= t,
//                   counted in a register; one integer atomicAdd per (CTA, plane) into counts[H].  The winner is the
//                   atomicMax of count << 32 | ~h (largest count, lowest h on ties).
//   (c) refit       the winner's on-plane points: centroid, then the six centred second moments, each an fp64 sum
//                   over tiles of 256 consecutive indices (off-plane points add +0) summed in index order by one CTA
//                   per tile, the tile partials in tile order; one thread runs the Jacobi of jacobi3.cuh.
//   (d) classify    every point against the refit plane: on / above / below, counted by warp-aggregated integer
//                   atomics; the plane flips when below > above; the kept (above) indices by CUB DeviceSelect::Flagged.
// No host synchronisation and no floating-point atomics: every kernel reads the winner from device memory, and a
// winning count below 3 (no plane) makes the refit a no-op and keeps every point.  Every fp32 / fp64 step is an
// explicit round-to-nearest intrinsic, so tests/plane_oracle.py restates planes, counts, the refit, the mask and the
// stats bit for bit.
#include <algorithm>
#include <cmath>

#include <cub/device/device_select.cuh>
#include <cub/iterator/counting_input_iterator.cuh>

#include "jacobi3.cuh"
#include "philox.cuh"
#include "workspace.h"

namespace ma {

constexpr int kPlThreads = 256;
constexpr int kPlPerThread = 4;                         // planes in each scoring thread's registers
constexpr int kPlPlanes = kPlThreads * kPlPerThread;    // planes per scoring CTA
constexpr int kPlPoints = 1024;                         // points per shared-memory stage of the scoring kernel
constexpr int kPlTile = 256;                            // indices per tile of the fixed-order fp64 sums
constexpr int kPlMaxN = 1 << 24;
constexpr int kPlMaxH = 65536;
constexpr uint32_t kPlTag0 = 0x504c414eu, kPlTag1 = 0x4d455348u, kPlTag2 = 0x414e5954u;  // "PLAN", "MESH", "ANYT"

// s(p) = ((nx px + ny py) + nz pz) + d, nothing contracted
__device__ __forceinline__ float pl_dist(float4 pl, float px, float py, float pz) {
  return __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(pl.x, px), __fmul_rn(pl.y, py)), __fmul_rn(pl.z, pz)), pl.w);
}

// the winner packed as count << 32 | ~h; a count below 3 means no plane
__device__ __forceinline__ bool pl_found(unsigned long long best) { return (best >> 32) >= 3ull; }

// small counters, zeroed together: best, valid hypotheses, on / above / below
struct PlCounters {
  unsigned long long best;
  int valid;
  int cls[3];
};

// ---------------------------------------------------------------- (a) hypotheses

__global__ void plane_hypothesis_kernel(const float* __restrict__ xyz, int n, int H, unsigned long long seed,
                                        float4* __restrict__ planes, PlCounters* __restrict__ ctr) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  bool ok = false;
  if (h < H) {
    const uint4 r = philox4x32_10((uint32_t)h, kPlTag0, kPlTag1, kPlTag2, seed);
    const uint32_t i0 = (uint32_t)(((unsigned long long)r.x * (uint32_t)n) >> 32);
    const uint32_t i1 = (uint32_t)(((unsigned long long)r.y * (uint32_t)n) >> 32);
    const uint32_t i2 = (uint32_t)(((unsigned long long)r.z * (uint32_t)n) >> 32);
    const float* a = xyz + 3 * (size_t)i0;
    const float* b = xyz + 3 * (size_t)i1;
    const float* c = xyz + 3 * (size_t)i2;
    const float ax = a[0], ay = a[1], az = a[2];
    const float ux = __fsub_rn(b[0], ax), uy = __fsub_rn(b[1], ay), uz = __fsub_rn(b[2], az);
    const float wx = __fsub_rn(c[0], ax), wy = __fsub_rn(c[1], ay), wz = __fsub_rn(c[2], az);
    const float mx = __fsub_rn(__fmul_rn(uy, wz), __fmul_rn(uz, wy));
    const float my = __fsub_rn(__fmul_rn(uz, wx), __fmul_rn(ux, wz));
    const float mz = __fsub_rn(__fmul_rn(ux, wy), __fmul_rn(uy, wx));
    const float l = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(mx, mx), __fmul_rn(my, my)), __fmul_rn(mz, mz)));
    float4 pl = make_float4(0.0f, 0.0f, 0.0f, INFINITY);
    if (l > 0.0f && l < INFINITY) {
      pl.x = __fdiv_rn(mx, l);
      pl.y = __fdiv_rn(my, l);
      pl.z = __fdiv_rn(mz, l);
      pl.w = -__fadd_rn(__fadd_rn(__fmul_rn(pl.x, ax), __fmul_rn(pl.y, ay)), __fmul_rn(pl.z, az));
      ok = true;
    }
    planes[h] = pl;
  }
  const unsigned votes = __ballot_sync(0xffffffffu, ok);
  if ((threadIdx.x & 31) == 0 && votes) atomicAdd(&ctr->valid, __popc(votes));
}

// ---------------------------------------------------------------- (b) scoring

// grid (point slices, ceil(H / kPlPlanes)); thread x of plane group y owns planes y kPlPlanes + x + q kPlThreads
__global__ void __launch_bounds__(kPlThreads) plane_score_kernel(const float* __restrict__ xyz, int n, int H, float t,
                                                                 const float4* __restrict__ planes,
                                                                 int* __restrict__ counts) {
  __shared__ float4 sp[kPlPoints];
  const int h0 = blockIdx.y * kPlPlanes + threadIdx.x;
  float4 pl[kPlPerThread];
  int cnt[kPlPerThread];
#pragma unroll
  for (int q = 0; q < kPlPerThread; q++) {
    const int h = h0 + q * kPlThreads;
    pl[q] = h < H ? planes[h] : make_float4(0.0f, 0.0f, 0.0f, INFINITY);
    cnt[q] = 0;
  }
  for (int base = blockIdx.x * kPlPoints; base < n; base += gridDim.x * kPlPoints) {
    const int m = min(kPlPoints, n - base);
    __syncthreads();
    for (int j = threadIdx.x; j < m; j += kPlThreads) {
      const float* p = xyz + 3 * (size_t)(base + j);
      sp[j] = make_float4(p[0], p[1], p[2], 0.0f);
    }
    __syncthreads();
#pragma unroll 4
    for (int j = 0; j < m; j++) {
      const float4 p = sp[j];
#pragma unroll
      for (int q = 0; q < kPlPerThread; q++) cnt[q] += fabsf(pl_dist(pl[q], p.x, p.y, p.z)) <= t ? 1 : 0;
    }
  }
#pragma unroll
  for (int q = 0; q < kPlPerThread; q++) {
    const int h = h0 + q * kPlThreads;
    if (h < H && cnt[q]) atomicAdd(counts + h, cnt[q]);
  }
}

// best = max over h of count << 32 | ~h: the warp's maximum (high word, then low word), one atomicMax per warp
__global__ void plane_winner_kernel(const int* __restrict__ counts, int H, PlCounters* __restrict__ ctr) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t hi = h < H ? (uint32_t)counts[h] : 0u, lo = h < H ? ~(uint32_t)h : 0u;
  const uint32_t whi = __reduce_max_sync(0xffffffffu, hi);
  const uint32_t wlo = __reduce_max_sync(0xffffffffu, hi == whi ? lo : 0u);
  if ((threadIdx.x & 31) == 0) atomicMax(&ctr->best, ((unsigned long long)whi << 32) | wlo);
}

// ---------------------------------------------------------------- (c) refit

// one CTA per tile of kPlTile indices: pass 0 the winner's on-plane x, y, z; pass 1 the six centred products
// (xx, xy, xz, yy, yz, zz) about cent; off-plane points give +0.  part[tile][a] = the tile's sum of term a in index order.
__global__ void __launch_bounds__(kPlTile) plane_tile_kernel(const float* __restrict__ xyz, int n, float t,
                                                             const float4* __restrict__ planes,
                                                             const PlCounters* __restrict__ ctr,
                                                             const double* __restrict__ cent, int pass,
                                                             double* __restrict__ part) {
  __shared__ double v[6][kPlTile + 1];
  const unsigned long long best = ctr->best;
  if (!pl_found(best)) return;
  const float4 pl = planes[~(uint32_t)best];
  const int i = blockIdx.x * kPlTile + threadIdx.x;
  double y[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  if (i < n) {
    const float* p = xyz + 3 * (size_t)i;
    if (fabsf(pl_dist(pl, p[0], p[1], p[2])) <= t) {
      if (pass == 0) {
        y[0] = p[0], y[1] = p[1], y[2] = p[2];
      } else {
        const double dx = __dsub_rn((double)p[0], cent[0]), dy = __dsub_rn((double)p[1], cent[1]);
        const double dz = __dsub_rn((double)p[2], cent[2]);
        y[0] = __dmul_rn(dx, dx), y[1] = __dmul_rn(dx, dy), y[2] = __dmul_rn(dx, dz);
        y[3] = __dmul_rn(dy, dy), y[4] = __dmul_rn(dy, dz), y[5] = __dmul_rn(dz, dz);
      }
    }
  }
#pragma unroll
  for (int a = 0; a < 6; a++) v[a][threadIdx.x] = y[a];
  __syncthreads();
  const int a = threadIdx.x;
  if (a < (pass == 0 ? 3 : 6)) {
    const int m = min(kPlTile, n - blockIdx.x * kPlTile);
    double s = 0.0;
    for (int k = 0; k < m; k++) s = __dadd_rn(s, v[a][k]);
    part[(size_t)blockIdx.x * 6 + a] = s;
  }
}

// the tile partials in tile order (thread a sums term a).  pass 0: cent = sums / count; pass 1: the moments, then the
// Jacobi by thread 0 and the refit plane fit = (n, d), n the fp32 rounding of the fp64 unit eigenvector n64 of the
// smallest eigenvalue, d = fp32(-((n64x cx + n64y cy) + n64z cz))
__global__ void plane_reduce_kernel(const double* __restrict__ part, int tiles, const PlCounters* __restrict__ ctr,
                                    int pass, double* __restrict__ cent, float4* __restrict__ fit) {
  __shared__ double c[6];
  const unsigned long long best = ctr->best;
  if (!pl_found(best)) {
    if (pass == 1 && threadIdx.x == 0) *fit = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    return;
  }
  const int a = threadIdx.x;
  if (a < (pass == 0 ? 3 : 6)) {
    double s = 0.0;
    for (int tl = 0; tl < tiles; tl++) s = __dadd_rn(s, part[(size_t)tl * 6 + a]);
    if (pass == 0) cent[a] = __ddiv_rn(s, (double)(best >> 32));
    else c[a] = s;
  }
  if (pass == 0) return;
  __syncthreads();
  if (threadIdx.x != 0) return;
  double n64[3];
  jacobi3_smallest(c, n64);
  const double d = -__dadd_rn(__dadd_rn(__dmul_rn(n64[0], cent[0]), __dmul_rn(n64[1], cent[1])),
                              __dmul_rn(n64[2], cent[2]));
  *fit = make_float4((float)n64[0], (float)n64[1], (float)n64[2], (float)d);
}

// ---------------------------------------------------------------- (d) classification

// cls[i] = 0 on (|s| <= t), 1 above (s > t), 2 below (s < -t) under the refit plane; 1 for every point when there
// is no plane.  ctr->cls[] += the counts (one atomic per warp and class)
__global__ void plane_classify_kernel(const float* __restrict__ xyz, int n, float t, const float4* __restrict__ fit,
                                      PlCounters* __restrict__ ctr, uint8_t* __restrict__ cls) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool found = pl_found(ctr->best);
  int k = -1;
  if (i < n) {
    k = 1;
    if (found) {
      const float* p = xyz + 3 * (size_t)i;
      const float s = pl_dist(*fit, p[0], p[1], p[2]);
      k = fabsf(s) <= t ? 0 : (s > t ? 1 : 2);
    }
    cls[i] = (uint8_t)k;
  }
  if (!found) return;
#pragma unroll
  for (int c = 0; c < 3; c++) {
    const unsigned votes = __ballot_sync(0xffffffffu, k == c);
    if ((threadIdx.x & 31) == 0 && votes) atomicAdd(ctr->cls + c, __popc(votes));
  }
}

// the flip rule: when below > above, the plane turns over and the below points become the kept side
__global__ void plane_keep_kernel(int n, const PlCounters* __restrict__ ctr, const uint8_t* __restrict__ cls,
                                  uint8_t* __restrict__ keep) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t side = ctr->cls[2] > ctr->cls[1] ? 2 : 1;
  keep[i] = cls[i] == side ? 1 : 0;
}

// stats = (found, nx, ny, nz, d, winning hypothesis, its count, valid hypotheses, on, above, below, kept), the plane
// and the counts after the flip
__global__ void plane_finish_kernel(const PlCounters* __restrict__ ctr, const float4* __restrict__ fit,
                                    const int64_t* __restrict__ n_kept, double* __restrict__ stats) {
  if (threadIdx.x != 0) return;
  const unsigned long long best = ctr->best;
  const bool flip = ctr->cls[2] > ctr->cls[1];
  float4 pl = *fit;
  if (flip) pl = make_float4(-pl.x, -pl.y, -pl.z, -pl.w);
  stats[0] = pl_found(best) ? 1.0 : 0.0;
  stats[1] = (double)pl.x;
  stats[2] = (double)pl.y;
  stats[3] = (double)pl.z;
  stats[4] = (double)pl.w;
  stats[5] = (double)(uint32_t)~(uint32_t)best;
  stats[6] = (double)(best >> 32);
  stats[7] = (double)ctr->valid;
  stats[8] = (double)ctr->cls[0];
  stats[9] = (double)(flip ? ctr->cls[2] : ctr->cls[1]);
  stats[10] = (double)(flip ? ctr->cls[1] : ctr->cls[2]);
  stats[11] = (double)*n_kept;
}

// ---------------------------------------------------------------- workspace

static bool pl_shape_ok(int n, int h) { return n >= 3 && n <= kPlMaxN && h >= 1 && h <= kPlMaxH; }
static int pl_tiles(int n) { return (n + kPlTile - 1) / kPlTile; }

static size_t pl_flag_bytes(int n) {
  size_t bytes = 0;
  cub::DeviceSelect::Flagged(nullptr, bytes, cub::CountingInputIterator<int64_t>(0), (uint8_t*)nullptr,
                             (int64_t*)nullptr, (int64_t*)nullptr, n);
  return bytes;
}

struct PlBuffers {
  float4* planes;
  int* counts;
  PlCounters* ctr;
  uint8_t* cls;
  double *part, *cent;
  float4* fit;
  void* cub;
  size_t cub_bytes, total;
};

static PlBuffers pl_buffers(int n, int h, void* ws) {
  Carver c(ws);
  PlBuffers b;
  b.planes = c.take<float4>(h);
  b.counts = c.take<int>(h);
  b.ctr = c.take<PlCounters>(1);
  b.cls = c.take<uint8_t>(n);
  b.part = c.take<double>((size_t)pl_tiles(n) * 6);
  b.cent = c.take<double>(3);
  b.fit = c.take<float4>(1);
  b.cub_bytes = pl_flag_bytes(n);
  b.cub = c.take<char>(b.cub_bytes);
  b.total = c.total;
  return b;
}

static StageEvents<5> pl_events;

// point slices of the scoring grid: about four CTAs per SM over all plane groups, at most one per stage of points
static int pl_score_slices(int n, int groups) {
  const int stages = (n + kPlPoints - 1) / kPlPoints;
  return std::max(1, std::min(stages, (4 * sm_count() + groups - 1) / groups));
}

}  // namespace ma

using namespace ma;

extern "C" {

size_t ma_remove_plane_workspace_bytes(int n, int h) {
  if (!pl_shape_ok(n, h)) return 0;
  return pl_buffers(n, h, nullptr).total;
}

void ma_remove_plane_set_events(void* const* events) { pl_events.set(events); }

int ma_remove_plane(const float* xyz, int n, int h, float t, unsigned long long seed, uint8_t* keep_out,
                    int64_t* kept_idx_out, int64_t* n_kept_out, int32_t* counts_out, float* planes_out,
                    double* stats_out, void* ws, void* stream) {
  if (!xyz || !keep_out || !kept_idx_out || !n_kept_out || !stats_out || !ws || !pl_shape_ok(n, h) ||
      !(t > 0.0f && t <= 1.0f)) {
    set_error("ma_remove_plane: bad arguments (3 <= n <= 2^24, 1 <= h <= %d, 0 < t <= 1)", kPlMaxH);
    return 1;
  }
  cudaStream_t st = (cudaStream_t)stream;
  PlBuffers b = pl_buffers(n, h, ws);
  if (planes_out) b.planes = reinterpret_cast<float4*>(planes_out);
  if (counts_out) b.counts = counts_out;
  const int tiles = pl_tiles(n), groups = (h + kPlPlanes - 1) / kPlPlanes;

  pl_events.mark(0, st);
  cudaError_t e = cudaMemsetAsync(b.ctr, 0, sizeof(PlCounters), st);
  if (e == cudaSuccess) e = cudaMemsetAsync(b.counts, 0, (size_t)h * 4, st);
  plane_hypothesis_kernel<<<blocks(h, kPlThreads), kPlThreads, 0, st>>>(xyz, n, h, seed, b.planes, b.ctr);
  count_launch(1);
  pl_events.mark(1, st);
  plane_score_kernel<<<dim3(pl_score_slices(n, groups), groups), kPlThreads, 0, st>>>(xyz, n, h, t, b.planes,
                                                                                        b.counts);
  plane_winner_kernel<<<blocks(h, kPlThreads), kPlThreads, 0, st>>>(b.counts, h, b.ctr);
  count_launch(2);
  pl_events.mark(2, st);
  plane_tile_kernel<<<tiles, kPlTile, 0, st>>>(xyz, n, t, b.planes, b.ctr, b.cent, 0, b.part);
  plane_reduce_kernel<<<1, 32, 0, st>>>(b.part, tiles, b.ctr, 0, b.cent, b.fit);
  plane_tile_kernel<<<tiles, kPlTile, 0, st>>>(xyz, n, t, b.planes, b.ctr, b.cent, 1, b.part);
  plane_reduce_kernel<<<1, 32, 0, st>>>(b.part, tiles, b.ctr, 1, b.cent, b.fit);
  count_launch(4);
  pl_events.mark(3, st);
  plane_classify_kernel<<<blocks(n, kPlThreads), kPlThreads, 0, st>>>(xyz, n, t, b.fit, b.ctr, b.cls);
  plane_keep_kernel<<<blocks(n, kPlThreads), kPlThreads, 0, st>>>(n, b.ctr, b.cls, keep_out);
  if (e == cudaSuccess)
    e = cub::DeviceSelect::Flagged(b.cub, b.cub_bytes, cub::CountingInputIterator<int64_t>(0), keep_out, kept_idx_out,
                                   n_kept_out, n, st);
  plane_finish_kernel<<<1, 32, 0, st>>>(b.ctr, b.fit, n_kept_out, stats_out);
  count_launch(3);
  pl_events.mark(4, st);
  return stage_status("ma_remove_plane", e);
}

}  // extern "C"
