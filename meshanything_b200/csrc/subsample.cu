// subsample.cu -- farthest-point subsampling of a point cloud (DESIGN.md section 1.4 defines it).
//
// The points arrive already in the output frame (metrics.to_output_frame), fp32 [N][3].  Every point carries D_i, the
// least fp32 d^2 = (dx dx + dy dy) + dz dz to the picks so far; pick t + 1 is the unpicked point of largest D_i, lowest
// index on ties.  One kernel runs every pick:
//   per pick   each thread reads the previous winner's coordinates, lowers the D of its points, and keeps the largest
//              key D_bits << 32 | ~i over its unpicked points (a picked point stores D = -1 and gets key 0; D >= +0
//              otherwise, so the bits order like the values, and N <= 2^24 keeps ~i, hence every real key, above 0);
//              warp and CTA maxima by __reduce_max_sync on the high then the low word.
//   one CTA    (N <= kFpsSmallN) the whole cloud in shared memory (SoA x | y | z | D); the CTA maximum is the winner.
//   grid       cooperative launch, one contiguous slice of the points per CTA, each CTA's maximum atomicMax-ed into a
//              fresh per-pick slot of zeroed workspace, then grid.sync(); the slot holds the winner.  The slices live in
//              shared memory when they fit (kFpsGridShared, up to ~1.8M points on 132 SMs), in global memory (SoA in the
//              workspace, L2-resident up to tens of MB) otherwise.
// The keys are unique, so the winner, and r2[t] = the high word of the maximum (the largest D; 0 once every point is
// picked), do not depend on the schedule: a call is bit-deterministic without floating-point atomics, and
// tests/subsample_oracle.py restates it bit for bit.
#include <cooperative_groups.h>

#include <algorithm>
#include <cmath>

#include "workspace.h"

namespace cg = cooperative_groups;

namespace ma {

constexpr int kFpsThreads = 1024;
constexpr int kFpsMaxN = 1 << 24;  // ~i of every index stays above 0 in the low word of a key
constexpr int kFpsSmallN = 8192;   // up to this many points: one CTA, no grid barrier

enum { kFpsAuto = 0, kFpsOneCta = 1, kFpsGridShared = 2, kFpsGridGlobal = 3 };

__device__ __forceinline__ float fps_d2(float x, float y, float z, float qx, float qy, float qz) {
  const float dx = __fsub_rn(x, qx), dy = __fsub_rn(y, qy), dz = __fsub_rn(z, qz);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

__device__ __forceinline__ unsigned long long fps_key(float d, int i) {
  return d < 0.0f ? 0ull : ((unsigned long long)__float_as_uint(d) << 32) | (uint32_t)~(uint32_t)i;
}

// maximum of a 64-bit key over the warp: the high words, then the low words of the lanes holding the largest high word
__device__ __forceinline__ unsigned long long fps_warp_max(unsigned long long k) {
  const uint32_t hi = (uint32_t)(k >> 32);
  const uint32_t top = __reduce_max_sync(0xffffffffu, hi);
  const uint32_t lo = __reduce_max_sync(0xffffffffu, hi == top ? (uint32_t)k : 0u);
  return ((unsigned long long)top << 32) | lo;
}

// kGrid: cooperative launch, slices of `slice` points per CTA, winners through slots[t]; otherwise one CTA.
// kShared: the slice in dynamic shared memory (4 slice floats); otherwise in soa = x[n] | y[n] | z[n] | D[n].
template <bool kGrid, bool kShared>
__global__ void __launch_bounds__(kFpsThreads, 1)
    fps_kernel(const float* __restrict__ xyz, int n, int m, int start, int slice, float* __restrict__ soa,
               unsigned long long* __restrict__ slots, int64_t* __restrict__ idx_out, float* __restrict__ r2_out) {
  extern __shared__ float fps_smem[];
  __shared__ unsigned long long red[kFpsThreads / 32];
  __shared__ unsigned long long bcast;
  const int lo = blockIdx.x * slice, cnt = max(min(n - lo, slice), 0);
  float* px = kShared ? fps_smem : soa + lo;
  float* py = kShared ? fps_smem + slice : soa + (size_t)n + lo;
  float* pz = kShared ? fps_smem + 2 * (size_t)slice : soa + 2 * (size_t)n + lo;
  float* pd = kShared ? fps_smem + 3 * (size_t)slice : soa + 3 * (size_t)n + lo;
  // every thread touches only its own points (j = threadIdx.x mod kFpsThreads) from here on: no barrier needed
  for (int j = threadIdx.x; j < cnt; j += kFpsThreads) {
    const size_t g = 3 * (size_t)(lo + j);
    px[j] = xyz[g];
    py[j] = xyz[g + 1];
    pz[j] = xyz[g + 2];
    pd[j] = INFINITY;
  }
  int w = start;
  for (int t = 0; t < m; t++) {
    const size_t g = 3 * (size_t)w;
    const float qx = __ldg(xyz + g), qy = __ldg(xyz + g + 1), qz = __ldg(xyz + g + 2);
    const int wl = w - lo;
    unsigned long long best = 0;
#pragma unroll 4
    for (int j = threadIdx.x; j < cnt; j += kFpsThreads) {
      const float old = pd[j];
      const float d = j == wl ? -1.0f : fminf(old, fps_d2(px[j], py[j], pz[j], qx, qy, qz));
      if (d != old) pd[j] = d;
      best = max(best, fps_key(d, lo + j));
    }
    best = fps_warp_max(best);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = best;
    __syncthreads();
    if (threadIdx.x < 32) {
      best = fps_warp_max(red[threadIdx.x]);
      if (threadIdx.x == 0) {
        if (!kGrid)
          bcast = best;
        else if (best)
          atomicMax(slots + t, best);
      }
    }
    unsigned long long win;
    if constexpr (kGrid) {
      cg::this_grid().sync();
      win = __ldcg(slots + t);
    } else {
      __syncthreads();
      win = bcast;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
      idx_out[t] = w;
      r2_out[t] = __uint_as_float((uint32_t)(win >> 32));
    }
    w = (int)~(uint32_t)win;  // the next pick (meaningless only after the last pick of M = N)
  }
}

// ---------------------------------------------------------------- host

static bool fps_shape_ok(int n, int m) { return n >= 1 && n <= kFpsMaxN && m >= 1 && m <= n; }

struct FpsBuffers {
  unsigned long long* slots;  // one per pick
  float* soa;                 // x | y | z | D of the global-memory path
  size_t total;
};

static FpsBuffers fps_buffers(int n, int m, void* ws) {
  Carver c(ws);
  FpsBuffers b;
  b.slots = c.take<unsigned long long>(m);
  b.soa = c.take<float>(4 * (size_t)n);
  b.total = c.total;
  return b;
}

static int g_fps_force = kFpsAuto;
static int g_fps_last = 0;

struct FpsPlan {
  int path, blocks, slice;
  size_t smem;
};

template <bool kGrid, bool kShared>
static cudaError_t fps_occupancy(size_t smem, int* occ) {
  auto* fn = fps_kernel<kGrid, kShared>;
  int dev = 0, optin = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  cudaFuncAttributes fa;
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, fn);
  if (e != cudaSuccess) return e;
  if (smem + fa.sharedSizeBytes > (size_t)optin) {
    *occ = 0;
    return cudaSuccess;
  }
  e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(occ, fn, kFpsThreads, smem);
  return e;
}

// the path (forced, or chosen from N) and its grid; false with the message set when it cannot run here
static bool fps_plan(int n, FpsPlan* p) {
  int dev = 0, sms = 0, coop = 0, occ = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev);
  if (e != cudaSuccess) {
    set_error("ma_farthest_point_sample: %s", cudaGetErrorString(e));
    return false;
  }
  const int need = (n + kFpsThreads - 1) / kFpsThreads;  // CTAs for one point per thread
  const int grid_slice = (n + std::min(sms, need) - 1) / std::min(sms, need);
  int path = g_fps_force;
  if (path == kFpsAuto && n <= kFpsSmallN) {
    path = kFpsOneCta;
  } else if (path == kFpsAuto) {  // the slices in shared memory when one CTA per SM can hold them
    int fits = 0;
    e = fps_occupancy<true, true>((size_t)grid_slice * 16, &fits);
    if (e != cudaSuccess) cudaGetLastError();
    path = e == cudaSuccess && fits >= 1 ? kFpsGridShared : kFpsGridGlobal;
  }
  p->path = path;
  if (path == kFpsOneCta) {
    p->blocks = 1, p->slice = n, p->smem = (size_t)n * 16;
    e = fps_occupancy<false, true>(p->smem, &occ);
  } else if (path == kFpsGridShared) {
    p->slice = grid_slice, p->smem = (size_t)grid_slice * 16;
    e = fps_occupancy<true, true>(p->smem, &occ);
  } else if (path == kFpsGridGlobal) {
    p->smem = 0;
    e = fps_occupancy<true, false>(0, &occ);
    p->slice = (n + std::min(occ * sms, need) - 1) / std::max(std::min(occ * sms, need), 1);
  } else {
    set_error("ma_farthest_point_sample: unknown path %d", path);
    return false;
  }
  if (e != cudaSuccess) {
    set_error("ma_farthest_point_sample: %s", cudaGetErrorString(e));
    cudaGetLastError();
    return false;
  }
  if (occ < 1) {
    set_error("ma_farthest_point_sample: path %d cannot hold %d points per CTA on this device", path, p->slice);
    return false;
  }
  if (path != kFpsOneCta && !coop) {
    set_error("ma_farthest_point_sample: the device does not support cooperative launches");
    return false;
  }
  p->blocks = (n + p->slice - 1) / p->slice;  // no empty CTA
  return true;
}

}  // namespace ma

using namespace ma;

extern "C" {

size_t ma_farthest_point_sample_workspace_bytes(int n, int m) {
  if (!fps_shape_ok(n, m)) return 0;
  return fps_buffers(n, m, nullptr).total;
}

int ma_farthest_point_sample_set_path(int path) {
  const int prev = g_fps_force;
  if (path >= kFpsAuto && path <= kFpsGridGlobal) g_fps_force = path;
  return prev;
}

int ma_farthest_point_sample_last_path(void) { return g_fps_last; }

int ma_farthest_point_sample(const float* xyz, int n, int m, int start, int64_t* out_idx, float* out_r2, void* ws,
                             void* stream) {
  if (!xyz || !out_idx || !out_r2 || !ws || !fps_shape_ok(n, m) || start < 0 || start >= n) {
    set_error("ma_farthest_point_sample: bad arguments (1 <= m <= n <= 2^24, 0 <= start < n, non-null pointers)");
    return 1;
  }
  FpsPlan p;
  if (!fps_plan(n, &p)) return 1;
  cudaStream_t st = (cudaStream_t)stream;
  FpsBuffers b = fps_buffers(n, m, ws);
  cudaError_t e = cudaSuccess;
  if (p.path == kFpsOneCta) {
    fps_kernel<false, true><<<1, kFpsThreads, p.smem, st>>>(xyz, n, m, start, p.slice, b.soa, b.slots, out_idx,
                                                            out_r2);
  } else {
    e = cudaMemsetAsync(b.slots, 0, (size_t)m * 8, st);
    void* args[] = {(void*)&xyz, &n, &m, &start, &p.slice, &b.soa, &b.slots, &out_idx, &out_r2};
    if (e == cudaSuccess)
      e = cudaLaunchCooperativeKernel(p.path == kFpsGridShared ? (const void*)fps_kernel<true, true>
                                                               : (const void*)fps_kernel<true, false>,
                                      dim3(p.blocks), dim3(kFpsThreads), args, p.smem, st);
  }
  count_launch(1);
  if (stage_status("ma_farthest_point_sample", e)) return 1;
  g_fps_last = p.path;
  return 0;
}

}  // extern "C"
