// knn_grid.cuh -- the exact kNN of DESIGN.md section 1.2 on a uniform grid, shared by normals.cu, outliers.cu and
// smooth.cu.
//
//   grid   knn_cell_kernel counts the points per cell of a G^3 grid of cubic cells (origin lo, `scale` cells per unit;
//          points outside are clamped into the border cells), a CUB exclusive scan gives the cell starts,
//          knn_scatter_kernel writes the points in cell order (float4: xyz and the original index).  The order inside a
//          cell is whatever the atomics give: nothing depends on it.
//   kNN    knn_grid_kernel, one thread per point: shells of cells by Chebyshev radius r = 0, 1, ... around the query's
//          cell, every candidate keyed by (fp32 d^2 bits << 32 | index), the k smallest keys kept sorted in shared
//          memory.  After shell r it stops when the k-th key's d^2 is below a lower bound of the distance to every cell
//          outside the shells (shrunk by a margin far above fp32 rounding), or when no cell is left.  Clamping keeps
//          that bound valid: a border cell only gains points farther out than its nominal box.  With a shell budget, a
//          query still unfinished after shell `budget` starts over on the compact list of occupied cells with their
//          true point boxes (knn_scan_boxes).  The grid and the budget therefore only change the speed: the result is
//          the exact kNN.
#pragma once

#include <cstdint>

#include <cub/device/device_scan.cuh>

namespace ma {

constexpr int kKnnBinThreads = 256;  // threads per CTA of knn_cell_kernel and knn_scatter_kernel
constexpr int kKnnThreads = 64;   // kNN threads per CTA: k x 64 x 8 B of shared memory for the top-k lists
constexpr int kKnnMaxK = 64;
constexpr int kKnnMaxG = 256;

// the grid: cell index floor((x - lo) * scale) per axis, clamped to [0, G); inv = 1 / scale is a cell's side
struct KnnGrid {
  float lo[3];
  float scale, inv;
  int G;
};

// grid cells per axis: about 4 k points per occupied cell of a surface spanning the grid, so that radius 1 mostly
// suffices
static inline int knn_grid_size(int n, int k) {
  const int g = (int)ceil(0.5 * sqrt((double)n / (double)k));
  return g < 1 ? 1 : (g > kKnnMaxG ? kKnnMaxG : g);
}

// the grid over the whole output frame [-0.5, 0.5]^3 (normals.cu, smooth.cu)
static inline KnnGrid knn_frame_grid(int n, int k) {
  const int G = knn_grid_size(n, k);
  return KnnGrid{{-0.5f, -0.5f, -0.5f}, (float)G, 1.0f / (float)G, G};
}

__device__ __forceinline__ int knn_cell1(float x, float lo, float scale, int G) {
  const int c = (int)floorf(__fmul_rn(__fsub_rn(x, lo), scale));
  return min(max(c, 0), G - 1);
}

static __global__ void knn_cell_kernel(const float* __restrict__ xyz, int n, KnnGrid g, uint32_t* __restrict__ cell,
                                       uint32_t* __restrict__ count) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* p = xyz + 3 * (size_t)i;
  const int G = g.G;
  const uint32_t c = ((uint32_t)knn_cell1(p[0], g.lo[0], g.scale, G) * G + knn_cell1(p[1], g.lo[1], g.scale, G)) * G +
                     knn_cell1(p[2], g.lo[2], g.scale, G);
  cell[i] = c;
  atomicAdd(count + c, 1u);
}

// count[c] is used up as a cursor: the point takes slot start[c] + (atomicSub's old value - 1)
static __global__ void knn_scatter_kernel(const float* __restrict__ xyz, int n, const uint32_t* __restrict__ cell,
                                          const uint32_t* __restrict__ start, uint32_t* __restrict__ count,
                                          float4* __restrict__ sorted) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t c = cell[i];
  const uint32_t slot = start[c] + atomicSub(count + c, 1u) - 1u;
  const float* p = xyz + 3 * (size_t)i;
  sorted[slot] = make_float4(p[0], p[1], p[2], __int_as_float(i));
}

// bytes of CUB scratch that knn_bin needs for a grid of `cells` cells
static inline size_t knn_bin_scan_bytes(size_t cells) {
  size_t bytes = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, bytes, (uint32_t*)nullptr, (uint32_t*)nullptr, (int)(cells + 1));
  return bytes;
}

// The grid step on stream st: zero count[cells + 1], bin the points, scan the counts into start[], scatter the
// points into sorted[] in cell order.  Stops at the first runtime error and returns it.  Launches are not counted.
static inline cudaError_t knn_bin(const float* xyz, int n, const KnnGrid& g, uint32_t* cell, uint32_t* count,
                                  uint32_t* start, float4* sorted, void* scan, size_t scan_bytes, cudaStream_t st) {
  const size_t cells = (size_t)g.G * g.G * g.G;
  const int nb = (n + kKnnBinThreads - 1) / kKnnBinThreads;
  cudaError_t e = cudaMemsetAsync(count, 0, (cells + 1) * 4, st);
  if (e != cudaSuccess) return e;
  knn_cell_kernel<<<nb, kKnnBinThreads, 0, st>>>(xyz, n, g, cell, count);
  e = cub::DeviceScan::ExclusiveSum(scan, scan_bytes, count, start, (int)(cells + 1), st);
  if (e != cudaSuccess) return e;
  knn_scatter_kernel<<<nb, kKnnBinThreads, 0, st>>>(xyz, n, cell, start, count, sorted);
  return cudaSuccess;
}

// offers the candidates sorted[t0, t1) to the sorted top-k list top[e * kKnnThreads] (m entries so far)
__device__ __forceinline__ void knn_offer(const float4* __restrict__ sorted, uint32_t t0, uint32_t t1, float4 q,
                                          int self, int k, unsigned long long* top, int& m) {
  for (uint32_t t = t0; t < t1; t++) {
    const float4 p = sorted[t];
    const int j = __float_as_int(p.w);
    if (j == self) continue;
    const float ex = __fsub_rn(q.x, p.x), ey = __fsub_rn(q.y, p.y), ez = __fsub_rn(q.z, p.z);
    const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey)), __fmul_rn(ez, ez));
    const unsigned long long key = ((unsigned long long)__float_as_uint(d2) << 32) | (uint32_t)j;
    if (m == k && key >= top[(size_t)(k - 1) * kKnnThreads]) continue;
    int e = m < k ? m++ : k - 1;
    while (e > 0 && top[(size_t)(e - 1) * kKnnThreads] > key) {
      top[(size_t)e * kKnnThreads] = top[(size_t)(e - 1) * kKnnThreads];
      e--;
    }
    top[(size_t)e * kKnnThreads] = key;
  }
}

// The search over boxes[2 b], boxes[2 b + 1] = (min xyz, first slot bits), (max xyz, end slot bits) of every occupied
// cell, from an empty list.  Pass 1: U = the least distance within which some cell holds k + 1 points (its farthest
// box corner), so at least k other points lie within U.  Pass 2: every cell whose box is nearer than U and than the
// current k-th key.  Both distances are fp32 and widened by a relative 1e-5, far above the rounding of d^2.
__device__ __forceinline__ void knn_scan_boxes(const float4* __restrict__ sorted, const float4* __restrict__ boxes,
                                               int nbox, float4 q, int self, int k, unsigned long long* top, int& m) {
  float u2 = INFINITY;
  for (int b = 0; b < nbox; b++) {
    const float4 lo = boxes[2 * b], hi = boxes[2 * b + 1];
    if (__float_as_uint(hi.w) - __float_as_uint(lo.w) < (uint32_t)k + 1u) continue;
    const float fx = fmaxf(fabsf(q.x - lo.x), fabsf(hi.x - q.x)), fy = fmaxf(fabsf(q.y - lo.y), fabsf(hi.y - q.y)),
                fz = fmaxf(fabsf(q.z - lo.z), fabsf(hi.z - q.z));
    u2 = fminf(u2, (fx * fx + fy * fy + fz * fz) * (1.0f + 1e-5f));
  }
  m = 0;
  for (int b = 0; b < nbox; b++) {
    const float4 lo = boxes[2 * b], hi = boxes[2 * b + 1];
    const float gx = fmaxf(fmaxf(lo.x - q.x, q.x - hi.x), 0.0f), gy = fmaxf(fmaxf(lo.y - q.y, q.y - hi.y), 0.0f),
                gz = fmaxf(fmaxf(lo.z - q.z, q.z - hi.z), 0.0f);
    const float l2 = (gx * gx + gy * gy + gz * gz) * (1.0f - 1e-5f);
    if (l2 > u2) continue;
    if (m == k && l2 > __uint_as_float((uint32_t)(top[(size_t)(k - 1) * kKnnThreads] >> 32))) continue;
    knn_offer(sorted, __float_as_uint(lo.w), __float_as_uint(hi.w), q, self, k, top, m);
  }
}

// knn[i][rank] (and d2_out[i][rank], the fp32 d^2 of the key, when not null).  kBudget: after shell `budget` an
// unfinished query scans the boxes; without it (the instance normals.cu runs) shells only, and no boxes are read.
template <bool kBudget>
__global__ void __launch_bounds__(kKnnThreads)
    knn_grid_kernel(const float4* __restrict__ sorted, const uint32_t* __restrict__ start, int n, int k, KnnGrid g,
                    int budget, const float4* __restrict__ boxes, const int* __restrict__ nbox,
                    int32_t* __restrict__ knn, float* __restrict__ d2_out) {
  extern __shared__ unsigned long long knn_top[];  // [k][kKnnThreads]: entry e of thread t at e * 64 + t
  const int s = blockIdx.x * kKnnThreads + threadIdx.x;
  if (s >= n) return;
  unsigned long long* top = knn_top + threadIdx.x;
  const float4 q = sorted[s];
  const int self = __float_as_int(q.w);
  const int G = g.G;
  const int cx = knn_cell1(q.x, g.lo[0], g.scale, G), cy = knn_cell1(q.y, g.lo[1], g.scale, G),
            cz = knn_cell1(q.z, g.lo[2], g.scale, G);
  const float inv = g.inv;
  int m = 0;
  for (int r = 0;; r++) {
    for (int dx = -r; dx <= r; dx++) {
      const int x = cx + dx;
      if (x < 0 || x >= G) continue;
      for (int dy = -r; dy <= r; dy++) {
        const int y = cy + dy;
        if (y < 0 || y >= G) continue;
        // the shell of radius r: whole z columns on its x / y faces, only dz = -r and +r inside them
        const int step = (r == 0 || dx == -r || dx == r || dy == -r || dy == r) ? 1 : 2 * r;
        for (int dz = -r; dz <= r; dz += step) {
          const int z = cz + dz;
          if (z < 0 || z >= G) continue;
          const uint32_t c = ((uint32_t)x * G + y) * G + z;
          knn_offer(sorted, start[c], start[c + 1], q, self, k, top, m);
        }
      }
    }
    // lower bound of the distance from q to any cell outside the cube [c - r, c + r]^3 (only the sides that have cells)
    float b = INFINITY;
    if (cx - r > 0) b = fminf(b, q.x - ((float)(cx - r) * inv + g.lo[0]));
    if (cx + r < G - 1) b = fminf(b, ((float)(cx + r + 1) * inv + g.lo[0]) - q.x);
    if (cy - r > 0) b = fminf(b, q.y - ((float)(cy - r) * inv + g.lo[1]));
    if (cy + r < G - 1) b = fminf(b, ((float)(cy + r + 1) * inv + g.lo[1]) - q.y);
    if (cz - r > 0) b = fminf(b, q.z - ((float)(cz - r) * inv + g.lo[2]));
    if (cz + r < G - 1) b = fminf(b, ((float)(cz + r + 1) * inv + g.lo[2]) - q.z);
    if (b == INFINITY) break;  // every cell has been searched
    if (m == k) {
      // margin: a point can sit ~1e-7 outside its cell after fp32 rounding, and d^2 carries a few ulps of error; a
      // strict < because an unseen point at the same d^2 with a lower index would still rank first
      const float bs = fmaxf(b - 1e-6f, 0.0f);
      if (__uint_as_float((uint32_t)(top[(size_t)(k - 1) * kKnnThreads] >> 32)) < bs * bs * (1.0f - 1e-5f)) break;
    }
    if (kBudget && r == budget) {
      knn_scan_boxes(sorted, boxes, *nbox, q, self, k, top, m);
      break;
    }
  }
  int32_t* out = knn + (size_t)self * k;
  for (int e = 0; e < k; e++) out[e] = (int32_t)(uint32_t)top[(size_t)e * kKnnThreads];
  if (d2_out) {
    float* o2 = d2_out + (size_t)self * k;
    for (int e = 0; e < k; e++) o2[e] = __uint_as_float((uint32_t)(top[(size_t)e * kKnnThreads] >> 32));
  }
}

}  // namespace ma
