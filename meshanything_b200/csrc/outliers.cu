// outliers.cu -- statistical and small-component outlier removal of a point cloud (DESIGN.md section 1.3 defines it).
//
// The points arrive already in the output frame (p' = (p - c) / L, metrics.to_output_frame), fp32 [N][3].
//   (a) grid      A robust cube: per axis the 1 % and 99 % quantiles from two 1024-bin histogram passes (the second
//                 inside the bins the first found), grown by 10 % on each side; its longest side holds G cells.  The
//                 host reads the 24-byte cube back, then knn_cell/scatter_kernel (knn_grid.cuh) sort the points into it,
//                 points outside clamped into the border cells.  The occupied cells are compacted (CUB DeviceSelect)
//                 and each gets the true box of its points (min / max, exact).
//   (b) kNN       knn_grid_kernel with a shell budget of kOlBudget: a query not finished by then (a far point, whose
//                 shells would run out to the whole grid) scans the occupied cells' boxes instead.  It also writes the
//                 fp32 d^2 of every neighbour.  The result is the exact kNN of section 1.2 whatever the grid.
//   (c) stats     d_i = (sum over ranks of fp32 sqrt(d^2)) / k in fp64; mu and the two-pass sigma as sums over tiles
//                 of 256 consecutive indices, each summed in index order, the tile partials summed in tile order by
//                 one thread; inlier iff d_i <= mu + std_ratio sigma.  No floating-point atomics.
//   (d) parts     connected components of the kNN graph restricted to the inliers: min-label hooking (atomicMin of
//                 the larger root onto the smaller) and pointer jumping, one 4-byte read-back per round; labels are
//                 minimum indices, so the result does not depend on the schedule.  Sizes by integer atomics; a
//                 component is kept iff size >= min_component n_inliers (fp64) or it is the largest (lowest label on
//                 ties).  The kept indices are compacted in ascending order (CUB DeviceSelect::Flagged).
// Every fp32 / fp64 step is an explicit round-to-nearest intrinsic, so tests/outliers_oracle.py restates d_i, mu,
// sigma, the threshold, the masks and the counts bit for bit.
#include <algorithm>
#include <cmath>

#include <cub/device/device_select.cuh>
#include <cub/iterator/counting_input_iterator.cuh>

#include "knn_grid.cuh"
#include "workspace.h"

namespace ma {

constexpr int kOlThreads = 256;
constexpr int kOlTile = 256;          // indices per tile of the fixed-order fp64 sums
constexpr int kOlBins = 1024;         // histogram bins per axis and pass
constexpr int kOlBudget = 2;          // shells (radius 0..2: 125 cells) before a query scans the occupied cells
constexpr int kOlMaxN = 1 << 24;      // the index part of a kNN key and the component labels
constexpr int kOlMaxRounds = 1024;    // connectivity rounds; every round with a hook lowers some root's parent
constexpr double kOlQuantile = 0.01;  // robust extent: [1 %, 99 %] per axis
constexpr float kOlPad = 0.1f;        // ... grown by 10 % of the extent on each side

// ---------------------------------------------------------------- (a) robust grid

// hist[a][b]: points whose coordinate a falls in bin b of [lo, lo + kOlBins w), clamped into the end bins
__global__ void outliers_hist_kernel(const float* __restrict__ xyz, int n, const float* __restrict__ box,
                                     uint32_t* __restrict__ hist) {
  __shared__ uint32_t h[3 * kOlBins];
  for (int t = threadIdx.x; t < 3 * kOlBins; t += blockDim.x) h[t] = 0;
  __syncthreads();
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    for (int a = 0; a < 3; a++) {
      const int b = (int)floorf((xyz[3 * (size_t)i + a] - box[a]) / box[3 + a]);
      atomicAdd(h + a * kOlBins + min(max(b, 0), kOlBins - 1), 1u);
    }
  }
  __syncthreads();
  for (int t = threadIdx.x; t < 3 * kOlBins; t += blockDim.x)
    if (h[t]) atomicAdd(hist + t, h[t]);
}

// one thread per axis: the bins holding the points of rank t and n - 1 - t; narrows box[a] to them (pass 0) or turns
// them into the robust extent of axis a (pass 1)
__global__ void outliers_range_kernel(const uint32_t* __restrict__ hist, int n, int pass, float* __restrict__ box,
                                      float* __restrict__ ext) {
  const int a = threadIdx.x;
  if (a >= 3) return;
  const uint32_t t = (uint32_t)(kOlQuantile * n), t2 = (uint32_t)n - 1u - t;
  uint32_t cum = 0;
  int blo = -1, bhi = kOlBins - 1;
  for (int b = 0; b < kOlBins; b++) {
    cum += hist[a * kOlBins + b];
    if (blo < 0 && cum > t) blo = b;
    if (cum > t2) {
      bhi = b;
      break;
    }
  }
  blo = max(blo, 0);
  const float lo = box[a] + (float)blo * box[3 + a], hi = box[a] + (float)(bhi + 1) * box[3 + a];
  if (pass == 0) {
    box[a] = lo;
    box[3 + a] = (hi - lo) / (float)kOlBins;
  } else {
    ext[a] = lo;
    ext[3 + a] = hi;
  }
}

struct OlOccupied {
  const uint32_t* start;
  __device__ __forceinline__ bool operator()(uint32_t c) const { return start[c + 1] > start[c]; }
};

// boxes[2 b], boxes[2 b + 1] = (min xyz, first slot), (max xyz, end slot) of occupied cell b
__global__ void outliers_box_kernel(const float4* __restrict__ sorted, const uint32_t* __restrict__ start,
                                    const uint32_t* __restrict__ occ, const int* __restrict__ nocc,
                                    float4* __restrict__ boxes) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= *nocc) return;
  const uint32_t c = occ[b], s = start[c], e = start[c + 1];
  float4 lo = sorted[s], hi = lo;
  for (uint32_t t = s + 1; t < e; t++) {
    const float4 p = sorted[t];
    lo.x = fminf(lo.x, p.x), lo.y = fminf(lo.y, p.y), lo.z = fminf(lo.z, p.z);
    hi.x = fmaxf(hi.x, p.x), hi.y = fmaxf(hi.y, p.y), hi.z = fmaxf(hi.z, p.z);
  }
  lo.w = __uint_as_float(s);
  hi.w = __uint_as_float(e);
  boxes[2 * b] = lo;
  boxes[2 * b + 1] = hi;
}

// ---------------------------------------------------------------- (c) statistics

__global__ void outliers_mean_kernel(const float* __restrict__ d2, int n, int k, double* __restrict__ dbar) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float* r = d2 + (size_t)i * k;
  double s = 0.0;
  for (int e = 0; e < k; e++) s = __dadd_rn(s, (double)__fsqrt_rn(r[e]));
  dbar[i] = __ddiv_rn(s, (double)k);
}

// one CTA per tile: the tile's values (x_i, or (x_i - mu)^2 when mu is given) summed in index order from 0
__global__ void __launch_bounds__(kOlTile) outliers_tile_kernel(const double* __restrict__ x, int n,
                                                                const double* __restrict__ mu,
                                                                double* __restrict__ part) {
  __shared__ double v[kOlTile];
  const int i = blockIdx.x * kOlTile + threadIdx.x;
  double y = 0.0;
  if (i < n) {
    y = x[i];
    if (mu) {
      const double d = __dsub_rn(y, *mu);
      y = __dmul_rn(d, d);
    }
  }
  v[threadIdx.x] = y;
  __syncthreads();
  if (threadIdx.x == 0) {
    const int m = min(kOlTile, n - blockIdx.x * kOlTile);
    double s = 0.0;
    for (int t = 0; t < m; t++) s = __dadd_rn(s, v[t]);
    part[blockIdx.x] = s;
  }
}

// the tile partials in tile order.  pass 0: stats[0] = mu; pass 1: stats[1] = sigma, stats[2] = mu + std_ratio sigma
__global__ void outliers_moment_kernel(const double* __restrict__ part, int tiles, int n, int pass, double std_ratio,
                                       double* __restrict__ stats) {
  if (threadIdx.x != 0) return;
  double s = 0.0;
  for (int t = 0; t < tiles; t++) s = __dadd_rn(s, part[t]);
  if (pass == 0) {
    stats[0] = __ddiv_rn(s, (double)n);
  } else {
    const double sigma = n > 1 ? __dsqrt_rn(__ddiv_rn(s, (double)(n - 1))) : 0.0;
    stats[1] = sigma;
    stats[2] = __dadd_rn(stats[0], __dmul_rn(std_ratio, sigma));
  }
}

// inl[i] = d_i <= threshold; parent[i] = i; counters[0] += inliers (one atomic per warp)
__global__ void outliers_inlier_kernel(const double* __restrict__ dbar, int n, const double* __restrict__ stats,
                                       uint8_t* __restrict__ inl, uint32_t* __restrict__ parent,
                                       int* __restrict__ counters) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool in = i < n && dbar[i] <= stats[2];
  if (i < n) {
    inl[i] = in ? 1 : 0;
    parent[i] = (uint32_t)i;
  }
  const unsigned votes = __ballot_sync(0xffffffffu, in);
  if ((threadIdx.x & 31) == 0 && votes) atomicAdd(counters, __popc(votes));
}

// ---------------------------------------------------------------- (d) components

// every kNN slot between two inliers of different trees hooks the larger root onto the smaller one
__global__ void outliers_hook_kernel(const int32_t* __restrict__ knn, int n, int k, const uint8_t* __restrict__ inl,
                                     uint32_t* parent, int* __restrict__ changed) {
  const size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (e >= (size_t)n * k) return;
  const int i = (int)(e / k), j = knn[e];
  if (!inl[i] || !inl[j]) return;
  volatile uint32_t* p = parent;
  const uint32_t a = p[i], b = p[j];
  if (a == b) return;
  atomicMin(parent + max(a, b), min(a, b));
  *changed = 1;
}

// pointer jumping: every vertex points at its root.  Every value read is an ancestor, old or new, and parents only
// decrease, so the walk ends and the result does not depend on the schedule.
__global__ void outliers_jump_kernel(int n, uint32_t* parent) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n) return;
  volatile uint32_t* p = parent;
  uint32_t r = p[v];
  for (uint32_t q = p[r]; q != r; q = p[r]) r = q;
  p[v] = r;
}

// size[root] += members (lanes with the same root add once)
__global__ void outliers_size_kernel(int n, const uint8_t* __restrict__ inl, const uint32_t* __restrict__ parent,
                                     uint32_t* __restrict__ size) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  const bool in = v < n && inl[v];
  const uint32_t r = in ? parent[v] : 0xffffffffu;
  const unsigned peers = __match_any_sync(0xffffffffu, r);
  if (in && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(size + r, (uint32_t)__popc(peers));
}

// per root: counters[1] += 1; largest = max of (size << 32 | ~root), the lowest root among the largest
__global__ void outliers_largest_kernel(int n, const uint8_t* __restrict__ inl, const uint32_t* __restrict__ parent,
                                        const uint32_t* __restrict__ size, unsigned long long* __restrict__ largest,
                                        int* __restrict__ counters) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n || !inl[v] || parent[v] != (uint32_t)v) return;
  atomicAdd(counters + 1, 1);
  atomicMax(largest, ((unsigned long long)size[v] << 32) | (uint32_t)~(uint32_t)v);
}

// keep[v]: an inlier whose component is large enough or the largest; counters[2] += dropped components
__global__ void outliers_keep_kernel(int n, const uint8_t* __restrict__ inl, const uint32_t* __restrict__ parent,
                                     const uint32_t* __restrict__ size, const unsigned long long* __restrict__ largest,
                                     double min_component, int* counters, uint8_t* __restrict__ keep) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n) return;
  if (!inl[v]) {
    keep[v] = 0;
    return;
  }
  const uint32_t r = parent[v];
  const bool big = r == ~(uint32_t)*largest || (double)size[r] >= __dmul_rn(min_component, (double)counters[0]);
  keep[v] = big ? 1 : 0;
  if (!big && r == (uint32_t)v) atomicAdd(counters + 2, 1);
}

// stats[3..7] = statistical inliers, components, components dropped, kept points, connectivity rounds
__global__ void outliers_finish_kernel(const int* __restrict__ counters, const int64_t* __restrict__ n_kept,
                                       int rounds, double* __restrict__ stats) {
  if (threadIdx.x != 0) return;
  stats[3] = (double)counters[0];
  stats[4] = (double)counters[1];
  stats[5] = (double)counters[2];
  stats[6] = (double)*n_kept;
  stats[7] = (double)rounds;
}

// ---------------------------------------------------------------- workspace

static bool ol_shape_ok(int n, int k) { return k >= 1 && k <= kKnnMaxK && n > k && n <= kOlMaxN; }

static size_t ol_occ_bytes(size_t cells) {
  size_t bytes = 0;
  cub::DeviceSelect::If(nullptr, bytes, cub::CountingInputIterator<uint32_t>(0), (uint32_t*)nullptr, (int*)nullptr,
                        (int)cells, OlOccupied{nullptr});
  return bytes;
}

static size_t ol_flag_bytes(int n) {
  size_t bytes = 0;
  cub::DeviceSelect::Flagged(nullptr, bytes, cub::CountingInputIterator<int64_t>(0), (uint8_t*)nullptr,
                             (int64_t*)nullptr, (int64_t*)nullptr, n);
  return bytes;
}

struct OlBuffers {
  float4* sorted;
  uint32_t *cell, *count, *start;
  void* cub;         // the largest CUB temporary, shared by the scan and both selections
  size_t cub_bytes;
  uint32_t* hist;
  float *box, *ext;
  uint32_t* occ;
  int* nocc;
  float4* boxes;
  int32_t* knn;
  float* d2;
  double *dbar, *part;
  uint8_t* inl;
  uint32_t *parent, *size;
  unsigned long long* largest;
  int* counters;
  size_t total;
};

static OlBuffers ol_buffers(int n, int k, void* ws) {
  const int G = knn_grid_size(n, k);
  const size_t cells = (size_t)G * G * G, nk = (size_t)n * k, nbox = std::min(cells, (size_t)n);
  Carver c(ws);
  OlBuffers b;
  b.cub_bytes = std::max(knn_bin_scan_bytes(cells), std::max(ol_occ_bytes(cells), ol_flag_bytes(n)));
  b.sorted = c.take<float4>(n);
  b.cell = c.take<uint32_t>(n);
  b.count = c.take<uint32_t>(cells + 1);
  b.start = c.take<uint32_t>(cells + 1);
  b.cub = c.take<char>(b.cub_bytes);
  b.hist = c.take<uint32_t>(3 * kOlBins);
  b.box = c.take<float>(6);
  b.ext = c.take<float>(6);
  b.occ = c.take<uint32_t>(nbox);
  b.nocc = c.take<int>(1);
  b.boxes = c.take<float4>(2 * nbox);
  b.knn = c.take<int32_t>(nk);
  b.d2 = c.take<float>(nk);
  b.dbar = c.take<double>(n);
  b.part = c.take<double>((n + kOlTile - 1) / kOlTile);
  b.inl = c.take<uint8_t>(n);
  b.parent = c.take<uint32_t>(n);
  b.size = c.take<uint32_t>(n);
  b.largest = c.take<unsigned long long>(1);
  b.counters = c.take<int>(4);
  b.total = c.total;
  return b;
}

// the cube over the robust extent ext = (lo[3], hi[3]): its longest side (grown by kOlPad on each side) in G cells
static KnnGrid ol_grid(const float* ext, int G) {
  float side = 0.0f;
  for (int a = 0; a < 3; a++) side = std::max(side, ext[3 + a] - ext[a]);
  side *= 1.0f + 2.0f * kOlPad;
  if (!(side >= 1e-6f)) side = 1e-6f;  // every robust extent empty (a cloud of identical points)
  KnnGrid g;
  for (int a = 0; a < 3; a++) g.lo[a] = 0.5f * (ext[a] + ext[3 + a]) - 0.5f * side;
  g.scale = (float)G / side;
  g.inv = 1.0f / g.scale;
  g.G = G;
  return g;
}

static StageEvents<5> ol_events;

}  // namespace ma

using namespace ma;

extern "C" {

size_t ma_remove_outliers_workspace_bytes(int n, int k) {
  if (!ol_shape_ok(n, k)) return 0;
  return ol_buffers(n, k, nullptr).total;
}

void ma_remove_outliers_set_events(void* const* events) { ol_events.set(events); }

int ma_remove_outliers(const float* xyz, int n, int k, double std_ratio, double min_component, uint8_t* keep_out,
                       int64_t* kept_idx_out, int64_t* n_kept_out, double* mean_dist_out, int32_t* knn_out,
                       double* stats_out, void* ws, void* stream) {
  if (!xyz || !keep_out || !kept_idx_out || !n_kept_out || !stats_out || !ws || !ol_shape_ok(n, k) ||
      !std::isfinite(std_ratio) || !std::isfinite(min_component) || min_component < 0.0) {
    set_error("ma_remove_outliers: bad arguments (1 <= k <= %d, k < n <= 2^24, finite std_ratio, finite "
              "min_component >= 0)", kKnnMaxK);
    return 1;
  }
  const char* what = "ma_remove_outliers";
  cudaStream_t st = (cudaStream_t)stream;
  OlBuffers b = ol_buffers(n, k, ws);
  if (knn_out) b.knn = knn_out;
  if (mean_dist_out) b.dbar = mean_dist_out;
  const int G = knn_grid_size(n, k);
  const size_t cells = (size_t)G * G * G, nk = (size_t)n * k, nbox = std::min(cells, (size_t)n);
  const int tiles = (n + kOlTile - 1) / kOlTile;
  size_t cub_bytes = b.cub_bytes;

  // (a) the robust cube: two histogram passes, the first over the whole frame [-0.5, 0.5]^3
  ol_events.mark(0, st);
  const float frame[6] = {-0.5f, -0.5f, -0.5f, 1.0f / kOlBins, 1.0f / kOlBins, 1.0f / kOlBins};
  cudaError_t e = cudaMemcpyAsync(b.box, frame, sizeof(frame), cudaMemcpyHostToDevice, st);
  const int hist_blocks = std::min(blocks(n, kOlThreads), 1024);
  for (int pass = 0; pass < 2 && e == cudaSuccess; pass++) {
    e = cudaMemsetAsync(b.hist, 0, 3 * kOlBins * 4, st);
    outliers_hist_kernel<<<hist_blocks, kOlThreads, 0, st>>>(xyz, n, b.box, b.hist);
    outliers_range_kernel<<<1, 32, 0, st>>>(b.hist, n, pass, b.box, b.ext);
    count_launch(2);
  }
  float ext_h[6];
  if (e == cudaSuccess) e = cudaMemcpyAsync(ext_h, b.ext, sizeof(ext_h), cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  if (stage_status(what, e)) return 1;
  const KnnGrid grid = ol_grid(ext_h, G);
  e = knn_bin(xyz, n, grid, b.cell, b.count, b.start, b.sorted, b.cub, cub_bytes, st);
  if (e != cudaSuccess) return stage_status(what, e);
  e = cub::DeviceSelect::If(b.cub, cub_bytes, cub::CountingInputIterator<uint32_t>(0), b.occ, b.nocc, (int)cells,
                            OlOccupied{b.start}, st);
  outliers_box_kernel<<<blocks(nbox, kOlThreads), kOlThreads, 0, st>>>(b.sorted, b.start, b.occ, b.nocc, b.boxes);
  count_launch(3);
  ol_events.mark(1, st);
  // (b) kNN with the fp32 d^2 of every neighbour
  knn_grid_kernel<true><<<(n + kKnnThreads - 1) / kKnnThreads, kKnnThreads,
                          (size_t)k * kKnnThreads * sizeof(unsigned long long), st>>>(
      b.sorted, b.start, n, k, grid, kOlBudget, b.boxes, b.nocc, b.knn, b.d2);
  count_launch(1);
  ol_events.mark(2, st);
  // (c) mean distances, mu, sigma, the statistical inliers
  if (e == cudaSuccess) e = cudaMemsetAsync(b.counters, 0, 4 * 4, st);
  outliers_mean_kernel<<<blocks(n, kOlThreads), kOlThreads, 0, st>>>(b.d2, n, k, b.dbar);
  outliers_tile_kernel<<<tiles, kOlTile, 0, st>>>(b.dbar, n, nullptr, b.part);
  outliers_moment_kernel<<<1, 32, 0, st>>>(b.part, tiles, n, 0, std_ratio, stats_out);
  outliers_tile_kernel<<<tiles, kOlTile, 0, st>>>(b.dbar, n, stats_out, b.part);
  outliers_moment_kernel<<<1, 32, 0, st>>>(b.part, tiles, n, 1, std_ratio, stats_out);
  outliers_inlier_kernel<<<blocks(n, kOlThreads), kOlThreads, 0, st>>>(b.dbar, n, stats_out, b.inl, b.parent,
                                                                       b.counters);
  count_launch(6);
  ol_events.mark(3, st);
  if (stage_status(what, e)) return 1;
  // (d) components of the inlier graph (skipped when min_component = 0: every inlier is kept)
  int rounds = 0;
  if (min_component > 0.0) {
    for (;;) {
      if (rounds == kOlMaxRounds) {
        set_error("ma_remove_outliers: connectivity did not finish in %d rounds", kOlMaxRounds);
        return 1;
      }
      rounds++;
      int changed = 0;
      e = cudaMemsetAsync(b.counters + 3, 0, 4, st);
      outliers_hook_kernel<<<blocks(nk, kOlThreads), kOlThreads, 0, st>>>(b.knn, n, k, b.inl, b.parent,
                                                                          b.counters + 3);
      outliers_jump_kernel<<<blocks(n, kOlThreads), kOlThreads, 0, st>>>(n, b.parent);
      count_launch(2);
      if (e == cudaSuccess) e = cudaMemcpyAsync(&changed, b.counters + 3, 4, cudaMemcpyDeviceToHost, st);
      if (e == cudaSuccess) e = cudaStreamSynchronize(st);
      if (stage_status(what, e)) return 1;
      if (changed == 0) break;
    }
    e = cudaMemsetAsync(b.size, 0, (size_t)n * 4, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(b.largest, 0, 8, st);
    outliers_size_kernel<<<blocks(n, kOlThreads), kOlThreads, 0, st>>>(n, b.inl, b.parent, b.size);
    outliers_largest_kernel<<<blocks(n, kOlThreads), kOlThreads, 0, st>>>(n, b.inl, b.parent, b.size, b.largest,
                                                                          b.counters);
    outliers_keep_kernel<<<blocks(n, kOlThreads), kOlThreads, 0, st>>>(n, b.inl, b.parent, b.size, b.largest,
                                                                       min_component, b.counters, keep_out);
    count_launch(3);
  } else if (e == cudaSuccess) {
    e = cudaMemcpyAsync(keep_out, b.inl, (size_t)n, cudaMemcpyDeviceToDevice, st);
  }
  cub_bytes = b.cub_bytes;
  if (e == cudaSuccess)
    e = cub::DeviceSelect::Flagged(b.cub, cub_bytes, cub::CountingInputIterator<int64_t>(0), keep_out, kept_idx_out,
                                   n_kept_out, n, st);
  outliers_finish_kernel<<<1, 32, 0, st>>>(b.counters, n_kept_out, rounds, stats_out);
  count_launch(1);
  ol_events.mark(4, st);
  return stage_status(what, e);
}

}  // extern "C"
