// objects.cu -- splitting a point cloud into objects: the connected components of the graph "d^2 <= e2", ordered by
// size, and the ones holding at least min_points points (DESIGN.md section 1.7 defines it).
//
// The points arrive already in the output frame (p' = (p - c) / L, metrics.to_output_frame), fp32 [N][3].
//   (a) grid      the bounding box by integer atomics on order-preserving float bits; a cell side h =
//                 max(e (1 + 1e-5) / 2, extent / 2^20), the cell of a point floor((x - lo) / h) per axis in fp64, a
//                 63-bit key (21 bits per axis); CUB radix sort of (key, index), run-length encoding of the occupied
//                 cells, an exclusive scan for their starts, the points gathered in cell order.  Two points with
//                 d^2 <= e2 are less than e (1 + 1e-6) apart, so their cells differ by at most 2 on every axis.
//   (b) union     union-find over the point indices in `labels` (ECL-CC hooking: the larger root under the smaller with
//                 atomicCAS, so every root is the lowest index of its tree).  A cell whose exact fp32 point box passes
//                 the pair formula is a clique: its points are hooked to its first (lowest) index at once.  One warp
//                 per cell A looks up the 62 cells after it in the 5^3 neighbourhood by binary search and skips a pair
//                 of cells whose box gap fails the formula or, for two cliques, whose roots already agree; otherwise
//                 the warp tests point pairs -- for two cliques only until the first pair within e2.  A final pass compresses every label to its root, the component minimum.
//   (c) order     sizes by warp-aggregated integer atomics; CUB sort (descending) of size << 24 | (2^24 - 1 - label);
//                 the objects are the prefix of clusters with size >= min_points; their offsets by a CUB scan, their
//                 indices by a stable CUB radix sort of (object rank, index).
// No host synchronisation and no floating-point atomics; labels are component minima, so the result does not depend
// on the schedule and tests/objects_oracle.py restates labels, indices, offsets and stats bit for bit.
#include <algorithm>
#include <cmath>

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_run_length_encode.cuh>
#include <cub/device/device_scan.cuh>

#include "workspace.h"

namespace ma {

constexpr int kObThreads = 256;
constexpr int kObMaxN = 1 << 24;
constexpr int kObAxisBits = 21;                          // cell coordinate bits per axis of the 63-bit key
constexpr uint32_t kObAxisMask = (1u << kObAxisBits) - 1u;
constexpr int kObReach = 2;                              // neighbour cells per axis and side (cell side >= e / 2)
constexpr int kObForward = 62;                           // the cells after the centre of the 5^3 block, in key order
constexpr uint32_t kObLabelMask = (1u << 24) - 1u;       // labels < 2^24 in the order keys

struct ObCounters {
  uint32_t box[6];            // order-preserving bits of min x, y, z (atomicMin) and max x, y, z (atomicMax)
  int runs;                   // occupied cells
  int next;                   // work counter of the pair kernel
  int clusters, objects, obj_points, largest_dropped;
};

__device__ __forceinline__ uint32_t ob_order(float x) {
  const uint32_t u = __float_as_uint(x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float ob_unorder(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

// the pair formula of section 1.7: (dx dx + dy dy) + dz dz in fp32, nothing contracted
__device__ __forceinline__ float ob_d2(float dx, float dy, float dz) {
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

__device__ __forceinline__ float ob_pair_d2(float4 p, float4 q) {
  return ob_d2(__fsub_rn(p.x, q.x), __fsub_rn(p.y, q.y), __fsub_rn(p.z, q.z));
}

// the grid from the bounding box: lo per axis and 1 / h, in fp64
struct ObGrid {
  double lo[3];
  double scale;
};

__device__ __forceinline__ ObGrid ob_grid(const ObCounters* ctr, float e) {
  ObGrid g;
  double ext = 0.0;
  for (int a = 0; a < 3; a++) {
    g.lo[a] = (double)ob_unorder(ctr->box[a]);
    ext = fmax(ext, (double)ob_unorder(ctr->box[3 + a]) - g.lo[a]);
  }
  const double h = fmax((double)e * (1.0 + 1e-5) / kObReach, ext / (double)(1 << 20));
  g.scale = 1.0 / h;
  return g;
}

__device__ __forceinline__ uint32_t ob_cell1(float x, double lo, double scale) {
  const double u = floor(((double)x - lo) * scale);
  return (uint32_t)fmin(fmax(u, 0.0), (double)kObAxisMask);
}

// ---------------------------------------------------------------- union-find (ECL-CC)

__device__ __forceinline__ int ob_find(int* parent, int x) {
  volatile int* p = parent;
  int cur = p[x];
  if (cur != x) {
    int next, prev = x;
    while (cur > (next = p[cur])) {
      p[prev] = next;   // path halving: every write lowers a parent to one of its ancestors
      prev = cur;
      cur = next;
    }
  }
  return cur;
}

// the root of x without writing: the final pass stores each label once, and a concurrent path-halving write could
// otherwise replace a stored root with an intermediate ancestor
__device__ __forceinline__ int ob_root(const int* parent, int x) {
  const volatile int* p = parent;
  int cur = x, next;
  while (cur > (next = p[cur])) cur = next;
  return cur;
}

__device__ __forceinline__ void ob_unite(int* parent, int a, int b) {
  int ra = ob_find(parent, a), rb = ob_find(parent, b);
  while (ra != rb) {
    if (ra < rb) {
      const int ret = atomicCAS(parent + rb, rb, ra);
      if (ret == rb) break;
      rb = ret;
    } else {
      const int ret = atomicCAS(parent + ra, ra, rb);
      if (ret == ra) break;
      ra = ret;
    }
  }
}

// ---------------------------------------------------------------- (a) grid

__global__ void objects_box_kernel(const float* __restrict__ xyz, int n, ObCounters* __restrict__ ctr) {
  uint32_t mn[3] = {~0u, ~0u, ~0u}, mx[3] = {0u, 0u, 0u};
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    for (int a = 0; a < 3; a++) {
      const uint32_t k = ob_order(xyz[3 * (size_t)i + a]);
      mn[a] = min(mn[a], k);
      mx[a] = max(mx[a], k);
    }
  for (int a = 0; a < 3; a++) {
    mn[a] = __reduce_min_sync(0xffffffffu, mn[a]);
    mx[a] = __reduce_max_sync(0xffffffffu, mx[a]);
  }
  if ((threadIdx.x & 31) == 0) {
    for (int a = 0; a < 3; a++) {
      atomicMin(ctr->box + a, mn[a]);
      atomicMax(ctr->box + 3 + a, mx[a]);
    }
  }
}

__global__ void objects_key_kernel(const float* __restrict__ xyz, int n, float e, const ObCounters* __restrict__ ctr,
                                   unsigned long long* __restrict__ key, int* __restrict__ val) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const ObGrid g = ob_grid(ctr, e);
  const float* p = xyz + 3 * (size_t)i;
  const unsigned long long cx = ob_cell1(p[0], g.lo[0], g.scale), cy = ob_cell1(p[1], g.lo[1], g.scale),
                           cz = ob_cell1(p[2], g.lo[2], g.scale);
  key[i] = (cx << (2 * kObAxisBits)) | (cy << kObAxisBits) | cz;
  val[i] = i;
}

__global__ void objects_gather_kernel(const float* __restrict__ xyz, int n, const int* __restrict__ val,
                                      float4* __restrict__ sorted) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const int i = val[s];
  const float* p = xyz + 3 * (size_t)i;
  sorted[s] = make_float4(p[0], p[1], p[2], __int_as_float(i));
}

// ---------------------------------------------------------------- (b) union

// one warp per cell (grid-stride): its exact point box (boxes[2 c], boxes[2 c + 1]); a clique iff the box's extents
// pass the pair formula, which then holds for every pair inside (each fp32 step is monotone in |dx|, |dy|, |dz|).
// parent of every point: the cell's first index (the lowest: the sort is stable) for a clique, itself otherwise.
__global__ void objects_cell_kernel(const float4* __restrict__ sorted, const int* __restrict__ start,
                                    const ObCounters* __restrict__ ctr, float e2, float4* __restrict__ boxes,
                                    uint8_t* __restrict__ clique, int* __restrict__ parent) {
  const int lane = threadIdx.x & 31;
  const int runs = ctr->runs;
  for (int c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; c < runs; c += (gridDim.x * blockDim.x) >> 5) {
    const int s0 = start[c], s1 = start[c + 1];
    float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
    for (int s = s0 + lane; s < s1; s += 32) {
      const float4 p = sorted[s];
      lo[0] = fminf(lo[0], p.x), lo[1] = fminf(lo[1], p.y), lo[2] = fminf(lo[2], p.z);
      hi[0] = fmaxf(hi[0], p.x), hi[1] = fmaxf(hi[1], p.y), hi[2] = fmaxf(hi[2], p.z);
    }
    for (int off = 16; off; off >>= 1)
      for (int a = 0; a < 3; a++) {
        lo[a] = fminf(lo[a], __shfl_xor_sync(0xffffffffu, lo[a], off));
        hi[a] = fmaxf(hi[a], __shfl_xor_sync(0xffffffffu, hi[a], off));
      }
    const bool cl = ob_d2(__fsub_rn(hi[0], lo[0]), __fsub_rn(hi[1], lo[1]), __fsub_rn(hi[2], lo[2])) <= e2;
    const int first = __float_as_int(sorted[s0].w);
    for (int s = s0 + lane; s < s1; s += 32) {
      const int i = __float_as_int(sorted[s].w);
      parent[i] = cl ? first : i;
    }
    if (lane == 0) {
      boxes[2 * (size_t)c] = make_float4(lo[0], lo[1], lo[2], 0.0f);
      boxes[2 * (size_t)c + 1] = make_float4(hi[0], hi[1], hi[2], 0.0f);
      clique[c] = cl ? 1 : 0;
    }
  }
}

// The warp tests the point pairs of cells [a0, a1) x [b0, b1) (same: one cell, pairs i < j only).  Lanes cover rows of
// w = min(nb, 32) columns, 32 / w rows per step.  With `cliques` both cells are cliques: the first pair within e2
// joins them and ends the test, which also ends when another warp has joined them already.  Otherwise every pair
// within e2 is united.  Warp-uniform control flow throughout.
__device__ void ob_test_pairs(const float4* __restrict__ sorted, int a0, int a1, int b0, int b1, bool same, bool cliques,
                              int rep_a, int rep_b, float e2, int* parent, int lane) {
  const int na = a1 - a0, nb = b1 - b0;
  const int w = min(nb, 32), rows = 32 / w, row = lane / w, col = lane % w;
  const int sweeps = (nb + w - 1) / w;
  for (int i0 = 0, step = 0; i0 < na; i0 += rows, step++) {
    if (cliques && step && (step & 63) == 0) {  // every 64 steps: stop if another warp has joined the two cells;
      int joined = 0;                           // lane 0 decides for the whole warp
      if (lane == 0) joined = ob_find(parent, rep_a) == ob_find(parent, rep_b);
      if (__shfl_sync(0xffffffffu, joined, 0)) return;
    }
    const int i = i0 + row;
    const bool row_ok = row < rows && i < na;
    const float4 p = row_ok ? sorted[a0 + i] : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    for (int k = 0; k < sweeps; k++) {
      const int j = col + k * w;
      bool hit = false;
      float4 q;
      if (row_ok && j < nb && (!same || j > i)) {
        q = sorted[b0 + j];
        hit = ob_pair_d2(p, q) <= e2;
      }
      if (cliques) {
        if (__any_sync(0xffffffffu, hit)) {
          if (lane == 0) ob_unite(parent, rep_a, rep_b);
          return;
        }
      } else if (hit) {
        ob_unite(parent, __float_as_int(p.w), __float_as_int(q.w));
      }
    }
  }
}

// one warp per occupied cell A, taken from a work counter: A's own pairs unless it is a clique, then the cells after
// it in the 5^3 neighbourhood (lane o < 62 looks up offset o by binary search among the cells after A)
__global__ void objects_pair_kernel(const float4* __restrict__ sorted, const unsigned long long* __restrict__ ukey,
                                    const int* __restrict__ start, const float4* __restrict__ boxes,
                                    const uint8_t* __restrict__ clique, ObCounters* __restrict__ ctr, float e2,
                                    int* __restrict__ parent) {
  const int lane = threadIdx.x & 31;
  const int runs = ctr->runs;
  for (;;) {
    int A = 0;
    if (lane == 0) A = atomicAdd(&ctr->next, 1);
    A = __shfl_sync(0xffffffffu, A, 0);
    if (A >= runs) return;
    const int a0 = start[A], a1 = start[A + 1];
    const bool cl_a = clique[A];
    const int rep_a = __float_as_int(sorted[a0].w);
    if (!cl_a) ob_test_pairs(sorted, a0, a1, a0, a1, true, false, rep_a, rep_a, e2, parent, lane);
    const unsigned long long ka = ukey[A];
    const int cx = (int)(ka >> (2 * kObAxisBits)), cy = (int)((ka >> kObAxisBits) & kObAxisMask),
              cz = (int)(ka & kObAxisMask);
    const float4 alo = boxes[2 * (size_t)A], ahi = boxes[2 * (size_t)A + 1];
    for (int base = 0; base < kObForward; base += 32) {
      const int o = base + lane;
      int B = -1;
      bool need = false;
      if (o < kObForward) {
        const int t = 63 + o;  // index in the 5^3 block; 62 is the centre, and index order is key order
        const int x = cx + t / 25 - kObReach, y = cy + (t / 5) % 5 - kObReach, z = cz + t % 5 - kObReach;
        if (x >= 0 && y >= 0 && z >= 0 && x <= (int)kObAxisMask && y <= (int)kObAxisMask && z <= (int)kObAxisMask) {
          const unsigned long long kb = ((unsigned long long)x << (2 * kObAxisBits)) |
                                        ((unsigned long long)y << kObAxisBits) | (unsigned long long)z;
          int lo = A + 1, hi = runs;
          while (lo < hi) {
            const int mid = (lo + hi) >> 1;
            if (ukey[mid] < kb) lo = mid + 1;
            else hi = mid;
          }
          if (lo < runs && ukey[lo] == kb) B = lo;
        }
      }
      if (B >= 0) {
        const float4 blo = boxes[2 * (size_t)B], bhi = boxes[2 * (size_t)B + 1];
        // the least gap per axis bounds every pair's d^2 from below
        const float gx = fmaxf(fmaxf(__fsub_rn(blo.x, ahi.x), __fsub_rn(alo.x, bhi.x)), 0.0f);
        const float gy = fmaxf(fmaxf(__fsub_rn(blo.y, ahi.y), __fsub_rn(alo.y, bhi.y)), 0.0f);
        const float gz = fmaxf(fmaxf(__fsub_rn(blo.z, ahi.z), __fsub_rn(alo.z, bhi.z)), 0.0f);
        if (ob_d2(gx, gy, gz) > e2) {
          B = -1;
        } else if (cl_a && clique[B]) {
          const int rep_b = __float_as_int(sorted[start[B]].w);
          if (ob_find(parent, rep_a) == ob_find(parent, rep_b)) B = -1;
          else need = true;
        } else {
          need = true;
        }
      }
      unsigned pend = __ballot_sync(0xffffffffu, need);
      while (pend) {
        const int src = __ffs(pend) - 1;
        pend &= pend - 1;
        const int b = __shfl_sync(0xffffffffu, B, src);
        const int b0 = start[b], b1 = start[b + 1];
        const bool both = cl_a && clique[b];
        ob_test_pairs(sorted, a0, a1, b0, b1, false, both, rep_a, __float_as_int(sorted[b0].w), e2, parent, lane);
      }
    }
  }
}

// labels[i] = the root of i (the component minimum); size[root] += 1 by warp-aggregated atomics; clusters counted
__global__ void objects_label_kernel(int n, int* __restrict__ labels, int* __restrict__ size,
                                     ObCounters* __restrict__ ctr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool in = i < n;
  const int r = in ? ob_root(labels, i) : -1;
  if (in) labels[i] = r;
  const unsigned act = __ballot_sync(0xffffffffu, in);
  if (!in) return;
  const unsigned peers = __match_any_sync(act, r);
  if ((threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(size + r, __popc(peers));
  const unsigned roots = __ballot_sync(act, r == i);
  if ((threadIdx.x & 31) == __ffs(act) - 1 && roots) atomicAdd(&ctr->clusters, __popc(roots));
}

// ---------------------------------------------------------------- (c) order and selection

// key[i] = size << 24 | (2^24 - 1 - i) for a root i, 0 otherwise; the object and dropped-cluster counts
__global__ void objects_order_key_kernel(int n, int min_points, const int* __restrict__ labels,
                                         const int* __restrict__ size, ObCounters* __restrict__ ctr,
                                         unsigned long long* __restrict__ key) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  int s = 0;
  if (i < n) {
    s = labels[i] == i ? size[i] : 0;
    key[i] = s ? ((unsigned long long)s << 24) | (kObLabelMask - (uint32_t)i) : 0ull;
  }
  const bool obj = s >= min_points;
  const unsigned objs = __ballot_sync(0xffffffffu, obj);
  const unsigned pts = __reduce_add_sync(0xffffffffu, obj ? (unsigned)s : 0u);
  const unsigned big = __reduce_max_sync(0xffffffffu, obj ? 0u : (unsigned)s);
  if ((threadIdx.x & 31) == 0) {
    if (objs) {
      atomicAdd(&ctr->objects, __popc(objs));
      atomicAdd(&ctr->obj_points, (int)pts);
    }
    if (big) atomicMax(&ctr->largest_dropped, (int)big);
  }
}

// the clusters in order: rank_of[label] = k; objsize[k] = its size for the objects (the first ctr->objects)
__global__ void objects_rank_kernel(int n, const unsigned long long* __restrict__ key,
                                    const ObCounters* __restrict__ ctr, int* __restrict__ rank_of,
                                    int64_t* __restrict__ objsize) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const unsigned long long kk = key[k];
  if (!kk) return;
  rank_of[kObLabelMask - (uint32_t)(kk & kObLabelMask)] = k;
  if (k < ctr->objects) objsize[k] = (int64_t)(kk >> 24);
}

// the object of every point (its rank), or `none` past every object, keyed for the stable sort by object
__global__ void objects_select_key_kernel(int n, uint32_t none, const int* __restrict__ labels,
                                          const int* __restrict__ rank_of, const ObCounters* __restrict__ ctr,
                                          uint32_t* __restrict__ key, int64_t* __restrict__ val) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int r = rank_of[labels[i]];
  key[i] = r < ctr->objects ? (uint32_t)r : none;
  val[i] = i;
}

// stats = (clusters, objects, points in objects, dropped clusters, points in dropped clusters, largest dropped)
__global__ void objects_finish_kernel(int n, const ObCounters* __restrict__ ctr, int64_t* __restrict__ stats) {
  if (threadIdx.x != 0) return;
  stats[0] = ctr->clusters;
  stats[1] = ctr->objects;
  stats[2] = ctr->obj_points;
  stats[3] = ctr->clusters - ctr->objects;
  stats[4] = n - ctr->obj_points;
  stats[5] = ctr->largest_dropped;
}

// ---------------------------------------------------------------- workspace

static bool ob_shape_ok(int n, int min_points) { return n >= 1 && n <= kObMaxN && min_points >= 1 && min_points <= n; }
static int ob_max_objects(int n, int min_points) { return n / min_points; }

// bits of the object keys: ranks 0 .. max_objects - 1 and `none` = max_objects
static int ob_select_bits(int max_objects) {
  int b = 1;
  while ((1ll << b) <= (long long)max_objects) b++;
  return b;
}

static size_t ob_cub_bytes(int n, int max_objects) {
  size_t b = 0, t = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, t, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                  (const int*)nullptr, (int*)nullptr, n, 0, 3 * kObAxisBits);
  b = std::max(b, t);
  cub::DeviceRunLengthEncode::Encode(nullptr, t, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                     (int*)nullptr, (int*)nullptr, n);
  b = std::max(b, t);
  cub::DeviceScan::ExclusiveSum(nullptr, t, (const int*)nullptr, (int*)nullptr, n + 1);
  b = std::max(b, t);
  cub::DeviceRadixSort::SortKeysDescending(nullptr, t, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                           n, 0, 49);
  b = std::max(b, t);
  cub::DeviceScan::ExclusiveSum(nullptr, t, (const int64_t*)nullptr, (int64_t*)nullptr, max_objects + 1);
  b = std::max(b, t);
  cub::DeviceRadixSort::SortPairs(nullptr, t, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const int64_t*)nullptr,
                                  (int64_t*)nullptr, n, 0, ob_select_bits(max_objects));
  return std::max(b, t);
}

struct ObBuffers {
  ObCounters* ctr;
  unsigned long long *key_a, *key_b;
  int *val_a, *val_b;
  unsigned long long* ukey;
  int *runlen, *start;
  float4 *sorted, *boxes;
  uint8_t* clique;
  int *size, *rank_of;
  int64_t* objsize;
  uint32_t *okey_a, *okey_b;
  int64_t* oval;
  void* cub;
  size_t cub_bytes, total;
};

static ObBuffers ob_buffers(int n, int min_points, void* ws) {
  const int mo = ob_max_objects(n, min_points);
  Carver c(ws);
  ObBuffers b;
  b.ctr = c.take<ObCounters>(1);
  b.key_a = c.take<unsigned long long>(n);
  b.key_b = c.take<unsigned long long>(n);
  b.val_a = c.take<int>(n);
  b.val_b = c.take<int>(n);
  b.ukey = c.take<unsigned long long>(n);
  b.runlen = c.take<int>((size_t)n + 1);
  b.start = c.take<int>((size_t)n + 1);
  b.sorted = c.take<float4>(n);
  b.boxes = c.take<float4>(2 * (size_t)n);
  b.clique = c.take<uint8_t>(n);
  b.size = c.take<int>(n);
  b.rank_of = c.take<int>(n);
  b.objsize = c.take<int64_t>((size_t)mo + 1);
  b.okey_a = c.take<uint32_t>(n);
  b.okey_b = c.take<uint32_t>(n);
  b.oval = c.take<int64_t>(n);
  b.cub_bytes = ob_cub_bytes(n, mo);
  b.cub = c.take<char>(b.cub_bytes);
  b.total = c.total;
  return b;
}

static StageEvents<4> ob_events;

// CTAs of the warp-per-cell kernels: 8 per SM, no more than one warp per point
static int ob_warp_blocks(int n) { return std::max(1, std::min(8 * sm_count(), blocks((size_t)n * 32, kObThreads))); }

}  // namespace ma

using namespace ma;

extern "C" {

size_t ma_split_objects_workspace_bytes(int n, int min_points) {
  if (!ob_shape_ok(n, min_points)) return 0;
  return ob_buffers(n, min_points, nullptr).total;
}

void ma_split_objects_set_events(void* const* events) { ob_events.set(events); }

int ma_split_objects(const float* xyz, int n, float e, int min_points, int32_t* labels_out, int64_t* indices_out,
                     int64_t* offsets_out, int64_t* stats_out, void* ws, void* stream) {
  const float e2 = e * e;
  if (!xyz || !labels_out || !indices_out || !offsets_out || !stats_out || !ws || !ob_shape_ok(n, min_points) ||
      !(e > 0.0f && e <= 1.0f) || !(e2 > 0.0f)) {
    set_error("ma_split_objects: bad arguments (1 <= n <= 2^24, 1 <= min_points <= n, 0 < e <= 1, e * e > 0 in fp32)");
    return 1;
  }
  cudaStream_t st = (cudaStream_t)stream;
  const ObBuffers b = ob_buffers(n, min_points, ws);
  const int mo = ob_max_objects(n, min_points), wblocks = ob_warp_blocks(n), nb = blocks(n, kObThreads);
  size_t tb = b.cub_bytes;

  ob_events.mark(0, st);
  cudaError_t e_ = cudaMemsetAsync(b.ctr, 0, sizeof(ObCounters), st);
  if (e_ == cudaSuccess) e_ = cudaMemsetAsync(b.ctr->box, 0xff, 3 * sizeof(uint32_t), st);
  if (e_ == cudaSuccess) e_ = cudaMemsetAsync(b.runlen, 0, (size_t)(n + 1) * 4, st);
  if (e_ == cudaSuccess) e_ = cudaMemsetAsync(b.size, 0, (size_t)n * 4, st);
  if (e_ == cudaSuccess) e_ = cudaMemsetAsync(b.objsize, 0, (size_t)(mo + 1) * 8, st);
  objects_box_kernel<<<std::min(nb, 1024), kObThreads, 0, st>>>(xyz, n, b.ctr);
  objects_key_kernel<<<nb, kObThreads, 0, st>>>(xyz, n, e, b.ctr, b.key_a, b.val_a);
  count_launch(2);
  if (e_ == cudaSuccess)
    e_ = cub::DeviceRadixSort::SortPairs(b.cub, tb, b.key_a, b.key_b, b.val_a, b.val_b, n, 0, 3 * kObAxisBits, st);
  tb = b.cub_bytes;
  if (e_ == cudaSuccess)
    e_ = cub::DeviceRunLengthEncode::Encode(b.cub, tb, b.key_b, b.ukey, b.runlen, &b.ctr->runs, n, st);
  tb = b.cub_bytes;
  if (e_ == cudaSuccess) e_ = cub::DeviceScan::ExclusiveSum(b.cub, tb, b.runlen, b.start, n + 1, st);
  objects_gather_kernel<<<nb, kObThreads, 0, st>>>(xyz, n, b.val_b, b.sorted);
  count_launch(1);
  ob_events.mark(1, st);
  objects_cell_kernel<<<wblocks, kObThreads, 0, st>>>(b.sorted, b.start, b.ctr, e2, b.boxes, b.clique, labels_out);
  objects_pair_kernel<<<wblocks, kObThreads, 0, st>>>(b.sorted, b.ukey, b.start, b.boxes, b.clique, b.ctr, e2,
                                                      labels_out);
  objects_label_kernel<<<nb, kObThreads, 0, st>>>(n, labels_out, b.size, b.ctr);
  count_launch(3);
  ob_events.mark(2, st);
  objects_order_key_kernel<<<nb, kObThreads, 0, st>>>(n, min_points, labels_out, b.size, b.ctr, b.key_a);
  count_launch(1);
  tb = b.cub_bytes;
  if (e_ == cudaSuccess) e_ = cub::DeviceRadixSort::SortKeysDescending(b.cub, tb, b.key_a, b.key_b, n, 0, 49, st);
  objects_rank_kernel<<<nb, kObThreads, 0, st>>>(n, b.key_b, b.ctr, b.rank_of, b.objsize);
  count_launch(1);
  tb = b.cub_bytes;
  if (e_ == cudaSuccess) e_ = cub::DeviceScan::ExclusiveSum(b.cub, tb, b.objsize, offsets_out, mo + 1, st);
  objects_select_key_kernel<<<nb, kObThreads, 0, st>>>(n, (uint32_t)mo, labels_out, b.rank_of, b.ctr, b.okey_a,
                                                       b.oval);
  count_launch(1);
  tb = b.cub_bytes;
  if (e_ == cudaSuccess)
    e_ = cub::DeviceRadixSort::SortPairs(b.cub, tb, b.okey_a, b.okey_b, b.oval, indices_out, n, 0, ob_select_bits(mo),
                                         st);
  objects_finish_kernel<<<1, 32, 0, st>>>(n, b.ctr, stats_out);
  count_launch(1);
  ob_events.mark(3, st);
  return stage_status("ma_split_objects", e_);
}

}  // extern "C"
