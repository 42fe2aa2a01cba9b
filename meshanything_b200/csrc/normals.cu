// normals.cu -- oriented normals of a bare point cloud for `--input_type pc` (DESIGN.md section 1.2 defines them).
//
// The points arrive already in the output frame (p' = (p - c) / L, metrics.to_output_frame), fp32 [N][3].
//   (a) grid      knn_cell_kernel / knn_scatter_kernel (knn_grid.cuh) sort the points into a G^3 grid over
//                 [-0.5, 0.5]^3 (lo = -0.5, scale = G), a CUB exclusive scan giving the cell starts.
//   (b) kNN       knn_grid_kernel (knn_grid.cuh), one thread per point, shells of cells until the k-th key's d^2 is
//                 below the bound of the next shell, without a shell budget: the exact kNN.
//   (c) PCA       normals_pca_kernel, one thread per point: fp64 centroid and covariance of the point and its
//                 neighbours in rank order, sequential sums of explicit __d*_rn operations, then the cyclic Jacobi
//                 of jacobi3.cuh; the eigenvector of the smallest diagonal entry, normalised in fp64, rounded to fp32.
//   (d) orient    Boruvka over the kNN graph.  Each vertex carries a word (component root << 1 | parity), the parity
//                 being its sign relative to that root.  A round: every component's minimum outgoing edge under the
//                 strict order (w, min(i,j), max(i,j)) by two 64/32-bit atomicMin passes over unique keys; each
//                 component hooks onto the component across that edge (of a mutual pair the larger root hooks) with
//                 parity = parity(x) ^ parity(y) ^ (u_x . u_y < 0); pointer jumping on single 32-bit words composes
//                 parities by XOR; every vertex is relabelled.  One 4-byte read-back per round (the number of hooks)
//                 decides whether another round runs.  Finally the point of largest |p'|^2 (lowest index on ties) of
//                 each component fixes the component's sign.
// Every fp32 step is an explicit round-to-nearest intrinsic, every fp64 step too (nvcc contracts fp64 as well), and
// every choice is a minimum over unique keys, so a call is bit-deterministic and tests/normals_oracle.py restates the
// neighbours, the unoriented and the oriented normals bit for bit.
#include "canon.cuh"
#include "jacobi3.cuh"
#include "knn_grid.cuh"
#include "workspace.h"

namespace ma {

constexpr int kNmThreads = 256;
constexpr int kNmMaxN = 1 << 24;    // vertex words hold the root in 31 bits; the index part of a kNN key in 32
constexpr int kNmMaxRounds = 64;    // Boruvka at least halves the components with an outgoing edge per round

__device__ __forceinline__ float nm_dot(float ax, float ay, float az, float bx, float by, float bz) {
  return __fadd_rn(__fadd_rn(__fmul_rn(ax, bx), __fmul_rn(ay, by)), __fmul_rn(az, bz));
}

// ---------------------------------------------------------------- (c) PCA + Jacobi

__global__ void normals_pca_kernel(const float* __restrict__ xyz, const int32_t* __restrict__ knn, int n, int k,
                                   float* __restrict__ uno) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int32_t* nb = knn + (size_t)i * k;
  const float* pi = xyz + 3 * (size_t)i;
  double sx = pi[0], sy = pi[1], sz = pi[2];
  for (int e = 0; e < k; e++) {
    const float* pj = xyz + 3 * (size_t)nb[e];
    sx = __dadd_rn(sx, (double)pj[0]);
    sy = __dadd_rn(sy, (double)pj[1]);
    sz = __dadd_rn(sz, (double)pj[2]);
  }
  const double cnt = (double)(k + 1);
  const double mx = __ddiv_rn(sx, cnt), my = __ddiv_rn(sy, cnt), mz = __ddiv_rn(sz, cnt);
  double c[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int e = -1; e < k; e++) {
    const float* pj = e < 0 ? pi : xyz + 3 * (size_t)nb[e];
    const double dx = __dsub_rn((double)pj[0], mx), dy = __dsub_rn((double)pj[1], my), dz = __dsub_rn((double)pj[2], mz);
    const double t[6] = {__dmul_rn(dx, dx), __dmul_rn(dx, dy), __dmul_rn(dx, dz),
                         __dmul_rn(dy, dy), __dmul_rn(dy, dz), __dmul_rn(dz, dz)};
    if (e < 0) {
#pragma unroll
      for (int a = 0; a < 6; a++) c[a] = t[a];
    } else {
#pragma unroll
      for (int a = 0; a < 6; a++) c[a] = __dadd_rn(c[a], t[a]);
    }
  }
  double v[3];
  jacobi3_smallest(c, v);
  float* o = uno + 3 * (size_t)i;
  o[0] = (float)v[0];
  o[1] = (float)v[1];
  o[2] = (float)v[2];
}

// ---------------------------------------------------------------- (d) orientation

constexpr uint32_t kNmDead = 0xffffffffu;  // weight bits of a kNN slot whose endpoints share a component for good

// w[slot] = bits of max(0, 1 - |u_i . u_j|); word[i] = i << 1 (own root, parity 0)
__global__ void normals_weight_kernel(const float* __restrict__ uno, const int32_t* __restrict__ knn, int n, int k,
                                      uint32_t* __restrict__ w, uint32_t* __restrict__ word) {
  const size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (e >= (size_t)n * k) return;
  const int i = (int)(e / k), j = knn[e];
  const float* a = uno + 3 * (size_t)i;
  const float* b = uno + 3 * (size_t)j;
  const float d = nm_dot(a[0], a[1], a[2], b[0], b[1], b[2]);
  w[e] = __float_as_uint(fmaxf(0.0f, __fsub_rn(1.0f, fabsf(d))));
  if (e % k == 0) word[i] = (uint32_t)i << 1;
}

__global__ void normals_clear_kernel(int n, unsigned long long* __restrict__ best1, uint32_t* __restrict__ best2) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  best1[i] = ~0ull;
  best2[i] = ~0u;
}

// pass 1: per component the least (w, min(i,j)) over its outgoing slots; slots found internal are marked dead
__global__ void normals_min1_kernel(const int32_t* __restrict__ knn, int n, int k, uint32_t* __restrict__ w,
                                    const uint32_t* __restrict__ word, unsigned long long* __restrict__ best1) {
  const size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (e >= (size_t)n * k) return;
  const uint32_t wb = w[e];
  if (wb == kNmDead) return;
  const uint32_t i = (uint32_t)(e / k), j = (uint32_t)knn[e];
  const uint32_t ci = word[i] >> 1, cj = word[j] >> 1;
  if (ci == cj) {
    w[e] = kNmDead;
    return;
  }
  const unsigned long long key = ((unsigned long long)wb << 32) | min(i, j);
  atomicMin(best1 + ci, key);
  atomicMin(best1 + cj, key);
}

// pass 2: among the slots that carry the winning (w, min) key, the least max(i,j)
__global__ void normals_min2_kernel(const int32_t* __restrict__ knn, int n, int k, const uint32_t* __restrict__ w,
                                    const uint32_t* __restrict__ word, const unsigned long long* __restrict__ best1,
                                    uint32_t* __restrict__ best2) {
  const size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (e >= (size_t)n * k) return;
  const uint32_t wb = w[e];
  if (wb == kNmDead) return;
  const uint32_t i = (uint32_t)(e / k), j = (uint32_t)knn[e];
  const uint32_t ci = word[i] >> 1, cj = word[j] >> 1;
  const unsigned long long key = ((unsigned long long)wb << 32) | min(i, j);
  if (key == best1[ci]) atomicMin(best2 + ci, max(i, j));
  if (key == best1[cj]) atomicMin(best2 + cj, max(i, j));
}

// per root c: hook[c] = (new parent << 1) | parity of c relative to it; hook[c] = c << 1 when c stays a root
__global__ void normals_hook_kernel(const float* __restrict__ uno, int n, const uint32_t* __restrict__ word,
                                    const unsigned long long* __restrict__ best1, const uint32_t* __restrict__ best2,
                                    uint32_t* __restrict__ hook, int* __restrict__ hooks) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= (uint32_t)n || (word[c] >> 1) != c) return;
  const unsigned long long b1 = best1[c];
  if (b1 == ~0ull) {
    hook[c] = c << 1;
    return;
  }
  const uint32_t a = (uint32_t)b1, b = best2[c];
  const uint32_t x = (word[a] >> 1) == c ? a : b, y = x == a ? b : a;
  const uint32_t d = word[y] >> 1;
  if (best1[d] == b1 && best2[d] == b && c < d) {  // both chose this edge: the smaller root stays
    hook[c] = c << 1;
    return;
  }
  const float* ux = uno + 3 * (size_t)x;
  const float* uy = uno + 3 * (size_t)y;
  const uint32_t flip = nm_dot(ux[0], ux[1], ux[2], uy[0], uy[1], uy[2]) < 0.0f ? 1u : 0u;
  hook[c] = (d << 1) | ((word[x] ^ word[y] ^ flip) & 1u);
  atomicAdd(hooks, 1);
}

// pointer jumping over the hook forest.  Each root only writes its own word, and any word it reads is a valid
// (ancestor, parity relative to it) pair, old or new: the result does not depend on the schedule.
__global__ void normals_jump_kernel(int n, const uint32_t* __restrict__ word, uint32_t* hook) {
  const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= (uint32_t)n || (word[c] >> 1) != c) return;
  volatile uint32_t* h = hook;
  uint32_t w = h[c];
  for (;;) {
    const uint32_t p = w >> 1, wp = h[p];
    if ((wp >> 1) == p) break;
    w = (wp & ~1u) | ((w ^ wp) & 1u);
    h[c] = w;
  }
}

__global__ void normals_relabel_kernel(int n, const uint32_t* __restrict__ hook, uint32_t* __restrict__ word) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n) return;
  const uint32_t w = word[v], r = hook[w >> 1];
  word[v] = (r & ~1u) | ((w ^ r) & 1u);
}

// per component the point of largest fp32 |p|^2, lowest index on ties: max of (bits << 32 | ~index)
__global__ void normals_far_kernel(const float* __restrict__ xyz, int n, const uint32_t* __restrict__ word,
                                   unsigned long long* __restrict__ far) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n) return;
  const float* p = xyz + 3 * (size_t)v;
  const float r2 = nm_dot(p[0], p[1], p[2], p[0], p[1], p[2]);
  atomicMax(far + (word[v] >> 1), ((unsigned long long)__float_as_uint(r2) << 32) | (uint32_t)~(uint32_t)v);
}

__global__ void normals_apply_kernel(const float* __restrict__ xyz, const float* __restrict__ uno, int n,
                                     const uint32_t* __restrict__ word, const unsigned long long* __restrict__ far,
                                     float* __restrict__ out) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= n) return;
  const uint32_t wv = word[v];
  const uint32_t f = ~(uint32_t)far[wv >> 1];
  const float* uf = uno + 3 * (size_t)f;
  const float* pf = xyz + 3 * (size_t)f;
  const uint32_t neg = nm_dot(uf[0], uf[1], uf[2], pf[0], pf[1], pf[2]) < 0.0f ? 1u : 0u;
  const bool flip = ((neg ^ word[f] ^ wv) & 1u) != 0;
  const float* u = uno + 3 * (size_t)v;
  out[3 * (size_t)v] = flip ? -u[0] : u[0];
  out[3 * (size_t)v + 1] = flip ? -u[1] : u[1];
  out[3 * (size_t)v + 2] = flip ? -u[2] : u[2];
}

// ---------------------------------------------------------------- workspace

static bool nm_shape_ok(int n, int k) { return k >= 1 && k <= kKnnMaxK && n > k && n <= kNmMaxN; }

struct NmBuffers {
  float4* sorted;
  uint32_t *cell, *count, *start;
  void* scan;
  size_t scan_bytes;
  int32_t* knn;
  float* uno;
  uint32_t *w, *word, *hook;
  unsigned long long* best1;
  uint32_t* best2;
  int* hooks;
  size_t total;
};

static NmBuffers nm_buffers(int n, int k, void* ws) {
  const int G = knn_frame_grid(n, k).G;
  const size_t cells = (size_t)G * G * G, nk = (size_t)n * k;
  Carver c(ws);
  NmBuffers b;
  b.sorted = c.take<float4>(n);
  b.cell = c.take<uint32_t>(n);
  b.count = c.take<uint32_t>(cells + 1);
  b.start = c.take<uint32_t>(cells + 1);
  b.scan_bytes = knn_bin_scan_bytes(cells);
  b.scan = c.take<char>(b.scan_bytes);
  b.knn = c.take<int32_t>(nk);
  b.uno = c.take<float>(3 * (size_t)n);
  b.w = c.take<uint32_t>(nk);
  b.word = c.take<uint32_t>(n);
  b.hook = c.take<uint32_t>(n);
  b.best1 = c.take<unsigned long long>(n);
  b.best2 = c.take<uint32_t>(n);
  b.hooks = c.take<int>(1);
  b.total = c.total;
  return b;
}

static StageEvents<5> nm_events;
static int g_nm_rounds = 0;

}  // namespace ma

using namespace ma;

extern "C" {

size_t ma_estimate_normals_workspace_bytes(int n, int k) {
  if (!nm_shape_ok(n, k)) return 0;
  return nm_buffers(n, k, nullptr).total;
}

void ma_estimate_normals_set_events(void* const* events) { nm_events.set(events); }

int ma_estimate_normals_last_rounds(void) { return g_nm_rounds; }

int ma_estimate_normals(const float* xyz, int n, int k, float* normals_out, int32_t* knn_out, float* unoriented_out,
                        void* ws, void* stream) {
  if (!xyz || !normals_out || !ws || !nm_shape_ok(n, k)) {
    set_error("ma_estimate_normals: bad arguments (1 <= k <= %d, k < n <= 2^24)", kKnnMaxK);
    return 1;
  }
  const char* what = "ma_estimate_normals";
  cudaStream_t st = (cudaStream_t)stream;
  NmBuffers b = nm_buffers(n, k, ws);
  if (knn_out) b.knn = knn_out;
  if (unoriented_out) b.uno = unoriented_out;
  const KnnGrid grid = knn_frame_grid(n, k);
  const size_t nk = (size_t)n * k;

  nm_events.mark(0, st);
  cudaError_t e = knn_bin(xyz, n, grid, b.cell, b.count, b.start, b.sorted, b.scan, b.scan_bytes, st);
  if (e != cudaSuccess) return stage_status(what, e);
  count_launch(3);
  nm_events.mark(1, st);
  knn_grid_kernel<false><<<(n + kKnnThreads - 1) / kKnnThreads, kKnnThreads,
                           (size_t)k * kKnnThreads * sizeof(unsigned long long), st>>>(b.sorted, b.start, n, k, grid, 0,
                                                                                       nullptr, nullptr, b.knn, nullptr);
  nm_events.mark(2, st);
  normals_pca_kernel<<<blocks(n, kNmThreads), kNmThreads, 0, st>>>(xyz, b.knn, n, k, b.uno);
  nm_events.mark(3, st);
  normals_weight_kernel<<<blocks(nk, kNmThreads), kNmThreads, 0, st>>>(b.uno, b.knn, n, k, b.w, b.word);
  count_launch(3);
  if (stage_status(what, e)) return 1;
  int rounds = 0;
  for (;;) {
    if (rounds == kNmMaxRounds) {
      set_error("ma_estimate_normals: Boruvka did not finish in %d rounds", kNmMaxRounds);
      return 1;
    }
    rounds++;
    int merged = 0;
    e = cudaMemsetAsync(b.hooks, 0, sizeof(int), st);
    normals_clear_kernel<<<blocks(n, kNmThreads), kNmThreads, 0, st>>>(n, b.best1, b.best2);
    normals_min1_kernel<<<blocks(nk, kNmThreads), kNmThreads, 0, st>>>(b.knn, n, k, b.w, b.word, b.best1);
    normals_min2_kernel<<<blocks(nk, kNmThreads), kNmThreads, 0, st>>>(b.knn, n, k, b.w, b.word, b.best1, b.best2);
    normals_hook_kernel<<<blocks(n, kNmThreads), kNmThreads, 0, st>>>(b.uno, n, b.word, b.best1, b.best2, b.hook,
                                                                      b.hooks);
    normals_jump_kernel<<<blocks(n, kNmThreads), kNmThreads, 0, st>>>(n, b.word, b.hook);
    normals_relabel_kernel<<<blocks(n, kNmThreads), kNmThreads, 0, st>>>(n, b.hook, b.word);
    count_launch(6);
    if (e == cudaSuccess) e = cudaMemcpyAsync(&merged, b.hooks, sizeof(int), cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    if (stage_status(what, e)) return 1;
    if (merged == 0) break;
  }
  g_nm_rounds = rounds;
  // the last round hooked nothing, so best1 is free again: it collects each component's farthest point
  e = cudaMemsetAsync(b.best1, 0, (size_t)n * 8, st);
  normals_far_kernel<<<blocks(n, kNmThreads), kNmThreads, 0, st>>>(xyz, n, b.word, b.best1);
  normals_apply_kernel<<<blocks(n, kNmThreads), kNmThreads, 0, st>>>(xyz, b.uno, n, b.word, b.best1, normals_out);
  count_launch(2);
  nm_events.mark(4, st);
  return stage_status(what, e);
}

}  // extern "C"
