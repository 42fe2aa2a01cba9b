// smooth.cu -- moving-least-squares smoothing of a point cloud for `--smooth` (DESIGN.md section 1.8 defines it).
//
// The points arrive already in the output frame (p' = (p - c) / L, metrics.to_output_frame), fp32 [N][3].
//   (a) grid      knn_bin (knn_grid.cuh): the points in cell order on a G^3 grid over [-0.5, 0.5]^3.
//   (b) kNN       knn_grid_kernel<false> (knn_grid.cuh): the exact kNN of section 1.2, self excluded.
//   (c) fit       smooth_fit_kernel, one thread per point, walking the points in cell order (neighbouring threads
//                 gather neighbouring rows): fp64 weights (1 - d^2 / H)^2 with H = 2 d^2 of the last neighbour, the
//                 weighted centroid and covariance, the cyclic Jacobi of jacobi3.cuh for the local frame (n, t1, t2),
//                 the weighted least-squares height field z = a . (1, u, v, u^2, uv, v^2) over (u, v) scaled by
//                 h = sqrt(H), solved by a 6x6 Cholesky in a fixed row order, and the projection of the point onto it.
//                 A Cholesky pivot at or below kSmPivot of M_00 = sum w, or a projection that moves the point by
//                 more than h, falls back to the projection onto the weighted plane.  Each warp adds its counts of the
//                 three outcomes with one integer atomic each.
// Every fp64 step is an explicit round-to-nearest intrinsic (nvcc contracts fp64 as well) and every sum runs in a fixed
// order, so a call is bit-deterministic and tests/smooth_oracle.py restates the neighbours, the normals, the flags and
// the points bit for bit.
#include "canon.cuh"
#include "jacobi3.cuh"
#include "knn_grid.cuh"
#include "workspace.h"

namespace ma {

constexpr int kSmThreads = 128;     // fit threads per CTA: at 130 registers, 3 CTAs (12 warps) fit on an SM
constexpr int kSmMaxN = 1 << 24;    // the index part of a kNN key and the cap shared by every point-cloud stage
constexpr int kSmMinK = 5;          // the quadratic has 6 coefficients: the point and at least 5 neighbours
constexpr double kSmPivot = 1e-9;   // Cholesky pivot threshold of the singular fallback, times M_00 (smooth_oracle.PIVOT)

enum SmFlag : int { kSmQuadratic = 0, kSmSingular = 1, kSmFar = 2 };

__device__ __forceinline__ double sm_dot(double ax, double ay, double az, double bx, double by, double bz) {
  return __dadd_rn(__dadd_rn(__dmul_rn(ax, bx), __dmul_rn(ay, by)), __dmul_rn(az, bz));
}

// (1 - d2 / H)^2; 1 when H == 0
__device__ __forceinline__ double sm_weight(double d2, double H) {
  if (H == 0.0) return 1.0;
  const double t = __dsub_rn(1.0, __ddiv_rn(d2, H));
  return __dmul_rn(t, t);
}

// (dx dx + dy dy) + dz dz in fp64 between fp32 points a and b
__device__ __forceinline__ double sm_d2(const float* a, const float* b) {
  const double dx = __dsub_rn((double)b[0], (double)a[0]), dy = __dsub_rn((double)b[1], (double)a[1]),
               dz = __dsub_rn((double)b[2], (double)a[2]);
  return sm_dot(dx, dy, dz, dx, dy, dz);
}

// column c of V divided by its fp64 length (selects, so that V stays in registers)
__device__ __forceinline__ void sm_column(const double V[3][3], int c, double v[3]) {
  double x[3];
#pragma unroll
  for (int a = 0; a < 3; a++) x[a] = c == 0 ? V[a][0] : (c == 1 ? V[a][1] : V[a][2]);
  jacobi3_unit(x[0], x[1], x[2], v);
}

constexpr int sm_tri(int a, int b) { return a * (a + 1) / 2 + b; }   // entry (a, b), b <= a, of a packed 6x6

// Smooths point i: q (fp64, before rounding), the unit normal n of its local frame, and the outcome.
__device__ __forceinline__ int smooth_point(const float* __restrict__ xyz, const int32_t* __restrict__ nb, int i, int k,
                                            double q[3], double n[3]) {
  const float* pi = xyz + 3 * (size_t)i;
  const double H = __dmul_rn(2.0, sm_d2(pi, xyz + 3 * (size_t)nb[k - 1]));
  // weighted centroid: the point itself (w = 1), then the neighbours in rank order
  double sw = 0.0, sx = 0.0, sy = 0.0, sz = 0.0;
  for (int e = -1; e < k; e++) {
    const float* pj = e < 0 ? pi : xyz + 3 * (size_t)nb[e];
    const double w = e < 0 ? 1.0 : sm_weight(sm_d2(pi, pj), H);
    sw = __dadd_rn(sw, w);
    sx = __dadd_rn(sx, __dmul_rn(w, (double)pj[0]));
    sy = __dadd_rn(sy, __dmul_rn(w, (double)pj[1]));
    sz = __dadd_rn(sz, __dmul_rn(w, (double)pj[2]));
  }
  const double mx = __ddiv_rn(sx, sw), my = __ddiv_rn(sy, sw), mz = __ddiv_rn(sz, sw);
  // weighted covariance, entries w (d_a d_b)
  double c[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int e = -1; e < k; e++) {
    const float* pj = e < 0 ? pi : xyz + 3 * (size_t)nb[e];
    const double w = e < 0 ? 1.0 : sm_weight(sm_d2(pi, pj), H);
    const double dx = __dsub_rn((double)pj[0], mx), dy = __dsub_rn((double)pj[1], my),
                 dz = __dsub_rn((double)pj[2], mz);
    c[0] = __dadd_rn(c[0], __dmul_rn(w, __dmul_rn(dx, dx)));
    c[1] = __dadd_rn(c[1], __dmul_rn(w, __dmul_rn(dx, dy)));
    c[2] = __dadd_rn(c[2], __dmul_rn(w, __dmul_rn(dx, dz)));
    c[3] = __dadd_rn(c[3], __dmul_rn(w, __dmul_rn(dy, dy)));
    c[4] = __dadd_rn(c[4], __dmul_rn(w, __dmul_rn(dy, dz)));
    c[5] = __dadd_rn(c[5], __dmul_rn(w, __dmul_rn(dz, dz)));
  }
  double d[3], V[3][3];
  jacobi3(c, d, V);
  const int cn = jacobi3_smallest_column(d);
  const int c1 = cn == 0 ? 1 : 0, c2 = cn == 2 ? 1 : 2;
  double t1[3], t2[3];
  sm_column(V, cn, n);
  sm_column(V, c1, t1);
  sm_column(V, c2, t2);
  const double px = pi[0], py = pi[1], pz = pi[2];
  bool ok = H != 0.0;   // all k + 1 points coincide: nothing to fit
  if (ok) {
    // normal equations M = sum w phi phi^T (lower triangle, row-major) and b = sum w phi z
    const double h = __dsqrt_rn(H);
    double M[21], b[6], up = 0.0, vp = 0.0;
#pragma unroll
    for (int a = 0; a < 21; a++) M[a] = 0.0;
#pragma unroll
    for (int a = 0; a < 6; a++) b[a] = 0.0;
    for (int e = -1; e < k; e++) {
      const float* pj = e < 0 ? pi : xyz + 3 * (size_t)nb[e];
      const double w = e < 0 ? 1.0 : sm_weight(sm_d2(pi, pj), H);
      const double rx = __dsub_rn((double)pj[0], mx), ry = __dsub_rn((double)pj[1], my),
                   rz = __dsub_rn((double)pj[2], mz);
      const double u = __ddiv_rn(sm_dot(rx, ry, rz, t1[0], t1[1], t1[2]), h);
      const double v = __ddiv_rn(sm_dot(rx, ry, rz, t2[0], t2[1], t2[2]), h);
      const double z = sm_dot(rx, ry, rz, n[0], n[1], n[2]);
      if (e < 0) {
        up = u;
        vp = v;
      }
      const double phi[6] = {1.0, u, v, __dmul_rn(u, u), __dmul_rn(u, v), __dmul_rn(v, v)};
#pragma unroll
      for (int a = 0; a < 6; a++) {
        const double wa = __dmul_rn(w, phi[a]);
#pragma unroll
        for (int c = 0; c <= a; c++) M[sm_tri(a, c)] = __dadd_rn(M[sm_tri(a, c)], __dmul_rn(wa, phi[c]));
        b[a] = __dadd_rn(b[a], __dmul_rn(wa, z));
      }
    }
    // Cholesky M = L L^T in place, row by row; a pivot at or below kSmPivot M_00 (the weight mass) is singular
    const double pivot_min = __dmul_rn(kSmPivot, M[0]);
#pragma unroll
    for (int a = 0; a < 6; a++) {
#pragma unroll
      for (int c = 0; c <= a; c++) {
        double s = M[sm_tri(a, c)];
#pragma unroll
        for (int t = 0; t < c; t++) s = __dsub_rn(s, __dmul_rn(M[sm_tri(a, t)], M[sm_tri(c, t)]));
        if (c == a) {
          if (!(s > pivot_min)) ok = false;
          M[sm_tri(a, a)] = __dsqrt_rn(s);
        } else {
          M[sm_tri(a, c)] = __ddiv_rn(s, M[sm_tri(c, c)]);
        }
      }
    }
    if (ok) {
      // L y = b, then L^T x = y, in place in b
#pragma unroll
      for (int a = 0; a < 6; a++) {
        double s = b[a];
#pragma unroll
        for (int t = 0; t < a; t++) s = __dsub_rn(s, __dmul_rn(M[sm_tri(a, t)], b[t]));
        b[a] = __ddiv_rn(s, M[sm_tri(a, a)]);
      }
#pragma unroll
      for (int a = 5; a >= 0; a--) {
        double s = b[a];
#pragma unroll
        for (int t = a + 1; t < 6; t++) s = __dsub_rn(s, __dmul_rn(M[sm_tri(t, a)], b[t]));
        b[a] = __ddiv_rn(s, M[sm_tri(a, a)]);
      }
      const double phi[6] = {1.0, up, vp, __dmul_rn(up, up), __dmul_rn(up, vp), __dmul_rn(vp, vp)};
      double z = __dmul_rn(b[0], phi[0]);
#pragma unroll
      for (int a = 1; a < 6; a++) z = __dadd_rn(z, __dmul_rn(b[a], phi[a]));
      const double uh = __dmul_rn(up, h), vh = __dmul_rn(vp, h);
#pragma unroll
      for (int a = 0; a < 3; a++) {
        const double m = a == 0 ? mx : (a == 1 ? my : mz);
        q[a] = __dadd_rn(__dadd_rn(__dadd_rn(m, __dmul_rn(uh, t1[a])), __dmul_rn(vh, t2[a])), __dmul_rn(z, n[a]));
      }
      const double ex = __dsub_rn(q[0], px), ey = __dsub_rn(q[1], py), ez = __dsub_rn(q[2], pz);
      if (!(sm_dot(ex, ey, ez, ex, ey, ez) > H)) return kSmQuadratic;
    }
  }
  // the weighted plane: q = p - ((p - m) . n) n
  const double s = sm_dot(__dsub_rn(px, mx), __dsub_rn(py, my), __dsub_rn(pz, mz), n[0], n[1], n[2]);
  q[0] = __dsub_rn(px, __dmul_rn(s, n[0]));
  q[1] = __dsub_rn(py, __dmul_rn(s, n[1]));
  q[2] = __dsub_rn(pz, __dmul_rn(s, n[2]));
  return ok ? kSmFar : kSmSingular;
}

// kCellOrder: thread s smooths the point in slot s of the cell-sorted copy; otherwise point s
template <bool kCellOrder>
__global__ void __launch_bounds__(kSmThreads)
    smooth_fit_kernel(const float* __restrict__ xyz, const float4* __restrict__ sorted, const int32_t* __restrict__ knn,
                      int n, int k, float* __restrict__ out, float* __restrict__ normal_out,
                      uint8_t* __restrict__ flag_out, unsigned long long* __restrict__ counts) {
  const int s = blockIdx.x * kSmThreads + threadIdx.x;
  int flag = -1;
  if (s < n) {
    const int i = kCellOrder ? __float_as_int(sorted[s].w) : s;
    double q[3], nv[3];
    flag = smooth_point(xyz, knn + (size_t)i * k, i, k, q, nv);
    out[3 * (size_t)i] = (float)q[0];
    out[3 * (size_t)i + 1] = (float)q[1];
    out[3 * (size_t)i + 2] = (float)q[2];
    if (normal_out) {
      normal_out[3 * (size_t)i] = (float)nv[0];
      normal_out[3 * (size_t)i + 1] = (float)nv[1];
      normal_out[3 * (size_t)i + 2] = (float)nv[2];
    }
    if (flag_out) flag_out[i] = (uint8_t)flag;
  }
  // one integer atomic per warp and outcome: the counts do not depend on the schedule
#pragma unroll
  for (int f = 0; f < 3; f++) {
    const unsigned m = __ballot_sync(0xffffffffu, flag == f);
    if ((threadIdx.x & 31) == 0 && m) atomicAdd(counts + f, (unsigned long long)__popc(m));
  }
}

// ---------------------------------------------------------------- workspace

static bool sm_shape_ok(int n, int k) { return k >= kSmMinK && k <= kKnnMaxK && n > k && n <= kSmMaxN; }

struct SmBuffers {
  float4* sorted;
  uint32_t *cell, *count, *start;
  void* scan;
  size_t scan_bytes;
  int32_t* knn;
  size_t total;
};

static SmBuffers sm_buffers(int n, int k, void* ws) {
  const int G = knn_frame_grid(n, k).G;
  const size_t cells = (size_t)G * G * G;
  Carver c(ws);
  SmBuffers b;
  b.sorted = c.take<float4>(n);
  b.cell = c.take<uint32_t>(n);
  b.count = c.take<uint32_t>(cells + 1);
  b.start = c.take<uint32_t>(cells + 1);
  b.scan_bytes = knn_bin_scan_bytes(cells);
  b.scan = c.take<char>(b.scan_bytes);
  b.knn = c.take<int32_t>((size_t)n * k);
  b.total = c.total;
  return b;
}

static StageEvents<4> sm_events;
static bool g_sm_cell_order = true;

}  // namespace ma

using namespace ma;

extern "C" {

size_t ma_smooth_points_workspace_bytes(int n, int k) {
  if (!sm_shape_ok(n, k)) return 0;
  return sm_buffers(n, k, nullptr).total;
}

void ma_smooth_points_set_events(void* const* events) { sm_events.set(events); }

void ma_smooth_points_set_order(int cell_order) { g_sm_cell_order = cell_order != 0; }

int ma_smooth_points(const float* xyz, int n, int k, float* out_xyz, float* normal_out, uint8_t* flag_out,
                     int32_t* knn_out, int64_t* stats_out, void* ws, void* stream) {
  if (!xyz || !out_xyz || !stats_out || !ws || !sm_shape_ok(n, k)) {
    set_error("ma_smooth_points: bad arguments (%d <= k <= %d, k < n <= 2^24)", kSmMinK, kKnnMaxK);
    return 1;
  }
  const char* what = "ma_smooth_points";
  cudaStream_t st = (cudaStream_t)stream;
  SmBuffers b = sm_buffers(n, k, ws);
  if (knn_out) b.knn = knn_out;
  const KnnGrid grid = knn_frame_grid(n, k);

  sm_events.mark(0, st);
  cudaError_t e = cudaMemsetAsync(stats_out, 0, 3 * sizeof(int64_t), st);
  if (e == cudaSuccess) e = knn_bin(xyz, n, grid, b.cell, b.count, b.start, b.sorted, b.scan, b.scan_bytes, st);
  if (e != cudaSuccess) return stage_status(what, e);
  count_launch(3);
  sm_events.mark(1, st);
  knn_grid_kernel<false><<<(n + kKnnThreads - 1) / kKnnThreads, kKnnThreads,
                           (size_t)k * kKnnThreads * sizeof(unsigned long long), st>>>(b.sorted, b.start, n, k, grid, 0,
                                                                                       nullptr, nullptr, b.knn, nullptr);
  sm_events.mark(2, st);
  unsigned long long* counts = reinterpret_cast<unsigned long long*>(stats_out);
  if (g_sm_cell_order)
    smooth_fit_kernel<true><<<blocks(n, kSmThreads), kSmThreads, 0, st>>>(xyz, b.sorted, b.knn, n, k, out_xyz,
                                                                          normal_out, flag_out, counts);
  else
    smooth_fit_kernel<false><<<blocks(n, kSmThreads), kSmThreads, 0, st>>>(xyz, b.sorted, b.knn, n, k, out_xyz,
                                                                           normal_out, flag_out, counts);
  count_launch(2);
  sm_events.mark(3, st);
  return stage_status(what, e);
}

}  // extern "C"
