// jacobi3.cuh -- eigenvectors of a symmetric 3x3 matrix by a fixed cyclic Jacobi (DESIGN.md section 1.2), shared by
// the per-point PCA of normals.cu, the plane refit of plane.cu and the local frame of smooth.cu.  Every fp64 step is an
// explicit round-to-nearest intrinsic (nvcc contracts fp64 as well), so tests/normals_oracle.py (jacobi,
// smallest_vector) restates it bit for bit.
#pragma once

namespace ma {

constexpr int kJacobiSweeps = 5;   // cyclic sweeps: 4 reach 4e-15 rad against LAPACK on separated spectra, 1 spare

// c = (xx, xy, xz, yy, yz, zz) -> the diagonal d and V (eigenvectors in its columns) after kJacobiSweeps sweeps over
// the pairs (0,1), (0,2), (1,2)
__device__ __forceinline__ void jacobi3(const double c[6], double d[3], double V[3][3]) {
  double A[3][3] = {{c[0], c[1], c[2]}, {c[1], c[3], c[4]}, {c[2], c[4], c[5]}};
#pragma unroll
  for (int a = 0; a < 3; a++)
#pragma unroll
    for (int b = 0; b < 3; b++) V[a][b] = a == b ? 1.0 : 0.0;
  for (int sweep = 0; sweep < kJacobiSweeps; sweep++) {
#pragma unroll
    for (int pr = 0; pr < 3; pr++) {
      const int p = pr == 2 ? 1 : 0, q = pr == 0 ? 1 : 2, r = 2 - pr;
      const double apq = A[p][q];
      if (apq == 0.0) continue;
      const double app = A[p][p], aqq = A[q][q];
      const double theta = __ddiv_rn(__dsub_rn(aqq, app), __dmul_rn(2.0, apq));
      double t = __ddiv_rn(1.0, __dadd_rn(fabs(theta), __dsqrt_rn(__dadd_rn(__dmul_rn(theta, theta), 1.0))));
      if (theta < 0.0) t = -t;
      const double cs = __ddiv_rn(1.0, __dsqrt_rn(__dadd_rn(__dmul_rn(t, t), 1.0)));
      const double sn = __dmul_rn(t, cs);
      const double tapq = __dmul_rn(t, apq);
      const double arp = A[r][p], arq = A[r][q];
      A[p][p] = __dsub_rn(app, tapq);
      A[q][q] = __dadd_rn(aqq, tapq);
      A[p][q] = A[q][p] = 0.0;
      A[r][p] = A[p][r] = __dsub_rn(__dmul_rn(cs, arp), __dmul_rn(sn, arq));
      A[r][q] = A[q][r] = __dadd_rn(__dmul_rn(sn, arp), __dmul_rn(cs, arq));
#pragma unroll
      for (int row = 0; row < 3; row++) {
        const double vp = V[row][p], vq = V[row][q];
        V[row][p] = __dsub_rn(__dmul_rn(cs, vp), __dmul_rn(sn, vq));
        V[row][q] = __dadd_rn(__dmul_rn(sn, vp), __dmul_rn(cs, vq));
      }
    }
  }
  d[0] = A[0][0];
  d[1] = A[1][1];
  d[2] = A[2][2];
}

// the column of V of the smallest diagonal entry (the lowest column on ties)
__device__ __forceinline__ int jacobi3_smallest_column(const double d[3]) {
  int m = 0;
  double dmin = d[0];
  if (d[1] < dmin) { m = 1; dmin = d[1]; }
  if (d[2] < dmin) m = 2;
  return m;
}

// (x, y, z) divided by its fp64 length
__device__ __forceinline__ void jacobi3_unit(double x, double y, double z, double v[3]) {
  const double ln = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, x), __dmul_rn(y, y)), __dmul_rn(z, z)));
  v[0] = __ddiv_rn(x, ln);
  v[1] = __ddiv_rn(y, ln);
  v[2] = __ddiv_rn(z, ln);
}

// c -> v: the column of V of the smallest diagonal entry (the lowest column on ties), divided by its fp64 length
__device__ __forceinline__ void jacobi3_smallest(const double c[6], double v[3]) {
  double d[3], V[3][3];
  jacobi3(c, d, V);
  double v0 = V[0][0], v1 = V[1][0], v2 = V[2][0], dmin = d[0];
  if (d[1] < dmin) { v0 = V[0][1]; v1 = V[1][1]; v2 = V[2][1]; dmin = d[1]; }
  if (d[2] < dmin) { v0 = V[0][2]; v1 = V[1][2]; v2 = V[2][2]; }
  jacobi3_unit(v0, v1, v2, v);
}

}  // namespace ma
