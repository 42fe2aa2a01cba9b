// jacobi3.cuh -- the eigenvector of the smallest eigenvalue of a symmetric 3x3 matrix by a fixed cyclic Jacobi
// (DESIGN.md section 1.2), shared by the per-point PCA of normals.cu and the plane refit of plane.cu.  Every fp64 step
// is an explicit round-to-nearest intrinsic (nvcc contracts fp64 as well), so tests/normals_oracle.py (jacobi,
// smallest_vector) restates it bit for bit.
#pragma once

namespace ma {

constexpr int kJacobiSweeps = 5;   // cyclic sweeps: 4 reach 4e-15 rad against LAPACK on separated spectra, 1 spare

// c = (xx, xy, xz, yy, yz, zz) -> v: after kJacobiSweeps sweeps over the pairs (0,1), (0,2), (1,2), the column of V of
// the smallest diagonal entry (the lowest column on ties), divided by its fp64 length
__device__ __forceinline__ void jacobi3_smallest(const double c[6], double v[3]) {
  double A[3][3] = {{c[0], c[1], c[2]}, {c[1], c[3], c[4]}, {c[2], c[4], c[5]}};
  double V[3][3] = {{1.0, 0.0, 0.0}, {0.0, 1.0, 0.0}, {0.0, 0.0, 1.0}};
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
  // the column of the smallest diagonal entry, the lowest column on ties
  double v0 = V[0][0], v1 = V[1][0], v2 = V[2][0], dmin = A[0][0];
  if (A[1][1] < dmin) { v0 = V[0][1]; v1 = V[1][1]; v2 = V[2][1]; dmin = A[1][1]; }
  if (A[2][2] < dmin) { v0 = V[0][2]; v1 = V[1][2]; v2 = V[2][2]; }
  const double ln = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(v0, v0), __dmul_rn(v1, v1)), __dmul_rn(v2, v2)));
  v[0] = __ddiv_rn(v0, ln);
  v[1] = __ddiv_rn(v1, ln);
  v[2] = __ddiv_rn(v2, ln);
}

}  // namespace ma
