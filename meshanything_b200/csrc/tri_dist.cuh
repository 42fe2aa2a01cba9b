// tri_dist.cuh -- the fixed fp32 point-triangle distance shared by watertight.cu (distance field of `--mc`),
// mesh_score.cu (Chamfer scoring of generated meshes) and colors.cu (`--transfer_colors`), and the barycentric weights
// of the nearest point that colors.cu adds.
//
// Every operation is an explicit round-to-nearest intrinsic, so nvcc cannot contract or reorder it and numpy restates
// it bit for bit (tests/watertight_oracle.py: tri_dist).  wt_tri_prep holds the per-face part of the formula, so that
// a kernel which evaluates one face against many points can compute it once; wt_tri_dist(p, wt_tri_prep(a, b, c)) and
// wt_tri_dist(p, a, b, c) are the same operations.
#pragma once

namespace ma {

struct wt_v3 { float x, y, z; };

__device__ __forceinline__ wt_v3 wt_sub(wt_v3 a, wt_v3 b) {
  return {__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y), __fsub_rn(a.z, b.z)};
}
__device__ __forceinline__ float wt_dot(wt_v3 a, wt_v3 b) {
  return __fadd_rn(__fadd_rn(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)), __fmul_rn(a.z, b.z));
}
__device__ __forceinline__ wt_v3 wt_cross(wt_v3 a, wt_v3 b) {
  return {__fsub_rn(__fmul_rn(a.y, b.z), __fmul_rn(a.z, b.y)), __fsub_rn(__fmul_rn(a.z, b.x), __fmul_rn(a.x, b.z)),
          __fsub_rn(__fmul_rn(a.x, b.y), __fmul_rn(a.y, b.x))};
}
// the parameter t in [0, 1] of the point of the segment [0, e] nearest to w (relative to the segment's start); 0 for a
// zero-length segment
__device__ __forceinline__ float wt_seg_t(wt_v3 w, wt_v3 e) {
  const float l = wt_dot(e, e);
  const float t = l > 0.0f ? __fdiv_rn(wt_dot(w, e), l) : 0.0f;
  return fminf(fmaxf(t, 0.0f), 1.0f);
}
// squared distance from w to the segment [0, e] at the parameter t of wt_seg_t
__device__ __forceinline__ float wt_seg2_at(wt_v3 w, wt_v3 e, float t) {
  const wt_v3 q = {__fsub_rn(w.x, __fmul_rn(t, e.x)), __fsub_rn(w.y, __fmul_rn(t, e.y)), __fsub_rn(w.z, __fmul_rn(t, e.z))};
  return wt_dot(q, q);
}
// squared distance from the point w (relative to the segment's start) to the segment [0, e]; a zero-length segment is
// its point
__device__ __forceinline__ float wt_seg2(wt_v3 w, wt_v3 e) { return wt_seg2_at(w, e, wt_seg_t(w, e)); }

// Euclidean distance from p to the triangle (a, b, c), from p - a, p - b, p - c and the face terms: the plane distance
// when p projects inside the triangle (all three edge tests >= 0), else the nearest of the three edges.  A degenerate
// face (zero normal) is its segments.
__device__ __forceinline__ float wt_tri_dist_terms(wt_v3 ap, wt_v3 bp, wt_v3 cp, wt_v3 ab, wt_v3 bc, wt_v3 ca, wt_v3 nrm,
                                                   float nn) {
  if (nn > 0.0f && wt_dot(wt_cross(ab, ap), nrm) >= 0.0f && wt_dot(wt_cross(bc, bp), nrm) >= 0.0f &&
      wt_dot(wt_cross(ca, cp), nrm) >= 0.0f) {
    const float h = wt_dot(ap, nrm);
    return __fsqrt_rn(__fdiv_rn(__fmul_rn(h, h), nn));
  }
  const float d2 = fminf(fminf(wt_seg2(ap, ab), wt_seg2(bp, bc)), wt_seg2(cp, ca));
  return __fsqrt_rn(d2);
}

__device__ __forceinline__ float wt_tri_dist(wt_v3 p, wt_v3 a, wt_v3 b, wt_v3 c) {
  const wt_v3 ab = wt_sub(b, a), bc = wt_sub(c, b), ca = wt_sub(a, c);
  const wt_v3 ap = wt_sub(p, a), bp = wt_sub(p, b), cp = wt_sub(p, c);
  const wt_v3 nrm = wt_cross(ab, wt_sub(c, a));
  const float nn = wt_dot(nrm, nrm);
  return wt_tri_dist_terms(ap, bp, cp, ab, bc, ca, nrm, nn);
}

// the per-face terms of wt_tri_dist computed once, for a kernel that measures one face against many points
struct wt_tri { wt_v3 a, b, c, ab, bc, ca, nrm; float nn; };

__device__ __forceinline__ wt_tri wt_tri_prep(wt_v3 a, wt_v3 b, wt_v3 c) {
  wt_tri t;
  t.a = a; t.b = b; t.c = c;
  t.ab = wt_sub(b, a); t.bc = wt_sub(c, b); t.ca = wt_sub(a, c);
  t.nrm = wt_cross(t.ab, wt_sub(c, a));
  t.nn = wt_dot(t.nrm, t.nrm);
  return t;
}

__device__ __forceinline__ float wt_tri_dist(wt_v3 p, const wt_tri& t) {
  return wt_tri_dist_terms(wt_sub(p, t.a), wt_sub(p, t.b), wt_sub(p, t.c), t.ab, t.bc, t.ca, t.nrm, t.nn);
}

// Barycentric weights (w[0], w[1], w[2]) of a, b, c at the point of the face nearest to p, in the region
// wt_tri_dist_terms measures p in (DESIGN.md section 1.9): inside, the three edge tests, each the weight of the vertex
// opposite its edge, over their sum s = (e_ab + e_bc) + e_ca (s > 0 always holds there unless the tests underflow; s == 0
// takes the segments); otherwise the nearest of the segments ab, bc, ca (the first on ties) with (1 - t, t) on its two
// ends.  A degenerate face (zero normal) is its segments.  Every weight lies in [0, 1].
__device__ __forceinline__ void wt_tri_bary(wt_v3 p, const wt_tri& t, float w[3]) {
  const wt_v3 ap = wt_sub(p, t.a), bp = wt_sub(p, t.b), cp = wt_sub(p, t.c);
  if (t.nn > 0.0f) {
    const float eab = wt_dot(wt_cross(t.ab, ap), t.nrm), ebc = wt_dot(wt_cross(t.bc, bp), t.nrm),
                eca = wt_dot(wt_cross(t.ca, cp), t.nrm);
    const float s = __fadd_rn(__fadd_rn(eab, ebc), eca);
    if (eab >= 0.0f && ebc >= 0.0f && eca >= 0.0f && s > 0.0f) {
      w[0] = __fdiv_rn(ebc, s);
      w[1] = __fdiv_rn(eca, s);
      w[2] = __fdiv_rn(eab, s);
      return;
    }
  }
  const float tab = wt_seg_t(ap, t.ab), tbc = wt_seg_t(bp, t.bc), tca = wt_seg_t(cp, t.ca);
  const float dab = wt_seg2_at(ap, t.ab, tab), dbc = wt_seg2_at(bp, t.bc, tbc), dca = wt_seg2_at(cp, t.ca, tca);
  if (dab <= dbc && dab <= dca) {
    w[0] = __fsub_rn(1.0f, tab); w[1] = tab; w[2] = 0.0f;
  } else if (dbc <= dca) {
    w[0] = 0.0f; w[1] = __fsub_rn(1.0f, tbc); w[2] = tbc;
  } else {
    w[0] = tca; w[1] = 0.0f; w[2] = __fsub_rn(1.0f, tca);
  }
}

}  // namespace ma
