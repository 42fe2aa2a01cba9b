// surface.cu -- mesh -> point cloud on the GPU: area-weighted surface sampling with face normals.
//
// Replaces `trimesh.Trimesh.sample(count, return_index=True)` + `mesh.face_normals[idx]` of the reference's
// pre-processing (/root/reference/mesh_to_pc.py:42-57): a face is drawn with probability proportional to its area
// (inverse CDF over the cumulative areas), a point uniformly inside it (two uniforms, reflected into the triangle --
// what trimesh.sample.sample_surface does), and the face's unit normal is appended.  Output fp16 [n][6], the dtype the
// reference feeds the encoder (np.float16, mesh_to_pc.py:53).  The random stream is Philox4x32-10 keyed by
// (seed, sample), not numpy's Mersenne twister: same distribution, different individual points.
#include "canon.cuh"
#include "internal.h"
#include "philox.cuh"

namespace ma {

// three uniforms in [0,1) for sample i
__device__ __forceinline__ float3 sf_philox3(unsigned long long seed, uint32_t i) {
  const uint4 c = philox4x32_10(i, 0x53555246u, 0x4d455348u, 0x414e5954u, seed);
  const float s = 1.0f / 16777216.0f;
  return make_float3((float)(c.x >> 8) * s, (float)(c.y >> 8) * s, (float)(c.z >> 8) * s);
}

__device__ __forceinline__ float3 sf_vertex(const float* v, int i) { return make_float3(v[3 * i], v[3 * i + 1], v[3 * i + 2]); }

// area[f] (double: the cumulative sum of up to millions of faces must stay monotone and exact enough for the search).
// Here and in surface_sample_kernel every operation carries an explicit rounding, so nvcc contracts nothing and the
// numpy restatement (tests/surface_oracle.py) reproduces the bits: DESIGN.md section 1.5.
__global__ void surface_area_kernel(const float* __restrict__ v, const int32_t* __restrict__ faces, int F, double* __restrict__ area) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const float3 a = sf_vertex(v, faces[3 * f]), b = sf_vertex(v, faces[3 * f + 1]), c = sf_vertex(v, faces[3 * f + 2]);
  const double ux = __dsub_rn(b.x, a.x), uy = __dsub_rn(b.y, a.y), uz = __dsub_rn(b.z, a.z);
  const double wx = __dsub_rn(c.x, a.x), wy = __dsub_rn(c.y, a.y), wz = __dsub_rn(c.z, a.z);
  const double nx = __dsub_rn(__dmul_rn(uy, wz), __dmul_rn(uz, wy));
  const double ny = __dsub_rn(__dmul_rn(uz, wx), __dmul_rn(ux, wz));
  const double nz = __dsub_rn(__dmul_rn(ux, wy), __dmul_rn(uy, wx));
  const double s = __dadd_rn(__dadd_rn(__dmul_rn(nx, nx), __dmul_rn(ny, ny)), __dmul_rn(nz, nz));
  area[f] = __dmul_rn(0.5, __dsqrt_rn(s));
}

// in-place inclusive scan by ONE CTA of 1024 threads walking the array in tiles (F is at most a few million), followed
// by a running maximum over the faces of positive area.  The Hillis-Steele sums alone are not monotone: two neighbours
// are summed in different orders, so the cumulative area can step down by an ulp, or up by one across a face of zero
// area, which the search below would then pick.  The maximum is exact and order-free: cum[i] = max over j <= i with
// area[j] > 0 of the sum up to j (0 before the first such face).  So cum never decreases, and a face of zero area has
// cum[i] = cum[i - 1]: it is never drawn.
__global__ void __launch_bounds__(1024) surface_scan_kernel(double* __restrict__ a, int F) {
  __shared__ double wsum[32], wmax[32];
  __shared__ double carry, mcarry;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) carry = mcarry = 0.0;
  __syncthreads();
  for (int base = 0; base < F; base += 1024) {
    const int i = base + tid;
    const double v = i < F ? a[i] : 0.0;
    double x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const double y = __shfl_up_sync(0xffffffffu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) wsum[warp] = x;
    __syncthreads();
    if (warp == 0) {
      double s = wsum[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const double y = __shfl_up_sync(0xffffffffu, s, o);
        if (lane >= o) s += y;
      }
      wsum[lane] = s;
    }
    __syncthreads();
    const double off = carry + (warp ? wsum[warp - 1] : 0.0);
    const double sum = x + off;
    double m = v > 0.0 ? sum : 0.0;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) m = fmax(m, __shfl_up_sync(0xffffffffu, m, o));  // lanes < o get their own m back
    if (lane == 31) wmax[warp] = m;
    __syncthreads();
    if (warp == 0) {
      double s = wmax[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) s = fmax(s, __shfl_up_sync(0xffffffffu, s, o));
      wmax[lane] = s;
    }
    __syncthreads();
    m = fmax(m, fmax(mcarry, warp ? wmax[warp - 1] : 0.0));
    if (i < F) a[i] = m;
    __syncthreads();
    if (tid == 1023) { carry = sum; mcarry = m; }
    __syncthreads();
  }
}

__global__ void surface_sample_kernel(const float* __restrict__ v, const int32_t* __restrict__ faces, int F,
                                      const double* __restrict__ cum, int n, unsigned long long seed,
                                      __half* __restrict__ out, int32_t* __restrict__ face_idx) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float3 u = sf_philox3(seed, (uint32_t)i);
  const double target = (double)u.x * cum[F - 1];
  int lo = 0, hi = F - 1;                       // first face whose cumulative area exceeds the target
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (cum[mid] > target) hi = mid; else lo = mid + 1;
  }
  const int f = lo;
  const float3 a = sf_vertex(v, faces[3 * f]), b = sf_vertex(v, faces[3 * f + 1]), c = sf_vertex(v, faces[3 * f + 2]);
  float r1 = u.y, r2 = u.z;
  if (fadd(r1, r2) > 1.0f) { r1 = fsub(1.0f, r1); r2 = fsub(1.0f, r2); }
  const float ux = fsub(b.x, a.x), uy = fsub(b.y, a.y), uz = fsub(b.z, a.z);
  const float wx = fsub(c.x, a.x), wy = fsub(c.y, a.y), wz = fsub(c.z, a.z);
  const float px = fadd(fadd(a.x, fmul(r1, ux)), fmul(r2, wx));
  const float py = fadd(fadd(a.y, fmul(r1, uy)), fmul(r2, wy));
  const float pz = fadd(fadd(a.z, fmul(r1, uz)), fmul(r2, wz));
  const float nx = fsub(fmul(uy, wz), fmul(uz, wy)), ny = fsub(fmul(uz, wx), fmul(ux, wz));
  const float nz = fsub(fmul(ux, wy), fmul(uy, wx));
  const float ln = __fsqrt_rn(fadd(fadd(fmul(nx, nx), fmul(ny, ny)), fmul(nz, nz)));
  const float inv = ln > 0.0f ? __fdiv_rn(1.0f, ln) : 1.0f;
  __half* o = out + (size_t)i * 6;
  o[0] = __float2half_rn(px); o[1] = __float2half_rn(py); o[2] = __float2half_rn(pz);
  o[3] = __float2half_rn(fmul(nx, inv)); o[4] = __float2half_rn(fmul(ny, inv)); o[5] = __float2half_rn(fmul(nz, inv));
  if (face_idx) face_idx[i] = f;
}

}  // namespace ma

using namespace ma;

extern "C" {

size_t ma_sample_surface_workspace_bytes(int n_faces) { return (size_t)(n_faces > 0 ? n_faces : 1) * sizeof(double) + 256; }

int ma_sample_surface(const float* vertices, const int32_t* faces, int n_faces, int n_samples, unsigned long long seed,
                      void* out_pc_normal, int32_t* out_face_idx, void* ws, void* stream) {
  if (!vertices || !faces || !out_pc_normal || !ws || n_faces <= 0 || n_samples <= 0) {
    set_error("ma_sample_surface: bad arguments");
    return 1;
  }
  cudaStream_t st = (cudaStream_t)stream;
  double* cum = reinterpret_cast<double*>(ws);
  surface_area_kernel<<<(n_faces + 255) / 256, 256, 0, st>>>(vertices, faces, n_faces, cum);
  surface_scan_kernel<<<1, 1024, 0, st>>>(cum, n_faces);
  surface_sample_kernel<<<(n_samples + 255) / 256, 256, 0, st>>>(vertices, faces, n_faces, cum, n_samples, seed,
                                                                  reinterpret_cast<__half*>(out_pc_normal), out_face_idx);
  count_launch(3);
  return check_launch("ma_sample_surface") ? 0 : 1;
}

}  // extern "C"
