// ghicp_device.cuh — device-side helpers shared by the translation units of libghicp_b200.so that evaluate
// the EXACT cost path (separately rounded IEEE operations in the reference's order) and the float32 Umeyama core.
// Include only from .cu files compiled with --fmad=false (see Makefile).
#pragma once
#include <cuda_fp16.h>

#include "ghicp_internal.h"

namespace ghicp_b200 {
namespace {

constexpr int TR = 8;              // source rows per CTA in the row sweeps
constexpr double MAXVALIUE = 9e20;  // initial mincd of the reference scans (src/ghicp_reg.cpp:618,711)

// ---------------------------------------------------------------------------------------------
// reductions
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int warp_sum_i(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// lexicographic (value, index) minimum: the reference keeps the FIRST minimum of an ascending scan
__device__ __forceinline__ void lexmin(double &v, int &i, double ov, int oi) {
  if (ov < v || (ov == v && oi < i)) { v = ov; i = oi; }
}
__device__ __forceinline__ void warp_lexmin(double &v, int &i) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    double ov = __shfl_xor_sync(0xffffffffu, v, o);
    int oi = __shfl_xor_sync(0xffffffffu, i, o);
    lexmin(v, i, ov, oi);
  }
}
// block-wide sum of K doubles with a fixed reduction tree (deterministic). Result valid in thread 0.
template <int K, int THREADS>
__device__ __forceinline__ void block_sum(double (&v)[K], double *smem /* [K][THREADS/32] */) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int NW = THREADS / 32;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    double w = warp_sum(v[k]);
    if (lane == 0) smem[k * NW + warp] = w;
  }
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int k = 0; k < K; ++k) {
      double w = (lane < NW) ? smem[k * NW + lane] : 0.0;
      w = warp_sum(w);
      v[k] = w;
    }
  }
  __syncthreads();
}

// The BSC feature-distance plane stores integer Hamming distances as IEEE half bits (exact for
// 0..2048): one HADD2.F32-class conversion per value on the streaming path instead of unpack + I2F.
__device__ __forceinline__ double h2d(unsigned int bits16) {
  return (double)__half2float(__ushort_as_half((unsigned short)bits16));
}

// ---------------------------------------------------------------------------------------------
// exact cost evaluation
// ---------------------------------------------------------------------------------------------
// EF.scale * sqrt(pow(dx,2) + pow(dy,2) + pow(dz,2))   (src/ghicp_reg.cpp:122)
__device__ __forceinline__ double ed_exact(double sx, double sy, double sz, double tx, double ty, double tz,
                                           double scale) {
  double dx = sx - tx, dy = sy - ty, dz = sz - tz;
  double d2 = (dx * dx + dy * dy) + dz * dz;
  return scale * sqrt(d2);
}
// FT: 0 = BSC, 2 = FPFH, 3 = None (enum order of include/utility.h:51-57)
template <int FT>
__device__ __forceinline__ double cd_exact(double ed, double fd, const CostParams &cp) {
  if (FT == GHICP_FT_BSC) return cp.WED * ed + cp.WFD * fd;             // src/ghicp_reg.cpp:259
  if (FT == GHICP_FT_FPFH) return 1.0 * ed / pow(fd, cp.ex);            // src/ghicp_reg.cpp:308
  return ed;                                                            // src/ghicp_reg.cpp:224
}

// ---------------------------------------------------------------------------------------------
// float32 3x3 SVD (one-sided Jacobi) and Umeyama from moments — PCL's
// TransformationEstimationSVD → Eigen::umeyama (no scaling) as called at src/ghicp_reg.cpp:857-866.
// A is first scaled by 2^-e, 2^e the power of two above its largest |entry| (JacobiSVD divides by the
// largest entry too): the sweep's alpha * beta then neither overflows (points spread over more than
// ~6e4 units) nor underflows, and every step commutes exactly with the power of two, so results are
// bit-identical to the unscaled sweep wherever that one stayed in range.  Zero or non-finite A: e = 0.
// ---------------------------------------------------------------------------------------------
__device__ void svd3_f32(const float A[9], float U[9], float S[3], float V[9]) {
  float amax = 0.f;
  bool finite = true;
  for (int i = 0; i < 9; ++i) { const float m = fabsf(A[i]); finite = finite && isfinite(m); amax = m > amax ? m : amax; }
  int e = 0;
  if (finite && amax > 0.f) frexpf(amax, &e);
  float a[9];
  for (int i = 0; i < 9; ++i) a[i] = ldexpf(A[i], -e);
  float v[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  const float tol = 1e-7f;
  for (int sweep = 0; sweep < 30; ++sweep) {
    int rotated = 0;
    for (int p = 0; p < 2; ++p) {
      for (int q = p + 1; q < 3; ++q) {
        float alpha = 0.f, beta = 0.f, gamma = 0.f;
        for (int i = 0; i < 3; ++i) {
          alpha = alpha + a[i * 3 + p] * a[i * 3 + p];
          beta = beta + a[i * 3 + q] * a[i * 3 + q];
          gamma = gamma + a[i * 3 + p] * a[i * 3 + q];
        }
        if (gamma == 0.f || fabsf(gamma) <= tol * sqrtf(alpha * beta)) continue;
        rotated = 1;
        float zeta = (beta - alpha) / (2.0f * gamma);
        float t = 1.0f / (fabsf(zeta) + sqrtf(1.0f + zeta * zeta));
        if (zeta < 0.f) t = -t;
        float c = 1.0f / sqrtf(1.0f + t * t);
        float s = c * t;
        for (int i = 0; i < 3; ++i) {
          float ap = a[i * 3 + p], aq = a[i * 3 + q];
          a[i * 3 + p] = c * ap - s * aq;
          a[i * 3 + q] = s * ap + c * aq;
          float vp = v[i * 3 + p], vq = v[i * 3 + q];
          v[i * 3 + p] = c * vp - s * vq;
          v[i * 3 + q] = s * vp + c * vq;
        }
      }
    }
    if (!rotated) break;
  }
  float sv[3];
  for (int k = 0; k < 3; ++k) {
    float n2 = 0.f;
    for (int i = 0; i < 3; ++i) n2 = n2 + a[i * 3 + k] * a[i * 3 + k];
    sv[k] = sqrtf(n2);
  }
  int idx[3] = {0, 1, 2};
  for (int i = 1; i < 3; ++i)
    for (int j = i; j > 0 && sv[idx[j]] > sv[idx[j - 1]]; --j) { int tmp = idx[j]; idx[j] = idx[j - 1]; idx[j - 1] = tmp; }
  float u[9];
  for (int k = 0; k < 3; ++k) {
    int src = idx[k];
    S[k] = sv[src];
    for (int i = 0; i < 3; ++i) {
      V[i * 3 + k] = v[i * 3 + src];
      u[i * 3 + k] = a[i * 3 + src];
    }
  }
  const float tiny = 1e-20f;
  for (int k = 0; k < 2; ++k)
    if (S[k] > tiny)
      for (int i = 0; i < 3; ++i) u[i * 3 + k] = u[i * 3 + k] / S[k];
  if (!(S[0] > tiny)) { u[0] = 1; u[3] = 0; u[6] = 0; }
  if (!(S[1] > tiny)) {
    float x = u[0], y = u[3], z = u[6];
    float bx, by, bz;
    if (fabsf(x) <= fabsf(y) && fabsf(x) <= fabsf(z)) { bx = 1; by = 0; bz = 0; }
    else if (fabsf(y) <= fabsf(z)) { bx = 0; by = 1; bz = 0; }
    else { bx = 0; by = 0; bz = 1; }
    float cx = y * bz - z * by, cy = z * bx - x * bz, cz = x * by - y * bx;
    float n = sqrtf(cx * cx + cy * cy + cz * cz);
    u[1] = cx / n; u[4] = cy / n; u[7] = cz / n;
  }
  if (S[2] > 1e-6f * S[0] && S[2] > tiny) {
    for (int i = 0; i < 3; ++i) u[i * 3 + 2] = u[i * 3 + 2] / S[2];
  } else {
    u[2] = u[3] * u[7] - u[6] * u[4];
    u[5] = u[6] * u[1] - u[0] * u[7];
    u[8] = u[0] * u[4] - u[3] * u[1];
  }
  for (int i = 0; i < 9; ++i) U[i] = u[i];
  for (int k = 0; k < 3; ++k) S[k] = ldexpf(S[k], e);
}
__device__ __forceinline__ float det3_f32(const float m[9]) {
  return m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) +
         m[2] * (m[3] * m[7] - m[4] * m[6]);
}
__device__ void umeyama_from_moments_f32(const float mu_s[3], const float mu_d[3], const float sigma[9],
                                         double Rt[16]) {
  float U[9], S[3], V[9];
  svd3_f32(sigma, U, S, V);
  float sgn[3] = {1.f, 1.f, 1.f};
  if (det3_f32(U) * det3_f32(V) < 0.f) sgn[2] = -1.f;
  float R[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      float acc = 0.f;
      for (int k = 0; k < 3; ++k) acc = acc + (U[i * 3 + k] * sgn[k]) * V[j * 3 + k];
      R[i * 3 + j] = acc;
    }
  float t[3];
  for (int i = 0; i < 3; ++i) {
    float acc = 0.f;
    for (int k = 0; k < 3; ++k) acc = acc + R[i * 3 + k] * mu_s[k];
    t[i] = mu_d[i] - acc;
  }
  for (int i = 0; i < 16; ++i) Rt[i] = 0.0;
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) Rt[j * 4 + i] = (double)R[i * 3 + j];
    Rt[12 + i] = (double)t[i];
  }
  Rt[15] = 1.0;
}

}  // namespace
}  // namespace ghicp_b200
