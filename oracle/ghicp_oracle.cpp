// ghicp_oracle.cpp — CPU oracle (TEST INFRASTRUCTURE ONLY; see ghicp_oracle.h for scope, citations
// and pinning status).  Restates the reference's scalar loops on flat arrays; copies no code.
//
// Build with -ffp-contract=off and no -march so every double/float operation is a separately
// rounded IEEE operation, like the reference built with "-O3" on x86-64 (CMakeLists.txt:5).
#include "ghicp_oracle.h"

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#ifdef _OPENMP
#include <omp.h>
#endif

namespace {

using clk = std::chrono::steady_clock;
static double ms_since(clk::time_point t0) {
  return std::chrono::duration<double, std::milli>(clk::now() - t0).count();
}

static orc_km_backend_fn g_km_backend = nullptr;

// ---------------------------------------------------------------------------------------------
// Hamming distance, byte-LUT popcount semantics (src/stereo_binary_feature.cpp:16-104).
// The LUT in the reference is the plain popcount table, so popcount of the XORed byte is identical.
// ---------------------------------------------------------------------------------------------
static inline int popcount8(unsigned char b) {
  int c = 0;
  while (b) { c += b & 1; b >>= 1; }
  return c;
}
static unsigned char g_lut[256];
static bool g_lut_ready = false;
static void init_lut() {
  if (g_lut_ready) return;
  for (int i = 0; i < 256; ++i) g_lut[i] = (unsigned char)popcount8((unsigned char)i);
  g_lut_ready = true;
}

// ---------------------------------------------------------------------------------------------
// 3x3 float32 SVD by one-sided (Hestenes) Jacobi, singular values sorted descending like
// Eigen::JacobiSVD.  A = U diag(S) V^T, row-major 3x3.  V is a product of rotations / column swaps.
// Like JacobiSVD, A is first divided by its scale: by 2^e, the power of two above its largest |entry|, which
// every step commutes with exactly (bit-identical results wherever the unscaled sweep stayed in range; no
// overflow of alpha * beta past ~6e4 units of spread).  Zero or non-finite A is left unscaled.
// ---------------------------------------------------------------------------------------------
static void svd3_f32(const float A[9], float U[9], float S[3], float V[9]) {
  float amax = 0.f;
  bool finite = true;
  for (int i = 0; i < 9; ++i) { const float m = std::fabs(A[i]); finite = finite && std::isfinite(m); amax = m > amax ? m : amax; }
  int e = 0;
  if (finite && amax > 0.f) std::frexp(amax, &e);
  float a[9];
  for (int i = 0; i < 9; ++i) a[i] = std::ldexp(A[i], -e);
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
        if (gamma == 0.f || std::fabs(gamma) <= tol * std::sqrt(alpha * beta)) continue;
        rotated = 1;
        float zeta = (beta - alpha) / (2.0f * gamma);
        float t = 1.0f / (std::fabs(zeta) + std::sqrt(1.0f + zeta * zeta));
        if (zeta < 0.f) t = -t;
        float c = 1.0f / std::sqrt(1.0f + t * t);
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
    sv[k] = std::sqrt(n2);
  }
  int idx[3] = {0, 1, 2};
  // sort descending (stable insertion)
  for (int i = 1; i < 3; ++i)
    for (int j = i; j > 0 && sv[idx[j]] > sv[idx[j - 1]]; --j) std::swap(idx[j], idx[j - 1]);
  float u[9];
  for (int k = 0; k < 3; ++k) {
    int src = idx[k];
    S[k] = sv[src];
    for (int i = 0; i < 3; ++i) {
      V[i * 3 + k] = v[i * 3 + src];
      u[i * 3 + k] = a[i * 3 + src];
    }
  }
  // normalise U columns; complete rank-deficient columns with cross products
  const float tiny = 1e-20f;
  for (int k = 0; k < 2; ++k) {
    if (S[k] > tiny) {
      for (int i = 0; i < 3; ++i) u[i * 3 + k] = u[i * 3 + k] / S[k];
    }
  }
  if (!(S[0] > tiny)) { u[0] = 1; u[3] = 0; u[6] = 0; }
  if (!(S[1] > tiny)) {
    // any unit vector orthogonal to u0
    float x = u[0], y = u[3], z = u[6];
    float bx, by, bz;
    if (std::fabs(x) <= std::fabs(y) && std::fabs(x) <= std::fabs(z)) { bx = 1; by = 0; bz = 0; }
    else if (std::fabs(y) <= std::fabs(z)) { bx = 0; by = 1; bz = 0; }
    else { bx = 0; by = 0; bz = 1; }
    float cx = y * bz - z * by, cy = z * bx - x * bz, cz = x * by - y * bx;
    float n = std::sqrt(cx * cx + cy * cy + cz * cz);
    u[1] = cx / n; u[4] = cy / n; u[7] = cz / n;
  }
  // third column: if sigma_3 is well separated from zero use the normalised column,
  // otherwise the cross product of the first two (then det U = +1).
  if (S[2] > 1e-6f * S[0] && S[2] > tiny) {
    for (int i = 0; i < 3; ++i) u[i * 3 + 2] = u[i * 3 + 2] / S[2];
  } else {
    u[2] = u[3] * u[7] - u[6] * u[4];
    u[5] = u[6] * u[1] - u[0] * u[7];
    u[8] = u[0] * u[4] - u[3] * u[1];
  }
  for (int i = 0; i < 9; ++i) U[i] = u[i];
  for (int k = 0; k < 3; ++k) S[k] = std::ldexp(S[k], e);
}

static inline float det3_f32(const float m[9]) {
  return m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) +
         m[2] * (m[3] * m[7] - m[4] * m[6]);
}

// Umeyama (no scaling) given float32 means and float32 covariance sigma = dst_c * src_c^T / n.
// (Eigen/src/Geometry/Umeyama.h as used by PCL's TransformationEstimationSVD; published algorithm
// restated: JacobiSVD(sigma), S = diag(1,1,sign(det U det V)), R = U S V^T, t = mu_d - R mu_s.)
static void umeyama_from_moments_f32(const float mu_s[3], const float mu_d[3], const float sigma[9],
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
  // column-major 4x4, cast<double>() of the float matrix (ghicp_reg.cpp:863-866)
  for (int i = 0; i < 16; ++i) Rt[i] = 0.0;
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) Rt[j * 4 + i] = (double)R[i * 3 + j];
    Rt[12 + i] = (double)t[i];
  }
  Rt[15] = 1.0;
}

static int rigid_fit_impl(const double *s, const double *t, int n, int solve_mode, double Rt[16]) {
  for (int i = 0; i < 16; ++i) Rt[i] = (i % 5 == 0) ? 1.0 : 0.0;
  if (n < 3) return 1;  // degenerate: identity (deviation: the reference would feed PCL anyway)
  const double *sx = s, *sy = s + n, *sz = s + 2 * (size_t)n;
  const double *tx = t, *ty = t + n, *tz = t + 2 * (size_t)n;
  float mu_s[3], mu_d[3], sigma[9];
  if (solve_mode == 0) {
    // PCL path: points cast to float (ghicp_reg.cpp:843-855), float32 means / demean / product.
    float ms[3] = {0, 0, 0}, md[3] = {0, 0, 0};
    for (int i = 0; i < n; ++i) {
      ms[0] += (float)sx[i]; ms[1] += (float)sy[i]; ms[2] += (float)sz[i];
      md[0] += (float)tx[i]; md[1] += (float)ty[i]; md[2] += (float)tz[i];
    }
    const float one_over_n = 1.0f / (float)n;
    for (int k = 0; k < 3; ++k) { mu_s[k] = ms[k] * one_over_n; mu_d[k] = md[k] * one_over_n; }
    float acc[9] = {0};
    for (int i = 0; i < n; ++i) {
      float ds[3] = {(float)sx[i] - mu_s[0], (float)sy[i] - mu_s[1], (float)sz[i] - mu_s[2]};
      float dd[3] = {(float)tx[i] - mu_d[0], (float)ty[i] - mu_d[1], (float)tz[i] - mu_d[2]};
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) acc[r * 3 + c] += dd[r] * ds[c];
    }
    for (int k = 0; k < 9; ++k) sigma[k] = one_over_n * acc[k];
  } else {
    // float64 moments (order-independent up to 1e-16), then rounded once to float32.
    double ms[3] = {0, 0, 0}, md[3] = {0, 0, 0};
    for (int i = 0; i < n; ++i) {
      ms[0] += sx[i]; ms[1] += sy[i]; ms[2] += sz[i];
      md[0] += tx[i]; md[1] += ty[i]; md[2] += tz[i];
    }
    double mus[3], mud[3];
    for (int k = 0; k < 3; ++k) { mus[k] = ms[k] / n; mud[k] = md[k] / n; }
    double acc[9] = {0};
    for (int i = 0; i < n; ++i) {
      double ds[3] = {sx[i] - mus[0], sy[i] - mus[1], sz[i] - mus[2]};
      double dd[3] = {tx[i] - mud[0], ty[i] - mud[1], tz[i] - mud[2]};
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) acc[r * 3 + c] += dd[r] * ds[c];
    }
    for (int k = 0; k < 3; ++k) { mu_s[k] = (float)mus[k]; mu_d[k] = (float)mud[k]; }
    for (int k = 0; k < 9; ++k) sigma[k] = (float)(acc[k] / n);
  }
  umeyama_from_moments_f32(mu_s, mu_d, sigma, Rt);
  return 0;
}

// ---------------------------------------------------------------------------------------------
// OPT-IN estimators (extensions: the reference loop never calls them; SURVEY.md §8a-9, §8f N4).
//   1 weighted point-to-point: weighted means / cross-covariance + the float32 Umeyama core above
//   2 point-to-plane LLS     : PCL TransformationEstimationPointToPlaneLLS (estimator of
//                              IterativeClosestPointWithNormals, src/common_reg.cpp:123-199); PCL is not in
//                              /root/reference: published algorithm restated, PARITY UNPINNED
//   3 yaw-only 4-DoF         : CRegistration::LLS_4DOF, src/common_reg.cpp:623-775, restated row by row:
//                              the 3n x 4 system is assembled EXPLICITLY every Gauss-Newton step like :661-685
//                              and solved through the normal equations (:689) — on purpose not the moment
//                              form the GPU kernel uses, so the two derivations check each other.
// ---------------------------------------------------------------------------------------------
static bool gauss_solve(int n, std::vector<double> A /* n x n row-major */, std::vector<double> b, double *x) {
  for (int c = 0; c < n; ++c) {
    int piv = c;
    for (int r = c + 1; r < n; ++r) if (std::fabs(A[(size_t)r * n + c]) > std::fabs(A[(size_t)piv * n + c])) piv = r;
    if (!(std::fabs(A[(size_t)piv * n + c]) > 0.0)) return false;
    if (piv != c) { for (int k = 0; k < n; ++k) std::swap(A[(size_t)piv * n + k], A[(size_t)c * n + k]); std::swap(b[piv], b[c]); }
    for (int r = c + 1; r < n; ++r) {
      const double f = A[(size_t)r * n + c] / A[(size_t)c * n + c];
      for (int k = c; k < n; ++k) A[(size_t)r * n + k] -= f * A[(size_t)c * n + k];
      b[r] -= f * b[c];
    }
  }
  for (int r = n - 1; r >= 0; --r) {
    double v = b[r];
    for (int k = r + 1; k < n; ++k) v -= A[(size_t)r * n + k] * x[k];
    x[r] = v / A[(size_t)r * n + r];
  }
  return true;
}

static int rigid_fit_ex_impl(int solver, const double *s, const double *t, const double *tn, const double *w, int n,
                             double Rt[16]) {
  for (int i = 0; i < 16; ++i) Rt[i] = (i % 5 == 0) ? 1.0 : 0.0;
  const double *sx = s, *sy = s + n, *sz = s + 2 * (size_t)n;
  const double *tx = t, *ty = t + n, *tz = t + 2 * (size_t)n;
  auto W = [&](int i) { return w ? w[i] : 1.0; };
  if (solver == 0 || solver == 1) {
    if (n < 3) return 1;
    double sw = 0, ms[3] = {0, 0, 0}, md[3] = {0, 0, 0};
    for (int i = 0; i < n; ++i) {
      sw += W(i);
      ms[0] += W(i) * sx[i]; ms[1] += W(i) * sy[i]; ms[2] += W(i) * sz[i];
      md[0] += W(i) * tx[i]; md[1] += W(i) * ty[i]; md[2] += W(i) * tz[i];
    }
    if (!(sw > 0.0)) return 1;
    double mus[3], mud[3];
    for (int k = 0; k < 3; ++k) { mus[k] = ms[k] / sw; mud[k] = md[k] / sw; }
    double acc[9] = {0};
    for (int i = 0; i < n; ++i) {
      const double ds[3] = {sx[i] - mus[0], sy[i] - mus[1], sz[i] - mus[2]};
      const double dd[3] = {tx[i] - mud[0], ty[i] - mud[1], tz[i] - mud[2]};
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) acc[r * 3 + c] += W(i) * (dd[r] * ds[c]);
    }
    float mu_s[3], mu_d[3], sigma[9];
    for (int k = 0; k < 3; ++k) { mu_s[k] = (float)mus[k]; mu_d[k] = (float)mud[k]; }
    for (int k = 0; k < 9; ++k) sigma[k] = (float)(acc[k] / sw);
    umeyama_from_moments_f32(mu_s, mu_d, sigma, Rt);
    return 0;
  }
  if (solver == 2) {
    if (n < 6 || !tn) return 1;
    const double *nx = tn, *ny = tn + n, *nz = tn + 2 * (size_t)n;
    std::vector<double> ATA(36, 0.0), ATb(6, 0.0);
    for (int i = 0; i < n; ++i) {
      const double row[6] = {nz[i] * sy[i] - ny[i] * sz[i], nx[i] * sz[i] - nz[i] * sx[i], ny[i] * sx[i] - nx[i] * sy[i],
                             nx[i], ny[i], nz[i]};
      const double d = nx[i] * tx[i] + ny[i] * ty[i] + nz[i] * tz[i] - nx[i] * sx[i] - ny[i] * sy[i] - nz[i] * sz[i];
      for (int r = 0; r < 6; ++r) {
        for (int c = 0; c < 6; ++c) ATA[r * 6 + c] += W(i) * (row[r] * row[c]);
        ATb[r] += W(i) * (row[r] * d);
      }
    }
    double x[6];
    double tr = 0; for (int k = 0; k < 6; ++k) tr += ATA[k * 7];
    // rank check through the smallest pivot of an LDL^T-free elimination: compare against the trace scale
    if (!gauss_solve(6, ATA, ATb, x)) return 1;
    for (int k = 0; k < 6; ++k) if (!std::isfinite(x[k])) return 1;
    (void)tr;
    const double al = x[0], be = x[1], ga = x[2];
    // PCL constructTransformationMatrix(alpha, beta, gamma, tx, ty, tz): R = Rz(gamma) Ry(beta) Rx(alpha)
    double R[3][3];
    R[0][0] = std::cos(ga) * std::cos(be);
    R[0][1] = -std::sin(ga) * std::cos(al) + std::cos(ga) * std::sin(be) * std::sin(al);
    R[0][2] = std::sin(ga) * std::sin(al) + std::cos(ga) * std::sin(be) * std::cos(al);
    R[1][0] = std::sin(ga) * std::cos(be);
    R[1][1] = std::cos(ga) * std::cos(al) + std::sin(ga) * std::sin(be) * std::sin(al);
    R[1][2] = -std::cos(ga) * std::sin(al) + std::sin(ga) * std::sin(be) * std::cos(al);
    R[2][0] = -std::sin(be);
    R[2][1] = std::cos(be) * std::sin(al);
    R[2][2] = std::cos(be) * std::cos(al);
    for (int i = 0; i < 3; ++i) {
      for (int j = 0; j < 3; ++j) Rt[j * 4 + i] = R[i][j];
      Rt[12 + i] = x[3 + i];
    }
    return 0;
  }
  if (solver == 3) {
    if (n < 2) return 1;  // src/common_reg.cpp:648 "Not enough control point number"
    double theta0 = 0.0, dtheta = 9999, eps = 1e-9;  // :643-646 (initial guess 0 deg)
    double sol[4] = {0, 0, 0, 0};
    int iter_num = 0;
    while (std::abs(dtheta) > eps && iter_num < 200) {  // :654 (the 200 cap is ours)
      std::vector<double> ATA(16, 0.0), ATb(4, 0.0);
      for (int j = 0; j < n; ++j) {
        const double A0[4] = {-sx[j] * std::sin(theta0) - sy[j] * std::cos(theta0), 1, 0, 0};   // :663-666
        const double A1[4] = {sx[j] * std::cos(theta0) - sy[j] * std::sin(theta0), 0, 1, 0};    // :668-671
        const double A2[4] = {0, 0, 0, 1};                                                      // :673-676
        const double b0 = tx[j] - sx[j] * std::cos(theta0) + sy[j] * std::sin(theta0);          // :679
        const double b1 = ty[j] - sx[j] * std::sin(theta0) - sy[j] * std::cos(theta0);          // :680
        const double b2 = tz[j] - sz[j];                                                        // :681
        const double *rows[3] = {A0, A1, A2};
        const double bb[3] = {b0, b1, b2};
        for (int q = 0; q < 3; ++q)
          for (int r = 0; r < 4; ++r) {
            for (int c = 0; c < 4; ++c) ATA[r * 4 + c] += W(j) * (rows[q][r] * rows[q][c]);
            ATb[r] += W(j) * (rows[q][r] * bb[q]);
          }
      }
      if (!gauss_solve(4, ATA, ATb, sol)) return 1;   // x = (A^T A)^-1 A^T b, :689
      dtheta = sol[0];
      theta0 += dtheta;
      ++iter_num;
    }
    const double theta = theta0;
    Rt[0] = std::cos(theta); Rt[4] = -std::sin(theta); Rt[12] = sol[1];   // :719-737
    Rt[1] = std::sin(theta); Rt[5] = std::cos(theta);  Rt[13] = sol[2];
    Rt[10] = 1.0;                                       Rt[14] = sol[3];
    return 0;
  }
  return -1;
}

// ---------------------------------------------------------------------------------------------
// KM restatement (src/km.cpp:13-126).  Same traversal order, same eps-tight test, slack reset once
// per x, recursive DFS (run orc from a thread with a large stack for big n).
// ---------------------------------------------------------------------------------------------
struct KmState {
  const double *G;
  int n;
  double eps;
  std::vector<int> match;
  std::vector<double> lx, ly, slack;
  std::vector<char> visx, visy;
};

static bool km_findpath(KmState &k, int x) {
  double tempDelta;
  k.visx[x] = 1;
  const double *row = k.G + (size_t)x * k.n;
  for (int y = 0; y < k.n; ++y) {
    if (k.visy[y]) continue;
    tempDelta = k.lx[x] + k.ly[y] - row[y];
    if (tempDelta < k.eps) {
      k.visy[y] = 1;
      if (k.match[y] == -1 || km_findpath(k, k.match[y])) {
        k.match[y] = x;
        return true;
      }
    } else {
      k.slack[y] = std::min(tempDelta, k.slack[y]);
    }
  }
  return false;
}

static void km_solve_impl(const double *G, int n, double eps, int *match_out) {
  KmState k;
  k.G = G; k.n = n; k.eps = eps;
  k.match.assign(n, -1);
  k.lx.assign(n, 0.0); k.ly.assign(n, 0.0); k.slack.assign(n, 0.0);
  k.visx.assign(n, 0); k.visy.assign(n, 0);
  const int INF2 = 1000;
  for (int i = 0; i < n; ++i) {
    k.lx[i] = G[(size_t)i * n];
    for (int j = 0; j < n; ++j) k.lx[i] = std::max(G[(size_t)i * n + j], k.lx[i]);
  }
  for (int x = 0; x < n; ++x) {
    for (int j = 0; j < n; ++j) k.slack[j] = INF2;
    while (true) {
      for (int i = 0; i < n; ++i) { k.visx[i] = 0; k.visy[i] = 0; }
      if (km_findpath(k, x)) break;
      double delta = INF2;
      for (int j = 0; j < n; ++j)
        if (!k.visy[j]) delta = std::min(delta, k.slack[j]);
      for (int i = 0; i < n; ++i)
        if (k.visx[i]) k.lx[i] -= delta;
      for (int i = 0; i < n; ++i) {
        if (k.visy[i]) k.ly[i] += delta;
        else k.slack[i] -= delta;
      }
    }
  }
  for (int i = 0; i < n; ++i) match_out[i] = k.match[i];
}

// Km::output + Calenergy (src/km.cpp:128-233), without the Corres.txt side effect (km.cpp:147-198).
static int km_output_impl(const double *G, int n, int sp, int tp, double penalty, const int *match,
                          std::vector<int> &SP, std::vector<int> &TP, std::vector<int> &SPout,
                          std::vector<int> &TPout, double *energy) {
  int cor_number = 0;
  for (int i = 0; i < n; ++i) {
    if (G[(size_t)match[i] * n + i] != -penalty) {
      SP.push_back(match[i]);
      TP.push_back(i);
      cor_number++;
    } else {
      if (sp >= tp) {
        SPout.push_back(match[i]);
        if (i < tp) TPout.push_back(i);
      } else {
        TPout.push_back(i);
        if (match[i] < sp) SPout.push_back(match[i]);
      }
    }
  }
  if (energy) {
    const int INF = 10000;
    double e = 0;
    for (int i = 0; i < n; ++i)
      if (G[(size_t)match[i] * n + i] != -INF) e -= G[(size_t)match[i] * n + i];
    *energy = e;
  }
  return cor_number;
}

}  // namespace

// ---------------------------------------------------------------------------------------------
struct orc_ctx {
  orc_config cfg;
  int N = 0, M = 0, V = 0, bits = 0, B = 0;
  std::vector<double> kpS, kpT;           // column-major N x 3 / M x 3
  std::vector<uint8_t> bscS, bscT;        // [V][N][B], [M][B]
  std::vector<float> fpfhS, fpfhT;        // [N][33], [M][33]
  std::vector<double> ED, FD, CD;         // row-major N x M
  // Energyfunction (ghicp_reg.h:15-42)
  int weight_changing_rate = 6;
  double penalty = 0, para1_penalty = 1.0, para2_penalty = 1.0, penalty_initial = 2.0;
  int min_cor = 10;
  double KM_eps = 0.01;
  float scale = 0;
  // GHRegistration state (ghicp_reg.h:77-117)
  int iteration_number = 0;
  double RMS = 99999;
  double FDM = 0, FDstd = 0, IoU = 0;
  bool converge = false;
  double converge_t_, converge_r_;
  float adjustweight_step_, adjustweight_ratio_, estimated_IoU_;
  bool use_6dof_case_;
  double nonmax;
  double Rt_tillnow[16];
  std::vector<int> SP, TP;
  std::vector<double> Spoint, Tpoint;     // column-major cor x 3
  double last_cd_mean = 0, last_cd_std = 0, last_energy = 0;
  // opt-in estimators (extension; 0 = the reference's SVD)
  int solver = 0;
  std::vector<double> tn;                 // target normals, column-major M x 3
};

extern "C" {

void orc_set_km_backend(orc_km_backend_fn fn) { g_km_backend = fn; }

orc_ctx *orc_create(const orc_config *cfg) {
  init_lut();
  orc_ctx *c = new orc_ctx();
  c->cfg = *cfg;
  // Energyfunction::init (ghicp_reg.h:26-41)
  c->penalty_initial = 2.0;
  c->para1_penalty = 1.0;
  c->para2_penalty = 1.0;
  c->min_cor = 10;
  c->weight_changing_rate = 6;
  c->KM_eps = 0.01;
  c->scale = 0.005 * cfg->bbx_magnitude;  // double product rounded to float, as the reference
  // GHRegistration ctor (ghicp_reg.h:77-117)
  c->iteration_number = 0;
  c->RMS = 99999;
  c->converge = false;
  c->nonmax = cfg->nonmax;
  c->adjustweight_ratio_ = cfg->adjust_ratio;
  c->adjustweight_step_ = cfg->adjust_step;
  c->converge_t_ = cfg->converge_t;  // float -> double
  c->converge_r_ = cfg->converge_r;
  c->estimated_IoU_ = cfg->estimated_iou;
  c->use_6dof_case_ = (cfg->dof == 6);
  for (int i = 0; i < 16; ++i) c->Rt_tillnow[i] = (i % 5 == 0) ? 1.0 : 0.0;
#ifdef _OPENMP
  if (cfg->num_threads > 0) omp_set_num_threads(cfg->num_threads);
#endif
  return c;
}

void orc_destroy(orc_ctx *c) { delete c; }

int orc_set_keypoints(orc_ctx *c, const double *sxyz, int N, const double *txyz, int M) {
  c->N = N; c->M = M;
  c->kpS.assign(sxyz, sxyz + 3 * (size_t)N);
  c->kpT.assign(txyz, txyz + 3 * (size_t)M);
  // Energyfunction::init resizes ED/FD/CD to N x M zero-filled (ghicp_reg.h:28-30)
  c->ED.assign((size_t)N * M, 0.0);
  c->FD.assign((size_t)N * M, 0.0);
  c->CD.assign((size_t)N * M, 0.0);
  return 0;
}

int orc_set_bsc(orc_ctx *c, const uint8_t *s_bits, int V, const uint8_t *t_bits, int bits) {
  c->V = V; c->bits = bits;
  c->B = (int)std::ceil((float)bits / 8.f);  // stereo_binary_feature.h:50
  c->bscS.assign(s_bits, s_bits + (size_t)V * c->N * c->B);
  c->bscT.assign(t_bits, t_bits + (size_t)c->M * c->B);
  return 0;
}

int orc_set_fpfh(orc_ctx *c, const float *s, const float *t) {
  c->fpfhS.assign(s, s + (size_t)c->N * 33);
  c->fpfhT.assign(t, t + (size_t)c->M * 33);
  return 0;
}

int orc_hamming(const uint8_t *a, const uint8_t *b, int nbytes) {
  init_lut();
  int one_count = 0;
  for (int i = 0; i < nbytes; ++i) one_count += g_lut[(unsigned char)(a[i] ^ b[i])];
  return one_count;
}

float orc_fpfh_distance(const float *his1, const float *his2) {
  // include/fpfh.hpp:135-165, float32 arithmetic, same accumulation order
  float d_correlation = 0, d_correlation_up = 0, d_correlation_down1 = 0, d_correlation_down2 = 0;
  float mean_his1 = 0, mean_his2 = 0;
  for (int i = 0; i < 33; i++) {
    mean_his1 += his1[i];
    mean_his2 += his2[i];
  }
  mean_his1 /= 33;
  mean_his2 /= 33;
  for (int i = 0; i < 33; i++) {
    d_correlation_up += (his1[i] - mean_his1) * (his2[i] - mean_his2);
    d_correlation_down1 += (his1[i] - mean_his1) * (his1[i] - mean_his1);
    d_correlation_down2 += (his2[i] - mean_his2) * (his2[i] - mean_his2);
  }
  // sqrt(float) resolves to the float overload under <cmath> + using namespace std in the reference
  d_correlation = d_correlation_up / std::sqrt(d_correlation_down1 * d_correlation_down2);
  return std::fabs(d_correlation);
}

int orc_build_fd(orc_ctx *c) {
  const int N = c->N, M = c->M;
  if (c->cfg.feature_type == ORC_FT_BSC) {
    const int B = c->B;
    const int V = c->use_6dof_case_ ? 4 : 2;  // ghicp_reg.cpp:178-182
    if (c->V < V) return -1;
#pragma omp parallel for schedule(static) if (c->cfg.num_threads > 1)
    for (int i = 0; i < N; ++i) {
      for (int j = 0; j < M; ++j) {
        const uint8_t *tj = &c->bscT[(size_t)j * B];
        int best = orc_hamming(&c->bscS[((size_t)0 * N + i) * B], tj, B);
        for (int v = 1; v < V; ++v)
          best = std::min(best, orc_hamming(&c->bscS[((size_t)v * N + i) * B], tj, B));
        c->FD[(size_t)i * M + j] = best;
      }
    }
  } else if (c->cfg.feature_type == ORC_FT_FPFH) {
#pragma omp parallel for schedule(static) if (c->cfg.num_threads > 1)
    for (int i = 0; i < N; ++i)
      for (int j = 0; j < M; ++j)
        c->FD[(size_t)i * M + j] = orc_fpfh_distance(&c->fpfhS[(size_t)i * 33], &c->fpfhT[(size_t)j * 33]);
  }
  return 0;
}

int orc_km_solve(const double *W, int n, double eps, int *match) {
  km_solve_impl(W, n, eps, match);
  return 0;
}

int orc_km_output(const double *W, int n, int sp, int tp, double penalty, const int *match, int *SP,
                  int *TP, int *SPout, int *nSPout, int *TPout, int *nTPout, double *energy) {
  std::vector<int> sp_v, tp_v, spo, tpo;
  int cor = km_output_impl(W, n, sp, tp, penalty, match, sp_v, tp_v, spo, tpo, energy);
  for (int i = 0; i < cor; ++i) { if (SP) SP[i] = sp_v[i]; if (TP) TP[i] = tp_v[i]; }
  if (SPout) for (size_t i = 0; i < spo.size(); ++i) SPout[i] = spo[i];
  if (TPout) for (size_t i = 0; i < tpo.size(); ++i) TPout[i] = tpo[i];
  if (nSPout) *nSPout = (int)spo.size();
  if (nTPout) *nTPout = (int)tpo.size();
  return cor;
}

int orc_rigid_fit_ex(int solver, const double *s, const double *t, const double *tn, const double *w, int n,
                     double Rt[16]) {
  return rigid_fit_ex_impl(solver, s, t, tn, w, n, Rt);
}

int orc_set_solver(orc_ctx *c, int solver, const double *target_normals) {
  if (solver < 0 || solver > 3 || solver == 1) return -1;
  if (solver == 2 && !target_normals) return -1;
  c->solver = solver;
  if (target_normals) c->tn.assign(target_normals, target_normals + 3 * (size_t)c->M);
  return 0;
}

int orc_rigid_fit(const double *s, const double *t, int n, int solve_mode, double Rt[16]) {
  return rigid_fit_impl(s, t, n, solve_mode, Rt);
}

// --- stages -----------------------------------------------------------------------------------

static void calED(orc_ctx *c) {  // ghicp_reg.cpp:114-139
  const int N = c->N, M = c->M;
  const double *sx = c->kpS.data(), *sy = sx + N, *sz = sy + N;
  const double *tx = c->kpT.data(), *ty = tx + M, *tz = ty + M;
#pragma omp parallel for schedule(static) if (c->cfg.num_threads > 1)
  for (int i = 0; i < N; ++i)
    for (int j = 0; j < M; ++j)
      c->ED[(size_t)i * M + j] =
          c->scale * std::sqrt(std::pow(sx[i] - tx[j], 2) + std::pow(sy[i] - ty[j], 2) + std::pow(sz[i] - tz[j], 2));
}

static void calCD_NF(orc_ctx *c) {  // ghicp_reg.cpp:216-243
  const size_t NM = (size_t)c->N * c->M;
  double CDsum = 0;
  if (c->cfg.num_threads > 1) {
#pragma omp parallel for reduction(+ : CDsum) schedule(static)
    for (size_t k = 0; k < NM; ++k) { c->CD[k] = c->ED[k]; CDsum += c->CD[k]; }
  } else {
    for (size_t k = 0; k < NM; ++k) { c->CD[k] = c->ED[k]; CDsum += c->CD[k]; }
  }
  double CDmean = CDsum / c->M / c->N;
  if (c->iteration_number > 1) c->penalty = c->RMS * c->para1_penalty * c->scale;
  else c->penalty = CDmean / c->penalty_initial;
  c->penalty = std::max(CDmean, 1.0);  // :239 overrides the lines above
  c->last_cd_mean = CDmean;
  c->last_cd_std = 0;
}

static void calCD_BSC(orc_ctx *c) {  // ghicp_reg.cpp:245-293
  const size_t NM = (size_t)c->N * c->M;
  double WFD = std::exp(-1.0 * c->iteration_number / c->weight_changing_rate);
  double WED = 1.0 - WFD;
  double CDsum = 0, CDstdsum = 0;
  if (c->cfg.num_threads > 1) {
#pragma omp parallel for reduction(+ : CDsum) schedule(static)
    for (size_t k = 0; k < NM; ++k) { c->CD[k] = WED * c->ED[k] + WFD * c->FD[k]; CDsum += c->CD[k]; }
  } else {
    for (size_t k = 0; k < NM; ++k) { c->CD[k] = WED * c->ED[k] + WFD * c->FD[k]; CDsum += c->CD[k]; }
  }
  double CDmean = CDsum / c->M / c->N;
  if (c->cfg.num_threads > 1) {
#pragma omp parallel for reduction(+ : CDstdsum) schedule(static)
    for (size_t k = 0; k < NM; ++k) CDstdsum += std::pow(c->CD[k] - CDmean, 2);
  } else {
    for (size_t k = 0; k < NM; ++k) CDstdsum += std::pow(c->CD[k] - CDmean, 2);
  }
  double CDstd = std::sqrt(CDstdsum / c->M / c->N);
  if (c->iteration_number > 1)
    c->penalty = c->RMS * c->para1_penalty * c->scale * WED + (c->FDM + c->para2_penalty * c->FDstd) * WFD;
  else
    c->penalty = (CDmean - c->penalty_initial * CDstd);
  c->penalty = std::max(c->penalty, 5.0);
  c->last_cd_mean = CDmean;
  c->last_cd_std = CDstd;
}

static void calCD_FPFH(orc_ctx *c) {  // ghicp_reg.cpp:295-341
  const size_t NM = (size_t)c->N * c->M;
  double CDsum = 0;
  const double ex = 1.0 / (c->iteration_number + 1);
  if (c->cfg.num_threads > 1) {
#pragma omp parallel for reduction(+ : CDsum) schedule(static)
    for (size_t k = 0; k < NM; ++k) { c->CD[k] = 1.0 * c->ED[k] / std::pow(c->FD[k], ex); CDsum += c->CD[k]; }
  } else {
    for (size_t k = 0; k < NM; ++k) { c->CD[k] = 1.0 * c->ED[k] / std::pow(c->FD[k], ex); CDsum += c->CD[k]; }
  }
  double CDmean = CDsum / c->N / c->M;
  if (c->iteration_number > 1)
    c->penalty = c->RMS * c->para1_penalty * c->scale * c->para2_penalty;
  else
    c->penalty = (CDmean / c->penalty_initial);
  c->last_cd_mean = CDmean;
  c->last_cd_std = 0;
}

static void gather_and_stats(orc_ctx *c) {
  // shared tail of findcorrespondence{KM,NNR,NN}: gather Spoint/Tpoint, RMSE, FDM, FDstd, RMS
  // (ghicp_reg.cpp:446-452,549-578 / 664-695 / 735-766)
  const int N = c->N, M = c->M;
  const int cor_number = (int)c->SP.size();
  c->Spoint.assign(3 * (size_t)cor_number, 0.0);
  c->Tpoint.assign(3 * (size_t)cor_number, 0.0);
  for (int i = 0; i < cor_number; ++i)
    for (int k = 0; k < 3; ++k) {
      c->Spoint[(size_t)k * cor_number + i] = c->kpS[(size_t)k * N + c->SP[i]];
      c->Tpoint[(size_t)k * cor_number + i] = c->kpT[(size_t)k * M + c->TP[i]];
    }
  double RMSE = 0, FDcul = 0;
  c->FDM = 0; c->FDstd = 0;
  const double *S = c->Spoint.data(), *T = c->Tpoint.data();
  for (int i = 0; i < cor_number; ++i) {
    RMSE += std::pow(S[i] - T[i], 2) + std::pow(S[cor_number + i] - T[cor_number + i], 2) +
            std::pow(S[2 * (size_t)cor_number + i] - T[2 * (size_t)cor_number + i], 2);
    c->FDM += c->FD[(size_t)c->SP[i] * M + c->TP[i]];
  }
  c->FDM /= cor_number;
  for (int i = 0; i < cor_number; ++i) FDcul += std::pow((c->FD[(size_t)c->SP[i] * M + c->TP[i]] - c->FDM), 2);
  c->FDstd = std::sqrt(FDcul / cor_number);
  RMSE /= cor_number;
  RMSE = std::sqrt(RMSE);
  c->RMS = RMSE;
}

static void findcorrespondenceKM(orc_ctx *c) {  // ghicp_reg.cpp:343-460
  const int N = c->N, M = c->M;
  int size = std::max(N, M);
  std::vector<double> graphweight((size_t)size * size);
  for (size_t k = 0; k < graphweight.size(); ++k) graphweight[k] = -c->penalty;
  for (int i = 0; i < N; ++i)
    for (int j = 0; j < M; ++j)
      if (c->CD[(size_t)i * M + j] < c->penalty) graphweight[(size_t)i * size + j] = -c->CD[(size_t)i * M + j];
  std::vector<int> match(size);
  if (c->cfg.use_ref_km && g_km_backend) g_km_backend(graphweight.data(), size, c->KM_eps, match.data());
  else km_solve_impl(graphweight.data(), size, c->KM_eps, match.data());
  c->SP.clear(); c->TP.clear();
  std::vector<int> SPout, TPout;
  km_output_impl(graphweight.data(), size, N, M, c->penalty, match.data(), c->SP, c->TP, SPout, TPout,
                 &c->last_energy);
  gather_and_stats(c);
}

static void findcorrespondenceNNR(orc_ctx *c) {  // ghicp_reg.cpp:605-698
  const int N = c->N, M = c->M;
  std::vector<int> SV(N), TV(M);
  const double MAXVALIUE = 9e20;
#pragma omp parallel for schedule(static) if (c->cfg.num_threads > 1)
  for (int i = 0; i < N; i++) {
    double mincd = MAXVALIUE; int minindex = 0;
    for (int j = 0; j < M; j++)
      if (c->CD[(size_t)i * M + j] < mincd) { mincd = c->CD[(size_t)i * M + j]; minindex = j; }
    SV[i] = minindex;
  }
#pragma omp parallel for schedule(static) if (c->cfg.num_threads > 1)
  for (int i = 0; i < M; i++) {
    double mincd = MAXVALIUE; int minindex = 0;
    for (int j = 0; j < N; j++)
      if (c->CD[(size_t)j * M + i] < mincd) { mincd = c->CD[(size_t)j * M + i]; minindex = j; }
    TV[i] = minindex;
  }
  c->SP.clear(); c->TP.clear();
  for (int i = 0; i < N; i++)
    if (TV[SV[i]] == i) { c->SP.push_back(i); c->TP.push_back(SV[i]); }
  gather_and_stats(c);
}

static void findcorrespondenceNN(orc_ctx *c) {  // ghicp_reg.cpp:700-769
  const int N = c->N, M = c->M;
  const double MAXVALIUE = 9e20;
  std::vector<int> best(N);
  std::vector<double> bestv(N);
#pragma omp parallel for schedule(static) if (c->cfg.num_threads > 1)
  for (int i = 0; i < N; i++) {
    double mincd = MAXVALIUE; int minindex = 0;
    for (int j = 0; j < M; j++)
      if (c->CD[(size_t)i * M + j] < mincd) { mincd = c->CD[(size_t)i * M + j]; minindex = j; }
    best[i] = minindex; bestv[i] = mincd;
  }
  c->SP.clear(); c->TP.clear();
  for (int i = 0; i < N; i++)
    if (bestv[i] < c->penalty) { c->SP.push_back(i); c->TP.push_back(best[i]); }
  gather_and_stats(c);
}

static void adjustweight(orc_ctx *c) {  // ghicp_reg.cpp:771-789
  if (c->estimated_IoU_ / c->IoU > c->adjustweight_ratio_) {
    c->para1_penalty += c->adjustweight_step_;
    c->para2_penalty += c->adjustweight_step_;
  } else if (c->IoU / c->estimated_IoU_ > c->adjustweight_ratio_) {
    c->para1_penalty -= c->adjustweight_step_;
    c->para2_penalty -= c->adjustweight_step_;
  }
}

static void transformestimation(orc_ctx *c, double Rt[16], orc_iter_stats *st) {  // ghicp_reg.cpp:791-927
  const int N = c->N, M = c->M;
  int cor_number = (int)c->SP.size();
  if (cor_number < c->min_cor) c->converge = 1;
  c->IoU = 1.0 * cor_number / (N + M - cor_number);
  if (c->solver == 0) {
    rigid_fit_impl(c->Spoint.data(), c->Tpoint.data(), cor_number, c->cfg.solve_mode, Rt);
  } else {
    std::vector<double> npair;
    if (c->solver == 2) {
      npair.assign(3 * (size_t)cor_number, 0.0);
      for (int i = 0; i < cor_number; ++i)
        for (int k = 0; k < 3; ++k) npair[(size_t)k * cor_number + i] = c->tn[(size_t)k * M + c->TP[i]];
    }
    rigid_fit_ex_impl(c->solver, c->Spoint.data(), c->Tpoint.data(), npair.empty() ? nullptr : npair.data(), nullptr,
                      cor_number, Rt);
  }
  double R[3][3], t[3];
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) R[i][j] = Rt[j * 4 + i];
    t[i] = Rt[12 + i];
  }
  double dx = t[0], dy = t[1], dz = t[2];
  double ax = std::atan2(R[2][1], R[2][2]);
  double ay = std::atan2(-R[2][0], std::sqrt(R[2][1] * R[2][1] + R[2][2] * R[2][2]));
  double az = std::atan2(R[0][1], R[0][0]);
  const double pi = 3.1415926;
  ax = ax / pi * 180; ay = ay / pi * 180; az = az / pi * 180;
  // Update (ghicp_reg.cpp:889-907); Eigen evaluates R*v as ((R0*x + R1*y) + R2*z), then + t
  double *sx = c->kpS.data(), *sy = sx + N, *sz = sy + N;
  for (int i = 0; i < N; i++) {
    double x = sx[i], y = sy[i], z = sz[i];
    sx[i] = ((R[0][0] * x + R[0][1] * y) + R[0][2] * z) + t[0];
    sy[i] = ((R[1][0] * x + R[1][1] * y) + R[1][2] * z) + t[1];
    sz[i] = ((R[2][0] * x + R[2][1] * y) + R[2][2] * z) + t[2];
  }
  double RMSEafter = 0;
  {
    double *px = c->Spoint.data(), *py = px + cor_number, *pz = py + cor_number;
    const double *qx = c->Tpoint.data(), *qy = qx + cor_number, *qz = qy + cor_number;
    for (int i = 0; i < cor_number; i++) {
      double x = px[i], y = py[i], z = pz[i];
      px[i] = ((R[0][0] * x + R[0][1] * y) + R[0][2] * z) + t[0];
      py[i] = ((R[1][0] * x + R[1][1] * y) + R[1][2] * z) + t[1];
      pz[i] = ((R[2][0] * x + R[2][1] * y) + R[2][2] * z) + t[2];
    }
    for (int i = 0; i < cor_number; ++i)
      RMSEafter += std::pow(px[i] - qx[i], 2) + std::pow(py[i] - qy[i], 2) + std::pow(pz[i] - qz[i], 2);
  }
  RMSEafter /= cor_number;
  RMSEafter = std::sqrt(RMSEafter);
  if (std::abs(dx) < c->converge_t_ && std::abs(dy) < c->converge_t_ && std::abs(dz) < c->converge_t_ &&
      std::abs(ax) < c->converge_r_ && std::abs(ay) < c->converge_r_ && std::abs(az) < c->converge_r_)
    c->converge = 1;
  st->rmse_after = RMSEafter;
  st->ax = ax; st->ay = ay; st->az = az;
}

int orc_iterate(orc_ctx *c, orc_iter_stats *st) {
  orc_iter_stats local;
  if (!st) st = &local;
  std::memset(st, 0, sizeof(*st));
  st->iteration = c->iteration_number;
  auto t0 = clk::now();
  calED(c);
  switch (c->cfg.feature_type) {
    case ORC_FT_BSC: calCD_BSC(c); break;
    case ORC_FT_FPFH: calCD_FPFH(c); break;
    case ORC_FT_NONE: calCD_NF(c); break;
    default: break;
  }
  st->t_cost_ms = ms_since(t0);
  t0 = clk::now();
  switch (c->cfg.corr_type) {
    case ORC_CT_KM: findcorrespondenceKM(c); break;
    case ORC_CT_NN: findcorrespondenceNN(c); break;
    case ORC_CT_NNR: findcorrespondenceNNR(c); break;
    default: break;
  }
  st->t_corr_ms = ms_since(t0);
  st->rmse = c->RMS;
  st->fdm = c->FDM;
  st->fdstd = c->FDstd;
  st->cor = (int)c->SP.size();
  st->warn_few_pairs = st->cor < c->min_cor;
  t0 = clk::now();
  double Rt[16];
  transformestimation(c, Rt, st);
  adjustweight(c);
  // Rt_tillnow = Rt_temp * Rt_tillnow (ghicp_reg.cpp:93), column-major
  double acc[16];
  for (int col = 0; col < 4; ++col)
    for (int row = 0; row < 4; ++row) {
      double s = 0;
      for (int k = 0; k < 4; ++k) s += Rt[k * 4 + row] * c->Rt_tillnow[col * 4 + k];
      acc[col * 4 + row] = s;
    }
  std::memcpy(c->Rt_tillnow, acc, sizeof(acc));
  st->t_solve_ms = ms_since(t0);
  std::memcpy(st->Rt, Rt, sizeof(Rt));
  std::memcpy(st->Rt_tillnow, c->Rt_tillnow, sizeof(acc));
  st->cd_mean = c->last_cd_mean;
  st->cd_std = c->last_cd_std;
  st->penalty = c->penalty;
  st->iou = c->IoU;
  st->para1 = c->para1_penalty;
  st->para2 = c->para2_penalty;
  st->km_energy = c->last_energy;
  st->converged = c->converge ? 1 : 0;
  c->iteration_number++;
  return 0;
}

int orc_run(orc_ctx *c, double Rt_final[16], int *iterations) {
  int it = 0;
  orc_iter_stats st;
  orc_build_fd(c);  // calFD_BSC / calFD_FPFH at the top of ghicp_reg (src/ghicp_reg.cpp:33-44)
  while (!c->converge) {
    orc_iterate(c, &st);
    ++it;
    if (c->cfg.max_iter > 0 && it >= c->cfg.max_iter) break;
  }
  std::memcpy(Rt_final, c->Rt_tillnow, sizeof(double) * 16);
  if (iterations) *iterations = it;
  return c->converge ? 0 : 1;
}

int orc_get_pairs(orc_ctx *c, int *sp, int *tp, int cap) {
  int n = (int)c->SP.size();
  for (int i = 0; i < n && i < cap; ++i) { sp[i] = c->SP[i]; tp[i] = c->TP[i]; }
  return n;
}

int orc_get_source(orc_ctx *c, double *sxyz) {
  std::memcpy(sxyz, c->kpS.data(), sizeof(double) * 3 * (size_t)c->N);
  return 0;
}

const double *orc_fd(orc_ctx *c) { return c->FD.data(); }
const double *orc_cd(orc_ctx *c) { return c->CD.data(); }

void orc_set_state(orc_ctx *c, int iteration, double rms, double fdm, double fdstd, double para1,
                   double para2) {
  c->iteration_number = iteration;
  c->RMS = rms; c->FDM = fdm; c->FDstd = fdstd;
  c->para1_penalty = para1; c->para2_penalty = para2;
}

}  // extern "C"
