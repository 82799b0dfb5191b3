// ghicp_solvers_math.h — the small dense solves behind the opt-in estimators of ghicp_solvers.cu, written as
// host+device functions so that the very code the kernel runs on thread 0 can also be exercised by a host test
// harness (tests/harness/solvers_math_harness.cpp) against the oracle — no GPU needed for that part of the check.
// Inputs are the reduced sums the kernel accumulates; see k_solve_alt for their definition.
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define GHICP_HD __host__ __device__
#else
#define GHICP_HD
#endif

namespace ghicp_b200 {

GHICP_HD inline void rt_identity(double Rt[16]) {
  for (int i = 0; i < 16; ++i) Rt[i] = (i % 5 == 0) ? 1.0 : 0.0;
}

// x = A^-1 b for a symmetric positive definite NN x NN system by Cholesky; false when A is not positive definite to
// working precision (degenerate geometry: e.g. all normals parallel).
template <int NN>
GHICP_HD inline bool chol_solve(double (&A)[NN][NN], double (&b)[NN], double (&x)[NN]) {
  double tr = 0.0;
  for (int i = 0; i < NN; ++i) tr += A[i][i];
  const double tiny = 1e-13 * tr;
  double L[NN][NN];
  for (int i = 0; i < NN; ++i)
    for (int j = 0; j <= i; ++j) {
      double v = A[i][j];
      for (int k = 0; k < j; ++k) v -= L[i][k] * L[j][k];
      if (i == j) {
        if (!(v > tiny)) return false;
        L[i][i] = sqrt(v);
      } else {
        L[i][j] = v / L[j][j];
      }
    }
  double y[NN];
  for (int i = 0; i < NN; ++i) {
    double v = b[i];
    for (int k = 0; k < i; ++k) v -= L[i][k] * y[k];
    y[i] = v / L[i][i];
  }
  for (int i = NN - 1; i >= 0; --i) {
    double v = y[i];
    for (int k = i + 1; k < NN; ++k) v -= L[k][i] * x[k];
    x[i] = v / L[i][i];
  }
  return true;
}

// Point-to-plane LLS (PCL TransformationEstimationPointToPlaneLLS).  acc[0..20] = upper triangle of A^T A in row order
// (rows [s x n, n]), acc[21..26] = A^T b (b = n.(t - s)).  Rt column-major 4x4, R = Rz(gamma) Ry(beta) Rx(alpha).
GHICP_HD inline bool pt2pl_from_normal_equations(const double acc[27], double Rt[16]) {
  double A[6][6], b[6], x[6];
  int q = 0;
  for (int i = 0; i < 6; ++i)
    for (int j = i; j < 6; ++j) { A[i][j] = acc[q]; A[j][i] = acc[q]; ++q; }
  for (int i = 0; i < 6; ++i) b[i] = acc[21 + i];
  if (!chol_solve<6>(A, b, x)) return false;
  const double al = x[0], be = x[1], ga = x[2];
  const double sa = sin(al), ca = cos(al), sb = sin(be), cb = cos(be), sg = sin(ga), cg = cos(ga);
  rt_identity(Rt);
  // PCL constructTransformationMatrix; column-major store Rt[col*4 + row]
  Rt[0] = cg * cb;  Rt[4] = -sg * ca + cg * sb * sa;  Rt[8] = sg * sa + cg * sb * ca;    Rt[12] = x[3];
  Rt[1] = sg * cb;  Rt[5] = cg * ca + sg * sb * sa;   Rt[9] = -cg * sa + sg * sb * ca;   Rt[13] = x[4];
  Rt[2] = -sb;      Rt[6] = cb * sa;                  Rt[10] = cb * ca;                  Rt[14] = x[5];
  return true;
}

// Deterministic double sine and cosine for |x| <= 2^20 (NaN beyond, and for a non-finite x): the same bits on the host and
// the device, because they use only correctly rounded + - * / in a fixed order (build without FMA contraction: nvcc
// --fmad=false, g++ -ffp-contract=off), where the device's and the C library's sin / cos may differ in the last bit.  The
// dense point-to-plane ICP (DESIGN.md §3.14) builds its rotation with them.  Method: the classic fdlibm / musl argument
// reduction by pi/2 in up to three rounds of a 33 + 33 + 33 + 53-bit split of pi/2, then their minimax kernels on
// [-pi/4, pi/4]; within 1 ulp of a correctly rounded result over the range.
namespace ghicp_sc {
constexpr double INVPIO2 = 6.36619772367581382433e-01, TOINT = 6755399441055744.0;   // 2 / pi, 1.5 * 2^52
constexpr double PIO2_1 = 1.57079632673412561417e+00, PIO2_1T = 6.07710050650619224932e-11;
constexpr double PIO2_2 = 6.07710050630396597660e-11, PIO2_2T = 2.02226624879595063154e-21;
constexpr double PIO2_3 = 2.02226624871116645580e-21, PIO2_3T = 8.47842766036889956997e-32;
constexpr double S1 = -1.66666666666666324348e-01, S2 = 8.33333333332248946124e-03, S3 = -1.98412698298579493134e-04,
                 S4 = 2.75573137070700676789e-06, S5 = -2.50507602534068634195e-08, S6 = 1.58969099521155010221e-10;
constexpr double C1 = 4.16666666666666019037e-02, C2 = -1.38888888888741095749e-03, C3 = 2.48015872894767294178e-05,
                 C4 = -2.75573143513906633035e-07, C5 = 2.08757232129817482790e-09, C6 = -1.13596475577881948265e-11;
// sin(x + y) and cos(x + y) for |x + y| <= pi/4, |y| tiny against x
GHICP_HD inline double ksin(double x, double y) {
  const double z = x * x, w = z * z;
  const double r = (S2 + z * (S3 + z * S4)) + (z * w) * (S5 + z * S6);
  const double v = z * x;
  return x - (((z * (0.5 * y - v * r)) - y) - v * S1);
}
GHICP_HD inline double kcos(double x, double y) {
  const double z = x * x, w = z * z;
  const double r = z * (C1 + z * (C2 + z * C3)) + (w * w) * (C4 + z * (C5 + z * C6));
  const double hz = 0.5 * z, u = 1.0 - hz;
  return u + (((1.0 - u) - hz) + (z * r - x * y));
}
// x = n pi/2 + (y0 + y1), |y0 + y1| <= pi/4 (about); returns n mod 4
GHICP_HD inline int rem_pio2(double x, double &y0, double &y1) {
  const double fn = (x * INVPIO2 + TOINT) - TOINT;   // x / (pi/2) rounded to the nearest integer
  double r = x - fn * PIO2_1;                        // exact: fn * PIO2_1 has at most 53 bits for |fn| < 2^20
  double w = fn * PIO2_1T;
  y0 = r - w;
  const double ax = x < 0.0 ? -x : x;
  if ((y0 < 0.0 ? -y0 : y0) < ax * 0x1p-16) {        // cancellation: second round, good to 118 bits
    double t = r;
    w = fn * PIO2_2;
    r = t - w;
    w = fn * PIO2_2T - ((t - r) - w);
    y0 = r - w;
    if ((y0 < 0.0 ? -y0 : y0) < ax * 0x1p-49) {      // third round, 151 bits
      t = r;
      w = fn * PIO2_3;
      r = t - w;
      w = fn * PIO2_3T - ((t - r) - w);
      y0 = r - w;
    }
  }
  y1 = (r - y0) - w;
  const double q = fn - 4.0 * (double)(long long)(fn * 0.25);   // fn mod 4 in -3 .. 3 (exact)
  return ((int)q + 4) & 3;
}
}  // namespace ghicp_sc

GHICP_HD inline void det_sincos(double x, double &s, double &c) {
  using namespace ghicp_sc;
  const double ax = x < 0.0 ? -x : x;
  if (!(ax <= 1048576.0)) { s = c = (x - x) / (x - x); return; }   // NaN (also for +-inf and NaN)
  if (ax < 0x1p-26) { s = x; c = 1.0; return; }                    // subnormals and tiny angles: exact to the last bit
  double y0 = x, y1 = 0.0;
  int n = 0;
  if (ax > 0.78539816339744827900) n = rem_pio2(x, y0, y1);   // beyond pi/4
  const double sn = ksin(y0, y1), cs = kcos(y0, y1);
  switch (n) {
    case 0: s = sn; c = cs; break;
    case 1: s = cs; c = -sn; break;
    case 2: s = -sn; c = -cs; break;
    default: s = -cs; c = sn; break;
  }
}

// Generalized ICP's per-pair metric (DESIGN.md §3.15): M = (R C_s R^T + C_t)^-1 with C = I - (1 - eps) n n^T, eps = 0.001
// (PCL's gicp_epsilon: the neighbourhood covariance with its singular values replaced by (1, 1, eps)), from the source and
// target k-NN normals ns, nt and R = the rotation of the transform at the start of the iteration (row-major, widened from
// float32).  All in double in a fixed order, so the kernel and the oracle agree bit for bit without FMA contraction.  The
// sum has eigenvalues >= 2 eps: M is positive definite.  M = {m00, m01, m02, m11, m12, m22}.
constexpr double GICP_EPSILON = 1e-3;
GHICP_HD inline void gicp_mahalanobis(const double R[9], const float ns[3], const float nt[3], double M[6]) {
  const double e = 1.0 - GICP_EPSILON;
  const double a[3] = {(double)ns[0], (double)ns[1], (double)ns[2]}, b[3] = {(double)nt[0], (double)nt[1], (double)nt[2]};
  double Cs[9], RC[9], S[6];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) Cs[3 * r + c] = (r == c ? 1.0 : 0.0) - e * (a[r] * a[c]);
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) RC[3 * r + c] = (R[3 * r] * Cs[c] + R[3 * r + 1] * Cs[3 + c]) + R[3 * r + 2] * Cs[6 + c];
  int q = 0;
  for (int r = 0; r < 3; ++r)
    for (int c = r; c < 3; ++c)   // (R C_s R^T)_rc + (C_t)_rc
      S[q++] = ((RC[3 * r] * R[3 * c] + RC[3 * r + 1] * R[3 * c + 1]) + RC[3 * r + 2] * R[3 * c + 2]) +
               ((r == c ? 1.0 : 0.0) - e * (b[r] * b[c]));
  // the inverse of the symmetric S by its cofactors
  const double c00 = S[3] * S[5] - S[4] * S[4], c01 = S[2] * S[4] - S[1] * S[5], c02 = S[1] * S[4] - S[2] * S[3];
  const double c11 = S[0] * S[5] - S[2] * S[2], c12 = S[1] * S[2] - S[0] * S[4], c22 = S[0] * S[3] - S[1] * S[1];
  const double det = (S[0] * c00 + S[1] * c01) + S[2] * c02;
  M[0] = c00 / det; M[1] = c01 / det; M[2] = c02 / det; M[3] = c11 / det; M[4] = c12 / det; M[5] = c22 / det;
}

// CRegistration::LLS_4DOF (src/common_reg.cpp:623-775) from the 12 moments
//   acc = { W, Sx, Sy, Sz, SX, SY, SZ, Q = sum w (x^2 + y^2), sum w xX, sum w yX, sum w xY, sum w yY }
// (x, y, z source; X, Y, Z target).  Per Gauss-Newton step the reference's normal equations (:661-689) are
//   [ Q  u  v  0 ] [dth]   [ c (xY - yX) - s (xX + yY) ]      u = -Sx s - Sy c,  v = Sx c - Sy s
//   [ u  W  0  0 ] [tx ] = [ SX - Sx c + Sy s           ]      (s, c = sin, cos of the current yaw)
//   [ v  0  W  0 ] [ty ]   [ SY - Sx s - Sy c           ]
//   [ 0  0  0  W ] [tz ]   [ SZ - Sz                    ]
// solved by eliminating the translation block.  Starts from yaw 0, stops when |dth| <= 1e-9 like :654.
GHICP_HD inline bool yaw4dof_from_moments(const double acc[12], double Rt[16]) {
  const double W = acc[0], Sx = acc[1], Sy = acc[2], Sz = acc[3], SX = acc[4], SY = acc[5], SZ = acc[6];
  const double Q = acc[7], xX = acc[8], yX = acc[9], xY = acc[10], yY = acc[11];
  if (!(W > 0.0)) return false;
  // Schur complement of the translation block = spread of the source about its centroid (independent of the yaw)
  const double den = Q - (Sx * Sx + Sy * Sy) / W;
  if (!(den > 1e-13 * Q)) return false;
  double theta = 0.0, tx = 0.0, ty = 0.0;
  for (int it = 0; it < 200; ++it) {
    const double sn = sin(theta), cs = cos(theta);
    const double u = -Sx * sn - Sy * cs, v = Sx * cs - Sy * sn;
    const double g0 = cs * (xY - yX) - sn * (xX + yY);
    const double g1 = SX - Sx * cs + Sy * sn;
    const double g2 = SY - Sx * sn - Sy * cs;
    const double dth = (g0 - (u * g1 + v * g2) / W) / den;
    tx = (g1 - u * dth) / W;
    ty = (g2 - v * dth) / W;
    theta += dth;
    if (!(fabs(dth) > 1e-9)) break;
  }
  const double tz = (SZ - Sz) / W;
  const double sn = sin(theta), cs = cos(theta);
  rt_identity(Rt);
  Rt[0] = cs; Rt[4] = -sn; Rt[12] = tx;
  Rt[1] = sn; Rt[5] = cs;  Rt[13] = ty;
  Rt[14] = tz;
  return true;
}

}  // namespace ghicp_b200
