// fpfh_oracle.cpp — the canonical FPFH definition (DESIGN.md §3.10), one thread, no grid.  TEST INFRASTRUCTURE ONLY:
// tests/fpfh_oracle.py compiles it (g++ -ffp-contract=off) and checks the product's kernels (ghicp_prep.cu, k_knn / k_normals /
// k_spfh / k_fpfh) against it.
//
// The reference's driver calls FPFHfeature::compute_fpfh_feature + keyfpfh (test/ghicp_main.cpp:120-127): PCL
// NormalEstimation (k-NN, k = 20) and FPFHEstimationOMP (k-NN, k = 20), include/fpfh.hpp:36-115.  PCL is not pinned, so the
// places where PCL / FLANN / Eigen leave a choice open get these fixed rules:
//   k-NN      exact, the k_eff = min(k, n) smallest d2 = (dx*dx + dy*dy) + dz*dz (float32, dx = q.x - p.x), the query itself
//             included, ascending (d2, index)  (FLANN's tie order is unspecified)
//   normal    covariance of the k_eff neighbours as double sums about the query point, (sum dd - sum d sum d / k) / (k - 1)
//             rounded once to float32; its eigenvectors by cyclic Jacobi in double, sign "largest component positive"
//             (Eigen's sign is unspecified); the smallest eigenvalue's (first index on ties), normalised in double,
//             rounded to float32, negated iff ((-p.x)*n.x + (-p.y)*n.y) + (-p.z)*n.z < 0 (viewpoint 0).  k_eff < 3: NaN.
//   SPFH      hist_incr = 100 / (k_eff - 1); per neighbour q != p (by index) computePairFeatures, pairs with |dp| == 0,
//             |v| == 0 or a NaN normal skipped (still counted in k_eff - 1); PCL's acos(|a1|) > acos(|a2|) is |a1| < |a2|;
//             f1 = atan2 in double, rounded to float; bins floor(11 * x) clamped to [0, 10]
//   non-finite points take no part: k_eff = min(k, finite points), the lists of finite points hold finite points only; a
//             non-finite point's list is itself k_eff times at d2 = 0, its normal NaN (status 1), its SPFH and FPFH zero
//   FPFH      the neighbours with d2 != 0, weight 1 / d2 (float), per bin float sums in k-NN order, per block double sums,
//             each block times (float)(100 / sum) when the sum is not 0; the point's own SPFH is not added
// Float operation order of the pair features — the same text in gh-icp_b200/csrc/ghicp_prep.cu:
//   dot(a, b)   = (a.x*b.x + a.y*b.y) + a.z*b.z
//   cross(a, b) = (a.y*b.z - a.z*b.y, a.z*b.x - a.x*b.z, a.x*b.y - a.y*b.x)
//   |a|         = sqrtf(dot(a, a)),  a / |a| = three divisions
#include <algorithm>
#include <cmath>
#include <cstring>
#include <utility>
#include <vector>

namespace {

float fpfh_d2(const float *q, const float *p) {
  const float dx = q[0] - p[0], dy = q[1] - p[1], dz = q[2] - p[2];
  return (dx * dx + dy * dy) + dz * dz;
}
float f3dot(const float a[3], const float b[3]) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }
void f3cross(const float a[3], const float b[3], float o[3]) {
  o[0] = a[1] * b[2] - a[2] * b[1];
  o[1] = a[2] * b[0] - a[0] * b[2];
  o[2] = a[0] * b[1] - a[1] * b[0];
}
int fpfh_bin(double x) {
  int h = (int)std::floor(11 * x);
  return h < 0 ? 0 : (h > 10 ? 10 : h);
}
// cyclic Jacobi on a symmetric 3x3 in double; columns of V = eigenvectors, "largest component positive"
void jacobi3(double a[3][3], double V[3][3], double w[3]) {
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) V[i][j] = (i == j) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 64; ++sweep) {
    double off = 0.0;
    for (int p = 0; p < 3; ++p) for (int q = p + 1; q < 3; ++q) off += a[p][q] * a[p][q];
    if (off == 0.0) break;
    for (int p = 0; p < 3; ++p)
      for (int q = p + 1; q < 3; ++q) {
        if (a[p][q] == 0.0) continue;
        const double theta = (a[q][q] - a[p][p]) / (2.0 * a[p][q]);
        const double t = (theta >= 0.0 ? 1.0 : -1.0) / (std::fabs(theta) + std::sqrt(theta * theta + 1.0));
        const double c = 1.0 / std::sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < 3; ++k) { const double x = a[k][p], y = a[k][q]; a[k][p] = c * x - s * y; a[k][q] = s * x + c * y; }
        for (int k = 0; k < 3; ++k) { const double x = a[p][k], y = a[q][k]; a[p][k] = c * x - s * y; a[q][k] = s * x + c * y; }
        for (int k = 0; k < 3; ++k) { const double x = V[k][p], y = V[k][q]; V[k][p] = c * x - s * y; V[k][q] = s * x + c * y; }
      }
  }
  for (int j = 0; j < 3; ++j) {
    w[j] = a[j][j];
    int big = 0;
    for (int i = 1; i < 3; ++i) if (std::fabs(V[i][j]) > std::fabs(V[big][j])) big = i;
    if (V[big][j] < 0.0) for (int i = 0; i < 3; ++i) V[i][j] = -V[i][j];
  }
}

struct State {
  const float *xyz; int n, k;   // k = k_eff
  std::vector<int> nb; std::vector<float> d2; std::vector<char> have_nb;
  std::vector<float> nrm; std::vector<char> have_nrm;
  std::vector<float> spfh; std::vector<char> have_spfh;

  bool finite(int i) const { const float *p = xyz + 3 * (size_t)i; return std::isfinite(p[0]) && std::isfinite(p[1]) && std::isfinite(p[2]); }
  const int *knn(int i) {   // brute force over the whole (finite) cloud
    if (!have_nb[i]) {
      std::vector<std::pair<float, int>> all;
      if (finite(i)) {
        for (int p = 0; p < n; ++p) if (finite(p)) all.push_back({fpfh_d2(xyz + 3 * (size_t)i, xyz + 3 * (size_t)p), p});
        std::partial_sort(all.begin(), all.begin() + k, all.end());
      } else {
        all.assign(k, {0.f, i});
      }
      for (int j = 0; j < k; ++j) { nb[(size_t)i * k + j] = all[j].second; d2[(size_t)i * k + j] = all[j].first; }
      have_nb[i] = 1;
    }
    return &nb[(size_t)i * k];
  }
  const float *normal(int i) {
    if (!have_nrm[i]) {
      float *o = &nrm[3 * (size_t)i];
      const float *q = xyz + 3 * (size_t)i;
      if (k < 3 || !finite(i)) {
        o[0] = o[1] = o[2] = std::nanf("");
      } else {
        const int *l = knn(i);
        double sd[3] = {0, 0, 0}, sdd[6] = {0, 0, 0, 0, 0, 0};
        for (int j = 0; j < k; ++j) {
          const float *p = xyz + 3 * (size_t)l[j];
          const float ex = p[0] - q[0], ey = p[1] - q[1], ez = p[2] - q[2];
          const double a = ex, b = ey, c = ez;
          sd[0] += a; sd[1] += b; sd[2] += c;
          sdd[0] += a * a; sdd[1] += a * b; sdd[2] += a * c; sdd[3] += b * b; sdd[4] += b * c; sdd[5] += c * c;
        }
        const double inv_n = 1.0 / k, alpha = 1.0 / (k - 1);
        const float cv[6] = {(float)((sdd[0] - sd[0] * sd[0] * inv_n) * alpha), (float)((sdd[1] - sd[0] * sd[1] * inv_n) * alpha),
                             (float)((sdd[2] - sd[0] * sd[2] * inv_n) * alpha), (float)((sdd[3] - sd[1] * sd[1] * inv_n) * alpha),
                             (float)((sdd[4] - sd[1] * sd[2] * inv_n) * alpha), (float)((sdd[5] - sd[2] * sd[2] * inv_n) * alpha)};
        double A[3][3] = {{cv[0], cv[1], cv[2]}, {cv[1], cv[3], cv[4]}, {cv[2], cv[4], cv[5]}}, V[3][3], w[3];
        jacobi3(A, V, w);
        int jm = 0;
        if (w[1] < w[jm]) jm = 1;
        if (w[2] < w[jm]) jm = 2;
        const double vx = V[0][jm], vy = V[1][jm], vz = V[2][jm];
        const double len = std::sqrt((vx * vx + vy * vy) + vz * vz);
        float nx = (float)(vx / len), ny = (float)(vy / len), nz = (float)(vz / len);
        if (((-q[0]) * nx + (-q[1]) * ny) + (-q[2]) * nz < 0.f) { nx = -nx; ny = -ny; nz = -nz; }
        o[0] = nx; o[1] = ny; o[2] = nz;
      }
      have_nrm[i] = 1;
    }
    return &nrm[3 * (size_t)i];
  }
  const float *spfh_of(int i) {
    if (!have_spfh[i]) {
      float *hist = &spfh[(size_t)i * 33];
      for (int b = 0; b < 33; ++b) hist[b] = 0.f;
      const float *np_ = normal(i);
      if (k > 1 && !std::isnan(np_[0])) {
        const float hist_incr = 100.0f / (float)(k - 1);
        const float inv2pi = 1.0f / (2.0f * 3.14159265358979323846f);
        const float *p = xyz + 3 * (size_t)i;
        const int *l = knn(i);
        for (int j = 0; j < k; ++j) {
          const int qi = l[j];
          if (qi == i) continue;
          const float *nq = normal(qi);
          if (std::isnan(nq[0])) continue;
          const float *q = xyz + 3 * (size_t)qi;
          float dp[3] = {q[0] - p[0], q[1] - p[1], q[2] - p[2]};
          const float f4 = std::sqrt(f3dot(dp, dp));
          if (f4 == 0.f) continue;
          const float a1 = f3dot(np_, dp) / f4, a2 = f3dot(nq, dp) / f4;
          float u[3], other[3], f3;
          if (std::fabs(a1) < std::fabs(a2)) {
            for (int c = 0; c < 3; ++c) { u[c] = nq[c]; other[c] = np_[c]; dp[c] = -dp[c]; }
            f3 = -a2;
          } else {
            for (int c = 0; c < 3; ++c) { u[c] = np_[c]; other[c] = nq[c]; }
            f3 = a1;
          }
          float v[3], w[3];
          f3cross(dp, u, v);
          const float vn = std::sqrt(f3dot(v, v));
          if (vn == 0.f) continue;
          v[0] = v[0] / vn; v[1] = v[1] / vn; v[2] = v[2] / vn;
          f3cross(u, v, w);
          const float f2 = f3dot(v, other);
          const float f1 = (float)std::atan2((double)f3dot(w, other), (double)f3dot(u, other));
          hist[fpfh_bin(((double)f1 + 3.14159265358979323846) * (double)inv2pi)] += hist_incr;
          hist[11 + fpfh_bin(((double)f2 + 1.0) * 0.5)] += hist_incr;
          hist[22 + fpfh_bin(((double)f3 + 1.0) * 0.5)] += hist_incr;
        }
      }
      have_spfh[i] = 1;
    }
    return &spfh[(size_t)i * 33];
  }
  void fpfh(int i, float *out) {
    float hist[33];
    double sum[3] = {0.0, 0.0, 0.0};
    for (int b = 0; b < 33; ++b) hist[b] = 0.f;
    const int *l = knn(i);
    for (int j = 0; j < k; ++j) {
      const float dd = d2[(size_t)i * k + j];
      if (dd == 0.f) continue;
      const float wgt = 1.0f / dd;
      const float *sq = spfh_of(l[j]);
      for (int b = 0; b < 33; ++b) {
        const float val = sq[b] * wgt;
        hist[b] += val;
        sum[b / 11] += (double)val;
      }
    }
    for (int b = 0; b < 33; ++b) out[b] = sum[b / 11] != 0.0 ? hist[b] * (float)(100.0 / sum[b / 11]) : hist[b];
  }
};

}  // namespace

extern "C" {

// Histograms at idx [nidx] (NULL: every point) into fpfh [nidx][33].  Only what those histograms read is computed (k-NN at
// the points, their neighbours and the neighbours' neighbours; normals of the last two), plus, when all_normals != 0, every
// point's k-NN and normal.  normals [n][3], status [n], nb_idx / nb_d2 [n][k_eff] (may be NULL) are written where
// computed; computed [n] (may be NULL) gets bit 0 = k-NN, bit 1 = normal.  Returns k_eff.
int fpfh_oracle(const float *xyz, int n, const int *idx, int nidx, int k, int all_normals, float *fpfh, float *normals,
                int *status, int *nb_idx, float *nb_d2, int *computed) {
  if (n <= 0 || k < 1) return -1;
  State S;
  int nfin = 0;
  for (int i = 0; i < n; ++i) nfin += std::isfinite(xyz[3 * (size_t)i]) && std::isfinite(xyz[3 * (size_t)i + 1]) && std::isfinite(xyz[3 * (size_t)i + 2]);
  S.xyz = xyz; S.n = n; S.k = k < nfin ? k : nfin;
  S.nb.assign((size_t)n * S.k, -1); S.d2.assign((size_t)n * S.k, 0.f); S.have_nb.assign(n, 0);
  S.nrm.assign(3 * (size_t)n, 0.f); S.have_nrm.assign(n, 0);
  S.spfh.assign((size_t)n * 33, 0.f); S.have_spfh.assign(n, 0);
  const int m = idx ? nidx : n;
  for (int t = 0; t < m; ++t) S.fpfh(idx ? idx[t] : t, fpfh + (size_t)t * 33);
  if (all_normals) for (int i = 0; i < n; ++i) S.normal(i);
  for (int i = 0; i < n; ++i) {
    if (S.have_nb[i]) {
      if (nb_idx) std::memcpy(nb_idx + (size_t)i * S.k, &S.nb[(size_t)i * S.k], sizeof(int) * S.k);
      if (nb_d2) std::memcpy(nb_d2 + (size_t)i * S.k, &S.d2[(size_t)i * S.k], sizeof(float) * S.k);
    }
    if (S.have_nrm[i]) {
      if (normals) std::memcpy(normals + 3 * (size_t)i, &S.nrm[3 * (size_t)i], sizeof(float) * 3);
      if (status) status[i] = (S.k < 3 || !S.finite(i)) ? 1 : 0;
    }
    if (computed) computed[i] = (S.have_nb[i] ? 1 : 0) | (S.have_nrm[i] ? 2 : 0);
  }
  return S.k;
}

}  // extern "C"
