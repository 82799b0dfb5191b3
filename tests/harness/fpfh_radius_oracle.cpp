// fpfh_radius_oracle.cpp — the canonical FPFH over radius neighbourhoods (DESIGN.md §3.10, "Radius neighbourhoods"), one
// thread, brute force.  TEST INFRASTRUCTURE ONLY: tests/fpfh_radius_oracle.py compiles it (g++ -ffp-contract=off) and checks
// the product's kernels (ghicp_prep.cu, prep_fpfh_radius) against it.
//
// CRegistration::compute_fpfh_feature (src/common_reg.cpp:373-389) = PCL NormalEstimation with radius search_radius, then
// FPFHEstimation with radius 2 search_radius.  The rules of the k-NN definition (fpfh_oracle.cpp, whose helpers this file
// includes) change only where radius neighbourhoods require it:
//   N_r(p)   every q of the cloud with d2(p, q) < r2: d2 = (dx*dx + dy*dy) + dz*dz (float32), r2 = r*r in float32; the query
//            and exact duplicates included; ascending (d2, index) (PCL's sorted KD-tree order, ties by index)
//   normal   the k-NN covariance / Jacobi / flip over N_rn(p); fewer than 3 points: NaN, status 1
//   SPFH     over N_rf(p), hist_incr = 100 / (|N_rf(p)| - 1); a point that is its own only neighbour: zero histogram
//   FPFH     over N_rf(p): weight 1 / d2, d2 == 0 skipped, float per-bin sums in list order, double per-block sums
#include "fpfh_oracle.cpp"

namespace {

struct RadState {
  const float *xyz; int n; float r2[2];          // [0] normal radius, [1] feature radius
  std::vector<std::vector<std::pair<float, int>>> nb[2]; std::vector<char> have_nb[2];
  std::vector<float> nrm; std::vector<char> have_nrm;
  std::vector<float> spfh; std::vector<char> have_spfh;

  const std::vector<std::pair<float, int>> &list(int w, int i) {
    if (!have_nb[w][i]) {
      auto &l = nb[w][i];
      for (int p = 0; p < n; ++p) {
        const float d = fpfh_d2(xyz + 3 * (size_t)i, xyz + 3 * (size_t)p);
        if (d < r2[w]) l.push_back({d, p});
      }
      std::sort(l.begin(), l.end());
      have_nb[w][i] = 1;
    }
    return nb[w][i];
  }
  const float *normal(int i) {
    if (!have_nrm[i]) {
      float *o = &nrm[3 * (size_t)i];
      const float *q = xyz + 3 * (size_t)i;
      const auto &l = list(0, i);
      const int k = (int)l.size();
      if (k < 3) {
        o[0] = o[1] = o[2] = std::nanf("");
      } else {
        double sd[3] = {0, 0, 0}, sdd[6] = {0, 0, 0, 0, 0, 0};
        for (int j = 0; j < k; ++j) {
          const float *p = xyz + 3 * (size_t)l[j].second;
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
      const auto &l = list(1, i);
      const int k = (int)l.size();
      const float *np_ = normal(i);
      if (k > 1 && !std::isnan(np_[0])) {
        const float hist_incr = 100.0f / (float)(k - 1);
        const float inv2pi = 1.0f / (2.0f * 3.14159265358979323846f);
        const float *p = xyz + 3 * (size_t)i;
        for (int j = 0; j < k; ++j) {
          const int qi = l[j].second;
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
    const auto &l = list(1, i);
    for (const auto &e : l) {
      if (e.first == 0.f) continue;
      const float wgt = 1.0f / e.first;
      const float *sq = spfh_of(e.second);
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

// Histograms at idx [nidx] (NULL: every point) into fpfh [nidx][33] with normal radius rn and feature radius rf.  Only what
// those histograms read is computed, plus every point's normal when all_normals != 0.  normals [n][3] and status [n] are
// written where computed (status 0 / 1); computed [n] (may be NULL) gets bit 0 = N_rn list, bit 1 = normal, bit 2 = N_rf list.
// Where list_w (0 = N_rn, 1 = N_rf) is 0 or 1, counts [n] (-1 where not built) and, when nb_idx / nb_d2 are not NULL, the
// lists concatenated in point order (capacity nb_cap entries) are written.  Returns the number of list entries written, or
// -1 on a bad argument / -2 when nb_cap is too small.
long long fpfh_radius_oracle(const float *xyz, int n, const int *idx, int nidx, float rn, float rf, int all_normals, float *fpfh,
                             float *normals, int *status, int *computed, int list_w, long long *counts, int *nb_idx, float *nb_d2,
                             long long nb_cap) {
  if (n <= 0) return -1;
  RadState S;
  S.xyz = xyz; S.n = n; S.r2[0] = rn * rn; S.r2[1] = rf * rf;
  for (int w = 0; w < 2; ++w) { S.nb[w].assign(n, {}); S.have_nb[w].assign(n, 0); }
  S.nrm.assign(3 * (size_t)n, 0.f); S.have_nrm.assign(n, 0);
  S.spfh.assign((size_t)n * 33, 0.f); S.have_spfh.assign(n, 0);
  const int m = idx ? nidx : n;
  for (int t = 0; t < m; ++t) S.fpfh(idx ? idx[t] : t, fpfh + (size_t)t * 33);
  if (all_normals) for (int i = 0; i < n; ++i) S.normal(i);
  if (list_w == 0 || list_w == 1) for (int i = 0; i < n; ++i) S.list(list_w, i);
  long long written = 0;
  for (int i = 0; i < n; ++i) {
    if (S.have_nrm[i]) {
      if (normals) std::memcpy(normals + 3 * (size_t)i, &S.nrm[3 * (size_t)i], sizeof(float) * 3);
      if (status) status[i] = std::isnan(S.nrm[3 * (size_t)i]) ? 1 : 0;
    }
    if (computed) computed[i] = (S.have_nb[0][i] ? 1 : 0) | (S.have_nrm[i] ? 2 : 0) | (S.have_nb[1][i] ? 4 : 0);
    if (list_w == 0 || list_w == 1) {
      const auto &l = S.nb[list_w][i];
      if (counts) counts[i] = (long long)l.size();
      for (const auto &e : l) {
        if (nb_idx || nb_d2) {
          if (written >= nb_cap) return -2;
          if (nb_idx) nb_idx[written] = e.second;
          if (nb_d2) nb_d2[written] = e.first;
        }
        ++written;
      }
    }
  }
  return written;
}

}  // extern "C"
