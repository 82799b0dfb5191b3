// icp_oracle.cpp — the canonical point-to-point ICP of DESIGN.md §3.13, one thread (TEST INFRASTRUCTURE, built with
// -ffp-contract=off so that every float32 operation is rounded separately).  tests/icp_oracle.py compiles it and checks the
// product's kernels (gh-icp_b200/csrc/ghicp_icp.cu) against it.
//   set-up      the finite source and target points take part (indices i, j count those); F = the guess rounded to float32;
//               W_i = P_i moved by F, ((F00 x + F01 y) + F02 z) + F03
//   iteration   j(i) = argmin_j knn_d2(W_i, Q_j), ties to the smallest j, d_i its float32 d2; reciprocal: keep (i, j(i)) when
//               argmin_i' knn_d2(Q_j, W_i') is i (ties to the smallest i'); trimmed (rho > 0): keep the floor(rho * (float)c)
//               smallest (d_i, i) of the c pairs; c < 3: stop (NO_CORRESPONDENCES); FP64 moments of the kept pairs (means,
//               then the demeaned cross-covariance) summed in the fixed tree below, rounded once to float32, the float32
//               Umeyama of the loop -> T; F <- T F (float32, each entry ((a0 + a1) + a2) + a3); W <- T W; then
//               DefaultConvergenceCriteria: k >= max_iterations, |cos| / |t|^2 within epsilon_T, |mse - prev| < 1e-12,
//               |mse - prev| / prev < epsilon_F, mse = sum d_i / c over the kept pairs (before T was applied)
//   fitness     the §3.12 fitness of the whole source moved by F with max_range = +inf, summed in k_ov_reduce's tree
// The sums' tree: blocks of 8192 consecutive points; thread t of 256 adds the points t, t + 256, ... of its block in that
// order; a halving tree over the 256 threads (x[t] += x[t + w], w = 128, 64, ..., 1); the blocks the same way (thread t adds
// blocks t, t + 256, ...).  Nearest neighbours: brute force, or a uniform grid of its own (rings stopped by a plain double
// bound with a strict comparison, so a point at the same d2 as the best is never left unvisited) — same bits.
#include "sac_oracle.cpp"   // svd3_f32 / umeyama_f32: the float32 Umeyama of the loop, the same text as the device code

#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <limits>
#include <utility>
#include <vector>

namespace {

const float FINF = std::numeric_limits<float>::infinity();

inline float icp_d2(float qx, float qy, float qz, const float *b) {
  const float dx = qx - b[0], dy = qy - b[1], dz = qz - b[2];
  return (dx * dx + dy * dy) + dz * dz;
}
inline bool finite3(const float *p) { return std::isfinite(p[0]) && std::isfinite(p[1]) && std::isfinite(p[2]); }
inline void move16(const float *m, const float *p, float *o) {
  for (int r = 0; r < 3; ++r) o[r] = ((m[4 * r] * p[0] + m[4 * r + 1] * p[1]) + m[4 * r + 2] * p[2]) + m[4 * r + 3];
}

// nearest point of B (n points) in (d2, index) order
struct Nearest {
  const float *B = nullptr;
  long long n = 0;
  bool grid = false;
  double mn[3] = {0, 0, 0}, h = 1.0;
  long long gm[3] = {0, 0, 0};
  std::vector<std::pair<uint64_t, int>> cells;   // (cell key, first sorted position)
  std::vector<int> order, start;
  uint64_t key(long long x, long long y, long long z) const { return ((uint64_t)x << 42) | ((uint64_t)y << 21) | (uint64_t)z; }
  long long coord(double v, int a) const {
    const double f = std::floor((v - mn[a]) / h);
    if (!(f > 0)) return 0;
    return f > (double)gm[a] ? gm[a] : (long long)f;
  }
  void build(const float *b, long long nb, bool use_grid) {
    B = b; n = nb; grid = use_grid;
    if (!grid) return;
    double mx[3];
    for (int a = 0; a < 3; ++a) { mn[a] = b[a]; mx[a] = b[a]; }
    for (long long j = 0; j < nb; ++j)
      for (int a = 0; a < 3; ++a) { mn[a] = std::min(mn[a], (double)b[3 * j + a]); mx[a] = std::max(mx[a], (double)b[3 * j + a]); }
    double ext = 0.0;
    for (int a = 0; a < 3; ++a) ext = std::max(ext, mx[a] - mn[a]);
    h = std::max(std::cbrt(std::max(ext * ext * ext, 1e-30) * 4.0 / (double)nb), ext / 1.0e6);
    if (!(h > 0)) h = 1.0;
    // a scan fills surfaces, not its box, and unevenly: shrink the cell by the occupancy a point sees (sum of squared cell
    // counts over n, ~ h^2 on a surface) towards ~8, at most 16x (any cell edge gives the same result; this one keeps a
    // million-point search fast)
    cells_at(b, nb, mx);
    double w = 0.0;
    for (size_t e = 0; e + 1 < start.size(); ++e) { const double c = start[e + 1] - start[e]; w += c * c; }
    const double f = std::max(std::sqrt(8.0 / std::max(w / (double)nb, 1e-30)), 1.0 / 16);
    if (f < 1.0 && h * f > ext / 1.0e6) { h *= f; cells_at(b, nb, mx); }
  }
  void cells_at(const float *b, long long nb, const double *mx) {
    for (int a = 0; a < 3; ++a) gm[a] = (long long)std::floor((mx[a] - mn[a]) / h);
    std::vector<std::pair<uint64_t, int>> kv((size_t)nb);
    for (long long j = 0; j < nb; ++j) kv[j] = {key(coord(b[3 * j], 0), coord(b[3 * j + 1], 1), coord(b[3 * j + 2], 2)), (int)j};
    std::sort(kv.begin(), kv.end());   // ascending index inside a cell
    order.resize((size_t)nb);
    cells.clear(); start.clear();
    for (long long j = 0; j < nb; ++j) {
      order[j] = kv[j].second;
      if (j == 0 || kv[j].first != kv[j - 1].first) cells.push_back({kv[j].first, (int)j});
    }
    for (auto &c : cells) start.push_back(c.second);
    start.push_back((int)nb);
  }
  static void take(float d, int j, float &best, int &bi) {
    if (d < best || (d == best && j < bi)) { best = d; bi = j; }
  }
  // d2 of the nearest point (+inf and idx -1 for a non-finite query)
  float query(const float *q, int &idx) const {
    idx = -1;
    float best = FINF;
    if (!finite3(q)) return FINF;
    if (!grid) {
      for (long long j = 0; j < n; ++j) take(icp_d2(q[0], q[1], q[2], B + 3 * j), (int)j, best, idx);
      return best;
    }
    long long c[3];
    for (int a = 0; a < 3; ++a) c[a] = coord(q[a], a);
    long long kmax = 0;
    for (int a = 0; a < 3; ++a) kmax = std::max(kmax, std::max(c[a], gm[a] - c[a]));
    double out2 = 0.0;   // how far the query lies outside its (clamped) cell, per axis
    for (int a = 0; a < 3; ++a) {
      const double lo = mn[a] + c[a] * h, hi = lo + h;
      const double d = q[a] < lo ? lo - q[a] : (q[a] > hi ? q[a] - hi : 0.0);
      out2 += d * d;
    }
    for (long long k = 0; k <= kmax; ++k) {
      for (long long x = std::max(c[0] - k, 0ll); x <= std::min(c[0] + k, gm[0]); ++x)
        for (long long y = std::max(c[1] - k, 0ll); y <= std::min(c[1] + k, gm[1]); ++y)
          for (long long z = std::max(c[2] - k, 0ll); z <= std::min(c[2] + k, gm[2]); ++z) {
            if (std::max(std::llabs(x - c[0]), std::max(std::llabs(y - c[1]), std::llabs(z - c[2]))) != k) continue;
            auto it = std::lower_bound(cells.begin(), cells.end(), std::make_pair(key(x, y, z), -1));
            if (it == cells.end() || it->first != key(x, y, z)) continue;
            const size_t e = (size_t)(it - cells.begin());
            for (int s = start[e]; s < start[e + 1]; ++s) take(icp_d2(q[0], q[1], q[2], B + 3 * (size_t)order[s]), order[s], best, idx);
          }
      // every point beyond ring k lies at least k h - 1e-6 h away on one axis: strictly farther than best, no tie possible
      const double lb = std::max(0.0, (double)k * h - 1e-6 * h);
      if ((double)best < (lb * lb + out2) * (1.0 - 1e-5)) break;
    }
    return best;
  }
};

struct Sum { double v[9]; unsigned long long n; };
void sum_add(Sum &x, const Sum &y) { for (int k = 0; k < 9; ++k) x.v[k] += y.v[k]; x.n += y.n; }
// the kernels' fixed tree (see the file header); point(p, acc) adds point p to acc
template <class A, class Pt, class Add>
A tree_sum(long long n, Pt point, Add add) {
  const int T = 256;
  const long long CH = 8192, nb = (n + CH - 1) / CH;
  auto tree = [&](std::vector<A> &x) {
    for (int w = T / 2; w > 0; w >>= 1)
      for (int t = 0; t < w; ++t) add(x[t], x[t + w]);
    return x[0];
  };
  std::vector<A> part((size_t)nb);
  for (long long b = 0; b < nb; ++b) {
    std::vector<A> th(T, A{});
    for (int t = 0; t < T; ++t)
      for (long long p = b * CH + t; p < std::min(b * CH + CH, n); p += T) point(p, th[t]);
    part[b] = tree(th);
  }
  std::vector<A> th(T, A{});
  for (int t = 0; t < T; ++t)
    for (long long b = t; b < nb; b += T) add(th[t], part[b]);
  return tree(th);
}

}  // namespace

// info = {iterations, state, converged, cor}; traces [max_it] (cor, mse), T_trace [max_it][16] (row-major T_k) and corr_trace
// [max_it][n_fin] (j(i) after the rejectors, -1: none, i over the finite source points) may be null; moved [ns][3] may be null.
extern "C" int icp_oracle(const float *P, long long ns, const float *Qall, long long nt_all, const double *G16, int max_it, int recip,
                          float rho, double eps_t, double eps_f, int grid, double *Rt16, int *info, double *mse_out,
                          double *fitness_out, int *cor_trace, double *mse_trace, float *T_trace, int *corr_trace, float *moved) {
  std::vector<float> Pf, Q;
  for (long long i = 0; i < ns; ++i) if (finite3(P + 3 * i)) Pf.insert(Pf.end(), P + 3 * i, P + 3 * i + 3);
  for (long long j = 0; j < nt_all; ++j) if (finite3(Qall + 3 * j)) Q.insert(Q.end(), Qall + 3 * j, Qall + 3 * j + 3);
  const long long n = (long long)Pf.size() / 3, nt = (long long)Q.size() / 3;
  if (n <= 0 || nt <= 0 || max_it < 1) return -1;
  float F[16];
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) F[4 * r + c] = G16 ? (float)G16[4 * c + r] : (r == c ? 1.f : 0.f);
  std::vector<float> W((size_t)3 * n), d2((size_t)n);
  std::vector<int> corr((size_t)n), rev((size_t)nt);
  for (long long i = 0; i < n; ++i) move16(F, &Pf[3 * i], &W[3 * i]);
  Nearest NQ;
  NQ.build(Q.data(), nt, grid != 0);
  double prev = DBL_MAX, mse = 0.0;
  int state = 0, k = 1;
  unsigned long long cor = 0;
  for (;; ++k) {
    for (long long i = 0; i < n; ++i) d2[i] = NQ.query(&W[3 * i], corr[i]);
    if (recip) {
      Nearest NW;
      NW.build(W.data(), n, grid != 0);
      std::vector<char> seen((size_t)nt, 0);
      for (long long i = 0; i < n; ++i)
        if (corr[i] >= 0 && !seen[corr[i]]) { seen[corr[i]] = 1; NW.query(&Q[3 * (size_t)corr[i]], rev[corr[i]]); }
      for (long long i = 0; i < n; ++i)
        if (corr[i] >= 0 && rev[corr[i]] != (int)i) corr[i] = -1;
    }
    if (rho > 0.f) {
      std::vector<std::pair<float, long long>> kept;
      for (long long i = 0; i < n; ++i) if (corr[i] >= 0) kept.push_back({d2[i], i});
      std::sort(kept.begin(), kept.end());
      const long long c = (long long)kept.size(), keep = (long long)std::floor(rho * (float)c);
      for (long long r = keep; r < c; ++r) corr[kept[r].second] = -1;
    }
    const Sum m1 = tree_sum<Sum>(n, [&](long long p, Sum &a) {
      const int j = corr[p];
      if (j < 0) return;
      for (int a3 = 0; a3 < 3; ++a3) { a.v[a3] += (double)W[3 * p + a3]; a.v[3 + a3] += (double)Q[3 * (size_t)j + a3]; }
      a.v[6] += (double)d2[p];
      ++a.n;
    }, sum_add);
    double mus[3], mud[3];
    for (int a = 0; a < 3; ++a) { mus[a] = m1.v[a] / (double)m1.n; mud[a] = m1.v[3 + a] / (double)m1.n; }
    const Sum m2 = tree_sum<Sum>(n, [&](long long p, Sum &a) {
      const int j = corr[p];
      if (j < 0) return;
      double ds[3], dd[3];
      for (int a3 = 0; a3 < 3; ++a3) { ds[a3] = (double)W[3 * p + a3] - mus[a3]; dd[a3] = (double)Q[3 * (size_t)j + a3] - mud[a3]; }
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) a.v[r * 3 + c] += dd[r] * ds[c];
    }, sum_add);
    cor = m1.n;
    mse = cor > 0 ? m1.v[6] / (double)cor : std::nan("");
    if (cor_trace) cor_trace[k - 1] = (int)cor;
    if (mse_trace) mse_trace[k - 1] = mse;
    if (corr_trace) std::copy(corr.begin(), corr.end(), corr_trace + (size_t)(k - 1) * n);
    float T[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    if (cor < 3) {
      state = 5;
      if (T_trace) std::copy(T, T + 16, T_trace + 16 * (size_t)(k - 1));
      break;
    }
    float mu_s[3], mu_d[3], sigma[9], R[9], t[3];
    for (int a = 0; a < 3; ++a) { mu_s[a] = (float)(m1.v[a] / (double)cor); mu_d[a] = (float)(m1.v[3 + a] / (double)cor); }
    for (int a = 0; a < 9; ++a) sigma[a] = (float)(m2.v[a] / (double)cor);
    umeyama_f32(mu_s, mu_d, sigma, R, t);
    for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) T[4 * r + c] = R[3 * r + c]; T[4 * r + 3] = t[r]; }
    if (T_trace) std::copy(T, T + 16, T_trace + 16 * (size_t)(k - 1));
    float Fn[16];
    for (int r = 0; r < 4; ++r)
      for (int c = 0; c < 4; ++c) Fn[4 * r + c] = ((T[4 * r] * F[c] + T[4 * r + 1] * F[4 + c]) + T[4 * r + 2] * F[8 + c]) + T[4 * r + 3] * F[12 + c];
    std::copy(Fn, Fn + 16, F);
    for (long long i = 0; i < n; ++i) { float o[3]; move16(T, &W[3 * i], o); std::copy(o, o + 3, &W[3 * i]); }
    if (k >= max_it) { state = 1; break; }
    const double cosa = 0.5 * ((((double)T[0] + (double)T[5]) + (double)T[10]) - 1.0);
    const double t2 = ((double)T[3] * (double)T[3] + (double)T[7] * (double)T[7]) + (double)T[11] * (double)T[11];
    if (cosa >= 1.0 - eps_t && t2 <= eps_t) { state = 2; break; }
    const double d = std::fabs(mse - prev);
    if (d < 1e-12) { state = 3; break; }
    if (d / prev < eps_f) { state = 4; break; }
    prev = mse;
  }
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) Rt16[4 * c + r] = (double)F[4 * r + c];
  info[0] = k; info[1] = state; info[2] = state != 5; info[3] = (int)cor;
  *mse_out = mse;
  // fitness: every source point moved by F, its nearest d2 (non-finite moved points take no part)
  struct Fit { double s; unsigned long long n; };
  std::vector<float> dall((size_t)ns);
  for (long long i = 0; i < ns; ++i) {
    float o[3];
    move16(F, P + 3 * i, o);
    if (moved) std::copy(o, o + 3, moved + 3 * i);
    int unused;
    dall[i] = NQ.query(o, unused);
  }
  const Fit f = tree_sum<Fit>(ns, [&](long long p, Fit &a) { if (dall[p] != FINF) { a.s += (double)dall[p]; ++a.n; } },
                              [](Fit &x, const Fit &y) { x.s += y.s; x.n += y.n; });
  *fitness_out = f.n > 0 ? f.s / (double)f.n : DBL_MAX;
  return 0;
}
