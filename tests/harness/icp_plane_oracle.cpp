// icp_plane_oracle.cpp — the canonical point-to-plane ICP of DESIGN.md §3.14, one thread (TEST INFRASTRUCTURE, built with
// -ffp-contract=off so that every float32 operation is rounded separately).  tests/icp_plane_oracle.py compiles it and checks
// the product's kernels (gh-icp_b200/csrc/ghicp_icp.cu, metric 1) against it.  The loop is icp_oracle.cpp's (§3.13) with
// another estimate; its nearest-neighbour search, fixed tree and fitness are that file's, included here.
//   set-up      N_j = the k-NN normal of §3.10 (fpfh_oracle.cpp's State::normal over the exact k_eff = min(k, n_t) nearest
//               targets of Q_j in (d2, index) order, the point itself included), (0.577, 0.577, 0.577) where it is not finite
//   estimate    c < 3: NO_CORRESPONDENCES; m = sum s / c from the pass-1 sums; per kept pair, in double from the float32
//               inputs, u = s - m, n = N_j, row r = [u_y n_z - u_z n_y, u_z n_x - u_x n_z, u_x n_y - u_y n_x, n],
//               b = (n_x (q_x - s_x) + n_y (q_y - s_y)) + n_z (q_z - s_z); the 21 sums r_a r_c (a <= c, row order) and the 6
//               sums r_a b in the same point blocks and per-thread order as pass 1, and the same halving trees applied to each
//               of the 27 components; chol_solve<6> (ghicp_solvers_math.h) -> x = (alpha, beta, gamma, t');
//               t = t' - omega x m, (omega x m) = (beta m_z - gamma m_y, gamma m_x - alpha m_z, alpha m_y - beta m_x);
//               refused, |angle| > 2^20 or a non-finite t: stop, SINGULAR (7), F unchanged;
//               T = PCL's constructTransformationMatrix with det_sincos, each entry in double, rounded once to float32
//   the rest    as point-to-point: F <- T F, W <- T W, DefaultConvergenceCriteria, fitness
#include "icp_oracle.cpp"   // Nearest, tree_sum, Sum, move16: the point-to-point oracle's search and sums
#include "fpfh_oracle.cpp"  // State::normal: the k-NN normal of §3.10
#include "../../gh-icp_b200/csrc/ghicp_solvers_math.h"   // chol_solve<6>, det_sincos: the text the device runs

namespace {

// the kk smallest (d2, index) of NQ's points around the finite point q, ascending (kk <= NQ.n); NQ's rings and bound
void knn(const Nearest &NQ, const float *q, int kk, std::vector<std::pair<float, int>> &out) {
  out.clear();
  if (!NQ.grid) {
    for (long long j = 0; j < NQ.n; ++j) out.push_back({icp_d2(q[0], q[1], q[2], NQ.B + 3 * j), (int)j});
  } else {
    long long c[3];
    for (int a = 0; a < 3; ++a) c[a] = NQ.coord(q[a], a);
    long long kmax = 0;
    for (int a = 0; a < 3; ++a) kmax = std::max(kmax, std::max(c[a], NQ.gm[a] - c[a]));
    double out2 = 0.0;
    for (int a = 0; a < 3; ++a) {
      const double lo = NQ.mn[a] + c[a] * NQ.h, hi = lo + NQ.h;
      const double d = q[a] < lo ? lo - q[a] : (q[a] > hi ? q[a] - hi : 0.0);
      out2 += d * d;
    }
    std::vector<std::pair<float, int>> tmp;
    for (long long k = 0; k <= kmax; ++k) {
      for (long long x = std::max(c[0] - k, 0ll); x <= std::min(c[0] + k, NQ.gm[0]); ++x)
        for (long long y = std::max(c[1] - k, 0ll); y <= std::min(c[1] + k, NQ.gm[1]); ++y)
          for (long long z = std::max(c[2] - k, 0ll); z <= std::min(c[2] + k, NQ.gm[2]); ++z) {
            if (std::max(std::llabs(x - c[0]), std::max(std::llabs(y - c[1]), std::llabs(z - c[2]))) != k) continue;
            auto it = std::lower_bound(NQ.cells.begin(), NQ.cells.end(), std::make_pair(NQ.key(x, y, z), -1));
            if (it == NQ.cells.end() || it->first != NQ.key(x, y, z)) continue;
            const size_t e = (size_t)(it - NQ.cells.begin());
            for (int s = NQ.start[e]; s < NQ.start[e + 1]; ++s)
              out.push_back({icp_d2(q[0], q[1], q[2], NQ.B + 3 * (size_t)NQ.order[s]), NQ.order[s]});
          }
      if ((long long)out.size() < kk) continue;
      tmp = out;
      std::nth_element(tmp.begin(), tmp.begin() + (kk - 1), tmp.end());
      // every point beyond ring k lies at least k h - 1e-6 h away on one axis: strictly farther than the kk-th
      const double lb = std::max(0.0, (double)k * NQ.h - 1e-6 * NQ.h);
      if ((double)tmp[kk - 1].first < (lb * lb + out2) * (1.0 - 1e-5)) break;
    }
  }
  std::partial_sort(out.begin(), out.begin() + kk, out.end());
  out.resize(kk);
}

// the target normals (nt >= 1 finite points Q, k in 3..32) into N [nt][3]
void plane_normals(const float *Q, long long nt, const Nearest &NQ, int k, float *N) {
  State S;
  S.xyz = Q; S.n = (int)nt; S.k = k < nt ? k : (int)nt;
  S.nb.assign((size_t)nt * S.k, -1); S.d2.assign((size_t)nt * S.k, 0.f); S.have_nb.assign((size_t)nt, 0);
  S.nrm.assign(3 * (size_t)nt, 0.f); S.have_nrm.assign((size_t)nt, 0);
  std::vector<std::pair<float, int>> l;
  for (long long j = 0; j < nt; ++j) {
    if (S.k >= 3) {   // the lists of fpfh_oracle.cpp's brute force, found through NQ (its grid, when it has one)
      knn(NQ, Q + 3 * j, S.k, l);
      for (int e = 0; e < S.k; ++e) { S.nb[(size_t)j * S.k + e] = l[e].second; S.d2[(size_t)j * S.k + e] = l[e].first; }
      S.have_nb[j] = 1;
    }
    const float *v = S.normal((int)j);
    const bool fin = std::isfinite(v[0]) && std::isfinite(v[1]) && std::isfinite(v[2]);
    for (int a = 0; a < 3; ++a) N[3 * j + a] = fin ? v[a] : 0.577f;   // CheckNormals
  }
}

struct Pl { double v[27]; };
void pl_add(Pl &x, const Pl &y) { for (int k = 0; k < 27; ++k) x.v[k] += y.v[k]; }

}  // namespace

// As icp_oracle, with the estimate of §3.14 (normal_k in 3..32); normals [n_fin_target][3] (may be null) receives the target
// normals the loop reads, over the finite target points in their order.  info[1] = 7: SINGULAR.
extern "C" int icp_plane_oracle(const float *P, long long ns, const float *Qall, long long nt_all, const double *G16, int max_it,
                                int recip, float rho, double eps_t, double eps_f, int grid, int normal_k, double *Rt16, int *info,
                                double *mse_out, double *fitness_out, int *cor_trace, double *mse_trace, float *T_trace,
                                int *corr_trace, float *moved, float *normals) {
  std::vector<float> Pf, Q;
  for (long long i = 0; i < ns; ++i) if (finite3(P + 3 * i)) Pf.insert(Pf.end(), P + 3 * i, P + 3 * i + 3);
  for (long long j = 0; j < nt_all; ++j) if (finite3(Qall + 3 * j)) Q.insert(Q.end(), Qall + 3 * j, Qall + 3 * j + 3);
  const long long n = (long long)Pf.size() / 3, nt = (long long)Q.size() / 3;
  if (n <= 0 || nt <= 0 || max_it < 1 || normal_k < 3 || normal_k > 32) return -1;
  float F[16];
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) F[4 * r + c] = G16 ? (float)G16[4 * c + r] : (r == c ? 1.f : 0.f);
  std::vector<float> W((size_t)3 * n), d2((size_t)n);
  std::vector<int> corr((size_t)n), rev((size_t)nt);
  for (long long i = 0; i < n; ++i) move16(F, &Pf[3 * i], &W[3 * i]);
  Nearest NQ;
  NQ.build(Q.data(), nt, grid != 0);
  std::vector<float> N(3 * (size_t)nt);
  plane_normals(Q.data(), nt, NQ, normal_k, N.data());
  if (normals) std::copy(N.begin(), N.end(), normals);
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
    double m[3];
    for (int a = 0; a < 3; ++a) m[a] = m1.v[a] / (double)m1.n;
    const Pl acc = tree_sum<Pl>(n, [&](long long p, Pl &a) {
      const int j = corr[p];
      if (j < 0) return;
      double s[3], q[3], nn[3], u[3];
      for (int a3 = 0; a3 < 3; ++a3) {
        s[a3] = (double)W[3 * p + a3]; q[a3] = (double)Q[3 * (size_t)j + a3]; nn[a3] = (double)N[3 * (size_t)j + a3];
        u[a3] = s[a3] - m[a3];
      }
      const double r[6] = {u[1] * nn[2] - u[2] * nn[1], u[2] * nn[0] - u[0] * nn[2], u[0] * nn[1] - u[1] * nn[0], nn[0], nn[1], nn[2]};
      const double b = (nn[0] * (q[0] - s[0]) + nn[1] * (q[1] - s[1])) + nn[2] * (q[2] - s[2]);
      int e = 0;
      for (int a6 = 0; a6 < 6; ++a6)
        for (int c = a6; c < 6; ++c) a.v[e++] += r[a6] * r[c];
      for (int a6 = 0; a6 < 6; ++a6) a.v[21 + a6] += r[a6] * b;
    }, pl_add);
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
    double A[6][6], b[6], x[6] = {0, 0, 0, 0, 0, 0};
    int e = 0;
    for (int i = 0; i < 6; ++i)
      for (int j = i; j < 6; ++j) { A[i][j] = acc.v[e]; A[j][i] = acc.v[e]; ++e; }
    for (int i = 0; i < 6; ++i) b[i] = acc.v[21 + i];
    bool ok = ghicp_b200::chol_solve<6>(A, b, x);
    const double al = x[0], be = x[1], ga = x[2];
    const double t[3] = {x[3] - (be * m[2] - ga * m[1]), x[4] - (ga * m[0] - al * m[2]), x[5] - (al * m[1] - be * m[0])};
    for (int i = 0; i < 3; ++i) ok = ok && std::fabs(x[i]) <= 1048576.0 && std::fabs(t[i]) <= DBL_MAX;
    if (!ok) {
      state = 7;
      if (T_trace) std::copy(T, T + 16, T_trace + 16 * (size_t)(k - 1));
      break;
    }
    double sa, ca, sb, cb, sg, cg;
    ghicp_b200::det_sincos(al, sa, ca); ghicp_b200::det_sincos(be, sb, cb); ghicp_b200::det_sincos(ga, sg, cg);
    const double Td[12] = {cg * cb, (-sg) * ca + (cg * sb) * sa, sg * sa + (cg * sb) * ca, t[0],
                           sg * cb, cg * ca + (sg * sb) * sa, (-cg) * sa + (sg * sb) * ca, t[1],
                           -sb, cb * sa, cb * ca, t[2]};
    for (int i = 0; i < 12; ++i) T[i] = (float)Td[i];
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
  info[0] = k; info[1] = state; info[2] = state != 5 && state != 7; info[3] = (int)cor;
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

// det_sincos of ghicp_solvers_math.h over x [n]
extern "C" void icp_det_sincos(const double *x, long long n, double *s, double *c) {
  for (long long i = 0; i < n; ++i) ghicp_b200::det_sincos(x[i], s[i], c[i]);
}
