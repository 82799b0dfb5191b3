// gicp_oracle.cpp — the canonical Generalized ICP of DESIGN.md §3.15, one thread (TEST INFRASTRUCTURE, built with
// -ffp-contract=off so that every float32 operation is rounded separately).  tests/gicp_oracle.py compiles it and checks the
// product's kernels (gh-icp_b200/csrc/ghicp_icp.cu, metric 2) against it.  The correspondences, the sum tree and the fitness
// are the point-to-point oracle's (icp_oracle.cpp), the k-NN normals the point-to-plane oracle's (icp_plane_oracle.cpp over
// fpfh_oracle.cpp), all included here unchanged.
//   set-up      F = the guess in float32, W = F P; N_s, N_t = the k-NN normals of the finite source and target points (CheckNormals'
//               substitute where not finite)
//   pairs       §3.13's nearest target of W_i, then the gate (double)d_i < 1e12, then reciprocity and trimming; c < 3: stop
//               (NO_CORRESPONDENCES, 5); m = sum q / c over the kept pairs (pass-1 sums), R = F's rotation widened to double,
//               M_i = gicp_mahalanobis(R, N_s,i, N_t,j) (ghicp_solvers_math.h)
//   inner       F_0 = F; for j = 0 .. 19: per kept pair in double from the float32 inputs, w = F_j P_i (move16), r0 = w - q,
//               u = w - m, J = [e_x x u, e_y x u, e_z x u, I]; the 21 upper-triangle sums of J^T M J (row order), the 6 of
//               J^T M r0 and f_j = sum r0^T M r0, each in the tree; j > 0 and f_j > f_{j-1}: F = F_{j-1}, end (rejected);
//               chol_solve<6>(H, -g) -> (alpha, beta, gamma, t'), t = t' - omega x m; refused, |angle| > 2^20 or a non-finite t:
//               SINGULAR (7), F = its value at the start of the iteration, stop; dT = constructTransformationMatrix with
//               det_sincos in double rounded once to float32, F_{j+1} = dT F_j (float32 product); end when
//               delta(F_{j+1}, F_j) < 1 (tolerance) or j + 1 = 20 (steps)
//   outer       W = F P; k >= max_iterations: ITERATIONS (1); delta(F at the start, F) < 1: TRANSFORM (2)
//   delta       PCL's: max over the 16 entries of |a - b| (float32 difference) times 1 / eps_r in the 3 x 3 block, 1 / eps_t
//               elsewhere (a NaN product is skipped)
#include "icp_plane_oracle.cpp"   // icp_oracle.cpp (Nearest, tree_sum, Sum, move16) and plane_normals (fpfh_oracle.cpp)

namespace {

struct Gs { double v[28]; };
void gs_add(Gs &x, const Gs &y) { for (int k = 0; k < 28; ++k) x.v[k] += y.v[k]; }

double gicp_delta(const float *a, const float *b, double eps_t, double eps_r) {
  const double rr = 1.0 / eps_r, rt = 1.0 / eps_t;
  double d = 0.0;
  for (int k = 0; k < 4; ++k)
    for (int l = 0; l < 4; ++l) {
      const double c = (k < 3 && l < 3 ? rr : rt) * (double)std::fabs(a[4 * k + l] - b[4 * k + l]);
      if (c > d) d = c;
    }
  return d;
}

void compose(const float *T, const float *F, float *out) {
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) out[4 * r + c] = ((T[4 * r] * F[c] + T[4 * r + 1] * F[4 + c]) + T[4 * r + 2] * F[8 + c]) + T[4 * r + 3] * F[12 + c];
}

}  // namespace

// As icp_oracle, with the estimate of §3.15 (normal_k in 3..32, eps_r > 0; eps_f is not read).  F_trace [max_it][16] (may be
// null) receives F after each iteration (row-major float32); inner [max_it][2] (may be null) each iteration's inner passes
// (sums evaluated) and how the inner loop ended (1 tolerance, 2 twenty steps, 3 a rejected step, 0 no inner loop);
// normals_s [n_fin_source][3] / normals_t [n_fin_target][3] (may be null) the normals the loop reads.
extern "C" int gicp_oracle(const float *P, long long ns, const float *Qall, long long nt_all, const double *G16, int max_it, int recip,
                           float rho, double eps_t, double eps_r, int grid, int normal_k, double *Rt16, int *info, double *mse_out,
                           double *fitness_out, int *cor_trace, double *mse_trace, float *F_trace, int *inner, int *corr_trace,
                           float *moved, float *normals_s, float *normals_t) {
  std::vector<float> Pf, Q;
  for (long long i = 0; i < ns; ++i) if (finite3(P + 3 * i)) Pf.insert(Pf.end(), P + 3 * i, P + 3 * i + 3);
  for (long long j = 0; j < nt_all; ++j) if (finite3(Qall + 3 * j)) Q.insert(Q.end(), Qall + 3 * j, Qall + 3 * j + 3);
  const long long n = (long long)Pf.size() / 3, nt = (long long)Q.size() / 3;
  if (n <= 0 || nt <= 0 || max_it < 1 || normal_k < 3 || normal_k > 32 || !(eps_r > 0.0)) return -1;
  float F[16];
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) F[4 * r + c] = G16 ? (float)G16[4 * c + r] : (r == c ? 1.f : 0.f);
  std::vector<float> W((size_t)3 * n), d2((size_t)n);
  std::vector<int> corr((size_t)n), rev((size_t)nt);
  for (long long i = 0; i < n; ++i) move16(F, &Pf[3 * i], &W[3 * i]);
  Nearest NQ, NP;
  NQ.build(Q.data(), nt, grid != 0);
  NP.build(Pf.data(), n, grid != 0);
  std::vector<float> Nt(3 * (size_t)nt), Ns(3 * (size_t)n);
  plane_normals(Q.data(), nt, NQ, normal_k, Nt.data());
  plane_normals(Pf.data(), n, NP, normal_k, Ns.data());
  if (normals_t) std::copy(Nt.begin(), Nt.end(), normals_t);
  if (normals_s) std::copy(Ns.begin(), Ns.end(), normals_s);
  double mse = 0.0;
  int state = 0, k = 1;
  unsigned long long cor = 0;
  std::vector<double> M((size_t)6 * n);
  for (;; ++k) {
    for (long long i = 0; i < n; ++i) {
      d2[i] = NQ.query(&W[3 * i], corr[i]);
      if (!((double)d2[i] < 1e12)) corr[i] = -1;   // gicp_reg's corr_dist_threshold 1e6, squared
    }
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
    cor = m1.n;
    mse = cor > 0 ? m1.v[6] / (double)cor : std::nan("");
    if (cor_trace) cor_trace[k - 1] = (int)cor;
    if (mse_trace) mse_trace[k - 1] = mse;
    if (corr_trace) std::copy(corr.begin(), corr.end(), corr_trace + (size_t)(k - 1) * n);
    if (inner) { inner[2 * (k - 1)] = 0; inner[2 * (k - 1) + 1] = 0; }
    if (cor < 3) {
      state = 5;
      if (F_trace) std::copy(F, F + 16, F_trace + 16 * (size_t)(k - 1));
      break;
    }
    double R[9], m[3];
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) R[3 * r + c] = (double)F[4 * r + c];
    for (int a = 0; a < 3; ++a) m[a] = m1.v[3 + a] / (double)cor;
    for (long long p = 0; p < n; ++p)
      if (corr[p] >= 0) ghicp_b200::gicp_mahalanobis(R, &Ns[3 * p], &Nt[3 * (size_t)corr[p]], &M[6 * p]);
    float Fs[16], Fj[16], Fp[16];
    std::copy(F, F + 16, Fs); std::copy(F, F + 16, Fj);
    double fprev = 0.0;
    int passes = 0, why = 0;
    for (int j = 0; j < 20 && why == 0 && state == 0; ++j) {
      ++passes;
      const Gs acc = tree_sum<Gs>(n, [&](long long p, Gs &a) {
        const int jj = corr[p];
        if (jj < 0) return;
        float w[3];
        move16(Fj, &Pf[3 * p], w);
        const double *Mp = &M[6 * p];
        const double q[3] = {(double)Q[3 * (size_t)jj], (double)Q[3 * (size_t)jj + 1], (double)Q[3 * (size_t)jj + 2]};
        const double r[3] = {(double)w[0] - q[0], (double)w[1] - q[1], (double)w[2] - q[2]};
        const double u[3] = {(double)w[0] - m[0], (double)w[1] - m[1], (double)w[2] - m[2]};
        const double J[3][3] = {{0.0, -u[2], u[1]}, {u[2], 0.0, -u[0]}, {-u[1], u[0], 0.0}};
        double MJ[3][3], Mr[3];
        for (int c = 0; c < 3; ++c) {
          MJ[c][0] = (Mp[0] * J[c][0] + Mp[1] * J[c][1]) + Mp[2] * J[c][2];
          MJ[c][1] = (Mp[1] * J[c][0] + Mp[3] * J[c][1]) + Mp[4] * J[c][2];
          MJ[c][2] = (Mp[2] * J[c][0] + Mp[4] * J[c][1]) + Mp[5] * J[c][2];
        }
        Mr[0] = (Mp[0] * r[0] + Mp[1] * r[1]) + Mp[2] * r[2];
        Mr[1] = (Mp[1] * r[0] + Mp[3] * r[1]) + Mp[4] * r[2];
        Mr[2] = (Mp[2] * r[0] + Mp[4] * r[1]) + Mp[5] * r[2];
        const double Mi[3][3] = {{Mp[0], Mp[1], Mp[2]}, {Mp[1], Mp[3], Mp[4]}, {Mp[2], Mp[4], Mp[5]}};
        int e = 0;
        for (int b = 0; b < 3; ++b) {
          for (int c = b; c < 3; ++c) a.v[e++] += (J[b][0] * MJ[c][0] + J[b][1] * MJ[c][1]) + J[b][2] * MJ[c][2];
          for (int c = 0; c < 3; ++c) a.v[e++] += MJ[b][c];
        }
        for (int b = 0; b < 3; ++b)
          for (int c = b; c < 3; ++c) a.v[e++] += Mi[b][c];
        for (int b = 0; b < 3; ++b) a.v[21 + b] += (J[b][0] * Mr[0] + J[b][1] * Mr[1]) + J[b][2] * Mr[2];
        for (int b = 0; b < 3; ++b) a.v[24 + b] += Mr[b];
        a.v[27] += (r[0] * Mr[0] + r[1] * Mr[1]) + r[2] * Mr[2];
      }, gs_add);
      const double f = acc.v[27];
      if (j > 0 && f > fprev) { std::copy(Fp, Fp + 16, Fj); why = 3; break; }
      double A[6][6], b[6], x[6] = {0, 0, 0, 0, 0, 0};
      int e = 0;
      for (int i = 0; i < 6; ++i)
        for (int jj = i; jj < 6; ++jj) { A[i][jj] = acc.v[e]; A[jj][i] = acc.v[e]; ++e; }
      for (int i = 0; i < 6; ++i) b[i] = -acc.v[21 + i];
      bool ok = ghicp_b200::chol_solve<6>(A, b, x);
      const double al = x[0], be = x[1], ga = x[2];
      const double t[3] = {x[3] - (be * m[2] - ga * m[1]), x[4] - (ga * m[0] - al * m[2]), x[5] - (al * m[1] - be * m[0])};
      for (int i = 0; i < 3; ++i) ok = ok && std::fabs(x[i]) <= 1048576.0 && std::fabs(t[i]) <= DBL_MAX;
      if (!ok) { state = 7; break; }
      double sa, ca, sb, cb, sg, cg;
      ghicp_b200::det_sincos(al, sa, ca); ghicp_b200::det_sincos(be, sb, cb); ghicp_b200::det_sincos(ga, sg, cg);
      const double Td[12] = {cg * cb, (-sg) * ca + (cg * sb) * sa, sg * sa + (cg * sb) * ca, t[0],
                             sg * cb, cg * ca + (sg * sb) * sa, (-cg) * sa + (sg * sb) * ca, t[1],
                             -sb, cb * sa, cb * ca, t[2]};
      float T[16] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1};
      for (int i = 0; i < 12; ++i) T[i] = (float)Td[i];
      float Fn[16];
      compose(T, Fj, Fn);
      const bool small = gicp_delta(Fn, Fj, eps_t, eps_r) < 1.0;
      std::copy(Fj, Fj + 16, Fp); std::copy(Fn, Fn + 16, Fj);
      fprev = f;
      if (small) why = 1;
      else if (j + 1 == 20) why = 2;
    }
    if (inner) { inner[2 * (k - 1)] = passes; inner[2 * (k - 1) + 1] = why; }
    if (state == 7) {
      if (F_trace) std::copy(F, F + 16, F_trace + 16 * (size_t)(k - 1));
      break;
    }
    std::copy(Fj, Fj + 16, F);
    if (F_trace) std::copy(F, F + 16, F_trace + 16 * (size_t)(k - 1));
    for (long long i = 0; i < n; ++i) move16(F, &Pf[3 * i], &W[3 * i]);
    if (k >= max_it) { state = 1; break; }
    if (gicp_delta(F, Fs, eps_t, eps_r) < 1.0) { state = 2; break; }
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
  const Fit fit = tree_sum<Fit>(ns, [&](long long p, Fit &a) { if (dall[p] != FINF) { a.s += (double)dall[p]; ++a.n; } },
                                [](Fit &x, const Fit &y) { x.s += y.s; x.n += y.n; });
  *fitness_out = fit.n > 0 ? fit.s / (double)fit.n : DBL_MAX;
  return 0;
}

// gicp_mahalanobis of ghicp_solvers_math.h over n pairs: R [9] row-major, ns / nt [n][3], M [n][6]
extern "C" void gicp_oracle_mahalanobis(const double *R, const float *ns, const float *nt, long long n, double *M) {
  for (long long i = 0; i < n; ++i) ghicp_b200::gicp_mahalanobis(R, ns + 3 * i, nt + 3 * i, M + 6 * i);
}
