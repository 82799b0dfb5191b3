// auction_sim.cpp — CPU model of the GPU auction (gh-icp_b200/csrc/ghicp_auction.cu) on a config-2-like
// KM instance (SURVEY.md §8d generator: BSC-441, V=4, 60 % overlap), used to choose the epsilon schedule /
// problem formulation for the dense first iterations WITHOUT a GPU: the number of synchronous (Jacobi)
// bidding rounds and the bidders per round are properties of the algorithm, not of the hardware.
//
//   g++ -O3 -march=native -fopenmp -std=c++17 tools/auction_sim.cpp -o tools/auction_sim
//   tools/auction_sim N it [mode ...]
//
// Development tool only: not part of the product, not used by tests or bench.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <string>
#include <vector>
#include <omp.h>

typedef long long ll;

struct Inst {
  int N = 0, M = 0;
  std::vector<ll> rp; std::vector<int> col; std::vector<double> g;   // CSR (persons = rows)
  std::vector<ll> cp; std::vector<int> row; std::vector<double> cg;  // CSC
  double penalty = 0, max_gain = 0;
};

static inline uint64_t splitmix(uint64_t &s) {
  uint64_t z = (s += 0x9E3779B97F4A7C15ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
static inline double u01(uint64_t &s) { return (splitmix(s) >> 11) * (1.0 / 9007199254740992.0); }

// iteration 0: CD = FD (WED = 0); iteration 1: CD = WED*scale*dist + WFD*FD with the source already aligned up to
// `misalign` metres; penalty = mean - 2 std (floor 5) in both (src/ghicp_reg.cpp:279-287).
static Inst make_instance(int N, int M, int it, uint64_t seed, double misalign) {
  const int bits = 441, W = 7, V = 4;
  const double p_one = 0.35, p_flip = 0.08, overlap = 0.6;
  uint64_t s = seed;
  std::vector<uint64_t> tb((size_t)M * W), sb((size_t)V * N * W);
  auto rnd_desc = [&](uint64_t *d, double p) {
    for (int w = 0; w < W; ++w) d[w] = 0;
    for (int k = 0; k < bits; ++k) if (u01(s) < p) d[k >> 6] |= 1ull << (k & 63);
  };
  for (int j = 0; j < M; ++j) rnd_desc(&tb[(size_t)j * W], p_one);
  for (size_t x = 0; x < (size_t)V * N; ++x) rnd_desc(&sb[x * W], p_one);
  const int K = (int)std::floor(overlap * std::min(N, M));
  std::vector<int> perm(M);
  for (int j = 0; j < M; ++j) perm[j] = j;
  for (int j = M - 1; j > 0; --j) std::swap(perm[j], perm[splitmix(s) % (uint64_t)(j + 1)]);
  for (int i = 0; i < K; ++i) {
    uint64_t fl[7];
    rnd_desc(fl, p_flip);
    for (int w = 0; w < W; ++w) sb[(size_t)i * W + w] = tb[(size_t)perm[i] * W + w] ^ fl[w];
  }
  // coordinates (only used for it >= 1)
  const double E[3] = {200, 200, 40};
  std::vector<double> T((size_t)M * 3), S((size_t)N * 3);
  std::mt19937_64 gen(seed ^ 0x1234567);
  std::normal_distribution<double> nd(0.0, 0.05);
  for (int j = 0; j < M; ++j) for (int k = 0; k < 3; ++k) T[(size_t)j * 3 + k] = u01(s) * E[k];
  for (int i = 0; i < N; ++i) for (int k = 0; k < 3; ++k) S[(size_t)i * 3 + k] = u01(s) * E[k];
  for (int i = 0; i < K; ++i) for (int k = 0; k < 3; ++k) S[(size_t)i * 3 + k] = T[(size_t)perm[i] * 3 + k] + nd(gen) + misalign * (k == 0 ? 1 : -0.5);
  const double scale = (double)(float)(0.005f * (float)(E[0] + E[1] + E[2]));
  const double WFD = it == 0 ? 1.0 : std::exp(-1.0 * it / 6.0), WED = 1.0 - WFD;

  auto cd_of = [&](int i, int j) -> double {
    int best = 1 << 30;
    for (int v = 0; v < V; ++v) {
      const uint64_t *a = &sb[((size_t)v * N + i) * W], *b = &tb[(size_t)j * W];
      int h = 0;
      for (int w = 0; w < W; ++w) h += __builtin_popcountll(a[w] ^ b[w]);
      best = std::min(best, h);
    }
    double cd = WFD * best;
    if (WED != 0.0) {
      double d2 = 0;
      for (int k = 0; k < 3; ++k) { double d = S[(size_t)i * 3 + k] - T[(size_t)j * 3 + k]; d2 += d * d; }
      cd += WED * scale * std::sqrt(d2);
    }
    return cd;
  };
  double sum = 0, sumsq = 0;
#pragma omp parallel for reduction(+ : sum, sumsq) schedule(dynamic, 64)
  for (int i = 0; i < N; ++i) {
    double a = 0, b = 0;
    for (int j = 0; j < M; ++j) { double c = cd_of(i, j); a += c; b += c * c; }
    sum += a; sumsq += b;
  }
  const double mean = sum / ((double)N * M), var = sumsq / ((double)N * M) - mean * mean;
  double penalty = mean - 2.0 * std::sqrt(var);
  if (penalty < 5.0) penalty = 5.0;
  Inst I; I.N = N; I.M = M; I.penalty = penalty;
  std::vector<std::vector<std::pair<int, double>>> rows(N);
#pragma omp parallel for schedule(dynamic, 64)
  for (int i = 0; i < N; ++i)
    for (int j = 0; j < M; ++j) { double c = cd_of(i, j); if (c < penalty) rows[i].push_back({j, penalty - c}); }
  I.rp.assign(N + 1, 0);
  for (int i = 0; i < N; ++i) I.rp[i + 1] = I.rp[i] + (ll)rows[i].size();
  I.col.resize(I.rp[N]); I.g.resize(I.rp[N]);
  for (int i = 0; i < N; ++i) for (size_t k = 0; k < rows[i].size(); ++k) { I.col[I.rp[i] + k] = rows[i][k].first; I.g[I.rp[i] + k] = rows[i][k].second; I.max_gain = std::max(I.max_gain, rows[i][k].second); }
  I.cp.assign(M + 1, 0);
  for (ll k = 0; k < I.rp[N]; ++k) I.cp[I.col[k] + 1]++;
  for (int j = 0; j < M; ++j) I.cp[j + 1] += I.cp[j];
  I.row.resize(I.rp[N]); I.cg.resize(I.rp[N]);
  std::vector<ll> cur(I.cp.begin(), I.cp.end() - 1);
  for (int i = 0; i < N; ++i) for (ll k = I.rp[i]; k < I.rp[i + 1]; ++k) { ll p = cur[I.col[k]]++; I.row[p] = i; I.cg[p] = I.g[k]; }
  fprintf(stderr, "instance N=%d M=%d it=%d: mean %.3f std %.3f penalty %.3f nnz %lld (%.1f / row) max gain %.3f\n", N, M, it, mean,
          std::sqrt(var), penalty, I.rp[N], (double)I.rp[N] / N, I.max_gain);
  return I;
}

// ---- the auction model -------------------------------------------------------------------------------
static inline unsigned tie_key(int who, int idx) {
  unsigned h = (unsigned)idx * 0x9E3779B1u ^ ((unsigned)who * 0x85EBCA77u + 0xC2B2AE3Du);
  h ^= h >> 15; h *= 0x2C1B3C6Du; h ^= h >> 12;
  return h;
}
static inline bool tie_less(int who, int a, int b) { unsigned ka = tie_key(who, a), kb = tie_key(who, b); return ka < kb || (ka == kb && a < b); }

struct Stats {
  ll rounds = 0, grid_rounds = 0, tail_rounds = 0, bids = 0, edges = 0;
  double est_us = 0;
  void add(const Stats &o) { rounds += o.rounds; grid_rounds += o.grid_rounds; tail_rounds += o.tail_rounds; bids += o.bids; edges += o.edges; est_us += o.est_us; }
};
// time model of one round (cost per full-grid round and per CTA-0 round: inputs of the model, not measurements)
static void account(Stats &st, ll n_active, ll edges, int small_n) {
  st.rounds++; st.bids += n_active; st.edges += edges;
  if (n_active > small_n) { st.grid_rounds++; st.est_us += 12.0 + (double)edges * 12.0 / 2.5e6; }   // 2.5 TB/s effective on the CSR
  else { st.tail_rounds++; st.est_us += 8.0 + 1.0 * std::ceil((double)n_active / 16.0) * std::max(1.0, (double)edges / std::max<ll>(1, n_active) / 256.0) * 4.0; }
}

struct Auction {
  // generic bipartite problem: P persons, O objects, person adjacency in CSR, object adjacency in CSC
  int P, O;
  const ll *rp; const int *col; const double *g;
  const ll *cp; const int *row; const double *cg;
  std::vector<double> price, profit;
  std::vector<int> assign, owner;  // assign: -1 unassigned, -2 dummy
  bool has_dummy = true;           // persons own a private zero-gain dummy
  int small_fwd = 64, small_rev = 64;
  Stats fwd, rev;

  void init() { price.assign(O, 0.0); profit.assign(P, 0.0); assign.assign(P, -1); owner.assign(O, -1); }

  // one forward phase: all persons in `act` bid until none is unassigned
  void forward(std::vector<int> act, double eps, ll max_rounds = 100000000) {
    std::vector<int> bid_obj(P), next;
    std::vector<double> bid_val(P), bid_gain(P);
    std::vector<uint64_t> bidmax(O, 0);
    ll rounds = 0;
    while (!act.empty() && rounds < max_rounds) {
      ll edges = 0;
      const int n = (int)act.size();
#pragma omp parallel for reduction(+ : edges) schedule(dynamic, 64) if (n > 256)
      for (int a = 0; a < n; ++a) {
        const int i = act[a];
        double best = -1e300, second = -1e300, bg = 0; int bi = -1;
        for (ll k = rp[i]; k < rp[i + 1]; ++k) {
          const int j = col[k]; const double v = g[k] - price[j];
          if (v > best || (v == best && bi >= 0 && tie_less(i, j, bi))) { second = best; best = v; bi = j; bg = g[k]; }
          else if (v > second) second = v;
        }
        edges += rp[i + 1] - rp[i];
        if (bi < 0 || (has_dummy && best <= 0.0)) { bid_obj[i] = -1; }
        else {
          const double wv = has_dummy ? std::max(second, 0.0) : second;
          double np = price[bi] + (best - wv) + eps;
          if (!has_dummy && second < -1e200) np = price[bi] + eps + 1e6;  // single option: unbeatable bid
          bid_obj[i] = bi; bid_val[i] = np; bid_gain[i] = bg;
        }
      }
      for (int a = 0; a < n; ++a) {
        const int i = act[a];
        if (bid_obj[i] < 0) { assign[i] = -2; profit[i] = 0; continue; }
        float f = (float)bid_val[i]; uint32_t fb; memcpy(&fb, &f, 4);
        uint64_t key = ((uint64_t)fb << 32) | (uint32_t)(i + 1);
        if (key > bidmax[bid_obj[i]]) bidmax[bid_obj[i]] = key;
      }
      next.clear();
      for (int a = 0; a < n; ++a) {
        const int i = act[a];
        if (assign[i] != -1) continue;
        const int j = bid_obj[i];
        if ((int)(bidmax[j] & 0xffffffffu) - 1 == i) {
          const int prev = owner[j];
          owner[j] = i; price[j] = bid_val[i]; assign[i] = j; profit[i] = bid_gain[i] - bid_val[i];
          if (prev >= 0) { assign[prev] = -1; next.push_back(prev); }
        } else next.push_back(i);
      }
      for (int a = 0; a < n; ++a) if (bid_obj[act[a]] >= 0) bidmax[bid_obj[act[a]]] = 0;
      account(fwd, n, edges, small_fwd);
      if (getenv("HIST")) fprintf(stderr, "%d ", n);
      if (getenv("TRACE") && n <= 2) { const int i = act[0]; fprintf(stderr, "    r%lld n=%d person %d -> obj %d price %.4f (incr %.4f) deg %lld\n", rounds, n, i, bid_obj[i], bid_obj[i] >= 0 ? bid_val[i] : 0.0, bid_obj[i] >= 0 ? bid_val[i] - (price[bid_obj[i]] == bid_val[i] ? 0 : 0) : 0.0, rp[i + 1] - rp[i]); }
      act.swap(next);
      ++rounds;
    }
  }
  // SYMMETRIC formulation (what the reference's padded n x n matrix is): every person can take EVERY object, non-candidate
  // objects at gain 0; all objects end up assigned, so there is no dummy, no free object and no reverse phase.
  // Jacobi rounds; a bidder looks at all O objects (the model does it by brute force; a kernel would use the candidate list
  // plus the globally cheapest objects).
  void forward_sym(std::vector<int> act, double eps, ll max_rounds = 100000000) {
    std::vector<int> bid_obj(P), next;
    std::vector<double> bid_val(P), bid_gain(P);
    std::vector<uint64_t> bidmax(O, 0);
    ll rounds = 0;
    while (!act.empty() && rounds < max_rounds) {
      ll edges = 0;
      const int n = (int)act.size();
#pragma omp parallel reduction(+ : edges)
      {
        std::vector<double> gg(O, 0.0);
#pragma omp for schedule(dynamic, 16)
        for (int a = 0; a < n; ++a) {
          const int i = act[a];
          for (ll k = rp[i]; k < rp[i + 1]; ++k) gg[col[k]] = g[k];
          double best = -1e300, second = -1e300, bg = 0; int bi = -1;
          for (int j = 0; j < O; ++j) {
            const double v = gg[j] - price[j];
            if (v > best || (v == best && bi >= 0 && tie_less(i, j, bi))) { second = best; best = v; bi = j; bg = gg[j]; }
            else if (v > second) second = v;
          }
          for (ll k = rp[i]; k < rp[i + 1]; ++k) gg[col[k]] = 0.0;
          edges += rp[i + 1] - rp[i];
          bid_obj[i] = bi; bid_val[i] = price[bi] + (best - second) + eps; bid_gain[i] = bg;
        }
      }
      for (int a = 0; a < n; ++a) {
        const int i = act[a];
        float f = (float)bid_val[i]; uint32_t fb; memcpy(&fb, &f, 4);
        uint64_t key = ((uint64_t)fb << 32) | (uint32_t)(i + 1);
        if (key > bidmax[bid_obj[i]]) bidmax[bid_obj[i]] = key;
      }
      next.clear();
      for (int a = 0; a < n; ++a) {
        const int i = act[a];
        const int j = bid_obj[i];
        if ((int)(bidmax[j] & 0xffffffffu) - 1 == i) {
          const int prev = owner[j];
          owner[j] = i; price[j] = bid_val[i]; assign[i] = j; profit[i] = bid_gain[i] - bid_val[i];
          if (prev >= 0) { assign[prev] = -1; next.push_back(prev); }
        } else next.push_back(i);
      }
      for (int a = 0; a < n; ++a) bidmax[bid_obj[act[a]]] = 0;
      account(fwd, n, edges, small_fwd);
      if (getenv("HIST")) fprintf(stderr, "%d ", n);
      act.swap(next);
      ++rounds;
    }
  }
  double free_price_sum() const { double D = 0; for (int j = 0; j < O; ++j) if (owner[j] < 0) D += price[j]; return D; }

  // reverse phase: free objects with positive price lower their price / attract persons
  // d_budget >= 0: stop as soon as D = sum of the prices of the objects still free (= the active list) is within the budget:
  // the bound OPT - ours <= n*eps + D holds at every round boundary (dual eps-feasibility is an invariant of the reverse
  // auction), so the rest of the displacement chains need not be followed.
  double d_budget = -1.0;
  ll rev_cut_round = -1;
  void reverse(double eps, ll max_rounds = 100000000) {
    std::vector<int> act, next;
    for (int j = 0; j < O; ++j) if (owner[j] < 0 && price[j] > 0.0) act.push_back(j);
    std::vector<int> bid_obj(O, -1); std::vector<double> bid_val(O), bid_aux(O);
    std::vector<uint64_t> bidmax(P, 0);
    ll rounds = 0;
    while (!act.empty() && rounds < max_rounds) {
      ll edges = 0;
      const int n = (int)act.size();
      if (d_budget >= 0.0) {
        double Dc = 0; for (int a = 0; a < n; ++a) Dc += price[act[a]];
        if (getenv("DTRACE") && (rounds % 50 == 0 || n <= 4)) fprintf(stderr, "    rev round %lld active %d D %.2f\n", rounds, n, Dc);
        if (Dc <= d_budget) { rev_cut_round = rounds; break; }
      }
#pragma omp parallel for reduction(+ : edges) schedule(dynamic, 64) if (n > 256)
      for (int a = 0; a < n; ++a) {
        const int j = act[a];
        double best = -1e300, second = -1e300; int bi = -1;
        for (ll k = cp[j]; k < cp[j + 1]; ++k) {
          const int i = row[k]; const double v = cg[k] - profit[i];
          if (v > best || (v == best && bi >= 0 && tie_less(j, i, bi))) { second = best; best = v; bi = i; }
          else if (v > second) second = v;
        }
        edges += cp[j + 1] - cp[j];
        if (bi < 0 || best <= eps) { bid_obj[j] = -1; }
        else { bid_obj[j] = bi; bid_val[j] = std::min(best, (best - second) + eps); bid_aux[j] = best; }
      }
      for (int a = 0; a < n; ++a) {
        const int j = act[a];
        if (bid_obj[j] < 0) { price[j] = 0.0; continue; }
        float f = (float)bid_val[j]; uint32_t fb; memcpy(&fb, &f, 4);
        uint64_t key = ((uint64_t)fb << 32) | (uint32_t)(j + 1);
        if (key > bidmax[bid_obj[j]]) bidmax[bid_obj[j]] = key;
      }
      next.clear();
      for (int a = 0; a < n; ++a) {
        const int j = act[a];
        const int i = bid_obj[j];
        if (i < 0) continue;
        if ((int)(bidmax[i] & 0xffffffffu) - 1 == j) {
          const int old = assign[i];
          assign[i] = j; owner[j] = i; price[j] = bid_aux[j] - bid_val[j]; profit[i] += bid_val[j];
          if (old >= 0) { owner[old] = -1; if (price[old] > 0.0) next.push_back(old); }
        } else next.push_back(j);
      }
      for (int a = 0; a < n; ++a) if (bid_obj[act[a]] >= 0) bidmax[bid_obj[act[a]]] = 0;
      account(rev, n, edges, small_rev);
      if (getenv("HISTR")) fprintf(stderr, "R%d ", n);
      act.swap(next);
      ++rounds;
    }
  }
  // a-posteriori optimality certificate: OPT - ours <= sum_i (best_i - cur_i) + sum_{free j} price_j
  // (dual: profit_i = max(0, max_k g_ik - p_k), p >= 0)
  void certificate(double &viol, double &D) const {
    double v = 0;
#pragma omp parallel for reduction(+ : v) schedule(dynamic, 64)
    for (int i = 0; i < P; ++i) {
      double best = 0.0, cur = 0.0;
      for (ll k = rp[i]; k < rp[i + 1]; ++k) { const double x = g[k] - price[col[k]]; best = std::max(best, x); if (col[k] == assign[i]) cur = x; }
      v += best - cur;
    }
    viol = v; D = free_price_sum();
  }
  // Price refinement for the FIXED matching: least prices p >= 0 with p_k >= p_a(i) + g_ik - g_ia(i) for matched i,
  // p_k >= g_ik for unmatched i (monotone Jacobi sweeps from p = 0 = Bellman-Ford longest paths), then the dual bound
  // G = sum_i max(0, max_k g_ik - p_k) + sum_j p_j - gain(X).  Returns G; sweeps used in *sweeps.
  double refine_prices(int max_sweeps, int *sweeps, double damp = 0.0) {
    std::vector<double> gia(P, 0.0);
    for (int i = 0; i < P; ++i) if (assign[i] >= 0) for (ll k = rp[i]; k < rp[i + 1]; ++k) if (col[k] == assign[i]) { gia[i] = g[k]; break; }
    std::vector<double> p(O, 0.0), np(O, 0.0);
    double bestG = 1e300; std::vector<double> bestp;
    int s = 0;
    for (; s < max_sweeps; ++s) {
      bool changed = false;
#pragma omp parallel for schedule(dynamic, 64) reduction(|| : changed)
      for (int k = 0; k < O; ++k) {
        double v = 0.0;
        for (ll e = cp[k]; e < cp[k + 1]; ++e) {
          const int i = row[e];
          if (assign[i] == k) continue;
          const double c = assign[i] >= 0 ? p[assign[i]] + cg[e] - gia[i] - damp : cg[e];
          v = std::max(v, c);
        }
        np[k] = std::max(p[k], v);
        if (np[k] > p[k] + 1e-12) changed = true;
      }
      p.swap(np);
      if (!changed) break;
      if ((s & 3) == 3 || s + 1 == max_sweeps) {
        double G = 0;
        for (int j = 0; j < O; ++j) G += p[j];
        for (int i = 0; i < P; ++i) { double b = 0; for (ll k = rp[i]; k < rp[i + 1]; ++k) b = std::max(b, g[k] - p[col[k]]); G += b; G -= gia[i]; }
        if (G < bestG) { bestG = G; bestp = p; }
      }
    }
    double G = 0;
    for (int j = 0; j < O; ++j) G += p[j];
    for (int i = 0; i < P; ++i) { double b = 0; for (ll k = rp[i]; k < rp[i + 1]; ++k) b = std::max(b, g[k] - p[col[k]]); G += b; G -= gia[i]; }
    if (G < bestG) { bestG = G; bestp = p; }
    *sweeps = s;
    return bestG;
  }
  double total_gain() const {
    double t = 0;
    for (int i = 0; i < P; ++i) if (assign[i] >= 0) { for (ll k = rp[i]; k < rp[i + 1]; ++k) if (col[k] == assign[i]) { t += g[k]; break; } }
    return t;
  }
};

static std::vector<int> persons_with_edges(const Auction &A) { std::vector<int> v; for (int i = 0; i < A.P; ++i) if (A.rp[i + 1] > A.rp[i]) v.push_back(i); return v; }

static std::vector<double> schedule(double e0, double div, double eps_last) {
  std::vector<double> e;
  while (e0 > eps_last * 1.0000001) { e.push_back(e0); e0 /= div; }
  e.push_back(eps_last);
  return e;
}

static void report(const char *name, const Auction &A, double gain, double D, double wall) {
  Stats t = A.fwd; t.add(A.rev);
  printf("%-34s gain %.3f  D %.1f | fwd rounds %lld (grid %lld) rev rounds %lld (grid %lld) | rev bids %lld rev edges %.3g | bids %lld edges %.3g | est %.2f ms  [cpu %.1fs]\n",
         name, gain, D, A.fwd.rounds, A.fwd.grid_rounds, A.rev.rounds, A.rev.grid_rounds, A.rev.bids, (double)A.rev.edges, t.bids, (double)t.edges, t.est_us * 1e-3, wall);
  fflush(stdout);
}

int main(int argc, char **argv) {
  const int N = argc > 1 ? atoi(argv[1]) : 8000;
  const int it = argc > 2 ? atoi(argv[2]) : 0;
  const double KM_eps = 0.01;
  Inst I = make_instance(N, N, it, 2, 0.03);
  const double avg_row = (double)I.rp[N] / N;
  int small = (int)(65536.0 / std::max(1.0, avg_row));
  small = std::max(16, std::min(2048, small));
  auto tnow = []() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
  auto mk = [&]() { Auction A; A.P = I.N; A.O = I.M; A.rp = I.rp.data(); A.col = I.col.data(); A.g = I.g.data(); A.cp = I.cp.data(); A.row = I.row.data(); A.cg = I.cg.data(); A.small_fwd = A.small_rev = small; A.init(); return A; };

  for (int a = 3; a < argc || a == 3; ++a) {
    std::string mode = a < argc ? argv[a] : "base";
    double t0 = tnow();
    if (mode == "base" || mode.rfind("e0=", 0) == 0 || mode.rfind("relax=", 0) == 0) {
      // the shipped schedule: e0 = max_gain/4 (penalty/4), /5, last = KM_eps/2, reverse after the last phase when D > budget
      double e0 = I.penalty / 4.0, relax = 0.0;
      if (mode.rfind("e0=", 0) == 0) e0 = atof(mode.c_str() + 3);
      if (mode.rfind("relax=", 0) == 0) relax = atof(mode.c_str() + 6);
      Auction A = mk();
      const double epsf = getenv("EPSF") ? atof(getenv("EPSF")) : 0.5;   // eps_last = epsf*KM_eps; D budget = (1-epsf)*KM_eps*n
      auto eps = schedule(e0, 5.0, epsf * KM_eps);
      for (size_t ph = 0; ph < eps.size(); ++ph) {
        if (ph > 0) { for (auto &p : A.price) p = std::max(0.0, p - relax * eps[ph - 1]); }
        std::fill(A.owner.begin(), A.owner.end(), -1); std::fill(A.assign.begin(), A.assign.end(), -1); std::fill(A.profit.begin(), A.profit.end(), 0.0);
        ll r0 = A.fwd.rounds;
        A.forward(persons_with_edges(A), eps[ph]);
        double cv, cD; A.certificate(cv, cD);
        fprintf(stderr, "  phase %zu eps %.4f: %lld rounds, D %.1f gain %.1f  certificate: viol %.2f + D %.2f\n", ph, eps[ph], A.fwd.rounds - r0, A.free_price_sum(), A.total_gain(), cv, cD);
      }
      double D = A.free_price_sum();
      if (getenv("DCUT")) A.d_budget = (1.0 - epsf) * KM_eps * N;
      if (D > (1.0 - epsf) * KM_eps * N) A.reverse(epsf * KM_eps);
      if (A.d_budget >= 0) fprintf(stderr, "  reverse cut at round %lld (budget %.1f), D left %.2f\n", A.rev_cut_round, A.d_budget, A.free_price_sum());
      report(mode.c_str(), A, A.total_gain(), D, tnow() - t0);
    } else if (mode.rfind("sym", 0) == 0) {
      // symmetric formulation + forward eps-scaling only.  sym[=e0[,div]]
      double e0 = I.penalty / 4.0, div = 5.0;
      if (mode.size() > 4) { e0 = atof(mode.c_str() + 4); const char *c = strchr(mode.c_str(), ','); if (c) div = atof(c + 1); }
      Auction A = mk();
      auto eps = schedule(e0, div, KM_eps * 0.999);   // no D term: the whole n*eps budget goes to eps
      std::vector<int> all(N); for (int i = 0; i < N; ++i) all[i] = i;
      for (size_t ph = 0; ph < eps.size(); ++ph) {
        std::fill(A.owner.begin(), A.owner.end(), -1); std::fill(A.assign.begin(), A.assign.end(), -1);
        ll r0 = A.fwd.rounds, b0 = A.fwd.bids;
        A.forward_sym(all, eps[ph]);
        fprintf(stderr, "  sym phase %zu eps %.4f: %lld rounds %lld bids, gain %.1f\n", ph, eps[ph], A.fwd.rounds - r0, A.fwd.bids - b0, A.total_gain());
      }
      report(mode.c_str(), A, A.total_gain(), 0.0, tnow() - t0);
    } else if (mode.rfind("warm", 0) == 0) {
      // warm start across ICP iterations: solve THIS iteration's instance with the shipped schedule, then the NEXT iteration's
      // instance (same descriptors and geometry, new metric weights / penalty) starting from those prices scaled by the ratio
      // of the feature weights, assignment empty.  warm=<eps0>: first epsilon of the second solve (0 = final epsilon only).
      Auction A0 = mk();
      { auto eps = schedule(I.penalty / 4.0, 5.0, 0.5 * KM_eps);
        for (size_t ph = 0; ph < eps.size(); ++ph) {
          std::fill(A0.owner.begin(), A0.owner.end(), -1); std::fill(A0.assign.begin(), A0.assign.end(), -1); std::fill(A0.profit.begin(), A0.profit.end(), 0.0);
          A0.forward(persons_with_edges(A0), eps[ph]);
        }
        if (A0.free_price_sum() > 0.5 * KM_eps * N) A0.reverse(0.5 * KM_eps); }
      fprintf(stderr, "  iteration %d solved: gain %.1f, %lld + %lld rounds\n", it, A0.total_gain(), A0.fwd.rounds, A0.rev.rounds);
      Inst J = make_instance(N, N, it + 1, 2, 0.03);
      const double w0 = it == 0 ? 1.0 : std::exp(-1.0 * it / 6.0), w1 = std::exp(-1.0 * (it + 1) / 6.0);
      Auction B; B.P = J.N; B.O = J.M; B.rp = J.rp.data(); B.col = J.col.data(); B.g = J.g.data(); B.cp = J.cp.data(); B.row = J.row.data(); B.cg = J.cg.data();
      const double avg = (double)J.rp[N] / N;
      B.small_fwd = B.small_rev = std::max(16, std::min(2048, (int)(65536.0 / std::max(1.0, avg)))); B.init();
      for (int j = 0; j < J.M; ++j) B.price[j] = A0.price[j] * (w1 / w0);
      double e0 = mode.size() > 5 ? atof(mode.c_str() + 5) : 0.0;
      auto eps = e0 > 0 ? schedule(e0, 5.0, 0.5 * KM_eps) : std::vector<double>(1, 0.5 * KM_eps);
      double t1 = tnow();
      for (size_t ph = 0; ph < eps.size(); ++ph) {
        std::fill(B.owner.begin(), B.owner.end(), -1); std::fill(B.assign.begin(), B.assign.end(), -1); std::fill(B.profit.begin(), B.profit.end(), 0.0);
        ll r0 = B.fwd.rounds;
        B.forward(persons_with_edges(B), eps[ph]);
        fprintf(stderr, "  warm phase %zu eps %.4f: %lld rounds, D %.1f gain %.1f\n", ph, eps[ph], B.fwd.rounds - r0, B.free_price_sum(), B.total_gain());
      }
      double D = B.free_price_sum();
      if (D > 0.5 * KM_eps * N) B.reverse(0.5 * KM_eps);
      report(mode.c_str(), B, B.total_gain(), D, tnow() - t1);
      // the same instance cold, for comparison
      Auction Cc; Cc.P = J.N; Cc.O = J.M; Cc.rp = J.rp.data(); Cc.col = J.col.data(); Cc.g = J.g.data(); Cc.cp = J.cp.data(); Cc.row = J.row.data(); Cc.cg = J.cg.data();
      Cc.small_fwd = Cc.small_rev = B.small_fwd; Cc.init();
      { auto ce = schedule(J.penalty / 4.0, 5.0, 0.5 * KM_eps);
        for (size_t ph = 0; ph < ce.size(); ++ph) {
          std::fill(Cc.owner.begin(), Cc.owner.end(), -1); std::fill(Cc.assign.begin(), Cc.assign.end(), -1); std::fill(Cc.profit.begin(), Cc.profit.end(), 0.0);
          Cc.forward(persons_with_edges(Cc), ce[ph]);
        }
        double Dc = Cc.free_price_sum();
        if (Dc > 0.5 * KM_eps * N) Cc.reverse(0.5 * KM_eps);
        report("  (next iteration, cold)", Cc, Cc.total_gain(), Dc, 0.0); }
    } else if (mode.rfind("dom", 0) == 0) {
      // dominance pre-matching: a pair (i, j) with g_ij >= (best other gain of row i, or 0) + (best other gain of column j, or 0)
      // belongs to some optimal matching (exchange argument: dropping whatever i and j hold instead loses at most those two
      // terms).  Fix such pairs, delete their row and column, repeat to a fixed point; then run the shipped schedule on what is
      // left.  Reports how much of the instance the sequential auction still has to resolve.
      std::vector<char> rdead(I.N, 0), cdead(I.M, 0);
      std::vector<int> fixed_row(I.N, -1);
      double fixed_gain = 0.0; int passes = 0; ll n_fixed = 0;
      for (;; ++passes) {
        std::vector<double> r1(I.N, 0.0), r2(I.N, 0.0), c1(I.M, 0.0), c2(I.M, 0.0);
        std::vector<int> rb(I.N, -1), cb(I.M, -1);
        for (int i = 0; i < I.N; ++i) { if (rdead[i]) continue;
          for (ll k = I.rp[i]; k < I.rp[i + 1]; ++k) { const int j = I.col[k]; if (cdead[j]) continue; const double v = I.g[k];
            if (v > r1[i]) { r2[i] = r1[i]; r1[i] = v; rb[i] = j; } else if (v > r2[i]) r2[i] = v;
            if (v > c1[j]) { c2[j] = c1[j]; c1[j] = v; cb[j] = i; } else if (v > c2[j]) c2[j] = v; } }
        ll now = 0;
        for (int i = 0; i < I.N; ++i) { if (rdead[i] || rb[i] < 0) continue; const int j = rb[i];
          if (cb[j] == i && r1[i] >= r2[i] + c2[j] && !cdead[j]) { rdead[i] = 1; cdead[j] = 1; fixed_row[i] = j; fixed_gain += r1[i]; ++now; } }
        n_fixed += now;
        if (now == 0 || passes > 50) break;
      }
      // reduced instance
      std::vector<int> rmap(I.N, -1), cmap(I.M, -1); int P = 0, O = 0;
      for (int i = 0; i < I.N; ++i) if (!rdead[i]) rmap[i] = P++;
      for (int j = 0; j < I.M; ++j) if (!cdead[j]) cmap[j] = O++;
      std::vector<ll> rp(P + 1, 0), cp(O + 1, 0); std::vector<int> col, row; std::vector<double> g, cg;
      for (int i = 0; i < I.N; ++i) { if (rdead[i]) continue;
        for (ll k = I.rp[i]; k < I.rp[i + 1]; ++k) if (!cdead[I.col[k]]) { col.push_back(cmap[I.col[k]]); g.push_back(I.g[k]); }
        rp[rmap[i] + 1] = (ll)col.size(); }
      for (int j = 0; j < I.M; ++j) { if (cdead[j]) continue;
        for (ll k = I.cp[j]; k < I.cp[j + 1]; ++k) if (!rdead[I.row[k]]) { row.push_back(rmap[I.row[k]]); cg.push_back(I.cg[k]); }
        cp[cmap[j] + 1] = (ll)row.size(); }
      fprintf(stderr, "  dominance: %lld pairs fixed in %d passes (gain %.1f); left %d x %d, %lld edges (was %lld)\n", n_fixed, passes + 1, fixed_gain, P, O, (ll)col.size(), I.rp[I.N]);
      Auction A; A.P = P; A.O = O; A.rp = rp.data(); A.col = col.data(); A.g = g.data(); A.cp = cp.data(); A.row = row.data(); A.cg = cg.data();
      const double avg = P ? (double)col.size() / P : 1.0;
      A.small_fwd = A.small_rev = std::max(16, std::min(2048, (int)(65536.0 / std::max(1.0, avg)))); A.init();
      double e0 = I.penalty / 4.0;
      if (mode.size() > 4) e0 = atof(mode.c_str() + 4);
      auto eps = e0 > 0 ? schedule(e0, 5.0, 0.5 * KM_eps) : std::vector<double>(1, 0.5 * KM_eps);
      for (size_t ph = 0; ph < eps.size(); ++ph) {
        std::fill(A.owner.begin(), A.owner.end(), -1); std::fill(A.assign.begin(), A.assign.end(), -1); std::fill(A.profit.begin(), A.profit.end(), 0.0);
        ll r0 = A.fwd.rounds;
        A.forward(persons_with_edges(A), eps[ph]);
        fprintf(stderr, "  phase %zu eps %.4f: %lld rounds, D %.1f gain %.1f\n", ph, eps[ph], A.fwd.rounds - r0, A.free_price_sum(), A.total_gain());
      }
      double D = A.free_price_sum();
      if (D > 0.5 * KM_eps * N) A.reverse(0.5 * KM_eps);
      report(mode.c_str(), A, A.total_gain() + fixed_gain, D, tnow() - t0);
    } else if (mode.rfind("dbl", 0) == 0) {
      // symmetric doubling: persons = rows + mirror columns, objects = columns + mirror rows; zero-gain edges
      // (i, i') and (j', j); forward auction only, standard epsilon scaling (all objects end up assigned)
      double e0 = I.penalty / 4.0, div = 5.0;
      if (mode.size() > 4) sscanf(mode.c_str() + 4, "%lf,%lf", &e0, &div);
      const int P = I.N + I.M;
      std::vector<ll> rp(P + 1, 0); std::vector<int> col; std::vector<double> g;
      for (int i = 0; i < I.N; ++i) { for (ll k = I.rp[i]; k < I.rp[i + 1]; ++k) { col.push_back(I.col[k]); g.push_back(I.g[k]); } col.push_back(I.M + i); g.push_back(0.0); rp[i + 1] = (ll)col.size(); }
      for (int j = 0; j < I.M; ++j) { for (ll k = I.cp[j]; k < I.cp[j + 1]; ++k) { col.push_back(I.M + I.row[k]); g.push_back(I.cg[k]); } col.push_back(j); g.push_back(0.0); rp[I.N + j + 1] = (ll)col.size(); }
      Auction A; A.P = P; A.O = P; A.rp = rp.data(); A.col = col.data(); A.g = g.data(); A.cp = nullptr; A.row = nullptr; A.cg = nullptr;
      A.has_dummy = false; A.small_fwd = small; A.init();
      auto eps = schedule(e0, div, KM_eps);
      for (size_t ph = 0; ph < eps.size(); ++ph) {
        std::fill(A.owner.begin(), A.owner.end(), -1); std::fill(A.assign.begin(), A.assign.end(), -1);
        ll r0 = A.fwd.rounds, b0 = A.fwd.bids;
        std::vector<int> all(P); for (int i = 0; i < P; ++i) all[i] = i;
        A.forward(all, eps[ph]);
        fprintf(stderr, "  phase %zu eps %.4f: %lld rounds %lld bids\n", ph, eps[ph], A.fwd.rounds - r0, A.fwd.bids - b0);
      }
      double ga = 0, gb = 0;
      for (int i = 0; i < I.N; ++i) if (A.assign[i] >= 0 && A.assign[i] < I.M) for (ll k = I.rp[i]; k < I.rp[i + 1]; ++k) if (I.col[k] == A.assign[i]) { ga += I.g[k]; break; }
      for (int j = 0; j < I.M; ++j) { int o = A.assign[I.N + j]; if (o >= I.M) for (ll k = I.cp[j]; k < I.cp[j + 1]; ++k) if (I.row[k] == o - I.M) { gb += I.cg[k]; break; } }
      fprintf(stderr, "  halves: real %.3f mirror %.3f\n", ga, gb);
      report(mode.c_str(), A, std::max(ga, gb), 0.0, tnow() - t0);
    } else if (mode.rfind("fr", 0) == 0) {
      // forward + reverse at EVERY phase (Bertsekas-Castanon scaling for the asymmetric problem)
      double e0 = I.penalty / 4.0, div = 5.0; int keep = 0;
      if (mode.size() > 3) sscanf(mode.c_str() + 3, "%lf,%lf,%d", &e0, &div, &keep);
      Auction A = mk();
      auto eps = schedule(e0, div, 0.5 * KM_eps);
      for (size_t ph = 0; ph < eps.size(); ++ph) {
        std::vector<int> act;
        if (ph == 0 || !keep) {
          std::fill(A.owner.begin(), A.owner.end(), -1); std::fill(A.assign.begin(), A.assign.end(), -1); std::fill(A.profit.begin(), A.profit.end(), 0.0);
          act = persons_with_edges(A);
        } else {
          // keep assignments that still satisfy eps-CS with the new eps
          for (int i = 0; i < A.P; ++i) {
            if (A.rp[i + 1] == A.rp[i]) continue;
            double best = 0.0;
            for (ll k = A.rp[i]; k < A.rp[i + 1]; ++k) best = std::max(best, A.g[k] - A.price[A.col[k]]);
            double mine = 0.0;
            if (A.assign[i] >= 0) for (ll k = A.rp[i]; k < A.rp[i + 1]; ++k) if (A.col[k] == A.assign[i]) { mine = A.g[k] - A.price[A.col[k]]; break; }
            if (mine < best - eps[ph]) { if (A.assign[i] >= 0) A.owner[A.assign[i]] = -1; A.assign[i] = -1; act.push_back(i); }
            else A.profit[i] = mine;
          }
        }
        ll r0 = A.fwd.rounds, r1 = A.rev.rounds;
        size_t nact = act.size();
        A.forward(act, eps[ph]);
        double D = A.free_price_sum();
        A.reverse(eps[ph]);
        double cv, cD; A.certificate(cv, cD);
        fprintf(stderr, "  phase %zu eps %.4f: active %zu fwd %lld rounds, D %.1f, rev %lld rounds, gain %.1f  certificate: viol %.2f + D %.2f\n", ph, eps[ph], nact, A.fwd.rounds - r0, D, A.rev.rounds - r1, A.total_gain(), cv, cD);
      }
      report(mode.c_str(), A, A.total_gain(), A.free_price_sum(), tnow() - t0);
    } else if (mode.rfind("sc=", 0) == 0) {
      // forward-only scaling: relax prices by relax*eps_prev at each phase start; after each phase: drop the price of
      // every free object to max(0, beta_j - eps) (no reassignment), certificate, stop when within budget
      double e0 = I.penalty / 4.0, div = 5.0, relax = 2.0, last = 0.5 * KM_eps; int carry = 0;
      sscanf(mode.c_str() + 3, "%lf,%lf,%lf,%lf,%d", &e0, &div, &relax, &last, &carry);
      Auction A = mk();
      auto eps = schedule(e0, div, last);
      const double budget = KM_eps * N;
      for (size_t ph = 0; ph < eps.size(); ++ph) {
        if (ph > 0) { for (auto &p : A.price) p = std::max(0.0, p - relax * eps[ph - 1]); }
        std::fill(A.owner.begin(), A.owner.end(), -1); std::fill(A.assign.begin(), A.assign.end(), -1); std::fill(A.profit.begin(), A.profit.end(), 0.0);
        ll r0 = A.fwd.rounds;
        A.forward(persons_with_edges(A), eps[ph]);
        double cv, cD; A.certificate(cv, cD);
        // price drop of free objects
        double Dd = 0; int nfree = 0;
        for (int j = 0; j < A.O; ++j) if (A.owner[j] < 0 && A.price[j] > 0.0) {
          double beta = -1e300;
          for (ll k = A.cp[j]; k < A.cp[j + 1]; ++k) beta = std::max(beta, A.cg[k] - A.profit[A.row[k]]);
          const double np = std::max(0.0, std::min(A.price[j], beta - eps[ph]));
          A.price[j] = np; Dd += np; nfree += np > 0;
        }
        double cv2, cD2; A.certificate(cv2, cD2);
        fprintf(stderr, "  phase %zu eps %.4f: %lld rounds gain %.1f  certificate: viol %.2f + D %.2f -> after drop viol %.2f + D %.2f (%d objects)  budget %.1f\n", ph, eps[ph], A.fwd.rounds - r0, A.total_gain(), cv, cD, cv2, cD2, nfree, budget);
        if (cv2 + cD2 <= budget) break;
        if (carry) {
          ll rr = A.rev.rounds; A.reverse(eps[ph]);
          double v3, D3; A.certificate(v3, D3);
          fprintf(stderr, "      + reverse %lld rounds -> gain %.1f certificate viol %.2f + D %.2f\n", A.rev.rounds - rr, A.total_gain(), v3, D3);
          if (v3 + D3 <= budget) break;
        } else if (eps[ph] < 2.0) {
          Auction B = A;   // try: reverse at this eps (cheap at coarse eps), then price refinement
          ll rr = B.rev.rounds; B.reverse(eps[ph]);
          int sw = 0; double G = B.refine_prices(200, &sw);
          fprintf(stderr, "      + reverse %lld rounds -> gain %.1f; price refinement: %d sweeps, dual bound gap G = %.3f\n", B.rev.rounds - rr, B.total_gain(), sw, G);
        }
      }
      report(mode.c_str(), A, A.total_gain(), A.free_price_sum(), tnow() - t0);
    } else if (mode.rfind("lvl=", 0) == 0) {
      // descending uniform price level: prices start at lambda; forward; then lambda /= 2: never-owned objects drop to
      // the new level, persons with violation > eps are released (their object keeps its price), forward again; ...
      double lam = atof(mode.c_str() + 4); const double e = 0.5 * KM_eps;
      Auction A = mk();
      std::fill(A.price.begin(), A.price.end(), lam);
      std::vector<char> touched(A.O, 0);
      std::vector<int> act = persons_with_edges(A);
      while (true) {
        ll r0 = A.fwd.rounds;
        A.forward(act, e);
        for (int j = 0; j < A.O; ++j) if (A.owner[j] >= 0) touched[j] = 1;
        double cv, cD; A.certificate(cv, cD);
        fprintf(stderr, "  level %.3f: %lld rounds, gain %.1f certificate viol %.2f + D %.2f\n", lam, A.fwd.rounds - r0, A.total_gain(), cv, cD);
        if (lam == 0.0) break;
        lam = lam < 0.5 ? 0.0 : lam * 0.5;
        for (int j = 0; j < A.O; ++j) if (A.owner[j] < 0) A.price[j] = std::min(A.price[j], lam);
        act.clear();
        for (int i = 0; i < A.P; ++i) {
          if (A.rp[i + 1] == A.rp[i]) continue;
          double best = 0.0, cur = 0.0;
          for (ll k = A.rp[i]; k < A.rp[i + 1]; ++k) { const double x = A.g[k] - A.price[A.col[k]]; best = std::max(best, x); if (A.col[k] == A.assign[i]) cur = x; }
          if (best - cur > e) { if (A.assign[i] >= 0) { A.owner[A.assign[i]] = -1; A.price[A.assign[i]] = std::min(A.price[A.assign[i]], lam); } A.assign[i] = -1; act.push_back(i); }
        }
        fprintf(stderr, "    -> level %.3f releases %zu persons\n", lam, act.size());
      }
      double D = A.free_price_sum();
      report(mode.c_str(), A, A.total_gain(), D, tnow() - t0);
    } else if (mode.rfind("single", 0) == 0) {
      Auction A = mk();
      double e = 0.5 * KM_eps;
      if (mode.size() > 7) e = atof(mode.c_str() + 7);
      A.forward(persons_with_edges(A), e);
      { double cv, cD; A.certificate(cv, cD); fprintf(stderr, "  single eps %.4f: certificate viol %.2f + D %.2f (budget %.1f)\n", e, cv, cD, KM_eps * N); }
      report("single phase", A, A.total_gain(), A.free_price_sum(), tnow() - t0);
    }
  }
  return 0;
}
