// ghicp_auction.cu — GPU replacement of Km::kmsolve (src/km.cpp:40-126) for the graph that
// findcorrespondenceKM builds (src/ghicp_reg.cpp:348-365).
//
// The reference solves a max-weight PERFECT matching on the padded n x n matrix w = -CD (CD < penalty)
// else -penalty, and then drops every matched pair whose weight == -penalty (src/km.cpp:162).  That is
// exactly the max-GAIN PARTIAL matching over the candidate edges g_ij = penalty - CD_ij > 0 (any partial
// matching completes to a perfect one with zero-gain edges).  We solve that sparse problem with an
// epsilon-scaled Jacobi forward auction (persons = source rows, objects = target columns, every person
// owns a private zero-gain dummy object) followed by a reverse auction that restores complementary
// slackness for objects left unassigned with a positive price (Bertsekas & Castanon's forward/reverse
// scheme for asymmetric assignment).  On termination with eps: total gain >= optimum - n_persons*eps,
// the same guarantee the reference's eps-tight Kuhn–Munkres gives with KM_eps (include/ghicp_reg.h:38).
//
// All tie-breaks are explicit (value, then smaller index), so the result does not depend on the
// order in which atomics land.
#include <algorithm>
#include <climits>
#include <cooperative_groups.h>
#include <cstdio>
#include <cstdlib>

#include "ghicp_internal.h"

namespace ghicp_b200 {

namespace {

constexpr int UNASSIGNED = -1;
constexpr int DUMMY = -2;
constexpr int AUC_BLOCK = 256;
constexpr int AUC_GRID = GHICP_SMS * 4;

__device__ __forceinline__ unsigned long long d2ull(double v) { return (unsigned long long)__double_as_longlong(v); }

// (best value, its index, second-best value) merge with explicit tie-breaks
struct Top2 {
  double best, second;
  int idx;
};
// Tie-break among equally valued options: a fixed pseudo-random order per bidder instead of "smallest
// index".  With integer costs (BSC iteration 0: CD = Hamming distance) whole groups of bidders are exactly
// indifferent between the same objects; index order would send them all to the same object and resolve
// one bidder per round, a hashed order spreads them and resolves the group in O(log) rounds.  The order
// is a pure function of (bidder, option), so results stay independent of thread scheduling.
__device__ __forceinline__ unsigned tie_key(int who, int idx) {
  unsigned h = (unsigned)idx * 0x9E3779B1u ^ ((unsigned)who * 0x85EBCA77u + 0xC2B2AE3Du);
  h ^= h >> 15; h *= 0x2C1B3C6Du; h ^= h >> 12;
  return h;
}
__device__ __forceinline__ bool tie_less(int who, int a, int b) {  // a before b ?
  const unsigned ka = tie_key(who, a), kb = tie_key(who, b);
  return ka < kb || (ka == kb && a < b);
}
__device__ __forceinline__ void top2_push_h(Top2 &t, double v, int idx, int who) {
  if (v > t.best || (v == t.best && t.idx >= 0 && tie_less(who, idx, t.idx))) {
    t.second = t.best;
    t.best = v;
    t.idx = idx;
  } else if (v > t.second) {
    t.second = v;
  }
}
__device__ __forceinline__ void top2_merge_h(Top2 &a, double ob, int oi, double os, int who) {
  if (ob > a.best || (ob == a.best && tie_less(who, oi, a.idx))) {
    double nb2 = fmax(a.best, os);
    a.best = ob; a.idx = oi; a.second = nb2;
  } else {
    a.second = fmax(a.second, ob);
  }
}
__device__ __forceinline__ void top2_push(Top2 &t, double v, int idx) {
  if (v > t.best || (v == t.best && idx < t.idx)) {
    t.second = t.best;
    t.best = v;
    t.idx = idx;
  } else if (v > t.second) {
    t.second = v;
  }
}
__device__ __forceinline__ void top2_merge(Top2 &a, double ob, int oi, double os) {
  if (ob > a.best || (ob == a.best && oi < a.idx)) {
    double nb2 = fmax(a.best, os);
    a.best = ob; a.idx = oi; a.second = nb2;
  } else {
    a.second = fmax(a.second, ob);
  }
}

struct AucArgs {
  const long long *rowptr; int n_chunks;  // row i spans rowptr[i*n_chunks] .. rowptr[(i+1)*n_chunks]
  const int *csr_col; const double *csr_gain;
  const long long *colptr; const int *csc_row; const double *csc_gain;
  double *price, *profit;
  int *assign, *owner;
  unsigned long long *bidmax; int *bidwin;
  int *bid_obj; double *bid_val, *bid_aux;
  int *counters;  // [0],[1]: ping-pong list sizes, [2]: base list size
  double eps;
  // Reverse phase: stop as soon as D = sum of the prices of the objects still free (= the active list) fits the budget.
  // Dual eps-feasibility (profit_i + price_j >= g_ij - eps on every edge, equality on matched pairs) is an invariant of
  // the reverse rounds, so OPT - ours <= n*eps + D holds at EVERY round boundary: the rest of the displacement chains
  // (thousands of rounds with a handful of bidders each) need not be followed.  D is kept in 2^-20 fixed point
  // (integer adds: the same value on every rank and run whatever order the atomics land in), each price rounded up.
  unsigned long long d_budget_fx;   // 0 = no early stop
};
constexpr double D_FX = 1048576.0;
__device__ __forceinline__ unsigned long long d_fx(double p) { return p > 0.0 ? (unsigned long long)(p * D_FX) + 1ull : 0ull; }
// counters (int[64]): [0],[1] list sizes, [2] base list size, [3] sticky round-limit flag, [4] cur, [5] rounds, [6] rounds
// of the whole solve, [8..9] bids (u64), [10] grid rounds, [32..33] / [34..35] D of list 0 / 1 (u64 fixed point), [36] 1 =
// the reverse phase stopped on the D budget
__device__ __forceinline__ unsigned long long *d_slot(int *counters, int which) {
  return reinterpret_cast<unsigned long long *>(&counters[32 + 2 * which]);
}

__global__ void k_auc_init(int n_rows, int n_cols, const long long *rowptr, int n_chunks, double *price,
                           int *base_list, int *counters, unsigned long long *bidmax, int *bidwin, int nmax) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_cols) price[i] = 0.0;
  if (i < nmax) { bidmax[i] = 0ull; bidwin[i] = INT_MAX; }
  if (i < n_rows) {
    if (rowptr[(size_t)(i + 1) * n_chunks] > rowptr[(size_t)i * n_chunks]) {
      int pos = atomicAdd(&counters[2], 1);
      base_list[pos] = i;
    }
  }
}

__global__ void k_auc_phase_start(int n_rows, int n_cols, const long long *rowptr, int n_chunks, int *assign,
                                  int *owner, double *profit) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_cols) owner[i] = -1;
  if (i < n_rows) {
    const bool has = rowptr[(size_t)(i + 1) * n_chunks] > rowptr[(size_t)i * n_chunks];
    assign[i] = has ? UNASSIGNED : DUMMY;
    profit[i] = 0.0;
  }
}

// ---- reverse round -------------------------------------------------------------------------------
// D = sum of the prices of objects left free: the exact amount by which complementary slackness is violated,
// i.e. the extra term of the optimality bound  OPT - ours <= |M*| * eps + D
__global__ void k_free_price_sum(int n_cols, const int *owner, const double *price, unsigned long long *out) {
  unsigned long long v = 0ull;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n_cols; j += gridDim.x * blockDim.x)
    if (owner[j] < 0) v += d_fx(price[j]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0 && v != 0ull) atomicAdd(out, v);
}
__global__ void k_rev_collect(int n_cols, const int *owner, const double *price, int *list, int *counters, int cur) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n_cols && owner[j] < 0 && price[j] > 0.0) {
    list[atomicAdd(&counters[cur], 1)] = j;
    atomicAdd(d_slot(counters, cur), d_fx(price[j]));
  }
}


// ---------------------------------------------------------------------------------------------
// Persistent cooperative bidding rounds.  One launch runs a whole forward (or
// reverse) phase: rounds with many active bidders use the whole grid with grid-wide barriers between
// bid / resolve / commit; once the active set is small (the long price-war tail) CTA 0 runs the rounds
// alone with __syncthreads, which removes the launch / grid-barrier latency from ~all of the rounds.
// ---------------------------------------------------------------------------------------------
namespace cg = cooperative_groups;
constexpr int PA_THREADS = 512;
constexpr int PA_SMALL = 1024;  // largest active set CTA 0 iterates alone (its lists and bid slots sit in shared memory)

// State written with plain stores (prices, profits, owners, assignments, bid slots, the active lists) may be read with plain,
// L1-cached loads: inside CTA 0's tail rounds the CTA's own stores go through the same L1, and every full-grid phase starts
// behind __threadfence() + grid.sync(), whose acquire makes the other CTAs' earlier stores visible to plain loads (CUDA's
// grid-synchronisation guarantee).  Words that ATOMICS modify (bid keys, counters, D slots) are always read at L2.
__device__ __forceinline__ int ldl2_i(const int *p) { return __ldcg(p); }   // counters (atomically updated): always L2
__device__ __forceinline__ unsigned long long pack_key(float v, int who) {  // v > 0
  return ((unsigned long long)__float_as_uint(v) << 32) | (unsigned)(who + 1);
}
__device__ __forceinline__ int key_who(unsigned long long k) { return (int)(unsigned)(k & 0xffffffffull) - 1; }

// one person bids (warp-cooperative). Returns nothing; writes bid slots / dummy assignment.
// scan edges [kb, ke) of person i: best / second-best value (and the gain of the best edge), warp-reduced
__device__ __forceinline__ void fwd_scan(const AucArgs &a, int i, int lane, long long kb, long long ke, Top2 &t,
                                         double &bgain) {
  t.best = -1e300; t.second = -1e300; t.idx = -1;
  bgain = 0.0;
  long long k = kb + lane;
  // 8 independent edge loads in flight per lane (the tail rounds are latency-bound)
  for (; k + 7 * 32 < ke; k += 8 * 32) {
    int j[8]; double g[8], p[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) { j[u] = a.csr_col[k + 32 * u]; g[u] = a.csr_gain[k + 32 * u]; }
#pragma unroll
    for (int u = 0; u < 8; ++u) p[u] = a.price[j[u]];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const double v = g[u] - p[u];
      if (v > t.best || (v == t.best && t.idx >= 0 && tie_less(i, j[u], t.idx))) bgain = g[u];
      top2_push_h(t, v, j[u], i);
    }
  }
  for (; k < ke; k += 32) {
    const int j = a.csr_col[k];
    const double g = a.csr_gain[k];
    const double v = g - a.price[j];
    if (v > t.best || (v == t.best && t.idx >= 0 && tie_less(i, j, t.idx))) bgain = g;
    top2_push_h(t, v, j, i);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    double ob = __shfl_xor_sync(0xffffffffu, t.best, o);
    int oi = __shfl_xor_sync(0xffffffffu, t.idx, o);
    double os = __shfl_xor_sync(0xffffffffu, t.second, o);
    double og = __shfl_xor_sync(0xffffffffu, bgain, o);
    if (oi >= 0) {
      if (t.idx < 0) { t.best = ob; t.idx = oi; t.second = os; bgain = og; }
      else {
        if (ob > t.best || (ob == t.best && tie_less(i, oi, t.idx))) bgain = og;
        top2_merge_h(t, ob, oi, os, i);
      }
    }
  }
}
// Bid slots: where a bidder leaves (target, value, auxiliary) between the bid half and the commit half of a round.
// Full-grid rounds: global arrays indexed by the bidder's id; CTA 0's tail rounds: SHARED memory indexed by the bidder's
// position in the active list (two L2 round trips less per round on the tail's dependent chain).
struct SlotsGlobal {
  int *o; double *v, *x;
  __device__ __forceinline__ void put(int k, int obj, double val, double aux) const { __stcg(&o[k], obj); __stcg(&v[k], val); __stcg(&x[k], aux); }
  __device__ __forceinline__ void none(int k) const { __stcg(&o[k], -1); }
  __device__ __forceinline__ int obj(int k) const { return o[k]; }
  __device__ __forceinline__ double val(int k) const { return v[k]; }
  __device__ __forceinline__ double aux(int k) const { return x[k]; }
};
struct SlotsShared {
  int *o; double *v, *x;
  __device__ __forceinline__ void put(int k, int obj, double val, double aux) const { o[k] = obj; v[k] = val; x[k] = aux; }
  __device__ __forceinline__ void none(int k) const { o[k] = -1; }
  __device__ __forceinline__ int obj(int k) const { return o[k]; }
  __device__ __forceinline__ double val(int k) const { return v[k]; }
  __device__ __forceinline__ double aux(int k) const { return x[k]; }
};
__device__ __forceinline__ SlotsGlobal global_slots(const AucArgs &a) { return SlotsGlobal{a.bid_obj, a.bid_val, a.bid_aux}; }

// one thread: turn (best, second) into a bid or retire to the private dummy
template <typename S>
__device__ __forceinline__ void fwd_finish(const AucArgs &a, int i, const Top2 &t, double bgain, const S &sl, int key) {
  if (t.idx < 0 || t.best <= 0.0) {
    __stcg(&a.assign[i], DUMMY);
    __stcg(&a.profit[i], 0.0);
    sl.none(key);
  } else {
    const double wv = fmax(t.second, 0.0);
    const double newprice = a.price[t.idx] + (t.best - wv) + a.eps;
    sl.put(key, t.idx, newprice, bgain);
    // One atomic decides the round's winner: the key orders bidders by their bid rounded to float32, then
    // by id.  ANY bidder may win a round as long as the price becomes its own (exact, double) bid: that is
    // a valid auction step (price rises by >= eps, the winner is eps-happy), so float32 ordering is enough.
    atomicMax(&a.bidmax[t.idx], pack_key((float)newprice, i));
  }
}
template <typename S>
__device__ __forceinline__ void fwd_bid_one(const AucArgs &a, int i, int lane, const S &sl, int key) {
  const long long b = a.rowptr[(size_t)i * a.n_chunks], e = a.rowptr[(size_t)(i + 1) * a.n_chunks];
  Top2 t;
  double bgain;
  fwd_scan(a, i, lane, b, e, t, bgain);
  if (lane == 0) fwd_finish(a, i, t, bgain, sl, key);
}
// returns via append(): persons that stay / become unassigned
template <typename S, typename Append>
__device__ __forceinline__ void fwd_commit_one(const AucArgs &a, int i, const S &sl, int key, Append append) {
  if (a.assign[i] != UNASSIGNED) return;
  const int j = sl.obj(key);
  if (key_who(__ldcg(&a.bidmax[j])) == i) {
    const int prev = a.owner[j];
    const double bv = sl.val(key);
    __stcg(&a.owner[j], i);
    __stcg(&a.price[j], bv);
    __stcg(&a.assign[i], j);
    __stcg(&a.profit[i], sl.aux(key) - bv);
    __stcg(&a.bidmax[j], 0ull);  // slot back to "no bid" (a loser reading 0 or the key sees "not me" either way)
    if (prev >= 0) { __stcg(&a.assign[prev], UNASSIGNED); append(prev, 0.0); }
  } else {
    append(i, 0.0);
  }
}

__device__ __forceinline__ void rev_scan(const AucArgs &a, int j, int lane, long long kb, long long ke, Top2 &t) {
  t.best = -1e300; t.second = -1e300; t.idx = -1;
  long long k = kb + lane;
  for (; k + 7 * 32 < ke; k += 8 * 32) {
    int i[8]; double g[8], pr[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) { i[u] = a.csc_row[k + 32 * u]; g[u] = a.csc_gain[k + 32 * u]; }
#pragma unroll
    for (int u = 0; u < 8; ++u) pr[u] = a.profit[i[u]];
#pragma unroll
    for (int u = 0; u < 8; ++u) top2_push_h(t, g[u] - pr[u], i[u], j);
  }
  for (; k < ke; k += 32) {
    const int i = a.csc_row[k];
    top2_push_h(t, a.csc_gain[k] - a.profit[i], i, j);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    double ob = __shfl_xor_sync(0xffffffffu, t.best, o);
    int oi = __shfl_xor_sync(0xffffffffu, t.idx, o);
    double os = __shfl_xor_sync(0xffffffffu, t.second, o);
    if (oi >= 0) {
      if (t.idx < 0) { t.best = ob; t.idx = oi; t.second = os; }
      else top2_merge_h(t, ob, oi, os, j);
    }
  }
}
template <typename S>
__device__ __forceinline__ void rev_finish(const AucArgs &a, int j, const Top2 &t, const S &sl, int key) {
  if (t.idx < 0 || t.best <= a.eps) {
    __stcg(&a.price[j], 0.0);   // nobody is worth attracting: price falls to the floor, object stays free
    sl.none(key);
  } else {
    const double delta = fmin(t.best, (t.best - t.second) + a.eps);
    sl.put(key, t.idx, delta, t.best);
    atomicMax(&a.bidmax[t.idx], pack_key((float)delta, j));
  }
}
template <typename S>
__device__ __forceinline__ void rev_offer_one(const AucArgs &a, int j, int lane, const S &sl, int key) {
  Top2 t;
  rev_scan(a, j, lane, a.colptr[j], a.colptr[j + 1], t);
  if (lane == 0) rev_finish(a, j, t, sl, key);
}
// short adjacency lists (a settled loop: about one candidate per keypoint): ONE THREAD per bidder walks its list; the
// (best, tie-ordered index, second) triple is the same whatever the partition of the list
template <bool REVERSE, typename S>
__device__ __forceinline__ void bid_serial(const AucArgs &a, int e, const S &sl, int key) {
  Top2 t;
  t.best = -1e300; t.second = -1e300; t.idx = -1;
  double bg = 0.0;
  long long k, ke;
  if (REVERSE) { k = a.colptr[e]; ke = a.colptr[e + 1]; }
  else { k = a.rowptr[(size_t)e * a.n_chunks]; ke = a.rowptr[(size_t)(e + 1) * a.n_chunks]; }
  const int *__restrict__ adj = REVERSE ? a.csc_row : a.csr_col;
  const double *__restrict__ gains = REVERSE ? a.csc_gain : a.csr_gain;
  const double *other = REVERSE ? a.profit : a.price;
  // four edges in flight: the two dependent loads of an edge (index, then the price / profit it points at) overlap
  for (; k + 3 < ke; k += 4) {
    int x[4]; double g[4], p[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) { x[u] = adj[k + u]; g[u] = gains[k + u]; }
#pragma unroll
    for (int u = 0; u < 4; ++u) p[u] = other[x[u]];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const double v = g[u] - p[u];
      if (!REVERSE && (v > t.best || (v == t.best && t.idx >= 0 && tie_less(e, x[u], t.idx)))) bg = g[u];
      top2_push_h(t, v, x[u], e);
    }
  }
  for (; k < ke; ++k) {
    const int x = adj[k];
    const double g = gains[k];
    const double v = g - other[x];
    if (!REVERSE && (v > t.best || (v == t.best && t.idx >= 0 && tie_less(e, x, t.idx)))) bg = g;
    top2_push_h(t, v, x, e);
  }
  if (REVERSE) rev_finish(a, e, t, sl, key); else fwd_finish(a, e, t, bg, sl, key);
}

template <typename S, typename Append>
__device__ __forceinline__ void rev_commit_one(const AucArgs &a, int j, const S &sl, int key, Append append) {
  const int i = sl.obj(key);
  if (i < 0) return;
  if (key_who(__ldcg(&a.bidmax[i])) == j) {
    const int old = a.assign[i];
    const double dl = sl.val(key);
    __stcg(&a.assign[i], j);
    __stcg(&a.owner[j], i);
    __stcg(&a.price[j], sl.aux(key) - dl);
    __stcg(&a.profit[i], a.profit[i] + dl);
    __stcg(&a.bidmax[i], 0ull);
    if (old >= 0) {
      __stcg(&a.owner[old], -1);
      const double po = a.price[old];
      if (po > 0.0) append(old, po);
    }
  } else {
    append(j, a.price[j]);
  }
}

// scan slice `slice` of G of the adjacency list of bidder e (warp-cooperative)
template <bool REVERSE>
__device__ __forceinline__ void split_scan(const AucArgs &a, int e, int G, int slice, int lane, Top2 &t, double &bg) {
  long long b, en;
  if (REVERSE) { b = a.colptr[e]; en = a.colptr[e + 1]; }
  else { b = a.rowptr[(size_t)e * a.n_chunks]; en = a.rowptr[(size_t)(e + 1) * a.n_chunks]; }
  const long long len = en - b;
  bg = 0.0;
  if (REVERSE) rev_scan(a, e, lane, b + len * slice / G, b + len * (slice + 1) / G, t);
  else fwd_scan(a, e, lane, b + len * slice / G, b + len * (slice + 1) / G, t, bg);
}
// merge the G partial results pt[0..G) of bidder e (the result does not depend on how the list was split:
// best value, the tie-order-preferred index among the options of that value, second-best value)
__device__ __forceinline__ void split_merge(int e, int G, const Top2 *pt, const double *pg, Top2 &t, double &bg) {
  t = pt[0]; bg = pg[0];
  for (int q = 1; q < G; ++q) {
    const Top2 o = pt[q];
    if (o.idx < 0) continue;
    if (t.idx < 0) { t = o; bg = pg[q]; continue; }
    if (o.best > t.best || (o.best == t.best && tie_less(e, o.idx, t.idx))) bg = pg[q];
    top2_merge_h(t, o.best, o.idx, o.second, e);
  }
}

template <bool REVERSE>
__global__ void __launch_bounds__(PA_THREADS, 2) k_auction_persistent(AucArgs a, int *list0, int *list1, int max_rounds,
                                                                      int small_n, int short_rows) {
  cg::grid_group grid = cg::this_grid();
  constexpr int NW = PA_THREADS / 32;
  __shared__ int s_n, s_next;
  __shared__ unsigned long long s_D, s_Dnext;
#if defined(GHICP_EMU_HOST)
  // the emulation shim maps __shared__ to ONE static per kernel; the split scans use these arrays in every block of the
  // (2-block) emulated grid at once, so each block gets its own copy there
  static Top2 s_pt_emu[4][NW];
  static double s_pg_emu[4][NW];
  Top2 *const s_pt = s_pt_emu[blockIdx.x & 3];
  double *const s_pg = s_pg_emu[blockIdx.x & 3];
#else
  __shared__ Top2 s_pt[NW];
  __shared__ double s_pg[NW];
#endif
  // CTA 0's tail rounds: active lists and bid slots in shared memory (used by block 0 only)
  __shared__ int s_list[2][PA_SMALL];
  __shared__ int s_bobj[PA_SMALL];
  __shared__ double s_bval[PA_SMALL], s_baux[PA_SMALL];
  const SlotsGlobal gsl = global_slots(a);
  int *lists[2] = {list0, list1};
  const int lane = threadIdx.x & 31;
  const int warp = threadIdx.x >> 5;
  const int gwarp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int gwarps = (gridDim.x * blockDim.x) >> 5;
  const int gtid = blockIdx.x * blockDim.x + threadIdx.x;
  const int gthreads = gridDim.x * blockDim.x;
  const bool cut_on = REVERSE && a.d_budget_fx != 0ull;
  bool cut = false;
  int cur = 0, rounds = 0;
  while (true) {
    const int n = ldl2_i(&a.counters[cur]);
    if (n == 0 || rounds >= max_rounds) break;
    // every thread of the grid reads the same D (written before the last grid barrier): a uniform decision
    if (cut_on && __ldcg(d_slot(a.counters, cur)) <= a.d_budget_fx) { cut = true; break; }
    if (n <= small_n) {
      // ---- tail: CTA 0 alone, block-level barriers only; the active lists and the bid slots live in shared memory
      if (blockIdx.x == 0) {
        int sc = 0;   // which of the two shared lists holds the current bidders
        for (int w = threadIdx.x; w < n; w += PA_THREADS) s_list[0][w] = lists[cur][w];
        if (threadIdx.x == 0) { s_n = n; s_D = __ldcg(d_slot(a.counters, cur)); }
        __syncthreads();
        const SlotsShared sl{s_bobj, s_bval, s_baux};
        while (true) {
          const int m = s_n;
          if (m == 0 || m > small_n || rounds >= max_rounds) break;
          if (cut_on && s_D <= a.d_budget_fx) break;   // the outer loop re-reads the same D and stops
          const int *list = s_list[sc];
          int *next = s_list[sc ^ 1];
          if (threadIdx.x == 0) { s_next = 0; s_Dnext = 0ull; atomicAdd((unsigned long long *)&a.counters[8], (unsigned long long)m); }
          if (m <= NW / 2) {
            // very few bidders: split every adjacency list over G warps so one round costs one short scan
            const int G = NW / m;
            const int bidder = warp / G, slice = warp % G;
            int i = -1;
            if (bidder < m) {
              i = list[bidder];
              Top2 t; double bg;
              split_scan<REVERSE>(a, i, G, slice, lane, t, bg);
              if (lane == 0) { s_pt[warp] = t; s_pg[warp] = bg; }
            }
            __syncthreads();
            if (bidder < m && slice == 0 && lane == 0) {
              Top2 t; double bg;
              split_merge(i, G, &s_pt[warp], &s_pg[warp], t, bg);
              if (m == 1) {
                // a single bidder cannot lose: bid and commit in one step (no key atomics, no second pass).
                // This is the common case of the tail: one displacement chain advancing one step per round.
                if (!REVERSE) {
                  if (t.idx < 0 || t.best <= 0.0) {
                    __stcg(&a.assign[i], DUMMY);
                    __stcg(&a.profit[i], 0.0);
                  } else {
                    const int j = t.idx;
                    const double newprice = a.price[j] + (t.best - fmax(t.second, 0.0)) + a.eps;
                    const int prev = a.owner[j];
                    __stcg(&a.owner[j], i);
                    __stcg(&a.price[j], newprice);
                    __stcg(&a.assign[i], j);
                    __stcg(&a.profit[i], bg - newprice);
                    if (prev >= 0) { __stcg(&a.assign[prev], UNASSIGNED); next[0] = prev; s_next = 1; }
                  }
                } else {
                  const int j = i;  // the list holds objects in the reverse phase
                  if (t.idx < 0 || t.best <= a.eps) {
                    __stcg(&a.price[j], 0.0);
                  } else {
                    const int who = t.idx;
                    const double delta = fmin(t.best, (t.best - t.second) + a.eps);
                    const int old = a.assign[who];
                    __stcg(&a.assign[who], j);
                    __stcg(&a.owner[j], who);
                    __stcg(&a.price[j], t.best - delta);
                    __stcg(&a.profit[who], a.profit[who] + delta);
                    if (old >= 0) {
                      __stcg(&a.owner[old], -1);
                      const double po = a.price[old];
                      if (po > 0.0) { next[0] = old; s_next = 1; s_Dnext = d_fx(po); }
                    }
                  }
                }
              } else if (REVERSE) rev_finish(a, i, t, sl, bidder); else fwd_finish(a, i, t, bg, sl, bidder);
            }
            if (m == 1) {   // committed above
              __syncthreads();
              cur ^= 1; sc ^= 1;
              ++rounds;
              if (threadIdx.x == 0) { s_n = s_next; s_D = s_Dnext; }
              __syncthreads();
              continue;
            }
          } else if (short_rows == 1 || (short_rows == 2 && m > 3 * NW)) {
            // one thread per bidder: short lists always; medium lists (<= 32 candidates) once the bidders outnumber the
            // CTA's warps three to one (16 warps walking 28 lists each in turn cost more than 512 threads walking one each)
            for (int w = threadIdx.x; w < m; w += PA_THREADS) bid_serial<REVERSE>(a, list[w], sl, w);
          } else {
            for (int w = warp; w < m; w += NW) {
              const int e = list[w];
              if (REVERSE) rev_offer_one(a, e, lane, sl, w); else fwd_bid_one(a, e, lane, sl, w);
            }
          }
          __syncthreads();
          for (int w = threadIdx.x; w < m; w += PA_THREADS) {
            const int e = list[w];
            auto app = [&](int x, double p) {
              next[atomicAdd(&s_next, 1)] = x;
              if (REVERSE) atomicAdd(&s_Dnext, d_fx(p));
            };
            if (REVERSE) rev_commit_one(a, e, sl, w, app); else fwd_commit_one(a, e, sl, w, app);
          }
          __syncthreads();
          cur ^= 1; sc ^= 1;
          ++rounds;
          if (threadIdx.x == 0) { s_n = s_next; s_D = s_Dnext; }
          __syncthreads();
        }
        // hand the current list back to the global arrays (the grid rounds, or the host, continue from there)
        {
          const int m = s_n;
          int *gl = lists[cur];
          for (int w = threadIdx.x; w < m; w += PA_THREADS) __stcg(&gl[w], s_list[sc][w]);
        }
        if (threadIdx.x == 0) {
          __stcg(&a.counters[cur], s_n);
          __stcg(d_slot(a.counters, cur), s_D);
          __stcg(&a.counters[4], cur);
          __stcg(&a.counters[5], rounds);
        }
      }
      __threadfence();
      grid.sync();
      cur = ldl2_i(&a.counters[4]);
      rounds = ldl2_i(&a.counters[5]);
      continue;
    }
    // ---- full-grid round
    const int *list = lists[cur];
    int *next = lists[cur ^ 1];
    if (gtid == 0) {
      __stcg(&a.counters[cur ^ 1], 0); __stcg(d_slot(a.counters, cur ^ 1), 0ull);
      atomicAdd((unsigned long long *)&a.counters[8], (unsigned long long)n); __stcg(&a.counters[10], ldl2_i(&a.counters[10]) + 1);
    }
    // warps per bidder: as many as the grid affords, so that a round with few bidders and long adjacency lists (the
    // dense first iterations: ~1400 candidates per keypoint) costs one short scan per warp instead of one long one
    int G = 1;
    {
      const long long tw = (long long)gridDim.x * NW;
      if (16ll * n <= tw) G = 16; else if (8ll * n <= tw) G = 8; else if (4ll * n <= tw) G = 4; else if (2ll * n <= tw) G = 2;
    }
    if (short_rows == 1 || (short_rows == 2 && n > 3 * gwarps)) {
      for (int w = gtid; w < n; w += gthreads) { const int e = list[w]; bid_serial<REVERSE>(a, e, gsl, e); }
    } else if (G > 1) {
      const int gpc = NW / G, grp = warp / G, slice = warp % G;
      const int w = blockIdx.x * gpc + grp;   // n <= gridDim.x * gpc by the choice of G
      int e = -1;
      if (w < n) {
        e = list[w];
        Top2 t; double bg;
        split_scan<REVERSE>(a, e, G, slice, lane, t, bg);
        if (lane == 0) { s_pt[warp] = t; s_pg[warp] = bg; }
      }
      __syncthreads();
      if (w < n && slice == 0 && lane == 0) {
        Top2 t; double bg;
        split_merge(e, G, &s_pt[warp], &s_pg[warp], t, bg);
        if (REVERSE) rev_finish(a, e, t, gsl, e); else fwd_finish(a, e, t, bg, gsl, e);
      }
    } else {
      for (int w = gwarp; w < n; w += gwarps) {
        const int e = list[w];
        if (REVERSE) rev_offer_one(a, e, lane, gsl, e); else fwd_bid_one(a, e, lane, gsl, e);
      }
    }
    __threadfence();
    grid.sync();
    for (int w = gtid; w < n; w += gthreads) {
      const int e = list[w];
      auto app = [&](int x, double p) {
        __stcg(&next[atomicAdd(&a.counters[cur ^ 1], 1)], x);
        if (REVERSE) atomicAdd(d_slot(a.counters, cur ^ 1), d_fx(p));
      };
      if (REVERSE) rev_commit_one(a, e, gsl, e, app); else fwd_commit_one(a, e, gsl, e, app);
    }
    __threadfence();
    grid.sync();
    cur ^= 1;
    ++rounds;
  }
  if (gtid == 0) {
    __stcg(&a.counters[4], cur);
    __stcg(&a.counters[6], ldl2_i(&a.counters[6]) + rounds);  // accumulated rounds of the whole solve
    if (cut) __stcg(&a.counters[36], 1);                       // stopped on the D budget: the list is not empty by design
    else if (ldl2_i(&a.counters[cur]) != 0) __stcg(&a.counters[3], 1);  // sticky: a phase hit the round limit
  }
}

// ---- CSC build ---------------------------------------------------------------------------------
__global__ void k_col_count(const int *__restrict__ csr_col, long long nnz, int *__restrict__ colcnt) {
  const long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < nnz) atomicAdd(&colcnt[csr_col[k]], 1);
}
__global__ void __launch_bounds__(AUC_BLOCK) k_csc_fill(int n_rows, const long long *rowptr, int n_chunks,
                                                         const int *csr_col, const double *csr_gain,
                                                         const long long *colptr, int *cursor, int *csc_row,
                                                         double *csc_gain) {
  const int lane = threadIdx.x & 31;
  const int warps = (gridDim.x * blockDim.x) >> 5;
  for (int i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < n_rows; i += warps) {
    const long long b = rowptr[(size_t)i * n_chunks], e = rowptr[(size_t)(i + 1) * n_chunks];
    for (long long k = b + lane; k < e; k += 32) {
      const int j = csr_col[k];
      const long long pos = colptr[j] + atomicAdd(&cursor[j], 1);
      csc_row[pos] = i;
      csc_gain[pos] = csr_gain[k];
    }
  }
}

}  // namespace

cudaError_t launch_build_csc(Ctx *c, int n_rows, int n_cols, long long nnz) {
  cudaError_t e;
  if ((e = cudaMemsetAsync(c->d_colcnt, 0, sizeof(int) * (size_t)(n_cols + 1), c->stream)) != cudaSuccess) return e;
  if (nnz > 0) {
    GHICP_LAUNCH(k_col_count, (unsigned)((nnz + 255) / 256), 256, 0, c->stream, c->d_csr_col, nnz, c->d_colcnt);
    c->launches++;
  }
  // cursor reuse: d_bid_obj is free before the auction starts
  {
    cudaError_t e = launch_scan_i32(c, c->d_colcnt, c->d_colptr, c->d_bid_obj, n_cols, nullptr);
    if (e != cudaSuccess) return e;
  }
  if (nnz > 0) {
    GHICP_LAUNCH(k_csc_fill, AUC_GRID, AUC_BLOCK, 0, c->stream, n_rows, c->d_rowptr, c->n_chunks, c->d_csr_col, c->d_csr_gain,
                                                       c->d_colptr, c->d_bid_obj, c->d_csc_row, c->d_csc_gain);
    c->launches++;
  }
  return cudaGetLastError();
}

// The settled route (km_auction_settled) and the general route (km_auction) must produce the same matching on the same
// graph: both fill the arguments, start the solve and launch the rounds through the functions below.

// eps of the single forward phase from zero prices (sparse graphs): free objects keep price 0 there (D = 0), so the whole
// optimality budget n*eps_final goes to eps.
static double single_phase_eps(double eps_final) { return 0.95 * eps_final; }

static AucArgs auc_args(const Ctx *c, double eps) {
  AucArgs a{};
  a.rowptr = c->d_rowptr; a.n_chunks = c->n_chunks; a.csr_col = c->d_csr_col; a.csr_gain = c->d_csr_gain;
  a.colptr = c->d_colptr; a.csc_row = c->d_csc_row; a.csc_gain = c->d_csc_gain;
  a.price = c->d_price; a.profit = c->d_profit; a.assign = c->d_assign; a.owner = c->d_owner;
  a.bidmax = c->d_bidmax; a.bidwin = c->d_bidwin; a.bid_obj = c->d_bid_obj; a.bid_val = c->d_bid_val;
  a.bid_aux = c->d_bid_aux; a.counters = c->d_counters;
  a.eps = eps;
  return a;
}

static int *base_list(Ctx *c) { return c->d_flags; }  // free during KM

// Start of a solve: counters zeroed, every price 0, the rows with candidates collected in the base list, no bids
static void auc_solve_start(Ctx *c, int n_rows, int n_cols) {
  const int nmax = std::max(n_rows, n_cols);
  cudaMemsetAsync(c->d_counters, 0, sizeof(int) * 64, c->stream);
  GHICP_LAUNCH(k_auc_init, (nmax + 255) / 256, 256, 0, c->stream, n_rows, n_cols, c->d_rowptr, c->n_chunks, c->d_price,
               base_list(c), c->d_counters, c->d_bidmax, c->d_bidwin, nmax);
  c->launches++;
  cudaMemsetAsync(c->d_bid_obj, 0xff, sizeof(int) * (size_t)nmax, c->stream);  // -1
}

// Start of a forward phase: every object free, every row with candidates unassigned and active (list 0 = the base list)
static void auc_phase_start(Ctx *c, int n_rows, int n_cols) {
  const int nmax = std::max(n_rows, n_cols);
  GHICP_LAUNCH(k_auc_phase_start, (nmax + 255) / 256, 256, 0, c->stream, n_rows, n_cols, c->d_rowptr, c->n_chunks,
               c->d_assign, c->d_owner, c->d_profit);
  c->launches++;
  cudaMemcpyAsync(c->d_list[0], base_list(c), sizeof(int) * (size_t)n_rows, cudaMemcpyDeviceToDevice, c->stream);
  cudaMemcpyAsync(&c->d_counters[0], &c->d_counters[2], sizeof(int), cudaMemcpyDeviceToDevice, c->stream);
}

// How the rounds run for adjacency lists of average length avg.  small_n: CTA 0 takes over the rounds alone once the active
// set is this small, i.e. once the expected work of a round (bidders x avg) is small enough that grid-wide barriers would
// dominate (long lists: a grid round gives every bidder up to 16 warps, CTA 0 alone only pays below ~16 bidders).
// short_rows: 1 = one thread walks a bidder's list (short lists), 2 = the same for medium lists once the bidders outnumber
// the warps, 0 = one or more warps per bidder.
struct RoundShape { int small_n, short_rows; };
static RoundShape round_shape(double avg) {
  const int sn = (int)(8192.0 / (avg > 1.0 ? avg : 1.0));
  return {std::min(std::max(sn, 16), PA_SMALL), avg <= 4.0 ? 1 : (avg <= 32.0 ? 2 : 0)};
}

// One persistent cooperative launch that runs a whole forward (REVERSE = false) or reverse phase from list 0
template <bool REVERSE>
static int launch_rounds(Ctx *c, const AucArgs &a, RoundShape rs) {
  static int blocks_per_sm = 0;   // all CTAs must be co-resident
  if (blocks_per_sm == 0) {
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks_per_sm, k_auction_persistent<REVERSE>, PA_THREADS, 0);
    if (blocks_per_sm < 1) blocks_per_sm = 1;
  }
  int n_sm = GHICP_SMS;
  cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, c->device);
  const dim3 grid(n_sm * blocks_per_sm);
  int *l0 = c->d_list[0], *l1 = c->d_list[1];
  int max_rounds = 4000000;
#if defined(GHICP_EMU_HOST)
  // host emulation: all blocks of the (small) grid run as fibers, the grid barrier is a rendezvous
  emu::launch_cooperative(grid, dim3(PA_THREADS), [&] { k_auction_persistent<REVERSE>(a, l0, l1, max_rounds, rs.small_n, rs.short_rows); });
  const cudaError_t e = cudaSuccess;
#else
  void *args[] = {(void *)&a, (void *)&l0, (void *)&l1, (void *)&max_rounds, (void *)&rs.small_n, (void *)&rs.short_rows};
  const cudaError_t e = cudaLaunchCooperativeKernel((void *)k_auction_persistent<REVERSE>, grid, dim3(PA_THREADS), args, 0, c->stream);
#endif
  if (e != cudaSuccess) {
    set_error(c, std::string(REVERSE ? "auction reverse launch: " : "auction forward launch: ") + cudaGetErrorString(e));
    return GHICP_E_CUDA;
  }
  c->launches++;
  return GHICP_OK;
}

// The settled loop's auction: ONE forward phase at single_phase_eps from zero prices (the sparse-graph schedule of
// km_auction: every object that ever received a bid stays owned, free objects keep price 0, D = 0, no reverse phase),
// enqueued without reading anything back.  Correct on any graph; chosen by the caller when last iteration's graph
// was sparse.
int km_auction_settled(Ctx *c, int n_rows, int n_cols, long long nnz_hint, double eps_final) {
  auc_solve_start(c, n_rows, n_cols);
  auc_phase_start(c, n_rows, n_cols);
  int rc;
  if ((rc = launch_rounds<false>(c, auc_args(c, single_phase_eps(eps_final)), round_shape((double)nnz_hint / std::max(n_rows, 1)))))
    return rc;
  cudaMemcpyAsync(c->h_counters, c->d_counters, sizeof(int) * 8, cudaMemcpyDeviceToHost, c->stream);
  return GHICP_OK;
}
int km_auction_settled_result(Ctx *c, KmResult *res) {   // after the iteration's stream synchronize
  if (c->h_counters[3] != 0) { set_error(c, "auction: round limit exceeded"); return GHICP_E_NOCONV; }
  if (res) { res->rounds = c->h_counters[6]; res->phases = 1; }
  return GHICP_OK;
}

int km_auction(Ctx *c, int n_rows, int n_cols, long long nnz, double eps_final, double max_gain, KmResult *res) {
  cudaStream_t st = c->stream;
  AucArgs a = auc_args(c, 0.0);
  const int nmax = std::max(n_rows, n_cols);
  auc_solve_start(c, n_rows, n_cols);

  // Split of the optimality budget n*eps_final: eps_last = epsf*eps_final for the forward phases (n*eps_last), the rest
  // for D = the prices of objects left free (the reverse phase runs while D exceeds it and stops as soon as it fits).
  // f = 0.1 where the D budget is worth having (large instances: it absorbs the last few dozen free objects and cuts the
  // reverse phase's tail: config 2, n = 50k, 693 rounds instead of 1375 at f = 0.5); f = 0.75 on small / medium instances,
  // whose budget n*KM_eps is below a handful of prices anyway and where the larger eps shortens the price wars instead
  // (measured, whole registration: config 4 (2.6k keypoints) 441 / 482 / 209 / 217 ms and config 5 (12.5k) 1549 / 765 / 731 / 839 ms
  // at f = 0.1 / 0.5 / 0.75 / 0.9)
  const double epsf = (eps_final * (double)nmax >= 250.0) ? 0.1 : 0.75;
  const double d_budget = (1.0 - epsf) * eps_final * (double)nmax;
  a.d_budget_fx = getenv("GHICP_AUCTION_NOCUT") ? 0ull : (unsigned long long)(d_budget * D_FX);
  // epsilon schedule
  std::vector<double> eps_list;
  {
    // Optimality bound at termination: OPT - ours <= n*eps_last + D  (D = prices of objects left free).
    // eps_last = epsf*eps_final leaves a budget of n*(1 - epsf)*eps_final for D, so the reverse auction (whose rounds are
    // long sequential displacement chains) only runs when D exceeds that budget.
    const double eps_last = epsf * eps_final;
    double e0 = max_gain / 4.0;
    while (e0 > eps_last * 1.0000001) { eps_list.push_back(e0); e0 /= 5.0; }
    eps_list.push_back(eps_last);
  }
  // Sparse candidate graphs (a settled loop: about one candidate per keypoint) need no epsilon scaling:
  // price wars are bounded by the few alternatives a person has, and a single forward phase from zero
  // prices leaves every free object at price zero (D = 0, no reverse auction).
  const bool single_phase = nnz <= (long long)(1.5 * (double)nmax) && getenv("GHICP_AUCTION_SCALING") == nullptr;
  if (nnz == 0 || single_phase) eps_list.assign(1, single_phase_eps(eps_final));

  RoundShape fwd = round_shape((double)nnz / std::max(n_rows, 1)), rev = round_shape((double)nnz / std::max(n_cols, 1));
  if (const char *ov = getenv("GHICP_AUCTION_SMALL"))   // test hook: 0 = grid rounds only
    fwd.small_n = rev.small_n = std::min(atoi(ov), PA_SMALL);
  const bool debug = getenv("GHICP_AUCTION_DEBUG") != nullptr;
  int last_rounds = 0, rc;
  bool ran_reverse = false;
  for (size_t ph = 0; ph < eps_list.size(); ++ph) {
    a.eps = eps_list[ph];
    auc_phase_start(c, n_rows, n_cols);
    cudaMemsetAsync(&c->d_counters[1], 0, sizeof(int), st);
    if ((rc = launch_rounds<false>(c, a, fwd))) return rc;
    // reverse: objects left free with a positive price.  Complementary slackness for free objects only
    // matters for the final optimality bound, so intermediate phases skip it (their leftover prices are
    // just the next phase's starting prices).
    bool need_reverse = false;
    if (ph + 1 == eps_list.size()) {
      unsigned long long *d_D = reinterpret_cast<unsigned long long *>(c->d_bid_aux);  // free scratch between rounds
      cudaMemsetAsync(d_D, 0, sizeof(unsigned long long), st);
      GHICP_LAUNCH(k_free_price_sum, GHICP_SMS, 256, 0, st, n_cols, c->d_owner, c->d_price, d_D);
      c->launches++;
      unsigned long long D_fx_host = 0ull;
      cudaMemcpyAsync(&D_fx_host, d_D, sizeof(unsigned long long), cudaMemcpyDeviceToHost, st);
      cudaMemcpyAsync(c->h_counters, c->d_counters, sizeof(int) * 8, cudaMemcpyDeviceToHost, st);  // final, unless the reverse runs
      cudaStreamSynchronize(st);
      const double D = (double)D_fx_host / D_FX;
      need_reverse = D > d_budget;
      if (debug) fprintf(stderr, "[auction] free-object price sum D = %.4f, budget %.4f -> reverse %s\n", D, d_budget, need_reverse ? "yes" : "skipped");
    }
    if (need_reverse) {
      ran_reverse = true;
      // the column-wise copy of the graph is only read by the reverse rounds: built here, on demand (a settled loop, one
      // forward phase from zero prices, never gets here)
      { cudaError_t e = launch_build_csc(c, n_rows, n_cols, nnz); if (e != cudaSuccess) { set_error(c, std::string("auction: CSC build: ") + cudaGetErrorString(e)); return GHICP_E_CUDA; } }
      cudaMemsetAsync(&c->d_counters[0], 0, sizeof(int) * 2, st);
      cudaMemsetAsync(&c->d_counters[32], 0, sizeof(int) * 5, st);   // D of both lists, the budget-stop flag
      GHICP_LAUNCH(k_rev_collect, (nmax + 255) / 256, 256, 0, st, n_cols, c->d_owner, c->d_price, c->d_list[0], c->d_counters, 0);
      c->launches++;
      cudaMemsetAsync(c->d_bid_obj, 0xff, sizeof(int) * (size_t)nmax, st);
      if ((rc = launch_rounds<true>(c, a, rev))) return rc;
      cudaMemsetAsync(c->d_bid_obj, 0xff, sizeof(int) * (size_t)nmax, st);
    }
    if (debug) {
      cudaMemcpyAsync(c->h_counters, c->d_counters, sizeof(int) * 64, cudaMemcpyDeviceToHost, st);
      cudaStreamSynchronize(st);
      fprintf(stderr, "[auction] phase %zu eps %.5f rounds %d (cum %d, grid rounds %d) bids(cum) %llu\n", ph, a.eps,
              c->h_counters[6] - last_rounds, c->h_counters[6], c->h_counters[10], *(unsigned long long *)&c->h_counters[8]);
      last_rounds = c->h_counters[6];
      if (need_reverse)
        fprintf(stderr, "[auction]   reverse %s: %d objects still free with a positive price, D left %.3f (budget %.3f)\n",
                c->h_counters[36] ? "stopped on the D budget" : "ran to completion", c->h_counters[c->h_counters[4] & 1],
                (double)*(unsigned long long *)&c->h_counters[32 + 2 * (c->h_counters[4] & 1)] / D_FX, d_budget);
    }
  }
  if (ran_reverse || debug) {
    cudaMemcpyAsync(c->h_counters, c->d_counters, sizeof(int) * 8, cudaMemcpyDeviceToHost, st);
    const cudaError_t e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) { set_error(c, std::string("auction: ") + cudaGetErrorString(e)); return GHICP_E_CUDA; }
  }
  if (c->h_counters[3] != 0) { set_error(c, "auction: round limit exceeded"); return GHICP_E_NOCONV; }
  if (res) { res->rounds = c->h_counters[6]; res->phases = (int)eps_list.size(); }
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) { set_error(c, std::string("auction: ") + cudaGetErrorString(e)); return GHICP_E_CUDA; }
  return GHICP_OK;
}

}  // namespace ghicp_b200
