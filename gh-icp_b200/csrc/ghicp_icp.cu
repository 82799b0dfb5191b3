// ghicp_icp.cu — point-to-point ICP on the dense clouds (DESIGN.md §3.13): the reference's CRegistration::icp_reg
// (src/common_reg.cpp:44-107), PCL's IterativeClosestPoint with its two options, reciprocal correspondences and the trimmed
// rejector.  Every stage of an iteration runs on the device; the host reads one small struct per iteration (pair count,
// convergence state, accumulated transform, work counters) to decide whether to go on.
//   k_icp_keys + sort   the working copy W's clamped target-cell keys, radix-sorted into the query order (the fitness-mode
//                       query order of ghicp_overlap.cu, redone every iteration because W moves)
//   k_icp_query         the hot path: the exact nearest target point of every W_i with its index, in (d2, index) order
//                       (ov_nearest<true> over the target grid ghicp_prep_overlap also keeps)
//   reciprocal          k_icp_mark / k_icp_compact the distinct targets j(i), a grid over W (prep_point_grid), k_icp_rev
//                       queries from those targets into W, k_icp_recip keeps (i, j) when j's nearest point of W is i
//   trimmed             k_icp_trim_keys: the u64 key (d2 bits, i) of every pair (non-negative float bits order like their
//                       values), radix sort, k_icp_trim_thr: the first key past floor(rho c), k_icp_trim_apply drops the rest
//   k_icp_sum<1, 2>     two-pass FP64 moments of the kept pairs over fixed point blocks and a fixed tree (means first, then
//   k_icp_total         the demeaned cross-covariance), as k_ov_reduce / k_ov_total: no floating-point atomic
//   k_icp_solve         one thread: the float32 Umeyama of the loop, F <- T F, DefaultConvergenceCriteria
//   k_icp_move          W <- T W (ov_move's formula)
// Point-to-plane (metric 1, DESIGN.md §3.14: the reference's CRegistration::ptplicp_reg, src/common_reg.cpp:123-199, PCL's
// IterativeClosestPointWithNormals with TransformationEstimationPointToPlaneLLS) keeps every stage above but the estimate:
//   k_icp_sum<1>        as above: the kept pairs' count, sum s (-> the centre m), sum d
//   k_icp_sum_pl        the 21 + 6 FP64 sums of the centred normal equations, rows [(s - m) x n_j, n_j], rhs n_j.(q_j - s),
//   k_icp_total_pl      over the same point blocks and thread tree as k_icp_sum, one component at a time
//   k_icp_solve_pl      one thread: chol_solve<6>, t = t' - omega x m, det_sincos, PCL's constructTransformationMatrix in double
//                       rounded once to float32, then k_icp_solve's F <- T F and convergence; a singular system stops the loop
// The target's normals (prep_knn_normals) are computed once per call, or kept on a pipeline result.
// Generalized ICP (metric 2, DESIGN.md §3.15: the reference's CRegistration::gicp_reg, src/common_reg.cpp:217-284, PCL's
// GeneralizedIterativeClosestPoint) keeps the correspondence stages, with k_icp_query<true> dropping pairs at d2 >= 1e12, and
// replaces the estimate by a Gauss-Newton minimisation of the Mahalanobis objective for the fixed pairs:
//   k_icp_sum<1>        as above: the kept pairs' count and sum q (-> the centre m)
//   k_gicp_begin        one thread: icp_begin, F_0 = F, R = F's rotation
//   k_gicp_mahal        M_i = gicp_mahalanobis(R, N_s,i, N_t,j) once per outer iteration, 6 doubles per pair
//   k_gicp_pass x 20    one inner step per launch: the 28 FP64 sums of J^T M J, J^T M r0, r0^T M r0 at F_j over k_icp_sum's
//                       point blocks and tree, then the last CTA to finish (an integer ticket) adds the blocks' partial sums
//                       in block order and runs gicp_step on one thread: accept or reject, chol_solve<6>, F_{j+1} = dT F_j;
//                       once the inner loop has ended the remaining launches return at once
//   k_gicp_end          one thread: F, then max_iterations and PCL's transformation delta
//   k_icp_move          W = F P, from the unmoved source
// Both clouds' normals (prep_knn_normals) are computed once per call, or kept on the pipeline results.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <vector>

#include "ghicp_internal.h"
#include "ghicp_device.cuh"
#include "ghicp_grid.cuh"
#include "ghicp_ovwalk.cuh"
#include "ghicp_solvers_math.h"

namespace ghicp_b200 {
namespace {

constexpr int IC_T = 128;            // threads per query / per-point CTA
constexpr int IC_RED_T = 256;        // threads per reduction CTA
constexpr int IC_RED_CHUNK = 8192;   // points per reduction CTA

struct IcpHead {                     // what the host reads after every iteration
  int state, cor;                    // ghicp_icp_state (0: running); kept pairs
  double mse;
  float F[16];                       // accumulated transform, row-major float32
  unsigned long long work[2];        // cells visited, candidates examined (every query so far)
};
struct IcpDev {
  IcpHead h;
  float T[16];                       // this iteration's transform, row-major float32
  double prev_mse;
  unsigned long long thr;            // trimmed: the smallest dropped (d2, i) key (~0: none dropped)
  int n_rev;                         // reciprocal: distinct targets to query
};
struct IcpSum { double v[9]; unsigned long long n; };   // pass 1: s, q, sum d; pass 2: sum (q - mu_q)(s - mu_s)^T
constexpr int IC_PL = 27;            // point-to-plane sums: the upper triangle of sum r r^T (row order), then sum r b
constexpr int IC_G = 28;             // GICP sums: the upper triangle of J^T M J (row order), J^T M r0, r0^T M r0
constexpr int GICP_INNER = 20;       // PCL's max_inner_iterations_
constexpr double GICP_GATE = 1e12;   // gicp_reg's corr_dist_threshold 1e6, squared: a pair is kept when d2 < this
struct GicpCtl {                     // the inner loop's state, on the device
  float Fs[16];                      // F at the start of the outer iteration (row-major float32)
  float Fj[16];                      // F_j: the transform the next pass evaluates
  float Fp[16];                      // F_{j-1}
  double R[9];                       // Fs's rotation, widened
  double m[3];                       // the centre: the kept target points' mean
  double fprev;                      // f_{j-1}
  int j, done;                       // the next pass's step; 1 once the inner loop has ended (the later passes return at once)
  unsigned ticket;                   // CTAs of the running pass that have written their partial sums
};

__device__ __forceinline__ void icp_move(const float *m, float x, float y, float z, float *o) {
  o[0] = ((m[0] * x + m[1] * y) + m[2] * z) + m[3];
  o[1] = ((m[4] * x + m[5] * y) + m[6] * z) + m[7];
  o[2] = ((m[8] * x + m[9] * y) + m[10] * z) + m[11];
}
// dst = src moved by the row-major float32 matrix m (device memory: the loop's T or F); dst may be src
__global__ void k_icp_move(const float *src, float *dst, long long n, const float *m) {
  const long long i = (long long)blockIdx.x * IC_T + threadIdx.x;
  if (i >= n) return;
  float o[3];
  icp_move(m, src[3 * i], src[3 * i + 1], src[3 * i + 2], o);
  dst[3 * i] = o[0]; dst[3 * i + 1] = o[1]; dst[3 * i + 2] = o[2];
}

// clamped target-cell key of each W_i, with its index (the cell order of the queries)
__global__ void k_icp_keys(const float *__restrict__ W, long long n, const OvGrid G, pu64 *__restrict__ keys, int *__restrict__ vals) {
  const long long t = (long long)blockIdx.x * IC_T + threadIdx.x;
  if (t >= n) return;
  keys[t] = ov_cell_key(G, W + 3 * t);
  vals[t] = (int)t;
}

// j(i) and d_i: the nearest target point of W_i in (d2, index) order, -1 / +inf for a non-finite W_i; GATE (GICP): no pair
// unless (double)d_i < 1e12
template <bool GATE>
__global__ void __launch_bounds__(IC_T) k_icp_query(const float *__restrict__ W, long long n, const int *__restrict__ perm,
                                                    const OvGrid G, int *__restrict__ corr, float *__restrict__ d2, IcpDev *dev) {
  const long long t = (long long)blockIdx.x * IC_T + threadIdx.x;
  unsigned long long cells = 0ull, cand = 0ull;
  if (t < n) {
    const long long i = perm[t];
    const GridRegs r = grid_regs(G.rg.g);   // per-thread registers, see k_pca
    int j = -1;
    const float d = ov_nearest<true>(r, G, W[3 * i], W[3 * i + 1], W[3 * i + 2], (double)INFINITY, -1.f, cells, cand, j);
    d2[i] = d;
    corr[i] = GATE && !((double)d < GICP_GATE) ? -1 : j;
  }
  ov_add_work(cells, cand, dev->h.work);
}

// reciprocal: the distinct targets of the pairs, compacted into list[0 .. n_rev) (any order: results are stored per target)
__global__ void k_icp_mark(const int *__restrict__ corr, long long n, unsigned char *__restrict__ flag) {
  const long long i = (long long)blockIdx.x * IC_T + threadIdx.x;
  if (i < n && corr[i] >= 0) flag[corr[i]] = 1;
}
__global__ void k_icp_compact(const unsigned char *__restrict__ flag, long long nt, int *__restrict__ list, IcpDev *dev) {
  const long long j = (long long)blockIdx.x * IC_T + threadIdx.x;
  const bool f = j < nt && flag[j];
  const unsigned m = __ballot_sync(0xffffffffu, f);
  const int lane = threadIdx.x & 31;
  int base = 0;
  if (lane == 0 && m) base = atomicAdd(&dev->n_rev, __popc(m));
  base = __shfl_sync(0xffffffffu, base, 0);
  if (f) list[base + __popc(m & ((1u << lane) - 1u))] = (int)j;
}
// rev[j] = the nearest point of W to Q_j in (d2, index) order, for the listed targets
__global__ void __launch_bounds__(IC_T) k_icp_rev(const float *__restrict__ Q, const int *__restrict__ list, const OvGrid Gw,
                                                  int *__restrict__ rev, IcpDev *dev) {
  const long long t = (long long)blockIdx.x * IC_T + threadIdx.x;
  unsigned long long cells = 0ull, cand = 0ull;
  if (t < dev->n_rev) {
    const int j = list[t];
    const GridRegs r = grid_regs(Gw.rg.g);
    int i = -1;
    ov_nearest<true>(r, Gw, Q[3 * (size_t)j], Q[3 * (size_t)j + 1], Q[3 * (size_t)j + 2], (double)INFINITY, -1.f, cells, cand, i);
    rev[j] = i;
  }
  ov_add_work(cells, cand, dev->h.work);
}
__global__ void k_icp_recip(int *__restrict__ corr, long long n, const int *__restrict__ rev) {
  const long long i = (long long)blockIdx.x * IC_T + threadIdx.x;
  if (i >= n) return;
  const int j = corr[i];
  if (j >= 0 && rev[j] != (int)i) corr[i] = -1;
}

// trimmed: (d2 bits, i) of every pair; ~0 for a point without one
__device__ __forceinline__ pu64 icp_trim_key(float d2, long long i) { return ((pu64)__float_as_uint(d2) << 32) | (pu64)(unsigned)i; }
__global__ void k_icp_trim_keys(const int *__restrict__ corr, const float *__restrict__ d2, long long n, pu64 *__restrict__ keys,
                                int *__restrict__ vals) {
  const long long i = (long long)blockIdx.x * IC_T + threadIdx.x;
  if (i >= n) return;
  keys[i] = corr[i] >= 0 ? icp_trim_key(d2[i], i) : ~0ull;
  vals[i] = (int)i;
}
// one thread: c = the pairs (sorted keys below ~0), keep = floor(rho * (float)c); thr = the first dropped key
__global__ void k_icp_trim_thr(const pu64 *__restrict__ sorted, long long n, float rho, IcpDev *dev) {
  long long lo = 0, hi = n;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (sorted[mid] != ~0ull) lo = mid + 1; else hi = mid;
  }
  const long long c = lo, keep = (long long)floorf(rho * (float)c);
  dev->thr = keep >= c ? ~0ull : sorted[keep];
}
__global__ void k_icp_trim_apply(int *__restrict__ corr, const float *__restrict__ d2, long long n, const IcpDev *dev) {
  const long long i = (long long)blockIdx.x * IC_T + threadIdx.x;
  if (i >= n) return;
  if (corr[i] >= 0 && icp_trim_key(d2[i], i) >= dev->thr) corr[i] = -1;
}

// moments of the kept pairs: thread t of block b sums the kept points b*CHUNK + t, + t + T, ... in that order, then a fixed
// halving tree over the block's threads; k_icp_total does the same over the blocks (tests/harness/icp_oracle.cpp restates it)
__device__ __forceinline__ void icp_sum_add(IcpSum &x, const IcpSum &y) {
  for (int k = 0; k < 9; ++k) x.v[k] += y.v[k];
  x.n += y.n;
}
__device__ void icp_tree(IcpSum *sh, const IcpSum &v, IcpSum *out) {
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int w = IC_RED_T / 2; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) icp_sum_add(sh[threadIdx.x], sh[threadIdx.x + w]);
    __syncthreads();
  }
  if (threadIdx.x == 0) *out = sh[0];
}
template <int PASS>
__global__ void __launch_bounds__(IC_RED_T) k_icp_sum(const float *__restrict__ W, const float *__restrict__ Q, const int *__restrict__ corr,
                                                      const float *__restrict__ d2, long long n, const IcpSum *__restrict__ m1,
                                                      IcpSum *__restrict__ part) {
  __shared__ IcpSum sh[IC_RED_T];
  const long long p0 = (long long)blockIdx.x * IC_RED_CHUNK, p1 = min(p0 + IC_RED_CHUNK, n);
  IcpSum v{};
  double mus[3] = {0, 0, 0}, mud[3] = {0, 0, 0};
  if (PASS == 2)
    for (int k = 0; k < 3; ++k) { mus[k] = m1->v[k] / (double)m1->n; mud[k] = m1->v[3 + k] / (double)m1->n; }
  for (long long p = p0 + threadIdx.x; p < p1; p += IC_RED_T) {
    const int j = corr[p];
    if (j < 0) continue;
    const double s[3] = {(double)W[3 * p], (double)W[3 * p + 1], (double)W[3 * p + 2]};
    const double q[3] = {(double)Q[3 * (size_t)j], (double)Q[3 * (size_t)j + 1], (double)Q[3 * (size_t)j + 2]};
    if (PASS == 1) {
      for (int k = 0; k < 3; ++k) { v.v[k] += s[k]; v.v[3 + k] += q[k]; }
      v.v[6] += (double)d2[p];
      ++v.n;
    } else {
      const double ds[3] = {s[0] - mus[0], s[1] - mus[1], s[2] - mus[2]};
      const double dd[3] = {q[0] - mud[0], q[1] - mud[1], q[2] - mud[2]};
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) v.v[r * 3 + c] += dd[r] * ds[c];
    }
  }
  icp_tree(sh, v, part + blockIdx.x);
}
__global__ void __launch_bounds__(IC_RED_T) k_icp_total(const IcpSum *__restrict__ part, int nb, IcpSum *__restrict__ out) {
  __shared__ IcpSum sh[IC_RED_T];
  IcpSum v{};
  for (int b = threadIdx.x; b < nb; b += IC_RED_T) icp_sum_add(v, part[b]);
  icp_tree(sh, v, out);
}

// point-to-plane pass 2: the 27 sums of the kept pairs' centred rows (m = the kept source mean of pass 1), the same point
// blocks and per-thread order as k_icp_sum; each of the 27 components then goes through k_icp_sum's halving tree in turn
// (one 2 KB shared array instead of 55 KB for all of them at once; tests/harness/icp_oracle.cpp restates it)
template <int NC>
__device__ void icp_tree_pl(double *sh, const double (&v)[NC], double *out) {
#pragma unroll
  for (int c = 0; c < NC; ++c) {
    sh[threadIdx.x] = v[c];
    __syncthreads();
    for (int w = IC_RED_T / 2; w > 0; w >>= 1) {
      if ((int)threadIdx.x < w) sh[threadIdx.x] += sh[threadIdx.x + w];
      __syncthreads();
    }
    if (threadIdx.x == 0) out[c] = sh[0];
    __syncthreads();
  }
}
__global__ void __launch_bounds__(IC_RED_T) k_icp_sum_pl(const float *__restrict__ W, const float *__restrict__ Q,
                                                         const float *__restrict__ N, const int *__restrict__ corr, long long n,
                                                         const IcpSum *__restrict__ m1, double *__restrict__ part) {
  __shared__ double sh[IC_RED_T];
  const long long p0 = (long long)blockIdx.x * IC_RED_CHUNK, p1 = min(p0 + IC_RED_CHUNK, n);
  double v[IC_PL];
#pragma unroll
  for (int c = 0; c < IC_PL; ++c) v[c] = 0.0;
  double m[3];
  for (int k = 0; k < 3; ++k) m[k] = m1->v[k] / (double)m1->n;
  for (long long p = p0 + threadIdx.x; p < p1; p += IC_RED_T) {
    const int j = corr[p];
    if (j < 0) continue;
    const double s[3] = {(double)W[3 * p], (double)W[3 * p + 1], (double)W[3 * p + 2]};
    const double q[3] = {(double)Q[3 * (size_t)j], (double)Q[3 * (size_t)j + 1], (double)Q[3 * (size_t)j + 2]};
    const double nn[3] = {(double)N[3 * (size_t)j], (double)N[3 * (size_t)j + 1], (double)N[3 * (size_t)j + 2]};
    const double u[3] = {s[0] - m[0], s[1] - m[1], s[2] - m[2]};
    const double r[6] = {u[1] * nn[2] - u[2] * nn[1], u[2] * nn[0] - u[0] * nn[2], u[0] * nn[1] - u[1] * nn[0], nn[0], nn[1], nn[2]};
    const double b = (nn[0] * (q[0] - s[0]) + nn[1] * (q[1] - s[1])) + nn[2] * (q[2] - s[2]);
    int e = 0;
#pragma unroll
    for (int a = 0; a < 6; ++a)
#pragma unroll
      for (int c = a; c < 6; ++c) v[e++] += r[a] * r[c];
#pragma unroll
    for (int a = 0; a < 6; ++a) v[21 + a] += r[a] * b;
  }
  icp_tree_pl(sh, v, part + (size_t)IC_PL * blockIdx.x);
}
__global__ void __launch_bounds__(IC_RED_T) k_icp_total_pl(const double *__restrict__ part, int nb, double *__restrict__ out) {
  __shared__ double sh[IC_RED_T];
  double v[IC_PL];
#pragma unroll
  for (int c = 0; c < IC_PL; ++c) v[c] = 0.0;
  for (int b = threadIdx.x; b < nb; b += IC_RED_T)
#pragma unroll
    for (int c = 0; c < IC_PL; ++c) v[c] += part[(size_t)IC_PL * b + c];
  icp_tree_pl(sh, v, out);
}

// the start of every solve: this iteration's pairs and mean squared distance, T_k = the identity; returns the pair count
__device__ unsigned long long icp_begin(IcpDev *dev, const IcpSum *__restrict__ m1) {
  IcpHead &h = dev->h;
  const unsigned long long c = m1->n;
  h.cor = (int)c;
  h.mse = c > 0 ? m1->v[6] / (double)c : (double)NAN;   // the distances found before T_k is applied, as PCL has it
  for (int i = 0; i < 16; ++i) dev->T[i] = (i % 5 == 0) ? 1.f : 0.f;
  return c;
}
// the float32 product T F of the loop (row-major), each entry ((a0 + a1) + a2) + a3
__device__ __forceinline__ void icp_compose(const float (&T)[16], const float *F, float (&out)[16]) {
  for (int r = 0; r < 4; ++r)
    for (int cc = 0; cc < 4; ++cc)
      out[r * 4 + cc] = ((T[r * 4] * F[cc] + T[r * 4 + 1] * F[4 + cc]) + T[r * 4 + 2] * F[8 + cc]) + T[r * 4 + 3] * F[12 + cc];
}
// F <- T_k F, and DefaultConvergenceCriteria with max_iterations_similar_transforms = 0
__device__ void icp_step(IcpDev *dev, const float (&T)[16], int k, int max_it, double eps_t, double eps_f) {
  IcpHead &h = dev->h;
  float F[16];
  icp_compose(T, h.F, F);
  for (int i = 0; i < 16; ++i) { dev->T[i] = T[i]; h.F[i] = F[i]; }
  if (k >= max_it) { h.state = GHICP_ICP_ITERATIONS; return; }
  const double cosa = 0.5 * ((((double)T[0] + (double)T[5]) + (double)T[10]) - 1.0);
  const double t2 = ((double)T[3] * (double)T[3] + (double)T[7] * (double)T[7]) + (double)T[11] * (double)T[11];
  if (cosa >= 1.0 - eps_t && t2 <= eps_t) { h.state = GHICP_ICP_TRANSFORM; return; }
  const double d = fabs(h.mse - dev->prev_mse);
  if (d < 1e-12) { h.state = GHICP_ICP_ABS_MSE; return; }
  if (d / dev->prev_mse < eps_f) { h.state = GHICP_ICP_REL_MSE; return; }
  dev->prev_mse = h.mse;
}

// one thread: T_k from the moments (the float32 Umeyama of the loop), then icp_step
__global__ void k_icp_solve(IcpDev *dev, const IcpSum *__restrict__ m1, const IcpSum *__restrict__ m2, int k, int max_it,
                            double eps_t, double eps_f) {
  const unsigned long long c = icp_begin(dev, m1);
  if (c < 3) { dev->h.state = GHICP_ICP_NO_CORRESPONDENCES; return; }
  float mu_s[3], mu_d[3], sigma[9];
  for (int a = 0; a < 3; ++a) { mu_s[a] = (float)(m1->v[a] / (double)c); mu_d[a] = (float)(m1->v[3 + a] / (double)c); }
  for (int a = 0; a < 9; ++a) sigma[a] = (float)(m2->v[a] / (double)c);
  double Rt[16];
  umeyama_from_moments_f32(mu_s, mu_d, sigma, Rt);
  float T[16];
  for (int r = 0; r < 4; ++r)
    for (int cc = 0; cc < 4; ++cc) T[r * 4 + cc] = (float)Rt[cc * 4 + r];
  icp_step(dev, T, k, max_it, eps_t, eps_f);
}

// one thread: T_k from the point-to-plane sums, then icp_step.  The normal equations are centred on the kept source mean m
// (x = (alpha, beta, gamma, t')), PCL's translation is t = t' - omega x m; a system chol_solve<6> refuses, or angles beyond
// det_sincos's range, stop the loop (GHICP_ICP_SINGULAR) with F unchanged
__global__ void k_icp_solve_pl(IcpDev *dev, const IcpSum *__restrict__ m1, const double *__restrict__ acc, int k, int max_it,
                               double eps_t, double eps_f) {
  const unsigned long long c = icp_begin(dev, m1);
  if (c < 3) { dev->h.state = GHICP_ICP_NO_CORRESPONDENCES; return; }
  double A[6][6], b[6], x[6] = {0, 0, 0, 0, 0, 0};
  int e = 0;
  for (int i = 0; i < 6; ++i)
    for (int j = i; j < 6; ++j) { A[i][j] = acc[e]; A[j][i] = acc[e]; ++e; }
  for (int i = 0; i < 6; ++i) b[i] = acc[21 + i];
  const double m[3] = {m1->v[0] / (double)c, m1->v[1] / (double)c, m1->v[2] / (double)c};
  bool ok = chol_solve<6>(A, b, x);
  const double al = x[0], be = x[1], ga = x[2];
  const double t[3] = {x[3] - (be * m[2] - ga * m[1]), x[4] - (ga * m[0] - al * m[2]), x[5] - (al * m[1] - be * m[0])};
  for (int i = 0; i < 3; ++i) ok = ok && fabs(x[i]) <= 1048576.0 && fabs(t[i]) <= DBL_MAX;   // false for NaN
  if (!ok) { dev->h.state = GHICP_ICP_SINGULAR; return; }
  double sa, ca, sb, cb, sg, cg;
  det_sincos(al, sa, ca); det_sincos(be, sb, cb); det_sincos(ga, sg, cg);
  const float T[16] = {(float)(cg * cb), (float)((-sg) * ca + (cg * sb) * sa), (float)(sg * sa + (cg * sb) * ca), (float)t[0],
                       (float)(sg * cb), (float)(cg * ca + (sg * sb) * sa), (float)((-cg) * sa + (sg * sb) * ca), (float)t[1],
                       (float)(-sb), (float)(cb * sa), (float)(cb * ca), (float)t[2],
                       0.f, 0.f, 0.f, 1.f};
  icp_step(dev, T, k, max_it, eps_t, eps_f);
}

// ---- Generalized ICP (metric 2) ---------------------------------------------------------------------------------------------
// PCL's GICP convergence measure between two float32 transforms: the largest |a_kl - b_kl| (float32 difference), scaled by
// 1 / eps_r in the 3 x 3 rotation block and by 1 / eps_t elsewhere (a NaN product, eps_t = 0 against no change, is skipped)
__device__ double gicp_delta(const float *a, const float *b, double eps_t, double eps_r) {
  const double rr = 1.0 / eps_r, rt = 1.0 / eps_t;
  double d = 0.0;
  for (int k = 0; k < 4; ++k)
    for (int l = 0; l < 4; ++l) {
      const double c = (k < 3 && l < 3 ? rr : rt) * (double)fabsf(a[4 * k + l] - b[4 * k + l]);
      if (c > d) d = c;
    }
  return d;
}

// one thread, once per outer iteration after k_icp_sum<1>: the pairs, F_0 = F, R, the centre m
__global__ void k_gicp_begin(IcpDev *dev, GicpCtl *g, const IcpSum *__restrict__ m1) {
  const unsigned long long c = icp_begin(dev, m1);
  g->j = 0;
  g->done = c < 3;
  if (c < 3) { dev->h.state = GHICP_ICP_NO_CORRESPONDENCES; return; }
  for (int i = 0; i < 16; ++i) { g->Fs[i] = dev->h.F[i]; g->Fj[i] = dev->h.F[i]; }
  for (int r = 0; r < 3; ++r)
    for (int cc = 0; cc < 3; ++cc) g->R[3 * r + cc] = (double)dev->h.F[4 * r + cc];
  for (int a = 0; a < 3; ++a) g->m[a] = m1->v[3 + a] / (double)c;
}

// the pairs' metric for the whole outer iteration, [n][6] (rows of dropped points are left as they are); the passes read it
// back rather than recompute it from the two normals: measured faster per outer iteration in 7 of 8 cases on an H100
// (DESIGN.md §3.15)
__global__ void k_gicp_mahal(const float *__restrict__ Ns, const float *__restrict__ Nt, const int *__restrict__ corr, long long n,
                             const GicpCtl *g, double *__restrict__ Mst) {
  const long long p = (long long)blockIdx.x * IC_T + threadIdx.x;
  if (p >= n || g->done) return;
  const int j = corr[p];
  if (j >= 0) gicp_mahalanobis(g->R, Ns + 3 * p, Nt + 3 * (size_t)j, Mst + 6 * p);
}

// one thread: the inner step on the pass's totals (acc) at F_j.  f_j > f_{j-1} rejects F_j (back to F_{j-1}) and ends the
// inner loop; else H x = -g by chol_solve<6>, t = t' - omega x m, dT = PCL's constructTransformationMatrix in double rounded
// once to float32, F_{j+1} = dT F_j; the loop ends when PCL's delta(F_{j+1}, F_j) < 1 or after 20 steps.  A system chol_solve
// refuses, an angle beyond det_sincos's range or a non-finite t stops the outer loop (SINGULAR) with F unchanged.
__device__ void gicp_step(IcpDev *dev, GicpCtl *g, const double *acc, double eps_t, double eps_r) {
  const double f = acc[IC_G - 1];
  if (g->j > 0 && f > g->fprev) {
    for (int i = 0; i < 16; ++i) g->Fj[i] = g->Fp[i];
    g->done = 1;
    return;
  }
  double A[6][6], b[6], x[6] = {0, 0, 0, 0, 0, 0};
  int e = 0;
  for (int i = 0; i < 6; ++i)
    for (int j = i; j < 6; ++j) { A[i][j] = acc[e]; A[j][i] = acc[e]; ++e; }
  for (int i = 0; i < 6; ++i) b[i] = -acc[21 + i];
  const double *m = g->m;
  bool ok = chol_solve<6>(A, b, x);
  const double al = x[0], be = x[1], ga = x[2];
  const double t[3] = {x[3] - (be * m[2] - ga * m[1]), x[4] - (ga * m[0] - al * m[2]), x[5] - (al * m[1] - be * m[0])};
  for (int i = 0; i < 3; ++i) ok = ok && fabs(x[i]) <= 1048576.0 && fabs(t[i]) <= DBL_MAX;   // false for NaN
  if (!ok) { dev->h.state = GHICP_ICP_SINGULAR; g->done = 1; return; }
  double sa, ca, sb, cb, sg, cg;
  det_sincos(al, sa, ca); det_sincos(be, sb, cb); det_sincos(ga, sg, cg);
  const float T[16] = {(float)(cg * cb), (float)((-sg) * ca + (cg * sb) * sa), (float)(sg * sa + (cg * sb) * ca), (float)t[0],
                       (float)(sg * cb), (float)(cg * ca + (sg * sb) * sa), (float)((-cg) * sa + (sg * sb) * ca), (float)t[1],
                       (float)(-sb), (float)(cb * sa), (float)(cb * ca), (float)t[2],
                       0.f, 0.f, 0.f, 1.f};
  float Fn[16];
  icp_compose(T, g->Fj, Fn);
  const bool small = gicp_delta(Fn, g->Fj, eps_t, eps_r) < 1.0;
  for (int i = 0; i < 16; ++i) { g->Fp[i] = g->Fj[i]; g->Fj[i] = Fn[i]; }
  g->fprev = f;
  g->j += 1;
  if (small || g->j >= GICP_INNER) g->done = 1;
}

// One inner step: the 28 sums at F_j (W = F_j P in place, icp_move's formula), thread t of block b over the kept points
// b*CHUNK + t, + t + T, ... and each component through the halving tree (k_icp_sum_pl's order); then the last CTA to take a
// ticket adds the blocks' sums as k_icp_total_pl does (block order, not arrival order: the same bits whichever CTA is last)
// and runs gicp_step.  Per kept pair, in double from the float32 inputs: r0 = w - q, u = w - m, J = [-[u]x, I] (the
// residual linearised as r0 + omega x u + t'), H += J^T M J, g += J^T M r0, f += r0^T M r0, M = k_gicp_mahal's.
__global__ void __launch_bounds__(IC_RED_T) k_gicp_pass(const float *__restrict__ P, const float *__restrict__ Q,
                                                        const double *__restrict__ Mst, const int *__restrict__ corr, long long n,
                                                        int nb, GicpCtl *g, IcpDev *dev, double *__restrict__ part, double eps_t,
                                                        double eps_r) {
  __shared__ double sh[IC_RED_T];
  __shared__ double tot[IC_G];
  __shared__ int last;
  if (g->done) return;   // the inner loop has ended: the same for every thread of the launch
  const long long p0 = (long long)blockIdx.x * IC_RED_CHUNK, p1 = min(p0 + IC_RED_CHUNK, n);
  double v[IC_G];
#pragma unroll
  for (int c = 0; c < IC_G; ++c) v[c] = 0.0;
  float F[16];
  for (int i = 0; i < 16; ++i) F[i] = g->Fj[i];
  double m[3];
  for (int a = 0; a < 3; ++a) m[a] = g->m[a];
  for (long long p = p0 + threadIdx.x; p < p1; p += IC_RED_T) {
    const int j = corr[p];
    if (j < 0) continue;
    float w[3];
    icp_move(F, P[3 * p], P[3 * p + 1], P[3 * p + 2], w);
    double M[6];
    for (int a = 0; a < 6; ++a) M[a] = Mst[6 * p + a];
    const double q[3] = {(double)Q[3 * (size_t)j], (double)Q[3 * (size_t)j + 1], (double)Q[3 * (size_t)j + 2]};
    const double r[3] = {(double)w[0] - q[0], (double)w[1] - q[1], (double)w[2] - q[2]};
    const double u[3] = {(double)w[0] - m[0], (double)w[1] - m[1], (double)w[2] - m[2]};
    // the rotation columns of J: e_x x u, e_y x u, e_z x u
    const double J[3][3] = {{0.0, -u[2], u[1]}, {u[2], 0.0, -u[0]}, {-u[1], u[0], 0.0}};
    double MJ[3][3], Mr[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      MJ[c][0] = (M[0] * J[c][0] + M[1] * J[c][1]) + M[2] * J[c][2];
      MJ[c][1] = (M[1] * J[c][0] + M[3] * J[c][1]) + M[4] * J[c][2];
      MJ[c][2] = (M[2] * J[c][0] + M[4] * J[c][1]) + M[5] * J[c][2];
    }
    Mr[0] = (M[0] * r[0] + M[1] * r[1]) + M[2] * r[2];
    Mr[1] = (M[1] * r[0] + M[3] * r[1]) + M[4] * r[2];
    Mr[2] = (M[2] * r[0] + M[4] * r[1]) + M[5] * r[2];
    const double Mi[3][3] = {{M[0], M[1], M[2]}, {M[1], M[3], M[4]}, {M[2], M[4], M[5]}};
    int e = 0;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
#pragma unroll
      for (int c = a; c < 3; ++c) v[e++] += (J[a][0] * MJ[c][0] + J[a][1] * MJ[c][1]) + J[a][2] * MJ[c][2];
#pragma unroll
      for (int c = 0; c < 3; ++c) v[e++] += MJ[a][c];
    }
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
      for (int c = a; c < 3; ++c) v[e++] += Mi[a][c];
#pragma unroll
    for (int a = 0; a < 3; ++a) v[21 + a] += (J[a][0] * Mr[0] + J[a][1] * Mr[1]) + J[a][2] * Mr[2];
#pragma unroll
    for (int a = 0; a < 3; ++a) v[24 + a] += Mr[a];
    v[27] += (r[0] * Mr[0] + r[1] * Mr[1]) + r[2] * Mr[2];
  }
  icp_tree_pl(sh, v, part + (size_t)IC_G * blockIdx.x);
  if (threadIdx.x == 0) {
    __threadfence();   // this block's sums before its ticket
    last = atomicAdd(&g->ticket, 1u) == (unsigned)(nb - 1);
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
#pragma unroll
  for (int c = 0; c < IC_G; ++c) v[c] = 0.0;
  for (int b = threadIdx.x; b < nb; b += IC_RED_T)
#pragma unroll
    for (int c = 0; c < IC_G; ++c) v[c] += __ldcg(part + (size_t)IC_G * b + c);
  icp_tree_pl(sh, v, tot);
  if (threadIdx.x == 0) {
    g->ticket = 0u;
    gicp_step(dev, g, tot, eps_t, eps_r);
  }
}

// one thread, after the inner steps: F, then k >= max_iterations (ITERATIONS) and PCL's delta(F_0, F) < 1 (TRANSFORM);
// NO_CORRESPONDENCES and SINGULAR leave F as it was
__global__ void k_gicp_end(IcpDev *dev, const GicpCtl *g, int k, int max_it, double eps_t, double eps_r) {
  IcpHead &h = dev->h;
  if (h.state != 0) return;
  for (int i = 0; i < 16; ++i) h.F[i] = g->Fj[i];
  if (k >= max_it) { h.state = GHICP_ICP_ITERATIONS; return; }
  if (gicp_delta(g->Fj, g->Fs, eps_t, eps_r) < 1.0) h.state = GHICP_ICP_TRANSFORM;
}

inline int iblk(long long n, int t) { return (int)((n + t - 1) / t); }

}  // namespace

cudaError_t icp_run(const float *d_src, int n_src, const float *d_all, int n_all, const OverlapTarget *t, const float *d_tgt,
                    const float *d_nrm, const float *d_nrm_s, const double *guess, const ghicp_icp_params *p, cudaEvent_t ev_iter,
                    cudaEvent_t ev_fit, ghicp_icp_result *out, float *h_moved, int *h_cor, double *h_mse) {
  const long long n = n_src, nt = t->n;
  const bool recip = p->reciprocal != 0, trim = p->trim_ratio > 0.f, plane = p->metric == 1, gicp = p->metric == 2;
  const int nb = iblk(n, IC_RED_CHUNK);
  DevBuf<float> W, d2, moved; DevBuf<int> corr, perm, rev, list; DevBuf<pu64> keys; DevBuf<unsigned char> flag;
  DevBuf<IcpDev> dev; DevBuf<IcpSum> part, tot; DevBuf<double> part_pl, tot_pl, Mst; DevBuf<GicpCtl> ctl;
  // every workspace of the loop first: running out of memory returns before anything is written (the reciprocal option's
  // grid over W is the exception: prep_point_grid allocates it every iteration, from the same pool)
  CUDA_TRY(W.alloc(3 * (size_t)n)); CUDA_TRY(d2.alloc((size_t)n)); CUDA_TRY(corr.alloc((size_t)n));
  CUDA_TRY(perm.alloc((size_t)n)); CUDA_TRY(keys.alloc((size_t)n));
  CUDA_TRY(dev.alloc(1)); CUDA_TRY(part.alloc((size_t)nb)); CUDA_TRY(tot.alloc(2));
  if (plane) { CUDA_TRY(part_pl.alloc((size_t)IC_PL * nb)); CUDA_TRY(tot_pl.alloc(IC_PL)); }
  if (gicp) {
    CUDA_TRY(part_pl.alloc((size_t)IC_G * nb)); CUDA_TRY(ctl.alloc(1)); CUDA_TRY(Mst.alloc(6 * (size_t)n));
    CUDA_TRY(cudaMemsetAsync(ctl.get(), 0, sizeof(GicpCtl), 0));
  }
  if (recip) { CUDA_TRY(rev.alloc((size_t)nt)); CUDA_TRY(list.alloc((size_t)nt)); CUDA_TRY(flag.alloc((size_t)nt)); }
  if (h_moved) CUDA_TRY(moved.alloc(3 * (size_t)n_all));
  IcpDev h0{};
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) h0.h.F[r * 4 + c] = guess ? (float)guess[c * 4 + r] : (r == c ? 1.f : 0.f);
  h0.prev_mse = DBL_MAX;
  CUDA_TRY(cudaMemcpyAsync(dev.get(), &h0, sizeof(h0), cudaMemcpyHostToDevice, 0));
  IcpDev *D = dev.get();
  const OvGrid G = ov_grid_of(t->pg);
  if (ev_iter) CUDA_TRY(cudaEventRecord(ev_iter, 0));
  GHICP_LAUNCH(k_icp_move, iblk(n, IC_T), IC_T, 0, 0, d_src, W.get(), n, D->h.F);   // W = P moved by the guess
  IcpHead hh{};
  std::vector<int> cor_tr;
  std::vector<double> mse_tr;
  int k = 1;
  for (;; ++k) {
    GHICP_LAUNCH(k_icp_keys, iblk(n, IC_T), IC_T, 0, 0, W.get(), n, G, keys.get(), perm.get());
    CUDA_TRY(prep_sort_pairs(0, keys.get(), perm.get(), n_src));
    if (gicp) GHICP_LAUNCH(k_icp_query<true>, iblk(n, IC_T), IC_T, 0, 0, W.get(), n, perm.get(), G, corr.get(), d2.get(), D);
    else GHICP_LAUNCH(k_icp_query<false>, iblk(n, IC_T), IC_T, 0, 0, W.get(), n, perm.get(), G, corr.get(), d2.get(), D);
    if (recip) {
      CUDA_TRY(cudaMemsetAsync(flag.get(), 0, (size_t)nt, 0));
      CUDA_TRY(cudaMemsetAsync(&D->n_rev, 0, sizeof(int), 0));
      GHICP_LAUNCH(k_icp_mark, iblk(n, IC_T), IC_T, 0, 0, corr.get(), n, flag.get());
      GHICP_LAUNCH(k_icp_compact, iblk(nt, IC_T), IC_T, 0, 0, flag.get(), nt, list.get(), D);
      PointGrid pw;
      CUDA_TRY(prep_point_grid(0, W.get(), n_src, n_src < 8 ? n_src : 8, 0.f, 0.0, &pw));
      GHICP_LAUNCH(k_icp_rev, iblk(nt, IC_T), IC_T, 0, 0, d_tgt, list.get(), ov_grid_of(pw), rev.get(), D);
      GHICP_LAUNCH(k_icp_recip, iblk(n, IC_T), IC_T, 0, 0, corr.get(), n, rev.get());
    }
    if (trim) {
      GHICP_LAUNCH(k_icp_trim_keys, iblk(n, IC_T), IC_T, 0, 0, corr.get(), d2.get(), n, keys.get(), perm.get());
      CUDA_TRY(prep_sort_pairs(0, keys.get(), perm.get(), n_src));
      GHICP_LAUNCH(k_icp_trim_thr, 1, 1, 0, 0, keys.get(), n, p->trim_ratio, D);
      GHICP_LAUNCH(k_icp_trim_apply, iblk(n, IC_T), IC_T, 0, 0, corr.get(), d2.get(), n, D);
    }
    GHICP_LAUNCH(k_icp_sum<1>, nb, IC_RED_T, 0, 0, W.get(), d_tgt, corr.get(), d2.get(), n, nullptr, part.get());
    GHICP_LAUNCH(k_icp_total, 1, IC_RED_T, 0, 0, part.get(), nb, tot.get());
    if (gicp) {
      GicpCtl *C = ctl.get();
      const double et = p->transformation_epsilon, er = p->rotation_epsilon;
      GHICP_LAUNCH(k_gicp_begin, 1, 1, 0, 0, D, C, tot.get());
      GHICP_LAUNCH(k_gicp_mahal, iblk(n, IC_T), IC_T, 0, 0, d_nrm_s, d_nrm, corr.get(), n, C, Mst.get());
      for (int j = 0; j < GICP_INNER; ++j)   // no read-back: the passes after the inner loop's end return at once
        GHICP_LAUNCH(k_gicp_pass, nb, IC_RED_T, 0, 0, d_src, d_tgt, Mst.get(), corr.get(), n, nb, C, D, part_pl.get(), et, er);
      GHICP_LAUNCH(k_gicp_end, 1, 1, 0, 0, D, C, k, p->max_iterations, et, er);
    } else if (plane) {
      GHICP_LAUNCH(k_icp_sum_pl, nb, IC_RED_T, 0, 0, W.get(), d_tgt, d_nrm, corr.get(), n, tot.get(), part_pl.get());
      GHICP_LAUNCH(k_icp_total_pl, 1, IC_RED_T, 0, 0, part_pl.get(), nb, tot_pl.get());
      GHICP_LAUNCH(k_icp_solve_pl, 1, 1, 0, 0, D, tot.get(), tot_pl.get(), k, p->max_iterations, p->transformation_epsilon,
                   p->fitness_epsilon);
    } else {
      GHICP_LAUNCH(k_icp_sum<2>, nb, IC_RED_T, 0, 0, W.get(), d_tgt, corr.get(), d2.get(), n, tot.get(), part.get());
      GHICP_LAUNCH(k_icp_total, 1, IC_RED_T, 0, 0, part.get(), nb, tot.get() + 1);
      GHICP_LAUNCH(k_icp_solve, 1, 1, 0, 0, D, tot.get(), tot.get() + 1, k, p->max_iterations, p->transformation_epsilon,
                   p->fitness_epsilon);
    }
    if (gicp) GHICP_LAUNCH(k_icp_move, iblk(n, IC_T), IC_T, 0, 0, d_src, W.get(), n, D->h.F);   // W = F P, as PCL moves its output
    else GHICP_LAUNCH(k_icp_move, iblk(n, IC_T), IC_T, 0, 0, W.get(), W.get(), n, D->T);
    CUDA_TRY(cudaGetLastError());
    // the one read-back of an iteration
    CUDA_TRY(cudaMemcpyAsync(&hh, &D->h, sizeof(hh), cudaMemcpyDeviceToHost, 0));
    CUDA_TRY(cudaStreamSynchronize(0));
    cor_tr.push_back(hh.cor);
    mse_tr.push_back(hh.mse);
    if (hh.state != 0) break;
  }
  if (ev_fit) CUDA_TRY(cudaEventRecord(ev_fit, 0));
  double Rt[16];
  for (int r = 0; r < 4; ++r)
    for (int c = 0; c < 4; ++c) Rt[c * 4 + r] = (double)hh.F[r * 4 + c];
  // PCL's getFitnessScore after align: the §3.12 fitness of the whole source moved by F, max_range = +inf
  ghicp_overlap_result ov{};
  CUDA_TRY(overlap_run(d_all, n_all, t, Rt, 1.f, (double)INFINITY, 1, nullptr, &ov, nullptr));
  if (h_moved) {
    GHICP_LAUNCH(k_icp_move, iblk(n_all, IC_T), IC_T, 0, 0, d_all, moved.get(), (long long)n_all, D->h.F);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(h_moved, moved.get(), 3 * sizeof(float) * (size_t)n_all, cudaMemcpyDeviceToHost, 0));
  }
  CUDA_TRY(cudaStreamSynchronize(0));
  ghicp_icp_result r{};
  std::memcpy(r.Rt, Rt, sizeof(Rt));
  r.mse = hh.mse;
  r.fitness = ov.fitness;
  r.iterations = k;
  r.state = hh.state;
  r.converged = hh.state != GHICP_ICP_NO_CORRESPONDENCES && hh.state != GHICP_ICP_SINGULAR;
  r.cor = hh.cor;
  r.cells_visited = (long long)hh.work[0];
  r.candidates = (long long)hh.work[1];
  *out = r;
  if (h_cor) std::copy(cor_tr.begin(), cor_tr.end(), h_cor);
  if (h_mse) std::copy(mse_tr.begin(), mse_tr.end(), h_mse);
  return cudaSuccess;
}

}  // namespace ghicp_b200
