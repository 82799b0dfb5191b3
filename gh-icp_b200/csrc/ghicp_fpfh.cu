// ghicp_fpfh.cu — MATRIX-FREE FPFH cost path (BASELINE.json config 3: 200k x 200k, FPFH-33, NN + reciprocal).
//
// The reference materialises FD = calFD_FPFH as N x M doubles (src/ghicp_reg.cpp:202-214; 320 GB at 200k x 200k,
// SURVEY.md §8a-5) and the stored-plane path of this library keeps it as N x M floats (160 GB at that size).
// Here nothing of size N x M exists: the row / column sweeps recompute
//     FD(i,j) = | sum_k (a_k - mean a)(b_k - mean b) / sqrt( sum (a-mean a)^2 * sum (b-mean b)^2 ) |
// (include/fpfh.hpp:135-165) on the fly from the centred histograms, in float32 and in the reference's operation
// order (serial sums over the 33 bins, separately rounded multiply and add: this file is compiled with --fmad=false),
// so every FD value — and therefore every CD double, every argmin and every gate decision — is bit-identical to the
// stored-plane kernels (k_fd_fpfh + k_rowsweep / k_colsweep in ghicp_kernels.cu) and to the oracle.
//
// Layouts: centred histograms are kept twice, 36 floats per keypoint (33 bins, sum of squares, 2 pad):
//   row-major   hc [n][36]  — staged into shared memory for the 8 rows (columns) a CTA owns
//   transposed  hcT[36][n]  — a thread's own column (row) histogram, read coalesced across the warp
// Per iteration algorithmic work: 33 multiply-adds + ~12 FP64 operations + one pow() per pair; bytes are O(N + M)
// per CTA row block (the 5.3 KB/keypoint-pair tiles stay in L2), i.e. the path is FP-pipe bound, not HBM bound.
#include <algorithm>
#include <climits>
#include <cmath>

#include "ghicp_internal.h"
#include "ghicp_device.cuh"

namespace ghicp_b200 {

namespace {

constexpr int HP = 36;            // histogram pitch (floats)
constexpr int MF_THREADS = 256;
constexpr int MF_CT = 8;          // target columns per CTA in the column sweep

// Per keypoint: mean (serial float sum / 33), centred histogram, serial sum of squares — the same arithmetic as
// k_fpfh_center (include/fpfh.hpp:139-155), written in both layouts.
__global__ void k_fpfh_center2(const float *__restrict__ h, float *__restrict__ hc, float *__restrict__ hcT, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float *p = h + (size_t)i * 33;
  float mean = 0.f;
  for (int k = 0; k < 33; ++k) mean += p[k];
  mean /= 33;
  float d = 0.f;
  float *q = hc + (size_t)i * HP;
  for (int k = 0; k < 33; ++k) {
    const float c = p[k] - mean;
    q[k] = c;
    hcT[(size_t)k * n + i] = c;
    d += c * c;
  }
  q[33] = d; q[34] = 0.f; q[35] = 0.f;
  hcT[(size_t)33 * n + i] = d;
  hcT[(size_t)34 * n + i] = 0.f;
  hcT[(size_t)35 * n + i] = 0.f;
}

// compute_fpfh_distance (include/fpfh.hpp:157-164) for one pair: `a` = 36 floats in shared memory (the CTA's row or
// column), `b` = the thread's own histogram in registers.  up accumulates serially over k = 0..32.
__device__ __forceinline__ float fpfh_fd(const float *__restrict__ a, const float (&b)[33], float bd) {
  float up = 0.f;
#pragma unroll
  for (int k = 0; k < 33; ++k) up += a[k] * b[k];
  return fabsf(up / sqrtf(a[33] * bd));
}

struct MfRowArgs {
  const double *s, *t;        // [3][N], [3][M]
  const float *sc;            // source centred histograms, row-major [N][36]
  const float *tcT;           // target centred histograms, transposed [36][M]
  int N, M, n_chunks, cols_per_chunk, row0, nloc;
  CostParams cp;
  double *part_cd; int *part_idx; double *part_stats;   // mode 0
  const DevIter *iter; int *cnt; const long long *rowptr; int *cursor;   // modes 1 / 2
  int *csr_col; double *csr_gain; float *csr_fd;
};

// Row sweep, same contract as k_rowsweep<GHICP_FT_FPFH, MODE> (ghicp_kernels.cu):
//   MODE 0: per-row first-argmin of CD + sum(cd - pivot), sum((cd - pivot)^2)   (src/ghicp_reg.cpp:295-341, 715-733)
//   MODE 1: per-row count of CD < penalty                                       (KM graph build, :358-365)
//   MODE 2: emit (j, penalty - CD, FD) for CD < penalty into the CSR
// One CTA owns TR source rows (histograms + coordinates in shared memory) and a chunk of target columns; a thread
// owns one column at a time: its histogram lives in 33 registers while the TR rows are swept.
template <int MODE>
__global__ void __launch_bounds__(MF_THREADS) k_rowsweep_mf(const MfRowArgs a) {
  __shared__ double s_src[3][TR];
  __shared__ __align__(16) float s_h[TR][HP];
  __shared__ double s_red[2 * (MF_THREADS / 32)];
  __shared__ double s_bv[TR][MF_THREADS / 32];
  __shared__ int s_bi[TR][MF_THREADS / 32];
  const int tid = threadIdx.x;
  const int i0 = a.row0 + blockIdx.x * TR;
  const int chunk = blockIdx.y;
  const int nrows = min(TR, a.row0 + a.nloc - i0);
  const int c0 = chunk * a.cols_per_chunk;
  const int c1 = min(a.M, c0 + a.cols_per_chunk);
  if (tid < 3 * TR) {
    const int k = tid / TR, r = tid % TR;
    s_src[k][r] = (r < nrows) ? a.s[(size_t)k * a.N + i0 + r] : 0.0;
  }
  for (int k = tid; k < TR * HP; k += MF_THREADS) {
    const int r = k / HP, q = k % HP;
    s_h[r][q] = (r < nrows) ? a.sc[(size_t)(i0 + r) * HP + q] : 0.f;
  }
  __syncthreads();

  double best[TR];
  int bidx[TR];
  int cnt[TR];
#pragma unroll
  for (int r = 0; r < TR; ++r) { best[r] = MAXVALIUE; bidx[r] = 0; cnt[r] = 0; }
  double sum = 0.0, sumsq = 0.0;
  double penalty = 0.0;
  if (MODE != 0) penalty = a.iter->penalty;

  const double *tx = a.t, *ty = a.t + a.M, *tz = a.t + 2 * (size_t)a.M;
  for (int j = c0 + tid; j < c1; j += MF_THREADS) {
    // the CTA's rows are re-read from shared memory for every column: without this barrier the compiler hoists
    // all TR x 34 loop-invariant loads out of the column loop and spills them to local memory
    asm volatile("" ::: "memory");
    float th[33];
#pragma unroll
    for (int k = 0; k < 33; ++k) th[k] = a.tcT[(size_t)k * a.M + j];
    const float td = a.tcT[(size_t)33 * a.M + j];
    const double cx = tx[j], cy = ty[j], cz = tz[j];
#pragma unroll
    for (int r = 0; r < TR; ++r) {
      if (r < nrows) {
        const float fdf = fpfh_fd(s_h[r], th, td);
        const double fd = (double)fdf;
        const double ed = ed_exact(s_src[0][r], s_src[1][r], s_src[2][r], cx, cy, cz, a.cp.scale);
        const double cd = cd_exact<GHICP_FT_FPFH>(ed, fd, a.cp);
        if (MODE == 0) {
          if (cd < best[r]) { best[r] = cd; bidx[r] = j; }
          const double d = cd - a.cp.pivot;
          sum += d;
          sumsq += d * d;
        } else if (MODE == 1) {
          cnt[r] += (cd < penalty) ? 1 : 0;
        } else {
          if (cd < penalty) {
            const size_t slot = (size_t)(i0 + r) * a.n_chunks + chunk;
            const long long pos = a.rowptr[slot] + atomicAdd(&a.cursor[slot], 1);
            a.csr_col[pos] = j;
            a.csr_gain[pos] = penalty - cd;
            a.csr_fd[pos] = fdf;
          }
        }
      }
    }
  }

  const int lane = tid & 31, warp = tid >> 5;
  if (MODE == 0) {
#pragma unroll
    for (int r = 0; r < TR; ++r) {
      warp_lexmin(best[r], bidx[r]);
      if (lane == 0) { s_bv[r][warp] = best[r]; s_bi[r][warp] = bidx[r]; }
    }
    const double ws = warp_sum(sum), wq = warp_sum(sumsq);
    if (lane == 0) { s_red[warp] = ws; s_red[MF_THREADS / 32 + warp] = wq; }
    __syncthreads();
    if (tid < nrows) {
      double v = s_bv[tid][0];
      int ix = s_bi[tid][0];
      for (int w = 1; w < MF_THREADS / 32; ++w) lexmin(v, ix, s_bv[tid][w], s_bi[tid][w]);
      a.part_cd[(size_t)(i0 + tid) * a.n_chunks + chunk] = v;
      a.part_idx[(size_t)(i0 + tid) * a.n_chunks + chunk] = ix;
    }
    if (tid == 0) {
      double S1 = 0.0, S2 = 0.0;
      for (int w = 0; w < MF_THREADS / 32; ++w) { S1 += s_red[w]; S2 += s_red[MF_THREADS / 32 + w]; }
      const size_t b = (size_t)blockIdx.y * gridDim.x + blockIdx.x;
      a.part_stats[2 * b] = S1;
      a.part_stats[2 * b + 1] = S2;
    }
  } else if (MODE == 1) {
#pragma unroll
    for (int r = 0; r < TR; ++r) {
      const int w = warp_sum_i(cnt[r]);
      if (lane == 0) s_bi[r][warp] = w;
    }
    __syncthreads();
    if (tid < nrows) {
      int tot = 0;
      for (int w = 0; w < MF_THREADS / 32; ++w) tot += s_bi[tid][w];
      a.cnt[(size_t)(i0 + tid) * a.n_chunks + chunk] = tot;
    }
  }
}

// Column sweep (NNR, src/ghicp_reg.cpp:637-650): per target column the first-argmin over the source rows of this
// context.  One CTA owns MF_CT columns (shared memory); a thread owns one source row at a time.
struct MfColArgs {
  const double *s, *t;
  const float *scT;           // source centred histograms, transposed [36][N]
  const float *tc;            // target centred histograms, row-major [M][36]
  int N, M, row0, nloc;
  CostParams cp;
  double *col_cd; int *col_idx;
};
__global__ void __launch_bounds__(MF_THREADS) k_colsweep_mf(const MfColArgs a) {
  __shared__ double s_t[3][MF_CT];
  __shared__ __align__(16) float s_h[MF_CT][HP];
  __shared__ double s_bv[MF_CT][MF_THREADS / 32];
  __shared__ int s_bi[MF_CT][MF_THREADS / 32];
  const int tid = threadIdx.x;
  const int j0 = blockIdx.x * MF_CT;
  const int ncols = min(MF_CT, a.M - j0);
  if (tid < 3 * MF_CT) {
    const int k = tid / MF_CT, c = tid % MF_CT;
    s_t[k][c] = (c < ncols) ? a.t[(size_t)k * a.M + j0 + c] : 0.0;
  }
  for (int k = tid; k < MF_CT * HP; k += MF_THREADS) {
    const int c = k / HP, q = k % HP;
    s_h[c][q] = (c < ncols) ? a.tc[(size_t)(j0 + c) * HP + q] : 0.f;
  }
  __syncthreads();
  double best[MF_CT];
  int bidx[MF_CT];
#pragma unroll
  for (int c = 0; c < MF_CT; ++c) { best[c] = MAXVALIUE; bidx[c] = 0; }
  const double *sxp = a.s, *syp = a.s + a.N, *szp = a.s + 2 * (size_t)a.N;
  for (int i = a.row0 + tid; i < a.row0 + a.nloc; i += MF_THREADS) {
    asm volatile("" ::: "memory");   // keep the CTA's column histograms in shared memory (see k_rowsweep_mf)
    float sh[33];
#pragma unroll
    for (int k = 0; k < 33; ++k) sh[k] = a.scT[(size_t)k * a.N + i];
    const float sd = a.scT[(size_t)33 * a.N + i];
    const double sx = sxp[i], sy = syp[i], sz = szp[i];
#pragma unroll
    for (int c = 0; c < MF_CT; ++c) {
      if (c < ncols) {
        // a[k] * b[k] and a[33] * bd commute exactly: same floats as the row sweep's (source, target) order
        const float fdf = fpfh_fd(s_h[c], sh, sd);
        const double ed = ed_exact(sx, sy, sz, s_t[0][c], s_t[1][c], s_t[2][c], a.cp.scale);
        const double cd = cd_exact<GHICP_FT_FPFH>(ed, (double)fdf, a.cp);
        if (cd < best[c]) { best[c] = cd; bidx[c] = i; }
      }
    }
  }
  const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
  for (int c = 0; c < MF_CT; ++c) {
    warp_lexmin(best[c], bidx[c]);
    if (lane == 0) { s_bv[c][warp] = best[c]; s_bi[c][warp] = bidx[c]; }
  }
  __syncthreads();
  if (tid < ncols) {
    double v = s_bv[tid][0];
    int ix = s_bi[tid][0];
    for (int w = 1; w < MF_THREADS / 32; ++w) lexmin(v, ix, s_bv[tid][w], s_bi[tid][w]);
    a.col_cd[j0 + tid] = v;
    a.col_idx[j0 + tid] = ix;
  }
}

// one pair from the row-major histograms (serial, same order)
__device__ __forceinline__ float fpfh_fd_pair(const float *__restrict__ a, const float *__restrict__ b) {
  float up = 0.f;
  for (int k = 0; k < 33; ++k) up += a[k] * b[k];
  return fabsf(up / sqrtf(a[33] * b[33]));
}
// FD of (row, its partner) for the pair statistics FDM / FDstd (src/ghicp_reg.cpp:745-760)
__global__ void k_rowfd_mf(const float *__restrict__ sc, const float *__restrict__ tc, const int *__restrict__ row_idx,
                           int row0, int nloc, float *__restrict__ row_fd) {
  const int i = row0 + blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= row0 + nloc) return;
  row_fd[i] = fpfh_fd_pair(sc + (size_t)i * HP, tc + (size_t)row_idx[i] * HP);
}
// Energyfunction::FD as doubles (test / debug entry point ghicp_get_fd)
__global__ void k_fd_to_double_mf(const float *__restrict__ sc, const float *__restrict__ tc, int N, int M, int row0,
                                  int nloc, double *__restrict__ out) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)N * M) return;
  const int i = (int)(idx / M), j = (int)(idx % M);
  if (i < row0 || i >= row0 + nloc) { out[idx] = 0.0; return; }
  out[idx] = (double)fpfh_fd_pair(sc + (size_t)i * HP, tc + (size_t)j * HP);
}


// =====================================================================================================================
// FAST path: FP32 filter + exact FP64 refinement (the scheme of ghicp_stream.cu with FD recomputed on the fly).
//
// Every decision the reference takes on doubles (row / column argmin with the first-minimum tie-break) is taken on the
// exactly evaluated CD of the few pairs an FP32 filter cannot rule out:
//   filter   cd32 = scale * dist32 * fd32^(-ex) dist32 from hi/lo-split centred coordinates (relative error ~2^-22),
//                                              fd32 = |<h_s, h_t>| of the L2-normalised centred histograms (33 FFMA),
//                                              fd^(-ex) = ex2(-ex * lg2(fd))  (MUFU)
//   bound    |fd32 - FD_reference| <= FF_G     (both are 33-term float dot products of vectors of norm <= 1; the
//                                              reference's own float evaluation carries the same kind of error)
//            => CD_exact >= LB = cd32 * (1 - FF_D0 - 1.5 * ex * FF_G / fd32)      while FF_G / fd32 <= 1/8;
//            below that (|correlation| < 6.4e-5, CD astronomically large) the rare path re-derives a bound from fd32 + FF_G
//   refine   every pair with LB <= thr(row) (or thr(column)) is evaluated EXACTLY (reference operation order), its CD
//            goes to atomicMin(rowbest / colbest) and to the candidate list; k_ff_resolve keeps the smallest index among
//            the candidates equal to the minimum.  thr = exact CD of a guess pair (last iteration's partner, or the FP32
//            argmin found by the PRE pass), so the true minimum always passes.
// Statistics: only the CD SUM is kept (FP32 values, FP64 accumulation).  In FPFH mode the mean is dominated by pairs of
// near-zero correlation (CD = ED / FD^ex is heavy-tailed) and cannot be reproduced by a filter, so the host only takes
// this path when no decision depends on it (NNR: no gate; NN from iteration 2 on: penalty = RMS*para1*scale*para2,
// src/ghicp_reg.cpp:327-330) and reports the estimate.
// =====================================================================================================================
constexpr int FF_THREADS = 256;
constexpr int FF_RB = 32;        // source rows staged in shared memory per step
constexpr int FF_ROWS = 1024;    // source rows per CTA
constexpr int FF_REC = 40;       // floats per source record: 33 normalised bins, hi xyz, lo xyz, row threshold
constexpr float FF_D0 = 3e-5f;   // relative slack: sqrt / lg2 / ex2 approximations, coordinate split, normalisation
constexpr float FF_G = 8e-6f;    // absolute bound on |fd32 - FD_reference|
typedef unsigned long long ffu64;

__device__ __forceinline__ float ff_lg2(float x) {
#if defined(GHICP_EMU_HOST)
  return log2f(x);
#else
  float r; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r;
#endif
}
__device__ __forceinline__ float ff_ex2(float x) {
#if defined(GHICP_EMU_HOST)
  return exp2f(x);
#else
  float r; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r;
#endif
}
__device__ __forceinline__ float ff_sqrt(float x) {
#if defined(GHICP_EMU_HOST)
  return sqrtf(x);
#else
  float r; asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r;
#endif
}
__device__ __forceinline__ ffu64 ff_ord64(double v) { return (ffu64)__double_as_longlong(v); }  // CD >= 0: monotone bits

struct FfArgs {
  const double *s, *t;          // exact coordinates [3][N], [3][M]
  const float *sc, *tc;         // exact path: centred histograms, row-major [n][36]
  const float *srec;            // filter: source records [N][FF_REC]
  const float *tnT;             // filter: normalised target histograms, transposed [36][M]
  const float *tco;             // filter: target coordinates hi xyz, lo xyz, transposed [6][M]
  int N, M, row0, nloc;
  CostParams cp;
  float scalef;                 // (float) cp.scale
  float exf;                    // (float) cp.ex
  float c1;                     // 1.5 * ex * FF_G
  float *thr_row, *thr_col;     // upper bounds of the exact minima (rounded up)
  ffu64 *rowguess, *colguess;   // PRE pass: packed (cd32 bits << 32 | index)
  ffu64 *rowbest, *colbest;     // exact minima, ordered-double bits
  int *rowidx, *colidx;
  Cand *cand[2]; int cand_cap;
  StreamDev *dev;
  double *part;                 // [grid] CD sums
};

// exact CD(i,j): reference operation order (include/fpfh.hpp:135-165, src/ghicp_reg.cpp:122, 308)
__device__ GHICP_NOINLINE double ff_exact_cd(const FfArgs &a, int i, int j) {
  const float fdf = fpfh_fd_pair(a.sc + (size_t)i * HP, a.tc + (size_t)j * HP);
  const double ed = ed_exact(a.s[i], a.s[(size_t)a.N + i], a.s[2 * (size_t)a.N + i], a.t[j], a.t[(size_t)a.M + j],
                             a.t[2 * (size_t)a.M + j], a.cp.scale);
  return cd_exact<GHICP_FT_FPFH>(ed, (double)fdf, a.cp);
}
// saturating like push_candidate (ghicp_stream.cu): the count stays below cap + resident threads and cannot wrap
__device__ __forceinline__ void ff_push(const FfArgs &a, int which, int i, int j, double cd) {
  if (*(volatile int *)&a.dev->cand_count[which] >= a.cand_cap) { a.dev->overflow = 1; return; }
  const int slot = atomicAdd(&a.dev->cand_count[which], 1);
  if (slot < a.cand_cap) {
    Cand c;
    c.i = i; c.j = j; c.cd = cd;
    a.cand[which][slot] = c;
  } else {
    a.dev->overflow = 1;
  }
}
// rare path: the filter could not rule the pair out.  fd32 so small that the first-order bound does not apply
// (FF_G / fd32 > 1/8) gets a bound from fd32 + FF_G >= FD_reference first.
__device__ GHICP_NOINLINE void ff_slow(const FfArgs &a, int which, int i, int j, float dist, float fd, float thr) {
  if (FF_G > 0.125f * fd) {
    const float lb2 = dist * ff_ex2(-a.exf * ff_lg2(fd + FF_G)) * (1.f - FF_D0);
    if (lb2 > thr) return;
  }
  const double e = ff_exact_cd(a, i, j);
  if (!(e == e)) return;  // NaN (degenerate histogram): never a minimum in the reference's '<' scans either
  if (which == 0) atomicMin(&a.rowbest[i], ff_ord64(e)); else atomicMin(&a.colbest[j], ff_ord64(e));
  ff_push(a, which, i, j, e);
}

// Per-iteration operands: centred coordinates split into hi + lo floats (their difference then carries a RELATIVE
// error of ~2^-23 even for nearly coincident points), written into the source records / the target SoA array.
__global__ void k_ff_prep(const double *__restrict__ s, const double *__restrict__ t, int N, int M, double cx, double cy,
                          double cz, float *__restrict__ srec, float *__restrict__ tco) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < N) {
    const double x = s[k] - cx, y = s[(size_t)N + k] - cy, z = s[2 * (size_t)N + k] - cz;
    const float xh = (float)x, yh = (float)y, zh = (float)z;
    float *r = srec + (size_t)k * FF_REC;
    r[33] = xh; r[34] = yh; r[35] = zh;
    r[36] = (float)(x - (double)xh); r[37] = (float)(y - (double)yh); r[38] = (float)(z - (double)zh);
  }
  if (k < M) {
    const double x = t[k] - cx, y = t[(size_t)M + k] - cy, z = t[2 * (size_t)M + k] - cz;
    const float xh = (float)x, yh = (float)y, zh = (float)z;
    tco[k] = xh; tco[(size_t)M + k] = yh; tco[2 * (size_t)M + k] = zh;
    tco[3 * (size_t)M + k] = (float)(x - (double)xh);
    tco[4 * (size_t)M + k] = (float)(y - (double)yh);
    tco[5 * (size_t)M + k] = (float)(z - (double)zh);
  }
}
// One-time: L2-normalised centred histograms for the filter (source: into the records; target: transposed)
__global__ void k_ff_normalise(const float *__restrict__ sc, const float *__restrict__ tc, int N, int M,
                               float *__restrict__ srec, float *__restrict__ tnT) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < N) {
    const float *h = sc + (size_t)k * HP;
    const float inv = h[33] > 0.f ? 1.0f / sqrtf(h[33]) : 0.f;
    float *r = srec + (size_t)k * FF_REC;
    for (int q = 0; q < 33; ++q) r[q] = h[q] * inv;
    for (int q = 33; q < FF_REC; ++q) r[q] = 0.f;
  }
  if (k < M) {
    const float *h = tc + (size_t)k * HP;
    const float inv = h[33] > 0.f ? 1.0f / sqrtf(h[33]) : 0.f;
    for (int q = 0; q < 33; ++q) tnT[(size_t)q * M + k] = h[q] * inv;
    for (int q = 33; q < HP; ++q) tnT[(size_t)q * M + k] = 0.f;
  }
}

// Thresholds: exact CD of the guess pairs (PRE pass argmin and / or last iteration's partner), rounded up.
__global__ void k_ff_seed(FfArgs a, const int *__restrict__ prev_row_idx, const int *__restrict__ prev_col_idx,
                          int have_prev, int use_guess, int with_cols, float *__restrict__ srec) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  const float INF = __uint_as_float(0x7f800000u);
  if (k >= a.row0 && k < a.row0 + a.nloc) {
    double best = 1e300;
    bool any = false;
    if (use_guess && a.rowguess[k] != ~0ull) {
      const int j = (int)(unsigned)(a.rowguess[k] & 0xffffffffull);
      const double e = ff_exact_cd(a, k, j);
      if (e == e && e < best) { best = e; any = true; }
    }
    if (have_prev) {
      const int j = prev_row_idx[k];
      if (j >= 0 && j < a.M) { const double e = ff_exact_cd(a, k, j); if (e == e && e < best) { best = e; any = true; } }
    }
    const float thr = any ? __double2float_ru(best * 1.0000001) : INF;
    a.thr_row[k] = thr;
    srec[(size_t)k * FF_REC + 39] = thr;
    a.rowbest[k] = ~0ull;
    a.rowidx[k] = INT_MAX;
    a.rowguess[k] = ~0ull;
  }
  if (with_cols && k < a.M) {
    double best = 1e300;
    bool any = false;
    if (use_guess && a.colguess[k] != ~0ull) {
      const int i = (int)(unsigned)(a.colguess[k] & 0xffffffffull);
      const double e = ff_exact_cd(a, i, k);
      if (e == e && e < best) { best = e; any = true; }
    }
    if (have_prev) {
      const int i = prev_col_idx[k];
      if (i >= a.row0 && i < a.row0 + a.nloc) { const double e = ff_exact_cd(a, i, k); if (e == e && e < best) { best = e; any = true; } }
    }
    a.thr_col[k] = any ? __double2float_ru(best * 1.0000001) : INF;
    a.colbest[k] = ~0ull;
    a.colidx[k] = INT_MAX;
    a.colguess[k] = ~0ull;
  }
}

// The sweep.  PRE = true: FP32 argmin per row (and column) -> guess pairs.  PRE = false: candidate gate + statistics.
// A thread owns TWO target columns (j and j + FF_THREADS; their normalised histograms and split coordinates stay in
// registers); the CTA walks FF_ROWS source rows, FF_RB at a time through shared memory.  One row's record is read from shared
// memory once (broadcast LDS.128) and serves both columns: the two 33-term dots are the two independent instruction
// streams, and the operand traffic per pair is half of the one-column form (ncu, round 2: LSU 31 % of the issue slots there).
constexpr int FF_CPT = 2;   // columns per thread
template <bool PRE, bool COLS>
__global__ void __launch_bounds__(FF_THREADS, 2) k_ff_sweep(const FfArgs a) {
  __shared__ __align__(16) float s_rec[FF_RB][FF_REC];
  __shared__ ffu64 s_guess[FF_RB];
  __shared__ double s_red[FF_THREADS / 32];
  const int tid = threadIdx.x, lane = tid & 31;
  const int i_begin = a.row0 + blockIdx.y * FF_ROWS;
  const int i_end = min(a.row0 + a.nloc, i_begin + FF_ROWS);
  const float INF = __uint_as_float(0x7f800000u);

  int jc[FF_CPT]; bool valid[FF_CPT];
  float ht[FF_CPT][33];
  float txh[FF_CPT], tyh[FF_CPT], tzh[FF_CPT], txl[FF_CPT], tyl[FF_CPT], tzl[FF_CPT], thr_c[FF_CPT], cmin[FF_CPT];
  int carg[FF_CPT];
#pragma unroll
  for (int c = 0; c < FF_CPT; ++c) {
    const int jraw = (blockIdx.x * FF_CPT + c) * FF_THREADS + tid;
    valid[c] = jraw < a.M;
    const int j = valid[c] ? jraw : a.M - 1;
    jc[c] = j;
#pragma unroll
    for (int k = 0; k < 33; ++k) ht[c][k] = a.tnT[(size_t)k * a.M + j];
    txh[c] = a.tco[j]; tyh[c] = a.tco[(size_t)a.M + j]; tzh[c] = a.tco[2 * (size_t)a.M + j];
    txl[c] = a.tco[3 * (size_t)a.M + j]; tyl[c] = a.tco[4 * (size_t)a.M + j]; tzl[c] = a.tco[5 * (size_t)a.M + j];
    thr_c[c] = (!PRE && COLS && valid[c]) ? a.thr_col[j] : -INF;
    cmin[c] = INF;   // PRE: running column minimum over this CTA's rows
    carg[c] = 0;
  }
  double dsum = 0.0;

  for (int ib = i_begin; ib < i_end; ib += FF_RB) {
    const int nb = min(FF_RB, i_end - ib);
    __syncthreads();
    for (int k = tid; k < nb * FF_REC; k += FF_THREADS) s_rec[k / FF_REC][k % FF_REC] = a.srec[(size_t)ib * FF_REC + k];
    if (PRE && tid < FF_RB) s_guess[tid] = ~0ull;
    __syncthreads();
    float fsum = 0.f;
    for (int r = 0; r < nb; ++r) {
      asm volatile("" ::: "memory");   // keep the records in shared memory (no hoisting into registers / local memory)
      const float *rec = s_rec[r];
      float cd32[FF_CPT], dist[FF_CPT], fd[FF_CPT], l[FF_CPT];
      {
        // the filter value of both columns and what the rare path needs; three independent partial sums per dot
        float d0[FF_CPT], d1[FF_CPT], d2s[FF_CPT];
#pragma unroll
        for (int c = 0; c < FF_CPT; ++c) { d0[c] = 0.f; d1[c] = 0.f; d2s[c] = 0.f; }
#pragma unroll
        for (int k = 0; k < 11; ++k) {
          const float r0 = rec[k], r1 = rec[11 + k], r2 = rec[22 + k];
#pragma unroll
          for (int c = 0; c < FF_CPT; ++c) {
            d0[c] = fmaf(r0, ht[c][k], d0[c]);
            d1[c] = fmaf(r1, ht[c][11 + k], d1[c]);
            d2s[c] = fmaf(r2, ht[c][22 + k], d2s[c]);
          }
        }
        const float sxh = rec[33], syh = rec[34], szh = rec[35], sxl = rec[36], syl = rec[37], szl = rec[38];
#pragma unroll
        for (int c = 0; c < FF_CPT; ++c) {
          const float dx = (sxh - txh[c]) + (sxl - txl[c]);
          const float dy = (syh - tyh[c]) + (syl - tyl[c]);
          const float dz = (szh - tzh[c]) + (szl - tzl[c]);
          const float d2 = fmaf(dz, dz, fmaf(dy, dy, dx * dx));
          fd[c] = fmaxf(fabsf((d0[c] + d1[c]) + d2s[c]), 1e-30f);
          dist[c] = a.scalef * ff_sqrt(d2);   // ED (src/ghicp_reg.cpp:122) in FP32
          l[c] = ff_lg2(fd[c]);
          cd32[c] = valid[c] ? dist[c] * ff_ex2(-a.exf * l[c]) : INF;
        }
      }
      if (PRE) {
        // warp argmin of the row over both columns of every lane: REDUX on the (non-negative) float bits, then the
        // smallest column index among the holders of the minimum (= the first minimum of the row scan)
        unsigned bmin = __float_as_uint(cd32[0]);
#pragma unroll
        for (int c = 1; c < FF_CPT; ++c) { const unsigned bc = __float_as_uint(cd32[c]); bmin = bc < bmin ? bc : bmin; }
        const unsigned m = __reduce_min_sync(0xffffffffu, bmin);
        if (m < 0x7f800000u) {
          unsigned jm = 0xffffffffu;
#pragma unroll
          for (int c = FF_CPT - 1; c >= 0; --c) if (__float_as_uint(cd32[c]) == m) jm = (unsigned)jc[c];   // jc ascending in c
          const unsigned jmin = __reduce_min_sync(0xffffffffu, jm);
          if (jm == jmin && jm != 0xffffffffu) atomicMin(&s_guess[r], ((ffu64)m << 32) | jmin);
        }
        if (COLS) {
#pragma unroll
          for (int c = 0; c < FF_CPT; ++c)
            if (cd32[c] < cmin[c]) { cmin[c] = cd32[c]; carg[c] = ib + r; }
        }
      } else {
        const float thr_r = rec[39];
#pragma unroll
        for (int c = 0; c < FF_CPT; ++c) {
          fsum += valid[c] ? cd32[c] : 0.f;
          const float rinv = ff_ex2(-l[c]);                         // ~ 1 / fd32
          // <= exact CD.  The first-order term only holds while FF_G / fd32 <= 1/8: below that the pair always takes the
          // rare path, which bounds it through fd32 + FF_G instead.
          const float lb = fd[c] < 8.f * FF_G ? -INF : cd32[c] * (1.f - FF_D0 - a.c1 * rinv);
          if (valid[c] && lb <= thr_r) ff_slow(a, 0, ib + r, jc[c], dist[c], fd[c], thr_r);
          if (COLS && valid[c] && lb <= thr_c[c]) ff_slow(a, 1, ib + r, jc[c], dist[c], fd[c], thr_c[c]);
        }
      }
    }
    if (PRE) {
      __syncthreads();
      if (tid < nb && s_guess[tid] != ~0ull) atomicMin(&a.rowguess[ib + tid], s_guess[tid]);
    } else {
      dsum += (double)fsum;   // at most FF_CPT * FF_RB FP32 values per partial
    }
  }
  if (PRE) {
    if (COLS) {
#pragma unroll
      for (int c = 0; c < FF_CPT; ++c)
        if (valid[c] && cmin[c] < INF) atomicMin(&a.colguess[jc[c]], ((ffu64)__float_as_uint(cmin[c]) << 32) | (unsigned)carg[c]);
    }
  } else {
    double v[1] = {dsum};
    block_sum<1, FF_THREADS>(v, s_red);
    if (tid == 0) a.part[(size_t)blockIdx.y * gridDim.x + blockIdx.x] = v[0];
  }
}

// this rank's CD sum -> xstats (the penalty rule runs in k_penalty); fixed order: deterministic
__global__ void __launch_bounds__(1024) k_ff_stats(const double *__restrict__ part, int n_parts, double *__restrict__ xstats,
                                                   int rank) {
  __shared__ double sm[32];
  double v[1] = {0.0};
  for (int p = threadIdx.x; p < n_parts; p += blockDim.x) v[0] += part[p];
  block_sum<1, 1024>(v, sm);
  if (threadIdx.x == 0) {
    xstats[4 * rank] = v[0];
    xstats[4 * rank + 1] = 0.0;   // the CD variance is not defined for FPFH (src/ghicp_reg.cpp:317-335 uses the mean only)
    xstats[4 * rank + 2] = 0.0;
  }
}
// first-minimum tie-break: among the candidates whose exact CD equals the minimum keep the smallest index
// (src/ghicp_reg.cpp:626, 641, 719)
__global__ void k_ff_resolve(const FfArgs a, int which) {
  const int n = min(a.dev->cand_count[which], a.cand_cap);
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
    const Cand c = a.cand[which][k];
    if (which == 0) {
      if (ff_ord64(c.cd) == a.rowbest[c.i]) atomicMin(&a.rowidx[c.i], c.j);
    } else {
      if (ff_ord64(c.cd) == a.colbest[c.j]) atomicMin(&a.colidx[c.j], c.i);
    }
  }
}
__global__ void k_ff_publish(const FfArgs a, double *row_cd, int *row_idx, double *col_cd, int *col_idx, double *xstats,
                             int rank) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k == 0) xstats[4 * rank + 2] = a.dev->overflow ? 1.0 : 0.0;   // travels with the statistics
  if (k >= a.row0 && k < a.row0 + a.nloc) {
    // not found: every CD of the row is NaN or >= 9e20 (clouds of ~1e10 units) -> the reference scan, which starts at
    // (9e20, 0) and takes a CD only when it is smaller, keeps (9e20, 0)
    const int j = a.rowidx[k];
    const double v = __longlong_as_double((long long)a.rowbest[k]);
    const bool found = j != INT_MAX && v < MAXVALIUE;
    row_cd[k] = found ? v : MAXVALIUE;
    row_idx[k] = found ? j : 0;
  }
  if (col_cd && k < a.M) {
    const int i = a.colidx[k];
    const double v = __longlong_as_double((long long)a.colbest[k]);
    const bool found = i != INT_MAX && v < MAXVALIUE;
    col_cd[k] = found ? v : MAXVALIUE;
    col_idx[k] = found ? i : 0;
  }
}
// ---- KM gate on the same filter (FPFH + KM from iteration 2 on: penalty = RMS*para1*scale*para2, src/ghicp_reg.cpp:327-330,
//      independent of this iteration's CD) -----------------------------------------------------------------------------
// Every row gets the SAME threshold, the penalty: the sweep then evaluates exactly every pair whose lower bound does not
// exceed it and leaves (i, j, CD_exact) in the candidate list; the pairs with CD < penalty (strict, :362) are the KM graph.
// They travel as the candidate block of the settled KM route (ghicp_stream.cu: one all-gather, CSR built on every rank).
__global__ void k_ff_gate_seed(FfArgs a, LoopScalars ls, DevIter *iter, float *__restrict__ srec) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  const double penalty = ls.RMS * ls.para1 * ls.scale * ls.para2;   // the expression of k_penalty: the same double
  if (k == 0) iter->penalty = penalty;
  if (k >= a.row0 && k < a.row0 + a.nloc) {
    const float thr = __double2float_ru(penalty * 1.0000001);
    a.thr_row[k] = thr;
    srec[(size_t)k * FF_REC + 39] = thr;
    a.rowbest[k] = ~0ull;
    a.rowidx[k] = INT_MAX;
    a.rowguess[k] = ~0ull;
  }
}
__global__ void k_ff_cand_block(const FfArgs a, const DevIter *iter, XBlockHdr *hdr, unsigned long long *__restrict__ key,
                                double *__restrict__ gain, float *__restrict__ fd, unsigned long long xuse) {
  const int n = min(a.dev->cand_count[0], a.cand_cap);
  const double penalty = iter->penalty;
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
    const Cand c = a.cand[0][k];
    if (c.cd < penalty) {
      const unsigned long long pos = atomicAdd(&hdr->count, 1ull);
      if (pos < xuse) {
        key[pos] = ((unsigned long long)(unsigned)c.i << 32) | (unsigned)c.j;
        gain[pos] = penalty - c.cd;
        fd[pos] = fpfh_fd_pair(a.sc + (size_t)c.i * HP, a.tc + (size_t)c.j * HP);
      }
    }
  }
}
__global__ void k_ff_block_hdr(const FfArgs a, const double *__restrict__ xstats_rank, XBlockHdr *hdr, unsigned long long xuse) {
  const bool ovf = hdr->count > xuse || a.dev->overflow != 0;
  hdr->stats[0] = xstats_rank[0]; hdr->stats[1] = xstats_rank[1];
  hdr->stats[2] = ovf ? 1.0 : 0.0;   // picked up by k_penalty as DevIter::overflow_any on every rank
  hdr->stats[3] = 0.0;
  if (ovf) hdr->count = 0ull;
}

__global__ void k_ff_reset(StreamDev *dev) {
  dev->cand_count[0] = 0; dev->cand_count[1] = 0; dev->overflow = 0;
}

}  // namespace

cudaError_t launch_fpfh_prepare(Ctx *c) {
  GHICP_LAUNCH(k_fpfh_center2, (c->N + 127) / 128, 128, 0, c->stream, c->d_fs, c->d_fsc, c->d_fscT, c->N);
  GHICP_LAUNCH(k_fpfh_center2, (c->M + 127) / 128, 128, 0, c->stream, c->d_ft, c->d_ftc, c->d_ftcT, c->M);
  c->launches += 2;
  return cudaGetLastError();
}

cudaError_t launch_rowsweep_mf(Ctx *c, int mode, const CostParams &cp) {
  MfRowArgs a{};
  a.s = c->d_s; a.t = c->d_t; a.sc = c->d_fsc; a.tcT = c->d_ftcT;
  a.N = c->N; a.M = c->M; a.n_chunks = c->n_chunks;
  a.row0 = c->r0; a.nloc = c->nloc;
  a.cols_per_chunk = (c->M + c->n_chunks - 1) / c->n_chunks;
  a.cp = cp;
  a.part_cd = c->d_part_cd; a.part_idx = c->d_part_idx; a.part_stats = c->d_part_stats;
  a.iter = c->d_iter; a.cnt = c->d_cnt; a.rowptr = c->d_rowptr; a.cursor = c->d_cursor;
  a.csr_col = c->d_csr_col; a.csr_gain = c->d_csr_gain; a.csr_fd = c->d_csr_fd;
  const dim3 grid((c->nloc + TR - 1) / TR, c->n_chunks);
  if (mode == SWEEP_ROWMIN) GHICP_LAUNCH(k_rowsweep_mf<SWEEP_ROWMIN>, grid, MF_THREADS, 0, c->stream, a);
  else if (mode == SWEEP_COUNT) GHICP_LAUNCH(k_rowsweep_mf<SWEEP_COUNT>, grid, MF_THREADS, 0, c->stream, a);
  else GHICP_LAUNCH(k_rowsweep_mf<SWEEP_FILL>, grid, MF_THREADS, 0, c->stream, a);
  c->launches++;
  return cudaGetLastError();
}

cudaError_t launch_colsweep_mf(Ctx *c, const CostParams &cp) {
  MfColArgs a{};
  a.s = c->d_s; a.t = c->d_t; a.scT = c->d_fscT; a.tc = c->d_ftc;
  a.N = c->N; a.M = c->M; a.row0 = c->r0; a.nloc = c->nloc; a.cp = cp;
  a.col_cd = c->d_col_cd; a.col_idx = c->d_col_idx;
  GHICP_LAUNCH(k_colsweep_mf, (c->M + MF_CT - 1) / MF_CT, MF_THREADS, 0, c->stream, a);
  c->launches++;
  return cudaGetLastError();
}

cudaError_t launch_rowfd_mf(Ctx *c) {
  if (c->nloc <= 0) return cudaSuccess;
  GHICP_LAUNCH(k_rowfd_mf, (c->nloc + 255) / 256, 256, 0, c->stream, c->d_fsc, c->d_ftc, c->d_row_idx, c->r0, c->nloc, c->d_row_fd);
  c->launches++;
  return cudaGetLastError();
}

cudaError_t launch_get_fd_mf(Ctx *c, double *d_out) {
  const size_t total = (size_t)c->N * c->M;
  GHICP_LAUNCH(k_fd_to_double_mf, (unsigned)((total + 255) / 256), 256, 0, c->stream, c->d_fsc, c->d_ftc, c->N, c->M, c->r0, c->nloc, d_out);
  c->launches++;
  return cudaGetLastError();
}


// ---- fast path launchers ---------------------------------------------------------------------------------------------
static FfArgs ff_args(Ctx *c, const CostParams &cp) {
  FfArgs a{};
  a.s = c->d_s; a.t = c->d_t; a.sc = c->d_fsc; a.tc = c->d_ftc;
  a.srec = c->d_ff_srec; a.tnT = c->d_ff_tnT; a.tco = c->d_ff_tco;
  a.N = c->N; a.M = c->M; a.row0 = c->r0; a.nloc = c->nloc;
  a.cp = cp;
  a.scalef = (float)cp.scale;
  a.exf = (float)cp.ex;
  a.c1 = 1.5f * (float)cp.ex * FF_G;
  a.thr_row = reinterpret_cast<float *>(c->d_row_thr); a.thr_col = reinterpret_cast<float *>(c->d_col_thr);
  a.rowguess = c->d_ff_rowguess; a.colguess = c->d_ff_colguess;
  a.rowbest = c->d_rowbest; a.colbest = c->d_colbest; a.rowidx = c->d_rowidx2; a.colidx = c->d_colidx2;
  a.cand[0] = c->d_cand[0]; a.cand[1] = c->d_cand[1]; a.cand_cap = c->cand_cap;
  a.dev = c->d_sdev;
  a.part = c->d_ff_part;
  return a;
}
static dim3 ff_grid(const Ctx *c) { return dim3((c->M + FF_CPT * FF_THREADS - 1) / (FF_CPT * FF_THREADS), (c->nloc + FF_ROWS - 1) / FF_ROWS); }
size_t fpfh_fast_parts(const Ctx *c) { const dim3 g = ff_grid(c); return (size_t)g.x * g.y; }
size_t fpfh_fast_rec_floats() { return FF_REC; }

// one-time (after launch_fpfh_prepare): normalised histograms for the filter; guesses cleared
cudaError_t launch_fpfh_fast_build(Ctx *c) {
  const int n = c->N > c->M ? c->N : c->M;
  GHICP_LAUNCH(k_ff_normalise, (n + 127) / 128, 128, 0, c->stream, c->d_fsc, c->d_ftc, c->N, c->M, c->d_ff_srec, c->d_ff_tnT);
  c->launches++;
  return cudaGetLastError();
}
// per iteration: split coordinates, counters
cudaError_t launch_fpfh_fast_prep(Ctx *c) {
  const int n = c->N > c->M ? c->N : c->M;
  GHICP_LAUNCH(k_ff_prep, (n + 255) / 256, 256, 0, c->stream, c->d_s, c->d_t, c->N, c->M, c->center[0], c->center[1],
               c->center[2], c->d_ff_srec, c->d_ff_tco);
  GHICP_LAUNCH(k_ff_reset, 1, 1, 0, c->stream, c->d_sdev);
  c->launches += 2;
  return cudaGetLastError();
}
cudaError_t launch_fpfh_fast_seed(Ctx *c, const CostParams &cp, bool with_cols, bool use_guess) {
  const FfArgs a = ff_args(c, cp);
  const int n = c->N > c->M ? c->N : c->M;
  // sharded: seed a column from this rank's own best row of the last iteration (see launch_stream_seed)
  const int *prev_cols = (c->world > 1 && c->d_colg_idx) ? c->d_colg_idx + (size_t)c->rank * (size_t)c->M : c->d_col_idx;
  GHICP_LAUNCH(k_ff_seed, (n + 255) / 256, 256, 0, c->stream, a, c->d_row_idx, prev_cols, c->have_prev ? 1 : 0,
               use_guess ? 1 : 0, with_cols ? 1 : 0, c->d_ff_srec);
  c->launches++;
  return cudaGetLastError();
}
cudaError_t launch_fpfh_fast_sweep(Ctx *c, const CostParams &cp, bool pre, bool with_cols) {
  const FfArgs a = ff_args(c, cp);
  const dim3 grid = ff_grid(c);
  void (*kern)(const FfArgs) = pre ? (with_cols ? k_ff_sweep<true, true> : k_ff_sweep<true, false>)
                                   : (with_cols ? k_ff_sweep<false, true> : k_ff_sweep<false, false>);
  GHICP_LAUNCH(kern, grid, FF_THREADS, 0, c->stream, a);
  c->launches++;
  return cudaGetLastError();
}
// statistics -> xstats, exact index resolution, publication into d_row_cd / d_row_idx (/ d_col_*)
cudaError_t launch_fpfh_fast_finish(Ctx *c, const CostParams &cp, bool with_cols) {
  const FfArgs a = ff_args(c, cp);
  GHICP_LAUNCH(k_ff_stats, 1, 1024, 0, c->stream, c->d_ff_part, (int)fpfh_fast_parts(c), c->d_xstats, c->rank);
  GHICP_LAUNCH(k_ff_resolve, GHICP_SMS * 4, 256, 0, c->stream, a, 0);
  if (with_cols) GHICP_LAUNCH(k_ff_resolve, GHICP_SMS * 4, 256, 0, c->stream, a, 1);
  const int n = c->N > c->M ? c->N : c->M;
  GHICP_LAUNCH(k_ff_publish, (n + 255) / 256, 256, 0, c->stream, a, c->d_row_cd, c->d_row_idx,
               with_cols ? c->d_col_cd : (double *)nullptr, with_cols ? c->d_col_idx : (int *)nullptr, c->d_xstats, c->rank);
  c->launches += with_cols ? 4 : 3;
  return cudaGetLastError();
}


// FPFH + KM, settled loop: thresholds = penalty, one filter sweep, candidate block (see k_ff_gate_seed)
cudaError_t launch_fpfh_gate_seed(Ctx *c, const CostParams &cp, const LoopScalars &ls) {
  const FfArgs a = ff_args(c, cp);
  const int n = c->N > c->M ? c->N : c->M;
  GHICP_LAUNCH(k_ff_gate_seed, (n + 255) / 256, 256, 0, c->stream, a, ls, c->d_iter, c->d_ff_srec);
  c->launches++;
  return cudaGetLastError();
}
cudaError_t launch_fpfh_cand_block(Ctx *c, const CostParams &cp) {
  const FfArgs a = ff_args(c, cp);
  XBlockHdr *hdr = reinterpret_cast<XBlockHdr *>(c->d_xsend);
  unsigned long long *key = reinterpret_cast<unsigned long long *>(hdr + 1);
  double *gain = reinterpret_cast<double *>(key + c->xuse);
  float *fd = reinterpret_cast<float *>(gain + c->xuse);
  cudaMemsetAsync(hdr, 0, sizeof(XBlockHdr), c->stream);
  GHICP_LAUNCH(k_ff_stats, 1, 1024, 0, c->stream, c->d_ff_part, (int)fpfh_fast_parts(c), c->d_xstats, c->rank);
  GHICP_LAUNCH(k_ff_cand_block, GHICP_SMS * 2, 256, 0, c->stream, a, c->d_iter, hdr, key, gain, fd, (unsigned long long)c->xuse);
  GHICP_LAUNCH(k_ff_block_hdr, 1, 1, 0, c->stream, a, c->d_xstats + 4 * c->rank, hdr, (unsigned long long)c->xuse);
  c->launches += 3;
  return cudaGetLastError();
}

}  // namespace ghicp_b200
