// ghicp_kernels.cu — cost build, correspondence scans, pair statistics, rigid solve and update kernels
// of the GH-ICP inner loop for sm_90a.  Compiled with --fmad=false: every arithmetic operation on
// the exact path is a separately rounded IEEE operation, in the reference's evaluation order, so
// CD(i,j) is bit-identical to the reference's double arithmetic (src/ghicp_reg.cpp:122,259,308).
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdio>
#include <cooperative_groups.h>
#include <cuda_fp16.h>

#include "ghicp_internal.h"
#include "ghicp_device.cuh"

namespace ghicp_b200 {
namespace cg = cooperative_groups;

namespace {

constexpr int SWEEP_THREADS = 256;
constexpr int COLS_PER_THREAD = 4;


// ---------------------------------------------------------------------------------------------
// BSC packing:  raw [V][N][B] bytes → words [V][W64][N]  (word-major planes, coalesced per word)
// ---------------------------------------------------------------------------------------------
__global__ void k_pack_bsc(const uint8_t *__restrict__ raw, uint64_t *__restrict__ words, int V, int n, int B,
                           int W64) {
  long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long total = (long long)V * W64 * n;
  if (idx >= total) return;
  int i = (int)(idx % n);
  int w = (int)((idx / n) % W64);
  int v = (int)(idx / ((long long)n * W64));
  const uint8_t *p = raw + ((size_t)v * n + i) * B;
  uint64_t word = 0;
#pragma unroll
  for (int b = 0; b < 8; ++b) {
    int byte = w * 8 + b;
    if (byte < B) word |= (uint64_t)p[byte] << (8 * b);
  }
  words[idx] = word;
}

// ---------------------------------------------------------------------------------------------
// calFD_BSC (src/ghicp_reg.cpp:143-200): FD[i][j] = min_v popcount(bscS[v][i] ^ bscT[0][j]) → the packed plane (fd_at).
// CTA = 128 threads = 128 target columns x 32 source rows; source words staged in shared memory.
// ---------------------------------------------------------------------------------------------
constexpr int FDB_ROWS = 32;
constexpr int FDB_THREADS = 128;
template <int V>
__global__ void __launch_bounds__(FDB_THREADS) k_fd_bsc(const uint64_t *__restrict__ bs,
                                                         const uint64_t *__restrict__ bt,
                                                         unsigned char *__restrict__ fdq, int hb, int N, int M,
                                                         size_t ldM, int W64, int row0, int nloc) {
#if defined(GHICP_EMU_HOST)
  uint64_t *s_words = reinterpret_cast<uint64_t *>(emu::dyn_smem());  // host emulation: the launch's dynamic shared memory
#else
  extern __shared__ uint64_t s_words[];  // [V][W64][FDB_ROWS]
#endif
  const int i0 = row0 + blockIdx.y * FDB_ROWS;
  const int iend = row0 + nloc;
  const int j = blockIdx.x * FDB_THREADS + threadIdx.x;
  for (int k = threadIdx.x; k < V * W64 * FDB_ROWS; k += FDB_THREADS) {
    int r = k % FDB_ROWS;
    int vw = k / FDB_ROWS;  // v*W64 + w
    int i = i0 + r;
    s_words[k] = (i < iend) ? bs[(size_t)vw * N + i] : 0ull;
  }
  __syncthreads();
  // every lane stays to the end: the high-bit words of the packed plane are OR-reduced over the 8 lanes of a quad block's lane
  const bool live = j < M;
  const int jj = live ? j : M - 1;
  for (int rc = 0; rc < FDB_ROWS; rc += 8) {
    int acc[8][V];
#pragma unroll
    for (int r = 0; r < 8; ++r)
#pragma unroll
      for (int v = 0; v < V; ++v) acc[r][v] = 0;
    for (int w = 0; w < W64; ++w) {
      const uint64_t tw = bt[(size_t)w * M + jj];
#pragma unroll
      for (int v = 0; v < V; ++v) {
        const uint64_t *sw = &s_words[(v * W64 + w) * FDB_ROWS + rc];
#pragma unroll
        for (int r = 0; r < 8; ++r) acc[r][v] += __popcll(sw[r] ^ tw);
      }
    }
    // rows i0 + rc ... + 7 are two whole quads (i0 - row0 and rc are multiples of 4)
#pragma unroll
    for (int qd = 0; qd < 2; ++qd) {
      unsigned hw[4] = {0u, 0u, 0u, 0u};
#pragma unroll
      for (int u = 0; u < FD_QUAD; ++u) {
        const int r = FD_QUAD * qd + u, i = i0 + rc + r;
        int m = acc[r][0];
#pragma unroll
        for (int v = 1; v < V; ++v) m = min(m, acc[r][v]);
        if (!live || i >= iend) m = 0;
        else fdq[fd_block_offset(ldM, hb, i - row0, j) + u * FD_PANEL + (j & (FD_PANEL - 1))] = (unsigned char)m;
        const int c = j & 7, wd = fd_hi_word(hb, u, c);
        const unsigned part = fd_hi_part(hb, u, c, (unsigned)m);
#pragma unroll
        for (int w = 0; w < 4; ++w) hw[w] |= (w == wd) ? part : 0u;
      }
      const int iq = i0 + rc + FD_QUAD * qd;
      for (int w = 0; w < hb; ++w) {
        const unsigned word = fd_lanes_or<8>(hw[w]);   // a warp's 32 columns are four whole lanes of the panel
        if ((j & 7) == 0 && live && iq < iend)
          reinterpret_cast<unsigned *>(fdq + fd_block_offset(ldM, hb, iq - row0, j) + FD_LOW_BYTES)[w * 32 + ((j & (FD_PANEL - 1)) >> 3)] = word;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// calFD_FPFH (src/ghicp_reg.cpp:202-214, include/fpfh.hpp:135-165), float32, reference op order.
// Stage 1 (per point): mean (serial float sum / 33), centred histogram, serial sum of squares.
// Stage 2 (per pair): serial float dot of centred histograms, / sqrt(d1*d2), fabs.
// ---------------------------------------------------------------------------------------------
__global__ void k_fpfh_center(const float *__restrict__ h, float *__restrict__ hc /*[n][36]*/, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float *p = h + (size_t)i * 33;
  float mean = 0.f;
  for (int k = 0; k < 33; ++k) mean += p[k];
  mean /= 33;
  float d = 0.f;
  float *q = hc + (size_t)i * 36;
  for (int k = 0; k < 33; ++k) {
    float c = p[k] - mean;
    q[k] = c;
    d += c * c;
  }
  q[33] = d;
  q[34] = 0.f;
  q[35] = 0.f;
}

constexpr int FPT = 16;  // tile edge
__global__ void __launch_bounds__(FPT *FPT) k_fd_fpfh(const float *__restrict__ sc, const float *__restrict__ tc,
                                                       float *__restrict__ fd, int N, int M, size_t ldM, int row0,
                                                       int nloc) {
  __shared__ float s_s[FPT][37];
  __shared__ float s_t[FPT][37];
  const int tx = threadIdx.x % FPT, ty = threadIdx.x / FPT;
  const int i0 = row0 + blockIdx.y * FPT, j0 = blockIdx.x * FPT;
  N = row0 + nloc;  // rows of this shard end here
  for (int k = threadIdx.x; k < FPT * 36; k += FPT * FPT) {
    int r = k / 36, q = k % 36;
    s_s[r][q] = (i0 + r < N) ? sc[(size_t)(i0 + r) * 36 + q] : 0.f;
    s_t[r][q] = (j0 + r < M) ? tc[(size_t)(j0 + r) * 36 + q] : 0.f;
  }
  __syncthreads();
  const int i = i0 + ty, j = j0 + tx;
  if (i >= N || j >= M) return;
  float up = 0.f;
#pragma unroll
  for (int k = 0; k < 33; ++k) up += s_s[ty][k] * s_t[tx][k];
  float d = up / sqrtf(s_s[ty][33] * s_t[tx][33]);
  fd[fd_index(ldM, i - row0, j)] = fabsf(d);
}

// ---------------------------------------------------------------------------------------------
// Row sweep: one CTA owns TR source rows and a chunk of target columns.
//   MODE 0: per-row first-argmin of CD + sum(cd - pivot), sum((cd - pivot)^2)
//           (calED + calCD_* + the NN scan, src/ghicp_reg.cpp:114-139, 216-341, 715-733)
//   MODE 1: per-row count of CD < penalty                       (KM graph build, :358-365)
//   MODE 2: emit (j, penalty - CD) for CD < penalty into the CSR
// ---------------------------------------------------------------------------------------------
struct SweepArgs {
  const double *s;  // [3][N]
  const double *t;  // [3][M]
  const unsigned char *fdq;  // packed BSC plane (fd_at)
  int hb;
  const float *fdf;
  size_t ldM;
  int N, M, n_chunks, cols_per_chunk;
  int row0, nloc;  // source rows [row0, row0 + nloc) held by this context
  CostParams cp;
  // mode 0
  double *part_cd; int *part_idx; double *part_stats;
  // mode 1/2
  const DevIter *iter;  // penalty
  int *cnt;
  const long long *rowptr;
  int *cursor;
  int *csr_col; double *csr_gain; float *csr_fd;
};

template <int FT, int MODE>
__global__ void __launch_bounds__(SWEEP_THREADS) k_rowsweep(const SweepArgs a) {
  __shared__ double s_src[3][TR];
  __shared__ double s_red[2 * (SWEEP_THREADS / 32)];
  __shared__ double s_bv[TR][SWEEP_THREADS / 32];
  __shared__ int s_bi[TR][SWEEP_THREADS / 32];
  const int tid = threadIdx.x;
  const int i0 = a.row0 + blockIdx.x * TR;
  const int chunk = blockIdx.y;
  const int nrows = min(TR, a.row0 + a.nloc - i0);
  const int c0 = chunk * a.cols_per_chunk;
  const int c1 = min(a.M, c0 + a.cols_per_chunk);
  if (tid < 3 * TR) {
    int k = tid / TR, r = tid % TR;
    s_src[k][r] = (r < nrows) ? a.s[(size_t)k * a.N + i0 + r] : 0.0;
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
  for (int j = c0 + tid * COLS_PER_THREAD; j < c1; j += SWEEP_THREADS * COLS_PER_THREAD) {
    double cx[COLS_PER_THREAD], cy[COLS_PER_THREAD], cz[COLS_PER_THREAD];
#pragma unroll
    for (int c = 0; c < COLS_PER_THREAD; ++c) {
      int jj = min(j + c, a.M - 1);
      cx[c] = tx[jj]; cy[c] = ty[jj]; cz[c] = tz[jj];
    }
#pragma unroll
    for (int r = 0; r < TR; ++r) {
      if (r < nrows) {
        const double sx = s_src[0][r], sy = s_src[1][r], sz = s_src[2][r];
        double fdv[COLS_PER_THREAD];
        if (FT == GHICP_FT_BSC) {
#pragma unroll
          for (int c = 0; c < COLS_PER_THREAD; ++c) fdv[c] = (double)fd_at(a.fdq, a.ldM, a.hb, i0 + r - a.row0, j + c);
        } else if (FT == GHICP_FT_FPFH) {
          const float4 q = *reinterpret_cast<const float4 *>(a.fdf + fd_index(a.ldM, i0 + r - a.row0, j));
          fdv[0] = (double)q.x; fdv[1] = (double)q.y; fdv[2] = (double)q.z; fdv[3] = (double)q.w;
        } else {
          fdv[0] = fdv[1] = fdv[2] = fdv[3] = 0.0;
        }
#pragma unroll
        for (int c = 0; c < COLS_PER_THREAD; ++c) {
          if (j + c < c1) {
            const double ed = ed_exact(sx, sy, sz, cx[c], cy[c], cz[c], a.cp.scale);
            const double cd = cd_exact<FT>(ed, fdv[c], a.cp);
            if (MODE == 0) {
              if (cd < best[r]) { best[r] = cd; bidx[r] = j + c; }
              const double d = cd - a.cp.pivot;
              sum += d;
              sumsq += d * d;
            } else if (MODE == 1) {
              cnt[r] += (cd < penalty) ? 1 : 0;
            } else {
              if (cd < penalty) {
                const size_t slot = (size_t)(i0 + r) * a.n_chunks + chunk;
                const long long pos = a.rowptr[slot] + atomicAdd(&a.cursor[slot], 1);
                a.csr_col[pos] = j + c;
                a.csr_gain[pos] = penalty - cd;
                a.csr_fd[pos] = (float)fdv[c];
              }
            }
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
    double ws = warp_sum(sum), wq = warp_sum(sumsq);
    if (lane == 0) { s_red[warp] = ws; s_red[SWEEP_THREADS / 32 + warp] = wq; }
    __syncthreads();
    if (tid < nrows) {
      double v = s_bv[tid][0];
      int ix = s_bi[tid][0];
      for (int w = 1; w < SWEEP_THREADS / 32; ++w) lexmin(v, ix, s_bv[tid][w], s_bi[tid][w]);
      a.part_cd[(size_t)(i0 + tid) * a.n_chunks + chunk] = v;
      a.part_idx[(size_t)(i0 + tid) * a.n_chunks + chunk] = ix;
    }
    if (tid == 0) {
      double S1 = 0.0, S2 = 0.0;
      for (int w = 0; w < SWEEP_THREADS / 32; ++w) { S1 += s_red[w]; S2 += s_red[SWEEP_THREADS / 32 + w]; }
      const size_t b = (size_t)blockIdx.y * gridDim.x + blockIdx.x;
      a.part_stats[2 * b] = S1;
      a.part_stats[2 * b + 1] = S2;
    }
  } else if (MODE == 1) {
#pragma unroll
    for (int r = 0; r < TR; ++r) {
      int w = warp_sum_i(cnt[r]);
      if (lane == 0) s_bi[r][warp] = w;
    }
    __syncthreads();
    if (tid < nrows) {
      int tot = 0;
      for (int w = 0; w < SWEEP_THREADS / 32; ++w) tot += s_bi[tid][w];
      a.cnt[(size_t)(i0 + tid) * a.n_chunks + chunk] = tot;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Column sweep (NNR, src/ghicp_reg.cpp:637-650): per target column first-argmin over source rows.
// CTA = CT columns x a chunk of rows; thread per row, CT running minima in registers.
// ---------------------------------------------------------------------------------------------
constexpr int CT = 8;
constexpr int COL_THREADS = 256;
struct ColArgs {
  const double *s, *t;
  const unsigned char *fdq;  // packed BSC plane (fd_at)
  int hb;
  const float *fdf;
  size_t ldM;
  int N, M;
  int row0, nloc;
  CostParams cp;
  double *col_cd; int *col_idx;
};
template <int FT>
__global__ void __launch_bounds__(COL_THREADS) k_colsweep(const ColArgs a) {
  __shared__ double s_t[3][CT];
  __shared__ double s_bv[CT][COL_THREADS / 32];
  __shared__ int s_bi[CT][COL_THREADS / 32];
  const int tid = threadIdx.x;
  const int j0 = blockIdx.x * CT;
  const int ncols = min(CT, a.M - j0);
  if (tid < 3 * CT) {
    int k = tid / CT, c = tid % CT;
    s_t[k][c] = (c < ncols) ? a.t[(size_t)k * a.M + j0 + c] : 0.0;
  }
  __syncthreads();
  double best[CT];
  int bidx[CT];
#pragma unroll
  for (int c = 0; c < CT; ++c) { best[c] = MAXVALIUE; bidx[c] = 0; }
  const double *sxp = a.s, *syp = a.s + a.N, *szp = a.s + 2 * (size_t)a.N;
  for (int i = a.row0 + tid; i < a.row0 + a.nloc; i += COL_THREADS) {
    const double sx = sxp[i], sy = syp[i], sz = szp[i];
    double fdv[CT];
    if (FT == GHICP_FT_BSC) {
#pragma unroll
      for (int c = 0; c < CT; ++c) fdv[c] = (double)fd_at(a.fdq, a.ldM, a.hb, i - a.row0, j0 + c);
    } else if (FT == GHICP_FT_FPFH) {
      const float4 q0 = *reinterpret_cast<const float4 *>(a.fdf + fd_index(a.ldM, i - a.row0, j0));
      const float4 q1 = *reinterpret_cast<const float4 *>(a.fdf + fd_index(a.ldM, i - a.row0, j0 + 4));
      fdv[0] = q0.x; fdv[1] = q0.y; fdv[2] = q0.z; fdv[3] = q0.w;
      fdv[4] = q1.x; fdv[5] = q1.y; fdv[6] = q1.z; fdv[7] = q1.w;
    } else {
#pragma unroll
      for (int c = 0; c < CT; ++c) fdv[c] = 0.0;
    }
#pragma unroll
    for (int c = 0; c < CT; ++c) {
      if (c < ncols) {
        const double ed = ed_exact(sx, sy, sz, s_t[0][c], s_t[1][c], s_t[2][c], a.cp.scale);
        const double cd = cd_exact<FT>(ed, fdv[c], a.cp);
        if (cd < best[c]) { best[c] = cd; bidx[c] = i; }
      }
    }
  }
  const int lane = tid & 31, warp = tid >> 5;
#pragma unroll
  for (int c = 0; c < CT; ++c) {
    warp_lexmin(best[c], bidx[c]);
    if (lane == 0) { s_bv[c][warp] = best[c]; s_bi[c][warp] = bidx[c]; }
  }
  __syncthreads();
  if (tid < ncols) {
    double v = s_bv[tid][0];
    int ix = s_bi[tid][0];
    for (int w = 1; w < COL_THREADS / 32; ++w) lexmin(v, ix, s_bv[tid][w], s_bi[tid][w]);
    a.col_cd[j0 + tid] = v;
    a.col_idx[j0 + tid] = ix;
  }
}

// ---------------------------------------------------------------------------------------------
// Finalise: merge per-chunk row minima, reduce statistics in a fixed order, apply the penalty rule
// (src/ghicp_reg.cpp:228-239, 264-287, 317-335).  One CTA.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) k_finalize(const double *__restrict__ part_cd,
                                                   const int *__restrict__ part_idx, int n_chunks, int row0, int nloc,
                                                   const double *__restrict__ part_stats, int n_parts,
                                                   double *__restrict__ row_cd, int *__restrict__ row_idx,
                                                   float *__restrict__ row_fd, const unsigned char *__restrict__ fdq, int hb,
                                                   const float *__restrict__ fdf, size_t fd_rows,
                                                   double *__restrict__ xstats /* [world][2] */, int rank) {
  __shared__ double smem[2 * 32];
  for (int i = row0 + threadIdx.x; i < row0 + nloc; i += blockDim.x) {
    double v = part_cd[(size_t)i * n_chunks];
    int ix = part_idx[(size_t)i * n_chunks];
    for (int c = 1; c < n_chunks; ++c) lexmin(v, ix, part_cd[(size_t)i * n_chunks + c], part_idx[(size_t)i * n_chunks + c]);
    row_cd[i] = v;
    row_idx[i] = ix;
    row_fd[i] = fdq ? (float)fd_at(fdq, fd_rows, hb, i - row0, ix) : (fdf ? fdf[fd_index(fd_rows, i - row0, ix)] : 0.f);
  }
  double acc[2] = {0.0, 0.0};
  for (int p = threadIdx.x; p < n_parts; p += blockDim.x) {
    acc[0] += part_stats[2 * p];
    acc[1] += part_stats[2 * p + 1];
  }
  block_sum<2, 1024>(acc, smem);
  if (threadIdx.x == 0) {
    xstats[4 * rank] = acc[0];
    xstats[4 * rank + 1] = acc[1];
    xstats[4 * rank + 2] = 0.0;
  }
}

// CD mean / std over the whole N x M matrix from the per-rank partial sums (fixed rank order: every rank
// computes bit-identical values) and the penalty rule (src/ghicp_reg.cpp:228-239, 264-287, 317-335).
__global__ void k_penalty(const double *__restrict__ xstats, int world, double pivot, int N, int M, int feature_type,
                          LoopScalars ls, DevIter *iter) {
  double S1 = 0.0, S2 = 0.0;
  double ovf = 0.0;
  for (int r = 0; r < world; ++r) { S1 += xstats[4 * r]; S2 += xstats[4 * r + 1]; ovf += xstats[4 * r + 2]; }
  iter->overflow_any = ovf > 0.0 ? 1 : 0;
  const double n = (double)N * (double)M;
  const double CDmean = pivot + S1 / M / N;
  double var = (S2 - S1 * S1 / n) / n;
  if (var < 0.0) var = 0.0;
  const double CDstd = sqrt(var);
  double penalty;
  if (feature_type == GHICP_FT_BSC) {
    if (ls.iteration > 1)
      penalty = ls.RMS * ls.para1 * ls.scale * ls.WED + (ls.FDM + ls.para2 * ls.FDstd) * ls.WFD;
    else
      penalty = (CDmean - ls.penalty_initial * CDstd);
    penalty = fmax(penalty, 5.0);
  } else if (feature_type == GHICP_FT_FPFH) {
    if (ls.iteration > 1)
      penalty = ls.RMS * ls.para1 * ls.scale * ls.para2;
    else
      penalty = (CDmean / ls.penalty_initial);
  } else {
    penalty = fmax(CDmean, 1.0);
  }
  iter->cd_sum_shift = S1;
  iter->cd_sumsq_shift = S2;
  iter->cd_mean = CDmean;
  iter->cd_std = (feature_type == GHICP_FT_BSC) ? CDstd : 0.0;
  iter->penalty = penalty;
}

// ---------------------------------------------------------------------------------------------
// Tiled ordered scan / compaction: every CTA owns TILE consecutive items (4 per thread); a first kernel
// leaves one sum per tile, the second adds up the tiles before its own (a few dozen values) and scans
// inside the tile.  Two short launches instead of one CTA walking the whole array.
// ---------------------------------------------------------------------------------------------
constexpr int TILE_THREADS = 256, TILE_ITEMS = 4, TILE = TILE_THREADS * TILE_ITEMS;

__device__ __forceinline__ long long block_exclusive_scan_256(long long v, long long *smem /*[9]*/, long long *total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  long long x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    long long y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) smem[warp] = x;
  __syncthreads();
  if (threadIdx.x == 0) {
    long long run = 0;
    for (int w = 0; w < TILE_THREADS / 32; ++w) { const long long t = smem[w]; smem[w] = run; run += t; }
    smem[TILE_THREADS / 32] = run;
  }
  __syncthreads();
  const long long excl = smem[warp] + x - v;
  *total = smem[TILE_THREADS / 32];
  __syncthreads();
  return excl;
}
// sum of tile_sum[stride * b], b < nb (every thread gets it)
__device__ __forceinline__ long long tiles_before(const long long *tile_sum, int stride, int nb, long long *smem) {
  long long p = 0;
  for (int b = threadIdx.x; b < nb; b += TILE_THREADS) p += tile_sum[(size_t)stride * b];
  long long tot;
  block_exclusive_scan_256(p, smem, &tot);
  return tot;
}

__global__ void __launch_bounds__(TILE_THREADS) k_tile_sum_i32(const int *__restrict__ cnt, long long L,
                                                               long long *__restrict__ tile_sum) {
  __shared__ long long smem[TILE_THREADS / 32 + 1];
  const long long base = (long long)blockIdx.x * TILE + threadIdx.x * TILE_ITEMS;
  long long v = 0;
#pragma unroll
  for (int q = 0; q < TILE_ITEMS; ++q)
    if (base + q < L) v += cnt[base + q];
  long long tot;
  block_exclusive_scan_256(v, smem, &tot);
  if (threadIdx.x == 0) tile_sum[blockIdx.x] = tot;
}
// counts[L] → ptr[L+1] (exclusive), total → *total_out (optional); cursor zeroed.
__global__ void __launch_bounds__(TILE_THREADS) k_tile_scan_i32(const int *__restrict__ cnt, long long L,
                                                                const long long *__restrict__ tile_sum,
                                                                long long *__restrict__ ptr, int *__restrict__ cursor,
                                                                long long *total_out) {
  __shared__ long long smem[TILE_THREADS / 32 + 1];
  const long long pre = tiles_before(tile_sum, 1, blockIdx.x, smem);
  const long long base = (long long)blockIdx.x * TILE + threadIdx.x * TILE_ITEMS;
  int cq[TILE_ITEMS];
  long long v = 0;
#pragma unroll
  for (int q = 0; q < TILE_ITEMS; ++q) {
    cq[q] = (base + q < L) ? cnt[base + q] : 0;
    v += cq[q];
  }
  long long tot;
  long long off = pre + block_exclusive_scan_256(v, smem, &tot);
#pragma unroll
  for (int q = 0; q < TILE_ITEMS; ++q) {
    if (base + q < L) {
      ptr[base + q] = off;
      cursor[base + q] = 0;
      off += cq[q];
    }
  }
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) {
    ptr[L] = pre + tot;
    if (total_out) *total_out = pre + tot;
  }
}

// kind 0: NN   keep row i iff row_cd[i] < penalty          (src/ghicp_reg.cpp:725-730)
// kind 1: NNR  keep row i iff col_idx[row_idx[i]] == i     (src/ghicp_reg.cpp:652-662)
// kind 2: KM   keep column j iff owner[j] >= 0; pairs ordered by target index (src/km.cpp:157-167)
struct SelArgs {
  int kind, n, n_cols;
  const double *row_cd;
  const int *row_idx, *col_idx, *owner;
  int *sp, *tp;
  const float *row_fd;
  float *pair_fd;
  DevIter *iter;
  double amb_rel;
  long long *tile_sum;  // [2][tiles]: kept, ambiguous
};
__device__ __forceinline__ bool sel_keep(const SelArgs &a, int k, double penalty) {
  if (a.kind == 0) return a.row_cd[k] < penalty;
  if (a.kind == 1) { const int j = a.row_idx[k]; return (j >= 0 && j < a.n_cols) ? (a.col_idx[j] == k) : false; }
  return a.owner[k] >= 0;
}
__global__ void __launch_bounds__(TILE_THREADS) k_select_count(const SelArgs a) {
  __shared__ long long smem[TILE_THREADS / 32 + 1];
  const double penalty = a.iter->penalty;
  const double band = a.amb_rel * fmax(1.0, fabs(penalty));
  const int base = blockIdx.x * TILE + threadIdx.x * TILE_ITEMS;
  long long v = 0;  // kept | ambiguous << 32
#pragma unroll
  for (int q = 0; q < TILE_ITEMS; ++q) {
    const int k = base + q;
    if (k < a.n) {
      v += sel_keep(a, k, penalty) ? 1 : 0;
      if (a.kind == 0 && a.amb_rel > 0.0 && fabs(a.row_cd[k] - penalty) <= band) v += 1ll << 32;
    }
  }
  long long tot;
  block_exclusive_scan_256(v, smem, &tot);
  if (threadIdx.x == 0) {
    a.tile_sum[2 * blockIdx.x] = tot & 0xffffffffll;
    a.tile_sum[2 * blockIdx.x + 1] = tot >> 32;
  }
}
__global__ void __launch_bounds__(TILE_THREADS) k_select_write(const SelArgs a) {
  __shared__ long long smem[TILE_THREADS / 32 + 1];
  const double penalty = a.iter->penalty;
  const long long pre = tiles_before(a.tile_sum, 2, blockIdx.x, smem);
  const int base = blockIdx.x * TILE + threadIdx.x * TILE_ITEMS;
  bool kq[TILE_ITEMS];
  long long v = 0;
#pragma unroll
  for (int q = 0; q < TILE_ITEMS; ++q) {
    kq[q] = (base + q < a.n) ? sel_keep(a, base + q, penalty) : false;
    v += kq[q] ? 1 : 0;
  }
  long long tot;
  long long off = pre + block_exclusive_scan_256(v, smem, &tot);
#pragma unroll
  for (int q = 0; q < TILE_ITEMS; ++q) {
    const int k = base + q;
    if (kq[q]) {
      if (a.kind == 2) { a.sp[off] = a.owner[k]; a.tp[off] = k; }
      else { a.sp[off] = k; a.tp[off] = a.row_idx[k]; a.pair_fd[off] = a.row_fd[k]; }
      ++off;
    }
  }
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) a.iter->cor = (int)(pre + tot);
  if (blockIdx.x == 0) {
    const long long amb = tiles_before(a.tile_sum + 1, 2, gridDim.x, smem);
    if (threadIdx.x == 0) a.iter->ambiguous = (int)amb;
  }
}


// ---------------------------------------------------------------------------------------------
// Pair statistics + rigid solve, one CTA (the pair list is at most max(N,M) long):
//  pass 1  RMSE, FDM, centroids            (src/ghicp_reg.cpp:549-558)
//  pass 2  FDstd, cross-covariance         (src/ghicp_reg.cpp:559-565; Umeyama sigma)
//  solve   float32 SVD, R, t               (src/ghicp_reg.cpp:857-866)
//  pass 3  RMSE after the update           (src/ghicp_reg.cpp:895-904)
// Moments are accumulated in float64 and rounded once to float32 (the reference/PCL accumulates in
// float32; the difference is O(1e-7) relative and documented in DESIGN.md).
// ---------------------------------------------------------------------------------------------
struct SolveArgs {
  const double *s, *t;
  const float *pair_fd;  // FD of every pair (gathered by the selection step), or nullptr
  size_t ldM;
  int N, M, feature_type;
  const int *sp, *tp;
  const double *sxyz_pairs, *txyz_pairs;  // stand-alone rigid fit: explicit point lists (column-major n x 3)
  int n_explicit;
  CostParams cp;
  DevIter *iter;
  double *part;  // [3][SOLVE_GRID_MAX][SOLVE_K] per-CTA partial sums of the cooperative variant
};
// COOP = false: one CTA of 1024 threads (stand-alone rigid fit).  COOP = true: a cooperative grid of
// SOLVE_GRID_MAX x 256 threads for the loop — per-CTA partial sums, grid barrier, then EVERY CTA adds the
// partials in CTA order (fixed tree: deterministic, identical on every rank) and carries on redundantly.
constexpr int SOLVE_GRID_MAX = 64;
constexpr int SOLVE_K = 12;  // widest reduction (10) rounded up
template <int K, int THREADS, bool COOP>
__device__ __forceinline__ void solve_sum(double (&v)[K], double *smem, double *part, double *s_tot) {
  block_sum<K, THREADS>(v, smem);
  if (COOP) {
    if (threadIdx.x == 0) {
#pragma unroll
      for (int k = 0; k < K; ++k) part[blockIdx.x * SOLVE_K + k] = v[k];
      __threadfence();
    }
    cg::this_grid().sync();
    if (threadIdx.x < K) {
      double t = 0.0;
      for (int b = 0; b < (int)gridDim.x; ++b) t += __ldcg(&part[b * SOLVE_K + threadIdx.x]);
      s_tot[threadIdx.x] = t;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < K; ++k) v[k] = s_tot[k];
    __syncthreads();
  }
}
template <bool COOP>
__global__ void __launch_bounds__(COOP ? 256 : 1024) k_solve(const SolveArgs a) {
  constexpr int SOLVE_THREADS = COOP ? 256 : 1024;
  __shared__ double smem[SOLVE_K * (SOLVE_THREADS / 32)];
  __shared__ double s_b[16];
  __shared__ double s_tot[SOLVE_K];
  const bool lead = blockIdx.x == 0 && threadIdx.x == 0;  // the one thread that publishes results
  const int p0 = blockIdx.x * SOLVE_THREADS + threadIdx.x, pstep = gridDim.x * SOLVE_THREADS;
  const bool explicit_pts = a.sxyz_pairs != nullptr;
  const int cor = explicit_pts ? a.n_explicit : a.iter->cor;
  auto load = [&](int p, double &sx, double &sy, double &sz, double &tx, double &ty, double &tz, double &fd) {
    if (explicit_pts) {
      sx = a.sxyz_pairs[p]; sy = a.sxyz_pairs[(size_t)cor + p]; sz = a.sxyz_pairs[2 * (size_t)cor + p];
      tx = a.txyz_pairs[p]; ty = a.txyz_pairs[(size_t)cor + p]; tz = a.txyz_pairs[2 * (size_t)cor + p];
      fd = 0.0;
    } else {
      const int i = a.sp[p], j = a.tp[p];
      sx = a.s[i]; sy = a.s[(size_t)a.N + i]; sz = a.s[2 * (size_t)a.N + i];
      tx = a.t[j]; ty = a.t[(size_t)a.M + j]; tz = a.t[2 * (size_t)a.M + j];
      fd = (a.pair_fd && a.feature_type != GHICP_FT_NONE) ? (double)a.pair_fd[p] : 0.0;
    }
  };
  // pass 1
  double acc1[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int p = p0; p < cor; p += pstep) {
    double sx, sy, sz, tx, ty, tz, fd;
    load(p, sx, sy, sz, tx, ty, tz, fd);
    const double dx = sx - tx, dy = sy - ty, dz = sz - tz;
    const double d2 = (dx * dx + dy * dy) + dz * dz;
    acc1[0] += d2;
    acc1[1] += fd;
    acc1[2] += sx; acc1[3] += sy; acc1[4] += sz;
    acc1[5] += tx; acc1[6] += ty; acc1[7] += tz;
    // CD of the kept pair (for Km::Calenergy, src/km.cpp:128-141)
    const double ed = a.cp.scale * sqrt(d2);
    double cd;
    if (a.feature_type == GHICP_FT_BSC) cd = a.cp.WED * ed + a.cp.WFD * fd;
    else if (a.feature_type == GHICP_FT_FPFH) cd = 1.0 * ed / pow(fd, a.cp.ex);
    else cd = ed;
    acc1[8] += cd;
  }
  solve_sum<9, SOLVE_THREADS, COOP>(acc1, smem, a.part, s_tot);
  if (threadIdx.x == 0) {
    if (lead) a.iter->km_cd_sum = acc1[8];
    s_b[0] = acc1[0];               // sum of squared distances
    s_b[1] = acc1[1] / cor;         // FDM (NaN when cor == 0, as the reference)
    for (int k = 0; k < 6; ++k) s_b[2 + k] = acc1[2 + k] / cor;  // centroids
  }
  __syncthreads();
  const double FDM = s_b[1];
  const double mus[3] = {s_b[2], s_b[3], s_b[4]}, mud[3] = {s_b[5], s_b[6], s_b[7]};
  // pass 2
  double acc2[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int p = p0; p < cor; p += pstep) {
    double sx, sy, sz, tx, ty, tz, fd;
    load(p, sx, sy, sz, tx, ty, tz, fd);
    const double ds[3] = {sx - mus[0], sy - mus[1], sz - mus[2]};
    const double dd[3] = {tx - mud[0], ty - mud[1], tz - mud[2]};
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c) acc2[r * 3 + c] += dd[r] * ds[c];
    const double e = fd - FDM;
    acc2[9] += e * e;
  }
  solve_sum<10, SOLVE_THREADS, COOP>(acc2, smem, a.part + SOLVE_GRID_MAX * SOLVE_K, s_tot);
  __shared__ double s_Rt[16];
  if (threadIdx.x == 0) {
    DevIter *it = a.iter;
    double RMSE = s_b[0] / cor;
    if (lead) {
      it->rmse = sqrt(RMSE);
      it->fdm = FDM;
      it->fdstd = sqrt(acc2[9] / cor);
      it->solve_degenerate = (cor >= 3) ? 0 : 1;
    }
    double Rt[16];
    for (int i = 0; i < 16; ++i) Rt[i] = (i % 5 == 0) ? 1.0 : 0.0;
    if (cor >= 3) {
      float mu_s[3], mu_d[3], sigma[9];
      for (int k = 0; k < 3; ++k) { mu_s[k] = (float)mus[k]; mu_d[k] = (float)mud[k]; }
      for (int k = 0; k < 9; ++k) sigma[k] = (float)(acc2[k] / cor);
      umeyama_from_moments_f32(mu_s, mu_d, sigma, Rt);
    }
    for (int i = 0; i < 16; ++i) { if (lead) it->Rt[i] = Rt[i]; s_Rt[i] = Rt[i]; }
  }
  __syncthreads();
  // pass 3: RMSE after the update; R*v evaluated as ((R0*x + R1*y) + R2*z) + t like Eigen
  double acc3[1] = {0};
  {
    const double R00 = s_Rt[0], R10 = s_Rt[1], R20 = s_Rt[2], R01 = s_Rt[4], R11 = s_Rt[5], R21 = s_Rt[6],
                 R02 = s_Rt[8], R12 = s_Rt[9], R22 = s_Rt[10], t0 = s_Rt[12], t1 = s_Rt[13], t2 = s_Rt[14];
    for (int p = p0; p < cor; p += pstep) {
      double sx, sy, sz, tx, ty, tz, fd;
      load(p, sx, sy, sz, tx, ty, tz, fd);
      const double nx = ((R00 * sx + R01 * sy) + R02 * sz) + t0;
      const double ny = ((R10 * sx + R11 * sy) + R12 * sz) + t1;
      const double nz = ((R20 * sx + R21 * sy) + R22 * sz) + t2;
      const double dx = nx - tx, dy = ny - ty, dz = nz - tz;
      acc3[0] += (dx * dx + dy * dy) + dz * dz;
    }
  }
  solve_sum<1, SOLVE_THREADS, COOP>(acc3, smem, a.part + 2 * SOLVE_GRID_MAX * SOLVE_K, s_tot);
  if (lead) a.iter->rmse_after = sqrt(acc3[0] / cor);
}

// KP.kpSXYZ.row(i) = (R * row^T + t)^T for ALL source keypoints (src/ghicp_reg.cpp:891-894)
__global__ void k_apply(double *__restrict__ s, int N, const DevIter *__restrict__ iter, int guard_overflow) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  if (guard_overflow && iter->overflow_any) return;   // settled KM iteration whose candidate block overflowed: redone by the host
  const double *Rt = iter->Rt;
  const double x = s[i], y = s[(size_t)N + i], z = s[2 * (size_t)N + i];
  s[i] = ((Rt[0] * x + Rt[4] * y) + Rt[8] * z) + Rt[12];
  s[(size_t)N + i] = ((Rt[1] * x + Rt[5] * y) + Rt[9] * z) + Rt[13];
  s[2 * (size_t)N + i] = ((Rt[2] * x + Rt[6] * y) + Rt[10] * z) + Rt[14];
}

__global__ void k_fd_to_double(const unsigned char *__restrict__ fdq, int hb, const float *__restrict__ fdf, size_t ldM,
                               int N, int M, int row0, int nloc, double *__restrict__ out) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)N * M) return;
  const int i = (int)(idx / M), j = (int)(idx % M);
  if (i < row0 || i >= row0 + nloc) { out[idx] = 0.0; return; }  // rows held by another rank
  out[idx] = fdq ? (double)fd_at(fdq, ldM, hb, i - row0, j) : (fdf ? (double)fdf[fd_index(ldM, i - row0, j)] : 0.0);
}

// KM: FD of every kept pair, looked up in the candidate CSR (every rank holds the full CSR, not the full plane)
__global__ void k_pair_fd_km(const int *__restrict__ sp, const int *__restrict__ tp, const DevIter *iter,
                             const long long *__restrict__ rowptr, const int *__restrict__ csr_col,
                             const float *__restrict__ csr_fd, float *__restrict__ pair_fd) {
  const int lane = threadIdx.x & 31;
  const int warps = (gridDim.x * blockDim.x) >> 5;
  const int cor = iter->cor;
  for (int p = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; p < cor; p += warps) {
    const int i = sp[p], j = tp[p];
    const long long b = rowptr[i], e = rowptr[i + 1];
    for (long long k = b + lane; k < e; k += 32)
      if (csr_col[k] == j) pair_fd[p] = csr_fd[k];
  }
}

// the same with ONE THREAD per pair: a settled loop has about one candidate per row, a warp per pair wastes 31 lanes
__global__ void k_pair_fd_km_thread(const int *__restrict__ sp, const int *__restrict__ tp, const DevIter *iter,
                                    const long long *__restrict__ rowptr, const int *__restrict__ csr_col,
                                    const float *__restrict__ csr_fd, float *__restrict__ pair_fd) {
  const int cor = iter->cor;
  for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < cor; p += gridDim.x * blockDim.x) {
    const int i = sp[p], j = tp[p];
    for (long long k = rowptr[i], e = rowptr[i + 1]; k < e; ++k)
      if (csr_col[k] == j) { pair_fd[p] = csr_fd[k]; break; }
  }
}

template <typename F>
cudaError_t dispatch_ft(int ft, F &&f) {
  switch (ft) {
    case GHICP_FT_BSC: return f(std::integral_constant<int, GHICP_FT_BSC>());
    case GHICP_FT_FPFH: return f(std::integral_constant<int, GHICP_FT_FPFH>());
    default: return f(std::integral_constant<int, GHICP_FT_NONE>());
  }
}

}  // namespace

// =============================================================================================
// launchers
// =============================================================================================
cudaError_t launch_pack_bsc(Ctx *c, const uint8_t *d_raw_s, const uint8_t *d_raw_t) {
  {
    long long total = (long long)c->V * c->W64 * c->N;
    GHICP_LAUNCH(k_pack_bsc, (unsigned)((total + 255) / 256), 256, 0, c->stream, d_raw_s, c->d_bs, c->V, c->N, c->Bbytes, c->W64);
    c->launches++;
  }
  {
    long long total = (long long)c->W64 * c->M;
    GHICP_LAUNCH(k_pack_bsc, (unsigned)((total + 255) / 256), 256, 0, c->stream, d_raw_t, c->d_bt, 1, c->M, c->Bbytes, c->W64);
    c->launches++;
  }
  return cudaGetLastError();
}

cudaError_t launch_fd_bsc(Ctx *c) {
  const int V = (c->cfg.dof == 6) ? 4 : 2;  // src/ghicp_reg.cpp:178-182
  dim3 grid((c->M + FDB_THREADS - 1) / FDB_THREADS, (c->nloc + FDB_ROWS - 1) / FDB_ROWS);
  size_t smem = (size_t)V * c->W64 * FDB_ROWS * sizeof(uint64_t);
  if (V == 4)
    GHICP_LAUNCH(k_fd_bsc<4>, grid, FDB_THREADS, smem, c->stream, c->d_bs, c->d_bt, reinterpret_cast<unsigned char *>(c->d_fd16), fd_hb(c->bits),
                 c->N, c->M, c->fd_rows, c->W64, c->r0, c->nloc);
  else
    GHICP_LAUNCH(k_fd_bsc<2>, grid, FDB_THREADS, smem, c->stream, c->d_bs, c->d_bt, reinterpret_cast<unsigned char *>(c->d_fd16), fd_hb(c->bits),
                 c->N, c->M, c->fd_rows, c->W64, c->r0, c->nloc);
  c->launches++;
  return cudaGetLastError();
}

cudaError_t launch_fd_fpfh(Ctx *c) {
  DevBuf<float> sc, tc;
  CUDA_TRY(sc.alloc((size_t)c->N * 36, c->stream));
  CUDA_TRY(tc.alloc((size_t)c->M * 36, c->stream));
  GHICP_LAUNCH(k_fpfh_center, (c->N + 127) / 128, 128, 0, c->stream, c->d_fs, sc.get(), c->N);
  GHICP_LAUNCH(k_fpfh_center, (c->M + 127) / 128, 128, 0, c->stream, c->d_ft, tc.get(), c->M);
  dim3 grid((c->M + FPT - 1) / FPT, (c->nloc + FPT - 1) / FPT);
  GHICP_LAUNCH(k_fd_fpfh, grid, FPT * FPT, 0, c->stream, sc.get(), tc.get(), c->d_fdf, c->N, c->M, c->fd_rows, c->r0, c->nloc);
  c->launches += 3;
  return cudaGetLastError();
}

cudaError_t launch_rowsweep(Ctx *c, int mode, const CostParams &cp) {
  SweepArgs a{};
  a.s = c->d_s; a.t = c->d_t; a.fdq = reinterpret_cast<const unsigned char *>(c->d_fd16); a.hb = fd_hb(c->bits); a.fdf = c->d_fdf; a.ldM = c->fd_rows;
  a.N = c->N; a.M = c->M; a.n_chunks = c->n_chunks;
  a.row0 = c->r0; a.nloc = c->nloc;
  int cpc = (c->M + c->n_chunks - 1) / c->n_chunks;
  cpc = (cpc + COLS_PER_THREAD - 1) / COLS_PER_THREAD * COLS_PER_THREAD;
  a.cols_per_chunk = cpc;
  a.cp = cp;
  a.part_cd = c->d_part_cd; a.part_idx = c->d_part_idx; a.part_stats = c->d_part_stats;
  a.iter = c->d_iter; a.cnt = c->d_cnt; a.rowptr = c->d_rowptr; a.cursor = c->d_cursor;
  a.csr_col = c->d_csr_col; a.csr_gain = c->d_csr_gain; a.csr_fd = c->d_csr_fd;
  dim3 grid((c->nloc + TR - 1) / TR, c->n_chunks);
  cudaError_t e = dispatch_ft(c->cfg.feature_type, [&](auto ft) {
    constexpr int FT = decltype(ft)::value;
    void (*kern)(const SweepArgs) = mode == SWEEP_ROWMIN ? k_rowsweep<FT, SWEEP_ROWMIN>
                                    : (mode == SWEEP_COUNT ? k_rowsweep<FT, SWEEP_COUNT> : k_rowsweep<FT, SWEEP_FILL>);
    GHICP_LAUNCH(kern, grid, SWEEP_THREADS, 0, c->stream, a);
    return cudaGetLastError();
  });
  c->launches++;
  return e;
}

cudaError_t launch_colsweep(Ctx *c, const CostParams &cp) {
  ColArgs a{};
  a.s = c->d_s; a.t = c->d_t; a.fdq = reinterpret_cast<const unsigned char *>(c->d_fd16); a.hb = fd_hb(c->bits); a.fdf = c->d_fdf; a.ldM = c->fd_rows;
  a.N = c->N; a.M = c->M; a.row0 = c->r0; a.nloc = c->nloc; a.cp = cp; a.col_cd = c->d_col_cd; a.col_idx = c->d_col_idx;
  dim3 grid((c->M + CT - 1) / CT);
  cudaError_t e = dispatch_ft(c->cfg.feature_type, [&](auto ft) {
    constexpr int FT = decltype(ft)::value;
    void (*kern)(const ColArgs) = k_colsweep<FT>;
    GHICP_LAUNCH(kern, grid, COL_THREADS, 0, c->stream, a);
    return cudaGetLastError();
  });
  c->launches++;
  return e;
}

cudaError_t launch_finalize_stats(Ctx *c, const CostParams &cp, const LoopScalars &ls) {
  (void)cp; (void)ls;
  const int n_parts = ((c->nloc + TR - 1) / TR) * c->n_chunks;
  GHICP_LAUNCH(k_finalize, 1, 1024, 0, c->stream, c->d_part_cd, c->d_part_idx, c->n_chunks, c->r0, c->nloc, c->d_part_stats,
                                        n_parts, c->d_row_cd, c->d_row_idx, c->d_row_fd, reinterpret_cast<const unsigned char *>(c->d_fd16), fd_hb(c->bits), c->d_fdf,
                                        c->fd_rows, c->d_xstats, c->rank);
  c->launches++;
  return cudaGetLastError();
}

cudaError_t launch_penalty(Ctx *c, double pivot, const LoopScalars &ls) {
  GHICP_LAUNCH(k_penalty, 1, 1, 0, c->stream, c->d_xstats, c->world, pivot, c->N, c->M, c->cfg.feature_type, ls, c->d_iter);
  c->launches++;
  return cudaGetLastError();
}
cudaError_t launch_pair_fd_km(Ctx *c) {
  const long long nmax = std::max(c->N, c->M);
  if (c->last_total_nnz >= 0 && c->last_total_nnz <= 4 * nmax) {   // short rows (hint: last iteration's edge count)
    GHICP_LAUNCH(k_pair_fd_km_thread, (unsigned)((nmax + 255) / 256), 256, 0, c->stream, c->d_sp, c->d_tp, c->d_iter, c->d_rowptr,
                 c->d_csr_col, c->d_csr_fd, c->d_pair_fd);
    c->launches++;
    return cudaGetLastError();
  }
  GHICP_LAUNCH(k_pair_fd_km, GHICP_SMS * 2, 256, 0, c->stream, c->d_sp, c->d_tp, c->d_iter, c->d_rowptr, c->d_csr_col, c->d_csr_fd,
                                               c->d_pair_fd);
  c->launches++;
  return cudaGetLastError();
}

cudaError_t launch_scan_i32(Ctx *c, const int *cnt, long long *ptr, int *cursor, long long L, long long *total_out) {
  const int tiles = (int)std::max<long long>(1, (L + TILE - 1) / TILE);
  if ((size_t)tiles > c->tile_cap) return cudaErrorInvalidValue;
  GHICP_LAUNCH(k_tile_sum_i32, tiles, TILE_THREADS, 0, c->stream, cnt, L, c->d_tile_sum);
  GHICP_LAUNCH(k_tile_scan_i32, tiles, TILE_THREADS, 0, c->stream, cnt, L, c->d_tile_sum, ptr, cursor, total_out);
  c->launches += 2;
  return cudaGetLastError();
}
cudaError_t launch_scan_counts(Ctx *c) {
  return launch_scan_i32(c, c->d_cnt, c->d_rowptr, c->d_cursor, (long long)c->N * c->n_chunks, &c->d_iter->nnz);
}

static cudaError_t launch_select(Ctx *c, SelArgs a) {
  const int tiles = std::max(1, (a.n + TILE - 1) / TILE);
  if ((size_t)tiles * 2 > c->tile_cap) return cudaErrorInvalidValue;
  a.iter = c->d_iter; a.sp = c->d_sp; a.tp = c->d_tp; a.tile_sum = c->d_tile_sum;
  GHICP_LAUNCH(k_select_count, tiles, TILE_THREADS, 0, c->stream, a);
  GHICP_LAUNCH(k_select_write, tiles, TILE_THREADS, 0, c->stream, a);
  c->launches += 2;
  return cudaGetLastError();
}
cudaError_t launch_select_nn(Ctx *c, double amb_rel) {
  SelArgs a{};
  a.kind = 0; a.n = c->N; a.n_cols = c->M; a.row_cd = c->d_row_cd; a.row_idx = c->d_row_idx;
  a.row_fd = c->d_row_fd; a.pair_fd = c->d_pair_fd; a.amb_rel = amb_rel;
  return launch_select(c, a);
}
cudaError_t launch_select_nnr(Ctx *c) {
  SelArgs a{};
  a.kind = 1; a.n = c->N; a.n_cols = c->M; a.row_cd = c->d_row_cd; a.row_idx = c->d_row_idx; a.col_idx = c->d_col_idx;
  a.row_fd = c->d_row_fd; a.pair_fd = c->d_pair_fd;
  return launch_select(c, a);
}
cudaError_t launch_select_km(Ctx *c) {
  SelArgs a{};
  a.kind = 2; a.n = c->M; a.n_cols = c->M; a.owner = c->d_owner;
  return launch_select(c, a);
}

cudaError_t launch_solve(Ctx *c, const CostParams &cp) {
  SolveArgs a{};
  a.cp = cp;
  a.s = c->d_s; a.t = c->d_t; a.pair_fd = c->d_pair_fd; a.ldM = c->fd_rows;
  a.N = c->N; a.M = c->M; a.feature_type = c->cfg.feature_type;
  a.sp = c->d_sp; a.tp = c->d_tp; a.sxyz_pairs = nullptr; a.txyz_pairs = nullptr; a.n_explicit = 0;
  a.iter = c->d_iter;
  a.part = c->d_solve_part;
  const int nmax = std::max(c->N, c->M);
  const int grid = std::min(SOLVE_GRID_MAX, std::max(1, (nmax + 1023) / 1024));
  void *args[] = {(void *)&a};
#if defined(GHICP_EMU_HOST)
  (void)args;   // host emulation: one block only (its grid barrier is then a block barrier), see tests/harness/cuda_emu
  void (*kern)(const SolveArgs) = k_solve<true>;
  GHICP_LAUNCH(kern, 1, 256, 0, c->stream, a);
  cudaError_t e = cudaSuccess;
#else
  cudaError_t e = cudaLaunchCooperativeKernel((void *)k_solve<true>, dim3(grid), dim3(256), args, 0, c->stream);
#endif
  c->launches++;
  return e != cudaSuccess ? e : cudaGetLastError();
}

cudaError_t launch_solve_explicit(cudaStream_t stream, const double *d_s, const double *d_t, int n, DevIter *d_iter) {
  SolveArgs a{};
  a.sxyz_pairs = d_s; a.txyz_pairs = d_t; a.n_explicit = n; a.iter = d_iter;
  a.feature_type = GHICP_FT_NONE;
  void (*kern)(const SolveArgs) = k_solve<false>;
  GHICP_LAUNCH(kern, 1, 1024, 0, stream, a);
  return cudaGetLastError();
}

cudaError_t launch_apply(Ctx *c, bool guard_overflow) {
  GHICP_LAUNCH(k_apply, (c->N + 255) / 256, 256, 0, c->stream, c->d_s, c->N, c->d_iter, guard_overflow ? 1 : 0);
  c->launches++;
  return cudaGetLastError();
}

cudaError_t launch_get_fd(Ctx *c, double *d_out) {
  const size_t total = (size_t)c->N * c->M;
  GHICP_LAUNCH(k_fd_to_double, (unsigned)((total + 255) / 256), 256, 0, c->stream, reinterpret_cast<const unsigned char *>(c->d_fd16), fd_hb(c->bits), c->d_fdf, c->fd_rows, c->N, c->M, c->r0, c->nloc, d_out);
  c->launches++;
  return cudaGetLastError();
}

}  // namespace ghicp_b200
