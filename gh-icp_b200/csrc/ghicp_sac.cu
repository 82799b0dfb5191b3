// ghicp_sac.cu — SAC-IA coarse alignment from FPFH histograms on the GPU: the reference's FPFHfeature::fpfhalign
// (include/fpfh.hpp:117-133, PCL SampleConsensusInitialAlignment with correspondence randomness 6) and
// CRegistration::Coarsereg_FPFHSAC (src/common_reg.cpp:393-423, randomness 15), on the canonical definition of DESIGN.md §3.11.
// Hypotheses are independent, so every stage runs all of them at once:
//   k_sac_sample     one thread per hypothesis: nr_samples distinct source indices (counter-based draws, ghicp_sac.h)
//   k_sac_compact    the distinct sampled indices -> a list (the only queries of the feature k-NN)
//   k_sac_feat_knn   one thread per listed index: the k nearest target histograms, target streamed through shared memory,
//                    top-k in registers as sorted (d2, index) keys (the k_knn idiom)
//   k_sac_estimate   one thread per hypothesis: the correspondence picks, FP64 moments, the hot path's float32 Umeyama
//   k_sac_score      the hot path: a CTA per (block of hypotheses, chunk of source points in shared memory), one exact
//                    nearest-neighbour query per (hypothesis, point) against the target's cell grid (ghicp_grid.cuh: the
//                    grid and ring_walk of k_knn with k = 1, stopped once the ring bound passes min(best, sqrt(thr))), the
//                    truncated error of each point as a 2^-32 fixed-point integer, warp-reduced, one 64-bit atomic per CTA
//                    and hypothesis: the sums are exact in any order
//   k_sac_pick       smallest (error, h) over the valid hypotheses
//   k_sac_fit        the chosen transform once more, per point, for the inlier count and the fitness (summed on the host in
//                    point order)
#include <algorithm>
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstring>
#include <vector>

#include "ghicp_internal.h"
#include "ghicp_device.cuh"
#include "ghicp_grid.cuh"
#include "ghicp_ovwalk.cuh"
#include "ghicp_sac.h"

namespace ghicp_b200 {
namespace {

using ghicp_sac::SAC_KMAX;
using ghicp_sac::SAC_MAX_SAMPLES;

constexpr int SAC_T = 128;        // threads per CTA of the per-hypothesis and per-point kernels
constexpr int FEAT_T = 64;        // queries per CTA of the feature k-NN (few queries: small CTAs spread over more SMs)
constexpr int FEAT_TILE = 64;     // target histograms per shared-memory tile
constexpr int SCORE_T = 256;      // threads per scoring CTA
constexpr int SCORE_HB = 4;       // hypotheses per scoring CTA
constexpr int SCORE_CHUNK = 1024; // source points per scoring CTA
constexpr int PICK_T = 1024;

struct SacArgs {
  const float *P, *Fs; int ns;        // source points [ns][3], histograms [ns][33]
  const float *Fq; int nt;            // target histograms [nt][33]
  int H, nsamp, ke;                   // hypotheses, samples per hypothesis, k_eff = min(k, nt)
  float msd, thr;                     // min_sample_distance, corr_dist_threshold (squared distances)
  unsigned long long seed;
  int *samp;                          // [H][nsamp] (-1 for an invalid hypothesis)
  int *valid;                         // [H]
  unsigned *dnext;                    // [H] draw number after the sample draws
  int *need, *slot;                   // [ns] sampled flag, position in the list
  int *list, *nlist;                  // distinct sampled indices (any order), their count
  int *knn;                           // [list][ke] target indices, ascending (d2, index)
  int *corr;                          // [H][nsamp]
  float *rt;                          // [H][12]: R row-major, then t
  unsigned long long *err;            // [H] fixed-point error sums
};

__global__ void k_sac_sample(const SacArgs a) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  if (h >= a.H) return;
  int s[SAC_MAX_SAMPLES];
  int n = 0, rej = 0;
  unsigned d = 0;
  bool ok = true;
  while (n < a.nsamp) {
    const int c = ghicp_sac::sac_index(ghicp_sac::sac_draw(a.seed, (unsigned)h, d++), a.ns);
    bool acc = true;
    for (int j = 0; j < n && acc; ++j)
      acc = s[j] != c && ghicp_sac::sac_sample_dist(a.P + 3 * (size_t)c, a.P + 3 * (size_t)s[j]) >= a.msd;
    if (acc) { s[n++] = c; rej = 0; }
    else if (++rej >= 3 * a.ns) { ok = false; break; }
  }
  for (int j = 0; j < a.nsamp; ++j) {
    const int v = ok ? s[j] : -1;
    a.samp[(size_t)h * a.nsamp + j] = v;
    if (ok) a.need[v] = 1;
  }
  a.valid[h] = ok ? 1 : 0;
  a.dnext[h] = d;
}

__global__ void k_sac_compact(const SacArgs a) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.ns || !a.need[i]) return;
  const int p = atomicAdd(a.nlist, 1);   // list order is irrelevant: each entry's neighbours depend on the index only
  a.list[p] = i;
  a.slot[i] = p;
}

__global__ void __launch_bounds__(FEAT_T) k_sac_feat_knn(const SacArgs a) {
  __shared__ float tile[FEAT_TILE * 33];
  const int nl = *a.nlist;
  if ((int)(blockIdx.x * FEAT_T) >= nl) return;   // the whole CTA
  const int q = blockIdx.x * FEAT_T + threadIdx.x;
  const bool active = q < nl;
  float f[33];
  const float *fs = a.Fs + 33 * (size_t)(active ? a.list[q] : 0);
#pragma unroll
  for (int b = 0; b < 33; ++b) f[b] = fs[b];
  pu64 key[SAC_KMAX];
#pragma unroll
  for (int j = 0; j < SAC_KMAX; ++j) key[j] = (j < SAC_KMAX - a.ke) ? 0ull : ~0ull;
  for (int t0 = 0; t0 < a.nt; t0 += FEAT_TILE) {
    const int cnt = min(FEAT_TILE, a.nt - t0);
    __syncthreads();
    for (int e = threadIdx.x; e < cnt * 33; e += FEAT_T) tile[e] = a.Fq[33 * (size_t)t0 + e];
    __syncthreads();
    if (active)
      for (int j = 0; j < cnt; ++j) knn_insert(key, knn_key(ghicp_sac::sac_feat_d2(f, tile + 33 * j), t0 + j));
  }
  if (!active) return;
#pragma unroll
  for (int j = 0; j < SAC_KMAX; ++j) {
    const int jj = j - (SAC_KMAX - a.ke);
    if (jj >= 0) a.knn[(size_t)q * a.ke + jj] = (int)(unsigned)key[j];
  }
}

// FP64 moments of the nr_samples pairs (the oracle's rigid fit with solve_mode 1), then the float32 Umeyama of the hot path
__global__ void k_sac_estimate(const SacArgs a, const float *__restrict__ Q) {
  const int h = blockIdx.x * blockDim.x + threadIdx.x;
  if (h >= a.H || !a.valid[h]) return;
  unsigned d = a.dnext[h];
  const int ns = a.nsamp;
  double ms[3] = {0, 0, 0}, md[3] = {0, 0, 0};
  for (int j = 0; j < ns; ++j) {
    const int s = a.samp[(size_t)h * ns + j];
    const unsigned long long r = ghicp_sac::sac_draw(a.seed, (unsigned)h, d++);
    const int c = a.knn[(size_t)a.slot[s] * a.ke + (int)(r % (unsigned long long)a.ke)];
    a.corr[(size_t)h * ns + j] = c;
    for (int k = 0; k < 3; ++k) { ms[k] += (double)a.P[3 * (size_t)s + k]; md[k] += (double)Q[3 * (size_t)c + k]; }
  }
  double mus[3], mud[3];
  for (int k = 0; k < 3; ++k) { mus[k] = ms[k] / ns; mud[k] = md[k] / ns; }
  double acc[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int j = 0; j < ns; ++j) {
    const int s = a.samp[(size_t)h * ns + j], c = a.corr[(size_t)h * ns + j];
    double ds[3], dd[3];
    for (int k = 0; k < 3; ++k) { ds[k] = (double)a.P[3 * (size_t)s + k] - mus[k]; dd[k] = (double)Q[3 * (size_t)c + k] - mud[k]; }
    for (int r = 0; r < 3; ++r)
      for (int cc = 0; cc < 3; ++cc) acc[r * 3 + cc] += dd[r] * ds[cc];
  }
  float mu_s[3], mu_d[3], sigma[9];
  for (int k = 0; k < 3; ++k) { mu_s[k] = (float)mus[k]; mu_d[k] = (float)mud[k]; }
  for (int k = 0; k < 9; ++k) sigma[k] = (float)(acc[k] / ns);
  double Rt[16];
  umeyama_from_moments_f32(mu_s, mu_d, sigma, Rt);
  float *o = a.rt + 12 * (size_t)h;
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) o[3 * i + j] = (float)Rt[j * 4 + i];
    o[9 + i] = (float)Rt[12 + i];
  }
}

// query cell coordinate, clamped into the grid (a query outside the box searches from the nearest boundary cell; the ring
// bound below still holds, since the query lies beyond that cell)
__device__ __forceinline__ int sac_cell(float v, float mn, float inv, int gmax) {
  const float f = floorf((v - mn) * inv);
  return !(f > 0.f) ? 0 : (f > (float)gmax ? gmax : (int)f);
}
// squared distance to the nearest target point when it is <= thr; otherwise some value > thr (the error term is 1 either way)
__device__ float sac_nn_d2(const GridRegs &r, const RingGrid &G, float qx, float qy, float qz, float thr) {
  {  // outside the box by more than sqrt(thr): no point can be within the threshold
    const double ex = qx < G.g.mnx ? (double)G.g.mnx - qx : (qx > G.mx[0] ? (double)qx - G.mx[0] : 0.0);
    const double ey = qy < G.g.mny ? (double)G.g.mny - qy : (qy > G.mx[1] ? (double)qy - G.mx[1] : 0.0);
    const double ez = qz < G.g.mnz ? (double)G.g.mnz - qz : (qz > G.mx[2] ? (double)qz - G.mx[2] : 0.0);
    if ((ex * ex + ey * ey) + ez * ez > (double)thr * (1.0 + 1e-5)) return INFINITY;
  }
  const int cx = sac_cell(qx, G.g.mnx, G.g.inv, G.gm[0]), cy = sac_cell(qy, G.g.mny, G.g.inv, G.gm[1]), cz = sac_cell(qz, G.g.mnz, G.g.inv, G.gm[2]);
  float best = INFINITY;
  ring_walk(r, G, cx, cy, cz, INT_MAX,   // no cap: the walk settles by the last ring at the latest
      [&](int s0, int s1) {
        for (int s = s0; s < s1; ++s) {
          const float d2 = knn_d2(qx, qy, qz, r.sorted[s]);
          best = d2 < best ? d2 : best;
        }
      },
      [&] { return best < thr ? (double)best : (double)thr; });
  return best;
}

__global__ void __launch_bounds__(SCORE_T) k_sac_score(const SacArgs a, const RingGrid G) {
  __shared__ float s_p[SCORE_CHUNK * 3];
  __shared__ float s_rt[SCORE_HB * 12];
  __shared__ int s_ok[SCORE_HB];
  __shared__ unsigned long long s_red[SCORE_HB][SCORE_T / 32];
  const int h0 = blockIdx.x * SCORE_HB, p0 = blockIdx.y * SCORE_CHUNK;
  const int cnt = min(SCORE_CHUNK, a.ns - p0);
  for (int e = threadIdx.x; e < cnt * 3; e += SCORE_T) s_p[e] = a.P[3 * (size_t)p0 + e];
  if (threadIdx.x < SCORE_HB) s_ok[threadIdx.x] = (h0 + (int)threadIdx.x < a.H) ? a.valid[h0 + threadIdx.x] : 0;
  for (int e = threadIdx.x; e < SCORE_HB * 12; e += SCORE_T) s_rt[e] = (h0 + e / 12 < a.H) ? a.rt[12 * (size_t)h0 + e] : 0.f;
  __syncthreads();
  const GridRegs r = grid_regs(G.g);   // per-thread registers, see k_pca
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int hb = 0; hb < SCORE_HB; ++hb) {
    if (!s_ok[hb]) continue;           // uniform over the CTA
    unsigned long long acc = 0ull;
    for (int p = threadIdx.x; p < cnt; p += SCORE_T) {
      float x, y, z;
      ov_move(s_rt + 12 * hb, s_p[3 * p], s_p[3 * p + 1], s_p[3 * p + 2], x, y, z);
      acc += ghicp_sac::sac_term_fx(sac_nn_d2(r, G, x, y, z, a.thr), a.thr);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) s_red[hb][warp] = acc;
  }
  __syncthreads();
  if (threadIdx.x < SCORE_HB && s_ok[threadIdx.x]) {
    unsigned long long t = 0ull;
    for (int w = 0; w < SCORE_T / 32; ++w) t += s_red[threadIdx.x][w];
    atomicAdd(a.err + h0 + threadIdx.x, t);
  }
}

// out[0] = h* (-1: every hypothesis invalid), out[1] = invalid hypotheses
__global__ void __launch_bounds__(PICK_T) k_sac_pick(const SacArgs a, int *__restrict__ out) {
  __shared__ unsigned long long s_e[PICK_T / 32];
  __shared__ int s_h[PICK_T / 32], s_inv[PICK_T / 32];
  unsigned long long be = ~0ull;
  int bh = INT_MAX, inv = 0;
  for (int h = threadIdx.x; h < a.H; h += PICK_T) {
    if (!a.valid[h]) { ++inv; continue; }
    const unsigned long long e = a.err[h];
    if (e < be || (e == be && h < bh)) { be = e; bh = h; }   // PCL replaces the best on a strict <: ties go to the first
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long oe = __shfl_xor_sync(0xffffffffu, be, o);
    const int oh = __shfl_xor_sync(0xffffffffu, bh, o);
    inv += __shfl_xor_sync(0xffffffffu, inv, o);
    if (oe < be || (oe == be && oh < bh)) { be = oe; bh = oh; }
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) { s_e[warp] = be; s_h[warp] = bh; s_inv[warp] = inv; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < PICK_T / 32; ++w) {
      if (s_e[w] < be || (s_e[w] == be && s_h[w] < bh)) { be = s_e[w]; bh = s_h[w]; }
      inv += s_inv[w];
    }
    out[0] = bh == INT_MAX ? -1 : bh;
    out[1] = inv;
  }
}

struct Rt12 { float v[12]; };
// per source point: the nearest target distance under the chosen transform when within the threshold, else +inf
__global__ void k_sac_fit(const SacArgs a, const RingGrid G, const Rt12 rt, float *__restrict__ d2o) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.ns) return;
  const GridRegs r = grid_regs(G.g);
  float x, y, z;
  ov_move(rt.v, a.P[3 * (size_t)i], a.P[3 * (size_t)i + 1], a.P[3 * (size_t)i + 2], x, y, z);
  const float d2 = sac_nn_d2(r, G, x, y, z, a.thr);
  d2o[i] = d2 <= a.thr ? d2 : INFINITY;
}

__global__ void k_sac_soa_to_aos(const double *__restrict__ soa, int n, float *__restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  for (int k = 0; k < 3; ++k) out[3 * (size_t)i + k] = (float)soa[(size_t)k * n + i];
}

inline int nblk(long long n, int t) { return (int)((n + t - 1) / t); }

}  // namespace

cudaError_t sac_points_from_soa(const double *d_soa, int n, float *d_xyz) {
  GHICP_LAUNCH(k_sac_soa_to_aos, nblk(n, SAC_T), SAC_T, 0, 0, d_soa, n, d_xyz);
  return cudaGetLastError();
}

cudaError_t sac_run(const float *d_P, const float *d_Fs, int ns, const float *d_Q, const float *d_Ft, int nt,
                    const ghicp_sac_params *p, ghicp_sac_result *out, SacDebug *dbg) {
  SacArgs a{};
  PointGrid pg;
  StageEvents<5> ev;
  DevBuf<int> samp, valid, need, slot, list, nlist, knn, corr, d_pick; DevBuf<unsigned> dnext;
  DevBuf<float> rts, d_d2; DevBuf<unsigned long long> err;
  int pick[2] = {-1, 0};
  Rt12 rt{};
  const int H = p->max_iterations;
  std::memset(out, 0, sizeof(*out));
  a.P = d_P; a.Fs = d_Fs; a.ns = ns; a.Fq = d_Ft; a.nt = nt;
  a.H = H; a.nsamp = p->nr_samples; a.ke = p->k_correspondences < nt ? p->k_correspondences : nt;
  a.msd = p->min_sample_distance; a.thr = p->corr_dist_threshold; a.seed = p->seed;
  const long long maxq = std::min((long long)ns, (long long)H * p->nr_samples);
  CUDA_TRY(ev.create());
  CUDA_TRY(samp.alloc((size_t)H * a.nsamp)); CUDA_TRY(valid.alloc((size_t)H)); CUDA_TRY(dnext.alloc((size_t)H));
  CUDA_TRY(need.alloc((size_t)ns)); CUDA_TRY(slot.alloc((size_t)ns)); CUDA_TRY(list.alloc((size_t)maxq)); CUDA_TRY(nlist.alloc(1));
  CUDA_TRY(knn.alloc((size_t)maxq * a.ke)); CUDA_TRY(corr.alloc((size_t)H * a.nsamp)); CUDA_TRY(rts.alloc((size_t)H * 12));
  CUDA_TRY(err.alloc((size_t)H)); CUDA_TRY(d_pick.alloc(2)); CUDA_TRY(d_d2.alloc((size_t)ns));
  a.samp = samp.get(); a.valid = valid.get(); a.dnext = dnext.get(); a.need = need.get(); a.slot = slot.get();
  a.list = list.get(); a.nlist = nlist.get(); a.knn = knn.get(); a.corr = corr.get(); a.rt = rts.get(); a.err = err.get();
  CUDA_TRY(cudaMemsetAsync(a.need, 0, sizeof(int) * (size_t)ns, 0)); CUDA_TRY(cudaMemsetAsync(a.nlist, 0, sizeof(int), 0));
  CUDA_TRY(cudaMemsetAsync(a.err, 0, sizeof(unsigned long long) * (size_t)H, 0));
  CUDA_TRY(cudaMemsetAsync(a.rt, 0, sizeof(float) * 12 * (size_t)H, 0));
  CUDA_TRY(cudaMemsetAsync(a.corr, 0xff, sizeof(int) * (size_t)H * a.nsamp, 0));
  CUDA_TRY(cudaEventRecord(ev[0], 0));
  GHICP_LAUNCH(k_sac_sample, nblk(H, SAC_T), SAC_T, 0, 0, a);
  GHICP_LAUNCH(k_sac_compact, nblk(ns, SAC_T), SAC_T, 0, 0, a);
  if (maxq > 0) GHICP_LAUNCH(k_sac_feat_knn, nblk(maxq, FEAT_T), FEAT_T, 0, 0, a);
  CUDA_TRY(cudaEventRecord(ev[1], 0));
  GHICP_LAUNCH(k_sac_estimate, nblk(H, SAC_T), SAC_T, 0, 0, a, d_Q);
  CUDA_TRY(cudaEventRecord(ev[2], 0));
  // Target grid: the k-NN cell rule (a few points per cell), but no finer than sqrt(thr) / 4, so that a query stops within
  // about five rings once no point can come within the threshold.  The result does not depend on the cell edge.
  const int kcell = nt < 8 ? nt : 8;
  CUDA_TRY(prep_point_grid(0, d_Q, nt, kcell, 0.f, std::sqrt((double)a.thr) / 4.0, &pg));
  dim3 grid((unsigned)nblk(H, SCORE_HB), (unsigned)nblk(ns, SCORE_CHUNK));
  GHICP_LAUNCH(k_sac_score, grid, SCORE_T, 0, 0, a, pg.rg);
  CUDA_TRY(cudaEventRecord(ev[3], 0));
  GHICP_LAUNCH(k_sac_pick, 1, PICK_T, 0, 0, a, d_pick.get());
  CUDA_TRY(cudaEventRecord(ev[4], 0));
  CUDA_TRY(cudaMemcpyAsync(pick, d_pick.get(), sizeof(pick), cudaMemcpyDeviceToHost, 0));
  CUDA_TRY(cudaStreamSynchronize(0));
  if (pick[0] >= 0) {
    CUDA_TRY(cudaMemcpy(rt.v, a.rt + 12 * (size_t)pick[0], sizeof(rt.v), cudaMemcpyDeviceToHost));
  } else {   // no valid hypothesis: the identity, scored like any transform
    rt.v[0] = rt.v[4] = rt.v[8] = 1.f;
  }
  GHICP_LAUNCH(k_sac_fit, nblk(ns, SAC_T), SAC_T, 0, 0, a, pg.rg, rt, d_d2.get());
  CUDA_TRY(cudaGetLastError());
  std::vector<float> d2((size_t)ns);
  CUDA_TRY(cudaMemcpyAsync(d2.data(), d_d2.get(), sizeof(float) * (size_t)ns, cudaMemcpyDeviceToHost, 0));
  CUDA_TRY(cudaStreamSynchronize(0));
  unsigned long long fx = 0ull;
  double fit = 0.0;
  int inl = 0;
  for (int i = 0; i < ns; ++i) {   // point order: the fitness sum is fixed
    fx += ghicp_sac::sac_term_fx(d2[i], a.thr);
    if (d2[i] <= a.thr) { fit += (double)d2[i]; ++inl; }
  }
  for (int i = 0; i < 16; ++i) out->Rt[i] = 0.0;
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) out->Rt[j * 4 + i] = (double)rt.v[3 * i + j];
    out->Rt[12 + i] = (double)rt.v[9 + i];
  }
  out->Rt[15] = 1.0;
  out->error = (double)fx / ghicp_sac::SAC_FX_ONE;
  out->fitness = inl > 0 ? fit / inl : DBL_MAX;   // PCL's getFitnessScore without a point in range
  out->inliers = inl;
  out->best_hypothesis = pick[0];
  out->invalid_hypotheses = pick[1];
  for (int k = 0; k < 4; ++k) out->stage_ms[k] = ev.ms(k, k + 1);
  if (dbg) {
    if (dbg->samples) CUDA_TRY(cudaMemcpy(dbg->samples, a.samp, sizeof(int) * (size_t)H * a.nsamp, cudaMemcpyDeviceToHost));
    if (dbg->valid) CUDA_TRY(cudaMemcpy(dbg->valid, a.valid, sizeof(int) * (size_t)H, cudaMemcpyDeviceToHost));
    if (dbg->corr) CUDA_TRY(cudaMemcpy(dbg->corr, a.corr, sizeof(int) * (size_t)H * a.nsamp, cudaMemcpyDeviceToHost));
    if (dbg->rt) CUDA_TRY(cudaMemcpy(dbg->rt, a.rt, sizeof(float) * 12 * (size_t)H, cudaMemcpyDeviceToHost));
    if (dbg->err) CUDA_TRY(cudaMemcpy(dbg->err, a.err, sizeof(unsigned long long) * (size_t)H, cudaMemcpyDeviceToHost));
    dbg->cell = pg.rg.cell;
  }
  return cudaSuccess;
}

}  // namespace ghicp_b200
