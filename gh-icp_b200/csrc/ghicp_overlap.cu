// ghicp_overlap.cu — overlap and fitness of a registration on the dense clouds (DESIGN.md §3.12): the reference's
// CRegistration::calOverlap (src/common_reg.cpp:294-317, the share of cloud A with a cloud-B point within thre_dis) and PCL's
// getFitnessScore (mean squared nearest-neighbour distance within max_range), for every point of A moved by a transform.
//   target grid   B's cell-sorted grid (prep_point_grid, the k-NN cell rule with 8 points per cell): independent of the
//                 threshold, so one grid serves every call on the same target (ghicp_prep_overlap keeps it)
//   k_ov_keys     (fitness mode) the moved points' clamped B-cell keys, radix-sorted into the query order
//   k_ov_query    the hot path: one exact nearest-neighbour query per point of A, a ring walk over B's grid like
//                 ghicp_grid.cuh's ring_walk, but every column is culled by a lower bound on its distance (cell extents
//                 clipped to B's box) and the walk stops once a true lower bound on every unvisited cell passes
//                 min(best, limit).  A query
//                 outside B's box walks only the cells that could hold a closer point.  Work counters: integer atomics.
//   k_ov_reduce   counts and double sums over contiguous point blocks, each in a fixed tree order; k_ov_total sums the
//   k_ov_total    blocks in a fixed order: two runs give identical bits, and no floating-point atomic is used
#include <algorithm>
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstdlib>
#include <cstring>

#include "ghicp_internal.h"
#include "ghicp_device.cuh"
#include "ghicp_grid.cuh"
#include "ghicp_ovwalk.cuh"

namespace ghicp_b200 {

namespace {

constexpr int OV_T = 128;         // threads per query CTA
constexpr int RED_T = 256;        // threads per reduction CTA
constexpr int RED_CHUNK = 8192;   // points per reduction CTA

struct OvArgs {
  const float *A; long long n;
  float rt[12];                   // R row-major, then t (float32, rounded once from the double matrix)
  float hit;                      // overlap-only mode: stop at the first d2 < hit (r*r); fitness mode: -1
  double lim;                     // exact up to this squared distance; beyond it the query reports +inf
  const int *perm;                // query order (nullptr: input order)
  float *d2;                      // [n]
  unsigned long long *work;       // [2] cells visited, candidates examined
};
struct OvPart { double fit, ov; unsigned long long n_fit, n_ov; };

// Nearest squared distance from q to B (ov_nearest of ghicp_ovwalk.cuh without the index)
__device__ float ov_nn_d2(const GridRegs &r, const OvGrid &G, float qx, float qy, float qz, double lim, float hit,
                          unsigned long long &cells, unsigned long long &cand) {
  int unused = -1;
  return ov_nearest<false>(r, G, qx, qy, qz, lim, hit, cells, cand, unused);
}

__global__ void __launch_bounds__(OV_T) k_ov_query(const OvArgs a, const OvGrid G) {
  const long long t = (long long)blockIdx.x * OV_T + threadIdx.x;
  unsigned long long cells = 0ull, cand = 0ull;
  if (t < a.n) {
    const long long i = a.perm ? (long long)a.perm[t] : t;
    const GridRegs r = grid_regs(G.rg.g);   // per-thread registers, see k_pca
    float x, y, z;
    ov_move(a.rt, a.A[3 * i], a.A[3 * i + 1], a.A[3 * i + 2], x, y, z);
    a.d2[i] = ov_nn_d2(r, G, x, y, z, a.lim, a.hit, cells, cand);
  }
  ov_add_work(cells, cand, a.work);
}

// clamped B-cell key of each moved point of A, with its index (the cell order of the queries)
__global__ void k_ov_keys(const OvArgs a, const OvGrid G, pu64 *__restrict__ keys, int *__restrict__ vals) {
  const long long t = (long long)blockIdx.x * OV_T + threadIdx.x;
  if (t >= a.n) return;
  float v[3];
  ov_move(a.rt, a.A[3 * t], a.A[3 * t + 1], a.A[3 * t + 2], v[0], v[1], v[2]);
  keys[t] = ov_cell_key(G, v);
  vals[t] = (int)t;
}

__device__ __forceinline__ void ov_part_add(OvPart &x, const OvPart &y) { x.fit += y.fit; x.ov += y.ov; x.n_fit += y.n_fit; x.n_ov += y.n_ov; }
// fixed-shape tree over the CTA's RED_T partials
__device__ void ov_tree(OvPart *sh, OvPart v, OvPart *out) {
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int w = RED_T / 2; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) ov_part_add(sh[threadIdx.x], sh[threadIdx.x + w]);
    __syncthreads();
  }
  if (threadIdx.x == 0) *out = sh[0];
}
__global__ void __launch_bounds__(RED_T) k_ov_reduce(const float *__restrict__ d2, long long n, float r2, double max_range,
                                                     int fitness, OvPart *__restrict__ part) {
  __shared__ OvPart sh[RED_T];
  const long long p0 = (long long)blockIdx.x * RED_CHUNK, p1 = min(p0 + RED_CHUNK, n);
  OvPart v{0.0, 0.0, 0ull, 0ull};
  for (long long p = p0 + threadIdx.x; p < p1; p += RED_T) {
    const float d = d2[p];
    if (d < r2) { v.ov += (double)d; ++v.n_ov; }
    if (fitness && d != INFINITY && (double)d <= max_range) { v.fit += (double)d; ++v.n_fit; }
  }
  ov_tree(sh, v, part + blockIdx.x);
}
__global__ void __launch_bounds__(RED_T) k_ov_total(const OvPart *__restrict__ part, int nb, OvPart *__restrict__ out) {
  __shared__ OvPart sh[RED_T];
  OvPart v{0.0, 0.0, 0ull, 0ull};
  for (int b = threadIdx.x; b < nb; b += RED_T) ov_part_add(v, part[b]);
  ov_tree(sh, v, out);
}

inline int oblk(long long n, int t) { return (int)((n + t - 1) / t); }

}  // namespace

cudaError_t overlap_target_build(const float *d_b, int n_b, OverlapTarget **out) {
  *out = nullptr;
  OverlapTarget *t = new OverlapTarget();
  t->n = n_b;
  const cudaError_t e = prep_point_grid(0, d_b, n_b, n_b < 8 ? n_b : 8, 0.f, 0.0, &t->pg);
  if (e != cudaSuccess) { delete t; return e; }
  *out = t;
  return cudaSuccess;
}
void overlap_target_free(OverlapTarget *t) { delete t; }

// GHICP_OVERLAP_ORDER=cell | input (test and measurement hook) overrides the query order overlap_run picks by mode
static int overlap_order(int dflt) {
  const char *s = getenv("GHICP_OVERLAP_ORDER");
  if (!s) return dflt;
  return std::strcmp(s, "cell") == 0 ? 1 : (std::strcmp(s, "input") == 0 ? 0 : dflt);
}

cudaError_t overlap_run(const float *d_a, int n_a, const OverlapTarget *t, const double *Rt, float thre_dis, double max_range,
                        int want_fitness, cudaEvent_t ev_queries, ghicp_overlap_result *out, float *h_d2_out) {
  const long long n = n_a;
  const float r2 = thre_dis * thre_dis;
  // fitness mode walks several cells per query: B-cell order keeps a warp's walks in the same cells (3 - 10x faster on an
  // H100, DESIGN.md §3.12); the overlap-only mode mostly stops in the first cell, and the sort costs more than it saves
  const bool cell_order = overlap_order(want_fitness ? 1 : 0) == 1;
  OvArgs a{};
  OvGrid G{};
  DevBuf<float> d2; DevBuf<unsigned long long> work; DevBuf<OvPart> part, tot;
  DevBuf<pu64> keys; DevBuf<int> perm;
  const int nb = oblk(n, RED_CHUNK);
  unsigned long long hwork[2] = {0ull, 0ull};
  OvPart h{};
  // every workspace first: running out of memory returns before anything is written
  CUDA_TRY(d2.alloc((size_t)n)); CUDA_TRY(work.alloc(2)); CUDA_TRY(part.alloc((size_t)nb)); CUDA_TRY(tot.alloc(1));
  if (cell_order) { CUDA_TRY(keys.alloc((size_t)n)); CUDA_TRY(perm.alloc((size_t)n)); }
  CUDA_TRY(cudaMemsetAsync(work.get(), 0, 2 * sizeof(unsigned long long), 0));
  a.A = d_a; a.n = n; a.d2 = d2.get(); a.work = work.get();
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) a.rt[3 * i + j] = Rt ? (float)Rt[j * 4 + i] : (i == j ? 1.f : 0.f);
    a.rt[9 + i] = Rt ? (float)Rt[12 + i] : 0.f;
  }
  a.hit = want_fitness ? -1.f : r2;
  a.lim = want_fitness ? std::max((double)r2, max_range) : (double)r2;
  G = ov_grid_of(t->pg);
  if (ev_queries) CUDA_TRY(cudaEventRecord(ev_queries, 0));
  if (cell_order) {
    GHICP_LAUNCH(k_ov_keys, oblk(n, OV_T), OV_T, 0, 0, a, G, keys.get(), perm.get());
    CUDA_TRY(prep_sort_pairs(0, keys.get(), perm.get(), n_a));
    a.perm = perm.get();
  }
  GHICP_LAUNCH(k_ov_query, oblk(n, OV_T), OV_T, 0, 0, a, G);
  GHICP_LAUNCH(k_ov_reduce, nb, RED_T, 0, 0, d2.get(), n, r2, max_range, want_fitness, part.get());
  GHICP_LAUNCH(k_ov_total, 1, RED_T, 0, 0, part.get(), nb, tot.get());
  CUDA_TRY(cudaGetLastError());
  CUDA_TRY(cudaMemcpyAsync(&h, tot.get(), sizeof(h), cudaMemcpyDeviceToHost, 0));
  CUDA_TRY(cudaMemcpyAsync(hwork, work.get(), sizeof(hwork), cudaMemcpyDeviceToHost, 0));
  if (h_d2_out) CUDA_TRY(cudaMemcpyAsync(h_d2_out, d2.get(), sizeof(float) * (size_t)n, cudaMemcpyDeviceToHost, 0));
  CUDA_TRY(cudaStreamSynchronize(0));
  out->n = n;
  out->overlap = (long long)h.n_ov;
  out->ratio = (float)((0.01 + (double)h.n_ov) / (double)n);   // src/common_reg.cpp:312
  out->overlap_rmse = (want_fitness && h.n_ov > 0) ? std::sqrt(h.ov / (double)h.n_ov) : NAN;
  out->n_fit = want_fitness ? (long long)h.n_fit : 0;
  out->fitness = !want_fitness ? NAN : (h.n_fit > 0 ? h.fit / (double)h.n_fit : DBL_MAX);   // PCL's getFitnessScore without a point in range
  out->cells_visited = (long long)hwork[0];
  out->candidates = (long long)hwork[1];
  return cudaSuccess;
}

}  // namespace ghicp_b200
