// ghicp_prep.cu — pre-processing that feeds the registration loop, on the GPU (SURVEY.md §8f row N1, BASELINE.json
// configs 4 / 5: "voxel 0.05 m downsample + curvature keypoint extract on-GPU"):
//   CFilter::voxelfilter                                   include/filter.hpp:28-88
//   PrincipleComponentAnalysis::CalculatePcaFeaturesOfPointCloud (radius) + CalculatePcaFeature   include/pca.h:133-165, 198-250
//   CKeypointDetect::pruneUnstablePoints / nonMaximaSuppression                                   include/keypoint_detect.hpp:132-191
// The reference does all three on one CPU thread with a KD-tree radius search per point.  Here:
//   voxel filter   = float32 voxel ids exactly as :54-63 -> stable radix sort of (id, index) -> run heads; keeps the
//                    smallest index of a voxel (the reference keeps "the first after an unstable std::sort") and
//                    reproduces its size bug (point 0 emitted once more for voxel id 0, :52 + :66)
//   radius search  = uniform grid with cell edge = radius: points sorted by cell id, 27-cell walk = 9 column runs (the three
//                    z-neighbours of a column are contiguous in the sorted order), lower-bound search of the occupied-cell table (no dense volume: a 5 M-point scan spans > 10^9 cells)
//   PCA            = double sums about the query point, rounded once to float32, cyclic Jacobi in float32
//   NMS            = the greedy scan "best unvisited first, erase its neighbours" (:169-188) is sequential; its result is
//                    the unique fixed point of  keep(r) <=> no kept k < r within the radius  (r = rank by curvature), which
//                    a few data-parallel rounds compute: a candidate is decided once all better-ranked neighbours are.
// Implementation-defined details of the reference (unstable sorts, PCL's neighbour order and float accumulation) get the
// canonical definitions documented in oracle/ghicp_prep_oracle.cpp; the oracle and these kernels agree bit for bit.
// Sort / scan plumbing = CUB (library code; under the host emulation shim: std::stable_sort / a loop).
#include <climits>
#include <cmath>
#include <cstdlib>
#include <cstring>

#include "ghicp_internal.h"
#include "ghicp_device.cuh"
#include "ghicp_grid.cuh"

#if !defined(GHICP_EMU_HOST)
#include <cub/cub.cuh>
#endif

namespace ghicp_b200 {

namespace {

constexpr int PT = 256;

// ---- plumbing: sort, scan (CUB under nvcc; the C++ library under the emulation shim) ----------------------------------
// Workspaces are DevBufs on stream 0 (the whole pre-processing runs on one stream), CUB's temporaries on the sort's stream.
#if defined(GHICP_EMU_HOST)
}  // namespace
}  // namespace ghicp_b200
#include <algorithm>
#include <vector>
namespace ghicp_b200 {
namespace {
cudaError_t sort_pairs(pu64 *keys, int *vals, int n, cudaStream_t) {   // stable, ascending keys
  std::vector<int> perm(n);
  for (int i = 0; i < n; ++i) perm[i] = i;
  std::stable_sort(perm.begin(), perm.end(), [&](int a, int b) { return keys[a] < keys[b]; });
  std::vector<pu64> k(n); std::vector<int> v(n);
  for (int i = 0; i < n; ++i) { k[i] = keys[perm[i]]; v[i] = vals[perm[i]]; }
  memcpy(keys, k.data(), sizeof(pu64) * n); memcpy(vals, v.data(), sizeof(int) * n);
  return cudaSuccess;
}
cudaError_t exclusive_scan(const int *in, int *out, int n, cudaStream_t) {   // out[n] = total
  int run = 0;
  for (int i = 0; i < n; ++i) { out[i] = run; run += in[i]; }
  out[n] = run;
  return cudaSuccess;
}
cudaError_t exclusive_scan64(const long long *in, long long *out, int n, cudaStream_t) {   // out[n] = total
  long long run = 0;
  for (int i = 0; i < n; ++i) { out[i] = run; run += in[i]; }
  out[n] = run;
  return cudaSuccess;
}
// every segment [off[r], off[r + 1]) of in sorted ascending into out (keys are distinct within a segment)
cudaError_t segmented_sort(const pu64 *in, pu64 *out, long long total, int m, const long long *off, cudaStream_t) {
  memcpy(out, in, sizeof(pu64) * (size_t)total);
  for (int r = 0; r < m; ++r) std::sort(out + off[r], out + off[r + 1]);
  return cudaSuccess;
}
#else
cudaError_t sort_pairs(pu64 *keys, int *vals, int n, cudaStream_t st) {   // stable LSD radix sort, ascending keys
  DevBuf<pu64> k2; DevBuf<int> v2; DevBuf<unsigned char> tmp; size_t tb = 0;
  CUDA_TRY(k2.alloc((size_t)n));
  CUDA_TRY(v2.alloc((size_t)n));
  CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, tb, keys, k2.get(), vals, v2.get(), n, 0, 64, st));
  CUDA_TRY(tmp.alloc(tb, st));
  CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp.get(), tb, keys, k2.get(), vals, v2.get(), n, 0, 64, st));
  CUDA_TRY(cudaMemcpyAsync(keys, k2.get(), sizeof(pu64) * (size_t)n, cudaMemcpyDeviceToDevice, st));
  CUDA_TRY(cudaMemcpyAsync(vals, v2.get(), sizeof(int) * (size_t)n, cudaMemcpyDeviceToDevice, st));
  return cudaSuccess;   // stream-ordered frees: no host synchronisation needed
}
cudaError_t exclusive_scan(const int *in, int *out, int n, cudaStream_t st) {   // out[n] = total (in[n] must be readable)
  DevBuf<unsigned char> tmp; size_t tb = 0;
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, tb, in, out, n + 1, st));
  CUDA_TRY(tmp.alloc(tb, st));
  return cub::DeviceScan::ExclusiveSum(tmp.get(), tb, in, out, n + 1, st);
}
cudaError_t exclusive_scan64(const long long *in, long long *out, int n, cudaStream_t st) {   // out[n] = total (in[n] readable)
  DevBuf<unsigned char> tmp; size_t tb = 0;
  CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, tb, in, out, n + 1, st));
  CUDA_TRY(tmp.alloc(tb, st));
  return cub::DeviceScan::ExclusiveSum(tmp.get(), tb, in, out, n + 1, st);
}
cudaError_t segmented_sort(const pu64 *in, pu64 *out, long long total, int m, const long long *off, cudaStream_t st);   // below
#endif

// ---- small device helpers ---------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned f2ord(float f) { const unsigned b = __float_as_uint(f); return (b & 0x80000000u) ? ~b : (b | 0x80000000u); }
__host__ __device__ inline float ord2f(unsigned u) {
  const unsigned b = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
  float f;
#if defined(__CUDA_ARCH__)
  f = __uint_as_float(b);
#else
  memcpy(&f, &b, 4);
#endif
  return f;
}

// cyclic Jacobi on a symmetric 3x3 (float32), eigenvalues descending; c = {xx, xy, xz, yy, yz, zz}
__device__ void sym3_eig_f32(const float c[6], float lam[3]) {
  float a[3][3] = {{c[0], c[1], c[2]}, {c[1], c[3], c[4]}, {c[2], c[4], c[5]}};
  for (int sweep = 0; sweep < 24; ++sweep) {
    const float off = fabsf(a[0][1]) + fabsf(a[0][2]) + fabsf(a[1][2]);
    const float diag = fabsf(a[0][0]) + fabsf(a[1][1]) + fabsf(a[2][2]);
    if (off <= 1e-12f * diag || off == 0.f) break;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        const float apq = a[p][q];
        if (apq == 0.f) continue;
        const float theta = (a[q][q] - a[p][p]) / (2.0f * apq);
        float t = 1.0f / (fabsf(theta) + sqrtf(theta * theta + 1.0f));
        if (theta < 0.f) t = -t;
        const float cs = 1.0f / sqrtf(t * t + 1.0f), sn = t * cs;
        const int r = 3 - p - q;
        const float app = a[p][p], aqq = a[q][q], arp = a[r][p], arq = a[r][q];
        a[p][p] = app - t * apq;
        a[q][q] = aqq + t * apq;
        a[p][q] = a[q][p] = 0.f;
        a[r][p] = a[p][r] = cs * arp - sn * arq;
        a[r][q] = a[q][r] = sn * arp + cs * arq;
      }
  }
  float l0 = a[0][0], l1 = a[1][1], l2 = a[2][2], tmp;
  if (l0 < l1) { tmp = l0; l0 = l1; l1 = tmp; }
  if (l1 < l2) { tmp = l1; l1 = l2; l2 = tmp; }
  if (l0 < l1) { tmp = l0; l0 = l1; l1 = tmp; }
  lam[0] = l0; lam[1] = l1; lam[2] = l2;
}

// ---- kernels ------------------------------------------------------------------------------------------------------------
// bounding box of the finite points ids[k] (or of all points when ids == nullptr): ordered-uint atomics, warp-reduced
// first.  box[6] counts the finite points, box[7] is the smallest k of a finite point.  Non-finite points are left out (f2ord
// would order +NaN above +inf and make the maximum NaN).
__global__ void k_bbox(const float *__restrict__ xyz, const int *__restrict__ ids, int n, unsigned *__restrict__ box) {
  unsigned lo[3] = {0xffffffffu, 0xffffffffu, 0xffffffffu}, hi[3] = {0u, 0u, 0u}, cnt = 0u, first = 0xffffffffu;
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
    const float *p = xyz + 3 * (size_t)(ids ? ids[k] : k);
    if (!finite3(p[0], p[1], p[2])) continue;
    ++cnt; first = (unsigned)k < first ? (unsigned)k : first;
#pragma unroll
    for (int a = 0; a < 3; ++a) { const unsigned u = f2ord(p[a]); lo[a] = u < lo[a] ? u : lo[a]; hi[a] = u > hi[a] ? u : hi[a]; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const unsigned l = __shfl_xor_sync(0xffffffffu, lo[a], o), h = __shfl_xor_sync(0xffffffffu, hi[a], o);
      lo[a] = l < lo[a] ? l : lo[a]; hi[a] = h > hi[a] ? h : hi[a];
    }
    const unsigned f = __shfl_xor_sync(0xffffffffu, first, o);
    cnt += __shfl_xor_sync(0xffffffffu, cnt, o); first = f < first ? f : first;
  }
  if ((threadIdx.x & 31) == 0) {
#pragma unroll
    for (int a = 0; a < 3; ++a) { atomicMin(&box[a], lo[a]); atomicMax(&box[3 + a], hi[a]); }
    if (cnt) { atomicAdd(&box[6], cnt); atomicMin(&box[7], first); }
  }
}
// voxel id of every point, float32 arithmetic as include/filter.hpp:54-63; a non-finite point gets id 0
__global__ void k_voxel_keys(const float *__restrict__ xyz, int n, float mnx, float mny, float mnz, float inv, pu64 mul_vx,
                             pu64 mul_vy, pu64 *__restrict__ keys, int *__restrict__ vals) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float x = xyz[3 * (size_t)i], y = xyz[3 * (size_t)i + 1], z = xyz[3 * (size_t)i + 2];
  vals[i] = i;
  if (!finite3(x, y, z)) { keys[i] = 0ull; return; }   // joins the voxel-0 run, which is never emitted
  const pu64 vx = (pu64)floorf((x - mnx) * inv), vy = (pu64)floorf((y - mny) * inv), vz = (pu64)floorf((z - mnz) * inv);
  keys[i] = vx * mul_vx + vy * mul_vy + vz;
}
// grid cell of the points ids[k] (or k): key + position k; non-finite points share the last key
__global__ void k_cell_keys(const float *__restrict__ xyz, const int *__restrict__ ids, int n, float mnx, float mny, float mnz,
                            float inv, pu64 *__restrict__ keys, int *__restrict__ vals) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const float *p = xyz + 3 * (size_t)(ids ? ids[k] : k);
  keys[k] = finite3(p[0], p[1], p[2]) ? cell_key(cell_coord(p[0], mnx, inv), cell_coord(p[1], mny, inv), cell_coord(p[2], mnz, inv))
                                      : ~0ull;   // after every cell a walk reads (no distance to it is < r2 anyway)
  vals[k] = k;
}
// heads of the runs of equal keys in a sorted array (flags[n] = 0 so that the scan yields the total)
__global__ void k_run_heads(const pu64 *__restrict__ keys, int n, int skip_zero_key, int *__restrict__ flags) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n) return;
  if (i == n) { flags[i] = 0; return; }
  const bool head = i == 0 || keys[i] != keys[i - 1];
  flags[i] = (head && !(skip_zero_key && keys[i] == 0ull)) ? 1 : 0;
}
// voxel filter output: [the first finite point (the reference's phantom voxel-0 entry)] + the first (smallest) index of
// every run
__global__ void k_voxel_emit(const int *__restrict__ vals, const int *__restrict__ flags, const int *__restrict__ pos, int n,
                             int head, int *__restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) out[0] = head;
  if (i < n && flags[i]) out[1 + pos[i]] = vals[i];
}
// table of occupied cells: ucell[u] = key, cstart[u] = first position in the sorted order (cstart[nu] = n)
__global__ void k_cell_table(const pu64 *__restrict__ keys, const int *__restrict__ flags, const int *__restrict__ pos, int n,
                             pu64 *__restrict__ ucell, int *__restrict__ cstart) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && flags[i]) { ucell[pos[i]] = keys[i]; cstart[pos[i]] = i; }
  if (i == n) cstart[pos[n]] = n;
}
// The three cells (x, y, cz - 1 .. cz + 1) of a grid column have consecutive keys (z is the low field), so their points are
// ONE contiguous run of the sorted order: one lower-bound search per column instead of three exact searches — 9 per point.
__device__ __forceinline__ void column_run(const GridArgs &g, int x, int y, int cz, int &s0, int &s1) {
  const pu64 klo = cell_key(x, y, cz > 0 ? cz - 1 : 0), khi = cell_key(x, y, cz + 1);
  int lo = 0, hi = g.nu;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (g.ucell[mid] < klo) lo = mid + 1; else hi = mid;
  }
  int u1 = lo;
  while (u1 < g.nu && g.ucell[u1] <= khi) ++u1;   // at most three cells
  s0 = g.cstart[lo]; s1 = g.cstart[u1];            // cstart holds nu + 1 entries
}
__device__ __forceinline__ void column_run_r(const GridRegs &g, int x, int y, int cz, int &s0, int &s1) {
  const pu64 klo = cell_key(x, y, cz > 0 ? cz - 1 : 0), khi = cell_key(x, y, cz + 1);
  int lo = 0, hi = g.nu;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (g.ucell[mid] < klo) lo = mid + 1; else hi = mid;
  }
  int u1 = lo;
  while (u1 < g.nu && g.ucell[u1] <= khi) ++u1;   // at most three cells
  s0 = g.cstart[lo]; s1 = g.cstart[u1];            // cstart holds nu + 1 entries
}
// radius PCA of every point (include/pca.h:133-165, 198-233): one thread per point
__global__ void k_pca(const GridArgs g, int n, float *__restrict__ lam, double *__restrict__ curvature, int *__restrict__ pt_num) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n) return;
  const GridRegs r = grid_regs(g);
  const int i = r.order[t];   // threads of a warp take points of the same cell: same 27 runs, loads broadcast instead of scattered
  const float qx = g.xyz[3 * (size_t)i], qy = g.xyz[3 * (size_t)i + 1], qz = g.xyz[3 * (size_t)i + 2];
  if (!finite3(qx, qy, qz)) {   // no neighbour: the outputs of an empty neighbourhood, never a keypoint
    pt_num[i] = 0; lam[3 * (size_t)i] = 0.f; lam[3 * (size_t)i + 1] = 0.f; lam[3 * (size_t)i + 2] = 0.f; curvature[i] = 0.0;
    return;
  }
  const int cx = cell_coord(qx, g.mnx, g.inv), cy = cell_coord(qy, g.mny, g.inv), cz = cell_coord(qz, g.mnz, g.inv);
  int cnt = 0;
  double sd[3] = {0, 0, 0}, sdd[6] = {0, 0, 0, 0, 0, 0};
  int rs0[9], rs1[9];   // the nine column runs, x slowest (the oracle's 27-cell order: x, y, z-fastest)
#pragma unroll
  for (int c9 = 0; c9 < 9; ++c9) {
    const int x = cx + c9 / 3 - 1, y = cy + c9 % 3 - 1;
    rs0[c9] = 0; rs1[c9] = 0;
    if (x >= 0 && y >= 0) column_run_r(r, x, y, cz, rs0[c9], rs1[c9]);
  }
#pragma unroll
  for (int c9 = 0; c9 < 9; ++c9)
    for (int s = rs0[c9]; s < rs1[c9]; ++s) {
      const float4 pt = r.sorted[s];
      const float ex = pt.x - qx, ey = pt.y - qy, ez = pt.z - qz;
      const float d2 = ex * ex + ey * ey + ez * ez;
      if (!(d2 < r.r2)) continue;
      ++cnt;
      const double a = ex, b = ey, c = ez;
      sd[0] += a; sd[1] += b; sd[2] += c;
      sdd[0] += a * a; sdd[1] += a * b; sdd[2] += a * c; sdd[3] += b * b; sdd[4] += b * c; sdd[5] += c * c;
    }
  pt_num[i] = cnt;
  float l[3] = {0.f, 0.f, 0.f};
  double curv = 0.0;
  if (cnt >= 3) {
    const double inv_n = 1.0 / cnt, alpha = 1.0 / (cnt - 1);
    const float cv[6] = {(float)((sdd[0] - sd[0] * sd[0] * inv_n) * alpha), (float)((sdd[1] - sd[0] * sd[1] * inv_n) * alpha),
                         (float)((sdd[2] - sd[0] * sd[2] * inv_n) * alpha), (float)((sdd[3] - sd[1] * sd[1] * inv_n) * alpha),
                         (float)((sdd[4] - sd[1] * sd[2] * inv_n) * alpha), (float)((sdd[5] - sd[2] * sd[2] * inv_n) * alpha)};
    sym3_eig_f32(cv, l);
    const double l1 = l[0], l2 = l[1], l3 = l[2];
    curv = (l1 + l2 + l3) == 0 ? 0.0 : l3 / (l1 + l2 + l3);
  }
  lam[3 * (size_t)i] = l[0]; lam[3 * (size_t)i + 1] = l[1]; lam[3 * (size_t)i + 2] = l[2];
  curvature[i] = curv;
}
// pruneUnstablePoints (include/keypoint_detect.hpp:132-147); flags[n] = 0
__global__ void k_prune(const float *__restrict__ lam, const int *__restrict__ pt_num, int n, float ratio_max, int min_pts,
                        int *__restrict__ flags) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n) return;
  if (i == n) { flags[i] = 0; return; }
  const float ratio1 = (float)((double)lam[3 * (size_t)i + 1] / (double)lam[3 * (size_t)i]);
  const float ratio2 = (float)((double)lam[3 * (size_t)i + 2] / (double)lam[3 * (size_t)i + 1]);
  flags[i] = (ratio1 < ratio_max && ratio2 < ratio_max && pt_num[i] > min_pts) ? 1 : 0;
}
// candidates in ascending index order + their sort keys: descending curvature (curvature >= 0: ordered double bits)
__global__ void k_cand_emit(const int *__restrict__ flags, const int *__restrict__ pos, const double *__restrict__ curvature, int n,
                            pu64 *__restrict__ keys, int *__restrict__ cand) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && flags[i]) {
    cand[pos[i]] = i;
    // descending curvature as an ascending unsigned key (total order on doubles: negative values can appear when the
    // smallest eigenvalue rounds below zero)
    const pu64 b = (pu64)__double_as_longlong(curvature[i]);
    const pu64 ord = (b >> 63) ? ~b : (b | 0x8000000000000000ull);
    keys[pos[i]] = ~ord;
  }
}
// one round of the data-parallel non-maximum suppression; state: 0 undecided, 1 kept, 2 suppressed
__global__ void k_nms_round(const GridArgs g, int m, int *__restrict__ state, int *__restrict__ undecided) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= m) return;
  const GridRegs gr = grid_regs(g);   // per-thread registers, see k_pca
  const int r = gr.order[t];   // candidates in cell order (see k_pca)
  if (state[r] != 0) return;
  const float *q = g.xyz + 3 * (size_t)g.ids[r];
  const float qx = q[0], qy = q[1], qz = q[2];
  const int cx = cell_coord(qx, g.mnx, g.inv), cy = cell_coord(qy, g.mny, g.inv), cz = cell_coord(qz, g.mnz, g.inv);
  int rs0[9], rs1[9];
#pragma unroll
  for (int c9 = 0; c9 < 9; ++c9) {
    const int x = cx + c9 / 3 - 1, y = cy + c9 % 3 - 1;
    rs0[c9] = 0; rs1[c9] = 0;
    if (x >= 0 && y >= 0) column_run_r(gr, x, y, cz, rs0[c9], rs1[c9]);
  }
  bool suppressed = false, blocked = false;
#pragma unroll
  for (int c9 = 0; c9 < 9; ++c9)
    for (int s = rs0[c9]; s < rs1[c9] && !suppressed; ++s) {
      const int k = gr.order[s];
      if (k >= r) continue;                          // only better-ranked candidates can suppress r
      const float4 p = gr.sorted[s];
      const float ex = p.x - qx, ey = p.y - qy, ez = p.z - qz;
      if (!(ex * ex + ey * ey + ez * ez < gr.r2)) continue;
      const int sk = state[k];
      if (sk == 1) suppressed = true;
      else if (sk == 0) blocked = true;
    }
  if (suppressed) state[r] = 2;
  else if (!blocked) state[r] = 1;
  else atomicAdd(undecided, 1);
}
__global__ void k_kept_flags(const int *__restrict__ state, int m, int *__restrict__ flags) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r > m) return;
  flags[r] = (r < m && state[r] == 1) ? 1 : 0;
}
__global__ void k_kp_emit(const int *__restrict__ flags, const int *__restrict__ pos, const int *__restrict__ cand, int m,
                          int *__restrict__ out) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r < m && flags[r]) out[pos[r]] = cand[r];
}

// points in cell order, padded to 16 bytes
__global__ void k_gather_sorted(const float *__restrict__ xyz, const int *__restrict__ ids, const int *__restrict__ order, int n,
                                float4 *__restrict__ sorted) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const int k = ids ? ids[order[s]] : order[s];
  sorted[s] = make_float4(xyz[3 * (size_t)k], xyz[3 * (size_t)k + 1], xyz[3 * (size_t)k + 2], 0.f);
}

inline int blocks(int n) { return (n + PT - 1) / PT; }

// Bounding box of the finite points ids[k] (k < n; all points when ids == nullptr), their number and the smallest such k
// (n when none).  Without a finite point the box is the origin, so that every grid built on it stays defined.
struct FiniteBox { float mn[3], mx[3]; int nfin, first; };
cudaError_t finite_box(cudaStream_t st, const float *d_xyz, const int *d_ids, int n, FiniteBox *b) {
  DevBuf<unsigned> d_box; unsigned h[8];
  const unsigned init[8] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0u, 0u, 0u, 0u, 0xffffffffu};
  CUDA_TRY(d_box.alloc(8));
  CUDA_TRY(cudaMemcpyAsync(d_box.get(), init, sizeof(init), cudaMemcpyHostToDevice, st));
  GHICP_LAUNCH(k_bbox, n < GHICP_SMS * 8 * PT ? blocks(n) : GHICP_SMS * 8, PT, 0, st, d_xyz, d_ids, n, d_box.get());
  CUDA_TRY(cudaMemcpyAsync(h, d_box.get(), sizeof(h), cudaMemcpyDeviceToHost, st)); CUDA_TRY(cudaStreamSynchronize(st));
  b->nfin = (int)h[6]; b->first = b->nfin ? (int)h[7] : n;
  for (int a = 0; a < 3; ++a) { b->mn[a] = b->nfin ? ord2f(h[a]) : 0.f; b->mx[a] = b->nfin ? ord2f(h[3 + a]) : 0.f; }
  return cudaSuccess;
}

// uniform grid over the points ids[k] (k < n); *out receives the device arrays g points into
cudaError_t build_grid(cudaStream_t st, const float *d_xyz, const int *d_ids, int n, float cell, GridArgs *g, GridBufs *out) {
  DevBuf<pu64> d_keys; DevBuf<int> d_flags, d_pos;
  GridBufs b;
  FiniteBox box;
  int nu = 0;
  CUDA_TRY(finite_box(st, d_xyz, d_ids, n, &box));
  g->mnx = box.mn[0]; g->mny = box.mn[1]; g->mnz = box.mn[2];
  g->inv = 1.0f / cell; g->r2 = cell * cell;
  CUDA_TRY(d_keys.alloc((size_t)n)); CUDA_TRY(b.order.alloc((size_t)n)); CUDA_TRY(d_flags.alloc((size_t)n + 1)); CUDA_TRY(d_pos.alloc((size_t)n + 1));
  GHICP_LAUNCH(k_cell_keys, blocks(n), PT, 0, st, d_xyz, d_ids, n, g->mnx, g->mny, g->mnz, g->inv, d_keys.get(), b.order.get());
  CUDA_TRY(sort_pairs(d_keys.get(), b.order.get(), n, st));
  GHICP_LAUNCH(k_run_heads, blocks(n + 1), PT, 0, st, d_keys.get(), n, 0, d_flags.get());
  CUDA_TRY(exclusive_scan(d_flags.get(), d_pos.get(), n, st));
  CUDA_TRY(cudaMemcpyAsync(&nu, d_pos.get() + n, sizeof(int), cudaMemcpyDeviceToHost, st)); CUDA_TRY(cudaStreamSynchronize(st));
  CUDA_TRY(b.ucell.alloc((size_t)nu)); CUDA_TRY(b.cstart.alloc((size_t)nu + 1));
  GHICP_LAUNCH(k_cell_table, blocks(n + 1), PT, 0, st, d_keys.get(), d_flags.get(), d_pos.get(), n, b.ucell.get(), b.cstart.get());
  CUDA_TRY(b.sorted.alloc((size_t)n));
  GHICP_LAUNCH(k_gather_sorted, blocks(n), PT, 0, st, d_xyz, d_ids, b.order.get(), n, b.sorted.get());
  g->xyz = d_xyz; g->ids = d_ids; g->order = b.order.get(); g->sorted = b.sorted.get(); g->ucell = b.ucell.get();
  g->cstart = b.cstart.get(); g->nu = nu;
  *out = std::move(b);
  return cudaSuccess;
}

}  // namespace

// CFilter::voxelfilter on device arrays: d_out (capacity n + 1) receives the kept indices in output order
cudaError_t prep_voxel_downsample(cudaStream_t st, const float *d_xyz, int n, float voxel_size, int *d_out, int *n_out) {
  DevBuf<pu64> d_keys; DevBuf<int> d_vals, d_flags, d_pos;
  FiniteBox box;
  *n_out = 0;
  if (n <= 0) return cudaSuccess;
  CUDA_TRY(finite_box(st, d_xyz, nullptr, n, &box));   // pcl::removeNaNFromPointCloud, then pcl::getMinMax3D
  if (box.nfin == 0) return cudaSuccess;
  const float *mn = box.mn, *mx = box.mx;
  const float inv = 1.0f / voxel_size;                                   // include/filter.hpp:30
  const float gy = mx[1] - mn[1], gz = mx[2] - mn[2];                    // :36
  const pu64 max_vy = (pu64)(ceilf(gy * inv) + 1), max_vz = (pu64)(ceilf(gz * inv) + 1);   // :39-40
  const pu64 mul_vx = max_vy * max_vz, mul_vy = max_vz;                  // :48-49
  CUDA_TRY(d_keys.alloc((size_t)n)); CUDA_TRY(d_vals.alloc((size_t)n)); CUDA_TRY(d_flags.alloc((size_t)n + 1)); CUDA_TRY(d_pos.alloc((size_t)n + 1));
  GHICP_LAUNCH(k_voxel_keys, blocks(n), PT, 0, st, d_xyz, n, mn[0], mn[1], mn[2], inv, mul_vx, mul_vy, d_keys.get(), d_vals.get());
  CUDA_TRY(sort_pairs(d_keys.get(), d_vals.get(), n, st));          // stable: ascending index inside a voxel
  // the reference's phantom entries {voxel 0, index 0} (:52) put point 0 of the finite cloud first and absorb the real voxel-0
  // run (and the non-finite points)
  GHICP_LAUNCH(k_run_heads, blocks(n + 1), PT, 0, st, d_keys.get(), n, 1, d_flags.get());
  CUDA_TRY(exclusive_scan(d_flags.get(), d_pos.get(), n, st));
  int runs = 0;
  CUDA_TRY(cudaMemcpyAsync(&runs, d_pos.get() + n, sizeof(int), cudaMemcpyDeviceToHost, st)); CUDA_TRY(cudaStreamSynchronize(st));
  GHICP_LAUNCH(k_voxel_emit, blocks(n), PT, 0, st, d_vals.get(), d_flags.get(), d_pos.get(), n, box.first, d_out);
  CUDA_TRY(cudaStreamSynchronize(st));
  *n_out = runs + 1;
  return cudaSuccess;
}

// keypointDetectionBasedOnCurvature on device arrays.  d_lam [n][3], d_curv [n], d_cnt [n], d_kp (capacity n).
cudaError_t prep_detect_keypoints(cudaStream_t st, const float *d_xyz, int n, float radius, float ratio_max, int min_pts,
                                  float nms_radius, float *d_lam, double *d_curv, int *d_cnt, int *d_kp, int *n_kp,
                                  int *nms_rounds) {
  GridArgs g{}, g2{};
  GridBufs grid, grid2;
  DevBuf<int> d_flags, d_pos, d_cand, d_state, d_und; DevBuf<pu64> d_keys;
  int m = 0, rounds = 0;
  *n_kp = 0;
  if (nms_rounds) *nms_rounds = 0;
  if (n <= 0) return cudaSuccess;
  CUDA_TRY(build_grid(st, d_xyz, nullptr, n, radius, &g, &grid));
  GHICP_LAUNCH(k_pca, blocks(n), PT, 0, st, g, n, d_lam, d_curv, d_cnt);
  CUDA_TRY(d_flags.alloc((size_t)n + 1)); CUDA_TRY(d_pos.alloc((size_t)n + 1));
  GHICP_LAUNCH(k_prune, blocks(n + 1), PT, 0, st, d_lam, d_cnt, n, ratio_max, min_pts, d_flags.get());
  CUDA_TRY(exclusive_scan(d_flags.get(), d_pos.get(), n, st));
  CUDA_TRY(cudaMemcpyAsync(&m, d_pos.get() + n, sizeof(int), cudaMemcpyDeviceToHost, st)); CUDA_TRY(cudaStreamSynchronize(st));
  if (m == 0) return cudaSuccess;
  CUDA_TRY(d_cand.alloc((size_t)m)); CUDA_TRY(d_keys.alloc((size_t)m));
  GHICP_LAUNCH(k_cand_emit, blocks(n), PT, 0, st, d_flags.get(), d_pos.get(), d_curv, n, d_keys.get(), d_cand.get());
  CUDA_TRY(sort_pairs(d_keys.get(), d_cand.get(), m, st));   // rank order: descending curvature, ties by ascending index (stable)
  CUDA_TRY(build_grid(st, d_xyz, d_cand.get(), m, nms_radius, &g2, &grid2));
  CUDA_TRY(d_state.alloc((size_t)m)); CUDA_TRY(d_und.alloc(1));
  CUDA_TRY(cudaMemsetAsync(d_state.get(), 0, sizeof(int) * (size_t)m, st));
  for (;;) {
    int und = 0;
    CUDA_TRY(cudaMemsetAsync(d_und.get(), 0, sizeof(int), st));
    GHICP_LAUNCH(k_nms_round, blocks(m), PT, 0, st, g2, m, d_state.get(), d_und.get());
    CUDA_TRY(cudaMemcpyAsync(&und, d_und.get(), sizeof(int), cudaMemcpyDeviceToHost, st)); CUDA_TRY(cudaStreamSynchronize(st));
    ++rounds;
    if (und == 0) break;
    if (rounds > m + 1) return cudaErrorInvalidValue;   // cannot happen: the best undecided rank decides every round
  }
  d_flags.reset(); d_pos.reset();
  CUDA_TRY(d_flags.alloc((size_t)m + 1)); CUDA_TRY(d_pos.alloc((size_t)m + 1));
  GHICP_LAUNCH(k_kept_flags, blocks(m + 1), PT, 0, st, d_state.get(), m, d_flags.get());
  CUDA_TRY(exclusive_scan(d_flags.get(), d_pos.get(), m, st));
  CUDA_TRY(cudaMemcpyAsync(n_kp, d_pos.get() + m, sizeof(int), cudaMemcpyDeviceToHost, st)); CUDA_TRY(cudaStreamSynchronize(st));
  GHICP_LAUNCH(k_kp_emit, blocks(m), PT, 0, st, d_flags.get(), d_pos.get(), d_cand.get(), m, d_kp);
  CUDA_TRY(cudaStreamSynchronize(st));
  if (nms_rounds) *nms_rounds = rounds;
  return cudaSuccess;
}


// ---- glue kernels of the device-resident pipeline (ghicp_prep_run, ghicp_capi.cu) --------------------------------------
namespace {
__global__ void k_gather_points(const float *__restrict__ xyz, const int *__restrict__ idx, int m, float *__restrict__ out) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= m) return;
  const size_t i = (size_t)idx[k];
  out[3 * (size_t)k] = xyz[3 * i]; out[3 * (size_t)k + 1] = xyz[3 * i + 1]; out[3 * (size_t)k + 2] = xyz[3 * i + 2];
}
// keypoint coordinates as the reference holds them: Eigen::MatrixX3d, column-major = SoA [3][nkp], float32 values widened
__global__ void k_kp_coords(const float *__restrict__ xyz, const int *__restrict__ kp, int nkp, double *__restrict__ soa) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= nkp) return;
  const size_t i = (size_t)kp[k];
  soa[k] = (double)xyz[3 * i]; soa[(size_t)nkp + k] = (double)xyz[3 * i + 1]; soa[2 * (size_t)nkp + k] = (double)xyz[3 * i + 2];
}
}  // namespace
cudaError_t prep_gather_points(cudaStream_t st, const float *d_xyz, const int *d_idx, int m, float *d_out) {
  if (m <= 0) return cudaSuccess;
  GHICP_LAUNCH(k_gather_points, blocks(m), PT, 0, st, d_xyz, d_idx, m, d_out);
  return cudaSuccess;
}
cudaError_t prep_kp_coords(cudaStream_t st, const float *d_xyz, const int *d_kp, int nkp, double *d_soa) {
  if (nkp <= 0) return cudaSuccess;
  GHICP_LAUNCH(k_kp_coords, blocks(nkp), PT, 0, st, d_xyz, d_kp, nkp, d_soa);
  return cudaSuccess;
}
// pcl::getMinMax3D of the finite points of a device cloud (the bounding box the driver takes its bbx_magnitude from,
// test/ghicp_main.cpp:91-93); *nfin (may be null) receives their number
cudaError_t prep_bounds(cudaStream_t st, const float *d_xyz, int n, float mn[3], float mx[3], int *nfin) {
  FiniteBox box;
  if (n <= 0) return cudaErrorInvalidValue;
  CUDA_TRY(finite_box(st, d_xyz, nullptr, n, &box));
  for (int a = 0; a < 3; ++a) { mn[a] = box.mn[a]; mx[a] = box.mx[a]; }
  if (nfin) *nfin = box.nfin;
  return cudaSuccess;
}

// =====================================================================================================================
// BSC descriptor encoder (SURVEY.md §8f row N2): BSCEncoder::extractBinaryFeatures, include/binary_feature_extraction.hpp
// :603-676 — per keypoint the weighted-PCA local frame (:940-1035, :123-160), the change of frame (:163-196, :1085-1138),
// the three projected Gaussian-weighted side x side grids (:197-373), the 9 side^2-bit descriptor (:464-565) and its
// re-arranged variants (:678-837).  The reference walks three KD-trees per keypoint on one thread; here one CTA per
// keypoint walks the 3 x 3 columns of a uniform grid (edge = search radius sqrt(3) R; a column's three cells are one contiguous
// run of the cell-sorted points) three times:
//   pass A  neighbour count, centroid and the weight sum            (double sums)
//   pass B  weighted covariance about the centroid                  (double sums, rounded once to float32)
//   thread 0: eigenvectors (cyclic Jacobi in double, sign "largest component positive"), the frame, the float32
//            Umeyama fit of the unit axes onto it and its inverse — the reference's own roundabout route to the rotation
//   pass C  every neighbour, moved to the frame in float32, adds exp(-d^2 / 2 delta^2) to the cells whose centre lies
//            within 1.5 cell edges in each projection.  The sums are FIXED-POINT integer atomics in shared memory
//            (weights are float32 in (2^-7, 1]: w * 2^40 is an exact integer), so the result does not depend on the order
//            in which threads arrive: the descriptor is deterministic run to run.
// Where the reference accumulates in float32 in KD-tree result order (covariance, depth sums) this kernel holds the exact
// sum instead; the two differ by float32 accumulation error (~1e-7 relative), which moves a descriptor bit only when a
// comparison is that close to its threshold — tests/ state the tolerance.  Variants 1..3 reproduce the reference's
// ReArrangeGrid quirk: the re-arranged grid is APPENDED to 3 side^2 empty cells (:693-695 after :788), so those
// descriptors carry the occupancy bits of the re-arranged grid at bit offset 3 side^2 and nothing else.
// =====================================================================================================================
namespace {

constexpr int BSC_T = 128;          // threads per keypoint
constexpr int BSC_RUNS = 9;         // 3 x 3 grid columns around the keypoint, each one contiguous run (column_run)
constexpr int BSC_MAX_SIDE = 9;     // grids up to 9 x 9 (the reference uses 7)
constexpr int BSC_MAX_CELLS = 3 * BSC_MAX_SIDE * BSC_MAX_SIDE;

struct BscArgs {
  GridArgs g;
  const int *kp; int nkp;
  float R; int side; const int *pairs; int V;
  unsigned char *bits; int nbytes; float *lrf; int *status;
};

// symmetric 3x3 eigen-decomposition in double (the convention of oracle/stub/Eigen/Eigenvalues, substitution S1)
__device__ void bsc_jacobi3(double a[3][3], double V[3][3], double w[3]) {
  for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) V[i][j] = (i == j) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 64; ++sweep) {
    double off = 0.0;
    for (int p = 0; p < 3; ++p) for (int q = p + 1; q < 3; ++q) off += a[p][q] * a[p][q];
    if (off == 0.0) break;
    for (int p = 0; p < 3; ++p)
      for (int q = p + 1; q < 3; ++q) {
        if (a[p][q] == 0.0) continue;
        const double theta = (a[q][q] - a[p][p]) / (2.0 * a[p][q]);
        const double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < 3; ++k) { const double x = a[k][p], y = a[k][q]; a[k][p] = c * x - s * y; a[k][q] = s * x + c * y; }
        for (int k = 0; k < 3; ++k) { const double x = a[p][k], y = a[q][k]; a[p][k] = c * x - s * y; a[q][k] = s * x + c * y; }
        for (int k = 0; k < 3; ++k) { const double x = V[k][p], y = V[k][q]; V[k][p] = c * x - s * y; V[k][q] = s * x + c * y; }
      }
  }
  for (int j = 0; j < 3; ++j) {
    w[j] = a[j][j];
    int big = 0;
    for (int i = 1; i < 3; ++i) if (fabs(V[i][j]) > fabs(V[big][j])) big = i;
    if (V[big][j] < 0.0) for (int i = 0; i < 3; ++i) V[i][j] = -V[i][j];
  }
}
// inverse of a 4x4 float matrix (column-major) through double Gauss-Jordan, rounded to float (substitution S2)
__device__ void bsc_inverse4(const float m[16], float out[16]) {
  double a[4][8];
  for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) { a[i][j] = (double)m[j * 4 + i]; a[i][4 + j] = (i == j) ? 1.0 : 0.0; }
  for (int c = 0; c < 4; ++c) {
    int p = c;
    for (int i = c + 1; i < 4; ++i) if (fabs(a[i][c]) > fabs(a[p][c])) p = i;
    for (int j = 0; j < 8; ++j) { const double t = a[c][j]; a[c][j] = a[p][j]; a[p][j] = t; }
    const double d = a[c][c];
    for (int j = 0; j < 8; ++j) a[c][j] /= d;
    for (int i = 0; i < 4; ++i) if (i != c) { const double f = a[i][c]; for (int j = 0; j < 8; ++j) a[i][j] -= f * a[c][j]; }
  }
  for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) out[j * 4 + i] = (float)a[i][4 + j];
}
__device__ __forceinline__ void bsc_cross(const float a[3], const float b[3], float o[3]) {
  o[0] = a[1] * b[2] - a[2] * b[1];
  o[1] = a[2] * b[0] - a[0] * b[2];
  o[2] = a[0] * b[1] - a[1] * b[0];
}
__device__ __forceinline__ void bsc_normalize(float a[3]) {
  float z = a[0] * a[0];
  z = z + a[1] * a[1];
  z = z + a[2] * a[2];
  if (z > 0.f) { const float n = sqrtf(z); a[0] = a[0] / n; a[1] = a[1] / n; a[2] = a[2] / n; }
}
// 64-bit add into a (lo, hi) pair of 32-bit shared words: two native atomics, the carry taken from the value the low word
// held before.  Sums modulo 2^64 whatever the order of arrival (two's complement values included).
__device__ __forceinline__ void bsc_add64(unsigned *lo, unsigned *hi, unsigned long long v) {
  const unsigned vlo = (unsigned)v, vhi = (unsigned)(v >> 32);
  const unsigned old = atomicAdd(lo, vlo);
  const unsigned up = vhi + ((unsigned)(old + vlo) < vlo ? 1u : 0u);
  if (up) atomicAdd(hi, up);
}
// index of the source cell of re-arranged cell k of one plane (ReArrange_2D :701-757)
__device__ __forceinline__ int bsc_rearranged(int tr, int k, int side) {
  const int i = k / side, j = k % side;
  return tr == 1 ? side * side - 1 - k : (tr == 2 ? (side - 1 - i) * side + j : i * side + side - 1 - j);
}

__global__ void __launch_bounds__(BSC_T) k_bsc(const BscArgs a) {
  __shared__ int s_lo[BSC_RUNS], s_pre[BSC_RUNS + 1];  // start of each column run in the sorted order, prefix sums of their lengths
  __shared__ unsigned s_num_lo[BSC_MAX_CELLS], s_num_hi[BSC_MAX_CELLS];   // 64-bit fixed-point sums as two 32-bit words:
  __shared__ unsigned s_dep_lo[BSC_MAX_CELLS], s_dep_hi[BSC_MAX_CELLS];   // native 32-bit shared atomics + explicit carry
  __shared__ float s_depth[BSC_MAX_CELLS], s_npw[BSC_MAX_CELLS];
  __shared__ double s_red[10 * (BSC_T / 32)];
  __shared__ double s_c[4];            // centroid, weight sum
  __shared__ float s_M[12];            // rows of the change of frame: x' = M[0..2].p + M[3] ...
  __shared__ double s_stat[3][4];      // per plane: mean / sd of the depth and of the density differences
  __shared__ int s_cnt;
  const GridArgs &g = a.g;
  const int q = blockIdx.x, tid = threadIdx.x;
  const int p = a.kp[q];
  const int side = a.side, S2 = side * side, cells = 3 * S2, nbits = 9 * S2;
  const float qx = g.xyz[3 * (size_t)p], qy = g.xyz[3 * (size_t)p + 1], qz = g.xyz[3 * (size_t)p + 2];
  if (tid < BSC_RUNS) {   // one contiguous run of the sorted points per grid column (x, y): its cells z - 1 .. z + 1
    const int cx = cell_coord(qx, g.mnx, g.inv) + tid / 3 - 1, cy = cell_coord(qy, g.mny, g.inv) + tid % 3 - 1;
    int lo = 0, hi = 0;   // a non-finite keypoint walks nothing: fewer than 3 neighbours below
    if (cx >= 0 && cy >= 0 && finite3(qx, qy, qz)) column_run(g, cx, cy, cell_coord(qz, g.mnz, g.inv), lo, hi);
    s_lo[tid] = lo; s_pre[tid + 1] = hi - lo;
  }
  for (int c = tid; c < cells; c += BSC_T) { s_num_lo[c] = 0u; s_num_hi[c] = 0u; s_dep_lo[c] = 0u; s_dep_hi[c] = 0u; }
  __syncthreads();
  if (tid == 0) { s_pre[0] = 0; for (int c = 0; c < BSC_RUNS; ++c) s_pre[c + 1] += s_pre[c]; }
  __syncthreads();
  const int total = s_pre[BSC_RUNS];   // candidates of this keypoint; every pass walks them flat, 128 at a time
  const double radius = sqrt(2.0) * (double)a.R;   // :956
  // ---- pass A: count, centroid sums, weight sum (:956-966) ----
  {
    double v[5] = {0, 0, 0, 0, 0};
    for (int idx = tid, c = 0; idx < total; idx += BSC_T) {
      while (idx >= s_pre[c + 1]) ++c;
      const float4 pt = g.sorted[s_lo[c] + (idx - s_pre[c])];
      const float x = pt.x, y = pt.y, z = pt.z;
      const float ex = x - qx, ey = y - qy, ez = z - qz;
      const float d2 = ex * ex + ey * ey + ez * ez;
      if (!(d2 < g.r2)) continue;
      v[0] += 1.0; v[1] += (double)x; v[2] += (double)y; v[3] += (double)z;
      v[4] += radius - (double)sqrtf(d2);
    }
    block_sum<5, BSC_T>(v, s_red);
    if (tid == 0) {
      s_cnt = (int)v[0];
      s_c[0] = v[1] / v[0]; s_c[1] = v[2] / v[0]; s_c[2] = v[3] / v[0]; s_c[3] = v[4];
    }
    __syncthreads();
  }
  const int cnt = s_cnt;
  if (cnt < 3) {   // the reference reads uninitialised axes here (:952): descriptor left zero, status 1
    for (int b = tid; b < a.V * a.nbytes; b += BSC_T) a.bits[((size_t)(b / a.nbytes) * a.nkp + q) * a.nbytes + b % a.nbytes] = 0;
    if (tid == 0) {
      if (a.status) a.status[q] = 1;
      if (a.lrf) { for (int c = 0; c < 9; ++c) a.lrf[12 * (size_t)q + c] = 0.f; a.lrf[12 * (size_t)q + 9] = qx; a.lrf[12 * (size_t)q + 10] = qy; a.lrf[12 * (size_t)q + 11] = qz; }
    }
    return;
  }
  // ---- pass B: weighted covariance about the centroid (:972-990) ----
  {
    double v[6] = {0, 0, 0, 0, 0, 0};
    const double cx = s_c[0], cy = s_c[1], cz = s_c[2];
    for (int idx = tid, c = 0; idx < total; idx += BSC_T) {
      while (idx >= s_pre[c + 1]) ++c;
      const float4 pt = g.sorted[s_lo[c] + (idx - s_pre[c])];
      const float x = pt.x, y = pt.y, z = pt.z;
      const float ex = x - qx, ey = y - qy, ez = z - qz;
      const float d2 = ex * ex + ey * ey + ez * ez;
      if (!(d2 < g.r2)) continue;
      const float weight = (float)(radius - (double)sqrtf(d2));
      const double dx = (double)x - cx, dy = (double)y - cy, dz = (double)z - cz, w = (double)weight;
      v[0] += w * dx * dx; v[1] += w * dx * dy; v[2] += w * dx * dz; v[3] += w * dy * dy; v[4] += w * dy * dz; v[5] += w * dz * dz;
    }
    block_sum<6, BSC_T>(v, s_red);
    if (tid == 0) {
      const float da = (float)s_c[3];
      const float c00 = (float)v[0] / da, c01 = (float)v[1] / da, c02 = (float)v[2] / da, c11 = (float)v[3] / da,
                  c12 = (float)v[4] / da, c22 = (float)v[5] / da;
      double A[3][3] = {{c00, c01, c02}, {c01, c11, c12}, {c02, c12, c22}}, Vv[3][3], w[3];
      bsc_jacobi3(A, Vv, w);
      const float ev[3] = {(float)w[0], (float)w[1], (float)w[2]};
      int imax = 0, imin = 0;
      float vmax = ev[0], vmin = ev[0];
      for (int i = 0; i < 3; ++i) {   // :998-1012
        if (ev[i] > vmax) { imax = i; vmax = ev[i]; }
        if (ev[i] < vmin) { imin = i; vmin = ev[i]; }
      }
      float principal[3], normal[3], ax[3], ay[3], az[3];
      for (int i = 0; i < 3; ++i) { principal[i] = (float)Vv[i][imax]; normal[i] = (float)Vv[i][imin]; }
      bsc_cross(principal, normal, ay);                 // middle direction :1022
      for (int i = 0; i < 3; ++i) ax[i] = principal[i];
      bsc_cross(ax, ay, az);                            // :148, before the normalisation
      bsc_normalize(ax); bsc_normalize(ay);             // :155-156
      if (a.lrf) {
        float *o = a.lrf + 12 * (size_t)q;
        for (int c = 0; c < 3; ++c) { o[c] = ax[c]; o[3 + c] = ay[c]; o[6 + c] = az[c]; }
        o[9] = qx; o[10] = qy; o[11] = qz;
      }
      if (a.status) a.status[q] = 0;
      // :1085-1138 — PCL's float32 Umeyama of the unit axes onto (ax, ay, az), the way the hot path's solve does it
      // (points (1,0,0), (0,1,0), (0,0,1) -> ax, ay, az; float32 means, demeaned products, 1/n), then the inverse
      const float third = 1.0f / 3.0f;
      float mu_s[3], mu_d[3], sigma[9];
      {
        float ms[3] = {0.f, 0.f, 0.f}, md[3] = {0.f, 0.f, 0.f};
        const float S[3][3] = {{1.f, 0.f, 0.f}, {0.f, 1.f, 0.f}, {0.f, 0.f, 1.f}};
        const float *D[3] = {ax, ay, az};
        for (int i = 0; i < 3; ++i) for (int c = 0; c < 3; ++c) { ms[c] += S[i][c]; md[c] += D[i][c]; }
        for (int c = 0; c < 3; ++c) { mu_s[c] = ms[c] * third; mu_d[c] = md[c] * third; }
        float acc[9] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        for (int i = 0; i < 3; ++i) {
          const float ds[3] = {S[i][0] - mu_s[0], S[i][1] - mu_s[1], S[i][2] - mu_s[2]};
          const float dd[3] = {D[i][0] - mu_d[0], D[i][1] - mu_d[1], D[i][2] - mu_d[2]};
          for (int r = 0; r < 3; ++r) for (int c = 0; c < 3; ++c) acc[r * 3 + c] += dd[r] * ds[c];
        }
        for (int k = 0; k < 9; ++k) sigma[k] = third * acc[k];
      }
      double Rt[16];
      umeyama_from_moments_f32(mu_s, mu_d, sigma, Rt);
      float M[16], Mi[16];
      for (int k = 0; k < 16; ++k) M[k] = (float)Rt[k];
      bsc_inverse4(M, Mi);
      for (int r = 0; r < 3; ++r) { s_M[4 * r] = Mi[r]; s_M[4 * r + 1] = Mi[4 + r]; s_M[4 * r + 2] = Mi[8 + r]; s_M[4 * r + 3] = Mi[12 + r]; }
    }
    __syncthreads();
  }
  // ---- pass C: the three projected grids (:197-310) ----
  const float R = a.R;
  const float unit = 2 * R / side;                                  // :72
  const float delta = (float)(unit * 0.5);                          // :205
  const float two_dd = 2 * delta * delta;
  const float rc = (float)(1.5 * unit), rc2 = rc * rc;              // search radius of a cell centre, squared like S4
  const double dep_scale = 1099511627776.0 / (double)R;             // 2^40 / R: depth * w / R in fixed point
  {
    const float m00 = s_M[0], m01 = s_M[1], m02 = s_M[2], m03 = s_M[3], m10 = s_M[4], m11 = s_M[5], m12 = s_M[6], m13 = s_M[7],
                m20 = s_M[8], m21 = s_M[9], m22 = s_M[10], m23 = s_M[11];
    for (int idx = tid, c = 0; idx < total; idx += BSC_T) {
        while (idx >= s_pre[c + 1]) ++c;
        const float4 pt = g.sorted[s_lo[c] + (idx - s_pre[c])];
        const float ex = pt.x - qx, ey = pt.y - qy, ez = pt.z - qz;
        const float d2 = ex * ex + ey * ey + ez * ez;
        if (!(d2 < g.r2)) continue;
        float loc[3];
        loc[0] = m00 * ex + m01 * ey + m02 * ez + m03;              // :193, rows summed left to right
        loc[1] = m10 * ex + m11 * ey + m12 * ez + m13;
        loc[2] = m20 * ex + m21 * ey + m22 * ez + m23;
#pragma unroll
        for (int pl = 0; pl < 3; ++pl) {
          const float u = loc[pl == 2 ? 1 : 0], v = loc[pl == 0 ? 1 : 2];
          const float depth = loc[pl == 0 ? 2 : (pl == 1 ? 1 : 0)] + R;   // :240, :274, :308
          // centres within 1.5 cell edges of u are among i0 - 1 .. i0 + 2, i0 = the cell row whose centre is just below u
          // (half a cell of margin against the rounding of this index; the float32 test below is the reference's)
          const int i0 = (int)floorf((u + R) / unit - 0.5f), j0 = (int)floorf((v + R) / unit - 0.5f);
#pragma unroll 1
          for (int i = (i0 - 1 < 0 ? 0 : i0 - 1); i <= i0 + 2 && i < side; ++i) {
            const float cu = (float)((i + 0.5) * unit - R);          // :226
            const float du = u - cu;
#pragma unroll 1
            for (int j = (j0 - 1 < 0 ? 0 : j0 - 1); j <= j0 + 2 && j < side; ++j) {
              const float cv = (float)((j + 0.5) * unit - R);
              const float dv = v - cv;
              const float dd = du * du + dv * dv;
              if (!(dd < rc2)) continue;
              const float wgt = (float)exp((double)(-dd / two_dd));  // :238 exp(float): rounded-to-nearest float32 exponential
              const int cell = i + j * side + pl * S2;
              bsc_add64(&s_num_lo[cell], &s_num_hi[cell], (unsigned long long)((double)wgt * 1099511627776.0));
              bsc_add64(&s_dep_lo[cell], &s_dep_hi[cell], (unsigned long long)__double2ll_rn((double)depth * (double)wgt * dep_scale));
            }
          }
        }
      }
  }
  __syncthreads();
  // ---- cells (:341-373) ----
  {
    const float area_n = (float)(3.14159265358979323846 * R * R);    // :346
    const float dens_n = (float)cnt / area_n;                        // :347
    const float area_g = unit * unit;
    for (int c = tid; c < cells; c += BSC_T) {
      const double num = (double)(((unsigned long long)s_num_hi[c] << 32) | s_num_lo[c]) * (1.0 / 1099511627776.0);
      const long long dep_fx = (long long)(((unsigned long long)s_dep_hi[c] << 32) | s_dep_lo[c]);
      float depth = 0.f;
      if (num != 0.0) depth = (float)(((double)dep_fx / dep_scale) / num);
      const float dens_g = (float)(num / (double)area_g);
      s_depth[c] = depth;
      s_npw[c] = (dens_n != 0.0f) ? dens_g / dens_n : 0.f;
    }
  }
  __syncthreads();
  // ---- per plane statistics of the pair differences (:498-527), one thread per plane, the reference's summation order ----
  if (tid < 3) {
    const int off = tid * S2;
    double mean_dep = 0.0, mean_den = 0.0, var_dep = 0.0, var_den = 0.0;
    for (int i = 0; i < S2; ++i) {
      mean_dep += (double)(s_depth[a.pairs[2 * i] + off] - s_depth[a.pairs[2 * i + 1] + off]);
      mean_den += (double)(s_npw[a.pairs[2 * i] + off] - s_npw[a.pairs[2 * i + 1] + off]);
    }
    mean_dep /= S2; mean_den /= S2;
    for (int i = 0; i < S2; ++i) {
      const double dep = (double)(s_depth[a.pairs[2 * i] + off] - s_depth[a.pairs[2 * i + 1] + off]);
      const double den = (double)(s_npw[a.pairs[2 * i] + off] - s_npw[a.pairs[2 * i + 1] + off]);
      var_dep += (dep - mean_dep) * (dep - mean_dep);
      var_den += (den - mean_den) * (den - mean_den);
    }
    s_stat[tid][0] = mean_dep; s_stat[tid][1] = sqrt(var_dep / S2); s_stat[tid][2] = mean_den; s_stat[tid][3] = sqrt(var_den / S2);
  }
  __syncthreads();
  // ---- bits: one thread per output byte ----
  const float T = 0.1f;
  for (int b = tid; b < a.V * a.nbytes; b += BSC_T) {
    const int v = b / a.nbytes, byte = b % a.nbytes;
    unsigned out = 0;
    for (int bit = 0; bit < 8; ++bit) {
      const int k = 8 * byte + bit;
      if (k >= nbits) break;
      bool on = false;
      if (v == 0) {
        if (k < cells) on = s_npw[k] > T;
        else {
          const int kk = k - cells, pl = kk / (2 * S2), r = kk % (2 * S2), i = r >> 1, off = pl * S2;
          const int pa = a.pairs[2 * i], pb = a.pairs[2 * i + 1];
          if ((r & 1) == 0) {
            const double dep = (double)(s_depth[pa + off] - s_depth[pb + off]);
            on = fabs(dep - s_stat[pl][0]) > s_stat[pl][1];          // :531
          } else if (!(s_npw[pa] < T && s_npw[pb] < T)) {             // :544 looks at the first plane whatever the plane
            const double den = (double)(s_npw[pa + off] - s_npw[pb + off]);
            on = fabs(den - s_stat[pl][2]) > s_stat[pl][3];          // :551
          }
        }
      } else if (k >= cells && k < 2 * cells) {                       // the appended re-arranged grid's occupancy bits
        const int kk = k - cells, pl = kk / S2;
        const int tr = (v == 1) ? (pl == 0 ? 1 : 2) : (v == 2 ? (pl == 0 ? 3 : (pl == 1 ? 2 : 1)) : (pl == 0 ? 2 : (pl == 1 ? 1 : 3)));   // :789, :804, :813
        on = s_npw[pl * S2 + bsc_rearranged(tr, kk % S2, side)] > T;
      }
      if (on) out |= 1u << bit;
    }
    a.bits[((size_t)v * a.nkp + q) * a.nbytes + byte] = (unsigned char)out;
  }
}

}  // namespace

// BSCEncoder::extractBinaryFeatures on device arrays.  d_kp [nkp] keypoint indices into d_xyz [n][3]; d_pairs [side^2][2];
// d_bits [V][nkp][ceil(9 side^2 / 8)] with V = 1 (dof_type 0), 2 (1..4), 4 (> 4); d_lrf [nkp][12] and d_status [nkp] may be null.
cudaError_t prep_bsc_extract(cudaStream_t st, const float *d_xyz, int n, const int *d_kp, int nkp, float R, int side,
                             const int *d_pairs, int dof_type, unsigned char *d_bits, float *d_lrf, int *d_status) {
  GridArgs g{};
  GridBufs grid;
  if (n <= 0 || nkp <= 0) return cudaSuccess;
  if (side < 1 || side > BSC_MAX_SIDE) return cudaErrorInvalidValue;
  const float search = (float)(sqrt(3.0) * (double)R);            // :643; squared in float32 like the radius of S4
  CUDA_TRY(build_grid(st, d_xyz, nullptr, n, search, &g, &grid));
  BscArgs a{};
  a.g = g; a.kp = d_kp; a.nkp = nkp; a.R = R; a.side = side; a.pairs = d_pairs;
  a.V = dof_type > 4 ? 4 : (dof_type > 0 ? 2 : 1);
  a.bits = d_bits; a.nbytes = (9 * side * side + 7) / 8; a.lrf = d_lrf; a.status = d_status;
  GHICP_LAUNCH(k_bsc, nkp, BSC_T, 0, st, a);
  CUDA_TRY(cudaStreamSynchronize(st));
  return cudaGetLastError();
}

// =====================================================================================================================
// FPFH estimator (DESIGN.md §3.10): FPFHfeature::compute_fpfh_feature + keyfpfh of the reference's driver
// (test/ghicp_main.cpp:120-127; include/fpfh.hpp:36-115 = PCL NormalEstimation + FPFHEstimationOMP, both k-NN with k = 20).
// PCL is not pinned, so the definition is the canonical one restated in tests/harness/fpfh_oracle.cpp; these kernels and
// that oracle agree bit for bit (k-NN lists, normals) and up to the double atan2 of the device math library (histograms).
//   k_knn      exact k nearest neighbours of every point, ascending (d2, index): rings of grid columns outward from the
//              query's cell (ring_walk; a column's z-range is one contiguous run of the cell-sorted points), stopped once the k-th
//              distance is below a conservative bound on every unvisited cell, exhaustive scan past FPFH_RING_CAP rings
//   k_normals  covariance of the k neighbours (k_pca's double sums), smallest eigenvector (bsc_jacobi3), flip to the origin
//   k_spfh     3 x 11 bin SPFH of every point a requested histogram reads (all points for the whole-cloud call)
//   k_fpfh     the 1 / d2 weighted sum of the neighbours' SPFH, each block normalised to 100 (own SPFH not added)
// =====================================================================================================================
namespace {

constexpr int FPFH_KMAX = 32;       // largest k: the top-k list lives in registers
constexpr int FPFH_RING_CAP = 4;    // a query not settled after this many rings scans the whole cloud (far outliers)

struct KnnArgs {
  RingGrid rg;
  int n, k;                         // k = k_eff = min(k, n)
  int *nb_idx; float *nb_d2;        // [n][k]
  unsigned long long *cand;         // candidates examined, summed over all queries
  int *fallbacks;                   // queries that took the exhaustive scan
  int *deferred, *n_deferred;       // optional: such queries are listed here instead (rows not written), for a wider scan
};

__global__ void k_knn(const KnnArgs a) {
  __shared__ unsigned long long s_cand;
  __shared__ int s_fb;
  if (threadIdx.x == 0) { s_cand = 0ull; s_fb = 0; }
  __syncthreads();
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < a.n) {
    const GridArgs &g = a.rg.g;
    const GridRegs r = grid_regs(g);     // per-thread registers, see k_pca
    const int i = r.order[t];            // threads of a warp take points of the same cell (see k_pca)
    const float qx = g.xyz[3 * (size_t)i], qy = g.xyz[3 * (size_t)i + 1], qz = g.xyz[3 * (size_t)i + 2];
    const int k = a.k;
    if (!finite3(qx, qy, qz)) {   // a non-finite point's list is itself at distance 0: an isolated point's zero histogram
      for (int j = 0; j < k; ++j) { a.nb_idx[(size_t)i * k + j] = i; a.nb_d2[(size_t)i * k + j] = 0.f; }
    } else {
      const int cx = cell_coord(qx, g.mnx, g.inv), cy = cell_coord(qy, g.mny, g.inv), cz = cell_coord(qz, g.mnz, g.inv);
      pu64 key[FPFH_KMAX];
#pragma unroll
      for (int j = 0; j < FPFH_KMAX; ++j) key[j] = (j < FPFH_KMAX - k) ? 0ull : ~0ull;
      long long cand = 0;
      const bool done = ring_walk(r, a.rg, cx, cy, cz, FPFH_RING_CAP,
          [&](int s0, int s1) {
            cand += s1 - s0;
            for (int s = s0; s < s1; ++s) knn_insert(key, knn_key(knn_d2(qx, qy, qz, r.sorted[s]), r.order[s]));
          },
          [&] { return key[FPFH_KMAX - 1] == ~0ull ? (double)INFINITY : (double)knn_key_d2(key[FPFH_KMAX - 1]); });
      if (!done) {   // far outlier (or a grid too fine for this cloud): exact by exhaustion
        atomicAdd(&s_fb, 1);
        if (a.deferred) {
          a.deferred[atomicAdd(a.n_deferred, 1)] = i;
        } else {
#pragma unroll
          for (int j = 0; j < FPFH_KMAX; ++j) key[j] = (j < FPFH_KMAX - k) ? 0ull : ~0ull;
          for (int s = 0; s < a.n; ++s) knn_insert(key, knn_key(knn_d2(qx, qy, qz, r.sorted[s]), r.order[s]));
          cand += a.n;
        }
      }
#pragma unroll
      for (int j = 0; j < FPFH_KMAX; ++j) {
        const int jj = j - (FPFH_KMAX - k);
        if (jj >= 0 && (done || !a.deferred)) {
          a.nb_idx[(size_t)i * k + jj] = (int)(unsigned)key[j];
          a.nb_d2[(size_t)i * k + jj] = knn_key_d2(key[j]);
        }
      }
      atomicAdd(&s_cand, (unsigned long long)cand);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) { atomicAdd(a.cand, s_cand); atomicAdd(a.fallbacks, s_fb); }
}

// Neighbour lists the estimator reads.  The normal, SPFH and FPFH arithmetic below is written once, over a list accessor:
//   FixedLists  the k-NN lists, [n][k] (k_knn)
//   CsrLists    the radius lists (k_rad_fill + segmented sort): row[point] -> 64-bit offsets into knn_key entries
// list(i) gives the first entry of point i's list and its length; id / dist2 read entry e.
struct FixedLists {
  const int *idx; const float *d2; int k;
  __device__ __forceinline__ size_t first(size_t i) const { return i * (size_t)k; }
  __device__ __forceinline__ int count(size_t) const { return k; }
  __device__ __forceinline__ int id(size_t e) const { return idx[e]; }
  __device__ __forceinline__ float dist2(size_t e) const { return d2[e]; }
};
struct CsrLists {
  const pu64 *key; const long long *off; const int *row;
  __device__ __forceinline__ size_t first(size_t i) const { return (size_t)off[row[i]]; }
  __device__ __forceinline__ int count(size_t i) const { const int r = row[i]; return (int)(off[r + 1] - off[r]); }
  __device__ __forceinline__ int id(size_t e) const { return (int)(unsigned)key[e]; }
  __device__ __forceinline__ float dist2(size_t e) const { return knn_key_d2(key[e]); }
};

// NormalEstimation::computePointNormal + flipNormalTowardsViewpoint (viewpoint 0) of point i over its list; a non-finite point
// (whose list is not read) or one with fewer than 3 neighbours gets a NaN normal and status 1
template <class L>
__device__ __forceinline__ void est_normal(const float *__restrict__ xyz, int i, const L &l, float *__restrict__ nrm,
                                           int *__restrict__ status) {
  const float qx = xyz[3 * (size_t)i], qy = xyz[3 * (size_t)i + 1], qz = xyz[3 * (size_t)i + 2];
  const bool fin = finite3(qx, qy, qz);
  const int k = fin ? l.count((size_t)i) : 0;
  const size_t b = fin ? l.first((size_t)i) : 0;
  if (k < 3) {
    const float nan = __uint_as_float(0x7fc00000u);
    nrm[3 * (size_t)i] = nan; nrm[3 * (size_t)i + 1] = nan; nrm[3 * (size_t)i + 2] = nan;
    if (status) status[i] = 1;
    return;
  }
  double sd[3] = {0, 0, 0}, sdd[6] = {0, 0, 0, 0, 0, 0};
  for (int j = 0; j < k; ++j) {   // list order; the sums of k_pca
    const size_t p = (size_t)l.id(b + j);
    const float ex = xyz[3 * p] - qx, ey = xyz[3 * p + 1] - qy, ez = xyz[3 * p + 2] - qz;
    const double a = ex, b = ey, c = ez;
    sd[0] += a; sd[1] += b; sd[2] += c;
    sdd[0] += a * a; sdd[1] += a * b; sdd[2] += a * c; sdd[3] += b * b; sdd[4] += b * c; sdd[5] += c * c;
  }
  const double inv_n = 1.0 / k, alpha = 1.0 / (k - 1);
  const float cv[6] = {(float)((sdd[0] - sd[0] * sd[0] * inv_n) * alpha), (float)((sdd[1] - sd[0] * sd[1] * inv_n) * alpha),
                       (float)((sdd[2] - sd[0] * sd[2] * inv_n) * alpha), (float)((sdd[3] - sd[1] * sd[1] * inv_n) * alpha),
                       (float)((sdd[4] - sd[1] * sd[2] * inv_n) * alpha), (float)((sdd[5] - sd[2] * sd[2] * inv_n) * alpha)};
  double A[3][3] = {{cv[0], cv[1], cv[2]}, {cv[1], cv[3], cv[4]}, {cv[2], cv[4], cv[5]}}, V[3][3], w[3];
  bsc_jacobi3(A, V, w);
  int jm = 0;                     // smallest eigenvalue, first index on ties
  if (w[1] < w[jm]) jm = 1;
  if (w[2] < w[jm]) jm = 2;
  const double vx = V[0][jm], vy = V[1][jm], vz = V[2][jm];
  const double len = sqrt((vx * vx + vy * vy) + vz * vz);
  float nx = (float)(vx / len), ny = (float)(vy / len), nz = (float)(vz / len);
  if (((-qx) * nx + (-qy) * ny) + (-qz) * nz < 0.f) { nx = -nx; ny = -ny; nz = -nz; }
  nrm[3 * (size_t)i] = nx; nrm[3 * (size_t)i + 1] = ny; nrm[3 * (size_t)i + 2] = nz;
  if (status) status[i] = 0;
}

// k-NN normals: one thread per point
__global__ void k_normals(const float *__restrict__ xyz, const int *__restrict__ nb_idx, int n, int k, float *__restrict__ nrm,
                          int *__restrict__ status) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  est_normal(xyz, i, FixedLists{nb_idx, nullptr, k}, nrm, status);
}

// points whose SPFH a requested histogram reads: the neighbours of every requested index
__global__ void k_fpfh_mark(const int *__restrict__ idx, int nidx, const int *__restrict__ nb_idx, int k, int *__restrict__ need) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nidx) return;
  const size_t p = (size_t)idx[t];
  for (int j = 0; j < k; ++j) need[nb_idx[p * k + j]] = 1;
}

// Float operation order of the pair features — the same text in tests/harness/fpfh_oracle.cpp:
//   dot(a, b)   = (a.x*b.x + a.y*b.y) + a.z*b.z
//   cross(a, b) = (a.y*b.z - a.z*b.y, a.z*b.x - a.x*b.z, a.x*b.y - a.y*b.x)
//   |a|         = sqrtf(dot(a, a)),  a / |a| = three divisions
__device__ __forceinline__ float f3dot(const float a[3], const float b[3]) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }
__device__ __forceinline__ void f3cross(const float a[3], const float b[3], float o[3]) {
  o[0] = a[1] * b[2] - a[2] * b[1];
  o[1] = a[2] * b[0] - a[0] * b[2];
  o[2] = a[0] * b[1] - a[1] * b[0];
}
__device__ __forceinline__ int fpfh_bin(double x) {   // x = the feature mapped to [0, 1]
  int h = (int)floor(11 * x);
  return h < 0 ? 0 : (h > 10 ? 10 : h);
}

// computePointSPFHSignature of point i over its list (the increments are all equal: the bins do not depend on list order)
template <class L>
__device__ __forceinline__ void est_spfh(const float *__restrict__ xyz, const float *__restrict__ nrm, int i, const L &l,
                                         float *__restrict__ spfh) {
  const int k = l.count((size_t)i);
  const size_t e0 = l.first((size_t)i);
  float hist[33];
  for (int b = 0; b < 33; ++b) hist[b] = 0.f;
  const float np[3] = {nrm[3 * (size_t)i], nrm[3 * (size_t)i + 1], nrm[3 * (size_t)i + 2]};
  if (k > 1 && np[0] == np[0]) {   // a NaN normal (fewer than 3 neighbours) takes part in no pair
    const float hist_incr = 100.0f / (float)(k - 1);
    const float inv2pi = 1.0f / (2.0f * 3.14159265358979323846f);
    const float p[3] = {xyz[3 * (size_t)i], xyz[3 * (size_t)i + 1], xyz[3 * (size_t)i + 2]};
    for (int j = 0; j < k; ++j) {
      const int qi = l.id(e0 + j);
      if (qi == i) continue;
      const float nq[3] = {nrm[3 * (size_t)qi], nrm[3 * (size_t)qi + 1], nrm[3 * (size_t)qi + 2]};
      if (nq[0] != nq[0]) continue;
      float dp[3] = {xyz[3 * (size_t)qi] - p[0], xyz[3 * (size_t)qi + 1] - p[1], xyz[3 * (size_t)qi + 2] - p[2]};
      const float f4 = sqrtf(f3dot(dp, dp));
      if (f4 == 0.f) continue;
      const float a1 = f3dot(np, dp) / f4, a2 = f3dot(nq, dp) / f4;
      float u[3], other[3], f3;
      if (fabsf(a1) < fabsf(a2)) {   // PCL's acos(|a1|) > acos(|a2|): the frame sits on q
        for (int c = 0; c < 3; ++c) { u[c] = nq[c]; other[c] = np[c]; dp[c] = -dp[c]; }
        f3 = -a2;
      } else {
        for (int c = 0; c < 3; ++c) { u[c] = np[c]; other[c] = nq[c]; }
        f3 = a1;
      }
      float v[3], w[3];
      f3cross(dp, u, v);
      const float vn = sqrtf(f3dot(v, v));
      if (vn == 0.f) continue;
      v[0] = v[0] / vn; v[1] = v[1] / vn; v[2] = v[2] / vn;
      f3cross(u, v, w);
      const float f2 = f3dot(v, other);
      const float f1 = (float)atan2((double)f3dot(w, other), (double)f3dot(u, other));
      hist[fpfh_bin(((double)f1 + 3.14159265358979323846) * (double)inv2pi)] += hist_incr;
      hist[11 + fpfh_bin(((double)f2 + 1.0) * 0.5)] += hist_incr;
      hist[22 + fpfh_bin(((double)f3 + 1.0) * 0.5)] += hist_incr;
    }
  }
  for (int b = 0; b < 33; ++b) spfh[(size_t)i * 33 + b] = hist[b];
}

// k-NN SPFH: one thread per needed point
__global__ void k_spfh(const float *__restrict__ xyz, const float *__restrict__ nrm, const int *__restrict__ nb_idx, int n, int k,
                       const int *__restrict__ need, float *__restrict__ spfh) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || (need && !need[i])) return;
  est_spfh(xyz, nrm, i, FixedLists{nb_idx, nullptr, k}, spfh);
}

// weightPointSPFHSignature of point p over its list into out [33]: float per-bin sums and double per-block sums in list order
template <class L>
__device__ __forceinline__ void est_fpfh(size_t p, const L &l, const float *__restrict__ spfh, float *__restrict__ out) {
  const int k = l.count(p);
  const size_t e0 = l.first(p);
  float hist[33];
  double sum[3] = {0.0, 0.0, 0.0};
#pragma unroll
  for (int b = 0; b < 33; ++b) hist[b] = 0.f;
  for (int j = 0; j < k; ++j) {
    const float d2 = l.dist2(e0 + j);
    if (d2 == 0.f) continue;                       // the point itself and its duplicates
    const float wgt = 1.0f / d2;
    const float *sq = spfh + (size_t)l.id(e0 + j) * 33;
#pragma unroll
    for (int b = 0; b < 33; ++b) {
      const float val = sq[b] * wgt;
      hist[b] += val;
      sum[b / 11] += (double)val;
    }
  }
#pragma unroll
  for (int b = 0; b < 33; ++b) {
    const float h = sum[b / 11] != 0.0 ? hist[b] * (float)(100.0 / sum[b / 11]) : hist[b];
    out[b] = h;
  }
}

// k-NN FPFH: one thread per requested index
__global__ void k_fpfh(const int *__restrict__ idx, int nidx, const int *__restrict__ nb_idx, const float *__restrict__ nb_d2, int k,
                       const float *__restrict__ spfh, float *__restrict__ out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nidx) return;
  est_fpfh((size_t)(idx ? idx[t] : t), FixedLists{nb_idx, nb_d2, k}, spfh, out + (size_t)t * 33);
}

// ---- radius neighbourhoods (DESIGN.md §3.10, "Radius neighbourhoods") ------------------------------------------------------
// N_r(p) = every q with d2(p, q) < r2 (knn_d2, r2 = r*r in float32), ascending (d2, index).  A query walks the columns
// (x, y) within `rings` cells of its own, each column's z-range cz - rings .. cz + rings being one run of the cell-sorted
// points.  rings = ceil(r / cell + slack) covers the float32 rounding of cell_coord, so the lists are exact.
struct RadWalk {
  GridArgs g;
  int rings; float r2;
};

// calls f(sorted position, d2) for every point of N_r(q) in walk order (not sorted); N_r of a non-finite q is empty
template <class F>
__device__ __forceinline__ void rad_walk(const GridRegs &r, const RadWalk &w, float qx, float qy, float qz, F &&f) {
  if (!finite3(qx, qy, qz)) return;
  const int cx = cell_coord(qx, w.g.mnx, w.g.inv), cy = cell_coord(qy, w.g.mny, w.g.inv), cz = cell_coord(qz, w.g.mnz, w.g.inv);
  const int R = w.rings, zlo = max(cz - R, 0), zhi = cz + R;
  for (int x = max(cx - R, 0); x <= cx + R; ++x)
    for (int y = max(cy - R, 0); y <= cy + R; ++y) {
      const int s0 = r.cstart[lower_cell(r, cell_key(x, y, zlo))], s1 = r.cstart[lower_cell(r, cell_key(x, y, zhi) + 1)];
      for (int s = s0; s < s1; ++s) {
        const float d2 = knn_d2(qx, qy, qz, r.sorted[s]);
        if (d2 < r.r2) f(s, d2);
      }
    }
}

// need[q] = 1 for every q in N_r(idx[t]) (the points whose SPFH the requested histograms read) and for idx[t] itself, which
// gives every requested point a list row (an empty one when it is not finite; a finite point is in its own N_r anyway)
__global__ void k_rad_mark(const RadWalk w, const int *__restrict__ idx, int nidx, int *__restrict__ need) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nidx) return;
  GridRegs r = grid_regs(w.g);   // per-thread registers, see k_pca
  r.r2 = w.r2;
  const float *q = w.g.xyz + 3 * (size_t)idx[t];
  need[idx[t]] = 1;
  rad_walk(r, w, q[0], q[1], q[2], [&](int s, float) { need[r.order[s]] = 1; });
}
// need[q] = 1 for every entry of the lists of rows [0, m)
__global__ void k_list_mark(const pu64 *__restrict__ key, const long long *__restrict__ off, int m, int *__restrict__ need) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= m) return;
  for (long long e = off[t]; e < off[t + 1]; ++e) need[(unsigned)key[e]] = 1;
}
// rows in cell order (warps walk the same columns): flags[s] = need[order[s]] (every point when need == nullptr), flags[n] = 0
__global__ void k_row_flags(const int *__restrict__ order, const int *__restrict__ need, int n, int *__restrict__ flags) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s > n) return;
  flags[s] = s < n && (!need || need[order[s]]) ? 1 : 0;
}
// rows[pos[s]] = order[s], row_of[order[s]] = pos[s] for the flagged positions (row_of holds -1 elsewhere)
__global__ void k_row_emit(const int *__restrict__ order, const int *__restrict__ flags, const int *__restrict__ pos, int n,
                           int *__restrict__ rows, int *__restrict__ row_of) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n || !flags[s]) return;
  rows[pos[s]] = order[s]; row_of[order[s]] = pos[s];
}
// |N_r(rows[t])| (cnt[m] = 0 so that the scan yields the total)
__global__ void k_rad_count(const RadWalk w, const int *__restrict__ rows, int m, long long *__restrict__ cnt) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t > m) return;
  if (t == m) { cnt[t] = 0; return; }
  GridRegs r = grid_regs(w.g);
  r.r2 = w.r2;
  const float *q = w.g.xyz + 3 * (size_t)rows[t];
  int c = 0;
  rad_walk(r, w, q[0], q[1], q[2], [&](int, float) { ++c; });
  cnt[t] = c;
}
// the entries knn_key(d2, q) of row t at off[t] .. off[t + 1], in walk order (the segmented sort orders them)
__global__ void k_rad_fill(const RadWalk w, const int *__restrict__ rows, int m, const long long *__restrict__ off,
                           pu64 *__restrict__ key) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= m) return;
  GridRegs r = grid_regs(w.g);
  r.r2 = w.r2;
  const float *q = w.g.xyz + 3 * (size_t)rows[t];
  pu64 *out = key + off[t];
  rad_walk(r, w, q[0], q[1], q[2], [&](int s, float d2) { *out++ = knn_key(d2, r.order[s]); });
}
// normals of every point: over its N_rn list where one was built (row_of >= 0), NaN with status 1 at a non-finite point, NaN
// with status 2 elsewhere
__global__ void k_rad_normals(const float *__restrict__ xyz, int n, const CsrLists l, float *__restrict__ nrm, int *__restrict__ status) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (l.row[i] >= 0 || !finite3(xyz[3 * (size_t)i], xyz[3 * (size_t)i + 1], xyz[3 * (size_t)i + 2])) {
    est_normal(xyz, i, l, nrm, status);
    return;
  }
  const float nan = __uint_as_float(0x7fc00000u);
  nrm[3 * (size_t)i] = nan; nrm[3 * (size_t)i + 1] = nan; nrm[3 * (size_t)i + 2] = nan;
  if (status) status[i] = 2;
}
// SPFH of the rows of the N_rf lists (one thread per row, rows in cell order)
__global__ void k_rad_spfh(const float *__restrict__ xyz, const float *__restrict__ nrm, const int *__restrict__ rows, int m,
                           const CsrLists l, float *__restrict__ spfh) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= m) return;
  est_spfh(xyz, nrm, rows[t], l, spfh);
}
__global__ void k_rad_fpfh(const int *__restrict__ idx, int nidx, const CsrLists l, const float *__restrict__ spfh, float *__restrict__ out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= nidx) return;
  est_fpfh((size_t)(idx ? idx[t] : t), l, spfh, out + (size_t)t * 33);
}
// the chunks of a segmented sort: first row of chunk c = first row whose offset is >= c * chunk (bounds[nchunks] = m)
__global__ void k_chunk_bounds(const long long *__restrict__ off, int m, long long chunk, int nchunks, int *__restrict__ bounds) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c > nchunks) return;
  if (c == nchunks) { bounds[c] = m; return; }
  const long long want = c * chunk;
  int lo = 0, hi = m;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (off[mid] < want) lo = mid + 1; else hi = mid; }
  bounds[c] = lo;
}
// int offsets of rows r0 .. r1 relative to off[r0]
__global__ void k_rel_offsets(const long long *__restrict__ off, int r0, int r1, int *__restrict__ rel) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (r0 + t > r1) return;
  rel[t] = (int)(off[r0 + t] - off[r0]);
}

#if !defined(GHICP_EMU_HOST)
// CUB's segmented sort counts items in int: the rows are sorted in chunks of at most 2^30 entries plus one row
cudaError_t segmented_sort(const pu64 *in, pu64 *out, long long total, int m, const long long *off, cudaStream_t st) {
  constexpr long long CHUNK = 1ll << 30;
  const int nch = (int)((total + CHUNK - 1) / CHUNK);
  if (nch == 0) return cudaSuccess;
  DevBuf<int> d_bounds, rel; DevBuf<unsigned char> tmp;
  size_t tmp_bytes = 0;
  std::vector<int> bounds(nch + 1);
  CUDA_TRY(d_bounds.alloc((size_t)nch + 1)); CUDA_TRY(rel.alloc((size_t)m + 1));
  GHICP_LAUNCH(k_chunk_bounds, blocks(nch + 1), PT, 0, st, off, m, CHUNK, nch, d_bounds.get());
  CUDA_TRY(cudaMemcpyAsync(bounds.data(), d_bounds.get(), sizeof(int) * (nch + 1), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  for (int c = 0; c < nch; ++c) {
    const int r0 = bounds[c], r1 = bounds[c + 1];
    if (r1 <= r0) continue;
    long long lo = 0, hi = 0;
    CUDA_TRY(cudaMemcpyAsync(&lo, off + r0, sizeof(lo), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(&hi, off + r1, sizeof(hi), cudaMemcpyDeviceToHost, st)); CUDA_TRY(cudaStreamSynchronize(st));
    if (hi - lo > INT_MAX) return cudaErrorInvalidValue;   // one row of more than 2^31 - 2^30 entries
    GHICP_LAUNCH(k_rel_offsets, blocks(r1 - r0 + 1), PT, 0, st, off, r0, r1, rel.get());
    size_t need = 0;
    CUDA_TRY(cub::DeviceSegmentedSort::SortKeys(nullptr, need, in + lo, out + lo, (int)(hi - lo), r1 - r0, rel.get(), rel.get() + 1, st));
    if (need > tmp_bytes) {
      tmp_bytes = need;
      CUDA_TRY(tmp.alloc(tmp_bytes, st));
    }
    CUDA_TRY(cub::DeviceSegmentedSort::SortKeys(tmp.get(), need, in + lo, out + lo, (int)(hi - lo), r1 - r0, rel.get(), rel.get() + 1, st));
  }
  return cudaSuccess;
}
#endif

}  // namespace

// The grid of a ring search over d_xyz [n][3] (see PointGrid).
cudaError_t prep_point_grid(cudaStream_t st, const float *d_xyz, int n, int ke, float cell_scale, double min_cell, PointGrid *out) {
  GridArgs g{};
  GridBufs grid;
  float mn[3], mx[3];
  *out = PointGrid();
  if (n <= 0 || ke <= 0) return cudaErrorInvalidValue;
  CUDA_TRY(prep_bounds(st, d_xyz, n, mn, mx, &out->nfin));
  // Cell edge from the data: a volume guess (k points per cell if the cloud filled its box), then corrected once by the
  // observed mean occupancy of the occupied cells assuming a surface (occupancy ~ edge^2), aiming at 0.4 k per cell —
  // enough for the k nearest to lie within one ring.  The results do not depend on it; the work per query does.
  double ext[3], emax = 0.0;
  for (int a = 0; a < 3; ++a) { ext[a] = (double)mx[a] - (double)mn[a]; emax = ext[a] > emax ? ext[a] : emax; }
  double cell = 1.0;
  if (emax > 0.0) {
    double vol = 1.0;
    for (int a = 0; a < 3; ++a) vol *= ext[a] > 1e-3 * emax ? ext[a] : 1e-3 * emax;
    cell = cbrt(vol * ke / n);
    CUDA_TRY(build_grid(st, d_xyz, nullptr, n, (float)cell, &g, &grid));
    const double occ = (double)n / g.nu;
    double f = sqrt(0.4 * ke / occ);
    f = f < 1.0 / 16 ? 1.0 / 16 : (f > 16.0 ? 16.0 : f);
    cell *= f;
    grid = GridBufs();
  }
  if (cell_scale > 0.f) cell *= cell_scale;
  if (cell < min_cell) cell = min_cell;
  if (cell < emax / 1048576.0) cell = emax / 1048576.0;   // cell coordinates stay below 2^20 (21-bit key fields)
  CUDA_TRY(build_grid(st, d_xyz, nullptr, n, (float)cell, &g, &out->buf));
  RingGrid &G = out->rg;
  G.g = g;
  G.gm[0] = cell_coord_host(mx[0], g.mnx, g.inv); G.gm[1] = cell_coord_host(mx[1], g.mny, g.inv); G.gm[2] = cell_coord_host(mx[2], g.mnz, g.inv);
  for (int a = 0; a < 3; ++a) G.mx[a] = mx[a];
  G.cell = (double)(float)cell;
  const int gmax = G.gm[0] > G.gm[1] ? (G.gm[0] > G.gm[2] ? G.gm[0] : G.gm[2]) : (G.gm[1] > G.gm[2] ? G.gm[1] : G.gm[2]);
  G.slack = 0.01 + (gmax + 2.0) / 1048576.0;
  return cudaSuccess;
}
cudaError_t prep_sort_pairs(cudaStream_t st, pu64 *keys, int *vals, int n) { return sort_pairs(keys, vals, n, st); }

// FPFH histograms at d_idx [nidx] (all points when d_idx == nullptr) of the cloud d_xyz [n][3]; d_normals [n][3] receives
// every point's normal, d_status [n] (may be null) 1 where fewer than 3 neighbours exist or the point is not finite,
// d_nb_idx / d_nb_d2 [n][k_eff] (may be null) the k-NN lists, k_eff = min(k, the number of finite points).  ev_mid (may be null) is recorded between the k-NN + normals and the SPFH + FPFH stages.
// cell_scale multiplies the data-derived cell edge (test hook).
namespace {
// The k-NN stage of the FPFH estimator: the grid, the k_eff-NN lists of every point (nb_idx / nb_d2 [n][*ke]) and their work
// counters (cand, fb), all allocated before the first launch; then k_knn and k_normals.  k_eff = min(k, finite points): the
// lists of the finite points hold finite points only.
cudaError_t knn_normals(cudaStream_t st, const float *d_xyz, int n, int k, float cell_scale, PointGrid *pg, DevBuf<int> *nb_idx,
                        DevBuf<float> *nb_d2, DevBuf<pu64> *cand, DevBuf<int> *fb, float *d_normals, int *d_status, int *ke_out) {
  CUDA_TRY(prep_point_grid(st, d_xyz, n, k < n ? k : n, cell_scale, 0.0, pg));
  const int ke = k < pg->nfin ? k : pg->nfin;
  *ke_out = ke;
  KnnArgs a{};
  a.rg = pg->rg; a.n = n; a.k = ke;
  CUDA_TRY(nb_idx->alloc((size_t)n * ke)); CUDA_TRY(nb_d2->alloc((size_t)n * ke));
  CUDA_TRY(cand->alloc(1)); CUDA_TRY(fb->alloc(1));
  CUDA_TRY(cudaMemsetAsync(cand->get(), 0, sizeof(pu64), st)); CUDA_TRY(cudaMemsetAsync(fb->get(), 0, sizeof(int), st));
  a.nb_idx = nb_idx->get(); a.nb_d2 = nb_d2->get(); a.cand = cand->get(); a.fallbacks = fb->get();
  GHICP_LAUNCH(k_knn, blocks(n), PT, 0, st, a);
  GHICP_LAUNCH(k_normals, blocks(n), PT, 0, st, d_xyz, nb_idx->get(), n, ke, d_normals, d_status);
  return cudaSuccess;
}

// PrincipleComponentAnalysis::CheckNormals (include/pca.h:258-271): a non-finite normal becomes (0.577, 0.577, 0.577)
__global__ void k_check_normals(float *__restrict__ nrm, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float *v = nrm + 3 * (size_t)i;
  if (!(isfinite(v[0]) && isfinite(v[1]) && isfinite(v[2]))) { v[0] = 0.577f; v[1] = 0.577f; v[2] = 0.577f; }
}
}  // namespace

cudaError_t prep_knn_normals(cudaStream_t st, const float *d_xyz, int n, int k, float *d_normals) {
  PointGrid pg;
  DevBuf<int> nb_idx, d_fb; DevBuf<float> nb_d2; DevBuf<pu64> d_cand;
  int ke = 0;
  if (n <= 0 || k < 3 || k > FPFH_KMAX) return cudaErrorInvalidValue;
  CUDA_TRY(knn_normals(st, d_xyz, n, k, 0.f, &pg, &nb_idx, &nb_d2, &d_cand, &d_fb, d_normals, nullptr, &ke));
  GHICP_LAUNCH(k_check_normals, blocks(n), PT, 0, st, d_normals, n);
  return cudaGetLastError();
}

cudaError_t prep_fpfh(cudaStream_t st, const float *d_xyz, int n, const int *d_idx, int nidx, int k, float cell_scale,
                      float *d_fpfh, float *d_normals, int *d_status, int *d_nb_idx, float *d_nb_d2, cudaEvent_t ev_mid,
                      FpfhStats *stats) {
  PointGrid pg;
  DevBuf<int> nb_idx, need, d_fb; DevBuf<float> nb_d2, spfh; DevBuf<pu64> d_cand;
  if (stats) *stats = FpfhStats{};
  if (n <= 0 || k < 3 || k > FPFH_KMAX) return cudaErrorInvalidValue;
  int ke = 0;
  CUDA_TRY(knn_normals(st, d_xyz, n, k, cell_scale, &pg, &nb_idx, &nb_d2, &d_cand, &d_fb, d_normals, d_status, &ke));
  if (d_nb_idx) CUDA_TRY(cudaMemcpyAsync(d_nb_idx, nb_idx.get(), sizeof(int) * (size_t)n * ke, cudaMemcpyDeviceToDevice, st));
  if (d_nb_d2) CUDA_TRY(cudaMemcpyAsync(d_nb_d2, nb_d2.get(), sizeof(float) * (size_t)n * ke, cudaMemcpyDeviceToDevice, st));
  if (ev_mid) CUDA_TRY(cudaEventRecord(ev_mid, st));
  CUDA_TRY(spfh.alloc((size_t)n * 33));
  if (d_idx) {
    CUDA_TRY(need.alloc((size_t)n));
    CUDA_TRY(cudaMemsetAsync(need.get(), 0, sizeof(int) * (size_t)n, st));
    if (nidx > 0) GHICP_LAUNCH(k_fpfh_mark, blocks(nidx), PT, 0, st, d_idx, nidx, nb_idx.get(), ke, need.get());
  }
  GHICP_LAUNCH(k_spfh, blocks(n), PT, 0, st, d_xyz, d_normals, nb_idx.get(), n, ke, need.get(), spfh.get());
  if (nidx > 0) GHICP_LAUNCH(k_fpfh, blocks(nidx), PT, 0, st, d_idx, nidx, nb_idx.get(), nb_d2.get(), ke, spfh.get(), d_fpfh);
  if (stats) {
    pu64 c = 0; int fb = 0;
    CUDA_TRY(cudaMemcpyAsync(&c, d_cand.get(), sizeof(c), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(&fb, d_fb.get(), sizeof(fb), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    stats->candidates = (long long)c; stats->fallbacks = fb; stats->cell = (float)pg.rg.cell; stats->queries = n;
  }
  return cudaGetLastError();
}

namespace {
// List rows in cell order: the points flagged in need (every point when need == nullptr).  rows [m], row_of [n] (-1: no row).
cudaError_t make_rows(cudaStream_t st, const int *order, const int *need, int n, int *flags, int *pos, DevBuf<int> *rows,
                      DevBuf<int> *row_of, int *m) {
  GHICP_LAUNCH(k_row_flags, blocks(n + 1), PT, 0, st, order, need, n, flags);
  CUDA_TRY(exclusive_scan(flags, pos, n, st));
  CUDA_TRY(cudaMemcpyAsync(m, pos + n, sizeof(int), cudaMemcpyDeviceToHost, st)); CUDA_TRY(cudaStreamSynchronize(st));
  CUDA_TRY(rows->alloc((size_t)*m)); CUDA_TRY(row_of->alloc((size_t)n));
  CUDA_TRY(cudaMemsetAsync(row_of->get(), 0xff, sizeof(int) * (size_t)n, st));
  GHICP_LAUNCH(k_row_emit, blocks(n), PT, 0, st, order, flags, pos, n, rows->get(), row_of->get());
  return cudaSuccess;
}
// The sorted N_r lists of rows [m]: count, 64-bit offsets, budget check (cudaErrorMemoryAllocation before the entries are
// allocated when *total > budget), fill, segmented sort into off [m + 1] and key [*total].
cudaError_t build_lists(cudaStream_t st, const RadWalk &w, const int *rows, int m, long long budget, DevBuf<long long> *off,
                        DevBuf<pu64> *key, long long *total) {
  DevBuf<long long> cnt; DevBuf<pu64> raw;
  *total = 0;
  CUDA_TRY(cnt.alloc((size_t)m + 1)); CUDA_TRY(off->alloc((size_t)m + 1));
  GHICP_LAUNCH(k_rad_count, blocks(m + 1), PT, 0, st, w, rows, m, cnt.get());
  CUDA_TRY(exclusive_scan64(cnt.get(), off->get(), m, st));
  CUDA_TRY(cudaMemcpyAsync(total, off->get() + m, sizeof(long long), cudaMemcpyDeviceToHost, st)); CUDA_TRY(cudaStreamSynchronize(st));
  if (*total > budget) return cudaErrorMemoryAllocation;
  CUDA_TRY(raw.alloc((size_t)*total)); CUDA_TRY(key->alloc((size_t)*total));
  if (m > 0) GHICP_LAUNCH(k_rad_fill, blocks(m), PT, 0, st, w, rows, m, off->get(), raw.get());
  return segmented_sort(raw.get(), key->get(), *total, m, off->get(), st);
}
// prep_fpfh_radius after the argument checks; *s receives the statistics as far as the call got
cudaError_t fpfh_radius_run(cudaStream_t st, const float *d_xyz, int n, const int *d_idx, int nidx, float rn, float rf,
                            long long nb_max, float *d_fpfh, float *d_normals, int *d_status, cudaEvent_t ev_lists,
                            cudaEvent_t ev_normals, FpfhRadiusStats *s) {
  GridArgs g{};
  GridBufs grid;
  DevBuf<int> need, flags, pos, rows_f, row_of_f, rows_n, row_of_n;
  DevBuf<long long> off_f, off_n; DevBuf<pu64> key_f, key_n;
  DevBuf<float> spfh;
  float mn[3], mx[3];
  int m_f = 0, m_n = 0;
  long long budget;
  {
    size_t fr = 0, tot = 0;
    CUDA_TRY(cudaMemGetInfo(&fr, &tot));
    budget = (long long)(fr / 2 / 16);
    if (nb_max > 0 && nb_max < budget) budget = nb_max;
  }
  s->budget = budget;
  // cell edge = the larger radius, widened by 2 % so that one ring covers the rounding of cell_coord (rings = 1), at least
  // the extent / 2^20 (21-bit key fields; more rings then)
  CUDA_TRY(prep_bounds(st, d_xyz, n, mn, mx));
  double emax = 0.0;
  for (int a = 0; a < 3; ++a) emax = (double)mx[a] - (double)mn[a] > emax ? (double)mx[a] - (double)mn[a] : emax;
  double cell = 1.02 * (double)(rn > rf ? rn : rf);
  if (cell < emax / 1048576.0) cell = emax / 1048576.0;
  CUDA_TRY(build_grid(st, d_xyz, nullptr, n, (float)cell, &g, &grid));
  int gmax = 0;
  for (int a = 0; a < 3; ++a) { const int c = cell_coord_host(mx[a], a == 0 ? g.mnx : (a == 1 ? g.mny : g.mnz), g.inv); gmax = c > gmax ? c : gmax; }
  // two cell coordinates of points closer than r differ by at most r / cell plus twice the float32 rounding of cell_coord
  // (< (gmax + 1) 2^-23 each); 0.01 covers the rounding of d2 against r2
  const double slack = 0.01 + (gmax + 2.0) / 1048576.0;
  const RadWalk wf{g, (int)ceil((double)rf * (double)g.inv + slack), rf * rf};
  const RadWalk wn{g, (int)ceil((double)rn * (double)g.inv + slack), rn * rn};
  s->cell = (float)cell; s->rings_f = wf.rings; s->rings_n = wn.rings;
  CUDA_TRY(flags.alloc((size_t)n + 1)); CUDA_TRY(pos.alloc((size_t)n + 1));
  if (d_idx) {   // rows of the rf lists: the requested points' rf-neighbours
    CUDA_TRY(need.alloc((size_t)n));
    CUDA_TRY(cudaMemsetAsync(need.get(), 0, sizeof(int) * (size_t)n, st));
    if (nidx > 0) GHICP_LAUNCH(k_rad_mark, blocks(nidx), PT, 0, st, wf, d_idx, nidx, need.get());
  }
  const int *order = grid.order.get();
  CUDA_TRY(make_rows(st, order, need.get(), n, flags.get(), pos.get(), &rows_f, &row_of_f, &m_f));
  if (const cudaError_t e = build_lists(st, wf, rows_f.get(), m_f, budget, &off_f, &key_f, &s->nb_f)) { s->needed = s->nb_f; return e; }
  if (d_idx) {   // rows of the rn lists: every point the SPFHs read
    CUDA_TRY(cudaMemsetAsync(need.get(), 0, sizeof(int) * (size_t)n, st));
    if (m_f > 0) GHICP_LAUNCH(k_list_mark, blocks(m_f), PT, 0, st, key_f.get(), off_f.get(), m_f, need.get());
  }
  CUDA_TRY(make_rows(st, order, need.get(), n, flags.get(), pos.get(), &rows_n, &row_of_n, &m_n));
  const cudaError_t en = build_lists(st, wn, rows_n.get(), m_n, budget - s->nb_f, &off_n, &key_n, &s->nb_n);
  s->needed = s->nb_f + s->nb_n;
  CUDA_TRY(en);
  s->spfh_points = m_f;
  if (ev_lists) CUDA_TRY(cudaEventRecord(ev_lists, st));
  const CsrLists lf{key_f.get(), off_f.get(), row_of_f.get()}, ln{key_n.get(), off_n.get(), row_of_n.get()};
  GHICP_LAUNCH(k_rad_normals, blocks(n), PT, 0, st, d_xyz, n, ln, d_normals, d_status);
  if (ev_normals) CUDA_TRY(cudaEventRecord(ev_normals, st));
  CUDA_TRY(spfh.alloc((size_t)n * 33));
  if (m_f > 0) GHICP_LAUNCH(k_rad_spfh, blocks(m_f), PT, 0, st, d_xyz, d_normals, rows_f.get(), m_f, lf, spfh.get());
  const int m_a = d_idx ? nidx : n;
  if (m_a > 0) GHICP_LAUNCH(k_rad_fpfh, blocks(m_a), PT, 0, st, d_idx, m_a, lf, spfh.get(), d_fpfh);
  CUDA_TRY(cudaStreamSynchronize(st));
  return cudaGetLastError();
}
}  // namespace

// FPFH over radius neighbourhoods (DESIGN.md §3.10, "Radius neighbourhoods"): normals over N_rn, SPFH and FPFH over N_rf, at
// d_idx [nidx] (every point when d_idx == nullptr) of d_xyz [n][3].  Only what the requested histograms read is computed:
// N_rf lists of the requested points' rf-neighbours, N_rn lists and normals of every point those SPFHs touch; d_normals [n][3]
// and d_status [n] (may be null) hold NaN / 2 at the points whose normal was not needed.  nb_max > 0 caps the list entries
// (both radii together) below the default budget (half the free device memory at 16 bytes per entry); over the budget the call
// returns cudaErrorMemoryAllocation with stats->needed set, before any output is written.  ev_lists / ev_normals (may be null)
// are recorded after the lists and after the normals.
cudaError_t prep_fpfh_radius(cudaStream_t st, const float *d_xyz, int n, const int *d_idx, int nidx, float rn, float rf,
                             long long nb_max, float *d_fpfh, float *d_normals, int *d_status, cudaEvent_t ev_lists,
                             cudaEvent_t ev_normals, FpfhRadiusStats *stats) {
  FpfhRadiusStats s;
  if (stats) *stats = s;
  if (n <= 0 || !(rn * rn > 0.f) || !(rf * rf > 0.f) || !std::isfinite(rn * rn) || !std::isfinite(rf * rf)) return cudaErrorInvalidValue;
  const cudaError_t e = fpfh_radius_run(st, d_xyz, n, d_idx, nidx, rn, rf, nb_max, d_fpfh, d_normals, d_status, ev_lists,
                                        ev_normals, &s);
  if (stats) *stats = s;
  return e;
}

// =====================================================================================================================
// Statistical outlier removal (DESIGN.md §3.16): CFilter::SORFilter (include/filter.hpp:90-102), PCL's
// StatisticalOutlierRemoval, on the canonical definition stated with ghicp_sor_filter in include/ghicp_b200.h.
//   k_knn + k_sor_listmean   k_eff <= 31: k_knn's k_eff + 1 nearest in registers, the point itself dropped, summed per thread
//   k_sor_dist     larger k_eff: one warp per finite point, k_knn's grid, ring_walk with k_knn's cap and bound, and its
//                  exhaustive fallback, over batches of 32 candidates, one per lane.  The k_eff smallest (d2, index) keys, k_eff up to 128, stay sorted
//                  in a per-warp list in shared memory; a batch's keys below the current k-th key are merged into it by rank.
//                  Only the mean distance leaves the warp: one float per point, no [n][k] lists.
//   k_sor_partial  fixed-order double sums of d (pass 0) or of (d - mean)^2 (pass 1), one per block of a fixed grid
//   k_sor_finish   one block: the fixed-order sum of the partials -> mean (pass 0), stddev and threshold (pass 1)
//   k_sor_flags + exclusive_scan + k_sor_emit: the kept indices, ascending
// No floating-point atomics: two runs give the same bits.
// =====================================================================================================================
namespace {

constexpr int SOR_KMAX = 128;       // largest mean_k
constexpr int SOR_T = 256;          // 8 warps per block, one query each
constexpr int SOR_DEFER_BLOCKS = 32;  // grid of the warp kernel over k_knn's deferred queries (rare: far outliers)
constexpr int SOR_RED = 256;        // blocks of the partial sums = threads of the final sum (fixed: it fixes the summation order)

struct SorArgs {
  RingGrid rg;
  int n, nfin, k;                   // points; the finite ones = the first nfin sorted positions (non-finite ones sort last); k = k_eff
  float *dist;                     // [n]
  unsigned long long *cand;         // candidates examined, summed over all queries
  int *fallbacks;                   // queries that took the exhaustive scan
  const int *qlist, *nq;            // optional: only the points qlist[0 .. *nq) (k_knn's deferred far outliers), grid-strided;
                                    // their fallbacks were counted by k_knn
};

// Merge the lanes' candidate keys c into the warp's ascending list cur[0 .. k) (~0ull = empty slot), writing nxt and swapping.
// Keys are distinct (d2, index) pairs, so every key's new slot is its rank in the union; slots >= k drop out.  Only keys
// below the current k-th key (kth) take part.  Warp-uniform control flow; the __syncwarp orders the writes of nxt before
// the next reads, and every read of cur before the next merge overwrites it.
__device__ __forceinline__ void sor_merge(pu64 *&cur, pu64 *&nxt, int k, int lane, pu64 c, pu64 &kth) {
  const unsigned acc = __ballot_sync(0xffffffffu, c < kth);
  if (acc == 0u) return;
  constexpr int E = SOR_KMAX / 32;  // list slots per lane: lane + 32 j
  pu64 e[E];
  int re[E];
#pragma unroll
  for (int j = 0; j < E; ++j) { const int t = lane + 32 * j; e[j] = t < k ? cur[t] : 0ull; re[j] = 0; }
  int rb = 0;                       // accepted batch keys below c
  for (unsigned m = acc; m; m &= m - 1) {
    const pu64 b = __shfl_sync(0xffffffffu, c, __ffs(m) - 1);
    rb += b < c ? 1 : 0;
#pragma unroll
    for (int j = 0; j < E; ++j) re[j] += b < e[j] ? 1 : 0;
  }
  if ((acc >> lane) & 1u) {
    int lo = 0, hi = k;             // list keys below c
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (cur[mid] < c) lo = mid + 1; else hi = mid;
    }
    if (lo + rb < k) nxt[lo + rb] = c;
  }
#pragma unroll
  for (int j = 0; j < E; ++j) {
    const int t = lane + 32 * j;
    if (t < k && t + re[j] < k) nxt[t + re[j]] = e[j];
  }
  __syncwarp();
  pu64 *const tmp = cur; cur = nxt; nxt = tmp;
  kth = cur[k - 1];
}
// sorted positions [s0, s1) as candidates of the query (point i), 32 per batch; the query itself is not its own neighbour
__device__ __forceinline__ void sor_scan(const GridRegs &g, int s0, int s1, int i, float qx, float qy, float qz, int k, int lane,
                                         pu64 *&cur, pu64 *&nxt, pu64 &kth) {
  for (int b = s0; b < s1; b += 32) {
    const int s = b + lane;
    pu64 c = ~0ull;
    if (s < s1) {
      const int p = g.order[s];
      if (p != i) c = knn_key(knn_d2(qx, qy, qz, g.sorted[s]), p);
    }
    sor_merge(cur, nxt, k, lane, c, kth);
  }
}
__device__ __forceinline__ void sor_reset(pu64 *cur, int k, int lane, pu64 &kth) {
  for (int t = lane; t < k; t += 32) cur[t] = ~0ull;
  __syncwarp();
  kth = ~0ull;
}

__global__ void __launch_bounds__(SOR_T) k_sor_dist(const SorArgs a) {
  __shared__ pu64 s_list[SOR_T / 32][2][SOR_KMAX];
  __shared__ unsigned long long s_cand;
  __shared__ int s_fb;
  if (threadIdx.x == 0) { s_cand = 0ull; s_fb = 0; }
  __syncthreads();
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int t = blockIdx.x * (SOR_T / 32) + w;   // sorted position: the warps of a block take points of the same cells
  const GridArgs &g = a.rg.g;
  if (!a.qlist && t >= a.nfin && t < a.n && lane == 0) a.dist[g.order[t]] = __uint_as_float(0x7fc00000u);   // non-finite
  const int nq = a.qlist ? *a.nq : a.nfin;
  const int step = a.qlist ? gridDim.x * (SOR_T / 32) : nq;   // without a list: at most one query per warp
  const GridRegs r = grid_regs(g);       // per-thread registers, see k_pca
  for (int q = t; q < nq; q += step) {
    const int i = a.qlist ? a.qlist[q] : r.order[q];
    const float qx = g.xyz[3 * (size_t)i], qy = g.xyz[3 * (size_t)i + 1], qz = g.xyz[3 * (size_t)i + 2];
    const int k = a.k;
    float d = 0.f;                       // k_eff = 0 (one finite point): distance 0
    long long cand = 0;
    bool fb = false;
    if (k > 0) {
      pu64 *cur = s_list[w][0], *nxt = s_list[w][1], kth;
      sor_reset(cur, k, lane, kth);
      const int cx = cell_coord(qx, g.mnx, g.inv), cy = cell_coord(qy, g.mny, g.inv), cz = cell_coord(qz, g.mnz, g.inv);
      const bool done = ring_walk(r, a.rg, cx, cy, cz, FPFH_RING_CAP,
          [&](int s0, int s1) {
            cand += s1 - s0;
            sor_scan(r, s0, s1, i, qx, qy, qz, k, lane, cur, nxt, kth);
          },
          [&] { return kth == ~0ull ? (double)INFINITY : (double)knn_key_d2(kth); });
      if (!done) {                       // far outlier: exact by exhaustion over the finite points
        sor_reset(cur, k, lane, kth);
        sor_scan(r, 0, a.nfin, i, qx, qy, qz, k, lane, cur, nxt, kth);
        cand += a.nfin;
        fb = true;
      }
      // square roots in parallel into the spare list, then one lane sums them in ascending d2 order
      for (int j = lane; j < k; j += 32) nxt[j] = (pu64)__double_as_longlong(sqrt((double)knn_key_d2(cur[j])));
      __syncwarp();
      double s = 0.0;
      for (int j = 0; j < k && lane == 0; ++j) s += __longlong_as_double((long long)nxt[j]);
      d = (float)(s / (double)k);
    }
    if (lane == 0) {
      a.dist[i] = d;
      atomicAdd(&s_cand, (unsigned long long)cand);
      if (fb && !a.qlist) atomicAdd(&s_fb, 1);
    }
    __syncwarp();                        // the next query's reset overwrites the lists lane 0 has just read
  }
  __syncthreads();
  if (threadIdx.x == 0) { atomicAdd(a.cand, s_cand); atomicAdd(a.fallbacks, s_fb); }
}

// pass 0: sum of d, pass 1: sum of (d - mean)^2, over the finite points (d not NaN) of this block's fixed share, tree-reduced
__global__ void __launch_bounds__(SOR_RED) k_sor_partial(const float *__restrict__ dist, int n, const double *__restrict__ stats,
                                                         int pass, double *__restrict__ partial) {
  __shared__ double s[SOR_RED];
  const double mean = pass ? stats[0] : 0.0;
  double acc = 0.0;
  for (int i = blockIdx.x * SOR_RED + threadIdx.x; i < n; i += SOR_RED * SOR_RED) {
    const float d = dist[i];
    if (d == d) { const double v = (double)d - mean; acc += pass ? v * v : v; }
  }
  s[threadIdx.x] = acc;
  __syncthreads();
  for (int o = SOR_RED / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) partial[blockIdx.x] = s[0];
}
// one block: stats[0] = mean (pass 0); stats[1] = stddev, stats[2] = threshold (pass 1)
__global__ void __launch_bounds__(SOR_RED) k_sor_finish(const double *__restrict__ partial, int nfin, double std_mul, int pass,
                                                        double *__restrict__ stats) {
  __shared__ double s[SOR_RED];
  s[threadIdx.x] = partial[threadIdx.x];
  __syncthreads();
  for (int o = SOR_RED / 2; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    if (pass == 0) {
      stats[0] = s[0] / (double)nfin;
    } else {
      const double sd = nfin > 1 ? sqrt(s[0] / (double)(nfin - 1)) : 0.0;
      stats[1] = sd;
      stats[2] = stats[0] + std_mul * sd;
    }
  }
}
// flags[i] = point i is kept (finite, d not above the threshold); flags[n] = 0
__global__ void k_sor_flags(const float *__restrict__ dist, int n, const double *__restrict__ stats, int *__restrict__ flags) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n) return;
  const float d = i < n ? dist[i] : 0.f;
  flags[i] = (i < n && d == d && !((double)d > stats[2])) ? 1 : 0;
}
__global__ void k_sor_emit(const int *__restrict__ flags, const int *__restrict__ pos, int n, int *__restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n && flags[i]) out[pos[i]] = i;
}
// The small-k path: d_p from k_knn's ascending (d2, index) list of k + 1 entries.  The list holds the k + 1 nearest of all
// finite points, p itself included unless k + 1 duplicates of p with smaller indices fill it; dropping p (or, without it, the
// last entry) leaves the k nearest OTHER points, whose square roots are added in list order as k_sor_dist adds them.
__global__ void k_sor_listmean(const float *__restrict__ xyz, int n, const int *__restrict__ nb_idx, const float *__restrict__ nb_d2,
                               int k, float *__restrict__ dist) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (!finite3(xyz[3 * (size_t)i], xyz[3 * (size_t)i + 1], xyz[3 * (size_t)i + 2])) { dist[i] = __uint_as_float(0x7fc00000u); return; }
  const size_t b = (size_t)i * (k + 1);
  double s = 0.0;
  for (int j = 0, taken = 0; j <= k && taken < k; ++j) {
    if (nb_idx[b + j] == i) continue;
    s += sqrt((double)nb_d2[b + j]);
    ++taken;
  }
  dist[i] = k > 0 ? (float)(s / (double)k) : 0.f;
}
// GHICP_SOR_FORCE_WARP=1 (test and benchmark hook) runs k_sor_dist at every k, so that both paths can be checked and timed at
// the same small k; results do not change, only the time does
bool sor_force_warp() {
  const char *e = getenv("GHICP_SOR_FORCE_WARP");
  return e && e[0] == '1';
}

}  // namespace

// ghicp_sor_filter on device arrays: d_out (capacity n) receives the kept indices, d_dist [n] every point's mean distance
// (NaN for a non-finite point); r every field.  The grid build allocates, launches and reads back its box and cell count;
// every later buffer is allocated before the distance kernels, and the one read-back after them, before the final
// synchronise, brings the kept count (with the statistics and work counters).  The distances come from k_knn's register
// top-k (k_eff + 1 <= FPFH_KMAX: its [n][k_eff + 1] lists, at most 1.3 GB at 5 M points, are summed by k_sor_listmean) or
// from k_sor_dist (larger k, no lists); both give the same bits, and at the k where both run k_knn is the faster
// (tools/bench_sor.py times both).
cudaError_t prep_sor_filter(cudaStream_t st, const float *d_xyz, int n, int mean_k, double std_mul, int *d_out, float *d_dist,
                            ghicp_sor_result *r) {
  StageEvents<5> ev;
  PointGrid pg;
  DevBuf<double> d_part, d_stats; DevBuf<int> d_flags, d_pos, d_fb, nb_idx, d_def; DevBuf<pu64> d_cand; DevBuf<float> nb_d2;
  *r = ghicp_sor_result{};
  if (n <= 0) return cudaSuccess;
  if (mean_k < 1 || mean_k > SOR_KMAX) return cudaErrorInvalidValue;
  CUDA_TRY(ev.create());
  CUDA_TRY(cudaEventRecord(ev[0], st));
  CUDA_TRY(prep_point_grid(st, d_xyz, n, mean_k + 1 < n ? mean_k + 1 : n, 0.f, 0.0, &pg));
  const int nfin = pg.nfin, k = nfin > 0 ? (mean_k < nfin - 1 ? mean_k : nfin - 1) : 0;
  CUDA_TRY(d_part.alloc(SOR_RED)); CUDA_TRY(d_stats.alloc(3));
  CUDA_TRY(d_flags.alloc((size_t)n + 1)); CUDA_TRY(d_pos.alloc((size_t)n + 1));
  CUDA_TRY(d_cand.alloc(1)); CUDA_TRY(d_fb.alloc(1));
  const bool lists = k + 1 <= FPFH_KMAX && !sor_force_warp();
  if (lists && nfin > 0) {
    CUDA_TRY(nb_idx.alloc((size_t)n * (k + 1))); CUDA_TRY(nb_d2.alloc((size_t)n * (k + 1)));
    CUDA_TRY(d_def.alloc((size_t)nfin + 1));
    CUDA_TRY(cudaMemsetAsync(d_def.get() + nfin, 0, sizeof(int), st));   // the deferred count
  }
  CUDA_TRY(cudaMemsetAsync(d_stats.get(), 0, 3 * sizeof(double), st));
  CUDA_TRY(cudaMemsetAsync(d_cand.get(), 0, sizeof(pu64), st)); CUDA_TRY(cudaMemsetAsync(d_fb.get(), 0, sizeof(int), st));
  CUDA_TRY(cudaEventRecord(ev[1], st));
  SorArgs a{};
  a.rg = pg.rg; a.n = n; a.nfin = nfin; a.k = k;
  a.dist = d_dist; a.cand = d_cand.get(); a.fallbacks = d_fb.get();
  if (lists) {
    if (nfin > 0) {
      KnnArgs b{};
      b.rg = pg.rg; b.n = n; b.k = k + 1;
      b.nb_idx = nb_idx.get(); b.nb_d2 = nb_d2.get(); b.cand = d_cand.get(); b.fallbacks = d_fb.get();
      b.deferred = d_def.get(); b.n_deferred = d_def.get() + nfin;
      GHICP_LAUNCH(k_knn, blocks(n), PT, 0, st, b);
    }
    GHICP_LAUNCH(k_sor_listmean, blocks(n), PT, 0, st, d_xyz, n, nb_idx.get(), nb_d2.get(), k, d_dist);
    if (nfin > 0) {   // the far outliers k_knn deferred: the warp kernel's 32-lane scan instead of one thread's
      a.qlist = d_def.get(); a.nq = d_def.get() + nfin;
      GHICP_LAUNCH(k_sor_dist, SOR_DEFER_BLOCKS, SOR_T, 0, st, a);
    }
  } else {
    GHICP_LAUNCH(k_sor_dist, (n + SOR_T / 32 - 1) / (SOR_T / 32), SOR_T, 0, st, a);
  }
  CUDA_TRY(cudaEventRecord(ev[2], st));
  if (nfin > 0)
    for (int pass = 0; pass < 2; ++pass) {
      GHICP_LAUNCH(k_sor_partial, SOR_RED, SOR_RED, 0, st, d_dist, n, d_stats.get(), pass, d_part.get());
      GHICP_LAUNCH(k_sor_finish, 1, SOR_RED, 0, st, d_part.get(), nfin, std_mul, pass, d_stats.get());
    }
  CUDA_TRY(cudaEventRecord(ev[3], st));
  GHICP_LAUNCH(k_sor_flags, blocks(n + 1), PT, 0, st, d_dist, n, d_stats.get(), d_flags.get());
  CUDA_TRY(exclusive_scan(d_flags.get(), d_pos.get(), n, st));
  int kept = 0, fb = 0;
  double stats[3];
  pu64 cand = 0;
  CUDA_TRY(cudaMemcpyAsync(&kept, d_pos.get() + n, sizeof(int), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaMemcpyAsync(stats, d_stats.get(), sizeof(stats), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaMemcpyAsync(&cand, d_cand.get(), sizeof(cand), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaMemcpyAsync(&fb, d_fb.get(), sizeof(fb), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  nb_idx.reset(); nb_d2.reset(); d_def.reset();
  if (kept > 0) GHICP_LAUNCH(k_sor_emit, blocks(n), PT, 0, st, d_flags.get(), d_pos.get(), n, d_out);
  CUDA_TRY(cudaEventRecord(ev[4], st));
  CUDA_TRY(cudaStreamSynchronize(st));
  r->n_finite = nfin; r->n_kept = kept; r->k_eff = k; r->fallbacks = fb;
  r->mean = stats[0]; r->stddev = stats[1]; r->threshold = stats[2];
  r->candidates = (long long)cand;
  for (int s = 0; s < 4; ++s) r->stage_ms[s] = ev.ms(s, s + 1);
  r->stage_ms[4] = ev.ms(0, 4);
  return cudaGetLastError();
}

}  // namespace ghicp_b200
