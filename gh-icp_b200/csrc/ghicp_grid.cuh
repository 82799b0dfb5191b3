// ghicp_grid.cuh — the cell-sorted uniform point grid of the pre-processing kernels (ghicp_prep.cu: radius PCA, NMS, the
// FPFH k-NN, SOR) and of the SAC-IA scoring (ghicp_sac.cu), which runs exact nearest-neighbour queries against the same
// index, and the ring walk those exact searches share.
// Points are sorted by cell key; ucell lists the occupied cells in key order and cstart their first sorted position.
#pragma once
#include "ghicp_internal.h"

namespace ghicp_b200 {

typedef unsigned long long pu64;

__device__ __forceinline__ pu64 cell_key(int cx, int cy, int cz) { return ((pu64)cx << 42) | ((pu64)cy << 21) | (pu64)cz; }
__device__ __forceinline__ int cell_coord(float v, float mn, float inv) { const int c = (int)floorf((v - mn) * inv); return c < 0 ? 0 : c; }
inline int cell_coord_host(float v, float mn, float inv) { const float f = (v - mn) * inv; const int c = (int)floorf(f); return c < 0 ? 0 : c; }
// Non-finite points take no part in the pre-processing (DESIGN.md §3.8): they bound no box, own no cell and find no neighbour.
__host__ __device__ __forceinline__ bool finite3(float x, float y, float z) { return isfinite(x) && isfinite(y) && isfinite(z); }

struct GridArgs {
  const float *xyz; const int *ids;      // point of position k = xyz[ids ? ids[k] : k]
  const int *order;                      // positions sorted by cell (ascending position inside a cell)
  const float4 *sorted;                  // the same points in that order (x y z _): a cell's run is read with coalesced 16-byte loads
  const pu64 *ucell; const int *cstart; int nu;
  float mnx, mny, mnz, inv, r2;
};
// Per-thread neighbour walks (k_pca, k_nms_round): every thread first resolves its nine column runs, then walks them in one
// flat loop nest, with the grid description copied into per-thread registers.  A form that walked "for dx, for dy
// { column_run; for s }" reading the grid description straight from the kernel parameters returned neighbour counts short
// for whole warps on hardware (its SASS re-loaded kernel parameters in per-warp uniform registers across the divergent
// per-thread loops), while the CPU emulation of the same source passed.
struct GridRegs {
  const float4 *sorted; const pu64 *ucell; const int *cstart; const int *order; int nu; float r2;
};
__device__ __forceinline__ GridRegs grid_regs(const GridArgs &g) {
  GridRegs r;
  r.sorted = g.sorted; r.ucell = g.ucell; r.cstart = g.cstart; r.order = g.order; r.nu = g.nu; r.r2 = g.r2;
  return r;
}
// first occupied cell with a key >= key
__device__ __forceinline__ int lower_cell(const GridRegs &g, pu64 key) {
  int lo = 0, hi = g.nu;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (g.ucell[mid] < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// Top-k lists of the k-NN searches (k_knn, and the feature k-NN of SAC-IA): (d2, index) as one ascending u64 key.  d2 >= 0,
// so its float bits order like the value; + 1 keeps key 0 free as the sentinel that pads the sorted list when k < K.
__device__ __forceinline__ pu64 knn_key(float d2, int idx) { return ((pu64)(__float_as_uint(d2) + 1u) << 32) | (unsigned)idx; }
__device__ __forceinline__ float knn_key_d2(pu64 key) { return __uint_as_float((unsigned)(key >> 32) - 1u); }

// sorted insertion with static indices only (the list stays in registers): the largest key sits in the last slot
template <int K>
__device__ __forceinline__ void knn_insert(pu64 (&key)[K], pu64 c) {
  if (!(c < key[K - 1])) return;
  key[K - 1] = c;
#pragma unroll
  for (int j = K - 1; j > 0; --j) {
    const pu64 lo = key[j - 1], hi = key[j];
    const bool sw = hi < lo;
    key[j - 1] = sw ? hi : lo; key[j] = sw ? lo : hi;
  }
}
// d2 = (dx*dx + dy*dy) + dz*dz, dx = q.x - p.x, every operation rounded separately (the oracle's fpfh_d2)
__device__ __forceinline__ float knn_d2(float qx, float qy, float qz, const float4 &p) {
  const float dx = qx - p.x, dy = qy - p.y, dz = qz - p.z;
  return (dx * dx + dy * dy) + dz * dz;
}

// A grid for ring searches as the kernels read it (prep_point_grid).
struct RingGrid {
  GridArgs g;
  int gm[3];                             // largest occupied cell coordinate per axis
  float mx[3];                           // maximum of the finite points' box (the minimum is g.mnx, g.mny, g.mnz)
  double cell, slack;                    // cell edge; cells of margin for the float32 rounding of cell_coord
};

// The ring walk of the exact nearest-neighbour searches (k_knn, k_sor_dist, SAC-IA's sac_nn_d2) from the cell (cx, cy, cz):
// rings 0, 1, ... of grid columns, dx then dy; a column on the ring's wall is its whole z-range clipped to the grid, one
// inside the wall its floor cell, then its ceiling cell.  col(s0, s1) receives each column's run [s0, s1) of sorted
// positions.  After each ring the walk is settled once the ring reaches the far side of the grid on every axis, or once
// bound() (a squared distance; +inf while nothing bounds the search) lies below every point of an unvisited cell, which is at
// least (ring - slack) cell edges away on some axis.  The (1 - 1e-5) margin is far more than the float32 rounding of knn_d2,
// and it is what keeps the results exact.  Returns false when rings 0 .. cap did not settle it.
// The scalar geometry is read once into locals (see GridRegs); the columns go through the per-thread copy r.
template <class Col, class Bound>
__device__ __forceinline__ bool ring_walk(const GridRegs &r, const RingGrid &G, int cx, int cy, int cz, int cap, Col &&col,
                                          Bound &&bound) {
  const int gx = G.gm[0], gy = G.gm[1], gz = G.gm[2];
  const double cell = G.cell, slack = G.slack;
  int rmax = cx;                         // the ring that reaches the far side of the grid on every axis
  rmax = max(rmax, gx - cx); rmax = max(rmax, cy); rmax = max(rmax, gy - cy); rmax = max(rmax, cz); rmax = max(rmax, gz - cz);
  for (int ring = 0; ring <= cap; ++ring) {
    for (int dx = -ring; dx <= ring; ++dx) {
      const int x = cx + dx;
      if (x < 0 || x > gx) continue;
      for (int dy = -ring; dy <= ring; ++dy) {
        const int y = cy + dy;
        if (y < 0 || y > gy) continue;
        const bool wall = max(abs(dx), abs(dy)) == ring;
        for (int zs = 0; zs < (wall ? 1 : 2); ++zs) {
          int zlo, zhi;
          if (wall) { zlo = max(cz - ring, 0); zhi = min(cz + ring, gz); }
          else { zlo = zhi = zs == 0 ? cz - ring : cz + ring; if (zlo < 0 || zlo > gz) continue; }
          if (zlo > zhi) continue;
          col(r.cstart[lower_cell(r, cell_key(x, y, zlo))], r.cstart[lower_cell(r, cell_key(x, y, zhi) + 1)]);
        }
      }
    }
    if (ring >= rmax) return true;
    const double lb = ((double)ring - slack) * cell;
    if (lb > 0.0 && bound() < lb * lb * (1.0 - 1e-5)) return true;
  }
  return false;
}

struct GridBufs {   // the device arrays GridArgs points into
  DevBuf<int> order, cstart; DevBuf<pu64> ucell; DevBuf<float4> sorted;
};
// A grid over all n points of d_xyz with the cell rule of the FPFH k-NN (k_eff neighbours wanted per query), for ring
// searches, and the device arrays it reads.
struct PointGrid {
  RingGrid rg{};
  int nfin = 0;                          // finite points
  GridBufs buf;
};
// cell edge = the k-NN rule times cell_scale (if > 0), at least min_cell, at least the extent / 2^20 (21-bit key fields)
cudaError_t prep_point_grid(cudaStream_t st, const float *d_xyz, int n, int ke, float cell_scale, double min_cell, PointGrid *out);
// stable ascending sort of (keys, vals) pairs in place, on the stream (the grid builder's radix sort)
cudaError_t prep_sort_pairs(cudaStream_t st, pu64 *keys, int *vals, int n);

}  // namespace ghicp_b200
