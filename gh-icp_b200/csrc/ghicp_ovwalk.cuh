// ghicp_ovwalk.cuh — the exact nearest-neighbour walk over a cloud's point grid shared by the overlap / fitness kernels
// (ghicp_overlap.cu, DESIGN.md §3.12) and the ICP kernels (ghicp_icp.cu, DESIGN.md §3.13): the grid as the walk reads it,
// the float32 move of a point, and the ring walk with its distance-culled columns.
#pragma once
#include <cmath>

#include "ghicp_internal.h"
#include "ghicp_grid.cuh"

namespace ghicp_b200 {

struct OverlapTarget {   // a cloud's grid for nearest-neighbour queries (prep_point_grid, 8 points per cell)
  PointGrid pg;
  int n = 0;
};

namespace {

struct OvGrid {   // the target grid as the query kernels read it
  RingGrid rg;
  double mn[3], ext[3];           // box minimum; box extent in cell edges
};
inline OvGrid ov_grid_of(const PointGrid &pg) {
  OvGrid G{};
  G.rg = pg.rg;
  G.mn[0] = pg.rg.g.mnx; G.mn[1] = pg.rg.g.mny; G.mn[2] = pg.rg.g.mnz;
  for (int k = 0; k < 3; ++k) G.ext[k] = ((double)pg.rg.mx[k] - G.mn[k]) / pg.rg.cell;
  return G;
}

// x' = ((R00 x + R01 y) + R02 z) + t0, float32, every operation rounded separately (also SAC-IA's move of a source point);
// rt = R row-major, then t
__device__ __forceinline__ void ov_move(const float *rt, float x, float y, float z, float &ox, float &oy, float &oz) {
  ox = ((rt[0] * x + rt[1] * y) + rt[2] * z) + rt[9];
  oy = ((rt[3] * x + rt[4] * y) + rt[5] * z) + rt[10];
  oz = ((rt[6] * x + rt[7] * y) + rt[8] * z) + rt[11];
}
// distance from u to the interval [lo, hi] (cell edges)
__device__ __forceinline__ double ov_gap(double u, double lo, double hi) { return u < lo ? lo - u : (u > hi ? u - hi : 0.0); }
// where the points of cells lo .. hi on one axis can lie: the cells widened by the rounding slack, clipped to B's box
__device__ __forceinline__ double ov_cells_gap(double u, int lo, int hi, double s, double ext) {
  return ov_gap(u, fmax((double)lo - s, 0.0), fmin((double)hi + 1.0 + s, ext));
}
// narrow [a, b] to the cells whose extent comes within w (cell edges) of u
__device__ __forceinline__ void ov_window(double u, double w, double s, int &a, int &b) {
  const double lo = u - w - 1.0 - s, hi = u + w + s;
  if (lo > (double)a) a = lo > (double)b ? b + 1 : (int)ceil(lo);
  if (hi < (double)b) b = hi < (double)a ? a - 1 : (int)floor(hi);
}

// Nearest squared distance (knn_d2) from q to B: exact when it is <= lim, +inf otherwise.  hit >= 0: stops at the first
// d2 < hit and returns it (overlap-only mode).  Bounds are compared in double against (1 - 1e-5) of their value, far more
// than the float32 rounding of knn_d2.
// IDX: idx (set to -1 by the caller) receives the index of the nearest point in (d2, index) order — the smallest index among
// the points at the smallest d2.  The pruning never skips such a point: every skip below is a strict comparison of a lower
// bound on a cell's distance, taken at (1 - 1e-5) of its value, against min(best, lim), so a point in a skipped cell is at
// least best / (1 - 1e-5) away in exact arithmetic, and its float32 knn_d2 (relative error below 1e-6) is still strictly
// greater than best: it cannot equal best, let alone win the tie.
template <bool IDX>
__device__ __forceinline__ float ov_nearest(const GridRegs &r, const OvGrid &G, float qx, float qy, float qz, double lim, float hit,
                                            unsigned long long &cells, unsigned long long &cand, int &idx) {
  // a non-finite moved point (a NaN return of an organised scan) has no nearest neighbour: +inf at once, no walk
  if (!(isfinite(qx) && isfinite(qy) && isfinite(qz))) return INFINITY;
  const double q[3] = {(double)qx, (double)qy, (double)qz};
  const double s = G.rg.slack, unit = G.rg.cell * G.rg.cell * (1.0 - 1e-5);
  double u[3], bg[3];
  int c[3];
  for (int a = 0; a < 3; ++a) {
    u[a] = (q[a] - G.mn[a]) / G.rg.cell;
    bg[a] = ov_gap(u[a], 0.0, G.ext[a]);
    c[a] = !(u[a] > 0.0) ? 0 : (u[a] >= (double)G.rg.gm[a] ? G.rg.gm[a] : (int)u[a]);
  }
  const double bg2 = (bg[0] * bg[0] + bg[1] * bg[1]) + bg[2] * bg[2];
  if (!(bg2 * unit <= lim)) return INFINITY;   // beyond the limit from B's box
  int kmax = 0;
  for (int a = 0; a < 3; ++a) kmax = max(kmax, max(c[a], G.rg.gm[a] - c[a]));
  float best = INFINITY;
  for (int k = 0;; ++k) {
    // columns of ring k: a wall column (max(|dx|, |dy|) == k) spans cz - k .. cz + k, an inner one only its floor and
    // ceiling cell; a column whose bound passes L (squared cell edges) is skipped
    double L = fmin((double)best, lim) / unit;
    if (bg2 > L) break;
    int x0 = max(c[0] - k, 0), x1 = min(c[0] + k, G.rg.gm[0]);
    ov_window(u[0], sqrt(L - bg[1] * bg[1] - bg[2] * bg[2]), s, x0, x1);
    for (int x = x0; x <= x1; ++x) {
      L = fmin((double)best, lim) / unit;
      const double gx = ov_cells_gap(u[0], x, x, s, G.ext[0]);
      const double wy = L - gx * gx - bg[2] * bg[2];
      if (wy < 0.0) continue;
      int y0 = max(c[1] - k, 0), y1 = min(c[1] + k, G.rg.gm[1]);
      ov_window(u[1], sqrt(wy), s, y0, y1);
      const bool xwall = abs(x - c[0]) == k;
      const int za = c[2] - k, zb = c[2] + k;   // the two cells of an inner column, or the run za .. zb of a wall column
      bool inner = false;                        // can an inner column of this row hold a closer point at all?
      if (!xwall) {
        const double wz0 = sqrt(fmax(L - gx * gx - bg[1] * bg[1], 0.0));
        inner = (za >= 0 && ov_cells_gap(u[2], za, za, s, G.ext[2]) <= wz0) ||
                (zb <= G.rg.gm[2] && ov_cells_gap(u[2], zb, zb, s, G.ext[2]) <= wz0);
      }
      for (int y = y0; y <= y1; ++y) {
        const bool wall = xwall || abs(y - c[1]) == k;
        if (!wall && !inner) { if (y < c[1] + k - 1) y = c[1] + k - 1; continue; }   // on to the far wall
        const double gy = ov_cells_gap(u[1], y, y, s, G.ext[1]);
        const double wz = L - gx * gx - gy * gy;
        if (wz < 0.0) continue;
        for (int part = 0; part < (wall ? 1 : 2); ++part) {
          int lo, hi;
          if (wall) { lo = max(za, 0); hi = min(zb, G.rg.gm[2]); }
          else { lo = hi = part == 0 ? za : zb; if (lo < 0 || lo > G.rg.gm[2]) continue; }
          ov_window(u[2], sqrt(wz), s, lo, hi);
          if (lo > hi) continue;
          cells += (unsigned long long)(hi - lo + 1);
          const int s0 = r.cstart[lower_cell(r, cell_key(x, y, lo))], s1 = r.cstart[lower_cell(r, cell_key(x, y, hi) + 1)];
          cand += (unsigned long long)(s1 - s0);
          for (int p = s0; p < s1; ++p) {
            const float d2 = knn_d2(qx, qy, qz, r.sorted[p]);
            if (d2 < hit) return d2;
            if (IDX) {
              const int j = r.order[p];
              if (d2 < best || (d2 == best && j < idx)) { best = d2; idx = j; }
            } else {
              best = d2 < best ? d2 : best;
            }
          }
        }
      }
    }
    if (k >= kmax) break;
    // a true lower bound on every cell outside the visited cube: it lies beyond ring k on some axis, and within B's box
    // on the two others
    L = fmin((double)best, lim) / unit;
    double lb = INFINITY;
    for (int a = 0; a < 3; ++a) {
      const double b1 = bg[(a + 1) % 3], b2 = bg[(a + 2) % 3], o2 = b1 * b1 + b2 * b2;
      if (c[a] - k - 1 >= 0) { const double d = ov_cells_gap(u[a], 0, c[a] - k - 1, s, G.ext[a]); lb = fmin(lb, d * d + o2); }
      if (c[a] + k + 1 <= G.rg.gm[a]) { const double d = ov_cells_gap(u[a], c[a] + k + 1, G.rg.gm[a], s, G.ext[a]); lb = fmin(lb, d * d + o2); }
    }
    if (lb > L) break;
  }
  if (hit >= 0.f) return best < hit ? best : INFINITY;
  return (double)best <= lim ? best : INFINITY;
}

// the key of v's cell in the grid, clamped into it (the cell order of the queries: k_ov_keys, k_icp_keys)
__device__ __forceinline__ pu64 ov_cell_key(const OvGrid &G, const float *v) {
  int c[3];
  for (int k = 0; k < 3; ++k) {
    const double f = floor(((double)v[k] - G.mn[k]) / G.rg.cell);
    c[k] = !(f > 0.0) ? 0 : (f > (double)G.rg.gm[k] ? G.rg.gm[k] : (int)f);
  }
  return cell_key(c[0], c[1], c[2]);
}

// warp-reduced integer work counters of the queries, work[0] += cells, work[1] += cand (every lane of the warp must call it)
__device__ __forceinline__ void ov_add_work(unsigned long long cells, unsigned long long cand, unsigned long long *work) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    cells += __shfl_xor_sync(0xffffffffu, cells, o);
    cand += __shfl_xor_sync(0xffffffffu, cand, o);
  }
  if ((threadIdx.x & 31) == 0 && (cells | cand)) { atomicAdd(work, cells); atomicAdd(work + 1, cand); }
}

}  // namespace
}  // namespace ghicp_b200
