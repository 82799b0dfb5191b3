// ghicp_prep_oracle.cpp — CPU ORACLE for the pre-processing that feeds the registration loop (SURVEY.md §8f row N1):
//   CFilter::voxelfilter                      include/filter.hpp:28-88
//   PrincipleComponentAnalysis (radius PCA)   include/pca.h:133-165, 198-250
//   CKeypointDetect::pruneUnstablePoints      include/keypoint_detect.hpp:132-147
//   CKeypointDetect::nonMaximaSuppression     include/keypoint_detect.hpp:149-191
// TEST INFRASTRUCTURE ONLY (see ghicp_oracle.h).  Restated on flat arrays, float32 where the reference computes in
// float32.  PARITY UNPINNED: the reference has no tests, and the arithmetic it delegates to PCL (pcl::getMinMax3D,
// KdTreeFLANN::radiusSearch, pcl::PCA -> Eigen::SelfAdjointEigenSolver<Matrix3f>) is not in /root/reference.
// Three places where the reference's result is implementation-defined or depends on an absent library are given a
// CANONICAL definition here (the CUDA path uses the same one, so the two agree bit for bit):
//   1. voxelfilter keeps "the first element of each run after std::sort" of an UNSTABLE sort (:71-83): canonical = the
//      point with the smallest index in the voxel.  The reference's size bug is reproduced: id_pairs is created with n
//      default entries {voxel 0, index 0} AND receives n push_backs (:52, :66), so point 0 is emitted once more as the
//      representative of voxel id 0.
//   2. PCA sums: radiusSearch returns neighbours sorted by distance and pcl::PCA accumulates in float; canonical = double
//      sums about the query point over the neighbours in grid-cell order (27 cells z-fastest, ascending index inside a
//      cell), rounded once to float32, then a cyclic Jacobi eigen-decomposition in float32.
//   3. nonMaximaSuppression sorts by curvature with an unstable sort and a '>' comparator (:120-130, :151): canonical tie
//      order = ascending point index.
// Neighbourhood test: squared distance < radius^2 (FLANN's RadiusResultSet keeps dist < radius), the query point included.
// Non-finite points take no part (pcl::removeNaNFromPointCloud, then the reference; indices stay those of the input): they
// bound no box, own no cell, have no neighbour (pt_num 0, eigenvalues and curvature 0) and are never emitted.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <map>
#include <numeric>
#include <vector>

namespace {

typedef unsigned long long ull;

bool finite3(const float *p) { return std::isfinite(p[0]) && std::isfinite(p[1]) && std::isfinite(p[2]); }

// cyclic Jacobi on a symmetric 3x3 (float32), eigenvalues sorted descending.  c = {xx, xy, xz, yy, yz, zz}
void sym3_eig_f32(const float c[6], float lam[3]) {
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

struct Grid {  // uniform grid, cell edge = radius; cells keyed by (cx << 42 | cy << 21 | cz)
  float minx, miny, minz, inv;
  std::map<ull, std::vector<int>> cells;  // ascending index inside a cell
  static ull key(int cx, int cy, int cz) { return ((ull)cx << 42) | ((ull)cy << 21) | (ull)cz; }
  int coord(float v, float mn) const { int c = (int)floorf((v - mn) * inv); return c < 0 ? 0 : c; }
  void build(const float *xyz, const int *ids, int n, float radius) {
    minx = miny = minz = INFINITY;
    for (int k = 0; k < n; ++k) {
      const float *p = xyz + 3 * (size_t)(ids ? ids[k] : k);
      if (finite3(p)) { minx = fminf(minx, p[0]); miny = fminf(miny, p[1]); minz = fminf(minz, p[2]); }
    }
    inv = 1.0f / radius;
    for (int k = 0; k < n; ++k) {
      const int i = ids ? ids[k] : k;
      const float *p = xyz + 3 * (size_t)i;
      if (finite3(p)) cells[key(coord(p[0], minx), coord(p[1], miny), coord(p[2], minz))].push_back(k);
    }
  }
  template <typename F>
  void for_neighbours(const float *q, F &&f) const {  // 27 cells, x slowest / z fastest, ascending position inside a cell
    if (!finite3(q)) return;
    const int cx = coord(q[0], minx), cy = coord(q[1], miny), cz = coord(q[2], minz);
    for (int dx = -1; dx <= 1; ++dx)
      for (int dy = -1; dy <= 1; ++dy)
        for (int dz = -1; dz <= 1; ++dz) {
          const int x = cx + dx, y = cy + dy, z = cz + dz;
          if (x < 0 || y < 0 || z < 0) continue;
          auto it = cells.find(key(x, y, z));
          if (it == cells.end()) continue;
          for (int k : it->second) f(k);
        }
  }
};

}  // namespace

extern "C" {

// CFilter::voxelfilter (include/filter.hpp:28-88).  xyz [n][3] float32.  out_idx (capacity n + 1) receives the indices of
// the kept points in output order (ascending voxel id).  Returns their number.
int orc_voxel_downsample(const float *xyz, int n, float voxel_size, int *out_idx) {
  int first = -1, nfin = 0;                                                            // the finite cloud: its size, its point 0
  for (int i = 0; i < n; ++i) if (finite3(xyz + 3 * (size_t)i)) { if (first < 0) first = i; ++nfin; }
  if (nfin == 0) return 0;
  const float inverse_voxel_size = 1.0f / voxel_size;                                  // :30
  float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};   // pcl::getMinMax3D, :33
  for (int i = 0; i < n; ++i)
    if (finite3(xyz + 3 * (size_t)i))
      for (int k = 0; k < 3; ++k) { mn[k] = fminf(mn[k], xyz[3 * (size_t)i + k]); mx[k] = fmaxf(mx[k], xyz[3 * (size_t)i + k]); }
  const float gap[3] = {mx[0] - mn[0], mx[1] - mn[1], mx[2] - mn[2]};                  // :36
  const ull max_vy = (ull)(ceilf(gap[1] * inverse_voxel_size) + 1);                    // :39-40
  const ull max_vz = (ull)(ceilf(gap[2] * inverse_voxel_size) + 1);
  const ull mul_vx = max_vy * max_vz, mul_vy = max_vz;                                 // :48-50
  std::vector<std::pair<ull, unsigned>> id_pairs((size_t)nfin, {0ull, (unsigned)first});   // :52: n default entries ...
  for (int i = 0; i < n; ++i) {                                                        // :54-68: ... plus n real ones
    if (!finite3(xyz + 3 * (size_t)i)) continue;
    const ull vx = (ull)floorf((xyz[3 * (size_t)i] - mn[0]) * inverse_voxel_size);
    const ull vy = (ull)floorf((xyz[3 * (size_t)i + 1] - mn[1]) * inverse_voxel_size);
    const ull vz = (ull)floorf((xyz[3 * (size_t)i + 2] - mn[2]) * inverse_voxel_size);
    id_pairs.push_back({vx * mul_vx + vy * mul_vy + vz, (unsigned)i});
  }
  std::sort(id_pairs.begin(), id_pairs.end());   // :71 sorts by voxel only (unstable); canonical: (voxel, index) order
  int m = 0;
  size_t b = 0;
  while (b < id_pairs.size()) {                  // :75-83
    out_idx[m++] = (int)id_pairs[b].second;
    size_t e = b + 1;
    while (e < id_pairs.size() && id_pairs[e].first == id_pairs[b].first) ++e;
    b = e;
  }
  return m;
}

// Radius PCA of every point (include/pca.h:133-165 + 198-233).  lam [n][3] float eigenvalues (descending, of the
// covariance normalised by count - 1 like pcl::PCA), curvature [n] double (:224-231), pt_num [n].
int orc_pca_curvature(const float *xyz, int n, float radius, float *lam, double *curvature, int *pt_num) {
  Grid g;
  g.build(xyz, nullptr, n, radius);
  const float r2 = radius * radius;
  for (int i = 0; i < n; ++i) {
    const float *q = xyz + 3 * (size_t)i;
    int cnt = 0;
    double sd[3] = {0, 0, 0}, sdd[6] = {0, 0, 0, 0, 0, 0};
    g.for_neighbours(q, [&](int k) {
      const float *p = xyz + 3 * (size_t)k;
      const float dx = p[0] - q[0], dy = p[1] - q[1], dz = p[2] - q[2];
      const float d2 = dx * dx + dy * dy + dz * dz;
      if (!(d2 < r2)) return;
      ++cnt;
      const double x = dx, y = dy, z = dz;
      sd[0] += x; sd[1] += y; sd[2] += z;
      sdd[0] += x * x; sdd[1] += x * y; sdd[2] += x * z; sdd[3] += y * y; sdd[4] += y * z; sdd[5] += z * z;
    });
    pt_num[i] = cnt;
    float l[3] = {0.f, 0.f, 0.f};
    double curv = 0.0;
    if (cnt >= 3) {                                                        // :203-204
      const double inv_n = 1.0 / cnt, alpha = 1.0 / (cnt - 1);
      const float c[6] = {(float)((sdd[0] - sd[0] * sd[0] * inv_n) * alpha), (float)((sdd[1] - sd[0] * sd[1] * inv_n) * alpha),
                          (float)((sdd[2] - sd[0] * sd[2] * inv_n) * alpha), (float)((sdd[3] - sd[1] * sd[1] * inv_n) * alpha),
                          (float)((sdd[4] - sd[1] * sd[2] * inv_n) * alpha), (float)((sdd[5] - sd[2] * sd[2] * inv_n) * alpha)};
      sym3_eig_f32(c, l);
      const double l1 = l[0], l2 = l[1], l3 = l[2];                        // :220-222 (float values held in doubles)
      curv = (l1 + l2 + l3) == 0 ? 0.0 : l3 / (l1 + l2 + l3);              // :224-231
    }
    lam[3 * (size_t)i] = l[0]; lam[3 * (size_t)i + 1] = l[1]; lam[3 * (size_t)i + 2] = l[2];
    curvature[i] = curv;
  }
  return 0;
}

// pruneUnstablePoints + nonMaximaSuppression (include/keypoint_detect.hpp:132-191).  Returns the keypoint count;
// kp_idx receives point indices in the order the reference emits them (descending curvature).
int orc_detect_keypoints(const float *xyz, int n, const float *lam, const double *curvature, const int *pt_num,
                         float ratio_max, int min_pts, float nms_radius, int *kp_idx) {
  std::vector<int> cand;
  for (int i = 0; i < n; ++i) {                                            // :134-144
    const float ratio1 = (float)((double)lam[3 * (size_t)i + 1] / (double)lam[3 * (size_t)i]);
    const float ratio2 = (float)((double)lam[3 * (size_t)i + 2] / (double)lam[3 * (size_t)i + 1]);
    if (ratio1 < ratio_max && ratio2 < ratio_max && pt_num[i] > min_pts) cand.push_back(i);
  }
  std::stable_sort(cand.begin(), cand.end(), [&](int a, int b) { return curvature[a] > curvature[b]; });   // :151
  const int m = (int)cand.size();
  Grid g;
  g.build(xyz, cand.data(), m, nms_radius);
  const float r2 = nms_radius * nms_radius;
  std::vector<char> visited(m, 0);
  int nk = 0;
  for (int r = 0; r < m; ++r) {                                            // :169-188: lowest unvisited rank first
    if (visited[r]) continue;
    kp_idx[nk++] = cand[r];
    const float *q = xyz + 3 * (size_t)cand[r];
    g.for_neighbours(q, [&](int k) {
      const float *p = xyz + 3 * (size_t)cand[k];
      const float dx = p[0] - q[0], dy = p[1] - q[1], dz = p[2] - q[2];
      if (dx * dx + dy * dy + dz * dz < r2) visited[k] = 1;
    });
    visited[r] = 1;
  }
  return nk;
}

}  // extern "C"
