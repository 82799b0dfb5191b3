// overlap_oracle.cpp — the canonical overlap and fitness of DESIGN.md §3.12, one thread (TEST INFRASTRUCTURE, built with
// -ffp-contract=off so that every float32 operation is rounded separately).
//   p_i   = a_i moved by the float32 transform: ((R00 x + R01 y) + R02 z) + t0 (R, t rounded once from the double matrix)
//   d2_i  = min over B of (dx*dx + dy*dy) + dz*dz, dx = p.x - b.x; reported when d2_i <= L = max(r*r, max_range), else +inf
//   overlap = #{d2_i < r*r} (r*r a float32 product), n_fit = #{finite d2_i <= max_range}; sums in double in point order.
// Two search modes give the same bits (a minimum does not depend on the visiting order): brute force over B, and a uniform
// grid of its own (cells hashed in a sorted table, rings stopped by a plain double bound) for clouds of a million points.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <limits>
#include <utility>
#include <vector>

namespace {

inline float d2f(float qx, float qy, float qz, const float *b) {
  const float dx = qx - b[0], dy = qy - b[1], dz = qz - b[2];
  return (dx * dx + dy * dy) + dz * dz;
}

struct Grid {
  double mn[3], h;
  long long gm[3];
  std::vector<std::pair<uint64_t, int>> cells;   // (cell key, first point) sorted
  std::vector<int> order;                        // points sorted by cell
  std::vector<int> start;                        // run start per table entry (+ end)
  const float *B;
  uint64_t key(long long x, long long y, long long z) const { return ((uint64_t)x << 42) | ((uint64_t)y << 21) | (uint64_t)z; }
  long long coord(double v, int a) const {
    double f = std::floor((v - mn[a]) / h);
    if (!(f > 0)) return 0;
    return f > (double)gm[a] ? gm[a] : (long long)f;
  }
  void build(const float *b, long long nb) {
    B = b;
    double mx[3];
    for (int a = 0; a < 3; ++a) { mn[a] = b[a]; mx[a] = b[a]; }
    for (long long j = 0; j < nb; ++j)
      for (int a = 0; a < 3; ++a) { mn[a] = std::min(mn[a], (double)b[3 * j + a]); mx[a] = std::max(mx[a], (double)b[3 * j + a]); }
    double ext = 0.0;
    for (int a = 0; a < 3; ++a) ext = std::max(ext, mx[a] - mn[a]);
    h = std::max(std::cbrt(std::max(ext * ext * ext, 1e-30) * 4.0 / (double)nb), ext / 1.0e6);
    if (!(h > 0)) h = 1.0;
    for (int a = 0; a < 3; ++a) gm[a] = (long long)std::floor((mx[a] - mn[a]) / h);
    std::vector<std::pair<uint64_t, int>> kv((size_t)nb);
    for (long long j = 0; j < nb; ++j) kv[j] = {key(coord(b[3 * j], 0), coord(b[3 * j + 1], 1), coord(b[3 * j + 2], 2)), (int)j};
    std::sort(kv.begin(), kv.end());
    order.resize((size_t)nb);
    for (long long j = 0; j < nb; ++j) {
      order[j] = kv[j].second;
      if (j == 0 || kv[j].first != kv[j - 1].first) { cells.push_back({kv[j].first, (int)j}); }
    }
    for (auto &c : cells) start.push_back(c.second);
    start.push_back((int)nb);
  }
  // exact minimum of d2f over B
  float nearest(float qx, float qy, float qz) const {
    const double q[3] = {qx, qy, qz};
    long long c[3];
    for (int a = 0; a < 3; ++a) c[a] = coord(q[a], a);
    long long kmax = 0;
    for (int a = 0; a < 3; ++a) kmax = std::max(kmax, std::max(c[a], gm[a] - c[a]));
    // how far the query lies outside the grid's box, per axis: every cell is at least that far on that axis
    double out2 = 0.0;
    for (int a = 0; a < 3; ++a) {
      const double lo = mn[a] + c[a] * h, hi = lo + h;
      const double d = q[a] < lo ? lo - q[a] : (q[a] > hi ? q[a] - hi : 0.0);
      out2 += d * d;
    }
    float best = std::numeric_limits<float>::infinity();
    for (long long k = 0; k <= kmax; ++k) {
      for (long long x = c[0] - k; x <= c[0] + k; ++x) {
        if (x < 0 || x > gm[0]) continue;
        for (long long y = c[1] - k; y <= c[1] + k; ++y) {
          if (y < 0 || y > gm[1]) continue;
          for (long long z = c[2] - k; z <= c[2] + k; ++z) {
            if (z < 0 || z > gm[2]) continue;
            if (std::max(std::llabs(x - c[0]), std::max(std::llabs(y - c[1]), std::llabs(z - c[2]))) != k) continue;
            auto it = std::lower_bound(cells.begin(), cells.end(), std::make_pair(key(x, y, z), -1));
            if (it == cells.end() || it->first != key(x, y, z)) continue;
            const size_t e = (size_t)(it - cells.begin());
            for (int s = start[e]; s < start[e + 1]; ++s) best = std::min(best, d2f(qx, qy, qz, B + 3 * (size_t)order[s]));
          }
        }
      }
      // a cell beyond ring k lies more than k h - 1e-6 h away on one axis (cells of points are computed in double here)
      // and outside the box on the others as the query is
      const double lb = std::max(0.0, (double)k * h - 1e-6 * h);
      if ((double)best < (lb * lb + out2) * (1.0 - 1e-5)) break;
    }
    return best;
  }
};

}  // namespace

extern "C" int overlap_oracle(const float *A, long long na, const float *B, long long nb, const double *Rt16, float r,
                              double max_range, int grid, float *d2, long long *counts /* overlap, n_fit */,
                              double *sums /* overlap sum, fit sum */) {
  if (na <= 0 || nb <= 0) return -1;
  float rt[12];
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) rt[3 * i + j] = Rt16 ? (float)Rt16[j * 4 + i] : (i == j ? 1.f : 0.f);
    rt[9 + i] = Rt16 ? (float)Rt16[12 + i] : 0.f;
  }
  const float r2 = r * r;
  const double L = std::max((double)r2, max_range);
  Grid G;
  if (grid) G.build(B, nb);
  long long ov = 0, nf = 0;
  double so = 0.0, sf = 0.0;
  for (long long i = 0; i < na; ++i) {
    const float x = A[3 * i], y = A[3 * i + 1], z = A[3 * i + 2];
    const float px = ((rt[0] * x + rt[1] * y) + rt[2] * z) + rt[9];
    const float py = ((rt[3] * x + rt[4] * y) + rt[5] * z) + rt[10];
    const float pz = ((rt[6] * x + rt[7] * y) + rt[8] * z) + rt[11];
    float best = std::numeric_limits<float>::infinity();
    if (grid) best = G.nearest(px, py, pz);
    else
      for (long long j = 0; j < nb; ++j) best = std::min(best, d2f(px, py, pz, B + 3 * j));
    if (!((double)best <= L)) best = std::numeric_limits<float>::infinity();
    d2[i] = best;
    if (best < r2) { ++ov; so += (double)best; }
    if (best != std::numeric_limits<float>::infinity() && (double)best <= max_range) { ++nf; sf += (double)best; }
  }
  counts[0] = ov; counts[1] = nf;
  sums[0] = so; sums[1] = sf;
  return 0;
}
