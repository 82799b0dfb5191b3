// sor_oracle.cpp — the canonical statistical outlier removal of DESIGN.md §3.16 (CFilter::SORFilter, PCL's
// StatisticalOutlierRemoval) on the CPU.  TEST INFRASTRUCTURE ONLY (tests/sor_oracle.py compiles and loads it).
// Written from the definition, not from the kernels:
//   F = the finite points, k_eff = min(mean_k, |F| - 1); for p in F the k_eff smallest float32 d2 = (dx*dx + dy*dy) + dz*dz
//   (dx = p.x - q.x) to the other points q of F (by index: duplicates of p count, at 0), in ascending (d2, index) order;
//   d_p = (float)(sum of sqrt((double)d2) in that order / k_eff), 0 when k_eff = 0; NaN for a non-finite point.
//   mean = sum d / |F|, stddev = sqrt(sum (d - mean)^2 / (|F| - 1)) (0 when |F| <= 1), both summed in index order;
//   threshold = mean + std_mul * stddev; kept = the finite p with !((double)d_p > threshold), ascending.
// Two neighbour searches, which must give the same bits: brute force (grid = 0) and a hashed uniform grid searched in
// Chebyshev rings of cells until no unvisited cell can hold a closer point (grid = 1; brute force past 16 rings; the
// queries run on all hardware threads).
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <thread>
#include <unordered_map>
#include <vector>

namespace {

typedef unsigned long long u64;

u64 key(float d2, int idx) {
  unsigned b;
  std::memcpy(&b, &d2, 4);
  return ((u64)b << 32) | (unsigned)idx;   // d2 >= 0: its bits order like its value
}
float key_d2(u64 k) {
  const unsigned b = (unsigned)(k >> 32);
  float f;
  std::memcpy(&f, &b, 4);
  return f;
}
float d2f(const float *p, const float *q) {
  const float dx = p[0] - q[0], dy = p[1] - q[1], dz = p[2] - q[2];
  return (dx * dx + dy * dy) + dz * dz;
}
bool finite3(const float *p) { return std::isfinite(p[0]) && std::isfinite(p[1]) && std::isfinite(p[2]); }

// d_p from the candidate keys (every other finite point, or a superset of the k nearest)
float mean_of_smallest(std::vector<u64> &c, int k) {
  if (k == 0) return 0.f;
  std::nth_element(c.begin(), c.begin() + (k - 1), c.end());
  std::sort(c.begin(), c.begin() + k);
  double s = 0.0;
  for (int j = 0; j < k; ++j) s += std::sqrt((double)key_d2(c[j]));
  return (float)(s / (double)k);
}

struct Grid {
  double mn[3], cell;
  long long ext[3];
  std::unordered_map<u64, std::vector<int>> cells;
  static u64 ck(long long x, long long y, long long z) { return ((u64)x << 42) | ((u64)y << 21) | (u64)z; }
  void coords(const float *p, long long c[3]) const {
    for (int a = 0; a < 3; ++a) c[a] = (long long)std::floor(((double)p[a] - mn[a]) / cell);
  }
};

}  // namespace

extern "C" int sor_oracle(const float *xyz, long long n, int mean_k, double std_mul, int grid, float *dist, int *kept,
                          long long *n_kept, double *stats, long long *counts) {
  std::vector<int> fin;
  for (long long i = 0; i < n; ++i) if (finite3(xyz + 3 * i)) fin.push_back((int)i);
  const long long nf = (long long)fin.size();
  const int k = nf > 0 ? (int)std::min<long long>(mean_k, nf - 1) : 0;
  const float nan = std::nanf("");
  for (long long i = 0; i < n; ++i) dist[i] = nan;
  std::vector<u64> c;
  if (!grid) {
    for (int p : fin) {
      c.clear();
      for (int q : fin) if (q != p) c.push_back(key(d2f(xyz + 3 * (size_t)p, xyz + 3 * (size_t)q), q));
      dist[p] = mean_of_smallest(c, k);
    }
  } else if (nf > 0) {
    Grid g;
    double mx[3];
    for (int a = 0; a < 3; ++a) { g.mn[a] = xyz[3 * (size_t)fin[0] + a]; mx[a] = g.mn[a]; }
    for (int p : fin)
      for (int a = 0; a < 3; ++a) { g.mn[a] = std::min(g.mn[a], (double)xyz[3 * (size_t)p + a]); mx[a] = std::max(mx[a], (double)xyz[3 * (size_t)p + a]); }
    double vol = 1.0, emax = 0.0;
    for (int a = 0; a < 3; ++a) emax = std::max(emax, mx[a] - g.mn[a]);
    for (int a = 0; a < 3; ++a) vol *= std::max(mx[a] - g.mn[a], 1e-3 * emax);
    // a volume guess, then corrected once for a surface's occupancy (aiming at about k / 2 points per occupied cell); the
    // result does not depend on the cell, only the work does
    g.cell = emax > 0.0 ? std::cbrt(vol * (k + 1) / (double)nf) : 1.0;
    for (int pass = 0; pass < 2; ++pass) {
      g.cell = std::max(g.cell, emax / 1048576.0);
      g.cells.clear();
      for (int a = 0; a < 3; ++a) g.ext[a] = (long long)std::floor((mx[a] - g.mn[a]) / g.cell);
      for (int p : fin) {
        long long cc[3];
        g.coords(xyz + 3 * (size_t)p, cc);
        g.cells[Grid::ck(cc[0], cc[1], cc[2])].push_back(p);
      }
      if (pass == 0 && emax > 0.0) g.cell *= std::min(16.0, std::max(1.0 / 16, std::sqrt(0.5 * (k + 1) * g.cells.size() / (double)nf)));
      else break;
    }
    // queries are independent: split them over the hardware threads (each writes only its own dist[p])
    auto run = [&](size_t f0, size_t f1) {
    std::vector<u64> c;
    for (size_t f = f0; f < f1; ++f) {
      const int p = fin[f];
      const float *q = xyz + 3 * (size_t)p;
      long long cc[3];
      g.coords(q, cc);
      long long rmax = 0;
      for (int a = 0; a < 3; ++a) rmax = std::max(rmax, std::max(cc[a], g.ext[a] - cc[a]));
      c.clear();
      bool done = k == 0;
      for (long long r = 0; !done && r <= 16; ++r) {
        for (long long x = cc[0] - r; x <= cc[0] + r; ++x)
          for (long long y = cc[1] - r; y <= cc[1] + r; ++y)
            for (long long z = cc[2] - r; z <= cc[2] + r; ++z) {
              if (std::max(std::llabs(x - cc[0]), std::max(std::llabs(y - cc[1]), std::llabs(z - cc[2]))) != r) continue;
              if (x < 0 || y < 0 || z < 0 || x > g.ext[0] || y > g.ext[1] || z > g.ext[2]) continue;
              auto it = g.cells.find(Grid::ck(x, y, z));
              if (it == g.cells.end()) continue;
              for (int o : it->second) if (o != p) c.push_back(key(d2f(q, xyz + 3 * (size_t)o), o));
            }
        if (r >= rmax) { done = true; break; }
        if ((long long)c.size() >= k) {   // every unvisited point is at least (r - 0.01) cells away on some axis
          std::nth_element(c.begin(), c.begin() + (k - 1), c.end());
          const double lb = ((double)r - 0.01) * g.cell;
          if (lb > 0.0 && (double)key_d2(c[k - 1]) < lb * lb * (1.0 - 1e-5)) done = true;
        }
      }
      if (!done) {                        // far outlier: brute force
        c.clear();
        for (int o : fin) if (o != p) c.push_back(key(d2f(q, xyz + 3 * (size_t)o), o));
      }
      dist[p] = mean_of_smallest(c, k);
    }
    };
    const size_t T = std::max(1u, std::min(64u, std::thread::hardware_concurrency()));
    std::vector<std::thread> pool;
    for (size_t t = 0; t < T; ++t) pool.emplace_back(run, fin.size() * t / T, fin.size() * (t + 1) / T);
    for (std::thread &t : pool) t.join();
  }
  double sum = 0.0, ss = 0.0;
  for (int p : fin) sum += (double)dist[p];
  const double mean = nf > 0 ? sum / (double)nf : 0.0;
  for (int p : fin) { const double v = (double)dist[p] - mean; ss += v * v; }
  const double sd = nf > 1 ? std::sqrt(ss / (double)(nf - 1)) : 0.0;
  const double thr = mean + std_mul * sd;
  long long m = 0;
  for (int p : fin) if (!((double)dist[p] > thr)) kept[m++] = p;
  *n_kept = m;
  stats[0] = mean; stats[1] = sd; stats[2] = thr;
  counts[0] = nf; counts[1] = k;
  return 0;
}
