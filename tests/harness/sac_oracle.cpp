// sac_oracle.cpp — the canonical SAC-IA definition (DESIGN.md §3.11), one thread.  TEST INFRASTRUCTURE ONLY: tests/sac_oracle.py
// compiles it (g++ -ffp-contract=off) and checks the product's kernels (gh-icp_b200/csrc/ghicp_sac.cu) against it.
//
// The reference's FPFHfeature::fpfhalign (include/fpfh.hpp:117-133) is PCL SampleConsensusInitialAlignment; PCL is not pinned
// and its std::rand() is global state, so the definition fixes (per hypothesis h = 0 .. H-1, independently):
//   samples   draws r = sac_draw(seed, h, d), d = 0, 1, ... (ghicp_sac.h, shared with the kernels); candidate sac_index(r, n_s),
//             accepted when it differs from every sample already chosen and sac_sample_dist to each of them >= min_sample_distance;
//             3 n_s rejections in a row: the hypothesis is invalid (never chosen, counted)
//   corresp.  per sample in sample order: the k_eff = min(k, n_t) nearest target histograms by sac_feat_d2 (float32, bins in
//             order), ascending (d2, index); position (next draw) mod k_eff
//   transform FP64 means and cross-covariance of the pairs, rounded once to float32, the float32 Umeyama of the loop
//   error     every source point moved in float32, ((R00 x + R01 y) + R02 z) + t0; exact nearest target by
//             (dx*dx + dy*dy) + dz*dz; term sac_term_fx (d2 / thr if d2 <= thr else 1, in units of 2^-32); summed as integers
//   choice    smallest error, ties to the smallest h
//   result    Rt = the float transform widened, error = sum * 2^-32, fitness = mean d2 over the points with d2 <= thr (point
//             order, double), inliers, h*, invalid count
// The nearest-neighbour search here is a hash-free sorted grid with cell edge >= sqrt(thr) and the 27 cells around the query:
// every point within the threshold lies in them, which is all the error and the fitness need — a different index from the
// kernels' ring walk on purpose.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <utility>
#include <vector>

#include "../../gh-icp_b200/csrc/ghicp_sac.h"

namespace {

using namespace ghicp_sac;

// ---- float32 SVD / Umeyama: the same text as the device code (gh-icp_b200/csrc/ghicp_device.cuh) and oracle/ghicp_oracle.cpp
void svd3_f32(const float A[9], float U[9], float S[3], float V[9]) {
  float amax = 0.f;   // scale by 2^-e, 2^e the power of two above max |A_ij| (zero or non-finite A: e = 0)
  bool finite = true;
  for (int i = 0; i < 9; ++i) { const float m = std::fabs(A[i]); finite = finite && std::isfinite(m); amax = m > amax ? m : amax; }
  int e = 0;
  if (finite && amax > 0.f) std::frexp(amax, &e);
  float a[9];
  for (int i = 0; i < 9; ++i) a[i] = std::ldexp(A[i], -e);
  float v[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  const float tol = 1e-7f;
  for (int sweep = 0; sweep < 30; ++sweep) {
    int rotated = 0;
    for (int p = 0; p < 2; ++p) {
      for (int q = p + 1; q < 3; ++q) {
        float alpha = 0.f, beta = 0.f, gamma = 0.f;
        for (int i = 0; i < 3; ++i) {
          alpha = alpha + a[i * 3 + p] * a[i * 3 + p];
          beta = beta + a[i * 3 + q] * a[i * 3 + q];
          gamma = gamma + a[i * 3 + p] * a[i * 3 + q];
        }
        if (gamma == 0.f || std::fabs(gamma) <= tol * std::sqrt(alpha * beta)) continue;
        rotated = 1;
        float zeta = (beta - alpha) / (2.0f * gamma);
        float t = 1.0f / (std::fabs(zeta) + std::sqrt(1.0f + zeta * zeta));
        if (zeta < 0.f) t = -t;
        float c = 1.0f / std::sqrt(1.0f + t * t);
        float s = c * t;
        for (int i = 0; i < 3; ++i) {
          float ap = a[i * 3 + p], aq = a[i * 3 + q];
          a[i * 3 + p] = c * ap - s * aq;
          a[i * 3 + q] = s * ap + c * aq;
          float vp = v[i * 3 + p], vq = v[i * 3 + q];
          v[i * 3 + p] = c * vp - s * vq;
          v[i * 3 + q] = s * vp + c * vq;
        }
      }
    }
    if (!rotated) break;
  }
  float sv[3];
  for (int k = 0; k < 3; ++k) {
    float n2 = 0.f;
    for (int i = 0; i < 3; ++i) n2 = n2 + a[i * 3 + k] * a[i * 3 + k];
    sv[k] = std::sqrt(n2);
  }
  int idx[3] = {0, 1, 2};
  for (int i = 1; i < 3; ++i)
    for (int j = i; j > 0 && sv[idx[j]] > sv[idx[j - 1]]; --j) std::swap(idx[j], idx[j - 1]);
  float u[9];
  for (int k = 0; k < 3; ++k) {
    int src = idx[k];
    S[k] = sv[src];
    for (int i = 0; i < 3; ++i) {
      V[i * 3 + k] = v[i * 3 + src];
      u[i * 3 + k] = a[i * 3 + src];
    }
  }
  const float tiny = 1e-20f;
  for (int k = 0; k < 2; ++k)
    if (S[k] > tiny)
      for (int i = 0; i < 3; ++i) u[i * 3 + k] = u[i * 3 + k] / S[k];
  if (!(S[0] > tiny)) { u[0] = 1; u[3] = 0; u[6] = 0; }
  if (!(S[1] > tiny)) {
    float x = u[0], y = u[3], z = u[6];
    float bx, by, bz;
    if (std::fabs(x) <= std::fabs(y) && std::fabs(x) <= std::fabs(z)) { bx = 1; by = 0; bz = 0; }
    else if (std::fabs(y) <= std::fabs(z)) { bx = 0; by = 1; bz = 0; }
    else { bx = 0; by = 0; bz = 1; }
    float cx = y * bz - z * by, cy = z * bx - x * bz, cz = x * by - y * bx;
    float n = std::sqrt(cx * cx + cy * cy + cz * cz);
    u[1] = cx / n; u[4] = cy / n; u[7] = cz / n;
  }
  if (S[2] > 1e-6f * S[0] && S[2] > tiny) {
    for (int i = 0; i < 3; ++i) u[i * 3 + 2] = u[i * 3 + 2] / S[2];
  } else {
    u[2] = u[3] * u[7] - u[6] * u[4];
    u[5] = u[6] * u[1] - u[0] * u[7];
    u[8] = u[0] * u[4] - u[3] * u[1];
  }
  for (int i = 0; i < 9; ++i) U[i] = u[i];
  for (int k = 0; k < 3; ++k) S[k] = std::ldexp(S[k], e);
}
float det3_f32(const float m[9]) {
  return m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) + m[2] * (m[3] * m[7] - m[4] * m[6]);
}
// R row-major [9], t [3]
void umeyama_f32(const float mu_s[3], const float mu_d[3], const float sigma[9], float R[9], float t[3]) {
  float U[9], S[3], V[9];
  svd3_f32(sigma, U, S, V);
  float sgn[3] = {1.f, 1.f, 1.f};
  if (det3_f32(U) * det3_f32(V) < 0.f) sgn[2] = -1.f;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      float acc = 0.f;
      for (int k = 0; k < 3; ++k) acc = acc + (U[i * 3 + k] * sgn[k]) * V[j * 3 + k];
      R[i * 3 + j] = acc;
    }
  for (int i = 0; i < 3; ++i) {
    float acc = 0.f;
    for (int k = 0; k < 3; ++k) acc = acc + R[i * 3 + k] * mu_s[k];
    t[i] = mu_d[i] - acc;
  }
}

void feat_knn(const float *f, const float *Ft, int nt, int ke, int *out) {
  std::vector<std::pair<float, int>> d((size_t)nt);
  for (int j = 0; j < nt; ++j) d[j] = {sac_feat_d2(f, Ft + 33 * (size_t)j), j};
  std::partial_sort(d.begin(), d.begin() + ke, d.end());   // pairs order by (d2, index)
  for (int j = 0; j < ke; ++j) out[j] = d[j].second;
}

// target points within the 27 cells of edge >= sqrt(thr) around a query = every point that can be within the threshold
struct NearGrid {
  double inv = 0.0, mn[3] = {0, 0, 0};
  std::vector<std::pair<uint64_t, int>> cells;   // (key, point), sorted
  const float *Q = nullptr;
  void build(const float *q, int n, float thr) {
    Q = q;
    for (int a = 0; a < 3; ++a) { mn[a] = q[a]; for (int i = 1; i < n; ++i) mn[a] = std::min(mn[a], (double)q[3 * (size_t)i + a]); }
    inv = 1.0 / (std::sqrt((double)thr) * 1.01 + 1e-30);
    cells.resize(n);
    for (int i = 0; i < n; ++i) cells[i] = {key(cell(q + 3 * (size_t)i, 0), cell(q + 3 * (size_t)i, 1), cell(q + 3 * (size_t)i, 2)), i};
    std::sort(cells.begin(), cells.end());
  }
  long long cell(const float *p, int a) const { return (long long)std::floor(((double)p[a] - mn[a]) * inv); }
  static uint64_t key(long long x, long long y, long long z) {
    return ((uint64_t)(x + (1 << 20)) << 42) | ((uint64_t)(y + (1 << 20)) << 21) | (uint64_t)(z + (1 << 20));
  }
  // +inf when nothing is within the 27 cells (keys of far cells may collide: extra real points never lower the true minimum)
  float nearest_d2(const float q[3]) const {
    float best = INFINITY;
    const long long cx = cell(q, 0), cy = cell(q, 1), cz = cell(q, 2);
    for (int dx = -1; dx <= 1; ++dx)
      for (int dy = -1; dy <= 1; ++dy)
        for (int dz = -1; dz <= 1; ++dz) {
          const uint64_t k = key(cx + dx, cy + dy, cz + dz);
          auto it = std::lower_bound(cells.begin(), cells.end(), std::make_pair(k, -1));
          for (; it != cells.end() && it->first == k; ++it) {
            const float *p = Q + 3 * (size_t)it->second;
            const float ex = q[0] - p[0], ey = q[1] - p[1], ez = q[2] - p[2];
            const float d2 = (ex * ex + ey * ey) + ez * ez;
            best = d2 < best ? d2 : best;
          }
        }
    return best;
  }
};

void move(const float R[9], const float t[3], const float *p, float o[3]) {
  for (int i = 0; i < 3; ++i) o[i] = ((R[3 * i] * p[0] + R[3 * i + 1] * p[1]) + R[3 * i + 2] * p[2]) + t[i];
}

}  // namespace

extern "C" {

// the float32 Umeyama of the hypotheses (and of icp_oracle.cpp's steps) on given float32 moments: R row-major [9], t [3]
void sac_oracle_umeyama(const float *mu_s, const float *mu_d, const float *sigma, float *R, float *t) {
  umeyama_f32(mu_s, mu_d, sigma, R, t);
}

// the k_eff nearest target histograms of the source histograms idx[m] (ascending (d2, index)); returns k_eff
int sac_oracle_feat_knn(const float *Fs, const int *idx, int m, const float *Ft, int nt, int k, int *out) {
  const int ke = std::min(k, nt);
  for (int i = 0; i < m; ++i) feat_knn(Fs + 33 * (size_t)idx[i], Ft, nt, ke, out + (size_t)i * ke);
  return ke;
}

// per-point nearest d2 (+inf beyond the threshold) under R (row-major) / t: the oracle's error search on its own
void sac_oracle_nearest(const float *P, int ns, const float *Q, int nt, const float *rt12, float thr, float *d2) {
  NearGrid g;
  g.build(Q, nt, thr);
  for (int i = 0; i < ns; ++i) {
    float x[3];
    move(rt12, rt12 + 9, P + 3 * (size_t)i, x);
    const float v = g.nearest_d2(x);
    d2[i] = v <= thr ? v : INFINITY;
  }
}

// The whole definition.  Per hypothesis: samples [H][nsamp] (-1 if invalid), valid [H], corr [H][nsamp] (-1 if invalid),
// rt [H][12] (zeros if invalid), err [H] (0 if invalid).  Result: Rt16 column-major, dres = {error, fitness},
// ires = {inliers, best hypothesis, invalid hypotheses}.
int sac_oracle(const float *P, const float *Fs, int ns, const float *Q, const float *Ft, int nt, int H, int nsamp, int k, float msd,
               float thr, unsigned long long seed, int *samples, int *valid, int *corr, float *rt, unsigned long long *err,
               double *Rt16, double *dres, int *ires) {
  const int ke = std::min(k, nt);
  NearGrid g;
  g.build(Q, nt, thr);
  std::vector<int> knn_cache((size_t)ns * ke, -1);
  std::vector<char> have((size_t)ns, 0);
  long long best = -1;
  unsigned long long best_err = 0;
  int invalid = 0;
  for (int h = 0; h < H; ++h) {
    int s[SAC_MAX_SAMPLES];
    int n = 0, rej = 0;
    uint32_t d = 0;
    bool ok = true;
    while (n < nsamp) {
      const int c = sac_index(sac_draw(seed, (uint32_t)h, d++), ns);
      bool acc = true;
      for (int j = 0; j < n && acc; ++j) acc = s[j] != c && sac_sample_dist(P + 3 * (size_t)c, P + 3 * (size_t)s[j]) >= msd;
      if (acc) { s[n++] = c; rej = 0; }
      else if (++rej >= 3 * ns) { ok = false; break; }
    }
    valid[h] = ok ? 1 : 0;
    float *o = rt + 12 * (size_t)h;
    for (int i = 0; i < 12; ++i) o[i] = 0.f;
    err[h] = 0;
    for (int j = 0; j < nsamp; ++j) { samples[(size_t)h * nsamp + j] = ok ? s[j] : -1; corr[(size_t)h * nsamp + j] = -1; }
    if (!ok) { ++invalid; continue; }
    int c[SAC_MAX_SAMPLES];
    for (int j = 0; j < nsamp; ++j) {
      if (!have[s[j]]) { feat_knn(Fs + 33 * (size_t)s[j], Ft, nt, ke, &knn_cache[(size_t)s[j] * ke]); have[s[j]] = 1; }
      const uint64_t r = sac_draw(seed, (uint32_t)h, d++);
      c[j] = knn_cache[(size_t)s[j] * ke + (int)(r % (uint64_t)ke)];
      corr[(size_t)h * nsamp + j] = c[j];
    }
    double ms[3] = {0, 0, 0}, md[3] = {0, 0, 0};
    for (int j = 0; j < nsamp; ++j)
      for (int a = 0; a < 3; ++a) { ms[a] += (double)P[3 * (size_t)s[j] + a]; md[a] += (double)Q[3 * (size_t)c[j] + a]; }
    double mus[3], mud[3];
    for (int a = 0; a < 3; ++a) { mus[a] = ms[a] / nsamp; mud[a] = md[a] / nsamp; }
    double acc[9] = {0};
    for (int j = 0; j < nsamp; ++j) {
      double ds[3], dd[3];
      for (int a = 0; a < 3; ++a) { ds[a] = (double)P[3 * (size_t)s[j] + a] - mus[a]; dd[a] = (double)Q[3 * (size_t)c[j] + a] - mud[a]; }
      for (int r = 0; r < 3; ++r)
        for (int cc = 0; cc < 3; ++cc) acc[r * 3 + cc] += dd[r] * ds[cc];
    }
    float mu_s[3], mu_d[3], sigma[9];
    for (int a = 0; a < 3; ++a) { mu_s[a] = (float)mus[a]; mu_d[a] = (float)mud[a]; }
    for (int a = 0; a < 9; ++a) sigma[a] = (float)(acc[a] / nsamp);
    umeyama_f32(mu_s, mu_d, sigma, o, o + 9);
    uint64_t e = 0;
    for (int i = 0; i < ns; ++i) {
      float x[3];
      move(o, o + 9, P + 3 * (size_t)i, x);
      e += sac_term_fx(g.nearest_d2(x), thr);
    }
    err[h] = e;
    if (best < 0 || e < best_err) { best = h; best_err = e; }   // strict <: ties keep the first
  }
  float R[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, t[3] = {0, 0, 0};
  if (best >= 0) { std::memcpy(R, rt + 12 * (size_t)best, sizeof(R)); std::memcpy(t, rt + 12 * (size_t)best + 9, sizeof(t)); }
  uint64_t e = 0;
  double fit = 0.0;
  int inl = 0;
  for (int i = 0; i < ns; ++i) {
    float x[3];
    move(R, t, P + 3 * (size_t)i, x);
    const float d2 = g.nearest_d2(x);
    e += sac_term_fx(d2, thr);
    if (d2 <= thr) { fit += (double)d2; ++inl; }
  }
  for (int i = 0; i < 16; ++i) Rt16[i] = 0.0;
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) Rt16[j * 4 + i] = (double)R[3 * i + j];
    Rt16[12 + i] = (double)t[i];
  }
  Rt16[15] = 1.0;
  dres[0] = (double)e / SAC_FX_ONE;
  dres[1] = inl > 0 ? fit / inl : DBL_MAX;
  ires[0] = inl; ires[1] = (int)best; ires[2] = invalid;
  return 0;
}

}  // extern "C"
