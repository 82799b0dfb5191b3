// ghicp_sac.h — the parts of the canonical SAC-IA definition (DESIGN.md §3.11) that the kernels (ghicp_sac.cu) and the CPU
// oracle (tests/harness/sac_oracle.cpp) must evaluate with the same text: the random draws, the sample distance and the
// fixed-point error term.  Host + device, no CUDA header needed.
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define GHICP_SAC_HD __host__ __device__ __forceinline__
#else
#define GHICP_SAC_HD inline
#endif

namespace ghicp_sac {

constexpr int SAC_MAX_SAMPLES = 8;   // nr_samples in 3 .. SAC_MAX_SAMPLES
constexpr int SAC_KMAX = 32;         // k_correspondences in 1 .. SAC_KMAX (the sorted top-k list lives in registers)
constexpr double SAC_FX_ONE = 4294967296.0;   // 2^32: one error unit of the fixed-point sums

// SplitMix64's finaliser (Steele, Lea, Flood: "Fast splittable pseudorandom number generators", 2014)
GHICP_SAC_HD uint64_t splitmix64_mix(uint64_t z) {
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
// Draw d of hypothesis h: output number c = h * 2^32 + d of the SplitMix64 stream whose state starts at mix(seed), i.e.
// mix(mix(seed) + (c + 1) * golden gamma).  Every (seed, h, d) names one draw, so hypotheses are independent of the order in
// which they are evaluated.  d counts the sample draws (rejected ones included) and then the correspondence picks.
GHICP_SAC_HD uint64_t sac_draw(uint64_t seed, uint32_t h, uint32_t d) {
  const uint64_t c = ((uint64_t)h << 32) | (uint64_t)d;
  return splitmix64_mix(splitmix64_mix(seed) + (c + 1ull) * 0x9E3779B97F4A7C15ull);
}
// candidate source index in [0, n): the high 32 bits scaled (Lemire's multiply-shift)
GHICP_SAC_HD int sac_index(uint64_t r, int n) { return (int)(((r >> 32) * (uint64_t)n) >> 32); }
// Euclidean distance of two float32 points, every operation rounded separately: sqrtf((dx*dx + dy*dy) + dz*dz), dx = a.x - b.x
GHICP_SAC_HD float sac_sample_dist(const float *a, const float *b) {
  const float dx = a[0] - b[0], dy = a[1] - b[1], dz = a[2] - b[2];
  return sqrtf((dx * dx + dy * dy) + dz * dz);
}
// squared L2 distance of two 33-bin histograms: float32, bins summed serially in bin order (no FMA: --fmad=false / -ffp-contract=off)
GHICP_SAC_HD float sac_feat_d2(const float *a, const float *b) {
  float d = 0.f;
  for (int j = 0; j < 33; ++j) {
    const float t = a[j] - b[j];
    d = d + t * t;
  }
  return d;
}
// PCL's TruncatedError per point: d2 / thr if d2 <= thr, else 1; as an integer multiple of 2^-32 (round to nearest even) so
// that the sum over the points is exact in any order.  term <= 1, so n points sum to at most n * 2^32 (< 2^64 for n < 2^32).
GHICP_SAC_HD uint64_t sac_term_fx(float d2, float thr) {
  if (!(d2 <= thr)) return (uint64_t)1 << 32;
  const double x = ((double)d2 / (double)thr) * SAC_FX_ONE;   // exact scaling by 2^32 of the double quotient
#if defined(__CUDA_ARCH__)
  return (uint64_t)__double2ull_rn(x);
#else
  return (uint64_t)nearbyint(x);                              // default rounding mode: to nearest even
#endif
}

}  // namespace ghicp_sac
