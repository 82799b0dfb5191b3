// sac_emu_harness.cpp — the SAC-IA kernels of gh-icp_b200/csrc/ghicp_sac.cu (sac_run) compiled as plain C++ against the host
// emulation shim (tests/harness/cuda_emu), every CUDA thread a fiber.  Unlike the C ABI it also hands back the per-hypothesis
// intermediates (samples, correspondences, transforms, integer errors).  TEST INFRASTRUCTURE ONLY (tests/test_sac_ia.py).
#define GHICP_EMU_HOST 1
#include "../../gh-icp_b200/csrc/ghicp_kernels.cu"
#include "../../gh-icp_b200/csrc/ghicp_auction.cu"
#include "../../gh-icp_b200/csrc/ghicp_fpfh.cu"
#include "../../gh-icp_b200/csrc/ghicp_solvers.cu"
#include "../../gh-icp_b200/csrc/ghicp_prep.cu"
#include "../../gh-icp_b200/csrc/ghicp_sac.cu"

namespace ghicp_b200 {
void set_error(Ctx *c, const std::string &msg) { if (c) c->err = msg; }   // the C ABI's error slot is not part of this build
}

extern "C" int emu_sac(const float *P, const float *Fs, int ns, const float *Q, const float *Ft, int nt, int H, int nsamp, int k,
                       float msd, float thr, unsigned long long seed, int *samples, int *valid, int *corr, float *rt,
                       unsigned long long *err, double *Rt16, double *dres /* error, fitness, cell */, int *ires /* inliers, best, invalid */) {
  ghicp_sac_params p{};
  p.max_iterations = H; p.nr_samples = nsamp; p.k_correspondences = k; p.min_sample_distance = msd; p.corr_dist_threshold = thr;
  p.seed = seed;
  ghicp_sac_result r{};
  ghicp_b200::SacDebug dbg;
  dbg.samples = samples; dbg.valid = valid; dbg.corr = corr; dbg.rt = rt; dbg.err = err;
  const cudaError_t e = ghicp_b200::sac_run(P, Fs, ns, Q, Ft, nt, &p, &r, &dbg);
  for (int i = 0; i < 16; ++i) Rt16[i] = r.Rt[i];
  dres[0] = r.error; dres[1] = r.fitness; dres[2] = dbg.cell;
  ires[0] = r.inliers; ires[1] = r.best_hypothesis; ires[2] = r.invalid_hypotheses;
  return (int)e;
}
