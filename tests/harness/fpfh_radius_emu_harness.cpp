// fpfh_radius_emu_harness.cpp — the radius FPFH estimator of gh-icp_b200/csrc/ghicp_prep.cu (prep_fpfh_radius: k_rad_mark,
// k_rad_count, k_rad_fill, the segmented sort, k_rad_normals, k_rad_spfh, k_rad_fpfh) compiled as plain C++ against the host
// emulation shim (tests/harness/cuda_emu), every CUDA thread a fiber.  Unlike the C ABI it also hands back the work counts
// and the grid it used.  TEST INFRASTRUCTURE ONLY (tests/test_fpfh_radius.py).
#define GHICP_EMU_HOST 1
#include "../../gh-icp_b200/csrc/ghicp_kernels.cu"
#include "../../gh-icp_b200/csrc/ghicp_auction.cu"
#include "../../gh-icp_b200/csrc/ghicp_fpfh.cu"
#include "../../gh-icp_b200/csrc/ghicp_solvers.cu"
#include "../../gh-icp_b200/csrc/ghicp_prep.cu"

namespace ghicp_b200 {
void set_error(Ctx *c, const std::string &msg) { if (c) c->err = msg; }   // the C ABI's error slot is not part of this build
}

// stats [8] = {normal-radius entries, feature-radius entries, SPFH points, rings (normal), rings (feature), entries counted,
// budget, -}; cell = grid cell edge
extern "C" int emu_fpfh_radius(const float *xyz, int n, const int *idx, int nidx, float rn, float rf, long long nb_max, float *fpfh,
                               float *normals, int *status, long long *stats, float *cell) {
  ghicp_b200::FpfhRadiusStats s;
  const cudaError_t e = ghicp_b200::prep_fpfh_radius(nullptr, xyz, n, idx, idx ? nidx : n, rn, rf, nb_max, fpfh, normals, status,
                                                     nullptr, nullptr, &s);
  stats[0] = s.nb_n; stats[1] = s.nb_f; stats[2] = s.spfh_points; stats[3] = s.rings_n; stats[4] = s.rings_f;
  stats[5] = s.needed; stats[6] = s.budget; stats[7] = 0;
  *cell = s.cell;
  return (int)e;
}
