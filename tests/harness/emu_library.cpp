// emu_library.cpp — the WHOLE C ABI of libghicp_b200.so built for the CPU through the host emulation shim
// (tests/harness/cuda_emu): ghicp_capi.cu (context, iteration orchestration, every extern "C" entry point) on top of ALL of
// the product's kernels — ghicp_kernels.cu, ghicp_stream.cu, ghicp_fdtc.cu, ghicp_auction.cu, ghicp_fpfh.cu,
// ghicp_solvers.cu, ghicp_prep.cu — every CUDA thread a fiber.  The PTX of ghicp_stream.cu (mbarrier, cp.async.bulk) and of
// ghicp_fdtc.cu (mbarrier, cp.async.bulk, wgmma s8 computed per thread on its accumulator fragment) has a host stand-in next
// to each asm statement.
// TEST INFRASTRUCTURE ONLY: tests/test_emulated_abi.py loads it explicitly to run the Python and C++ host layers, the
// command-line driver and the GPU test functions themselves on a machine without a GPU.  The product never loads it;
// libghicp_b200.so has no CPU path.
#define GHICP_EMU_HOST 1
#include "../../gh-icp_b200/csrc/ghicp_kernels.cu"
#include "../../gh-icp_b200/csrc/ghicp_auction.cu"
#include "../../gh-icp_b200/csrc/ghicp_fpfh.cu"
#include "../../gh-icp_b200/csrc/ghicp_solvers.cu"
#include "../../gh-icp_b200/csrc/ghicp_prep.cu"
#include "../../gh-icp_b200/csrc/ghicp_comm.cu"
#include "../../gh-icp_b200/csrc/ghicp_stream.cu"

#include "../../gh-icp_b200/csrc/ghicp_fdtc.cu"

#include "../../gh-icp_b200/csrc/ghicp_capi.cu"

// test controls of the shim's device allocations (tests/test_alloc_failures.py)
extern "C" long long ghicp_emu_live_allocations(void) { return emu_live_allocs; }
extern "C" void ghicp_emu_fail_allocation(long long k) { emu_fail_countdown = k; }   // the k-th allocation from now fails; -1: none
