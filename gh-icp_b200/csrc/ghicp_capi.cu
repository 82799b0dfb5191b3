// ghicp_capi.cu — the C ABI of include/ghicp_b200.h: context management and the per-iteration
// orchestration of GHRegistration::ghicp_reg's loop body (src/ghicp_reg.cpp:49-103).
// Heavy work = CUDA kernels on the ctx stream; the scalar tail of an iteration (Euler angles,
// convergence test, adjustweight, Rt accumulation — src/ghicp_reg.cpp:870-914, 771-789, 93) runs on
// the host from one small read-back per iteration.  There is NO CPU fallback: without a CUDA device
// every entry point fails with GHICP_E_NODEV.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstddef>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>

#include "ghicp_internal.h"
#include "ghicp_sac.h"

#if defined(GHICP_EMU_HOST)
// The CPU emulation of the whole library (tests/harness/emu_library.cpp) compiles the product's .cu files as ONE translation
// unit and lists the kernel files it includes; the SAC-IA kernels join it here, next to the entry points that call them.
// nvcc builds ghicp_sac.cu, ghicp_overlap.cu and ghicp_icp.cu as translation units of their own (Makefile SRCS).
#include "ghicp_sac.cu"
#include "ghicp_overlap.cu"
#include "ghicp_icp.cu"
#endif

namespace ghicp_b200 {

static std::string g_last_error;
static std::mutex g_err_mu;

void set_error(Ctx *c, const std::string &msg) {
  if (c) c->err = msg;
  std::lock_guard<std::mutex> lk(g_err_mu);
  g_last_error = msg;
}

// The ABI code of a CUDA call's result.  On an error: "<who>: <CUDA's message>" becomes the last error (of the context c,
// when given, and of the process), the error is cleared from the runtime, and the code is GHICP_E_NOMEM for an allocation
// failure, GHICP_E_CUDA otherwise.
static int cuda_status(cudaError_t e, const char *who, Ctx *c = nullptr) {
  if (e == cudaSuccess) return GHICP_OK;
  set_error(c, std::string(who) + ": " + cudaGetErrorString(e));
  cudaGetLastError();
  return e == cudaErrorMemoryAllocation ? GHICP_E_NOMEM : GHICP_E_CUDA;
}

#define CK(c, call)                                                \
  do {                                                             \
    cudaError_t e__ = (call);                                      \
    if (e__ != cudaSuccess) return cuda_status(e__, #call, (c));   \
  } while (0)

// The start of every stand-alone and pipeline entry point: a device must exist (GHICP_E_NODEV otherwise) and becomes current
static int enter_device(int device, const char *who) {
  if (ghicp_device_count() <= 0) { set_error(nullptr, std::string(who) + ": no CUDA device"); return GHICP_E_NODEV; }
  return cuda_status(cudaSetDevice(device), who);
}

template <typename T>
static int dev_alloc(Ctx *c, T **p, size_t count) {
  if (*p) { cudaFree(*p); *p = nullptr; }
  if (count == 0) count = 1;
  cudaError_t e = cudaMalloc((void **)p, count * sizeof(T));
  if (e != cudaSuccess) {
    *p = nullptr;
    set_error(c, std::string("cudaMalloc failed: ") + cudaGetErrorString(e));
    cudaGetLastError();
    return GHICP_E_NOMEM;
  }
  return GHICP_OK;
}
// small page-locked workspaces (read-backs): allocated once per context, kept across resizes
template <typename T>
static int host_alloc_once(Ctx *c, T **p, size_t bytes) {
  if (*p) return GHICP_OK;
  if (cudaMallocHost((void **)p, bytes) != cudaSuccess) {
    cudaGetLastError();
    *p = nullptr;
    set_error(c, "cudaMallocHost failed (page-locked workspace)");
    return GHICP_E_NOMEM;
  }
  return GHICP_OK;
}
template <typename T>
static void dev_free(T **p) {
  if (*p) { cudaFree(*p); *p = nullptr; }
}

// Is this host pointer page-locked (cudaMallocHost / ghicp_host_alloc / cudaHostRegister)?  Then the DMA engine reads or
// writes it directly and the pinned staging copy is skipped.
static bool is_pinned(const void *p) {
  cudaPointerAttributes at{};
  if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return at.type == cudaMemoryTypeHost;
}

static int use_device(Ctx *c) { return cuda_status(cudaSetDevice(c->device), "cudaSetDevice", c); }

static void free_all(Ctx *c) {
  dev_free(&c->d_s); dev_free(&c->d_t);
  dev_free(&c->d_bs); dev_free(&c->d_bt); dev_free(&c->d_fd16);
  dev_free(&c->d_fs); dev_free(&c->d_ft); dev_free(&c->d_fdf);
  dev_free(&c->d_fsc); dev_free(&c->d_fscT); dev_free(&c->d_ftc); dev_free(&c->d_ftcT); dev_free(&c->d_tn);
  dev_free(&c->d_ff_srec); dev_free(&c->d_ff_tnT); dev_free(&c->d_ff_tco); dev_free(&c->d_ff_part);
  dev_free(&c->d_ff_rowguess); dev_free(&c->d_ff_colguess); c->fpfh_fast_ready = false;
  dev_free(&c->d_part_cd); dev_free(&c->d_part_idx); dev_free(&c->d_part_stats);
  dev_free(&c->d_row_cd); dev_free(&c->d_row_idx); dev_free(&c->d_col_cd); dev_free(&c->d_col_idx);
  dev_free(&c->d_flags); dev_free(&c->d_sp); dev_free(&c->d_tp); dev_free(&c->d_iter);
  dev_free(&c->d_cnt); dev_free(&c->d_rowptr); dev_free(&c->d_cursor);
  dev_free(&c->d_csr_col); dev_free(&c->d_csr_gain); dev_free(&c->d_colptr); dev_free(&c->d_colcnt);
  dev_free(&c->d_csc_row); dev_free(&c->d_csc_gain);
  dev_free(&c->d_price); dev_free(&c->d_profit); dev_free(&c->d_assign); dev_free(&c->d_owner);
  dev_free(&c->d_bidmax); dev_free(&c->d_bidwin); dev_free(&c->d_bid_obj); dev_free(&c->d_bid_val);
  dev_free(&c->d_bid_aux); dev_free(&c->d_list[0]); dev_free(&c->d_list[1]); dev_free(&c->d_counters);
  dev_free(&c->d_row_fd); dev_free(&c->d_pair_fd); dev_free(&c->d_csr_fd); dev_free(&c->d_xstats);
  dev_free(&c->d_colg_cd); dev_free(&c->d_colg_idx);
  if (c->h_rowptr_cut) { cudaFreeHost(c->h_rowptr_cut); c->h_rowptr_cut = nullptr; }
  dev_free(&c->d_S4); dev_free(&c->d_T4); dev_free(&c->d_sdev); dev_free(&c->d_row_thr); dev_free(&c->d_col_thr);
  dev_free(&c->d_rowbest); dev_free(&c->d_colbest); dev_free(&c->d_rowidx2); dev_free(&c->d_colidx2);
  dev_free(&c->d_cand[0]); dev_free(&c->d_cand[1]);
  dev_free(&c->d_emit); c->emit_cap = 0;
  dev_free(&c->d_xsend); dev_free(&c->d_xrecv); dev_free(&c->d_xcounts); c->xcap = 0;
  if (c->h_xcounts) { cudaFreeHost(c->h_xcounts); c->h_xcounts = nullptr; }
  dev_free(&c->d_tile_sum); c->tile_cap = 0; dev_free(&c->d_solve_part);
  if (c->h_sdev) { cudaFreeHost(c->h_sdev); c->h_sdev = nullptr; }
  if (c->h_iter) { cudaFreeHost(c->h_iter); c->h_iter = nullptr; }
  if (c->h_counters) { cudaFreeHost(c->h_counters); c->h_counters = nullptr; }
  if (c->h_stage) { cudaFreeHost(c->h_stage); c->h_stage = nullptr; c->h_stage_cap = 0; }
  c->csr_cap = c->csc_cap = 0;
}

static void reset_loop_state(Ctx *c) {
  // Energyfunction::init (include/ghicp_reg.h:26-41) + GHRegistration ctor (include/ghicp_reg.h:77-117)
  c->penalty_initial = 2.0;
  c->para1 = 1.0;
  c->para2 = 1.0;
  c->min_cor = 10;
  c->weight_changing_rate = 6;
  c->KM_eps = (c->cfg.km_eps > 0.0) ? c->cfg.km_eps : 0.01;
  c->scale_f = 0.005 * c->cfg.bbx_magnitude;  // double product rounded to float (ghicp_reg.h:40)
  c->iteration = 0;
  c->RMS = 99999;
  c->FDM = 0; c->FDstd = 0; c->IoU = 0;
  c->converge = false;
  c->last_mean = 0.0;
  for (int i = 0; i < 16; ++i) c->Rt_tillnow[i] = (i % 5 == 0) ? 1.0 : 0.0;
  c->RouteHistory::reset();
}

static int ensure_edges(Ctx *c, long long nnz) {
  const size_t need = (size_t)std::max<long long>(nnz, 1);
  int rc;
  if (need > c->csr_cap) {
    size_t cap = need + need / 8 + 1024;
    if ((rc = dev_alloc(c, &c->d_csr_col, cap))) return rc;
    if ((rc = dev_alloc(c, &c->d_csr_gain, cap))) return rc;
    if ((rc = dev_alloc(c, &c->d_csr_fd, cap))) return rc;
    c->csr_cap = cap;
  }
  if (need > c->csc_cap) {
    size_t cap = need + need / 8 + 1024;
    if ((rc = dev_alloc(c, &c->d_csc_row, cap))) return rc;
    if ((rc = dev_alloc(c, &c->d_csc_gain, cap))) return rc;
    c->csc_cap = cap;
  }
  return GHICP_OK;
}

// workspaces that depend on (N, M)
static int alloc_workspaces(Ctx *c) {
  const int N = c->N, M = c->M;
  // contiguous blocks of source rows per rank (SURVEY.md §8e); Npad = arrays that get all-gathered
  c->shard = (N + c->world - 1) / c->world;
  c->Npad = c->shard * c->world;
  c->r0 = std::min(N, c->rank * c->shard);
  c->nloc = std::max(0, std::min(N, c->r0 + c->shard) - c->r0);
  const int nmax = std::max(c->Npad, M);
  const int row_ctas = (N + 7) / 8;
  int want = (GHICP_SMS * 4 + row_ctas - 1) / row_ctas;
  int lim = std::max(1, M / 2048);
  c->n_chunks = std::max(1, std::min(want, lim));
  if (c->cfg.corr_type == GHICP_CT_KM || c->world > 1) c->n_chunks = 1;  // one CSR / result segment per row
  int rc;
  const size_t L = (size_t)c->Npad * c->n_chunks;
  if ((rc = dev_alloc(c, &c->d_part_cd, L))) return rc;
  if ((rc = dev_alloc(c, &c->d_part_idx, L))) return rc;
  c->part_stats_cap = std::max((size_t)row_ctas * c->n_chunks * 2, (size_t)stream_num_parts(c) * 2);
  if ((rc = dev_alloc(c, &c->d_part_stats, c->part_stats_cap))) return rc;
  // streaming path
  if ((rc = dev_alloc(c, &c->d_S4, 4 * (size_t)c->Npad))) return rc;
  if ((rc = dev_alloc(c, &c->d_T4, 4 * (size_t)M))) return rc;
  if ((rc = dev_alloc(c, &c->d_sdev, 1))) return rc;
  if ((rc = host_alloc_once(c, &c->h_sdev, sizeof(StreamDev)))) return rc;
  if ((rc = dev_alloc(c, &c->d_row_thr, (size_t)c->Npad))) return rc;
  if ((rc = dev_alloc(c, &c->d_col_thr, (size_t)M))) return rc;
  if ((rc = dev_alloc(c, &c->d_rowbest, (size_t)c->Npad))) return rc;
  if ((rc = dev_alloc(c, &c->d_colbest, (size_t)M))) return rc;
  if ((rc = dev_alloc(c, &c->d_rowidx2, (size_t)c->Npad))) return rc;
  if ((rc = dev_alloc(c, &c->d_colidx2, (size_t)M))) return rc;
  if (c->cfg.corr_type != GHICP_CT_KM || c->cfg.feature_type == GHICP_FT_FPFH) {   // (FPFH + KM: the filter's KM gate lists its hits there)
    c->cand_cap = (int)std::min<size_t>((size_t)96 * nmax + (1u << 20), (size_t)1 << 28);
    if ((rc = dev_alloc(c, &c->d_cand[0], (size_t)c->cand_cap))) return rc;
    if (c->cfg.corr_type == GHICP_CT_NNR) { if ((rc = dev_alloc(c, &c->d_cand[1], (size_t)c->cand_cap))) return rc; }
    // GHICP_CAND_CAP_MAX lowers the capacity the kernels see (test hook: forces the overflow -> all-double redo at any size)
    if (const char *ov = getenv("GHICP_CAND_CAP_MAX")) {
      const long long v = atoll(ov);
      if (v >= 1) c->cand_cap = (int)std::min<long long>(c->cand_cap, v);
    }
  }
  c->tile_cap = 2 * ((std::max(L, (size_t)nmax) + 1023) / 1024 + 1);
  if ((rc = dev_alloc(c, &c->d_tile_sum, c->tile_cap))) return rc;
  if ((rc = dev_alloc(c, &c->d_solve_part, (size_t)3 * 64 * 12))) return rc;
  CK(c, cudaMemset(c->d_sdev, 0, sizeof(StreamDev)));
  if ((rc = comm_warmup(c))) return rc;
  if ((rc = dev_alloc(c, &c->d_row_cd, (size_t)c->Npad))) return rc;
  if ((rc = dev_alloc(c, &c->d_row_idx, (size_t)c->Npad))) return rc;
  if ((rc = dev_alloc(c, &c->d_row_fd, (size_t)c->Npad))) return rc;
  if ((rc = dev_alloc(c, &c->d_pair_fd, (size_t)nmax))) return rc;
  if ((rc = dev_alloc(c, &c->d_xstats, (size_t)4 * c->world))) return rc;
  CK(c, cudaMemset(c->d_xstats, 0, sizeof(double) * 4 * c->world));
  CK(c, cudaMemset(c->d_row_idx, 0, sizeof(int) * (size_t)c->Npad));
  if (c->world > 1 && c->cfg.corr_type == GHICP_CT_NNR) {
    if ((rc = dev_alloc(c, &c->d_colg_cd, (size_t)c->world * M))) return rc;
    if ((rc = dev_alloc(c, &c->d_colg_idx, (size_t)c->world * M))) return rc;
  }
  if ((rc = host_alloc_once(c, &c->h_rowptr_cut, sizeof(long long) * (c->world + 1)))) return rc;
  if ((rc = dev_alloc(c, &c->d_col_cd, (size_t)M))) return rc;
  if ((rc = dev_alloc(c, &c->d_col_idx, (size_t)M))) return rc;
  if ((rc = dev_alloc(c, &c->d_flags, (size_t)nmax))) return rc;
  if ((rc = dev_alloc(c, &c->d_sp, (size_t)nmax))) return rc;
  if ((rc = dev_alloc(c, &c->d_tp, (size_t)nmax))) return rc;
  if ((rc = dev_alloc(c, &c->d_iter, 1))) return rc;
  if ((rc = host_alloc_once(c, &c->h_iter, sizeof(DevIter)))) return rc;
  if ((rc = host_alloc_once(c, &c->h_counters, sizeof(int) * 64))) return rc;
  if (c->cfg.corr_type == GHICP_CT_KM) {
    if ((rc = dev_alloc(c, &c->d_cnt, L + 2))) return rc;
    if ((rc = dev_alloc(c, &c->d_rowptr, L + 1))) return rc;
    if ((rc = dev_alloc(c, &c->d_cursor, L + 1))) return rc;
    if ((rc = dev_alloc(c, &c->d_colptr, (size_t)M + 1))) return rc;
    if ((rc = dev_alloc(c, &c->d_colcnt, (size_t)M + 1))) return rc;
    if ((rc = dev_alloc(c, &c->d_price, (size_t)M))) return rc;
    if ((rc = dev_alloc(c, &c->d_profit, (size_t)c->Npad))) return rc;
    if ((rc = dev_alloc(c, &c->d_assign, (size_t)c->Npad))) return rc;
    if ((rc = dev_alloc(c, &c->d_owner, (size_t)M))) return rc;
    if ((rc = dev_alloc(c, &c->d_bidmax, (size_t)nmax))) return rc;
    if ((rc = dev_alloc(c, &c->d_bidwin, (size_t)nmax))) return rc;
    if ((rc = dev_alloc(c, &c->d_bid_obj, (size_t)nmax))) return rc;
    if ((rc = dev_alloc(c, &c->d_bid_val, (size_t)nmax))) return rc;
    if ((rc = dev_alloc(c, &c->d_bid_aux, (size_t)nmax))) return rc;
    if ((rc = dev_alloc(c, &c->d_list[0], (size_t)nmax))) return rc;
    if ((rc = dev_alloc(c, &c->d_list[1], (size_t)nmax))) return rc;
    if ((rc = dev_alloc(c, &c->d_counters, 64))) return rc;
    // edge list of the KM count pass: generous for a settled loop (a few edges per keypoint); denser graphs
    // take the two-pass count + fill route (their time is the auction's anyway)
    const size_t plane = (size_t)std::max(c->nloc, 1) * (size_t)M;
    c->emit_cap = std::min(plane, std::max((size_t)1 << 21, (size_t)32 * (size_t)(c->nloc + M)));
    // settled iterations (ghicp_stream.cu: k_emit_check ...): one candidate block per rank.  Its capacity is the same on
    // every rank (the choice between the settled and the general route must be: both contain collectives) and the
    // edge list never holds less; the CSR / CSC arrays can take every block full, so nothing is allocated mid-loop.
    c->xcap = (std::max((size_t)8192, (size_t)4 * (size_t)c->shard) + 3) & ~(size_t)3;
    c->emit_cap = std::max(c->emit_cap, c->xcap);
    if ((rc = dev_alloc(c, &c->d_emit, c->emit_cap))) return rc;
    if ((rc = dev_alloc(c, &c->d_xsend, xblock_bytes(c->xcap)))) return rc;
    if (c->world > 1) { if ((rc = dev_alloc(c, &c->d_xrecv, xblock_bytes(c->xcap) * (size_t)c->world))) return rc; }
    if ((rc = dev_alloc(c, &c->d_xcounts, (size_t)c->world))) return rc;
    if ((rc = host_alloc_once(c, &c->h_xcounts, sizeof(unsigned long long) * (size_t)c->world))) return rc;
    if ((rc = ensure_edges(c, (long long)(c->xcap * (size_t)c->world)))) return rc;
  }
  return GHICP_OK;
}

// New keypoint counts: workspaces of the new size; descriptors, FD plane, normals, loop state and route history start over
static int resize_keypoints(Ctx *c, int N, int M) {
  if (N == c->N && M == c->M) return GHICP_OK;
  c->N = N; c->M = M;
  int rc;
  if ((rc = dev_alloc(c, &c->d_s, 3 * (size_t)N)) || (rc = dev_alloc(c, &c->d_t, 3 * (size_t)M)) || (rc = alloc_workspaces(c))) {
    c->N = c->M = 0;   // half-sized workspaces must not pass for a configured context: every later call answers "keypoints not set"
    return rc;
  }
  c->have_bsc = c->have_fpfh = c->fd_built = c->have_normals = false;
  reset_loop_state(c);
  return GHICP_OK;
}

static int build_fd(Ctx *c) {
  if (c->fd_built) return GHICP_OK;
  if (c->cfg.feature_type == GHICP_FT_BSC) {
    if (!c->have_bsc) { set_error(c, "build_fd: BSC descriptors not set"); return GHICP_E_ARG; }
    const int Vneed = (c->cfg.dof == 6) ? 4 : 2;
    if (c->V < Vneed) { set_error(c, "build_fd: not enough BSC source variants for dof"); return GHICP_E_ARG; }
    if (c->bits > 2048) { set_error(c, "build_fd: BSC descriptors longer than 2048 bits are not supported (12-bit FD plane)"); return GHICP_E_ARG; }
    c->fd_rows = (size_t)std::max(c->nloc, 1);
    const size_t plane_bytes = fd_plane_bytes(c->fd_rows, c->M, fd_hb(c->bits));
    int rc = dev_alloc(c, &c->d_fd16, (plane_bytes + 1) / 2);
    if (rc) return rc;
    CK(c, cudaMemsetAsync(c->d_fd16, 0, plane_bytes, c->stream));  // zero the quad / panel padding
    // tensor-core build (wgmma s8) when the descriptor fits its shared-memory tiling, else POPC
    cudaError_t e = (getenv("GHICP_FD_POPC") != nullptr) ? cudaErrorNotSupported : launch_fd_bsc_tc(c);
    if (e == cudaErrorNotSupported) { cudaGetLastError(); CK(c, launch_fd_bsc(c)); }
    else CK(c, e);
  } else if (c->cfg.feature_type == GHICP_FT_FPFH) {
    if (!c->have_fpfh) { set_error(c, "build_fd: FPFH descriptors not set"); return GHICP_E_ARG; }
    c->fd_rows = (size_t)std::max(c->nloc, 1);
    // Stored float plane (4*N*M bytes, fpfh_matrix_free = -1) or matrix-free (ghicp_fpfh.cu: FD recomputed inside the sweeps,
    // O(N+M) memory).  Both give bit-identical FD / CD values.  Auto (0) is matrix-free for every correspondence mode: NN / NNR
    // sweeps then run the FP32-filter fast path, several times faster than the all-double kernels with the same
    // correspondences; KM runs the exact sweeps in iterations 0-1 and the filter's gate after.
    const size_t plane_bytes = fd_elems(c->fd_rows, c->M) * sizeof(float);
    const bool mf = c->cfg.fpfh_matrix_free >= 0 || getenv("GHICP_FPFH_MATRIX_FREE") != nullptr;
    c->fpfh_mf = mf;
    int rc;
    if (mf) {
      dev_free(&c->d_fdf);
      if ((rc = dev_alloc(c, &c->d_fsc, (size_t)c->N * 36))) return rc;
      if ((rc = dev_alloc(c, &c->d_fscT, (size_t)c->N * 36))) return rc;
      if ((rc = dev_alloc(c, &c->d_ftc, (size_t)c->M * 36))) return rc;
      if ((rc = dev_alloc(c, &c->d_ftcT, (size_t)c->M * 36))) return rc;
      CK(c, launch_fpfh_prepare(c));
      // operands of the FP32 filter (NN / NNR filter route, the KM gate of the settled route)
      c->fpfh_fast_ready = false;
      if ((rc = dev_alloc(c, &c->d_ff_srec, (size_t)c->N * fpfh_fast_rec_floats()))) return rc;
      if ((rc = dev_alloc(c, &c->d_ff_tnT, (size_t)c->M * 36))) return rc;
      if ((rc = dev_alloc(c, &c->d_ff_tco, (size_t)c->M * 6))) return rc;
      if ((rc = dev_alloc(c, &c->d_ff_part, fpfh_fast_parts(c)))) return rc;
      if ((rc = dev_alloc(c, &c->d_ff_rowguess, (size_t)c->Npad))) return rc;
      if ((rc = dev_alloc(c, &c->d_ff_colguess, (size_t)c->M))) return rc;
      CK(c, cudaMemsetAsync(c->d_ff_rowguess, 0xff, sizeof(unsigned long long) * (size_t)c->Npad, c->stream));
      CK(c, cudaMemsetAsync(c->d_ff_colguess, 0xff, sizeof(unsigned long long) * (size_t)c->M, c->stream));
      CK(c, launch_fpfh_fast_build(c));
      c->fpfh_fast_ready = true;
    } else {
      if ((rc = dev_alloc(c, &c->d_fdf, fd_elems(c->fd_rows, c->M)))) return rc;
      CK(c, cudaMemsetAsync(c->d_fdf, 0, plane_bytes, c->stream));
      CK(c, launch_fd_fpfh(c));
    }
  }
  c->fd_built = true;
  return GHICP_OK;
}

static CostParams make_cost_params(const Ctx *c) {
  CostParams cp;
  cp.scale = (double)c->scale_f;
  cp.WFD = std::exp(-1.0 * c->iteration / c->weight_changing_rate);  // src/ghicp_reg.cpp:247
  cp.WED = 1.0 - cp.WFD;
  cp.ex = 1.0 / (c->iteration + 1);                                   // src/ghicp_reg.cpp:308
  cp.pivot = c->last_mean;
  return cp;
}
static LoopScalars make_loop_scalars(const Ctx *c, const CostParams &cp) {
  LoopScalars ls;
  ls.iteration = c->iteration;
  ls.RMS = c->RMS; ls.FDM = c->FDM; ls.FDstd = c->FDstd;
  ls.para1 = c->para1; ls.para2 = c->para2;
  ls.scale = cp.scale; ls.WED = cp.WED; ls.WFD = cp.WFD;
  ls.penalty_initial = c->penalty_initial;
  return ls;
}

// Candidate edges a rank's block carries this iteration: twice the largest per-rank share of the last one (same on every
// rank; the latency-bound all-gather carries what the graph needs, not what the buffers could hold).  GHICP_KM_XUSE_MAX caps
// it (test hook: forces the overflow -> general-route fallback).
static size_t settled_block_size(const Ctx *c) {
  size_t x = std::min(c->xcap, ((size_t)std::max<long long>(1024, 2 * c->last_max_local_nnz + 256) + 3) & ~(size_t)3);
  if (const char *ov = getenv("GHICP_KM_XUSE_MAX")) {
    const long long v = atoll(ov);
    if (v >= 4) x = std::min(x, (size_t)v & ~(size_t)3);
  }
  return x;
}

// How one iteration computes its costs and correspondences (DESIGN.md §7).  Every route ends in the same solve and host tail.
enum class Route {
  FpfhFilter,       // FPFH, matrix-free: FP32 filter over on-the-fly FD + exact refinement (NN / NNR)
  Stream,           // BSC or no feature: streaming filter pass + exact refinement (NN / NNR)
  FpfhKmSettled,    // FPFH + KM, settled loop: the FP32 filter as the KM gate
  StreamKmSettled,  // BSC + KM, settled loop: one streaming pass, one all-gather, no host round trip
  StreamKmGeneral,  // BSC / no feature + KM: [statistics pass] + count pass [+ fill pass], CSR cuts read by the host
  Exact,            // all-double kernels
};

static Route choose_route(const Ctx *c) {
  const int ft = c->cfg.feature_type, ct = c->cfg.corr_type;
  const bool stream = c->use_fast && (ft == GHICP_FT_NONE || ft == GHICP_FT_BSC);
  const bool fpfh_filter = c->use_fast && ft == GHICP_FT_FPFH && c->fpfh_mf && c->fpfh_fast_ready &&
                           getenv("GHICP_FPFH_EXACT") == nullptr;
  if (ct != GHICP_CT_KM) {
    // FPFH: the filter is taken when no decision depends on the CD mean, which a filter cannot reproduce in FPFH mode
    // (heavy-tailed ED / FD^ex): NNR has no gate, NN's penalty is RMS*para1*scale*para2 from iteration 2 on
    // (src/ghicp_reg.cpp:327-330).
    if (fpfh_filter && (ct == GHICP_CT_NNR || c->iteration >= 2)) return Route::FpfhFilter;
    return stream ? Route::Stream : Route::Exact;
  }
  // Settled KM iteration?  Decided from quantities every rank holds identically (both routes contain collectives).
  const RouteHistory &h = *c;
  const long long nmax = std::max(c->N, c->M);
  const bool sparse_history = c->iteration >= 2 && !h.km_settled_off && c->xcap > 0 && h.last_total_nnz >= 0 &&
                              (double)h.last_total_nnz <= 1.5 * (double)nmax && h.last_max_local_nnz >= 0 &&
                              (size_t)h.last_max_local_nnz + (size_t)h.last_max_local_nnz / 2 + 64 <= c->xcap &&
                              getenv("GHICP_KM_GENERAL") == nullptr && getenv("GHICP_KM_FILL") == nullptr;   // test hooks: general route
  // FPFH + KM, settled loop: the FP32 filter as the KM gate (penalty = RMS*para1*scale*para2 from iteration 2 on)
  if (fpfh_filter && c->d_cand[0] && sparse_history) return Route::FpfhKmSettled;
  if (!stream) return Route::Exact;
  return (ft != GHICP_FT_NONE && sparse_history) ? Route::StreamKmSettled : Route::StreamKmGeneral;
}

// What a route hands to the solve and the host tail.
struct RouteResult {
  long long nnz = 0;          // KM candidate edges (-1: the device's count, read after the final synchronize)
  KmResult kres;
  int stream_passes = 0;      // > 0: ev[4] / ev[5] were recorded around the route's main streaming pass
  long long candidates = 0;   // NN / NNR filter routes: candidates the filter passed to exact evaluation
  bool exact_redo = false;    // a filter route asks for the all-double redo of its cost stage (which then skips ev[1])
  bool out_of_range = false;  // ... because its operands left the FP32 filter's window (StreamDev::out_of_range)
};

// Seed pre-pass (FP32 minima only) before an NN / NNR filter pass?  It keeps the refinement cheap whenever last iteration's
// partners are not a tight bound: the first iterations (the metric mix changes fastest) or after many candidates.
static bool want_prepass(const Ctx *c, bool cols) {
  const long long cand_budget = 6ll * ((long long)c->nloc + (cols ? c->M : 0));
  return !c->have_prev || c->iteration <= 2 || c->last_cands > cand_budget;
}

// Tail of the NN / NNR filter routes: exchange, penalty, selection, read-back.  A candidate buffer overflow (on any rank), or
// an NN gate decision inside the error band of the fast statistics (amb_rel > 0), asks for the all-double redo (rare).
static int nn_tail(Ctx *c, const LoopScalars &ls, bool cols, double amb_rel, RouteResult *r) {
  int rc;
  if ((rc = comm_exchange(c, EX_STATS | EX_ROWS | (cols ? EX_COLS : 0)))) return rc;
  CK(c, launch_penalty(c, 0.0, ls));
  if (cols && c->world > 1) CK(c, launch_colmerge(c));
  CK(c, cudaEventRecord(c->ev[1], c->stream));
  CK(c, cols ? launch_select_nnr(c) : launch_select_nn(c, amb_rel));
  CK(c, cudaMemcpyAsync(c->h_sdev, c->d_sdev, sizeof(StreamDev), cudaMemcpyDeviceToHost, c->stream));
  CK(c, cudaMemcpyAsync(c->h_iter, c->d_iter, sizeof(DevIter), cudaMemcpyDeviceToHost, c->stream));
  CK(c, cudaStreamSynchronize(c->stream));
  r->candidates = c->last_cands = (long long)c->h_sdev->cand_count[0] + (cols ? c->h_sdev->cand_count[1] : 0);
  r->out_of_range = c->h_sdev->out_of_range != 0;
  r->exact_redo = c->h_iter->overflow_any || (!cols && c->h_iter->ambiguous > 0);
  if (!r->exact_redo) c->have_prev = true;
  return GHICP_OK;
}

static int route_fpfh_filter(Ctx *c, const CostParams &cp, const LoopScalars &ls, RouteResult *r) {
  const bool cols = c->cfg.corr_type == GHICP_CT_NNR;
  const bool prepass = want_prepass(c, cols);
  CK(c, launch_fpfh_fast_prep(c));
  if (prepass) { CK(c, launch_fpfh_fast_sweep(c, cp, true, cols)); ++r->stream_passes; }
  CK(c, launch_fpfh_fast_seed(c, cp, cols, prepass));
  CK(c, cudaEventRecord(c->ev[4], c->stream));
  CK(c, launch_fpfh_fast_sweep(c, cp, false, cols));
  CK(c, cudaEventRecord(c->ev[5], c->stream));
  ++r->stream_passes;
  CK(c, launch_fpfh_fast_finish(c, cp, cols));
  CK(c, launch_rowfd_mf(c));
  return nn_tail(c, ls, cols, 0.0, r);
}

// one pass = calED + calCD + row (and column) scans + statistics
static int route_stream(Ctx *c, const CostParams &cp, const LoopScalars &ls, RouteResult *r) {
  const bool cols = c->cfg.corr_type == GHICP_CT_NNR;
  const bool prepass = want_prepass(c, cols);
  CK(c, launch_stream_prep(c, cp, 0));
  CK(c, launch_stream_seed(c, cp, cols));
  if (prepass) { CK(c, launch_stream(c, cp, cols ? SM_PRE_COLS : SM_PRE, true)); ++r->stream_passes; }
  CK(c, cudaEventRecord(c->ev[4], c->stream));
  CK(c, launch_stream(c, cp, cols ? SM_NNR : SM_NN, !prepass));
  CK(c, cudaEventRecord(c->ev[5], c->stream));
  ++r->stream_passes;
  CK(c, launch_finalize_fast(c));
  CK(c, launch_stream_resolve(c, cp, cols));
  // the NN gate depends on this iteration's statistics only for Ft=None and for BSC iterations 0-1
  const bool stats_dependent = c->cfg.feature_type == GHICP_FT_NONE || c->iteration <= 1;
  return nn_tail(c, ls, cols, stats_dependent ? 1e-5 : 0.0, r);
}

// Tail of the two settled KM routes: ONE all-gather of the per-rank candidate blocks (none on one GPU), then CSR / CSC,
// statistics, single-phase auction and selection; the host reads nothing until the iteration's final synchronize.
static int km_settled_tail(Ctx *c, const LoopScalars &ls, RouteResult *r) {
  int rc;
  if ((rc = comm_allgather_bytes(c, c->d_xsend, c->d_xrecv, xblock_bytes(c->xuse)))) return rc;   // the iteration's one exchange
  CK(c, launch_xbuild(c));
  CK(c, launch_penalty(c, 0.0, ls));        // CD mean / std of all ranks' sums (+ the overflow flag); same penalty
  CK(c, cudaEventRecord(c->ev[1], c->stream));
  r->stream_passes = 1;
  if ((rc = km_auction_settled(c, c->N, c->M, c->last_total_nnz, c->KM_eps))) return rc;
  CK(c, launch_select_km(c));
  CK(c, launch_pair_fd_km(c));
  CK(c, cudaMemcpyAsync(c->h_sdev, c->d_sdev, sizeof(StreamDev), cudaMemcpyDeviceToHost, c->stream));
  CK(c, cudaMemcpyAsync(c->h_xcounts, c->d_xcounts, sizeof(unsigned long long) * (size_t)c->world, cudaMemcpyDeviceToHost, c->stream));
  r->nnz = -1;  // filled from h_sdev after the final synchronize
  return GHICP_OK;
}

// FPFH + KM, settled loop: one filter sweep with every row's threshold at the penalty; the exactly evaluated hits with
// CD < penalty are the KM graph and travel as this rank's candidate block
static int route_fpfh_km_settled(Ctx *c, const CostParams &cp, const LoopScalars &ls, RouteResult *r) {
  c->xuse = settled_block_size(c);
  CK(c, launch_fpfh_fast_prep(c));
  CK(c, launch_fpfh_gate_seed(c, cp, ls));
  CK(c, cudaEventRecord(c->ev[4], c->stream));
  CK(c, launch_fpfh_fast_sweep(c, cp, false, false));
  CK(c, cudaEventRecord(c->ev[5], c->stream));
  CK(c, launch_fpfh_cand_block(c, cp));
  return km_settled_tail(c, ls, r);
}

// BSC + KM, settled loop (sparse candidate graph, penalty independent of this iteration's CD): one pass over the FD plane,
// the gate hits checked exactly where they were found.  A block overflow (the flag travels with the statistics, k_apply then
// leaves the keypoints alone) sends the iteration through the general route.
static int route_stream_km_settled(Ctx *c, const CostParams &cp, const LoopScalars &ls, RouteResult *r) {
  c->emit_on = true;
  c->xuse = settled_block_size(c);
  CK(c, launch_stream_prep(c, cp, 0));
  CK(c, cudaMemsetAsync(c->d_cnt, 0, sizeof(int) * ((size_t)c->Npad + 2), c->stream));
  CK(c, launch_penalty_only(c, ls));        // src/ghicp_reg.cpp:279-282: independent of this iteration's CD
  CK(c, launch_stream_gate(c, cp));
  CK(c, cudaEventRecord(c->ev[4], c->stream));
  CK(c, launch_stream(c, cp, SM_COUNT, true));
  CK(c, cudaEventRecord(c->ev[5], c->stream));
  CK(c, launch_finalize_fast(c));
  CK(c, launch_emit_check(c, cp));
  return km_settled_tail(c, ls, r);
}

// The KM graph's size and per-rank shares (share(k) = candidate edges of rank k), noted for the next route choice
template <class Share>
static void note_km_graph(Ctx *c, long long total, Share share) {
  RouteHistory &h = *c;
  h.last_total_nnz = total;
  h.last_local_nnz = share(c->rank);
  h.last_max_local_nnz = 0;
  for (int k = 0; k < c->world; ++k) h.last_max_local_nnz = std::max(h.last_max_local_nnz, share(k));
}

// End of the general KM routes: read back the edge count and penalty (sharded: and the CSR offsets at the shard boundaries),
// make room for the edges, fill(nnz) enqueues this rank's edges, note the graph's shares, auction, selection, pairs' FD.
template <class Fill>
static int km_general_tail(Ctx *c, RouteResult *r, Fill fill) {
  CK(c, cudaMemcpyAsync(c->h_iter, c->d_iter, sizeof(DevIter), cudaMemcpyDeviceToHost, c->stream));
  if (c->world > 1)
    for (int k = 0; k <= c->world; ++k)
      CK(c, cudaMemcpyAsync(c->h_rowptr_cut + k, c->d_rowptr + std::min(c->N, k * c->shard), sizeof(long long),
                            cudaMemcpyDeviceToHost, c->stream));
  CK(c, cudaStreamSynchronize(c->stream));
  if (c->h_iter->overflow_any) {
    // only the streaming route sets it here (k_finalize_fast): its gate ran outside the FP32 filter's window, and nothing
    // has been applied yet, so the all-double route takes the iteration over
    r->exact_redo = r->out_of_range = true;
    return GHICP_OK;
  }
  const long long nnz = c->h_iter->nnz;
  const double penalty = c->h_iter->penalty;
  int rc;
  if ((rc = ensure_edges(c, nnz)) || (rc = fill(nnz))) return rc;
  note_km_graph(c, nnz, [&](int k) { return c->world > 1 ? c->h_rowptr_cut[k + 1] - c->h_rowptr_cut[k] : nnz; });
  c->km_settled_off = false;
  if ((rc = km_auction(c, c->N, c->M, nnz, c->KM_eps, std::max(penalty, c->KM_eps), &r->kres))) return rc;
  CK(c, launch_select_km(c));
  CK(c, launch_pair_fd_km(c));
  r->nnz = nnz;
  return GHICP_OK;
}

// BSC / no feature + KM, general: [statistics pass] + count pass + [fill pass] over the FD plane
static int route_stream_km_general(Ctx *c, const CostParams &cp, const LoopScalars &ls, RouteResult *r) {
  int rc;
  // the penalty needs this iteration's CD statistics for Ft=None and in iterations 0-1: a statistics pass with the gate off
  // (thr = -1) comes first, then the count pass; otherwise the penalty is known and the first pass counts
  const bool stats_first = c->cfg.feature_type == GHICP_FT_NONE || c->iteration <= 1;
  // the edge list pays off on sparse candidate graphs; on a dense one (first iterations) its single append
  // counter would serialise millions of hits, so it is switched on from last iteration's count
  c->emit_on = c->last_local_nnz >= 0 && (size_t)c->last_local_nnz + (size_t)c->last_local_nnz / 2 <= c->emit_cap;
  CK(c, launch_stream_prep(c, cp, 0));
  CK(c, cudaMemsetAsync(c->d_cnt, 0, sizeof(int) * ((size_t)c->Npad + 2), c->stream));
  if (!stats_first) {
    CK(c, launch_penalty_only(c, ls));      // src/ghicp_reg.cpp:279-282: independent of this iteration's CD
    CK(c, launch_stream_gate(c, cp));
  }
  CK(c, cudaEventRecord(c->ev[4], c->stream));
  CK(c, launch_stream(c, cp, SM_COUNT, true));
  CK(c, cudaEventRecord(c->ev[5], c->stream));
  CK(c, launch_finalize_fast(c));
  if ((rc = comm_exchange(c, EX_STATS))) return rc;
  CK(c, launch_penalty(c, 0.0, ls));
  if (stats_first) CK(c, launch_stream_gate(c, cp));
  CK(c, cudaEventRecord(c->ev[1], c->stream));
  if (stats_first) CK(c, launch_stream(c, cp, SM_COUNT, false));
  r->stream_passes = stats_first ? 2 : 1;
  if ((rc = comm_gather_counts(c))) return rc;
  CK(c, launch_scan_rows(c));
  CK(c, cudaMemcpyAsync(c->h_sdev, c->d_sdev, sizeof(StreamDev), cudaMemcpyDeviceToHost, c->stream));
  rc = km_general_tail(c, r, [&](long long nnz) -> int {
    if (nnz <= 0) return GHICP_OK;
    // this rank's gate hits were appended to the edge list by the count pass (when the list was on and did
    // not overflow): scatter them; otherwise stream the plane a second time (fill pass)
    const unsigned long long emitted = c->h_sdev->emit_count;
    const bool force_fill = getenv("GHICP_KM_FILL") != nullptr;  // test hook: always take the fill pass
    if (c->emit_on && emitted <= (unsigned long long)c->emit_cap && !force_fill) {
      if (emitted > 0) CK(c, launch_emit_scatter(c, cp, emitted));
    } else {
      ++r->stream_passes;
      CK(c, launch_stream(c, cp, SM_FILL, false));
    }
    CK(c, launch_csr_check(c, cp));
    if (c->world > 1) {
      if ((rc = comm_gather_edges(c, c->h_rowptr_cut))) return rc;
      CK(c, launch_count_valid(c, nnz));
    }
    return GHICP_OK;
  });
  if (rc) return rc;
  CK(c, cudaMemcpyAsync(c->h_sdev, c->d_sdev, sizeof(StreamDev), cudaMemcpyDeviceToHost, c->stream));
  r->nnz = -1;  // filled from h_sdev after the final synchronize
  return GHICP_OK;
}

// Row stage of the all-double kernels: row minima and CD statistics (+ the partners' FD for matrix-free FPFH)
static int exact_row_stage(Ctx *c, const CostParams &cp, const LoopScalars &ls) {
  const bool mf = (c->cfg.feature_type == GHICP_FT_FPFH) && c->fpfh_mf;   // matrix-free FPFH: FD recomputed inside the sweeps
  CK(c, mf ? launch_rowsweep_mf(c, SWEEP_ROWMIN, cp) : launch_rowsweep(c, SWEEP_ROWMIN, cp));
  CK(c, launch_finalize_stats(c, cp, ls));
  if (mf) CK(c, launch_rowfd_mf(c));
  return GHICP_OK;
}

// All-double route (FPFH; forced; or the redo after a filter route): calED + calCD_* (+ the row scan of NN / NNR)
static int route_exact(Ctx *c, const CostParams &cp, const LoopScalars &ls, RouteResult *r) {
  const int ct = c->cfg.corr_type;
  const bool mf = (c->cfg.feature_type == GHICP_FT_FPFH) && c->fpfh_mf;
  const bool sharded = c->world > 1;
  int rc;
  if ((rc = exact_row_stage(c, cp, ls))) return rc;
  if (ct == GHICP_CT_NNR) CK(c, mf ? launch_colsweep_mf(c, cp) : launch_colsweep(c, cp));
  if ((rc = comm_exchange(c, EX_STATS | EX_ROWS | (ct == GHICP_CT_NNR ? EX_COLS : 0)))) return rc;
  CK(c, launch_penalty(c, cp.pivot, ls));
  if (ct == GHICP_CT_NNR && sharded) CK(c, launch_colmerge(c));
  if (!r->exact_redo) CK(c, cudaEventRecord(c->ev[1], c->stream));
  if (ct != GHICP_CT_KM) {
    CK(c, ct == GHICP_CT_NN ? launch_select_nn(c) : launch_select_nnr(c));
    c->have_prev = true;
    return GHICP_OK;
  }
  // sharded: every rank counts, fills and checks the candidates of ITS rows with the all-double kernels; counts and
  // edges travel like on the streaming path's general route (all-gather of the counts, one broadcast group of the edges)
  if (sharded) CK(c, cudaMemsetAsync(c->d_cnt, 0, sizeof(int) * ((size_t)c->Npad + 2), c->stream));
  CK(c, mf ? launch_rowsweep_mf(c, SWEEP_COUNT, cp) : launch_rowsweep(c, SWEEP_COUNT, cp));
  if (sharded && (rc = comm_gather_counts(c))) return rc;
  CK(c, launch_scan_counts(c));
  return km_general_tail(c, r, [&](long long nnz) -> int {
    if (nnz <= 0) return GHICP_OK;
    CK(c, mf ? launch_rowsweep_mf(c, SWEEP_FILL, cp) : launch_rowsweep(c, SWEEP_FILL, cp));
    return sharded ? comm_gather_edges(c, c->h_rowptr_cut) : GHICP_OK;
  });
}

// Host tail of an iteration (scalars only): convergence, IoU, Euler angles, adjustweight, Rt_tillnow, statistics; warnings
static int host_tail(Ctx *c, const RouteResult &r, bool redone, ghicp_iter_stats *out) {
  const DevIter &h = *c->h_iter;
  const int cor_number = h.cor;
  c->last_cor = cor_number;
  c->RMS = h.rmse;   // src/ghicp_reg.cpp:578, 695, 766
  c->FDM = h.fdm;
  c->FDstd = h.fdstd;
  c->last_mean = h.cd_mean;
  int warnings = 0;
  if (cor_number < c->min_cor) { c->converge = true; warnings |= GHICP_W_FEW_PAIRS; }  // :796-797
  c->IoU = 1.0 * cor_number / (c->N + c->M - cor_number);                                // :799
  double R[3][3], t[3];
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) R[i][j] = h.Rt[j * 4 + i];
    t[i] = h.Rt[12 + i];
  }
  const double dx = t[0], dy = t[1], dz = t[2];
  double ax = std::atan2(R[2][1], R[2][2]);
  double ay = std::atan2(-R[2][0], std::sqrt(R[2][1] * R[2][1] + R[2][2] * R[2][2]));
  double az = std::atan2(R[0][1], R[0][0]);
  const double pi = 3.1415926;  // src/ghicp_reg.cpp:876
  ax = ax / pi * 180; ay = ay / pi * 180; az = az / pi * 180;
  const double conv_t = (double)c->cfg.converge_t, conv_r = (double)c->cfg.converge_r;
  if (std::abs(dx) < conv_t && std::abs(dy) < conv_t && std::abs(dz) < conv_t && std::abs(ax) < conv_r &&
      std::abs(ay) < conv_r && std::abs(az) < conv_r)
    c->converge = true;  // :909-914
  // adjustweight (:771-789)
  if (c->cfg.estimated_iou / c->IoU > c->cfg.adjust_ratio) {
    c->para1 += c->cfg.adjust_step;
    c->para2 += c->cfg.adjust_step;
  } else if (c->IoU / c->cfg.estimated_iou > c->cfg.adjust_ratio) {
    c->para1 -= c->cfg.adjust_step;
    c->para2 -= c->cfg.adjust_step;
  }
  // Rt_tillnow = Rt_temp * Rt_tillnow (:93)
  double acc[16];
  for (int col = 0; col < 4; ++col)
    for (int row = 0; row < 4; ++row) {
      double s = 0;
      for (int k = 0; k < 4; ++k) s += h.Rt[k * 4 + row] * c->Rt_tillnow[col * 4 + k];
      acc[col * 4 + row] = s;
    }
  std::memcpy(c->Rt_tillnow, acc, sizeof(acc));

  if (out) {
    std::memset(out, 0, sizeof(*out));
    out->iteration = c->iteration;
    out->cor = cor_number;
    out->converged = c->converge ? 1 : 0;
    out->warnings = warnings;
    std::memcpy(out->Rt, h.Rt, sizeof(double) * 16);
    std::memcpy(out->Rt_tillnow, c->Rt_tillnow, sizeof(double) * 16);
    out->cd_mean = h.cd_mean; out->cd_std = h.cd_std; out->penalty = h.penalty;
    out->rmse = h.rmse; out->rmse_after = h.rmse_after; out->fdm = h.fdm; out->fdstd = h.fdstd;
    out->iou = c->IoU; out->para1 = c->para1; out->para2 = c->para2;
    const int n = std::max(c->N, c->M);
    out->km_energy = (c->cfg.corr_type == GHICP_CT_KM) ? h.km_cd_sum + (double)(n - cor_number) * h.penalty : 0.0;
    out->ax = ax; out->ay = ay; out->az = az;
    out->nnz = r.nnz; out->km_rounds = r.kres.rounds; out->km_phases = r.kres.phases;
    out->gpu_launches = c->launches;
    out->exact_fallback = (r.exact_redo ? 1 : 0) | (redone ? 2 : 0) | (r.out_of_range ? 4 : 0);
    float ms;
    cudaEventElapsedTime(&ms, c->ev[0], c->ev[1]); out->ms_cost = ms;
    cudaEventElapsedTime(&ms, c->ev[1], c->ev[2]); out->ms_corr = ms;
    cudaEventElapsedTime(&ms, c->ev[2], c->ev[3]); out->ms_solve = ms;
    cudaEventElapsedTime(&ms, c->ev[0], c->ev[3]); out->ms_total = ms;
    if (r.stream_passes > 0) { cudaEventElapsedTime(&ms, c->ev[4], c->ev[5]); out->ms_stream = ms; }
    out->stream_passes = r.stream_passes;
    out->candidates = r.candidates;
  }
  c->iteration++;
  return warnings;
}

static int iterate_impl(Ctx *c, ghicp_iter_stats *out) {
  if (c->N <= 0 || c->M <= 0) { set_error(c, "iterate: keypoints not set"); return GHICP_E_ARG; }
  if (c->cfg.solver == GHICP_SOLVER_POINT_TO_PLANE && !c->have_normals) {
    set_error(c, "iterate: GHICP_SOLVER_POINT_TO_PLANE needs ghicp_set_target_normals");
    return GHICP_E_ARG;
  }
  int rc;
  if ((rc = build_fd(c))) return rc;
  const CostParams cp = make_cost_params(c);
  const LoopScalars ls = make_loop_scalars(c, cp);
  RouteResult r;
  bool redone = false;   // reported as bit 1 of ghicp_iter_stats.exact_fallback
  for (;;) {
    const Route route = choose_route(c);
    const bool settled = route == Route::FpfhKmSettled || route == Route::StreamKmSettled;
    r = RouteResult();
    c->launches = 0;
    CK(c, cudaEventRecord(c->ev[0], c->stream));
    switch (route) {
      case Route::FpfhFilter: rc = route_fpfh_filter(c, cp, ls, &r); break;
      case Route::Stream: rc = route_stream(c, cp, ls, &r); break;
      case Route::FpfhKmSettled: rc = route_fpfh_km_settled(c, cp, ls, &r); break;
      case Route::StreamKmSettled: rc = route_stream_km_settled(c, cp, ls, &r); break;
      case Route::StreamKmGeneral: rc = route_stream_km_general(c, cp, ls, &r); break;
      case Route::Exact: rc = route_exact(c, cp, ls, &r); break;
    }
    if (rc == GHICP_OK && r.exact_redo) rc = route_exact(c, cp, ls, &r);
    if (rc) return rc;
    CK(c, cudaEventRecord(c->ev[2], c->stream));
    // transformestimation (numeric core) + update of all source keypoints
    CK(c, launch_solve(c, cp));
    // opt-in estimators replace the transform (and the RMSE after it); the pair statistics stay k_solve's
    if (c->cfg.solver != GHICP_SOLVER_SVD) CK(c, launch_solve_alt(c, c->cfg.solver));
    CK(c, launch_apply(c, settled));
    CK(c, cudaEventRecord(c->ev[3], c->stream));
    CK(c, cudaMemcpyAsync(c->h_iter, c->d_iter, sizeof(DevIter), cudaMemcpyDeviceToHost, c->stream));
    CK(c, cudaStreamSynchronize(c->stream));
    if (!settled) break;
    if (!c->h_iter->overflow_any) {
      if ((rc = km_auction_settled_result(c, &r.kres))) return rc;
      note_km_graph(c, c->h_iter->nnz, [&](int k) { return (long long)c->h_xcounts[k]; });
      break;
    }
    // some rank's candidate block overflowed: nothing was updated; the iteration runs again on the general route
    c->km_settled_off = true;
    redone = true;
  }
  if (r.nnz < 0) r.nnz = (long long)c->h_sdev->nnz_valid;
  return host_tail(c, r, redone, out);
}

}  // namespace ghicp_b200

using namespace ghicp_b200;

extern "C" {

int ghicp_abi_version(void) { return GHICP_ABI_VERSION; }

int ghicp_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

const char *ghicp_last_error(const ghicp_ctx *ctx) {
  const Ctx *c = reinterpret_cast<const Ctx *>(ctx);
  if (c) return c->err.c_str();
  return g_last_error.c_str();
}

int ghicp_create(const ghicp_config *cfg, ghicp_ctx **out) {
  if (!cfg || !out) { set_error(nullptr, "ghicp_create: null argument"); return GHICP_E_ARG; }
  *out = nullptr;
  if (ghicp_device_count() <= 0) {
    set_error(nullptr, "ghicp_create: no CUDA device visible (this library has no CPU fallback)");
    return GHICP_E_NODEV;
  }
  if (cfg->device < 0 || cfg->device >= ghicp_device_count()) { set_error(nullptr, "ghicp_create: bad device"); return GHICP_E_ARG; }
  if (cfg->corr_type < GHICP_CT_NN || cfg->corr_type > GHICP_CT_KM) { set_error(nullptr, "ghicp_create: bad corr_type"); return GHICP_E_ARG; }
  if (cfg->feature_type != GHICP_FT_BSC && cfg->feature_type != GHICP_FT_FPFH && cfg->feature_type != GHICP_FT_NONE) {
    set_error(nullptr, "ghicp_create: feature_type must be BSC, FPFH or None (RoPS is 'Not passed yet' in the reference, test/ghicp_main.cpp:130-134)");
    return GHICP_E_ARG;
  }
  if (cfg->solver != GHICP_SOLVER_SVD && cfg->solver != GHICP_SOLVER_POINT_TO_PLANE && cfg->solver != GHICP_SOLVER_YAW_4DOF) {
    set_error(nullptr, "ghicp_create: solver must be SVD (reference), POINT_TO_PLANE or YAW_4DOF (WEIGHTED_SVD is stand-alone: ghicp_rigid_fit_ex)");
    return GHICP_E_ARG;
  }
  Ctx *c = new Ctx();
  c->cfg = *cfg;
  c->device = cfg->device;
  int rc = use_device(c);
  if (rc) { delete c; return rc; }
  if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess) {
    cudaGetLastError();
    set_error(nullptr, "ghicp_create: cudaStreamCreateWithFlags failed");
    delete c;
    return GHICP_E_CUDA;
  }
  for (auto &e : c->ev) cudaEventCreate(&e);
  reset_loop_state(c);
  c->use_fast = (cfg->force_exact == 0);
  *out = reinterpret_cast<ghicp_ctx *>(c);
  return GHICP_OK;
}

int ghicp_destroy(ghicp_ctx *ctx) {
  Ctx *c = reinterpret_cast<Ctx *>(ctx);
  if (!c) return GHICP_OK;
  use_device(c);
  cudaStreamSynchronize(c->stream);
  comm_destroy(c);
  free_all(c);
  for (auto &e : c->ev) if (e) cudaEventDestroy(e);
  if (c->stream) cudaStreamDestroy(c->stream);
  delete c;
  return GHICP_OK;
}

int ghicp_set_keypoints(ghicp_ctx *ctx, const double *sxyz, int N, const double *txyz, int M) {
  Ctx *c = reinterpret_cast<Ctx *>(ctx);
  if (!c || !sxyz || !txyz || N <= 0 || M <= 0) { set_error(c, "set_keypoints: bad argument"); return GHICP_E_ARG; }
  int rc;
  if ((rc = use_device(c))) return rc;
  if ((rc = resize_keypoints(c, N, M))) return rc;
  const size_t need = 3 * ((size_t)N + M) * sizeof(double);
  if (need > c->h_stage_cap) {
    if (c->h_stage) cudaFreeHost(c->h_stage);
    if (cudaMallocHost((void **)&c->h_stage, need) != cudaSuccess) {
      cudaGetLastError();
      c->h_stage = nullptr; c->h_stage_cap = 0;
      set_error(c, "set_keypoints: cudaMallocHost of the staging buffer failed");
      return GHICP_E_NOMEM;
    }
    c->h_stage_cap = need;
  }
  // pageable -> pinned staging, pipelined with the DMA: the target is staged while the source is in flight,
  // and the centroid is taken while the target is in flight.  Page-locked caller buffers are read by the DMA directly.
  double *hs = c->h_stage, *ht = c->h_stage + 3 * (size_t)N;
  const bool pin_s = is_pinned(sxyz), pin_t = is_pinned(txyz);
  if (pin_s) hs = const_cast<double *>(sxyz); else std::memcpy(hs, sxyz, 3 * (size_t)N * sizeof(double));
  CK(c, cudaMemcpyAsync(c->d_s, hs, 3 * (size_t)N * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  if (pin_t) ht = const_cast<double *>(txyz); else std::memcpy(ht, txyz, 3 * (size_t)M * sizeof(double));
  CK(c, cudaMemcpyAsync(c->d_t, ht, 3 * (size_t)M * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  {  // centre of the FP32 filter coordinates: target centroid
    double cx = 0, cy = 0, cz = 0;
    for (int j = 0; j < M; ++j) { cx += ht[j]; cy += ht[(size_t)M + j]; cz += ht[2 * (size_t)M + j]; }
    c->center[0] = cx / M; c->center[1] = cy / M; c->center[2] = cz / M;
  }
  CK(c, cudaStreamSynchronize(c->stream));
  return GHICP_OK;
}

int ghicp_set_bsc(ghicp_ctx *ctx, const uint8_t *s_bits, int V, const uint8_t *t_bits, int bits) {
  Ctx *c = reinterpret_cast<Ctx *>(ctx);
  if (!c || !s_bits || !t_bits || V <= 0 || V > 4 || bits <= 0 || bits > 65535 || c->N <= 0) {
    set_error(c, "set_bsc: bad argument or keypoints not set");
    return GHICP_E_ARG;
  }
  int rc;
  if ((rc = use_device(c))) return rc;
  c->V = V; c->bits = bits;
  c->Bbytes = (int)std::ceil((float)bits / 8.f);  // include/stereo_binary_feature.h:50
  c->W64 = (c->Bbytes + 7) / 8;
  if ((rc = dev_alloc(c, &c->d_bs, (size_t)V * c->W64 * c->N))) return rc;
  if ((rc = dev_alloc(c, &c->d_bt, (size_t)c->W64 * c->M))) return rc;
  uint8_t *raw_s = nullptr, *raw_t = nullptr;
  const size_t ns = (size_t)V * c->N * c->Bbytes, nt = (size_t)c->M * c->Bbytes;
  if ((rc = dev_alloc(c, &raw_s, ns))) return rc;
  if ((rc = dev_alloc(c, &raw_t, nt))) { dev_free(&raw_s); return rc; }
  cudaError_t e = cudaMemcpyAsync(raw_s, s_bits, ns, cudaMemcpyHostToDevice, c->stream);
  if (e == cudaSuccess) e = cudaMemcpyAsync(raw_t, t_bits, nt, cudaMemcpyHostToDevice, c->stream);
  if (e == cudaSuccess) e = launch_pack_bsc(c, raw_s, raw_t);
  if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
  dev_free(&raw_s); dev_free(&raw_t);
  if (e != cudaSuccess) { set_error(c, std::string("set_bsc: ") + cudaGetErrorString(e)); return GHICP_E_CUDA; }
  c->have_bsc = true;
  c->fd_built = false;
  return GHICP_OK;
}

// Keypoints::setFPFHfeature from host (ghicp_set_fpfh) or device (ghicp_set_from_prep) histograms [N][33], [M][33]
static int set_fpfh_from(Ctx *c, const float *s, const float *t, cudaMemcpyKind kind) {
  int rc;
  if ((rc = use_device(c))) return rc;
  if ((rc = dev_alloc(c, &c->d_fs, (size_t)c->N * 33))) return rc;
  if ((rc = dev_alloc(c, &c->d_ft, (size_t)c->M * 33))) return rc;
  CK(c, cudaMemcpyAsync(c->d_fs, s, (size_t)c->N * 33 * sizeof(float), kind, c->stream));
  CK(c, cudaMemcpyAsync(c->d_ft, t, (size_t)c->M * 33 * sizeof(float), kind, c->stream));
  CK(c, cudaStreamSynchronize(c->stream));
  c->have_fpfh = true;
  c->fd_built = false;
  return GHICP_OK;
}

int ghicp_set_fpfh(ghicp_ctx *ctx, const float *s, const float *t) {
  Ctx *c = reinterpret_cast<Ctx *>(ctx);
  if (!c || !s || !t || c->N <= 0) { set_error(c, "set_fpfh: bad argument or keypoints not set"); return GHICP_E_ARG; }
  return set_fpfh_from(c, s, t, cudaMemcpyHostToDevice);
}

int ghicp_set_target_normals(ghicp_ctx *ctx, const double *nxyz) {
  Ctx *c = reinterpret_cast<Ctx *>(ctx);
  if (!c || !nxyz || c->M <= 0) { set_error(c, "set_target_normals: bad argument or keypoints not set"); return GHICP_E_ARG; }
  int rc;
  if ((rc = use_device(c))) return rc;
  if ((rc = dev_alloc(c, &c->d_tn, 3 * (size_t)c->M))) return rc;
  CK(c, cudaMemcpyAsync(c->d_tn, nxyz, 3 * (size_t)c->M * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  CK(c, cudaStreamSynchronize(c->stream));
  c->have_normals = true;
  return GHICP_OK;
}

int ghicp_set_solver(ghicp_ctx *ctx, int solver) {
  Ctx *c = reinterpret_cast<Ctx *>(ctx);
  if (!c || (solver != GHICP_SOLVER_SVD && solver != GHICP_SOLVER_POINT_TO_PLANE && solver != GHICP_SOLVER_YAW_4DOF)) {
    set_error(c, "set_solver: solver must be SVD (reference), POINT_TO_PLANE or YAW_4DOF");
    return GHICP_E_ARG;
  }
  c->cfg.solver = solver;
  return GHICP_OK;
}

int ghicp_build_fd(ghicp_ctx *ctx) {
  Ctx *c = reinterpret_cast<Ctx *>(ctx);
  if (!c) return GHICP_E_ARG;
  int rc;
  if ((rc = use_device(c))) return rc;
  if ((rc = build_fd(c))) return rc;
  CK(c, cudaStreamSynchronize(c->stream));
  return GHICP_OK;
}

int ghicp_iterate(ghicp_ctx *ctx, ghicp_iter_stats *out) {
  Ctx *c = reinterpret_cast<Ctx *>(ctx);
  if (!c) return GHICP_E_ARG;
  int rc;
  if ((rc = use_device(c))) return rc;
  return iterate_impl(c, out);
}

int ghicp_run(ghicp_ctx *ctx, double Rt_final[16], int *iterations) {
  Ctx *c = reinterpret_cast<Ctx *>(ctx);
  if (!c || !Rt_final) return GHICP_E_ARG;
  int rc;
  if ((rc = use_device(c))) return rc;
  int it = 0;
  while (!c->converge) {  // src/ghicp_reg.cpp:49
    ghicp_iter_stats st;
    rc = iterate_impl(c, &st);
    if (rc < 0) return rc;
    ++it;
    if (c->cfg.max_iter > 0 && it >= c->cfg.max_iter) break;
  }
  std::memcpy(Rt_final, c->Rt_tillnow, sizeof(double) * 16);  // :104
  if (iterations) *iterations = it;
  return c->converge ? GHICP_OK : GHICP_E_NOCONV;
}

int ghicp_get_pairs(ghicp_ctx *ctx, int *sp, int *tp, int cap, int *n) {
  Ctx *c = reinterpret_cast<Ctx *>(ctx);
  if (!c || !n) return GHICP_E_ARG;
  int rc;
  if ((rc = use_device(c))) return rc;
  const int cor = c->last_cor;
  *n = cor;
  const int k = std::min(cor, cap);
  // both lists in flight at once, one synchronize (page-locked destinations are written by the DMA directly)
  if (k > 0 && sp) CK(c, cudaMemcpyAsync(sp, c->d_sp, sizeof(int) * (size_t)k, cudaMemcpyDeviceToHost, c->stream));
  if (k > 0 && tp) CK(c, cudaMemcpyAsync(tp, c->d_tp, sizeof(int) * (size_t)k, cudaMemcpyDeviceToHost, c->stream));
  CK(c, cudaStreamSynchronize(c->stream));
  return GHICP_OK;
}

int ghicp_get_source(ghicp_ctx *ctx, double *sxyz) {
  Ctx *c = reinterpret_cast<Ctx *>(ctx);
  if (!c || !sxyz || c->N <= 0) return GHICP_E_ARG;
  int rc;
  if ((rc = use_device(c))) return rc;
  CK(c, cudaMemcpyAsync(sxyz, c->d_s, 3 * (size_t)c->N * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
  CK(c, cudaStreamSynchronize(c->stream));
  return GHICP_OK;
}

// Page-locked host memory for the caller's coordinate / result buffers: set_keypoints, get_pairs and get_source then move
// the data with one DMA each, no staging copy.
int ghicp_host_alloc(size_t bytes, void **out) {
  if (!out || bytes == 0) return GHICP_E_ARG;
  if (ghicp_device_count() <= 0) { set_error(nullptr, "host_alloc: no CUDA device"); return GHICP_E_NODEV; }
  if (cudaMallocHost(out, bytes) != cudaSuccess) { cudaGetLastError(); *out = nullptr; return GHICP_E_NOMEM; }
  return GHICP_OK;
}
int ghicp_host_free(void *p) {
  if (p && cudaFreeHost(p) != cudaSuccess) { cudaGetLastError(); return GHICP_E_CUDA; }
  return GHICP_OK;
}

int ghicp_get_rt(ghicp_ctx *ctx, double Rt[16]) {
  Ctx *c = reinterpret_cast<Ctx *>(ctx);
  if (!c || !Rt) return GHICP_E_ARG;
  std::memcpy(Rt, c->Rt_tillnow, sizeof(double) * 16);
  return GHICP_OK;
}

int ghicp_get_fd(ghicp_ctx *ctx, double *fd) {
  Ctx *c = reinterpret_cast<Ctx *>(ctx);
  if (!c || !fd || c->N <= 0) return GHICP_E_ARG;
  int rc;
  if ((rc = use_device(c))) return rc;
  if ((rc = build_fd(c))) return rc;
  double *d_out = nullptr;
  if ((rc = dev_alloc(c, &d_out, (size_t)c->N * c->M))) return rc;
  const bool mf = c->cfg.feature_type == GHICP_FT_FPFH && c->fpfh_mf;
  cudaError_t e = mf ? launch_get_fd_mf(c, d_out) : launch_get_fd(c, d_out);
  if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
  if (e == cudaSuccess) e = cudaMemcpy(fd, d_out, (size_t)c->N * c->M * sizeof(double), cudaMemcpyDeviceToHost);
  dev_free(&d_out);
  if (e != cudaSuccess) { set_error(c, std::string("get_fd: ") + cudaGetErrorString(e)); return GHICP_E_CUDA; }
  return GHICP_OK;
}

int ghicp_probe_rowmin(ghicp_ctx *ctx, int *idx, double *cd, double *cd_mean, double *cd_std, double *penalty) {
  Ctx *c = reinterpret_cast<Ctx *>(ctx);
  if (!c || c->N <= 0) return GHICP_E_ARG;
  int rc;
  if ((rc = use_device(c))) return rc;
  if ((rc = build_fd(c))) return rc;
  const CostParams cp = make_cost_params(c);
  const LoopScalars ls = make_loop_scalars(c, cp);
  if ((rc = exact_row_stage(c, cp, ls))) return rc;
  if ((rc = comm_exchange(c, EX_STATS | EX_ROWS))) return rc;
  CK(c, launch_penalty(c, cp.pivot, ls));
  CK(c, cudaMemcpyAsync(c->h_iter, c->d_iter, sizeof(DevIter), cudaMemcpyDeviceToHost, c->stream));
  CK(c, cudaStreamSynchronize(c->stream));
  if (idx) CK(c, cudaMemcpy(idx, c->d_row_idx, sizeof(int) * (size_t)c->N, cudaMemcpyDeviceToHost));
  if (cd) CK(c, cudaMemcpy(cd, c->d_row_cd, sizeof(double) * (size_t)c->N, cudaMemcpyDeviceToHost));
  if (cd_mean) *cd_mean = c->h_iter->cd_mean;
  if (cd_std) *cd_std = c->h_iter->cd_std;
  if (penalty) *penalty = c->h_iter->penalty;
  return GHICP_OK;
}

int ghicp_set_state(ghicp_ctx *ctx, int iteration, double rms, double fdm, double fdstd, double para1, double para2) {
  Ctx *c = reinterpret_cast<Ctx *>(ctx);
  if (!c) return GHICP_E_ARG;
  c->iteration = iteration;
  c->RMS = rms; c->FDM = fdm; c->FDstd = fdstd; c->para1 = para1; c->para2 = para2;
  return GHICP_OK;
}

int ghicp_reset(ghicp_ctx *ctx) {
  Ctx *c = reinterpret_cast<Ctx *>(ctx);
  if (!c) return GHICP_E_ARG;
  reset_loop_state(c);
  c->last_cor = 0;
  return GHICP_OK;
}

// ---- stand-alone stages ------------------------------------------------------------------------
int ghicp_km_solve(int device, const double *W, int n, int sp, int tp, double eps, double penalty, int *match,
                   double *energy, int *rounds) {
  if (!W || !match || n <= 0 || sp <= 0 || tp <= 0 || sp > n || tp > n || !(eps > 0.0)) {
    set_error(nullptr, "km_solve: bad argument");
    return GHICP_E_ARG;
  }
  ghicp_config cfg;
  std::memset(&cfg, 0, sizeof(cfg));
  cfg.feature_type = GHICP_FT_NONE;
  cfg.corr_type = GHICP_CT_KM;
  cfg.dof = 6;
  cfg.device = device;
  ghicp_ctx *ctx = nullptr;
  int rc = ghicp_create(&cfg, &ctx);
  if (rc) return rc;
  Ctx *c = reinterpret_cast<Ctx *>(ctx);
  c->N = sp; c->M = tp;
  rc = alloc_workspaces(c);
  if (rc) { ghicp_destroy(ctx); return rc; }
  // candidate edges: weight != -penalty  (src/km.cpp:162), gain = penalty + w = penalty - CD
  std::vector<long long> rowptr((size_t)sp * c->n_chunks + 1, 0);
  std::vector<int> col;
  std::vector<double> gain;
  double max_gain = eps;
  for (int i = 0; i < sp; ++i) {
    for (int j = 0; j < tp; ++j) {
      const double w = W[(size_t)i * n + j];
      if (w != -penalty) {
        const double g = penalty + w;
        if (g > 0.0) { col.push_back(j); gain.push_back(g); max_gain = std::max(max_gain, g); }
      }
    }
    for (int k = 0; k < c->n_chunks; ++k) rowptr[(size_t)i * c->n_chunks + k + 1] = (long long)col.size();
  }
  // (all of row i's edges live in chunk 0: rowptr[i*n_chunks] = start, the other chunk slots = end)
  const long long nnz = (long long)col.size();
  if ((rc = ensure_edges(c, nnz))) { ghicp_destroy(ctx); return rc; }
  cudaMemcpy(c->d_rowptr, rowptr.data(), sizeof(long long) * rowptr.size(), cudaMemcpyHostToDevice);
  if (nnz > 0) {
    cudaMemcpy(c->d_csr_col, col.data(), sizeof(int) * (size_t)nnz, cudaMemcpyHostToDevice);
    cudaMemcpy(c->d_csr_gain, gain.data(), sizeof(double) * (size_t)nnz, cudaMemcpyHostToDevice);
  }
  KmResult kres;   // (the column-wise copy the reverse rounds read is built inside km_auction, when they run)
  rc = km_auction(c, sp, tp, nnz, eps, max_gain, &kres);
  if (rc) { set_error(nullptr, c->err); ghicp_destroy(ctx); return rc; }
  std::vector<int> owner(tp);
  cudaMemcpy(owner.data(), c->d_owner, sizeof(int) * (size_t)tp, cudaMemcpyDeviceToHost);
  double en = 0.0;
  int kept = 0;
  for (int y = 0; y < n; ++y) match[y] = -1;
  for (int y = 0; y < tp; ++y) {
    if (owner[y] >= 0) { match[y] = owner[y]; en -= W[(size_t)owner[y] * n + y]; ++kept; }
  }
  en += (double)(n - kept) * penalty;
  if (energy) *energy = en;
  if (rounds) *rounds = kres.rounds;
  ghicp_destroy(ctx);
  return GHICP_OK;
}

// solver < 0: the loop's SVD solve (launch_solve_explicit); otherwise launch_solve_alt_explicit with that solver
static cudaError_t rigid_fit_run(int solver, const double *s, const double *t, const double *tn, const double *w, int n,
                                 DevIter *h) {
  const size_t b3 = 3 * (size_t)n * sizeof(double);
  DevBuf<double> d_s, d_t, d_n, d_w; DevBuf<DevIter> d_iter;
  CUDA_TRY(d_s.alloc(3 * (size_t)n)); CUDA_TRY(d_t.alloc(3 * (size_t)n));
  if (tn) CUDA_TRY(d_n.alloc(3 * (size_t)n));
  if (w) CUDA_TRY(d_w.alloc((size_t)n));
  CUDA_TRY(d_iter.alloc(1));
  CUDA_TRY(cudaMemcpy(d_s.get(), s, b3, cudaMemcpyHostToDevice));
  CUDA_TRY(cudaMemcpy(d_t.get(), t, b3, cudaMemcpyHostToDevice));
  if (tn) CUDA_TRY(cudaMemcpy(d_n.get(), tn, b3, cudaMemcpyHostToDevice));
  if (w) CUDA_TRY(cudaMemcpy(d_w.get(), w, (size_t)n * sizeof(double), cudaMemcpyHostToDevice));
  CUDA_TRY(cudaMemset(d_iter.get(), 0, sizeof(DevIter)));
  CUDA_TRY(solver < 0 ? launch_solve_explicit(0, d_s.get(), d_t.get(), n, d_iter.get())
                      : launch_solve_alt_explicit(0, solver, d_s.get(), d_t.get(), d_n.get(), d_w.get(), n, d_iter.get()));
  return cudaMemcpy(h, d_iter.get(), sizeof(DevIter), cudaMemcpyDeviceToHost);
}

int ghicp_rigid_fit(int device, const double *s, const double *t, int n, double Rt[16]) {
  if (!s || !t || !Rt || n <= 0) { set_error(nullptr, "rigid_fit: bad argument"); return GHICP_E_ARG; }
  int rc;
  if ((rc = enter_device(device, "rigid_fit"))) return rc;
  DevIter h;
  if ((rc = cuda_status(rigid_fit_run(-1, s, t, nullptr, nullptr, n, &h), "rigid_fit"))) return rc;
  std::memcpy(Rt, h.Rt, sizeof(double) * 16);
  return GHICP_OK;
}

int ghicp_rigid_fit_ex(int device, int solver, const double *s, const double *t, const double *tn, const double *w,
                       int n, double Rt[16]) {
  if (!s || !t || !Rt || n <= 0 || solver < GHICP_SOLVER_SVD || solver > GHICP_SOLVER_YAW_4DOF) {
    set_error(nullptr, "rigid_fit_ex: bad argument");
    return GHICP_E_ARG;
  }
  if (solver == GHICP_SOLVER_POINT_TO_PLANE && !tn) { set_error(nullptr, "rigid_fit_ex: point-to-plane needs target normals"); return GHICP_E_ARG; }
  int rc;
  if ((rc = enter_device(device, "rigid_fit_ex"))) return rc;
  DevIter h;
  if ((rc = cuda_status(rigid_fit_run(solver, s, t, tn, w, n, &h), "rigid_fit_ex"))) return rc;
  std::memcpy(Rt, h.Rt, sizeof(double) * 16);
  return h.solve_degenerate ? GHICP_W_FEW_PAIRS : GHICP_OK;
}

// ---- pre-processing ----------------------------------------------------------------------------------------------
static cudaError_t voxel_downsample_run(const float *xyz, int n, float voxel_size, int *out_idx, int *n_out) {
  DevBuf<float> d_xyz; DevBuf<int> d_out;
  CUDA_TRY(d_xyz.alloc(3 * (size_t)n)); CUDA_TRY(d_out.alloc((size_t)n + 1));
  CUDA_TRY(cudaMemcpy(d_xyz.get(), xyz, 3 * (size_t)n * sizeof(float), cudaMemcpyHostToDevice));
  int m = 0;
  CUDA_TRY(prep_voxel_downsample(0, d_xyz.get(), n, voxel_size, d_out.get(), &m));
  if (m > 0) CUDA_TRY(cudaMemcpy(out_idx, d_out.get(), (size_t)m * sizeof(int), cudaMemcpyDeviceToHost));
  *n_out = m;
  return cudaSuccess;
}
int ghicp_voxel_downsample(int device, const float *xyz, int n, float voxel_size, int *out_idx, int *n_out) {
  if (!xyz || !out_idx || !n_out || n <= 0 || !(voxel_size > 0.f)) { set_error(nullptr, "voxel_downsample: bad argument"); return GHICP_E_ARG; }
  if (int rc = enter_device(device, "voxel_downsample")) return rc;
  return cuda_status(voxel_downsample_run(xyz, n, voxel_size, out_idx, n_out), "voxel_downsample");
}

static bool sor_args_ok(int mean_k, double std_mul) { return mean_k >= 1 && mean_k <= 128 && std::isfinite(std_mul); }
static cudaError_t sor_filter_run(const float *xyz, int n, int mean_k, double std_mul, int *out_idx, float *mean_dist,
                                  ghicp_sor_result *r) {
  DevBuf<float> d_xyz, d_dist; DevBuf<int> d_out;
  ghicp_sor_result res;
  CUDA_TRY(d_xyz.alloc(3 * (size_t)n)); CUDA_TRY(d_dist.alloc((size_t)n)); CUDA_TRY(d_out.alloc((size_t)n));
  CUDA_TRY(cudaMemcpy(d_xyz.get(), xyz, 3 * (size_t)n * sizeof(float), cudaMemcpyHostToDevice));
  CUDA_TRY(prep_sor_filter(0, d_xyz.get(), n, mean_k, std_mul, d_out.get(), d_dist.get(), &res));
  if (res.n_kept > 0) CUDA_TRY(cudaMemcpy(out_idx, d_out.get(), (size_t)res.n_kept * sizeof(int), cudaMemcpyDeviceToHost));
  if (mean_dist) CUDA_TRY(cudaMemcpy(mean_dist, d_dist.get(), (size_t)n * sizeof(float), cudaMemcpyDeviceToHost));
  *r = res;
  return cudaSuccess;
}
int ghicp_sor_filter(int device, const float *xyz, int n, int mean_k, double std_mul, int *out_idx, float *mean_dist,
                     ghicp_sor_result *r) {
  if (!xyz || !out_idx || !r || n < 0 || !sor_args_ok(mean_k, std_mul)) { set_error(nullptr, "sor_filter: bad argument"); return GHICP_E_ARG; }
  if (int rc = enter_device(device, "sor_filter")) return rc;
  if (n == 0) { *r = ghicp_sor_result{}; return GHICP_OK; }
  return cuda_status(sor_filter_run(xyz, n, mean_k, std_mul, out_idx, mean_dist, r), "sor_filter");
}

static cudaError_t detect_keypoints_run(const float *xyz, int n, float radius, float ratio_max, int min_pts, float nms_radius,
                                        int *kp_idx, int *n_kp, float *lam, double *curvature, int *pt_num) {
  DevBuf<float> d_xyz, d_lam; DevBuf<double> d_curv; DevBuf<int> d_cnt, d_kp;
  CUDA_TRY(d_xyz.alloc(3 * (size_t)n)); CUDA_TRY(d_lam.alloc(3 * (size_t)n)); CUDA_TRY(d_curv.alloc((size_t)n));
  CUDA_TRY(d_cnt.alloc((size_t)n)); CUDA_TRY(d_kp.alloc((size_t)n));
  CUDA_TRY(cudaMemcpy(d_xyz.get(), xyz, 3 * (size_t)n * sizeof(float), cudaMemcpyHostToDevice));
  int m = 0, rounds = 0;
  CUDA_TRY(prep_detect_keypoints(0, d_xyz.get(), n, radius, ratio_max, min_pts, nms_radius, d_lam.get(), d_curv.get(), d_cnt.get(),
                                 d_kp.get(), &m, &rounds));
  if (m > 0) CUDA_TRY(cudaMemcpy(kp_idx, d_kp.get(), (size_t)m * sizeof(int), cudaMemcpyDeviceToHost));
  if (lam) CUDA_TRY(cudaMemcpy(lam, d_lam.get(), 3 * (size_t)n * sizeof(float), cudaMemcpyDeviceToHost));
  if (curvature) CUDA_TRY(cudaMemcpy(curvature, d_curv.get(), (size_t)n * sizeof(double), cudaMemcpyDeviceToHost));
  if (pt_num) CUDA_TRY(cudaMemcpy(pt_num, d_cnt.get(), (size_t)n * sizeof(int), cudaMemcpyDeviceToHost));
  *n_kp = m;
  return cudaSuccess;
}
int ghicp_detect_keypoints(int device, const float *xyz, int n, float radius, float ratio_max, int min_pts, float nms_radius,
                           int *kp_idx, int *n_kp, float *lam, double *curvature, int *pt_num) {
  if (!xyz || !kp_idx || !n_kp || n <= 0 || !(radius > 0.f) || !(nms_radius > 0.f)) { set_error(nullptr, "detect_keypoints: bad argument"); return GHICP_E_ARG; }
  if (int rc = enter_device(device, "detect_keypoints")) return rc;
  return cuda_status(detect_keypoints_run(xyz, n, radius, ratio_max, min_pts, nms_radius, kp_idx, n_kp, lam, curvature, pt_num),
                     "detect_keypoints");
}

static cudaError_t bsc_extract_run(const float *xyz, int n, const int *kp_idx, int nkp, float extract_radius, int side,
                                   const int *pairs, int dof_type, unsigned char *features, float *lrf, int *status) {
  const int V = dof_type > 4 ? 4 : (dof_type > 0 ? 2 : 1), S2 = side * side;
  const size_t nbytes = (size_t)(9 * S2 + 7) / 8, out_bytes = (size_t)V * nkp * nbytes;
  DevBuf<float> d_xyz, d_lrf; DevBuf<int> d_kp, d_pairs, d_status; DevBuf<unsigned char> d_bits;
  CUDA_TRY(d_xyz.alloc(3 * (size_t)n)); CUDA_TRY(d_kp.alloc((size_t)nkp)); CUDA_TRY(d_pairs.alloc(2 * (size_t)S2));
  CUDA_TRY(d_bits.alloc(out_bytes)); CUDA_TRY(d_lrf.alloc(12 * (size_t)nkp)); CUDA_TRY(d_status.alloc((size_t)nkp));
  CUDA_TRY(cudaMemcpy(d_xyz.get(), xyz, 3 * (size_t)n * sizeof(float), cudaMemcpyHostToDevice));
  CUDA_TRY(cudaMemcpy(d_kp.get(), kp_idx, (size_t)nkp * sizeof(int), cudaMemcpyHostToDevice));
  CUDA_TRY(cudaMemcpy(d_pairs.get(), pairs, 2 * (size_t)S2 * sizeof(int), cudaMemcpyHostToDevice));
  CUDA_TRY(prep_bsc_extract(0, d_xyz.get(), n, d_kp.get(), nkp, extract_radius, side, d_pairs.get(), dof_type, d_bits.get(),
                            d_lrf.get(), d_status.get()));
  CUDA_TRY(cudaMemcpy(features, d_bits.get(), out_bytes, cudaMemcpyDeviceToHost));
  if (lrf) CUDA_TRY(cudaMemcpy(lrf, d_lrf.get(), 12 * (size_t)nkp * sizeof(float), cudaMemcpyDeviceToHost));
  if (status) CUDA_TRY(cudaMemcpy(status, d_status.get(), (size_t)nkp * sizeof(int), cudaMemcpyDeviceToHost));
  return cudaSuccess;
}
int ghicp_bsc_extract(int device, const float *xyz, int n, const int *kp_idx, int nkp, float extract_radius, int voxel_side_num,
                      const int *pairs, int dof_type, unsigned char *features, int *n_variants, float *lrf, int *status) {
  if (!xyz || !kp_idx || !pairs || !features || n <= 0 || nkp <= 0 || !(extract_radius > 0.f) || voxel_side_num < 1 ||
      voxel_side_num > 9) {
    set_error(nullptr, "bsc_extract: bad argument");
    return GHICP_E_ARG;
  }
  const int S2 = voxel_side_num * voxel_side_num;
  for (int i = 0; i < nkp; ++i) if (kp_idx[i] < 0 || kp_idx[i] >= n) { set_error(nullptr, "bsc_extract: keypoint index out of range"); return GHICP_E_ARG; }
  for (int i = 0; i < 2 * S2; ++i) if (pairs[i] < 0 || pairs[i] >= S2) { set_error(nullptr, "bsc_extract: sampling pair out of range"); return GHICP_E_ARG; }
  int rc;
  if ((rc = enter_device(device, "bsc_extract"))) return rc;
  if ((rc = cuda_status(bsc_extract_run(xyz, n, kp_idx, nkp, extract_radius, voxel_side_num, pairs, dof_type, features, lrf, status),
                        "bsc_extract")))
    return rc;
  if (n_variants) *n_variants = dof_type > 4 ? 4 : (dof_type > 0 ? 2 : 1);
  return GHICP_OK;
}

// ---- device-resident pipeline: raw cloud -> down-sampled cloud -> keypoints -> descriptors ---------------------------------
struct ghicp_prep {
  int device = 0;
  int n = 0, n_down = 0, n_kp = 0, V = 0, side = 0, nbytes = 0;
  DevBuf<float> d_down;           // [n_down][3]
  DevBuf<int> d_kp;               // [n_kp] indices into d_down
  DevBuf<double> d_kp_xyz;        // [3][n_kp]
  DevBuf<unsigned char> d_bits;   // [V][n_kp][nbytes]
  DevBuf<float> d_fpfh;           // [n_kp][33] after ghicp_prep_fpfh
  float bbox_min[3] = {0, 0, 0}, bbox_max[3] = {0, 0, 0};
  float stage_ms[5] = {0, 0, 0, 0, 0};
  bool sor = false;                     // made by ghicp_prep_run_sor with the filter on
  ghicp_sor_result sor_result{};
  int n_voxel = 0;                      // the down-sampled cloud's size before the filter
  float sor_ms = 0.f;
  FpfhStats fpfh_stats;
  OverlapTarget *ov_target = nullptr;   // the down-sampled cloud's grid as an overlap target, after ghicp_prep_overlap
  DevBuf<float> icp_nrm;                // [n_down][3] k-NN normals, after ghicp_prep_icp with metric 1 (target) or 2 (either)
  int icp_nrm_k = 0;                    // their k (0: none)
  std::mutex ov_mu;                     // guards ov_target and the normals: concurrent first calls on one result build once
};

int ghicp_prep_destroy(ghicp_prep *h) {
  if (!h) return GHICP_OK;
  cudaSetDevice(h->device);
  overlap_target_free(h->ov_target);
  delete h;
  return GHICP_OK;
}

// events: 0 start, 1 uploaded, 2 voxel filter, 3 outlier filter (mean_k > 0; else right after 2), 4 keypoints, 5 end
static cudaError_t prep_run_stages(const float *xyz, int n, const ghicp_prep_params *p, const int *bsc_pairs, bool want_bsc,
                                   int sor_k, double sor_std, ghicp_prep *h) {
  const int side = h->side;
  StageEvents<6> ev;
  DevBuf<float> d_xyz, d_lam, d_lrf, d_dist; DevBuf<double> d_curv;
  DevBuf<int> d_keep, d_cnt, d_kpbuf, d_pairs, d_status;
  CUDA_TRY(ev.create());
  CUDA_TRY(d_xyz.alloc(3 * (size_t)n)); CUDA_TRY(d_keep.alloc((size_t)n + 1));
  CUDA_TRY(cudaEventRecord(ev[0], 0));
  CUDA_TRY(cudaMemcpyAsync(d_xyz.get(), xyz, 3 * (size_t)n * sizeof(float), cudaMemcpyHostToDevice, 0));
  CUDA_TRY(cudaEventRecord(ev[1], 0));
  int n_down = 0, n_kp = 0, rounds = 0;
  CUDA_TRY(prep_voxel_downsample(0, d_xyz.get(), n, p->voxel_size, d_keep.get(), &n_down));
  if (n_down <= 0) { h->n_down = 0; return cudaSuccess; }   // no finite point: ghicp_prep_run refuses the cloud
  CUDA_TRY(h->d_down.alloc(3 * (size_t)n_down));
  CUDA_TRY(prep_gather_points(0, d_xyz.get(), d_keep.get(), n_down, h->d_down.get()));
  CUDA_TRY(cudaEventRecord(ev[2], 0));
  d_xyz.reset(); d_keep.reset();
  if (sor_k > 0) {   // the outlier filter on the down-sampled cloud; the kept points replace it
    DevBuf<float> kept;
    h->n_voxel = n_down;
    CUDA_TRY(d_keep.alloc((size_t)n_down)); CUDA_TRY(d_dist.alloc((size_t)n_down));
    CUDA_TRY(prep_sor_filter(0, h->d_down.get(), n_down, sor_k, sor_std, d_keep.get(), d_dist.get(), &h->sor_result));
    n_down = h->sor_result.n_kept;
    if (n_down <= 0) { h->n_down = 0; return cudaSuccess; }   // nothing kept: refused like a cloud without a finite point
    CUDA_TRY(kept.alloc(3 * (size_t)n_down));
    CUDA_TRY(prep_gather_points(0, h->d_down.get(), d_keep.get(), n_down, kept.get()));
    h->d_down = std::move(kept);
    d_keep.reset(); d_dist.reset();
  }
  CUDA_TRY(cudaEventRecord(ev[3], 0));
  CUDA_TRY(prep_bounds(0, h->d_down.get(), n_down, h->bbox_min, h->bbox_max));
  CUDA_TRY(d_lam.alloc(3 * (size_t)n_down)); CUDA_TRY(d_curv.alloc((size_t)n_down));
  CUDA_TRY(d_cnt.alloc((size_t)n_down)); CUDA_TRY(d_kpbuf.alloc((size_t)n_down));
  CUDA_TRY(prep_detect_keypoints(0, h->d_down.get(), n_down, p->neighborhood_radius, p->ratio_max, p->min_pts, p->nms_radius,
                                 d_lam.get(), d_curv.get(), d_cnt.get(), d_kpbuf.get(), &n_kp, &rounds));
  CUDA_TRY(cudaEventRecord(ev[4], 0));
  h->n_down = n_down; h->n_kp = n_kp;
  if (n_kp > 0) {
    CUDA_TRY(h->d_kp.alloc((size_t)n_kp));
    CUDA_TRY(cudaMemcpyAsync(h->d_kp.get(), d_kpbuf.get(), (size_t)n_kp * sizeof(int), cudaMemcpyDeviceToDevice, 0));
    CUDA_TRY(h->d_kp_xyz.alloc(3 * (size_t)n_kp));
    CUDA_TRY(prep_kp_coords(0, h->d_down.get(), h->d_kp.get(), n_kp, h->d_kp_xyz.get()));
    if (want_bsc) {
      h->V = p->dof_type > 4 ? 4 : (p->dof_type > 0 ? 2 : 1);
      h->nbytes = (9 * side * side + 7) / 8;
      CUDA_TRY(h->d_bits.alloc((size_t)h->V * n_kp * h->nbytes));
      CUDA_TRY(d_pairs.alloc(2 * (size_t)side * side)); CUDA_TRY(d_lrf.alloc(12 * (size_t)n_kp)); CUDA_TRY(d_status.alloc((size_t)n_kp));
      CUDA_TRY(cudaMemcpyAsync(d_pairs.get(), bsc_pairs, 2 * (size_t)side * side * sizeof(int), cudaMemcpyHostToDevice, 0));
      CUDA_TRY(prep_bsc_extract(0, h->d_down.get(), n_down, h->d_kp.get(), n_kp, p->bsc_radius, side, d_pairs.get(), p->dof_type,
                                h->d_bits.get(), d_lrf.get(), d_status.get()));
    }
  }
  CUDA_TRY(cudaEventRecord(ev[5], 0));
  CUDA_TRY(cudaStreamSynchronize(0));
  h->stage_ms[0] = ev.ms(0, 1); h->stage_ms[1] = ev.ms(1, 2); h->stage_ms[2] = ev.ms(3, 4); h->stage_ms[3] = ev.ms(4, 5);
  h->stage_ms[4] = ev.ms(0, 5);
  h->sor_ms = ev.ms(2, 3);
  return cudaSuccess;
}
int ghicp_prep_run(int device, const float *xyz, int n, const ghicp_prep_params *p, const int *bsc_pairs, ghicp_prep **out) {
  return ghicp_prep_run_sor(device, xyz, n, p, bsc_pairs, 0, 0.0, out);
}
int ghicp_prep_run_sor(int device, const float *xyz, int n, const ghicp_prep_params *p, const int *bsc_pairs, int mean_k,
                       double std_mul, ghicp_prep **out) {
  if (!xyz || !p || !out || n <= 0 || !(p->voxel_size > 0.f) || !(p->neighborhood_radius > 0.f) || !(p->nms_radius > 0.f) ||
      (mean_k != 0 && !sor_args_ok(mean_k, std_mul))) {
    set_error(nullptr, "prep_run: bad argument");
    return GHICP_E_ARG;
  }
  const bool want_bsc = p->bsc_radius > 0.f;
  const int side = p->bsc_side > 0 ? p->bsc_side : 7;
  if (want_bsc && (!bsc_pairs || side > 9)) { set_error(nullptr, "prep_run: BSC needs the sampling pattern and voxel_side_num <= 9"); return GHICP_E_ARG; }
  if (want_bsc) for (int i = 0; i < 2 * side * side; ++i) if (bsc_pairs[i] < 0 || bsc_pairs[i] >= side * side) { set_error(nullptr, "prep_run: sampling pair out of range"); return GHICP_E_ARG; }
  int rc;
  if ((rc = enter_device(device, "prep_run"))) return rc;
  ghicp_prep *h = new ghicp_prep();
  h->device = device; h->n = n; h->side = side; h->sor = mean_k > 0;
  if ((rc = cuda_status(prep_run_stages(xyz, n, p, bsc_pairs, want_bsc, mean_k, std_mul, h), "prep_run"))) { ghicp_prep_destroy(h); return rc; }
  if (h->n_down <= 0) {
    const bool filtered = h->sor && h->n_voxel > 0;
    ghicp_prep_destroy(h);
    set_error(nullptr, filtered ? "prep_run: the outlier filter kept no point" : "prep_run: the cloud has no finite point");
    return GHICP_E_ARG;
  }
  *out = h;
  return GHICP_OK;
}

int ghicp_prep_sor_info(const ghicp_prep *h, ghicp_sor_result *r, int *n_voxel, float *ms) {
  if (!h || !h->sor) { set_error(nullptr, "prep_sor_info: the result was made without the outlier filter"); return GHICP_E_ARG; }
  if (r) *r = h->sor_result;
  if (n_voxel) *n_voxel = h->n_voxel;
  if (ms) *ms = h->sor_ms;
  return GHICP_OK;
}

int ghicp_prep_info(const ghicp_prep *h, int *n_down, int *n_kp, int *n_variants, float bbox_min[3], float bbox_max[3], float stage_ms[5]) {
  if (!h) return GHICP_E_ARG;
  if (n_down) *n_down = h->n_down;
  if (n_kp) *n_kp = h->n_kp;
  if (n_variants) *n_variants = h->V;
  if (bbox_min) std::memcpy(bbox_min, h->bbox_min, sizeof(float) * 3);
  if (bbox_max) std::memcpy(bbox_max, h->bbox_max, sizeof(float) * 3);
  if (stage_ms) std::memcpy(stage_ms, h->stage_ms, sizeof(float) * 5);
  return GHICP_OK;
}

static cudaError_t prep_get_run(const ghicp_prep *h, float *down_xyz, int *kp_idx, double *kp_xyz, unsigned char *bsc_bits) {
  if (down_xyz && h->n_down > 0) CUDA_TRY(cudaMemcpy(down_xyz, h->d_down.get(), 3 * (size_t)h->n_down * sizeof(float), cudaMemcpyDeviceToHost));
  if (kp_idx && h->n_kp > 0) CUDA_TRY(cudaMemcpy(kp_idx, h->d_kp.get(), (size_t)h->n_kp * sizeof(int), cudaMemcpyDeviceToHost));
  if (kp_xyz && h->n_kp > 0) CUDA_TRY(cudaMemcpy(kp_xyz, h->d_kp_xyz.get(), 3 * (size_t)h->n_kp * sizeof(double), cudaMemcpyDeviceToHost));
  if (bsc_bits && h->d_bits.get()) CUDA_TRY(cudaMemcpy(bsc_bits, h->d_bits.get(), (size_t)h->V * h->n_kp * h->nbytes, cudaMemcpyDeviceToHost));
  return cudaSuccess;
}
int ghicp_prep_get(const ghicp_prep *h, float *down_xyz, int *kp_idx, double *kp_xyz, unsigned char *bsc_bits) {
  if (!h) return GHICP_E_ARG;
  if (int rc = enter_device(h->device, "prep_get")) return rc;
  return cuda_status(prep_get_run(h, down_xyz, kp_idx, kp_xyz, bsc_bits), "prep_get");
}

int ghicp_set_from_prep(ghicp_ctx *ctx, const ghicp_prep *src, const ghicp_prep *tgt) {
  Ctx *c = reinterpret_cast<Ctx *>(ctx);
  if (!c || !src || !tgt || src->n_kp <= 0 || tgt->n_kp <= 0) { set_error(c, "set_from_prep: bad argument or a cloud without keypoints"); return GHICP_E_ARG; }
  if (src->device != c->device || tgt->device != c->device) { set_error(c, "set_from_prep: pipeline results live on another device"); return GHICP_E_ARG; }
  int rc;
  if ((rc = use_device(c))) return rc;
  const int N = src->n_kp, M = tgt->n_kp;
  if ((rc = resize_keypoints(c, N, M))) return rc;
  CK(c, cudaMemcpyAsync(c->d_s, src->d_kp_xyz.get(), 3 * (size_t)N * sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
  CK(c, cudaMemcpyAsync(c->d_t, tgt->d_kp_xyz.get(), 3 * (size_t)M * sizeof(double), cudaMemcpyDeviceToDevice, c->stream));
  {  // centre of the FP32 filter coordinates = target centroid (scalars only; the 24 M bytes read back are not re-uploaded)
    std::vector<double> ht(3 * (size_t)M);
    CK(c, cudaMemcpyAsync(ht.data(), tgt->d_kp_xyz.get(), 3 * (size_t)M * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    CK(c, cudaStreamSynchronize(c->stream));
    double cx = 0, cy = 0, cz = 0;
    for (int j = 0; j < M; ++j) { cx += ht[j]; cy += ht[(size_t)M + j]; cz += ht[2 * (size_t)M + j]; }
    c->center[0] = cx / M; c->center[1] = cy / M; c->center[2] = cz / M;
  }
  if (c->cfg.feature_type == GHICP_FT_BSC) {
    const int Vneed = (c->cfg.dof == 6) ? 4 : 2;
    if (!src->d_bits.get() || !tgt->d_bits.get() || src->V < Vneed || src->nbytes != tgt->nbytes) {
      set_error(c, "set_from_prep: BSC context needs descriptors (source with the context's dof variants, same length)");
      return GHICP_E_ARG;
    }
    const int bits = 9 * src->side * src->side;
    c->V = src->V; c->bits = bits;
    c->Bbytes = src->nbytes;
    c->W64 = (c->Bbytes + 7) / 8;
    if ((rc = dev_alloc(c, &c->d_bs, (size_t)c->V * c->W64 * c->N))) return rc;
    if ((rc = dev_alloc(c, &c->d_bt, (size_t)c->W64 * c->M))) return rc;
    CK(c, launch_pack_bsc(c, src->d_bits.get(), tgt->d_bits.get()));   // the target's variant 0 = its first [M][B] block
    CK(c, cudaStreamSynchronize(c->stream));
    c->have_bsc = true;
    c->fd_built = false;
  }
  if (c->cfg.feature_type == GHICP_FT_FPFH && src->d_fpfh.get() && tgt->d_fpfh.get()) {
    if ((rc = set_fpfh_from(c, src->d_fpfh.get(), tgt->d_fpfh.get(), cudaMemcpyDeviceToDevice))) return rc;
  }
  return GHICP_OK;
}

// ---- FPFH estimator ----------------------------------------------------------------------------------------------------
// GHICP_FPFH_CELL_SCALE (test hook) scales the k-NN grid's cell edge; results must not change, only the work per query
static float fpfh_cell_scale() {
  const char *s = getenv("GHICP_FPFH_CELL_SCALE");
  const float v = s ? (float)atof(s) : 0.f;
  return v > 0.f ? v : 1.f;
}

static cudaError_t fpfh_extract_run(const float *xyz, int n, const int *idx, int nidx, int k, float *fpfh, float *normals, int *status) {
  DevBuf<float> d_xyz, d_fpfh, d_nrm; DevBuf<int> d_status, d_idx;
  CUDA_TRY(d_xyz.alloc(3 * (size_t)n)); CUDA_TRY(d_fpfh.alloc((size_t)nidx * 33 + 1)); CUDA_TRY(d_nrm.alloc(3 * (size_t)n));
  CUDA_TRY(d_status.alloc((size_t)n));
  if (idx) CUDA_TRY(d_idx.alloc((size_t)nidx + 1));
  CUDA_TRY(cudaMemcpy(d_xyz.get(), xyz, 3 * (size_t)n * sizeof(float), cudaMemcpyHostToDevice));
  if (idx && nidx > 0) CUDA_TRY(cudaMemcpy(d_idx.get(), idx, (size_t)nidx * sizeof(int), cudaMemcpyHostToDevice));
  CUDA_TRY(prep_fpfh(0, d_xyz.get(), n, d_idx.get(), nidx, k, fpfh_cell_scale(), d_fpfh.get(), d_nrm.get(), d_status.get(), nullptr,
                     nullptr, nullptr, nullptr));
  if (nidx > 0) CUDA_TRY(cudaMemcpy(fpfh, d_fpfh.get(), (size_t)nidx * 33 * sizeof(float), cudaMemcpyDeviceToHost));
  if (normals) CUDA_TRY(cudaMemcpy(normals, d_nrm.get(), 3 * (size_t)n * sizeof(float), cudaMemcpyDeviceToHost));
  if (status) CUDA_TRY(cudaMemcpy(status, d_status.get(), (size_t)n * sizeof(int), cudaMemcpyDeviceToHost));
  return cudaSuccess;
}
int ghicp_fpfh_extract(int device, const float *xyz, int n, const int *idx, int nidx, int k, float *fpfh, float *normals, int *status) {
  if (!xyz || n <= 0 || k < 3 || k > 32 || (idx && nidx < 0) || (nidx > 0 && !fpfh)) { set_error(nullptr, "fpfh_extract: bad argument"); return GHICP_E_ARG; }
  if (!idx) nidx = n;
  if (idx) for (int i = 0; i < nidx; ++i) if (idx[i] < 0 || idx[i] >= n) { set_error(nullptr, "fpfh_extract: index out of range"); return GHICP_E_ARG; }
  if (int rc = enter_device(device, "fpfh_extract")) return rc;
  return cuda_status(fpfh_extract_run(xyz, n, idx, nidx, k, fpfh, normals, status), "fpfh_extract");
}

static cudaError_t prep_fpfh_run(ghicp_prep *h, int k, float ms[3]) {
  StageEvents<3> ev;
  DevBuf<float> d_nrm;
  CUDA_TRY(ev.create());
  if (!h->d_fpfh.get()) CUDA_TRY(h->d_fpfh.alloc((size_t)h->n_kp * 33 + 1));
  CUDA_TRY(d_nrm.alloc(3 * (size_t)h->n_down));
  CUDA_TRY(cudaEventRecord(ev[0], 0));
  CUDA_TRY(prep_fpfh(0, h->d_down.get(), h->n_down, h->d_kp.get(), h->n_kp, k, fpfh_cell_scale(), h->d_fpfh.get(), d_nrm.get(), nullptr,
                     nullptr, nullptr, ev[1], &h->fpfh_stats));
  CUDA_TRY(cudaEventRecord(ev[2], 0));
  CUDA_TRY(cudaStreamSynchronize(0));
  ms[0] = ev.ms(0, 1); ms[1] = ev.ms(1, 2); ms[2] = ev.ms(0, 2);
  return cudaSuccess;
}
int ghicp_prep_fpfh(ghicp_prep *h, int k, float stage_ms[3]) {
  if (!h || k < 3 || k > 32 || h->n_kp <= 0) { set_error(nullptr, "prep_fpfh: bad argument or a cloud without keypoints"); return GHICP_E_ARG; }
  int rc;
  if ((rc = enter_device(h->device, "prep_fpfh"))) return rc;
  float ms[3] = {0.f, 0.f, 0.f};
  if ((rc = cuda_status(prep_fpfh_run(h, k, ms), "prep_fpfh"))) {
    h->d_fpfh.reset();   // a failed call leaves no histograms behind
    return rc;
  }
  if (stage_ms) std::memcpy(stage_ms, ms, sizeof(ms));
  return GHICP_OK;
}

int ghicp_prep_get_fpfh(const ghicp_prep *h, float *fpfh) {
  if (!h || !fpfh || !h->d_fpfh.get()) { set_error(nullptr, "prep_get_fpfh: no histograms (call ghicp_prep_fpfh first)"); return GHICP_E_ARG; }
  if (int rc = enter_device(h->device, "prep_get_fpfh")) return rc;
  if (h->n_kp <= 0) return GHICP_OK;
  return cuda_status(cudaMemcpy(fpfh, h->d_fpfh.get(), (size_t)h->n_kp * 33 * sizeof(float), cudaMemcpyDeviceToHost), "prep_get_fpfh");
}

int ghicp_prep_fpfh_stats(const ghicp_prep *h, long long *candidates, int *queries, int *fallbacks, float *cell) {
  if (!h || !h->d_fpfh.get()) { set_error(nullptr, "prep_fpfh_stats: no histograms (call ghicp_prep_fpfh first)"); return GHICP_E_ARG; }
  if (candidates) *candidates = h->fpfh_stats.candidates;
  if (queries) *queries = h->fpfh_stats.queries;
  if (fallbacks) *fallbacks = h->fpfh_stats.fallbacks;
  if (cell) *cell = h->fpfh_stats.cell;
  return GHICP_OK;
}

// ---- FPFH over radius neighbourhoods -------------------------------------------------------------------------------------
// GHICP_FPFH_NB_MAX=<entries> (test hook) lowers the neighbour-list budget, forcing the GHICP_E_NOMEM path at any size
static long long fpfh_nb_max() {
  const char *s = getenv("GHICP_FPFH_NB_MAX");
  return s ? atoll(s) : 0;
}
static bool radii_ok(float rn, float rf, const char *who) {
  // the lists compare against r*r in float32: a radius whose square is 0 or infinite is refused with the others
  const bool ok = std::isfinite(rn) && std::isfinite(rf) && rn > 0.f && rf > 0.f && rn * rn > 0.f && rf * rf > 0.f &&
                  std::isfinite(rn * rn) && std::isfinite(rf * rf);
  if (!ok) set_error(nullptr, std::string(who) + ": normal_radius and feature_radius must be positive and finite");
  return ok;
}
static int fpfh_radius_status(cudaError_t e, const FpfhRadiusStats &s, const char *who) {
  if (e == cudaErrorMemoryAllocation && s.needed > s.budget) {
    cudaGetLastError();
    set_error(nullptr, std::string(who) + ": the neighbour lists need at least " + std::to_string(s.needed) + " entries, the budget is " +
                           std::to_string(s.budget) + " entries (16 bytes each)");
    return GHICP_E_NOMEM;
  }
  return cuda_status(e, who);
}

static cudaError_t fpfh_extract_radius_run(const float *xyz, int n, const int *idx, int nidx, float rn, float rf, float *fpfh,
                                           float *normals, int *status, FpfhRadiusStats *s) {
  DevBuf<float> d_xyz, d_fpfh, d_nrm; DevBuf<int> d_status, d_idx;
  CUDA_TRY(d_xyz.alloc(3 * (size_t)n)); CUDA_TRY(d_fpfh.alloc((size_t)nidx * 33 + 1)); CUDA_TRY(d_nrm.alloc(3 * (size_t)n));
  CUDA_TRY(d_status.alloc((size_t)n));
  if (idx) CUDA_TRY(d_idx.alloc((size_t)nidx + 1));
  CUDA_TRY(cudaMemcpy(d_xyz.get(), xyz, 3 * (size_t)n * sizeof(float), cudaMemcpyHostToDevice));
  if (idx && nidx > 0) CUDA_TRY(cudaMemcpy(d_idx.get(), idx, (size_t)nidx * sizeof(int), cudaMemcpyHostToDevice));
  CUDA_TRY(prep_fpfh_radius(0, d_xyz.get(), n, d_idx.get(), nidx, rn, rf, fpfh_nb_max(), d_fpfh.get(), d_nrm.get(), d_status.get(),
                            nullptr, nullptr, s));
  if (nidx > 0) CUDA_TRY(cudaMemcpy(fpfh, d_fpfh.get(), (size_t)nidx * 33 * sizeof(float), cudaMemcpyDeviceToHost));
  if (normals) CUDA_TRY(cudaMemcpy(normals, d_nrm.get(), 3 * (size_t)n * sizeof(float), cudaMemcpyDeviceToHost));
  if (status) CUDA_TRY(cudaMemcpy(status, d_status.get(), (size_t)n * sizeof(int), cudaMemcpyDeviceToHost));
  return cudaSuccess;
}
int ghicp_fpfh_extract_radius(int device, const float *xyz, int n, const int *idx, int nidx, float normal_radius,
                              float feature_radius, float *fpfh, float *normals, int *status) {
  if (!xyz || n <= 0 || (idx && nidx < 0) || ((idx ? nidx : n) > 0 && !fpfh)) { set_error(nullptr, "fpfh_extract_radius: bad argument"); return GHICP_E_ARG; }
  if (!radii_ok(normal_radius, feature_radius, "fpfh_extract_radius")) return GHICP_E_ARG;
  if (!idx) nidx = n;
  if (idx) for (int i = 0; i < nidx; ++i) if (idx[i] < 0 || idx[i] >= n) { set_error(nullptr, "fpfh_extract_radius: index out of range"); return GHICP_E_ARG; }
  if (int rc = enter_device(device, "fpfh_extract_radius")) return rc;
  FpfhRadiusStats s;
  const cudaError_t e = fpfh_extract_radius_run(xyz, n, idx, nidx, normal_radius, feature_radius, fpfh, normals, status, &s);
  return fpfh_radius_status(e, s, "fpfh_extract_radius");
}

static cudaError_t prep_fpfh_radius_run(ghicp_prep *h, float rn, float rf, float ms[4], FpfhRadiusStats *s) {
  StageEvents<4> ev;
  DevBuf<float> d_nrm, d_out;
  CUDA_TRY(ev.create());
  // into a fresh buffer: histograms a failed call leaves behind are never mistaken for results
  CUDA_TRY(d_out.alloc((size_t)h->n_kp * 33 + 1));
  CUDA_TRY(d_nrm.alloc(3 * (size_t)h->n_down));
  CUDA_TRY(cudaEventRecord(ev[0], 0));
  CUDA_TRY(prep_fpfh_radius(0, h->d_down.get(), h->n_down, h->d_kp.get(), h->n_kp, rn, rf, fpfh_nb_max(), d_out.get(), d_nrm.get(),
                            nullptr, ev[1], ev[2], s));
  CUDA_TRY(cudaEventRecord(ev[3], 0));
  CUDA_TRY(cudaStreamSynchronize(0));
  ms[0] = ev.ms(0, 1); ms[1] = ev.ms(1, 2); ms[2] = ev.ms(2, 3); ms[3] = ev.ms(0, 3);
  h->d_fpfh = std::move(d_out);
  return cudaSuccess;
}
int ghicp_prep_fpfh_radius(ghicp_prep *h, float normal_radius, float feature_radius, float stage_ms[4], long long work[3]) {
  if (!h || h->n_kp <= 0) { set_error(nullptr, "prep_fpfh_radius: bad argument or a cloud without keypoints"); return GHICP_E_ARG; }
  if (!radii_ok(normal_radius, feature_radius, "prep_fpfh_radius")) return GHICP_E_ARG;
  int rc;
  if ((rc = enter_device(h->device, "prep_fpfh_radius"))) return rc;
  FpfhRadiusStats s;
  float ms[4] = {0.f, 0.f, 0.f, 0.f};
  if ((rc = fpfh_radius_status(prep_fpfh_radius_run(h, normal_radius, feature_radius, ms, &s), s, "prep_fpfh_radius"))) return rc;
  if (stage_ms) std::memcpy(stage_ms, ms, sizeof(ms));
  if (work) { work[0] = s.nb_n; work[1] = s.nb_f; work[2] = s.spfh_points; }
  return GHICP_OK;
}

// ---- SAC-IA coarse alignment -------------------------------------------------------------------------------------------
static bool sac_params_ok(const ghicp_sac_params *p, const char *who) {
  const char *why = nullptr;
  if (!p) why = "no parameters";
  else if (p->max_iterations < 1) why = "max_iterations must be >= 1";
  else if (p->nr_samples < 3 || p->nr_samples > ghicp_sac::SAC_MAX_SAMPLES) why = "nr_samples must be in 3..8";
  else if (p->k_correspondences < 1 || p->k_correspondences > ghicp_sac::SAC_KMAX) why = "k_correspondences must be in 1..32";
  else if (!(p->min_sample_distance >= 0.f) || !std::isfinite(p->min_sample_distance)) why = "min_sample_distance must be finite and >= 0";
  else if (!(p->corr_dist_threshold > 0.f) || !std::isfinite(p->corr_dist_threshold)) why = "corr_dist_threshold must be finite and > 0";
  if (why) set_error(nullptr, std::string(who) + ": " + why);
  return why == nullptr;
}

static cudaError_t sac_ia_run(const float *src_xyz, const float *src_fpfh, int n_s, const float *tgt_xyz, const float *tgt_fpfh,
                              int n_t, const ghicp_sac_params *p, ghicp_sac_result *out) {
  DevBuf<float> d_p, d_fs, d_q, d_ft;
  CUDA_TRY(d_p.alloc(3 * (size_t)n_s)); CUDA_TRY(d_fs.alloc(33 * (size_t)n_s));
  CUDA_TRY(d_q.alloc(3 * (size_t)n_t)); CUDA_TRY(d_ft.alloc(33 * (size_t)n_t));
  CUDA_TRY(cudaMemcpyAsync(d_p.get(), src_xyz, 3 * (size_t)n_s * sizeof(float), cudaMemcpyHostToDevice, 0));
  CUDA_TRY(cudaMemcpyAsync(d_fs.get(), src_fpfh, 33 * (size_t)n_s * sizeof(float), cudaMemcpyHostToDevice, 0));
  CUDA_TRY(cudaMemcpyAsync(d_q.get(), tgt_xyz, 3 * (size_t)n_t * sizeof(float), cudaMemcpyHostToDevice, 0));
  CUDA_TRY(cudaMemcpyAsync(d_ft.get(), tgt_fpfh, 33 * (size_t)n_t * sizeof(float), cudaMemcpyHostToDevice, 0));
  return sac_run(d_p.get(), d_fs.get(), n_s, d_q.get(), d_ft.get(), n_t, p, out, nullptr);
}
int ghicp_sac_ia(int device, const float *src_xyz, const float *src_fpfh, int n_s, const float *tgt_xyz, const float *tgt_fpfh,
                 int n_t, const ghicp_sac_params *p, ghicp_sac_result *out) {
  if (!src_xyz || !src_fpfh || !tgt_xyz || !tgt_fpfh || !out || n_s <= 0 || n_t <= 0) {
    set_error(nullptr, "sac_ia: bad argument (null array or empty cloud)");
    return GHICP_E_ARG;
  }
  if (!sac_params_ok(p, "sac_ia")) return GHICP_E_ARG;
  if (int rc = enter_device(device, "sac_ia")) return rc;
  return cuda_status(sac_ia_run(src_xyz, src_fpfh, n_s, tgt_xyz, tgt_fpfh, n_t, p, out), "sac_ia");
}

static cudaError_t prep_sac_ia_run(const ghicp_prep *src, const ghicp_prep *tgt, const ghicp_sac_params *p, ghicp_sac_result *out) {
  DevBuf<float> d_p, d_q;
  CUDA_TRY(d_p.alloc(3 * (size_t)src->n_kp)); CUDA_TRY(d_q.alloc(3 * (size_t)tgt->n_kp));
  CUDA_TRY(sac_points_from_soa(src->d_kp_xyz.get(), src->n_kp, d_p.get()));   // exact: the doubles are widened floats
  CUDA_TRY(sac_points_from_soa(tgt->d_kp_xyz.get(), tgt->n_kp, d_q.get()));
  return sac_run(d_p.get(), src->d_fpfh.get(), src->n_kp, d_q.get(), tgt->d_fpfh.get(), tgt->n_kp, p, out, nullptr);
}
int ghicp_prep_sac_ia(const ghicp_prep *src, const ghicp_prep *tgt, const ghicp_sac_params *p, ghicp_sac_result *out) {
  if (!src || !tgt || !out || src->n_kp <= 0 || tgt->n_kp <= 0 || !src->d_fpfh.get() || !tgt->d_fpfh.get()) {
    set_error(nullptr, "prep_sac_ia: bad argument, a cloud without keypoints or without histograms (call ghicp_prep_fpfh first)");
    return GHICP_E_ARG;
  }
  if (src->device != tgt->device) { set_error(nullptr, "prep_sac_ia: the two pipeline results live on different devices"); return GHICP_E_ARG; }
  if (!sac_params_ok(p, "prep_sac_ia")) return GHICP_E_ARG;
  if (int rc = enter_device(src->device, "prep_sac_ia")) return rc;
  return cuda_status(prep_sac_ia_run(src, tgt, p, out), "prep_sac_ia");
}

// ---- overlap and fitness on the dense clouds ---------------------------------------------------------------------------
static bool finite_point(const float *p) { return std::isfinite(p[0]) && std::isfinite(p[1]) && std::isfinite(p[2]); }
// the finite points of xyz [n][3]: xyz itself when every point is finite, else a copy in *store
static const float *finite_points(const float *xyz, int n, std::vector<float> *store, int *n_out) {
  int j = 0;
  while (j < n && finite_point(xyz + 3 * (size_t)j)) ++j;
  *n_out = n;
  if (j == n) return xyz;
  store->reserve(3 * (size_t)n);
  for (int i = 0; i < n; ++i)
    if (finite_point(xyz + 3 * (size_t)i)) store->insert(store->end(), xyz + 3 * (size_t)i, xyz + 3 * (size_t)i + 3);
  *n_out = (int)(store->size() / 3);
  return store->data();
}
static bool overlap_args_ok(float thre_dis, double max_range, const char *who) {
  // thre_dis * thre_dis is compared in float32: a radius whose square is 0 or infinite is refused with the others
  const bool ok = std::isfinite(thre_dis) && thre_dis > 0.f && thre_dis * thre_dis > 0.f && std::isfinite(thre_dis * thre_dis) &&
                  max_range >= 0.0;   // false for NaN; +inf allowed (PCL's default)
  if (!ok) set_error(nullptr, std::string(who) + ": thre_dis must be positive and finite, max_range >= 0 (+inf allowed)");
  return ok;
}
static bool overlap_rt_ok(const double *Rt, const char *who) {
  if (Rt)
    for (int i = 0; i < 16; ++i)
      if (!std::isfinite(Rt[i])) { set_error(nullptr, std::string(who) + ": non-finite transform"); return false; }
  return true;
}

// Both overlap entries write *out (and d2) only once every stage succeeded.
static cudaError_t cloud_overlap_run(const float *a_xyz, int n_a, const float *b_xyz, int n_b, const double *Rt, float thre_dis,
                                     double max_range, int want_fitness, ghicp_overlap_result *out, float *d2) {
  StageEvents<3> ev;
  DevBuf<float> d_a, d_b;
  ghicp_overlap_result r{};
  CUDA_TRY(ev.create());
  CUDA_TRY(d_a.alloc(3 * (size_t)n_a)); CUDA_TRY(d_b.alloc(3 * (size_t)n_b));
  CUDA_TRY(cudaMemcpyAsync(d_a.get(), a_xyz, 3 * (size_t)n_a * sizeof(float), cudaMemcpyHostToDevice, 0));
  CUDA_TRY(cudaMemcpyAsync(d_b.get(), b_xyz, 3 * (size_t)n_b * sizeof(float), cudaMemcpyHostToDevice, 0));
  CUDA_TRY(cudaEventRecord(ev[0], 0));
  OverlapTarget *t = nullptr;
  CUDA_TRY(overlap_target_build(d_b.get(), n_b, &t));
  const cudaError_t e = overlap_run(d_a.get(), n_a, t, Rt, thre_dis, max_range, want_fitness, ev[1], &r, d2);
  overlap_target_free(t);
  CUDA_TRY(e);
  CUDA_TRY(cudaEventRecord(ev[2], 0));
  CUDA_TRY(cudaStreamSynchronize(0));
  r.stage_ms[0] = ev.ms(0, 1); r.stage_ms[1] = ev.ms(1, 2); r.stage_ms[2] = ev.ms(0, 2);
  *out = r;
  return cudaSuccess;
}
int ghicp_cloud_overlap(int device, const float *a_xyz, int n_a, const float *b_xyz, int n_b, const double Rt[16],
                        float thre_dis, double max_range, int want_fitness, ghicp_overlap_result *out, float *d2) {
  if (!a_xyz || !b_xyz || !out || n_a <= 0 || n_b <= 0 || (d2 && !want_fitness)) {
    set_error(nullptr, "cloud_overlap: bad argument (null array, empty cloud, or d2 without want_fitness)");
    return GHICP_E_ARG;
  }
  if (!overlap_args_ok(thre_dis, max_range, "cloud_overlap") || !overlap_rt_ok(Rt, "cloud_overlap")) return GHICP_E_ARG;
  // B's non-finite points (the NaN returns of an organised scan) are left out of the grid, as PCL's KdTreeFLANN leaves them
  // out of its tree; they can be no one's nearest point
  std::vector<float> b_store;
  int nb_fin = 0;
  b_xyz = finite_points(b_xyz, n_b, &b_store, &nb_fin);
  if (nb_fin <= 0) { set_error(nullptr, "cloud_overlap: cloud B has no finite point"); return GHICP_E_ARG; }
  if (int rc = enter_device(device, "cloud_overlap")) return rc;
  return cuda_status(cloud_overlap_run(a_xyz, n_a, b_xyz, nb_fin, Rt, thre_dis, max_range, want_fitness, out, d2), "cloud_overlap");
}

static cudaError_t prep_overlap_run(const ghicp_prep *a, ghicp_prep *tb, const double *Rt, float thre_dis, double max_range,
                                    int want_fitness, ghicp_overlap_result *out) {
  StageEvents<3> ev;
  ghicp_overlap_result r{};
  CUDA_TRY(ev.create());
  CUDA_TRY(cudaEventRecord(ev[0], 0));
  std::lock_guard<std::mutex> lk(tb->ov_mu);   // held while the grid is read: a concurrent first call waits for the build
  const bool cached = tb->ov_target != nullptr;
  if (!cached) CUDA_TRY(overlap_target_build(tb->d_down.get(), tb->n_down, &tb->ov_target));
  CUDA_TRY(overlap_run(a->d_down.get(), a->n_down, tb->ov_target, Rt, thre_dis, max_range, want_fitness, ev[1], &r, nullptr));
  CUDA_TRY(cudaEventRecord(ev[2], 0));
  CUDA_TRY(cudaStreamSynchronize(0));
  if (!cached) r.stage_ms[0] = ev.ms(0, 1);
  r.stage_ms[1] = ev.ms(1, 2); r.stage_ms[2] = ev.ms(0, 2);
  *out = r;
  return cudaSuccess;
}
int ghicp_prep_overlap(const ghicp_prep *a, const ghicp_prep *b, const double Rt[16], float thre_dis, double max_range,
                       int want_fitness, ghicp_overlap_result *out) {
  if (!a || !b || !out || a->n_down <= 0 || b->n_down <= 0) { set_error(nullptr, "prep_overlap: bad argument or an empty cloud"); return GHICP_E_ARG; }
  if (a->device != b->device) { set_error(nullptr, "prep_overlap: the two pipeline results live on different devices"); return GHICP_E_ARG; }
  if (!overlap_args_ok(thre_dis, max_range, "prep_overlap") || !overlap_rt_ok(Rt, "prep_overlap")) return GHICP_E_ARG;
  if (int rc = enter_device(a->device, "prep_overlap")) return rc;
  ghicp_prep *tb = const_cast<ghicp_prep *>(b);   // the grid is a cache of the target's down-sampled cloud, not its state
  return cuda_status(prep_overlap_run(a, tb, Rt, thre_dis, max_range, want_fitness, out), "prep_overlap");
}

// ---- point-to-point, point-to-plane and Generalized ICP on the dense clouds ------------------------------------------------
static_assert(offsetof(ghicp_icp_params, rotation_epsilon) == 40 && sizeof(ghicp_icp_params) == 48,
              "ghicp_icp_params: rotation_epsilon took the place of reserved[2]; the layout must not move");
static bool icp_params_ok(const ghicp_icp_params *p, const double *guess, const char *who) {
  const bool ok = p && p->max_iterations >= 1 && p->trim_ratio >= 0.f && p->trim_ratio <= 1.f &&   // false for NaN
                  p->transformation_epsilon >= 0.0 && p->fitness_epsilon >= 0.0;
  if (!ok) {
    set_error(nullptr, std::string(who) + ": max_iterations must be >= 1, trim_ratio in [0, 1], the epsilons >= 0");
    return false;
  }
  const bool k_ok = p->normal_k >= 3 && p->normal_k <= 32;
  if (p->metric != 0 && !(p->metric == 1 && k_ok) &&
      !(p->metric == 2 && k_ok && p->rotation_epsilon > 0.0 && p->rotation_epsilon <= DBL_MAX)) {   // false for NaN
    set_error(nullptr, std::string(who) + ": metric must be 0 (point-to-point), 1 (point-to-plane, with normal_k in 3..32) or 2 "
                                          "(GICP, with normal_k in 3..32 and a finite rotation_epsilon > 0)");
    return false;
  }
  return overlap_rt_ok(guess, who);
}
// the status of a finished ICP call: its warning bit, if any
static int icp_warnings(const ghicp_icp_result *r) {
  return r->state == GHICP_ICP_NO_CORRESPONDENCES ? GHICP_W_FEW_PAIRS : (r->state == GHICP_ICP_SINGULAR ? GHICP_W_SINGULAR : GHICP_OK);
}

// Both ICP entries write *out, moved and the traces only once every stage succeeded.
static cudaError_t cloud_icp_run(const float *src, int n_s, const float *src_fin, int ns_fin, const float *tgt, int n_t,
                                 const double *guess, const ghicp_icp_params *p, ghicp_icp_result *out, float *moved, int *cor_trace,
                                 double *mse_trace) {
  StageEvents<4> ev;
  DevBuf<float> d_all, d_fin, d_t, d_nrm, d_nrm_s;
  ghicp_icp_result r{};
  CUDA_TRY(ev.create());
  CUDA_TRY(d_all.alloc(3 * (size_t)n_s)); CUDA_TRY(d_t.alloc(3 * (size_t)n_t));
  if (src_fin != src) CUDA_TRY(d_fin.alloc(3 * (size_t)ns_fin));
  if (p->metric != 0) CUDA_TRY(d_nrm.alloc(3 * (size_t)n_t));
  if (p->metric == 2) CUDA_TRY(d_nrm_s.alloc(3 * (size_t)ns_fin));
  CUDA_TRY(cudaMemcpyAsync(d_all.get(), src, 3 * (size_t)n_s * sizeof(float), cudaMemcpyHostToDevice, 0));
  if (src_fin != src) CUDA_TRY(cudaMemcpyAsync(d_fin.get(), src_fin, 3 * (size_t)ns_fin * sizeof(float), cudaMemcpyHostToDevice, 0));
  CUDA_TRY(cudaMemcpyAsync(d_t.get(), tgt, 3 * (size_t)n_t * sizeof(float), cudaMemcpyHostToDevice, 0));
  CUDA_TRY(cudaEventRecord(ev[0], 0));
  OverlapTarget *t = nullptr;
  CUDA_TRY(overlap_target_build(d_t.get(), n_t, &t));
  std::vector<int> cor(cor_trace ? p->max_iterations : 0);
  std::vector<double> mse(mse_trace ? p->max_iterations : 0);
  const float *d_src = src_fin != src ? d_fin.get() : d_all.get();
  cudaError_t e = p->metric != 0 ? prep_knn_normals(0, d_t.get(), n_t, p->normal_k, d_nrm.get()) : cudaSuccess;
  if (e == cudaSuccess && p->metric == 2) e = prep_knn_normals(0, d_src, ns_fin, p->normal_k, d_nrm_s.get());
  if (e == cudaSuccess)
    e = icp_run(d_src, ns_fin, d_all.get(), n_s, t, d_t.get(), d_nrm.get(), d_nrm_s.get(), guess, p, ev[1], ev[2], &r, moved,
                cor_trace ? cor.data() : nullptr, mse_trace ? mse.data() : nullptr);
  overlap_target_free(t);
  CUDA_TRY(e);
  CUDA_TRY(cudaEventRecord(ev[3], 0));
  CUDA_TRY(cudaStreamSynchronize(0));
  r.stage_ms[0] = ev.ms(0, 1); r.stage_ms[1] = ev.ms(1, 2); r.stage_ms[2] = ev.ms(2, 3); r.stage_ms[3] = ev.ms(0, 3);
  *out = r;
  if (cor_trace) std::copy(cor.begin(), cor.begin() + r.iterations, cor_trace);
  if (mse_trace) std::copy(mse.begin(), mse.begin() + r.iterations, mse_trace);
  return cudaSuccess;
}
int ghicp_cloud_icp(int device, const float *src_xyz, int n_s, const float *tgt_xyz, int n_t, const double guess[16],
                    const ghicp_icp_params *p, ghicp_icp_result *out, float *moved, int *cor_trace, double *mse_trace) {
  if (!src_xyz || !tgt_xyz || !out || n_s <= 0 || n_t <= 0) {
    set_error(nullptr, "cloud_icp: bad argument (null array or empty cloud)");
    return GHICP_E_ARG;
  }
  if (!icp_params_ok(p, guess, "cloud_icp")) return GHICP_E_ARG;
  // non-finite points take no part (PCL's KdTreeFLANN leaves them out of its tree; their moved copies find no neighbour)
  std::vector<float> s_store, t_store;
  int ns_fin = 0, nt_fin = 0;
  const float *s_fin = finite_points(src_xyz, n_s, &s_store, &ns_fin);
  const float *t_fin = finite_points(tgt_xyz, n_t, &t_store, &nt_fin);
  if (ns_fin <= 0 || nt_fin <= 0) { set_error(nullptr, "cloud_icp: the source or the target has no finite point"); return GHICP_E_ARG; }
  if (int rc = enter_device(device, "cloud_icp")) return rc;
  if (int rc = cuda_status(cloud_icp_run(src_xyz, n_s, s_fin, ns_fin, t_fin, nt_fin, guess, p, out, moved, cor_trace, mse_trace),
                           "cloud_icp"))
    return rc;
  return icp_warnings(out);
}

// a pipeline result's k-NN normals for k, kept on it (the caller holds its ov_mu); *built = false when they were already
// there.  New normals go into a fresh buffer: the cache changes only once they exist.
static cudaError_t prep_icp_normals(ghicp_prep *h, int k, bool *built) {
  *built = h->icp_nrm_k != k;
  if (!*built) return cudaSuccess;
  DevBuf<float> nrm;
  CUDA_TRY(nrm.alloc(3 * (size_t)h->n_down));
  CUDA_TRY(prep_knn_normals(0, h->d_down.get(), h->n_down, k, nrm.get()));
  h->icp_nrm = std::move(nrm);
  h->icp_nrm_k = k;
  return cudaSuccess;
}

// the caches and the loop, under the locks prep_icp_run holds; *cached: the grid and every normal needed were there
static cudaError_t prep_icp_locked(ghicp_prep *sb, ghicp_prep *tb, const double *guess, const ghicp_icp_params *p,
                                   StageEvents<4> &ev, ghicp_icp_result *r, bool *cached) {
  bool built = false;
  *cached = tb->ov_target != nullptr;
  if (!*cached) CUDA_TRY(overlap_target_build(tb->d_down.get(), tb->n_down, &tb->ov_target));
  if (p->metric != 0) { CUDA_TRY(prep_icp_normals(tb, p->normal_k, &built)); *cached = *cached && !built; }
  if (p->metric == 2) { CUDA_TRY(prep_icp_normals(sb, p->normal_k, &built)); *cached = *cached && !built; }
  return icp_run(sb->d_down.get(), sb->n_down, sb->d_down.get(), sb->n_down, tb->ov_target, tb->d_down.get(), tb->icp_nrm.get(),
                 sb->icp_nrm.get(), guess, p, ev[1], ev[2], r, nullptr, nullptr, nullptr);
}

static cudaError_t prep_icp_run(ghicp_prep *sb, ghicp_prep *tb, const double *guess, const ghicp_icp_params *p,
                                ghicp_icp_result *out) {
  StageEvents<4> ev;
  ghicp_icp_result r{};
  CUDA_TRY(ev.create());
  CUDA_TRY(cudaEventRecord(ev[0], 0));
  // the grid ghicp_prep_overlap keeps, and the normals, under the target's lock; GICP also keeps the source's normals, under
  // both locks taken together (std::scoped_lock avoids the deadlock of (a, b) and (b, a) at once; one lock when a == b)
  bool cached = false;
  if (p->metric == 2 && sb != tb) {
    std::scoped_lock lk(tb->ov_mu, sb->ov_mu);
    CUDA_TRY(prep_icp_locked(sb, tb, guess, p, ev, &r, &cached));
  } else {
    std::scoped_lock lk(tb->ov_mu);
    CUDA_TRY(prep_icp_locked(sb, tb, guess, p, ev, &r, &cached));
  }
  CUDA_TRY(cudaEventRecord(ev[3], 0));
  CUDA_TRY(cudaStreamSynchronize(0));
  if (!cached) r.stage_ms[0] = ev.ms(0, 1);
  r.stage_ms[1] = ev.ms(1, 2); r.stage_ms[2] = ev.ms(2, 3); r.stage_ms[3] = ev.ms(0, 3);
  *out = r;
  return cudaSuccess;
}
int ghicp_prep_icp(const ghicp_prep *source, const ghicp_prep *target, const double guess[16], const ghicp_icp_params *p,
                   ghicp_icp_result *out) {
  if (!source || !target || !out || source->n_down <= 0 || target->n_down <= 0) {
    set_error(nullptr, "prep_icp: bad argument or an empty cloud");
    return GHICP_E_ARG;
  }
  if (source->device != target->device) { set_error(nullptr, "prep_icp: the two pipeline results live on different devices"); return GHICP_E_ARG; }
  if (!icp_params_ok(p, guess, "prep_icp")) return GHICP_E_ARG;
  if (int rc = enter_device(source->device, "prep_icp")) return rc;
  // the grid and the normals are caches of the down-sampled clouds, not the results' state
  ghicp_prep *sb = const_cast<ghicp_prep *>(source), *tb = const_cast<ghicp_prep *>(target);
  if (int rc = cuda_status(prep_icp_run(sb, tb, guess, p, out), "prep_icp")) return rc;
  return icp_warnings(out);
}

int ghicp_set_initial_transform(ghicp_ctx *ctx, const double Rt[16]) {
  Ctx *c = reinterpret_cast<Ctx *>(ctx);
  if (!c || !Rt) { set_error(c, "set_initial_transform: bad argument"); return GHICP_E_ARG; }
  if (c->N <= 0) { set_error(c, "set_initial_transform: keypoints not set"); return GHICP_E_ARG; }
  if (c->iteration != 0) { set_error(c, "set_initial_transform: only before iteration 0 (after ghicp_reset, re-upload the source first)"); return GHICP_E_ARG; }
  for (int i = 0; i < 16; ++i)
    if (!std::isfinite(Rt[i])) { set_error(c, "set_initial_transform: non-finite matrix"); return GHICP_E_ARG; }
  int rc;
  if ((rc = use_device(c))) return rc;
  // the update of every iteration (k_apply) with this transform
  CK(c, cudaMemcpyAsync(c->d_iter->Rt, Rt, sizeof(double) * 16, cudaMemcpyHostToDevice, c->stream));
  CK(c, launch_apply(c, false));
  CK(c, cudaStreamSynchronize(c->stream));
  double acc[16];   // Rt_tillnow = Rt * Rt_tillnow, as after an iteration
  for (int col = 0; col < 4; ++col)
    for (int row = 0; row < 4; ++row) {
      double s = 0;
      for (int k = 0; k < 4; ++k) s += Rt[k * 4 + row] * c->Rt_tillnow[col * 4 + k];
      acc[col * 4 + row] = s;
    }
  std::memcpy(c->Rt_tillnow, acc, sizeof(acc));
  return GHICP_OK;
}

// The sampling pattern of the grid-pair comparisons for voxel_side_num = 7: what the reference's BSCEncoder constructor
// generates with build_sample_pattern = true (include/binary_feature_extraction.hpp:75-103) in a process that has not called
// srand — glibc's rand() sequence for seed 1 — i.e. the sample_pattern.txt a user of the reference produces; the reference
// itself ships none.  Generated by tests/golden/make_bsc_golden.py through the reference's own constructor.
static const int kBscPattern7[49][2] = {
    {15, 39}, {37, 5}, {29, 10}, {24, 23}, {8, 17}, {9, 47}, {6, 18},
    {20, 21}, {17, 22}, {3, 21}, {30, 47}, {33, 48}, {29, 5}, {5, 0},
    {45, 47}, {10, 30}, {8, 35}, {9, 16}, {8, 18}, {19, 14}, {41, 45},
    {41, 9}, {23, 15}, {38, 26}, {42, 43}, {46, 4}, {22, 31}, {9, 27},
    {32, 5}, {31, 47}, {40, 39}, {38, 0}, {12, 3}, {23, 31}, {17, 16},
    {32, 14}, {30, 7}, {35, 24}, {33, 28}, {18, 4}, {7, 16}, {8, 29},
    {47, 18}, {12, 35}, {28, 43}, {39, 20}, {39, 28}, {25, 7}, {31, 0},
};
int ghicp_bsc_default_pattern(int voxel_side_num, int *pairs) {
  if (!pairs || voxel_side_num != 7) { set_error(nullptr, "bsc_default_pattern: only voxel_side_num = 7 has a shipped pattern"); return GHICP_E_ARG; }
  for (int i = 0; i < 49; ++i) { pairs[2 * i] = kBscPattern7[i][0]; pairs[2 * i + 1] = kBscPattern7[i][1]; }
  return GHICP_OK;
}

int ghicp_comm_unique_id(void *id128) {
  if (!id128) return GHICP_E_ARG;
  return comm_unique_id(id128);
}
int ghicp_comm_init(ghicp_ctx *ctx, const void *id128, int rank, int world) {
  Ctx *c = reinterpret_cast<Ctx *>(ctx);
  if (!c || (!id128 && world > 1)) return GHICP_E_ARG;
  int rc;
  if ((rc = use_device(c))) return rc;
  return comm_init(c, id128, rank, world);
}

}  // extern "C"
