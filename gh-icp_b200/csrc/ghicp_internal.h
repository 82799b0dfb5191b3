// ghicp_internal.h — internal declarations shared by the translation units of libghicp_b200.so.
// Not part of the ABI (the ABI is include/ghicp_b200.h).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <string>
#include <vector>

#include "../../include/ghicp_b200.h"

// Kernel launch: the <<< >>> syntax under nvcc.  The kernel-LOGIC harness (tests/harness, g++ -DGHICP_EMU_HOST with the
// host emulation shim of tests/harness/cuda_emu) compiles a few .cu files as plain C++ and runs every CUDA thread as a
// fiber on the CPU; those files launch through this macro.  The product is always built by nvcc.
#if defined(GHICP_EMU_HOST)
#define GHICP_LAUNCH(kernel, grid, block, smem, stream, ...) emu::launch((grid), (block), [&] { kernel(__VA_ARGS__); }, (smem))
#define GHICP_NOINLINE __attribute__((noinline))
#else
#define GHICP_NOINLINE __noinline__
#define GHICP_LAUNCH(kernel, grid, block, smem, stream, ...) kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
#endif

namespace ghicp_b200 {

// SM count of the H100 SXM the fixed grid-stride launch geometries are sized for (a multiple of it keeps every SM busy);
// launches that must match the device query cudaDevAttrMultiProcessorCount instead.
constexpr int GHICP_SMS = 132;

// ---- host plumbing of the stages around the loop: temporary device memory, events, early return on error ----------------
// Return the error of a cudaError_t call from the enclosing function (which returns cudaError_t); the DevBufs in scope free
// their arrays on the way out.
#define CUDA_TRY(call)                                      \
  do {                                                      \
    const cudaError_t e__ = (call);                         \
    if (e__ != cudaSuccess) return e__;                     \
  } while (0)

// The pool keeps what it has handed out once (release threshold = unlimited), so the second scan of a pair allocates
// nothing new.  Set once per process, for the device current at the first DevBuf allocation.
inline void pool_init() {
#if !defined(GHICP_EMU_HOST)
  static const bool done = [] {
    int dev = 0;
    cudaMemPool_t pool;
    if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
      unsigned long long thr = ~0ull;
      cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
    }
    return true;
  }();
  (void)done;
#endif
}

// A temporary device array from the device's stream-ordered pool, freed (stream-ordered, on the stream it was allocated on)
// when it goes out of scope or at reset().  A cudaMalloc / cudaFree pair per temporary costs more host time than all the
// kernels of a 1 M-point scan together, cudaFree being a device-wide synchronisation.  Move-only.
template <typename T>
class DevBuf {
 public:
  DevBuf() = default;
  DevBuf(const DevBuf &) = delete;
  DevBuf &operator=(const DevBuf &) = delete;
  DevBuf(DevBuf &&o) noexcept : p_(o.p_), st_(o.st_) { o.p_ = nullptr; }
  DevBuf &operator=(DevBuf &&o) noexcept {
    if (this != &o) { reset(); p_ = o.p_; st_ = o.st_; o.p_ = nullptr; }
    return *this;
  }
  ~DevBuf() { reset(); }

  // n elements (one when n = 0, so that an empty array still has an address); frees what the buffer held first
  cudaError_t alloc(size_t n, cudaStream_t st = 0) {
    reset();
    pool_init();
    st_ = st;
    const cudaError_t e = cudaMallocAsync((void **)&p_, (n ? n : 1) * sizeof(T), st);
    if (e != cudaSuccess) p_ = nullptr;
    return e;
  }
  T *get() const { return p_; }
  void reset() {
    if (p_) cudaFreeAsync(p_, st_);
    p_ = nullptr;
  }

 private:
  T *p_ = nullptr;
  cudaStream_t st_ = 0;
};

// The events that time the stages of one call, destroyed with it
template <int N>
struct StageEvents {
  cudaEvent_t ev[N] = {};
  StageEvents() = default;
  StageEvents(const StageEvents &) = delete;
  StageEvents &operator=(const StageEvents &) = delete;
  ~StageEvents() {
    for (cudaEvent_t e : ev)
      if (e) cudaEventDestroy(e);
  }
  cudaError_t create() {
    for (cudaEvent_t &e : ev) CUDA_TRY(cudaEventCreate(&e));
    return cudaSuccess;
  }
  cudaEvent_t operator[](int i) const { return ev[i]; }
  float ms(int from, int to) const {   // elapsed time between two recorded events
    float t = 0.f;
    cudaEventElapsedTime(&t, ev[from], ev[to]);
    return t;
  }
};

// Feature-distance plane layout: PANEL-MAJOR.  The N x M plane is stored as ceil(M/256) column panels, each
// a dense row-major [rows][256] block, so the 256-column panel a warp sweeps down the source rows is one
// perfectly sequential HBM stream instead of short reads at a row stride.  fd_index / fd_elems address the
// float FPFH plane in this order.
constexpr int FD_PANEL = 256;
__host__ __device__ inline size_t fd_index(size_t rows, int i, int j) {
  return ((size_t)(j >> 8) * rows + (size_t)i) * FD_PANEL + (size_t)(j & (FD_PANEL - 1));
}
__host__ __device__ inline size_t fd_elems(size_t rows, int M) { return (size_t)((M + FD_PANEL - 1) / FD_PANEL) * rows * FD_PANEL; }

// The BSC plane holds integer Hamming distances 0 ... bits (<= 2048), PACKED exactly into 8 + hb bits per value:
//   hb = 1 for bits <= 511, 2 for bits <= 1023, 4 up to 2048 (fd_hb).
// Panels as above; inside a panel the rows are grouped in QUADS (4 rows: one k_stream TMA stage).  A quad block is
//   [4][256] low bytes (row-major)  |  [hb][32] 32-bit words of high bits (word h of lane l at h * 32 + l)
// where "lane" l = column / 8 of the panel: a lane's 8 columns x 4 rows are 16 column PAIRS k = 4 * row + column / 2, and
// the high bits of pair k, value e (= column & 1) sit in word k / (16 / hb) at bit hb * (k % (16 / hb)) + 16 e.  Shifting
// a word so that a pair lands on bits 8 and 24 puts both high parts right above their low bytes (k_stream's decode).
// Rows are padded to whole quads and columns to whole panels; padding holds zeros.
constexpr int FD_QUAD = 4;
constexpr int FD_LOW_BYTES = FD_QUAD * FD_PANEL;   // 1024
__host__ __device__ inline int fd_hb(int bits) { return bits <= 511 ? 1 : bits <= 1023 ? 2 : 4; }
__host__ __device__ inline size_t fd_block_bytes(int hb) { return (size_t)FD_LOW_BYTES + 128 * (size_t)hb; }   // 1152 / 1280 / 1536
__host__ __device__ inline size_t fd_quads(size_t rows) { return (rows + FD_QUAD - 1) / FD_QUAD; }
__host__ __device__ inline size_t fd_plane_bytes(size_t rows, int M, int hb) {
  return (size_t)((M + FD_PANEL - 1) / FD_PANEL) * fd_quads(rows) * fd_block_bytes(hb);
}
// byte offset of the quad block holding rows 4 (i / 4) ... of the panel of column j
__host__ __device__ inline size_t fd_block_offset(size_t rows, int hb, int i, int j) {
  return ((size_t)(j >> 8) * fd_quads(rows) + (size_t)(i >> 2)) * fd_block_bytes(hb);
}
// high-bit word (0 ... hb-1) and bit position of value (u, c): row u of the quad, column c of the lane
// (pair k = 4u + c/2 in word k / (16/hb) at hb * (k mod 16/hb); hb = 1, 2, 4 -> log2(hb) = hb >> 1, shifts instead of divisions)
__host__ __device__ inline int fd_hi_word(int hb, int u, int c) { return (4 * u + (c >> 1)) >> (4 - (hb >> 1)); }
__host__ __device__ inline int fd_hi_bit(int hb, int u, int c) {
  return hb * ((4 * u + (c >> 1)) & ((16 >> (hb >> 1)) - 1)) + 16 * (c & 1);
}
// exact decode of FD(i, j), i relative to the plane's first row
__host__ __device__ inline unsigned fd_at(const void *plane, size_t rows, int hb, int i, int j) {
  const unsigned char *blk = static_cast<const unsigned char *>(plane) + fd_block_offset(rows, hb, i, j);
  const int u = i & 3, col = j & (FD_PANEL - 1), c = col & 7;
  const unsigned hi = reinterpret_cast<const unsigned *>(blk + FD_LOW_BYTES)[fd_hi_word(hb, u, c) * 32 + (col >> 3)];
  return (unsigned)blk[u * FD_PANEL + col] | (((hi >> fd_hi_bit(hb, u, c)) & ((1u << hb) - 1u)) << 8);
}
// OR of v over aligned groups of WIDTH lanes (the encoders' high-bit words); every lane of the warp must take part
template <int WIDTH>
__device__ __forceinline__ unsigned fd_lanes_or(unsigned v) {
#if !defined(GHICP_EMU_HOST)
  if (WIDTH == 32) return __reduce_or_sync(0xffffffffu, v);
#endif
#pragma unroll
  for (int o = 1; o < WIDTH; o <<= 1) v |= __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// encoder side: value v's contribution to its high-bit word (the words of a quad and lane are the OR over its 32 values)
__host__ __device__ inline unsigned fd_hi_part(int hb, int u, int c, unsigned v) { return (v >> 8) << fd_hi_bit(hb, u, c); }

// ---- small device-side structs -----------------------------------------------------------------
// Parameters of one cost evaluation CD(i,j) (src/ghicp_reg.cpp:122, 224, 259, 308).
struct CostParams {
  double scale;    // (double)Energyfunction::scale
  double WED, WFD; // BSC weights (src/ghicp_reg.cpp:247-249)
  double ex;       // FPFH exponent 1/(it+1) (src/ghicp_reg.cpp:308)
  double pivot;    // shift used for the one-pass variance accumulation
};

// Host-owned loop scalars passed to the device penalty rule (src/ghicp_reg.cpp:230-239, 279-287, 327-335).
struct LoopScalars {
  int iteration;
  double RMS, FDM, FDstd, para1, para2;
  double scale, WED, WFD, penalty_initial;
};

// Scalars produced on the device by one iteration and read back once at its end.
struct DevIter {
  double cd_sum_shift, cd_sumsq_shift;  // sums of (cd - pivot), (cd - pivot)^2
  double cd_mean, cd_std, penalty;
  int cor;
  int overflow_any;     // some rank's candidate buffer overflowed (streaming path)
  double rmse, fdm, fdstd, rmse_after;
  double km_cd_sum;     // sum of CD over kept pairs
  double Rt[16];        // column-major
  long long nnz;
  int solve_degenerate; // cor < 3: identity returned
  int ambiguous;        // NN gate decisions within the fast-statistics error band of the penalty
};

// ---- streaming (fast) path ----------------------------------------------------------------------
struct Cand {  // a pair the FP32 filter could not rule out, with its exactly evaluated CD
  int i, j;
  double cd;
};
struct StreamDev {  // device-resident scalars of the streaming path
  unsigned r2max_bits;   // max squared centred norm of any keypoint (float bits)
  float margin;          // bound on |cd32 - cd64|
  float thr_hi;          // KM superset gate
  int cand_count[2];     // row / column candidates (saturating: at most cand_cap + resident threads)
  int overflow;          // some candidate did not fit below cand_cap
  unsigned long long nnz_valid;
  unsigned long long emit_count;  // KM: gate hits appended to the edge list by the count pass (may exceed its capacity)
  int out_of_range;      // A * R^2 outside the window of k_margin's error bound (stream_in_window): all-double route
};
// Where the FP32 filter of ghicp_stream.cu keeps every operand and partial sum of d2' = A*|s - t|^2 a normal float (A = the
// squared ED weight, R2 = the largest squared centred norm): A*R2 in [2^-80, 2^120] (the sums stay below 4*A*R2, the
// rounding error 2^-150 of a subnormal and the flush of sqrt.approx.ftz stay far below the margin), |T.xyz| = 2*A*|t| below
// 2^120, and R2 in [2^-100, 2^100] for the coordinates themselves.  A = 0 (BSC iteration 0: no ED term) is always inside.
// About 10^-5 ... 10^10 units of cloud extent for the usual bbx_magnitude weight (bbx_magnitude ~ 3x the extent).
constexpr double STREAM_WINDOW_LO = 0x1p-80, STREAM_WINDOW_HI = 0x1p120;
__host__ __device__ inline bool stream_in_window(double A, double R2) {
  if (!(R2 >= 0x1p-100 && R2 <= 0x1p100)) return false;
  if (A == 0.0) return true;
  const double P = A * R2;
  return P >= STREAM_WINDOW_LO && P <= STREAM_WINDOW_HI && 4.0 * A * A * R2 <= 0x1p240;
}

struct StreamArgs {
  const unsigned char *fd;   // packed BSC FD plane (fd_at) or nullptr (no feature)
  size_t fd_rows;            // rows of the plane held by this context
  int fd_hb;                 // high bits per value of the plane (fd_hb)
  int N, M;
  int row0, nloc;            // source rows [row0, row0 + nloc) streamed by this context
  int rb;                    // source rows per CTA of this launch (<= ST_RB, a multiple of the batch)
  const float4 *S4, *T4;
  const double *s, *t;
  double scale, WED, WFD;
  float b;               // feature weight in the filter's (kappa-scaled) domain (an fp16 value when x2_ok)
  double kappa;          // scale of the filter domain relative to CD
  StreamDev *dev;
  unsigned *row_thr_init; unsigned long long *rowbest; int *rowidx;
  unsigned *col_thr_init; unsigned long long *colbest; int *colidx;
  Cand *cand[2]; int cand_cap;
  double *part_stats;
  int *cnt; const long long *rowptr; int *cursor; int *csr_col;
  float *row_fd;   // FD of (row, its partner)
  float *csr_fd;   // FD of every CSR entry
  unsigned long long *emit; unsigned long long emit_cap;  // KM edge list: (row << 32 | col) per gate hit
};

// header of the per-rank candidate block of a settled KM iteration (ghicp_stream.cu: k_emit_check)
struct XBlockHdr {
  unsigned long long count;   // candidate edges that follow (0 when the rank overflowed: stats[2] = 1)
  double stats[4];            // the rank's partial CD sums (sum, sum of squares), overflow flag, spare
  unsigned long long pad[3];  // 64 bytes: the arrays behind it stay 16-byte aligned
};

// What the choice of an iteration's route (ghicp_capi.cu: choose_route) remembers of earlier iterations; part of the
// context (Ctx derives from it).  Reset when the keypoints change size and by ghicp_reset.
struct RouteHistory {
  bool have_prev = false;             // d_row_idx / d_col_idx hold last iteration's partners
  long long last_cands = 0;           // candidates the filter passed to exact evaluation last iteration
  long long last_local_nnz = -1;      // KM candidate edges in this context's rows last iteration (-1: no history)
  long long last_total_nnz = -1;      // candidate edges of the whole graph last iteration (-1: no history)
  long long last_max_local_nnz = -1;  // largest per-rank share of them
  bool km_settled_off = false;        // the last settled attempt overflowed: take the general route once
  void reset() { *this = RouteHistory(); }
};

// ---- the context ----------------------------------------------------------------------------------
struct Ctx : RouteHistory {
  ghicp_config cfg{};
  int device = 0;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  std::string err;

  int N = 0, M = 0;
  size_t fd_rows = 0;  // rows of the FD plane held by this context
  // coordinates, SoA doubles
  double *d_s = nullptr;  // [3][N]
  double *d_t = nullptr;  // [3][M]
  // BSC
  int V = 0, bits = 0, Bbytes = 0, W64 = 0;
  uint64_t *d_bs = nullptr;  // [V][W64][N]
  uint64_t *d_bt = nullptr;  // [W64][M]
  uint16_t *d_fd16 = nullptr;  // packed FD plane, fd_plane_bytes(fd_rows, M, fd_hb(bits)) bytes (allocated in 16-bit units)
  // FPFH
  float *d_fs = nullptr, *d_ft = nullptr;  // raw [N][33], [M][33]
  float *d_fdf = nullptr;                  // stored float FD plane, panel-major (fd_index)
  // matrix-free FPFH (ghicp_fpfh.cu): centred histograms, row-major [n][36] and transposed [36][n]; no N x M array
  bool fpfh_mf = false;
  float *d_fsc = nullptr, *d_fscT = nullptr, *d_ftc = nullptr, *d_ftcT = nullptr;
  // FPFH fast path (FP32 filter + exact refinement): source records [N][40], normalised target histograms [36][M],
  // split target coordinates [6][M], per-CTA CD sums, PRE-pass guesses
  bool fpfh_fast_ready = false;
  float *d_ff_srec = nullptr, *d_ff_tnT = nullptr, *d_ff_tco = nullptr;
  double *d_ff_part = nullptr;
  unsigned long long *d_ff_rowguess = nullptr, *d_ff_colguess = nullptr;
  // opt-in solvers (ghicp_solvers.cu)
  double *d_tn = nullptr;  // target normals [3][M]
  bool have_normals = false;
  bool have_bsc = false, have_fpfh = false, fd_built = false;

  // per-iteration workspaces
  int n_chunks = 1;
  double *d_part_cd = nullptr;   // [N][n_chunks]
  int *d_part_idx = nullptr;     // [N][n_chunks]
  double *d_part_stats = nullptr;  // [grid][2]
  size_t part_stats_cap = 0;
  double *d_row_cd = nullptr;  // [N]
  int *d_row_idx = nullptr;    // [N]
  double *d_col_cd = nullptr;  // [M]
  int *d_col_idx = nullptr;    // [M]
  int *d_flags = nullptr;      // [max(N,M)]
  int *d_sp = nullptr, *d_tp = nullptr;  // [max(N,M)]
  DevIter *d_iter = nullptr;
  DevIter *h_iter = nullptr;  // pinned
  double *h_stage = nullptr;  // pinned staging for coordinates
  size_t h_stage_cap = 0;

  // KM
  int *d_cnt = nullptr;          // [N*n_chunks + 1]
  long long *d_rowptr = nullptr; // [N*n_chunks + 1]
  int *d_cursor = nullptr;       // [N*n_chunks]
  int *d_csr_col = nullptr; double *d_csr_gain = nullptr; size_t csr_cap = 0;
  long long *d_colptr = nullptr; // [M+1]
  int *d_colcnt = nullptr;       // [M+1]
  int *d_csc_row = nullptr; double *d_csc_gain = nullptr; size_t csc_cap = 0;
  // auction state
  double *d_price = nullptr;   // [M]
  double *d_profit = nullptr;  // [N]
  int *d_assign = nullptr;     // [N] person -> object (-1 unassigned, -2 dummy)
  int *d_owner = nullptr;      // [M] object -> person (-1 none)
  unsigned long long *d_bidmax = nullptr;  // [max(N,M)]
  int *d_bidwin = nullptr;     // [max(N,M)]
  int *d_bid_obj = nullptr; double *d_bid_val = nullptr;  // [max(N,M)]
  double *d_bid_aux = nullptr; // [max(N,M)]
  int *d_list[2] = {nullptr, nullptr};  // active lists [max(N,M)]
  int *d_counters = nullptr;   // [64] (layout: ghicp_auction.cu)
  int *h_counters = nullptr;   // pinned [64]

  // streaming path
  bool use_fast = true;
  bool x2_ok = true;         // column-pair FP32 variant usable this iteration (feature weight exact in fp16)
  double kappa = 1.0;
  float b_eff = 0.f;
  double center[3] = {0, 0, 0};
  float *d_S4 = nullptr, *d_T4 = nullptr;   // float4[N], float4[M]
  StreamDev *d_sdev = nullptr;
  StreamDev *h_sdev = nullptr;              // pinned
  unsigned *d_row_thr = nullptr, *d_col_thr = nullptr;
  unsigned long long *d_rowbest = nullptr, *d_colbest = nullptr;
  int *d_rowidx2 = nullptr, *d_colidx2 = nullptr;
  Cand *d_cand[2] = {nullptr, nullptr};
  int cand_cap = 0;
  long long *d_tile_sum = nullptr;          // per-tile sums of the tiled scan / selection kernels
  size_t tile_cap = 0;
  double *d_solve_part = nullptr;           // per-CTA partial sums of the cooperative solve kernel
  unsigned long long *d_emit = nullptr;     // KM edge list of the count pass
  size_t emit_cap = 0;
  bool emit_on = false;                     // this iteration's count pass appends to the list

  // host loop state (include/ghicp_reg.h:173-202)
  int iteration = 0;
  double RMS = 99999, FDM = 0, FDstd = 0, IoU = 0;
  double para1 = 1.0, para2 = 1.0, penalty_initial = 2.0;
  int min_cor = 10, weight_changing_rate = 6;
  double KM_eps = 0.01;
  float scale_f = 0.f;
  bool converge = false;
  double Rt_tillnow[16];
  double last_mean = 0.0;
  int launches = 0;
  int last_cor = 0;

  // multi-GPU: source rows [r0, r0 + nloc) live here; target replicated; one exchange per iteration
  void *nccl_comm = nullptr;
  int rank = 0, world = 1;
  int r0 = 0, nloc = 0, shard = 0, Npad = 0;
  float *d_row_fd = nullptr;    // [Npad]
  float *d_pair_fd = nullptr;   // [max(N,M)]
  float *d_csr_fd = nullptr;    // [csr_cap]
  double *d_xstats = nullptr;   // [world][2] partial CD sums
  unsigned long long *d_colg_cd = nullptr;  // [world][M] gathered column minima (ordered-double bits)
  int *d_colg_idx = nullptr;                // [world][M]
  long long *h_rowptr_cut = nullptr;        // pinned [world + 1] CSR offsets at the shard boundaries
  // settled KM iteration: one candidate block per rank, one all-gather, no host round trip inside the iteration
  size_t xcap = 0;                          // candidate edges a block can carry (allocation)
  size_t xuse = 0;                          // ... and carries this iteration: 2 x last iteration's largest share (same on every rank)
  unsigned char *d_xsend = nullptr;         // this rank's block
  unsigned char *d_xrecv = nullptr;         // [world] blocks (world > 1)
  unsigned long long *d_xcounts = nullptr;  // [world] edges per block (device)
  unsigned long long *h_xcounts = nullptr;  // pinned copy
};

struct KmResult {
  int rounds = 0, phases = 0;
};

// ---- modes the orchestration passes to the launchers --------------------------------------------------
// launch_stream (k_stream's MODE): NN / NNR filter pass, KM count / fill pass, FP32 seed pre-pass (rows / rows + columns)
enum StreamMode { SM_NN = 0, SM_NNR = 1, SM_COUNT = 2, SM_FILL = 3, SM_PRE = 4, SM_PRE_COLS = 5 };
// launch_rowsweep / launch_rowsweep_mf (mode, an int holding one of these): row minima + CD statistics, KM candidate count
// (needs the penalty in d_iter), KM fill
enum SweepMode { SWEEP_ROWMIN = 0, SWEEP_COUNT = 1, SWEEP_FILL = 2 };
// comm_exchange: what the grouped all-gather carries (OR of the bits)
enum ExchangeBits { EX_STATS = 1, EX_ROWS = 2, EX_COLS = 4 };

// ---- launchers (ghicp_kernels.cu) ---------------------------------------------------------------
cudaError_t launch_pack_bsc(Ctx *c, const uint8_t *d_raw_s, const uint8_t *d_raw_t);
cudaError_t launch_fd_bsc(Ctx *c);
cudaError_t launch_fd_bsc_tc(Ctx *c);  // wgmma path; cudaErrorNotSupported when the shape does not fit
cudaError_t launch_fd_fpfh(Ctx *c);
cudaError_t launch_rowsweep(Ctx *c, int mode, const CostParams &cp);
cudaError_t launch_colsweep(Ctx *c, const CostParams &cp);
cudaError_t launch_finalize_stats(Ctx *c, const CostParams &cp, const LoopScalars &ls);
cudaError_t launch_select_nn(Ctx *c, double amb_rel = 0.0);    // flags from row minima + penalty, compaction → d_sp/d_tp, cor
cudaError_t launch_select_nnr(Ctx *c);
cudaError_t launch_select_km(Ctx *c);    // from d_owner
cudaError_t launch_solve(Ctx *c, const CostParams &cp);  // stats + umeyama + rmse_after → d_iter
cudaError_t launch_apply(Ctx *c, bool guard_overflow = false);   // guard: no update when DevIter::overflow_any is set
cudaError_t launch_solve_explicit(cudaStream_t stream, const double *d_s, const double *d_t, int n, DevIter *d_iter);
cudaError_t launch_get_fd(Ctx *c, double *d_out);
cudaError_t launch_scan_counts(Ctx *c);  // d_cnt → d_rowptr, nnz → d_iter->nnz
// counts[L] → ptr[L + 1] (exclusive scan), cursor[L] zeroed, total → *total_out (device pointer, may be null)
cudaError_t launch_scan_i32(Ctx *c, const int *cnt, long long *ptr, int *cursor, long long L, long long *total_out);
cudaError_t launch_penalty(Ctx *c, double pivot, const LoopScalars &ls);
cudaError_t launch_pair_fd_km(Ctx *c);
cudaError_t launch_colmerge(Ctx *c);
cudaError_t launch_count_valid(Ctx *c, long long nnz);

// ---- matrix-free FPFH (ghicp_fpfh.cu): same contracts as launch_rowsweep / launch_colsweep, FD recomputed on the fly
cudaError_t launch_fpfh_prepare(Ctx *c);   // centred histograms in both layouts
cudaError_t launch_rowsweep_mf(Ctx *c, int mode, const CostParams &cp);
cudaError_t launch_colsweep_mf(Ctx *c, const CostParams &cp);
cudaError_t launch_rowfd_mf(Ctx *c);       // d_row_fd[i] = FD(i, d_row_idx[i]) for this context's rows
cudaError_t launch_get_fd_mf(Ctx *c, double *d_out);
// FPFH fast path: FP32 filter over on-the-fly FD + exact FP64 refinement of the candidates (NN / NNR)
size_t fpfh_fast_parts(const Ctx *c);      // per-CTA partial sums the sweep writes
size_t fpfh_fast_rec_floats();             // floats per source record
cudaError_t launch_fpfh_fast_build(Ctx *c);                                   // once, after launch_fpfh_prepare
cudaError_t launch_fpfh_fast_prep(Ctx *c);                                    // per iteration
cudaError_t launch_fpfh_fast_seed(Ctx *c, const CostParams &cp, bool with_cols, bool use_guess);
cudaError_t launch_fpfh_fast_sweep(Ctx *c, const CostParams &cp, bool pre, bool with_cols);
cudaError_t launch_fpfh_fast_finish(Ctx *c, const CostParams &cp, bool with_cols);
// FPFH + KM (settled loop): the filter as the KM gate, candidates into this rank's block of the settled route
cudaError_t launch_fpfh_gate_seed(Ctx *c, const CostParams &cp, const LoopScalars &ls);
cudaError_t launch_fpfh_cand_block(Ctx *c, const CostParams &cp);

// ---- opt-in solvers (ghicp_solvers.cu) -------------------------------------------------------------
// Overwrites iter->Rt and iter->rmse_after from the pair list in the ctx (after launch_solve produced the statistics)
cudaError_t launch_solve_alt(Ctx *c, int solver);
// stand-alone: explicit column-major n x 3 point lists (+ normals, + weights, either may be null)
cudaError_t launch_solve_alt_explicit(cudaStream_t stream, int solver, const double *d_s, const double *d_t,
                                      const double *d_tn, const double *d_w, int n, DevIter *d_iter);

// ---- pre-processing (ghicp_prep.cu): voxel filter, radius PCA / curvature, keypoint pruning + NMS, on device arrays ----
cudaError_t prep_voxel_downsample(cudaStream_t st, const float *d_xyz, int n, float voxel_size, int *d_out, int *n_out);
cudaError_t prep_detect_keypoints(cudaStream_t st, const float *d_xyz, int n, float radius, float ratio_max, int min_pts,
                                  float nms_radius, float *d_lam, double *d_curv, int *d_cnt, int *d_kp, int *n_kp,
                                  int *nms_rounds);
// BSCEncoder::extractBinaryFeatures (include/binary_feature_extraction.hpp:603-676) on device arrays, see ghicp_prep.cu
cudaError_t prep_bsc_extract(cudaStream_t st, const float *d_xyz, int n, const int *d_kp, int nkp, float R, int side,
                             const int *d_pairs, int dof_type, unsigned char *d_bits, float *d_lrf, int *d_status);

// FPFHfeature::compute_fpfh_feature + keyfpfh (include/fpfh.hpp:36-115) on device arrays, see ghicp_prep.cu
struct FpfhStats {
  long long candidates = 0;   // k-NN candidates examined, all queries together
  int queries = 0;            // k-NN queries (every point of the cloud)
  int fallbacks = 0;          // queries that took the exhaustive scan
  float cell = 0.f;           // grid cell edge used
};
cudaError_t prep_fpfh(cudaStream_t st, const float *d_xyz, int n, const int *d_idx, int nidx, int k, float cell_scale,
                      float *d_fpfh, float *d_normals, int *d_status, int *d_nb_idx, float *d_nb_d2, cudaEvent_t ev_mid,
                      FpfhStats *stats);
// The k-NN normals of prep_fpfh alone (k in 3..32, k_eff = min(k, n)), with CheckNormals' substitute (0.577, 0.577, 0.577)
// where a normal is not finite (fewer than 3 neighbours): d_normals [n][3].  The k-NN lists are allocated before any launch.
cudaError_t prep_knn_normals(cudaStream_t st, const float *d_xyz, int n, int k, float *d_normals);
// The same estimator over radius neighbourhoods (CRegistration::compute_fpfh_feature, src/common_reg.cpp:373-389), see
// ghicp_prep.cu
struct FpfhRadiusStats {
  long long nb_n = 0, nb_f = 0;   // list entries at the normal / the feature radius
  long long needed = 0;           // entries counted (both radii); > budget: the call returned cudaErrorMemoryAllocation
  long long budget = 0;           // entry budget of the call
  int spfh_points = 0;            // points whose SPFH was computed
  int rings_n = 0, rings_f = 0;   // grid rings walked per query
  float cell = 0.f;               // grid cell edge
};
cudaError_t prep_fpfh_radius(cudaStream_t st, const float *d_xyz, int n, const int *d_idx, int nidx, float rn, float rf,
                             long long nb_max, float *d_fpfh, float *d_normals, int *d_status, cudaEvent_t ev_lists,
                             cudaEvent_t ev_normals, FpfhRadiusStats *stats);

// SAC-IA coarse alignment from FPFH histograms (ghicp_sac.cu, DESIGN.md §3.11) on device arrays: source points [ns][3] and
// histograms [ns][33], target likewise; parameters already checked.  dbg (may be null): host arrays that receive the
// per-hypothesis intermediates (any may be null) and the scoring grid's cell edge — for tests and tools.
struct SacDebug {
  int *samples = nullptr;             // [H][nr_samples], -1 for an invalid hypothesis
  int *valid = nullptr;               // [H]
  int *corr = nullptr;                // [H][nr_samples] target indices
  float *rt = nullptr;                // [H][12]: R row-major, then t
  unsigned long long *err = nullptr;  // [H] error sums in units of 2^-32
  double cell = 0.0;
};
cudaError_t sac_run(const float *d_P, const float *d_Fs, int ns, const float *d_Q, const float *d_Ft, int nt,
                    const ghicp_sac_params *p, ghicp_sac_result *out, SacDebug *dbg);
cudaError_t sac_points_from_soa(const double *d_soa, int n, float *d_xyz);   // [3][n] doubles -> [n][3] floats

// Overlap and fitness on the dense clouds (ghicp_overlap.cu, DESIGN.md §3.12).  OverlapTarget = B's grid, independent of the
// threshold and reusable across calls.  overlap_run fills every field of out but stage_ms; h_d2_out (host, may be null)
// receives the per-point d2.  ev_queries (may be null) is recorded after the workspaces are allocated.
struct OverlapTarget;
cudaError_t overlap_target_build(const float *d_b, int n_b, OverlapTarget **out);
void overlap_target_free(OverlapTarget *t);
cudaError_t overlap_run(const float *d_a, int n_a, const OverlapTarget *t, const double *Rt, float thre_dis, double max_range,
                        int want_fitness, cudaEvent_t ev_queries, ghicp_overlap_result *out, float *h_d2_out);

// ICP on the dense clouds (ghicp_icp.cu): point-to-point (p->metric 0, DESIGN.md §3.13), point-to-plane (1, §3.14) or
// Generalized ICP (2, §3.15).  d_src [n_src][3] = the finite source points (the loop's), d_all [n_all][3] = the whole source
// (fitness and h_moved); t = the target's grid over d_tgt; d_nrm [n_tgt][3] = the target's normals (prep_knn_normals; read
// by metrics 1 and 2), d_nrm_s [n_src][3] = d_src's normals (metric 2 only); parameters already checked.  Fills every field
// of out but stage_ms; h_moved, h_cor, h_mse (host, may be null) receive the moved source and the per-iteration traces.
// ev_iter / ev_fit (may be null) are recorded before the first iteration and before the fitness.
cudaError_t icp_run(const float *d_src, int n_src, const float *d_all, int n_all, const OverlapTarget *t, const float *d_tgt,
                    const float *d_nrm, const float *d_nrm_s, const double *guess, const ghicp_icp_params *p, cudaEvent_t ev_iter,
                    cudaEvent_t ev_fit, ghicp_icp_result *out, float *h_moved, int *h_cor, double *h_mse);

// CFilter::SORFilter (ghicp_sor_filter, DESIGN.md §3.16) on device arrays, see ghicp_prep.cu: d_out (capacity n) receives the
// kept indices, d_dist [n] every point's mean distance; *r every field.  mean_k in 1..128.
cudaError_t prep_sor_filter(cudaStream_t st, const float *d_xyz, int n, int mean_k, double std_mul, int *d_out, float *d_dist,
                            ghicp_sor_result *r);

// glue of the device-resident pipeline (ghicp_prep_run)
cudaError_t prep_gather_points(cudaStream_t st, const float *d_xyz, const int *d_idx, int m, float *d_out);
cudaError_t prep_kp_coords(cudaStream_t st, const float *d_xyz, const int *d_kp, int nkp, double *d_soa);
cudaError_t prep_bounds(cudaStream_t st, const float *d_xyz, int n, float mn[3], float mx[3], int *nfin = nullptr);

// ---- streaming path (ghicp_stream.cu) -----------------------------------------------------------
cudaError_t launch_stream_prep(Ctx *c, const CostParams &cp, int for_km_gate);
cudaError_t launch_stream_gate(Ctx *c, const CostParams &cp);
cudaError_t launch_stream_seed(Ctx *c, const CostParams &cp, bool with_cols);
cudaError_t launch_stream(Ctx *c, const CostParams &cp, StreamMode mode, bool stats);
cudaError_t launch_stream_resolve(Ctx *c, const CostParams &cp, bool with_cols);
cudaError_t launch_finalize_fast(Ctx *c);
cudaError_t launch_penalty_only(Ctx *c, const LoopScalars &ls);
cudaError_t launch_scan_rows(Ctx *c);
cudaError_t launch_emit_scatter(Ctx *c, const CostParams &cp, unsigned long long n_emitted);
cudaError_t launch_csr_check(Ctx *c, const CostParams &cp);
int stream_num_parts(const Ctx *c);
size_t xblock_bytes(size_t xcap);
cudaError_t launch_emit_check(Ctx *c, const CostParams &cp);   // this rank's gate hits, checked exactly -> d_xsend
cudaError_t launch_xbuild(Ctx *c);                             // gathered blocks -> statistics + CSR, all on the device

// ---- KM (ghicp_auction.cu) ----------------------------------------------------------------------
// Solves max-gain partial matching on the CSR in the ctx (rows = persons). Result in d_owner/d_assign.
int km_auction(Ctx *c, int n_rows, int n_cols, long long nnz, double eps_final, double max_gain,
               KmResult *res);
cudaError_t launch_build_csc(Ctx *c, int n_rows, int n_cols, long long nnz);
// settled loop (sparse graph): the same single forward phase, edge count read on the device, nothing read back;
// counters land in h_counters with the iteration's final copy (km_auction_settled_result after the synchronize)
int km_auction_settled(Ctx *c, int n_rows, int n_cols, long long nnz_hint, double eps_final);
int km_auction_settled_result(Ctx *c, KmResult *res);

// ---- multi-GPU exchange (ghicp_comm.cu) ------------------------------------------------------------
int comm_unique_id(void *id128);
int comm_init(Ctx *c, const void *id128, int rank, int world);
void comm_destroy(Ctx *c);
int comm_warmup(Ctx *c);
int comm_exchange(Ctx *c, int what);         // what: OR of ExchangeBits
int comm_gather_counts(Ctx *c);
int comm_gather_edges(Ctx *c, const long long *cut);
int comm_allgather_bytes(Ctx *c, const void *send, void *recv, size_t bytes);   // the one exchange of a settled KM iteration

// misc
void set_error(Ctx *c, const std::string &msg);

}  // namespace ghicp_b200
