// ghicp_stream.cu — the streaming cost/correspondence kernel of the GH-ICP inner loop (sm_90a).
//
// One pass over the N x M feature-distance plane (packed, 9 / 10 / 12 bits per pair — the only O(N*M) HBM traffic of an
// iteration) fuses calED + calCD_* + the NN / NNR scans or the KM candidate gate
// (src/ghicp_reg.cpp:114-139, 216-293, 348-365, 622-650, 715-733) and the CD mean / std reductions
// (:228, 264-272).  ED and CD are never stored.
//
// Arithmetic: the bulk runs in FP32 as a FILTER with a rigorous error margin; every decision the
// reference takes on doubles (row / column argmin, the CD < penalty gate) is re-evaluated in FP64 with the
// reference's exact operation order for the few pairs the filter cannot rule out, so index results are
// identical to the all-double evaluation (and to the oracle).  The filter evaluates
//      d2' = A*|s - t|^2 = S.w + T.w + S.x*T.x + S.y*T.y + S.z*T.z      (3 FFMA + 1 FADD)
// with S = (s_c, A|s_c|^2), T = (-2A t_c, A|t_c|^2), A = (scale*WED)^2, coordinates centred on the target
// centroid, then cd32 = sqrt.approx(d2') + WFD*fd.   |cd32 - cd64| <= margin (see k_margin).
//
// Thread mapping: a warp owns a 256-column panel (lane = 8 consecutive columns whose T operands stay in
// registers) and sweeps ST_RB source rows, one quad block of the packed plane (4 rows, ghicp_internal.h) per TMA stage;
// per row a lane reads its 8 low bytes, per quad its hb words of high bits, and decodes in registers.  Row minima are
// warp-reduced with one REDUX per row.
#include <climits>
#include <cstdlib>
#include <cuda_fp16.h>

#include "ghicp_internal.h"

namespace ghicp_b200 {

namespace {

constexpr int ST_THREADS = 256;
constexpr int ST_WARPS = ST_THREADS / 32;
constexpr int ST_CPL = 8;                         // columns per lane
constexpr int ST_PANEL = 32 * ST_CPL;             // columns per warp
constexpr int ST_CTA_COLS = ST_WARPS * ST_PANEL;  // 2048
constexpr int ST_RB = 256;                        // source rows per CTA (upper bound; StreamArgs::rb is what a launch uses)
constexpr int ST_RB_MIN = 64;
constexpr int ST_CTAS_PER_SM = 2;                 // k_stream's residency bound, and the slots stream_rows_per_cta fills
constexpr int ST_UNROLL = FD_QUAD;   // rows per batch = one quad block of the packed plane (part of its format)
constexpr unsigned INF_BITS = 0x7f800000u;
// TMA staging of the FD plane: every warp runs its own ring of stages in at most ST_RING_BYTES; a stage holds ST_QPS
// consecutive quad blocks of the warp's 256-column panel (fd_block_bytes(hb) = 1152 / 1280 / 1536 B each), brought in by ONE
// cp.async.bulk (TMA engine, UBLKCP) and signalled on one mbarrier per stage.  No registers are tied up by loads in flight.
// Four quads per stage (two stages) measured fastest on the H100: fewer, larger copies beat more bytes in flight.
constexpr int ST_RING_BYTES = 12 * 1024;   // per warp
constexpr int ST_DYN_SMEM = ST_WARPS * ST_RING_BYTES;
constexpr int ST_QPS = 4;                  // quad blocks (batches) per stage
template <int HB> __host__ __device__ constexpr int st_quad_bytes() { return FD_LOW_BYTES + 128 * HB; }
template <int HB> __host__ __device__ constexpr int st_stage_bytes() { return ST_QPS * st_quad_bytes<HB>(); }
template <int HB> __host__ __device__ constexpr int st_stages() { return ST_RING_BYTES / st_stage_bytes<HB>(); }
constexpr int ST_MAX_STAGES = ST_RING_BYTES / (ST_QPS * (FD_LOW_BYTES + 128));

#if defined(GHICP_EMU_HOST)
__device__ __forceinline__ void fence_proxy_async() {}     // one OS thread: program order is memory order
__device__ __forceinline__ void fence_mbarrier_init() {}
// Host emulation (tests/harness/cuda_emu/emu_mbarrier.h): an mbarrier is modelled inside its own 64-bit word, a bulk copy
// is a memcpy that completes its bytes at once, a waiting fiber yields.
__device__ __forceinline__ void mbar_init(unsigned long long *bar, int count) { emu::bar_init(bar, count); }
__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, unsigned bytes) { emu::bar_arrive_expect_tx(bar, bytes); }
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, unsigned parity) { emu::bar_wait(bar, parity); }
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, unsigned bytes, unsigned long long *bar) { emu::bulk_copy(dst, src, bytes, bar); }
__device__ __forceinline__ unsigned byte_perm(unsigned x, unsigned y, unsigned sel) {   // PRMT, default mode
  const unsigned long long xy = ((unsigned long long)y << 32) | x;
  unsigned r = 0;
  for (int n = 0; n < 4; ++n) r |= (unsigned)((xy >> (8 * ((sel >> (4 * n)) & 7))) & 0xffu) << (8 * n);
  return r;
}
#else
__device__ __forceinline__ unsigned byte_perm(unsigned x, unsigned y, unsigned sel) { return __byte_perm(x, y, sel); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_mbarrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long *bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, unsigned parity) {
  unsigned ok;
  do {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  } while (!ok);
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, unsigned bytes, unsigned long long *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

#endif

// Column pairs travel as one 64-bit value (two floats); Hopper has no packed f32x2 arithmetic, so fma2 / add2 are two scalar
// operations with one rounding each.
typedef unsigned long long u64;
__device__ __forceinline__ u64 pack2(float lo, float hi) { return ((u64)__float_as_uint(hi) << 32) | __float_as_uint(lo); }
__device__ __forceinline__ void unpack2(u64 v, float &lo, float &hi) { lo = __uint_as_float((unsigned)v); hi = __uint_as_float((unsigned)(v >> 32)); }
__device__ __forceinline__ u64 fma2(u64 a, u64 b, u64 c) {
  float al, ah, bl, bh, cl, ch; unpack2(a, al, ah); unpack2(b, bl, bh); unpack2(c, cl, ch);
  return pack2(fmaf(al, bl, cl), fmaf(ah, bh, ch));
}
__device__ __forceinline__ u64 add2(u64 a, u64 b) {
  float al, ah, bl, bh; unpack2(a, al, ah); unpack2(b, bl, bh);
  return pack2(__fadd_rn(al, bl), __fadd_rn(ah, bh));
}
#if defined(GHICP_EMU_HOST)
// Host emulation of the PTX-only operations: the approximate square root becomes the exact one (inside the filter's error
// budget).
__device__ __forceinline__ float sqrt_approx(float x) { return sqrtf(x); }
#else
__device__ __forceinline__ float sqrt_approx(float x) {
  float r;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
  return r;
}
#endif
__device__ __forceinline__ unsigned long long ord64(double v) {  // CD >= 0: bit pattern is monotone
  return (unsigned long long)__double_as_longlong(v);
}
__device__ __forceinline__ float half_lo(unsigned w) { return __half2float(__ushort_as_half((unsigned short)(w & 0xffffu))); }
__device__ __forceinline__ float half_hi(unsigned w) { return __half2float(__ushort_as_half((unsigned short)(w >> 16))); }

// Decode of column pair p (columns 2p, 2p+1 of the lane) of quad row u from the staged quad block: lo4 = the 4 low bytes
// of columns 4 (p / 2) ..., hw = the lane's high-bit words.  One PRMT spreads the two low bytes to bits 0 and 16, one shift
// brings the pair's high bits to bits 8 (and 24) and one LOP3 ORs them in: two 16-bit patterns fd0, fd1.  Read as fp16, a
// pattern v <= 2048 is exactly v * 2^-24 (subnormal below 1024, exponent field 1 below 2048, 2^-13 for 2048), so the usual
// fp16 -> f32 conversion yields f = fd * 2^-24 exactly, and fmaf(f, 2^24 b, dist) == fmaf(fd, b, dist) bit for bit: the
// product is exact either way and the FMA rounds once.
template <int HB>
__device__ __forceinline__ void fd_pair(unsigned lo4, const unsigned (&hw)[HB], int u, int p, float &f0, float &f1) {
  constexpr int PPW = 16 / HB;                       // pairs per high-bit word
  constexpr unsigned MASK = HB == 1 ? 0x01000100u : HB == 2 ? 0x03000300u : 0x0f000f00u;
  const int k = 4 * u + p;
  const int sh = HB * (k % PPW) - 8;
  const unsigned hv = sh >= 0 ? hw[k / PPW] >> sh : hw[k / PPW] << -sh;
  const unsigned h2 = byte_perm(lo4, 0u, (p & 1) ? 0x4342u : 0x4140u) | (hv & MASK);
  f0 = half_lo(h2);
  f1 = half_hi(h2);
}

// exact CD(i,j), the reference's operation order, no FMA contraction (src/ghicp_reg.cpp:122,224,259)
__device__ GHICP_NOINLINE double exact_cd(const StreamArgs &a, int i, int j) {
  const double sx = a.s[i], sy = a.s[(size_t)a.N + i], sz = a.s[2 * (size_t)a.N + i];
  const double tx = a.t[j], ty = a.t[(size_t)a.M + j], tz = a.t[2 * (size_t)a.M + j];
  const double dx = __dsub_rn(sx, tx), dy = __dsub_rn(sy, ty), dz = __dsub_rn(sz, tz);
  const double d2 = __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
  const double ed = __dmul_rn(a.scale, __dsqrt_rn(d2));
  if (a.fd) {
    const double fd = (double)fd_at(a.fd, a.fd_rows, a.fd_hb, i - a.row0, j);
    return __dadd_rn(__dmul_rn(a.WED, ed), __dmul_rn(a.WFD, fd));
  }
  return ed;
}

// ---------------------------------------------------------------------------------------------
// per-iteration operand preparation
// ---------------------------------------------------------------------------------------------
__global__ void k_prep(const double *__restrict__ s, const double *__restrict__ t, int N, int M, double cx,
                       double cy, double cz, double A, float4 *__restrict__ S4, float4 *__restrict__ T4,
                       StreamDev *dev) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  float r2 = 0.f;
  if (k < N) {
    const double x = s[k] - cx, y = s[(size_t)N + k] - cy, z = s[2 * (size_t)N + k] - cz;
    const double n2 = x * x + y * y + z * z;
    S4[k] = make_float4((float)x, (float)y, (float)z, (float)(A * n2));
    r2 = fmaxf(r2, __double2float_ru(n2));
  }
  if (k < M) {
    const double x = t[k] - cx, y = t[(size_t)M + k] - cy, z = t[2 * (size_t)M + k] - cz;
    const double n2 = x * x + y * y + z * z;
    T4[k] = make_float4((float)(-2.0 * A * x), (float)(-2.0 * A * y), (float)(-2.0 * A * z), (float)(A * n2));
    r2 = fmaxf(r2, __double2float_ru(n2));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) r2 = fmaxf(r2, __shfl_xor_sync(0xffffffffu, r2, o));
  if ((threadIdx.x & 31) == 0) atomicMax(&dev->r2max_bits, __float_as_uint(r2));
}

// Error bound of the FP32 filter.  d2' carries <= 32*2^-24*A*R^2 absolute error (input roundings of
// S, T + 1 add + 3 fma on magnitudes <= 4*A*R^2, R = max centred norm), so |sqrt(d2'_32) - a*dist| <=
// sqrt(that); sqrt.approx, the fd FFMA and the float weight add 2^-21-relative terms.
// The bound holds while every operand and partial sum is a normal float (STREAM_WINDOW_*): below it a rounding costs up to
// 2^-150 absolutely and sqrt.approx.ftz flushes d2' to 0, above it S.w / T.w overflow and d2' becomes NaN.  Outside the
// window StreamDev::out_of_range sends the iteration to the all-double route (exact_fallback bit 2).
__global__ void k_margin(StreamDev *dev, double A, double a, double b, double fdmax, const DevIter *iter,
                         int use_iter_penalty, double rel_slack, double kappa) {
  const double R2 = (double)__uint_as_float(dev->r2max_bits);
  const double E = 32.0 * 5.9604644775390625e-08 * A * R2;
  const double R = sqrt(R2);
  double m = sqrt(E) * 1.001 + 9.5367431640625e-07 * (2.0 * a * R + b * fdmax) + 1e-30;
  dev->margin = __double2float_ru(m);
  dev->cand_count[0] = 0;
  dev->cand_count[1] = 0;
  dev->overflow = 0;
  dev->out_of_range = !stream_in_window(A, R2);
  dev->nnz_valid = 0;
  dev->emit_count = 0;
  if (use_iter_penalty) {
    // KM gate: superset threshold = penalty*(1+slack) + margin, rounded up
    const double p = iter->penalty * kappa;   // thresholds live in the scaled domain
    dev->thr_hi = __double2float_ru(p + fabs(p) * rel_slack + m);
  } else {
    dev->thr_hi = -1.f;
  }
}

// Seeds of the running row / column minima: CD of last iteration's partner under the current geometry
// is an upper bound of the new minimum (exactly evaluated, rounded up).
__global__ void k_seed(StreamArgs a, const int *__restrict__ prev_row_idx, const int *__restrict__ prev_col_idx,
                       int have_prev) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= a.row0 && k < a.row0 + a.nloc) {
    unsigned bits = INF_BITS;
    if (have_prev) {
      int j = prev_row_idx[k];
      if (j >= 0 && j < a.M) bits = __float_as_uint(__double2float_ru(a.kappa * exact_cd(a, k, j) * 1.0000001));
    }
    a.row_thr_init[k] = bits;
    a.rowbest[k] = ~0ull;
    a.rowidx[k] = INT_MAX;
  }
  if (a.col_thr_init && k < a.M) {
    unsigned bits = INF_BITS;
    if (have_prev) {
      int i = prev_col_idx[k];
      if (i >= a.row0 && i < a.row0 + a.nloc) bits = __float_as_uint(__double2float_ru(a.kappa * exact_cd(a, i, k) * 1.0000001));
    }
    a.col_thr_init[k] = bits;
    a.colbest[k] = ~0ull;
    a.colidx[k] = INT_MAX;
  }
}

// ---------------------------------------------------------------------------------------------
// the streaming kernel
// ---------------------------------------------------------------------------------------------
// Saturating: once the count has reached the cap nobody adds to it, so it stays below cap + resident threads and cannot wrap
// past INT_MAX into a negative slot that passes the bound (a far outlier widens the margin enough for billions of pushes).
__device__ __forceinline__ void push_candidate(const StreamArgs &a, int which, int i, int j, double cd) {
  if (*(volatile int *)&a.dev->cand_count[which] >= a.cand_cap) { a.dev->overflow = 1; return; }
  const int slot = atomicAdd(&a.dev->cand_count[which], 1);
  if (slot < a.cand_cap) {
    Cand c;
    c.i = i; c.j = j; c.cd = cd;
    a.cand[which][slot] = c;
  } else {
    a.dev->overflow = 1;
  }
}

// slow paths (rare): kept out of line so the streaming loop stays compact in the instruction cache
__device__ GHICP_NOINLINE void slow_row(const StreamArgs &a, int i, int j, float cdv, float lim) {
  if (cdv <= lim) {
    const double e = exact_cd(a, i, j);
    atomicMin(&a.rowbest[i], ord64(e));
    push_candidate(a, 0, i, j, e);
  }
}
__device__ GHICP_NOINLINE void slow_col(const StreamArgs &a, int i, int j, float cdv, float lim) {
  if (cdv <= lim) {
    const double e = exact_cd(a, i, j);
    atomicMin(&a.colbest[j], ord64(e));
    push_candidate(a, 1, i, j, e);
  }
}

// KM count pass, rare path: a warp-row with `total` gate hits (bit c of mask8 = column j0 + c of this lane).
// Besides the per-row count the hits are appended to a global edge list, so that the CSR can be scattered
// from the list instead of streaming the plane a second time (the fill pass stays as the overflow fallback).
__device__ GHICP_NOINLINE void emit_hits(const StreamArgs &a, int *s_cnt_r, int row, int j0, unsigned mask8, int total,
                                       int lane) {
  if (lane == 0) atomicAdd(s_cnt_r, total);
  if (a.emit_cap == 0) return;  // list switched off (dense graph expected): count only, the fill pass follows
  unsigned long long base = 0;
  if (lane == 0) base = atomicAdd(&a.dev->emit_count, (unsigned long long)total);
  base = __shfl_sync(0xffffffffu, base, 0);
  const int c8 = __popc(mask8);
  int incl = c8;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += y;
  }
  unsigned long long pos = base + (unsigned long long)(incl - c8);
  while (mask8) {
    const int c = __ffs(mask8) - 1;
    mask8 &= mask8 - 1;
    if (pos < a.emit_cap) a.emit[pos] = ((unsigned long long)(unsigned)row << 32) | (unsigned)(j0 + c);
    ++pos;
  }
}

template <int MODE, bool HAS_FD, bool STATS, bool FULL, int HB, bool X2>
__device__ __forceinline__ void sweep(const StreamArgs &a, const float4 *s_S4, const float *s_S8, unsigned *s_thr, int *s_cnt,
                                      int r0, int nrows, int j0, int lane, double &dsum, double &dsq,
                                      unsigned char *ring, unsigned long long *bars) {
  float Tx[ST_CPL], Ty[ST_CPL], Tz[ST_CPL], Tw[ST_CPL];
  float colrun[ST_CPL];
#pragma unroll
  for (int c = 0; c < ST_CPL; ++c) {
    const int j = j0 + c;
    if (FULL || j < a.M) {
      const float4 T = a.T4[j];
      Tx[c] = T.x; Ty[c] = T.y; Tz[c] = T.z; Tw[c] = T.w;
      colrun[c] = (MODE == SM_NNR || MODE == SM_PRE_COLS) ? __uint_as_float(a.col_thr_init[j]) : 0.f;
    } else {
      Tx[c] = Ty[c] = Tz[c] = 0.f;
      Tw[c] = __uint_as_float(INF_BITS);  // cd = +inf: never a minimum, never below a threshold
      colrun[c] = (MODE == SM_PRE_COLS) ? __uint_as_float(INF_BITS) : -1.f;  // never triggers / never written
    }
  }
  u64 Tx2[ST_CPL / 2], Ty2[ST_CPL / 2], Tz2[ST_CPL / 2], Tw2[ST_CPL / 2];
  if (X2) {
#pragma unroll
    for (int p = 0; p < ST_CPL / 2; ++p) {
      Tx2[p] = pack2(Tx[2 * p], Tx[2 * p + 1]); Ty2[p] = pack2(Ty[2 * p], Ty[2 * p + 1]);
      Tz2[p] = pack2(Tz[2 * p], Tz[2 * p + 1]); Tw2[p] = pack2(Tw[2 * p], Tw[2 * p + 1]);
    }
  }
  const float margin = a.dev->margin;
  const float m2 = 2.f * margin;
  if (MODE == SM_NNR) {
#pragma unroll
    for (int c = 0; c < ST_CPL; ++c) colrun[c] += m2;   // (padding columns: cd = +inf never passes a finite threshold)
  }
  const float thr_hi = a.dev->thr_hi;
  const float b24 = a.b * 16777216.f;   // 2^24 b, exact: the decoded FD values carry the factor 2^-24 (fd_pair)
  // ---- TMA ring bookkeeping (warp-private) ----
  constexpr int STAGES = st_stages<HB>(), STAGE_BYTES = st_stage_bytes<HB>(), QUAD_BYTES = st_quad_bytes<HB>();
  const int panel = j0 - lane * ST_CPL;
  // rows are padded to whole quads (r0 - row0 is a multiple of 4): a batch is one whole quad block, a stage ST_QPS of them
  // (fewer in the CTA's last stage)
  const unsigned char *panel_base = HAS_FD ? a.fd + fd_block_offset(a.fd_rows, HB, r0 - a.row0, panel) : nullptr;
  const int nbatch = (nrows + ST_UNROLL - 1) / ST_UNROLL;
  const int nstage = (nbatch + ST_QPS - 1) / ST_QPS;
  auto issue = [&](int st) {  // lane 0 only
    const int slot = st % STAGES;
    const unsigned bytes = (unsigned)(min(ST_QPS, nbatch - st * ST_QPS) * QUAD_BYTES);
    mbar_expect_tx(&bars[slot], bytes);
    bulk_g2s(ring + slot * STAGE_BYTES, panel_base + (size_t)st * STAGE_BYTES, bytes, &bars[slot]);
  };
  // (the first STAGES stages were issued by the kernel prologue, before the operand staging)

  for (int rb = 0; rb < nrows; rb += ST_UNROLL) {
    uint2 lo[ST_UNROLL];
    unsigned hw[HB];
    // per-batch base addresses: everything inside the unrolled rows is base + immediate
    const int kb = rb / ST_UNROLL, kst = kb / ST_QPS;
    const unsigned char *qbase = HAS_FD ? ring + (kst % STAGES) * STAGE_BYTES + (kb % ST_QPS) * QUAD_BYTES : nullptr;
    if (HAS_FD) {
      if (kb % ST_QPS == 0) mbar_wait(&bars[kst % STAGES], (unsigned)((kst / STAGES) & 1));
#pragma unroll
      for (int w = 0; w < HB; ++w) hw[w] = reinterpret_cast<const unsigned *>(qbase + FD_LOW_BYTES)[w * 32 + lane];
    }
    float psum = 0.f, psq = 0.f;
    u64 psum2 = 0ull, psq2 = 0ull;
    const float *s8base = s_S8 + rb * 8;
    const float4 *s4base = s_S4 + rb;
    unsigned *thrbase = s_thr + rb;
    auto compute_row = [&](const int u, float (&cd)[ST_CPL]) {
        const float4 S = X2 ? make_float4(0.f, 0.f, 0.f, 0.f) : s4base[u];
        if (HAS_FD)  // just-in-time read of this row's 8 low bytes from the staged quad block
          lo[u] = *reinterpret_cast<const uint2 *>(qbase + u * FD_PANEL + lane * ST_CPL);
                if (X2) {
          const ulonglong2 sA = *reinterpret_cast<const ulonglong2 *>(s8base + u * 8);      // (sx,sx) (sy,sy)
          const ulonglong2 sB = *reinterpret_cast<const ulonglong2 *>(s8base + u * 8 + 4);  // (sz,sz) (sw,sw)
#pragma unroll
          for (int p = 0; p < ST_CPL / 2; ++p) {
            u64 acc = add2(Tw2[p], sB.y);
            acc = fma2(sB.x, Tz2[p], acc);
            acc = fma2(sA.y, Ty2[p], acc);
            acc = fma2(sA.x, Tx2[p], acc);
            float d0, d1;
            unpack2(acc, d0, d1);
            d0 = sqrt_approx(fabsf(d0));   // |.|: a slightly negative d2' (cancellation) stays inside the margin
            d1 = sqrt_approx(fabsf(d1));
            if (HAS_FD) {
              float f0, f1;
              fd_pair<HB>(p < 2 ? lo[u].x : lo[u].y, hw, u, p, f0, f1);
              cd[2 * p] = fmaf(f0, b24, d0);
              cd[2 * p + 1] = fmaf(f1, b24, d1);
            } else {
              cd[2 * p] = d0;
              cd[2 * p + 1] = d1;
            }
            if (STATS && FULL) {
              const u64 c2 = pack2(cd[2 * p], cd[2 * p + 1]);
              psum2 = add2(psum2, c2);
              psq2 = fma2(c2, c2, psq2);
            }
          }
          if (STATS && !FULL) {
#pragma unroll
            for (int c = 0; c < ST_CPL; ++c)
              if (j0 + c < a.M) { psum += cd[c]; psq = fmaf(cd[c], cd[c], psq); }
          }
        } else {
        float fdf[ST_CPL];
        if (HAS_FD) {
#pragma unroll
          for (int p = 0; p < ST_CPL / 2; ++p) fd_pair<HB>(p < 2 ? lo[u].x : lo[u].y, hw, u, p, fdf[2 * p], fdf[2 * p + 1]);
        }
#pragma unroll
        for (int c = 0; c < ST_CPL; ++c) {
          float d2 = fmaf(S.x, Tx[c], fmaf(S.y, Ty[c], fmaf(S.z, Tz[c], Tw[c] + S.w)));
          d2 = fmaxf(d2, 0.f);
          const float dist = sqrt_approx(d2);
          if (HAS_FD) {
            cd[c] = fmaf(fdf[c], b24, dist);
          } else {
            cd[c] = dist;
          }
        }
        if (STATS) {
#pragma unroll
          for (int c = 0; c < ST_CPL; ++c) {
            if (FULL || (j0 + c < a.M)) {
              psum += cd[c];
              psq = fmaf(cd[c], cd[c], psq);
            }
          }
        }
        }
    };
    // do_rows = false: the batch-level test has shown that no row of the batch can touch its running minimum
    auto decide_row = [&](const int u, const float (&cd)[ST_CPL], const bool do_rows) {
      const int r = rb + u;
        if (MODE == SM_PRE || MODE == SM_PRE_COLS) {
          // seed pass: FP32 row (and column) minima only, no decisions
          if (do_rows) {
            float m8 = fminf(fminf(fminf(cd[0], cd[1]), fminf(cd[2], cd[3])), fminf(fminf(cd[4], cd[5]), fminf(cd[6], cd[7])));
            const unsigned wmin = __reduce_min_sync(0xffffffffu, __float_as_uint(m8));
            if (lane == 0 && wmin < thrbase[u]) atomicMin(&thrbase[u], wmin);
          }
          if (MODE == SM_PRE_COLS) {
#pragma unroll
            for (int c = 0; c < ST_CPL; ++c) colrun[c] = fminf(colrun[c], cd[c]);
          }
        } else if (MODE == SM_NN || MODE == SM_NNR) {
          float m8 = fminf(fminf(fminf(cd[0], cd[1]), fminf(cd[2], cd[3])), fminf(fminf(cd[4], cd[5]), fminf(cd[6], cd[7])));
          const unsigned wmin = do_rows ? __reduce_min_sync(0xffffffffu, __float_as_uint(m8)) : INF_BITS;
          const float run = __uint_as_float(thrbase[u]);
          if (do_rows && __uint_as_float(wmin) <= run + m2) {  // warp-uniform, rare once the running minimum is tight
            // the row argmin is within 2*margin of the smallest value of ANY set that contains it
            const float lim = fminf(run, __uint_as_float(wmin)) + m2;
#pragma unroll
            for (int c = 0; c < ST_CPL; ++c) slow_row(a, r0 + r, j0 + c, cd[c], lim);
            if (lane == 0) atomicMin(&s_thr[r], wmin);
          }
          if (MODE == SM_NNR && do_rows) {
            // columns: every value within 2*margin of the column's seed (an upper bound of its minimum up to one margin:
            // last iteration's partner evaluated exactly, or the FP32 minimum of the seed pass) is evaluated exactly.
            // The threshold is FIXED for the sweep (colrun holds seed + 2*margin): a running minimum would only save
            // refinements that are already rare, at the price of two more instructions per pair.
            bool hit = false;
#pragma unroll
            for (int c = 0; c < ST_CPL; ++c) hit |= (cd[c] <= colrun[c]);
            if (hit) {
#pragma unroll
              for (int c = 0; c < ST_CPL; ++c) slow_col(a, r0 + r, j0 + c, cd[c], colrun[c]);
            }
            // rare path only: tighten (a column without a seed — its last partner lives on another rank — starts at
            // +inf and must not send its whole length to the exact evaluation)
#pragma unroll
            for (int c = 0; c < ST_CPL; ++c) colrun[c] = fminf(colrun[c], cd[c] + m2);
          }
        } else {
          // KM gate on the superset threshold (exactly re-checked per CSR entry afterwards)
          unsigned mask8 = 0;
#pragma unroll
          for (int c = 0; c < ST_CPL; ++c) mask8 |= (cd[c] < thr_hi) ? (1u << c) : 0u;
          const int c8 = __popc(mask8);
          const int total = __reduce_add_sync(0xffffffffu, c8);
          if (total) {
            if (MODE == SM_COUNT) {
              emit_hits(a, &s_cnt[r], r0 + r, j0, mask8, total, lane);
            } else {
              int base = 0;
              if (lane == 0) base = atomicAdd(&a.cursor[r0 + r], total);
              base = __shfl_sync(0xffffffffu, base, 0);
              int incl = c8;
#pragma unroll
              for (int o = 1; o < 32; o <<= 1) {
                const int y = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += y;
              }
              long long pos = a.rowptr[r0 + r] + base + (incl - c8);
#pragma unroll
              for (int c = 0; c < ST_CPL; ++c)
                if (cd[c] < thr_hi) a.csr_col[pos++] = j0 + c;
            }
          }
        }
          };
    if (rb + ST_UNROLL <= nrows) {
      // full batch: all arithmetic of the ST_UNROLL rows first (4 x 8 independent chains in flight), then
      // the per-row reductions / rare branches
      float cdm[ST_UNROLL][ST_CPL];
#pragma unroll
      for (int u = 0; u < ST_UNROLL; ++u) compute_row(u, cdm[u]);
      if (MODE == SM_COUNT || MODE == SM_FILL) {
        // one gate test per batch: the minimum of the ST_UNROLL x ST_CPL values against the threshold
        // (hits are a few 1e-5 of the plane once the loop has settled)
        float bm[ST_CPL];
#pragma unroll
        for (int cc = 0; cc < ST_CPL; ++cc) {
          bm[cc] = cdm[0][cc];
#pragma unroll
          for (int u = 1; u < ST_UNROLL; ++u) bm[cc] = fminf(bm[cc], cdm[u][cc]);
        }
        const float m8 = fminf(fminf(fminf(bm[0], bm[1]), fminf(bm[2], bm[3])), fminf(fminf(bm[4], bm[5]), fminf(bm[6], bm[7])));
        if (__any_sync(0xffffffffu, m8 < thr_hi)) {
#pragma unroll
          for (int u = 0; u < ST_UNROLL; ++u) decide_row(u, cdm[u], true);
        }
      } else {
        // one vote per batch: does any lane hold a value that can touch the running minimum of its row?
        // (for the seed passes: strictly below it)
        bool touch = false;
#pragma unroll
        for (int u = 0; u < ST_UNROLL; ++u) {
          const float (&cd)[ST_CPL] = cdm[u];
          const float m8 = fminf(fminf(fminf(cd[0], cd[1]), fminf(cd[2], cd[3])), fminf(fminf(cd[4], cd[5]), fminf(cd[6], cd[7])));
          const float run = __uint_as_float(thrbase[u]);
          touch |= (MODE == SM_PRE || MODE == SM_PRE_COLS) ? (m8 < run) : (m8 <= run + m2);
        }
        if (MODE == SM_NNR) {
          // ... or one that can touch its column's threshold (minimum over the batch's rows per column first)
#pragma unroll
          for (int cc = 0; cc < ST_CPL; ++cc) {
            float bmc = cdm[0][cc];
#pragma unroll
            for (int u = 1; u < ST_UNROLL; ++u) bmc = fminf(bmc, cdm[u][cc]);
            touch |= (bmc <= colrun[cc]);
          }
        }
        const bool do_rows = __any_sync(0xffffffffu, touch);
#pragma unroll
        for (int u = 0; u < ST_UNROLL; ++u) decide_row(u, cdm[u], do_rows);
      }
    } else {
#pragma unroll
      for (int u = 0; u < ST_UNROLL; ++u) {
        if (rb + u < nrows) {
          float cd1[ST_CPL];
          compute_row(u, cd1);
          decide_row(u, cd1, true);
        }
      }
    }
    if (HAS_FD && (kb % ST_QPS == ST_QPS - 1 || kb == nbatch - 1)) {
      // every lane has consumed the stage's values: hand it back to the TMA engine for stage kst + STAGES
      __syncwarp();
      if (lane == 0 && kst + STAGES < nstage) {
        fence_proxy_async();
        issue(kst + STAGES);
      }
    }
    if (STATS) {
      if (X2 && FULL) {
        float a0, a1, b0, b1;
        unpack2(psum2, a0, a1);
        unpack2(psq2, b0, b1);
        dsum += (double)a0 + (double)a1;
        dsq += (double)b0 + (double)b1;
      }
      dsum += (double)psum;
      dsq += (double)psq;
    }
  }
  if (MODE == SM_PRE_COLS) {
#pragma unroll
    for (int c = 0; c < ST_CPL; ++c)
      if (FULL || (j0 + c < a.M)) atomicMin(&a.col_thr_init[j0 + c], __float_as_uint(colrun[c]));
  }
}

// two CTAs per SM: the FD variants are held there by their 2 x 96 KB rings anyway, and a tighter bound only costs spills
template <int MODE, bool HAS_FD, bool STATS, int HB, bool X2>
__global__ void __launch_bounds__(ST_THREADS, ST_CTAS_PER_SM) k_stream(const StreamArgs a) {
  __shared__ __align__(16) float s_S8[X2 ? ST_RB * 8 : 8];
#if defined(GHICP_EMU_HOST)
  unsigned char *s_ring = reinterpret_cast<unsigned char *>(emu::dyn_smem());   // host emulation: the launch's dynamic shared memory
#else
  extern __shared__ __align__(128) unsigned char s_ring[];   // [ST_WARPS][ST_RING_BYTES] when HAS_FD
#endif
  __shared__ __align__(8) unsigned long long s_bar[ST_WARPS][ST_MAX_STAGES];
  __shared__ float4 s_S4[ST_RB];
  __shared__ unsigned s_thr[ST_RB];
  __shared__ int s_cnt[ST_RB];
  __shared__ double s_red[2][ST_WARPS];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int r0 = a.row0 + blockIdx.y * a.rb;
  const int nrows = min(a.rb, a.row0 + a.nloc - r0);
  if (HAS_FD) {
    // start the FD stream first: the operand staging below overlaps with the first bulk copies in flight
    constexpr int STAGES = st_stages<HB>(), STAGE_BYTES = st_stage_bytes<HB>(), QUAD_BYTES = st_quad_bytes<HB>();
    const int panel0 = blockIdx.x * ST_CTA_COLS + warp * ST_PANEL;
    if (lane == 0) {
      for (int st = 0; st < STAGES; ++st) mbar_init(&s_bar[warp][st], 1);
      fence_mbarrier_init();
      if (panel0 < a.M) {
        const unsigned char *pb = a.fd + fd_block_offset(a.fd_rows, HB, r0 - a.row0, panel0);
        const int nbatch = (nrows + ST_UNROLL - 1) / ST_UNROLL;
        const int nstage = (nbatch + ST_QPS - 1) / ST_QPS;
        for (int st = 0; st < min(STAGES, nstage); ++st) {
          const unsigned bytes = (unsigned)(min(ST_QPS, nbatch - st * ST_QPS) * QUAD_BYTES);
          mbar_expect_tx(&s_bar[warp][st], bytes);
          bulk_g2s(s_ring + warp * ST_RING_BYTES + st * STAGE_BYTES, pb + (size_t)st * STAGE_BYTES, bytes, &s_bar[warp][st]);
        }
      }
    }
    __syncwarp();
  }
  for (int r = tid; r < ST_RB; r += ST_THREADS) {
    const float4 Sv = (r < nrows) ? a.S4[r0 + r] : make_float4(0.f, 0.f, 0.f, 0.f);
    s_S4[r] = Sv;
    if (X2) {
      float *d = s_S8 + r * 8;
      d[0] = d[1] = Sv.x; d[2] = d[3] = Sv.y; d[4] = d[5] = Sv.z; d[6] = d[7] = Sv.w;
    }
    s_thr[r] = ((MODE == SM_NN || MODE == SM_NNR || MODE == SM_PRE || MODE == SM_PRE_COLS) && r < nrows) ? a.row_thr_init[r0 + r] : INF_BITS;
    s_cnt[r] = 0;
  }
  __syncthreads();
  unsigned char *ring = HAS_FD ? s_ring + warp * ST_RING_BYTES : nullptr;
  const int panel = blockIdx.x * ST_CTA_COLS + warp * ST_PANEL;
  const int j0 = panel + lane * ST_CPL;
  double dsum = 0.0, dsq = 0.0;
  if (panel < a.M) {
    if (panel + ST_PANEL <= a.M)
      sweep<MODE, HAS_FD, STATS, true, HB, X2>(a, s_S4, s_S8, s_thr, s_cnt, r0, nrows, j0, lane, dsum, dsq, ring, s_bar[warp]);
    else
      sweep<MODE, HAS_FD, STATS, false, HB, X2>(a, s_S4, s_S8, s_thr, s_cnt, r0, nrows, j0, lane, dsum, dsq, ring, s_bar[warp]);
  }
  if (STATS) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      dsum += __shfl_xor_sync(0xffffffffu, dsum, o);
      dsq += __shfl_xor_sync(0xffffffffu, dsq, o);
    }
    if (lane == 0) { s_red[0][warp] = dsum; s_red[1][warp] = dsq; }
  }
  __syncthreads();
  if (STATS && tid == 0) {
    double S1 = 0.0, S2 = 0.0;
    for (int w = 0; w < ST_WARPS; ++w) { S1 += s_red[0][w]; S2 += s_red[1][w]; }
    const size_t blk = (size_t)blockIdx.y * gridDim.x + blockIdx.x;
    a.part_stats[2 * blk] = S1;
    a.part_stats[2 * blk + 1] = S2;
  }
  if (MODE == SM_COUNT) {
    for (int r = tid; r < nrows; r += ST_THREADS)
      if (s_cnt[r]) atomicAdd(&a.cnt[r0 + r], s_cnt[r]);
  }
  if (MODE == SM_PRE || MODE == SM_PRE_COLS) {
    for (int r = tid; r < nrows; r += ST_THREADS) atomicMin(&a.row_thr_init[r0 + r], s_thr[r]);
  }
}

// exact index resolution: among the candidates whose exact CD equals the row (column) minimum keep the
// smallest index — the reference's first-minimum tie-break (src/ghicp_reg.cpp:626, 641, 719).
__global__ void k_resolve(const StreamArgs a, int which) {
  const int n = min(a.dev->cand_count[which], a.cand_cap);
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
    const Cand c = a.cand[which][k];
    if (which == 0) {
      if (ord64(c.cd) == a.rowbest[c.i]) atomicMin(&a.rowidx[c.i], c.j);
    } else {
      if (ord64(c.cd) == a.colbest[c.j]) atomicMin(&a.colidx[c.j], c.i);
    }
  }
}
__global__ void k_publish(const StreamArgs a, double *row_cd, int *row_idx, double *col_cd, int *col_idx,
                          double *xstats, int rank) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k == 0) xstats[4 * rank + 2] = (a.dev->overflow || a.dev->out_of_range) ? 1.0 : 0.0;  // travels with the statistics
  if (k >= a.row0 && k < a.row0 + a.nloc) {
    row_cd[k] = __longlong_as_double((long long)a.rowbest[k]);
    const int j = a.rowidx[k];
    row_idx[k] = j;
    a.row_fd[k] = (a.fd && j >= 0 && j < a.M) ? (float)fd_at(a.fd, a.fd_rows, a.fd_hb, k - a.row0, j) : 0.f;
  }
  if (col_cd && k < a.M) {
    col_cd[k] = __longlong_as_double((long long)a.colbest[k]);
    col_idx[k] = a.colidx[k];
  }
}

// fast statistics: this rank's partial sums of CD and CD^2 (the penalty rule runs in k_penalty)
__global__ void __launch_bounds__(1024) k_finalize_fast(const double *__restrict__ part_stats, int n_parts,
                                                        double *__restrict__ xstats, int rank, double kappa,
                                                        const StreamDev *dev) {
  __shared__ double sm[2][32];
  double a0 = 0.0, a1 = 0.0;
  for (int p = threadIdx.x; p < n_parts; p += blockDim.x) { a0 += part_stats[2 * p]; a1 += part_stats[2 * p + 1]; }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) { a0 += __shfl_xor_sync(0xffffffffu, a0, o); a1 += __shfl_xor_sync(0xffffffffu, a1, o); }
  if (lane == 0) { sm[0][warp] = a0; sm[1][warp] = a1; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double S1 = 0.0, S2 = 0.0;
    for (int w = 0; w < 32; ++w) { S1 += sm[0][w]; S2 += sm[1][w]; }
    xstats[4 * rank] = S1 / kappa;               // back from the filter's scaled domain
    xstats[4 * rank + 1] = S2 / (kappa * kappa);
    xstats[4 * rank + 2] = dev->out_of_range ? 1.0 : 0.0;   // k_penalty: DevIter::overflow_any (KM general route: redo)
  }
}
// BSC iterations > 1: the penalty does not depend on this iteration's statistics (src/ghicp_reg.cpp:279-282)
__global__ void k_penalty_only(LoopScalars ls, DevIter *iter) {
  double penalty = ls.RMS * ls.para1 * ls.scale * ls.WED + (ls.FDM + ls.para2 * ls.FDstd) * ls.WFD;
  iter->penalty = fmax(penalty, 5.0);
}

// KM: exact re-check of every CSR entry the FP32 gate let through; gain = penalty - CD (> 0 for true
// candidates, src/ghicp_reg.cpp:362-363); entries that fail get gain = -1e300 (ignored by the auction).
__global__ void __launch_bounds__(256) k_csr_check(const StreamArgs a, const DevIter *iter, double *csr_gain) {
  const int lane = threadIdx.x & 31;
  const int warps = (gridDim.x * blockDim.x) >> 5;
  const double penalty = iter->penalty;
  int valid = 0;
  for (int i = a.row0 + ((blockIdx.x * blockDim.x + threadIdx.x) >> 5); i < a.row0 + a.nloc; i += warps) {
    const long long b = a.rowptr[i], e = a.rowptr[i + 1];
    for (long long k = b + lane; k < e; k += 32) {
      const int j = a.csr_col[k];
      const double cd = exact_cd(a, i, j);
      a.csr_fd[k] = a.fd ? (float)fd_at(a.fd, a.fd_rows, a.fd_hb, i - a.row0, j) : 0.f;
      if (cd < penalty) { csr_gain[k] = penalty - cd; ++valid; }
      else csr_gain[k] = -1e300;
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) valid += __shfl_xor_sync(0xffffffffu, valid, o);
  if (lane == 0 && valid) atomicAdd(&a.dev->nnz_valid, (unsigned long long)valid);
}

// CSR columns from the edge list of the count pass (order inside a row is arbitrary, as with the fill pass:
// the auction breaks ties by a hash of (row, col), not by position)
__global__ void k_emit_scatter(const StreamArgs a, unsigned long long n) {
  for (unsigned long long k = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; k < n;
       k += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned long long e = a.emit[k];
    const int row = (int)(e >> 32), col = (int)(unsigned)e;
    const long long pos = a.rowptr[row] + atomicAdd(&a.cursor[row], 1);
    a.csr_col[pos] = col;
  }
}


// ---- settled KM iteration: the candidate graph travels as ONE block per rank, no host round trip -----------------------
// Block layout (bytes): XBlockHdr | keys[xcap] (row << 32 | col) | gains[xcap] (double) | fds[xcap] (float).
// Every rank gate-checks its own hits exactly (k_emit_check), ONE all-gather moves the blocks, and every rank builds
// the same CSR from all of them (k_xcount -> tiled scan -> k_xscatter; the order inside a row is arbitrary: the auction
// breaks ties by a hash of (row, col), never by position).
__global__ void __launch_bounds__(256) k_emit_check(const StreamArgs a, const DevIter *iter, const double *__restrict__ xstats_rank,
                                                    XBlockHdr *hdr, unsigned long long *__restrict__ xkey,
                                                    double *__restrict__ xgain, float *__restrict__ xfd, unsigned long long xcap) {
  const unsigned long long count = a.dev->emit_count;
  const bool ovf = count > xcap || count > a.emit_cap || a.dev->out_of_range;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    hdr->count = ovf ? 0ull : count;
    hdr->stats[0] = xstats_rank[0]; hdr->stats[1] = xstats_rank[1];
    hdr->stats[2] = ovf ? 1.0 : 0.0;   // picked up by k_penalty as DevIter::overflow_any (on every rank)
    hdr->stats[3] = 0.0;
  }
  if (ovf) return;
  const double penalty = iter->penalty;
  for (unsigned long long k = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; k < count;
       k += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned long long e = a.emit[k];
    const int i = (int)(e >> 32), j = (int)(unsigned)e;
    const double cd = exact_cd(a, i, j);
    xkey[k] = e;
    xgain[k] = cd < penalty ? penalty - cd : -1e300;   // src/ghicp_reg.cpp:362-363 (strict <)
    xfd[k] = a.fd ? (float)fd_at(a.fd, a.fd_rows, a.fd_hb, i - a.row0, j) : 0.f;
  }
}
__device__ __forceinline__ const XBlockHdr *xblock_hdr(const unsigned char *blocks, size_t block_bytes, int r) {
  return reinterpret_cast<const XBlockHdr *>(blocks + (size_t)r * block_bytes);
}
// per-row candidate counts over all blocks (blockIdx.y = rank); block (0, r) also unpacks the rank's partial CD sums
__global__ void k_xcount(const unsigned char *__restrict__ blocks, size_t block_bytes, unsigned long long xcap, int *__restrict__ cnt,
                         double *__restrict__ xstats, unsigned long long *__restrict__ xcounts) {
  const int r = blockIdx.y;
  const XBlockHdr *h = xblock_hdr(blocks, block_bytes, r);
  if (blockIdx.x == 0 && threadIdx.x < 4) xstats[4 * r + threadIdx.x] = h->stats[threadIdx.x];
  if (blockIdx.x == 0 && threadIdx.x == 4) xcounts[r] = h->count;
  const unsigned long long count = h->count < xcap ? h->count : xcap;
  const unsigned long long *key = reinterpret_cast<const unsigned long long *>(h + 1);
  for (unsigned long long k = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; k < count;
       k += (unsigned long long)gridDim.x * blockDim.x)
    atomicAdd(&cnt[(int)(key[k] >> 32)], 1);
}
__global__ void k_xscatter(const unsigned char *__restrict__ blocks, size_t block_bytes, unsigned long long xcap,
                           const long long *__restrict__ rowptr, int *__restrict__ cursor, int *__restrict__ csr_col,
                           double *__restrict__ csr_gain, float *__restrict__ csr_fd, StreamDev *dev) {
  const int r = blockIdx.y;
  const XBlockHdr *h = xblock_hdr(blocks, block_bytes, r);
  const unsigned long long count = h->count < xcap ? h->count : xcap;
  const unsigned long long *key = reinterpret_cast<const unsigned long long *>(h + 1);
  const double *gain = reinterpret_cast<const double *>(key + xcap);
  const float *fd = reinterpret_cast<const float *>(gain + xcap);
  int valid = 0;
  for (unsigned long long k = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; k < count;
       k += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned long long e = key[k];
    const int row = (int)(e >> 32);
    const long long pos = rowptr[row] + atomicAdd(&cursor[row], 1);
    const double g = gain[k];
    csr_col[pos] = (int)(unsigned)e;
    csr_gain[pos] = g;
    csr_fd[pos] = fd[k];
    valid += g > 0.0 ? 1 : 0;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) valid += __shfl_xor_sync(0xffffffffu, valid, o);
  if ((threadIdx.x & 31) == 0 && valid) atomicAdd(&dev->nnz_valid, (unsigned long long)valid);
}

}  // namespace

// =============================================================================================
static int stream_rows_per_cta(const Ctx *c);
static StreamArgs make_args(Ctx *c, const CostParams &cp) {
  StreamArgs a{};
  a.fd = (c->cfg.feature_type == GHICP_FT_BSC) ? reinterpret_cast<const unsigned char *>(c->d_fd16) : nullptr;
  a.fd_rows = c->fd_rows; a.fd_hb = fd_hb(c->bits); a.N = c->N; a.M = c->M;
  a.row0 = c->r0; a.nloc = c->nloc; a.rb = stream_rows_per_cta(c);
  a.row_fd = c->d_row_fd; a.csr_fd = c->d_csr_fd;
  a.S4 = reinterpret_cast<const float4 *>(c->d_S4); a.T4 = reinterpret_cast<const float4 *>(c->d_T4);
  a.s = c->d_s; a.t = c->d_t;
  a.scale = cp.scale; a.WED = cp.WED; a.WFD = cp.WFD;
  a.b = c->b_eff; a.kappa = c->kappa;
  a.dev = c->d_sdev;
  a.row_thr_init = c->d_row_thr; a.rowbest = c->d_rowbest; a.rowidx = c->d_rowidx2;
  a.col_thr_init = nullptr; a.colbest = c->d_colbest; a.colidx = c->d_colidx2;
  a.cand[0] = c->d_cand[0]; a.cand[1] = c->d_cand[1]; a.cand_cap = c->cand_cap;
  a.part_stats = c->d_part_stats;
  a.cnt = c->d_cnt; a.rowptr = c->d_rowptr; a.cursor = c->d_cursor; a.csr_col = c->d_csr_col;
  a.emit = c->d_emit; a.emit_cap = (c->d_emit && c->emit_on) ? (unsigned long long)c->emit_cap : 0ull;
  return a;
}

// Source rows per CTA.  The grid is (column blocks) x (row blocks) CTAs of equal cost, two resident per SM: with 256 rows a
// sharded rank's last wave is mostly empty (6250 rows x 50k columns: 625 CTAs on 296 slots = 3 waves for 2.1 waves of
// work).  Pick the height (multiple of the batch, 64 ... 256) that minimises waves x rows — 180 rows in that example:
// 875 CTAs, 2.96 waves.
static int stream_rows_per_cta(const Ctx *c) {
  static int slots = 0;
  if (slots == 0) {
    int n_sm = GHICP_SMS;
    cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, c->device);
    slots = ST_CTAS_PER_SM * (n_sm > 0 ? n_sm : GHICP_SMS);
  }
  const long long gx = (c->M + ST_CTA_COLS - 1) / ST_CTA_COLS;
  const int nloc = c->nloc > 0 ? c->nloc : 1;
  // many waves: the scheduler's dynamic CTA placement already hides the quantisation and shorter CTAs only add prologues
  // (measured at 1 / 2 GPUs, 16.6 / 8.3 waves: 236 rows cost +1.4 % / +0.7 %); few waves: the empty tail is real (4 GPUs: -2 %)
  if (gx * ((nloc + ST_RB - 1) / ST_RB) > 6ll * slots) return ST_RB;
  int best = ST_RB;
  long long best_cost = -1;
  for (int rb = ST_RB; rb >= ST_RB_MIN; rb -= ST_UNROLL) {
    const long long ctas = gx * ((nloc + rb - 1) / rb);
    const long long waves = (ctas + slots - 1) / slots;
    const long long cost = waves * (rb + 6);   // + the CTA's prologue / epilogue, in row equivalents
    if (best_cost < 0 || cost < best_cost) { best_cost = cost; best = rb; }
  }
  return best;
}
static dim3 stream_grid(const Ctx *c) {
  const int rb = stream_rows_per_cta(c);
  return dim3((c->M + ST_CTA_COLS - 1) / ST_CTA_COLS, (c->nloc + rb - 1) / rb);
}
int stream_num_parts(const Ctx *c) {   // upper bound over every admissible CTA height (sizes d_part_stats)
  return (int)(((c->M + ST_CTA_COLS - 1) / ST_CTA_COLS) * ((c->nloc + ST_RB_MIN - 1) / ST_RB_MIN));
}
static int stream_num_parts_now(const Ctx *c) {
  dim3 g = stream_grid(c);
  return (int)(g.x * g.y);
}

cudaError_t launch_stream_prep(Ctx *c, const CostParams &cp, int for_km_gate) {
  const bool bsc = c->cfg.feature_type == GHICP_FT_BSC;
  // The filter works in a domain scaled by kappa = half(WFD)/WFD (|kappa - 1| <= 2^-11) so that the feature
  // weight is exactly representable in fp16 and cd32 = fmaf(fd, w_h, dist): argmin and threshold tests are
  // invariant under the positive scaling; sums are scaled back in k_finalize_fast.
  double kappa = 1.0;
  c->x2_ok = true;
  c->b_eff = 0.f;
  if (bsc) {
    const __half wh = __float2half_rn((float)cp.WFD);
    const float whf = __half2float(wh);
    if (cp.WFD >= 6.2e-5 && whf > 0.f) {
      kappa = (double)whf / cp.WFD;
      c->b_eff = whf;
    } else {           // weight below the fp16 normal range: scalar FFMA path with the float weight
      c->x2_ok = false;
      c->b_eff = (float)cp.WFD;
    }
  }
  c->kappa = kappa;
  const double a = (bsc ? cp.scale * cp.WED : cp.scale) * kappa;
  const double A = a * a;
  const double b = bsc ? (double)c->b_eff : 0.0;
  const int n = c->N > c->M ? c->N : c->M;
  cudaMemsetAsync(&c->d_sdev->r2max_bits, 0, sizeof(unsigned), c->stream);
  GHICP_LAUNCH(k_prep, (n + 255) / 256, 256, 0, c->stream, c->d_s, c->d_t, c->N, c->M, c->center[0], c->center[1], c->center[2], A,
                                                 reinterpret_cast<float4 *>(c->d_S4), reinterpret_cast<float4 *>(c->d_T4),
                                                 c->d_sdev);
  GHICP_LAUNCH(k_margin, 1, 1, 0, c->stream, c->d_sdev, A, a, b, (double)c->bits, c->d_iter, for_km_gate, 1e-5, kappa);
  c->launches += 2;
  return cudaGetLastError();
}
// refresh only the KM superset threshold (penalty has been (re)computed on the device)
cudaError_t launch_stream_gate(Ctx *c, const CostParams &cp) {
  const bool bsc = c->cfg.feature_type == GHICP_FT_BSC;
  const double a = (bsc ? cp.scale * cp.WED : cp.scale) * c->kappa;
  GHICP_LAUNCH(k_margin, 1, 1, 0, c->stream, c->d_sdev, a * a, a, bsc ? (double)c->b_eff : 0.0, (double)c->bits, c->d_iter, 1, 1e-5,
                                   c->kappa);
  c->launches++;
  return cudaGetLastError();
}

cudaError_t launch_stream_seed(Ctx *c, const CostParams &cp, bool with_cols) {
  StreamArgs a = make_args(c, cp);
  if (with_cols) a.col_thr_init = c->d_col_thr;
  const int n = c->N > c->M ? c->N : c->M;
  // sharded NNR: a column is seeded from this rank's OWN best row of the last iteration (its slice of the gathered per-rank
  // column minima), not from the merged winner, which mostly lives on another rank and would leave the column unseeded
  const int *prev_cols = (c->world > 1 && c->d_colg_idx) ? c->d_colg_idx + (size_t)c->rank * (size_t)c->M : c->d_col_idx;
  GHICP_LAUNCH(k_seed, (n + 255) / 256, 256, 0, c->stream, a, c->d_row_idx, prev_cols, c->have_prev ? 1 : 0);
  c->launches++;
  return cudaGetLastError();
}

// stats: accumulate sum / sumsq of CD
cudaError_t launch_stream(Ctx *c, const CostParams &cp, StreamMode mode, bool stats) {
  StreamArgs a = make_args(c, cp);
  if (mode == SM_NNR || mode == SM_PRE_COLS) a.col_thr_init = c->d_col_thr;
  const dim3 grid = stream_grid(c);
  const bool fd = a.fd != nullptr;
#if defined(GHICP_EMU_HOST)
#define GHICP_STREAM_OPT_IN_SMEM(kernel) (void)0
#else
#define GHICP_STREAM_OPT_IN_SMEM(kernel) cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, ST_DYN_SMEM)
#endif
#define LAUNCH_FD(MODE, ST, HB)                                                                                \
  do {                                                                                                         \
    if (c->x2_ok) {                                                                                            \
      GHICP_STREAM_OPT_IN_SMEM((k_stream<MODE, true, ST, HB, true>));                                          \
      GHICP_LAUNCH((k_stream<MODE, true, ST, HB, true>), grid, ST_THREADS, ST_DYN_SMEM, c->stream, a);         \
    } else {                                                                                                   \
      GHICP_STREAM_OPT_IN_SMEM((k_stream<MODE, true, ST, HB, false>));                                         \
      GHICP_LAUNCH((k_stream<MODE, true, ST, HB, false>), grid, ST_THREADS, ST_DYN_SMEM, c->stream, a);        \
    }                                                                                                          \
  } while (0)
#define LAUNCH(MODE, FD, ST)                                                                                   \
  do {                                                                                                         \
    if (FD) {                                                                                                  \
      if (a.fd_hb == 1) LAUNCH_FD(MODE, ST, 1);                                                                \
      else if (a.fd_hb == 2) LAUNCH_FD(MODE, ST, 2);                                                           \
      else LAUNCH_FD(MODE, ST, 4);                                                                             \
    } else if (c->x2_ok) {                                                                                     \
      GHICP_LAUNCH((k_stream<MODE, false, ST, 1, true>), grid, ST_THREADS, 0, c->stream, a);                   \
    } else {                                                                                                   \
      GHICP_LAUNCH((k_stream<MODE, false, ST, 1, false>), grid, ST_THREADS, 0, c->stream, a);                  \
    }                                                                                                          \
  } while (0)
#define PICK(MODE)                                      \
  do {                                                  \
    if (fd) { if (stats) LAUNCH(MODE, true, true); else LAUNCH(MODE, true, false); }   \
    else    { if (stats) LAUNCH(MODE, false, true); else LAUNCH(MODE, false, false); } \
  } while (0)
  switch (mode) {
    case SM_NN: PICK(SM_NN); break;
    case SM_NNR: PICK(SM_NNR); break;
    case SM_COUNT: PICK(SM_COUNT); break;
    case SM_PRE: PICK(SM_PRE); break;
    case SM_PRE_COLS: PICK(SM_PRE_COLS); break;
    default:
      if (fd) LAUNCH(SM_FILL, true, false); else LAUNCH(SM_FILL, false, false);
      break;
  }
#undef PICK
#undef LAUNCH
#undef LAUNCH_FD
  c->launches++;
  return cudaGetLastError();
}

cudaError_t launch_stream_resolve(Ctx *c, const CostParams &cp, bool with_cols) {
  StreamArgs a = make_args(c, cp);
  GHICP_LAUNCH(k_resolve, GHICP_SMS * 4, 256, 0, c->stream, a, 0);
  if (with_cols) GHICP_LAUNCH(k_resolve, GHICP_SMS * 4, 256, 0, c->stream, a, 1);
  const int n = c->N > c->M ? c->N : c->M;
  GHICP_LAUNCH(k_publish, (n + 255) / 256, 256, 0, c->stream, a, c->d_row_cd, c->d_row_idx, with_cols ? c->d_col_cd : nullptr,
                                                    with_cols ? c->d_col_idx : nullptr, c->d_xstats, c->rank);
  c->launches += with_cols ? 3 : 2;
  return cudaGetLastError();
}

cudaError_t launch_finalize_fast(Ctx *c) {
  GHICP_LAUNCH(k_finalize_fast, 1, 1024, 0, c->stream, c->d_part_stats, stream_num_parts_now(c), c->d_xstats, c->rank, c->kappa,
               c->d_sdev);
  c->launches++;
  return cudaGetLastError();
}
cudaError_t launch_penalty_only(Ctx *c, const LoopScalars &ls) {
  GHICP_LAUNCH(k_penalty_only, 1, 1, 0, c->stream, ls, c->d_iter);
  c->launches++;
  return cudaGetLastError();
}
// NNR with sharded rows: per-rank column minima (ordered-double bits, row index) gathered as [world][M];
// keep the lexicographic minimum (ranks own ascending row ranges, so equal values keep the smaller row).
__global__ void k_colmerge(const unsigned long long *__restrict__ g_cd, const int *__restrict__ g_idx, int world, int M,
                           double *__restrict__ col_cd, int *__restrict__ col_idx) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= M) return;
  unsigned long long best = g_cd[j];
  int bi = g_idx[j];
  for (int r = 1; r < world; ++r) {
    const unsigned long long v = g_cd[(size_t)r * M + j];
    const int i = g_idx[(size_t)r * M + j];
    if (v < best || (v == best && i < bi)) { best = v; bi = i; }
  }
  col_cd[j] = __longlong_as_double((long long)best);
  col_idx[j] = bi;
}
cudaError_t launch_colmerge(Ctx *c) {
  GHICP_LAUNCH(k_colmerge, (c->M + 255) / 256, 256, 0, c->stream, c->d_colg_cd, c->d_colg_idx, c->world, c->M, c->d_col_cd, c->d_col_idx);
  c->launches++;
  return cudaGetLastError();
}
__global__ void k_count_valid(const double *__restrict__ gain, long long nnz, StreamDev *dev) {
  long long k = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  int v = 0;
  for (; k < nnz; k += (long long)gridDim.x * blockDim.x) v += gain[k] > 0.0 ? 1 : 0;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0 && v) atomicAdd(&dev->nnz_valid, (unsigned long long)v);
}
cudaError_t launch_count_valid(Ctx *c, long long nnz) {
  cudaMemsetAsync(&c->d_sdev->nnz_valid, 0, sizeof(unsigned long long), c->stream);
  GHICP_LAUNCH(k_count_valid, GHICP_SMS * 4, 256, 0, c->stream, c->d_csr_gain, nnz, c->d_sdev);
  c->launches++;
  return cudaGetLastError();
}
cudaError_t launch_scan_rows(Ctx *c) {
  return launch_scan_i32(c, c->d_cnt, c->d_rowptr, c->d_cursor, c->N, &c->d_iter->nnz);
}
cudaError_t launch_emit_scatter(Ctx *c, const CostParams &cp, unsigned long long n_emitted) {
  StreamArgs a = make_args(c, cp);
  const unsigned long long want = (n_emitted + 255) / 256;
  const int blocks = (int)std::min<unsigned long long>(std::max<unsigned long long>(want, 1), (unsigned long long)GHICP_SMS * 8);
  GHICP_LAUNCH(k_emit_scatter, blocks, 256, 0, c->stream, a, n_emitted);
  c->launches++;
  return cudaGetLastError();
}
cudaError_t launch_csr_check(Ctx *c, const CostParams &cp) {
  StreamArgs a = make_args(c, cp);
  GHICP_LAUNCH(k_csr_check, GHICP_SMS * 4, 256, 0, c->stream, a, c->d_iter, c->d_csr_gain);
  c->launches++;
  return cudaGetLastError();
}


// ---- settled KM iteration (see the kernels above) -------------------------------------------------------------------
size_t xblock_bytes(size_t xcap) { return sizeof(XBlockHdr) + xcap * (sizeof(unsigned long long) + sizeof(double) + sizeof(float)); }
cudaError_t launch_emit_check(Ctx *c, const CostParams &cp) {
  StreamArgs a = make_args(c, cp);
  unsigned char *blk = c->d_xsend;
  XBlockHdr *hdr = reinterpret_cast<XBlockHdr *>(blk);
  unsigned long long *key = reinterpret_cast<unsigned long long *>(hdr + 1);
  double *gain = reinterpret_cast<double *>(key + c->xuse);
  float *fd = reinterpret_cast<float *>(gain + c->xuse);
  GHICP_LAUNCH(k_emit_check, GHICP_SMS * 2, 256, 0, c->stream, a, c->d_iter, c->d_xstats + 4 * c->rank, hdr, key, gain, fd,
               (unsigned long long)c->xuse);
  c->launches++;
  return cudaGetLastError();
}
// gathered blocks -> d_xstats, CSR (d_rowptr / d_csr_*), DevIter::nnz, StreamDev::nnz_valid; no host involvement
cudaError_t launch_xbuild(Ctx *c) {
  const unsigned char *blocks = c->world > 1 ? c->d_xrecv : c->d_xsend;
  const size_t bb = xblock_bytes(c->xuse);
  cudaMemsetAsync(c->d_cnt, 0, sizeof(int) * ((size_t)c->Npad + 2), c->stream);
  cudaMemsetAsync(&c->d_sdev->nnz_valid, 0, sizeof(unsigned long long), c->stream);
  const dim3 grid(32, c->world);
  GHICP_LAUNCH(k_xcount, grid, 256, 0, c->stream, blocks, bb, (unsigned long long)c->xuse, c->d_cnt, c->d_xstats, c->d_xcounts);
  c->launches++;
  cudaError_t e = launch_scan_rows(c);
  if (e != cudaSuccess) return e;
  GHICP_LAUNCH(k_xscatter, grid, 256, 0, c->stream, blocks, bb, (unsigned long long)c->xuse, c->d_rowptr, c->d_cursor, c->d_csr_col,
               c->d_csr_gain, c->d_csr_fd, c->d_sdev);
  c->launches++;
  return cudaGetLastError();
}

}  // namespace ghicp_b200
