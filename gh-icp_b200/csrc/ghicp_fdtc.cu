// ghicp_fdtc.cu — one-time BSC feature-distance build on the Hopper tensor cores (wgmma, integer kind).
//
// calFD_BSC (src/ghicp_reg.cpp:143-200): FD[i][j] = min_v Hamming(bscS[v][i], bscT[0][j]).
// With descriptor bits mapped to +/-1 int8 (padding = 0) the Hamming distance is an integer GEMM:
//      dot(a, b) = (#equal bits) - (#different bits) = bits - 2 * Hamming   =>   Hamming = (bits - dot) / 2
// exactly (int32 accumulation of +/-1 products).  One CTA keeps a B tile = TN (source, variant) rows resident in shared
// memory and streams 64-row target tiles (A) through a ring of K-chunk stages (cp.async.bulk, one mbarrier per stage).
// Two consumer warpgroups each own half of the B tile's columns and issue wgmma.mma_async m64n32k32.s32.s8.s8 from shared
// memory into register accumulators; after a tile's last K-chunk they take the min over the V variants (adjacent
// accumulator columns: in-thread pairs, plus one lane shuffle for V = 4) and store into the packed panel-major FD plane (ghicp_internal.h: fd_at).
// Operands sit in shared memory in the canonical K-major no-swizzle layout [k-chunk(16 B)][row][16 B]
// (8-row x 16-byte core matrices back to back: SBO = 128 B between row groups, LBO = rows * 16 B between k-chunks).
#include <cstdlib>
#include <cuda_fp16.h>

#include "ghicp_internal.h"

namespace ghicp_b200 {

namespace {

constexpr int TC_TM = 64;         // target rows per A tile (wgmma M)
constexpr int TC_NCH = 32;        // B columns per wgmma instruction (N)
constexpr int TC_CONSUMERS = 2;   // warpgroups; each owns TN / 2 columns of the B tile
constexpr int TC_THREADS = TC_CONSUMERS * 128 + 32;   // + one producer warp
constexpr int KC_BYTES = 128;     // K bytes per row and ring stage (4 wgmma K-steps)
constexpr int KC_STAGES = 4;

#if !defined(GHICP_EMU_HOST)
__device__ __forceinline__ unsigned smem_u32(const void *p) { return (unsigned)__cvta_generic_to_shared(p); }
#endif

// bits -> +/-1 int8, written directly in the TILE-CANONICAL layout the MMA reads from shared memory:
//   out[tile][k-chunk (16 B)][R rows][16 B]      (R = rows per tile; padding rows / bits are 0)
// so that a whole operand tile is ONE contiguous block = one cp.async.bulk.  Logical row = (i - i0) * V + v.
// words: [Vw][W64][n] word-major planes.
__global__ void k_unpack_pm1(const uint64_t *__restrict__ words, int V, int n, int W64, int bits, int KP, int R,
                             int i0, int n_rows_logical, int8_t *__restrict__ out) {
  const int chunks = KP / 16;
  const int n_tiles = (n_rows_logical + R - 1) / R;
  const long long total = (long long)n_tiles * R * chunks;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int r = (int)(idx % R);
  const int c = (int)((idx / R) % chunks);
  const int tile = (int)(idx / ((long long)R * chunks));
  const long long row = (long long)tile * R + r;
  uint32_t o[4] = {0, 0, 0, 0};
  if (row < n_rows_logical) {
    const int i = i0 + (int)(row / V), v = (int)(row % V);
    const int k0 = c * 16;
    const int w = k0 >> 6;
    const uint64_t word = (w < W64) ? words[((size_t)v * W64 + w) * n + i] : 0ull;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      uint32_t pack = 0;
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        const int k = k0 + q * 4 + b;
        int8_t val = 0;
        if (k < bits) val = ((word >> (k & 63)) & 1ull) ? 1 : -1;
        pack |= (uint32_t)(uint8_t)val << (8 * b);
      }
      o[q] = pack;
    }
  }
  *reinterpret_cast<uint4 *>(out + idx * 16) = make_uint4(o[0], o[1], o[2], o[3]);
}

#if defined(GHICP_EMU_HOST)
// Host emulation (tests/harness/cuda_emu): mbarriers and bulk copies as in emu_mbarrier.h; one wgmma m64n32k32 s8 is, for
// the calling thread, the 16 accumulator elements of its fragment computed from the two no-swizzle K-major tiles (the
// layout k_unpack_pm1 writes), so the fragment mapping of the epilogue is exercised as on the device.
__device__ __forceinline__ void mbar_init1(unsigned long long *b, int count) { emu::bar_init(b, count); }
__device__ __forceinline__ void mbar_wait_parity(unsigned long long *b, unsigned parity) { emu::bar_wait(b, parity); }
__device__ __forceinline__ void mbar_arrive(unsigned long long *b) { emu::bar_arrive(b); }
__device__ __forceinline__ void bulk_load(void *dst, const void *src, unsigned bytes, unsigned long long *bar) {
  emu::bar_arrive_expect_tx(bar, bytes);
  emu::bulk_copy(dst, src, bytes, bar);
}
// A: first 16-byte k-chunk of this K = 32 step of the 64-row stage (k-chunks TC_TM * 16 bytes apart); B: first k-chunk of the
// step at the instruction's first column (k-chunks TN * 16 bytes apart)
inline void emu_wgmma_s8(int d[16], const unsigned char *A, const unsigned char *B, int TN, bool accumulate) {
  const int tid = (int)(emu::cur()->tidx.x & 127), warp = tid >> 5, lane = tid & 31;
  for (int e = 0; e < 16; ++e) {
    const int m = warp * 16 + (lane >> 2) + 8 * ((e >> 1) & 1);
    const int n = 8 * (e >> 2) + 2 * (lane & 3) + (e & 1);
    int acc = accumulate ? d[e] : 0;
    for (int kk = 0; kk < 32; ++kk)
      acc += (int)(signed char)A[(size_t)(kk >> 4) * TC_TM * 16 + (size_t)m * 16 + (kk & 15)] *
             (int)(signed char)B[(size_t)(kk >> 4) * TN * 16 + (size_t)n * 16 + (kk & 15)];
    d[e] = acc;
  }
}
#else
__device__ __forceinline__ void mbar_init1(unsigned long long *b, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(b)), "r"(count));
}
__device__ __forceinline__ void mbar_wait_parity(unsigned long long *b, unsigned parity) {
  unsigned ok;
  do {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(smem_u32(b)), "r"(parity) : "memory");
  } while (!ok);
}
__device__ __forceinline__ void mbar_arrive(unsigned long long *b) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(b)) : "memory");
}
// One logical tile copy = several bulk copies of at most 4 KB in flight (a single large cp.async.bulk is serviced with little
// memory-level parallelism), all completing on one mbarrier.
__device__ __forceinline__ void bulk_load(void *dst, const void *src, unsigned bytes, unsigned long long *bar) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
  constexpr unsigned PIECE = 4096;
  for (unsigned off = 0; off < bytes; off += PIECE) {
    const unsigned n = (bytes - off < PIECE) ? (bytes - off) : PIECE;
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32((unsigned char *)dst + off)), "l"((const unsigned char *)src + off), "r"(n), "r"(smem_u32(bar)) : "memory");
  }
}

__device__ __forceinline__ uint64_t make_desc(unsigned smem_addr, unsigned lbo_bytes, unsigned sbo_bytes) {
  // SM90 shared-memory matrix descriptor: start address [0,14) (>>4), leading byte offset [16,30) (>>4),
  // stride byte offset [32,46) (>>4), base offset [49,52) = 0, layout type [62,64) = 0 (no swizzle)
  return (uint64_t)((smem_addr >> 4) & 0x3FFFu) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16) |
         ((uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32);
}

__device__ __forceinline__ void wgmma_s8(int d[16], uint64_t adesc, uint64_t bdesc, unsigned accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k32.s32.s8.s8 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p;\n\t}\n"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]),
        "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
#endif

// keeps the compiler from moving accumulator registers across the asynchronous MMA window
template <int NC>
__device__ __forceinline__ void fence_acc(int (&acc)[NC][16]) {
#if !defined(GHICP_EMU_HOST)
#pragma unroll
  for (int c = 0; c < NC; ++c)
#pragma unroll
    for (int e = 0; e < 16; ++e) asm volatile("" : "+r"(acc[c][e])::"memory");
#else
  (void)acc;
#endif
}

// B tile: TN (source, variant) rows x KP bytes, resident.  A tiles: TC_TM target rows, streamed in K-chunks of KC_BYTES through
// KC_STAGES ring stages (warp 8 loads; every consumer warp hands a stage back on its `empty` barrier once its MMAs retired).
template <int V, int TN, int HB>
__global__ void __launch_bounds__(TC_THREADS, 1)
k_fd_bsc_tc(const int8_t *__restrict__ T8c, const int8_t *__restrict__ S8c, unsigned char *__restrict__ fdq, int M,
            size_t fd_rows, int row0, int nloc, int bits, int KP) {
#if defined(GHICP_EMU_HOST)
  unsigned char *smem = reinterpret_cast<unsigned char *>(emu::dyn_smem());   // host emulation: the launch's dynamic shared memory
#else
  extern __shared__ __align__(128) unsigned char smem[];
#endif
  // barriers: full[KC_STAGES] stage landed, empty[KC_STAGES] stage consumed, [2 * KC_STAGES] B tile landed
  __shared__ __align__(8) unsigned long long s_bar[2 * KC_STAGES + 1];
  constexpr int NC = TN / TC_CONSUMERS / TC_NCH;    // wgmma instructions per K-step and warpgroup
  constexpr int SRC_PER_TILE = TN / V;
  constexpr unsigned STAGE_BYTES = (unsigned)TC_TM * KC_BYTES;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const unsigned b_bytes = (unsigned)TN * KP, a_bytes = (unsigned)TC_TM * KP;
  unsigned char *Bs = smem;
  unsigned char *ring = smem + b_bytes;
  const int src_base = row0 + blockIdx.x * SRC_PER_TILE;   // first source row of this CTA's B tile
  const int n_ttiles = (M + TC_TM - 1) / TC_TM;
  const int n_kc = (KP + KC_BYTES - 1) / KC_BYTES;

  if (tid == 0) {
    for (int s = 0; s < KC_STAGES; ++s) {
      mbar_init1(&s_bar[s], 1);
      mbar_init1(&s_bar[KC_STAGES + s], TC_CONSUMERS * 4);
    }
    mbar_init1(&s_bar[2 * KC_STAGES], 1);
#if !defined(GHICP_EMU_HOST)
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
#endif
  }
  __syncthreads();

  if (warp == TC_CONSUMERS * 4) {
    // ===== producer (one thread) =====
    if (lane == 0) {
      bulk_load(Bs, S8c + (size_t)blockIdx.x * b_bytes, b_bytes, &s_bar[2 * KC_STAGES]);
      const long long n_chunks = (long long)n_ttiles * n_kc;
      for (long long g = 0; g < n_chunks; ++g) {
        const int st = (int)(g % KC_STAGES);
        const int t = (int)(g / n_kc), kc = (int)(g % n_kc);
        if (g >= KC_STAGES) mbar_wait_parity(&s_bar[KC_STAGES + st], (unsigned)(((g / KC_STAGES) - 1) & 1));
        const int kb = min(KC_BYTES, KP - kc * KC_BYTES);   // K bytes of this chunk (a multiple of 32)
        bulk_load(ring + (size_t)st * STAGE_BYTES, T8c + (size_t)t * a_bytes + (size_t)kc * KC_BYTES * TC_TM,
                  (unsigned)kb * TC_TM, &s_bar[st]);
      }
    }
    return;
  }

  // ===== consumer warpgroups: wgmma into registers, then min over variants -> packed FD plane =====
  const int wg = warp >> 2, wl = warp & 3;
  const int col0 = wg * (TN / TC_CONSUMERS);   // first B row (column of D) of this warpgroup
  int acc[NC][16];
#if !defined(GHICP_EMU_HOST)
  const unsigned b_addr = smem_u32(Bs), ring_addr = smem_u32(ring);
#endif
  mbar_wait_parity(&s_bar[2 * KC_STAGES], 0);   // B landed
  long long g = 0;
  for (int t = 0; t < n_ttiles; ++t) {
    for (int kc = 0; kc < n_kc; ++kc, ++g) {
      const int st = (int)(g % KC_STAGES);
      mbar_wait_parity(&s_bar[st], (unsigned)((g / KC_STAGES) & 1));
      const int ks = min(KC_BYTES, KP - kc * KC_BYTES) / 32;
#if defined(GHICP_EMU_HOST)
      for (int k = 0; k < ks; ++k) {
        const int kg = kc * (KC_BYTES / 32) + k;   // K-step index inside the B tile
        for (int c = 0; c < NC; ++c)
          emu_wgmma_s8(acc[c], ring + (size_t)st * STAGE_BYTES + (size_t)k * 2 * TC_TM * 16,
                       Bs + (size_t)kg * 2 * TN * 16 + (size_t)(col0 + c * TC_NCH) * 16, TN, kc > 0 || k > 0);
      }
#else
      fence_acc(acc);
      asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
      for (int k = 0; k < ks; ++k) {
        const int kg = kc * (KC_BYTES / 32) + k;
        const uint64_t adesc = make_desc(ring_addr + (unsigned)st * STAGE_BYTES + (unsigned)k * 2u * TC_TM * 16u, TC_TM * 16u, 128u);
        const unsigned accumulate = (kc > 0 || k > 0) ? 1u : 0u;
#pragma unroll
        for (int c = 0; c < NC; ++c) {
          const uint64_t bdesc = make_desc(b_addr + (unsigned)kg * 2u * TN * 16u + (unsigned)(col0 + c * TC_NCH) * 16u, TN * 16u, 128u);
          wgmma_s8(acc[c], adesc, bdesc, accumulate);
        }
      }
      asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
      asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
      fence_acc(acc);
#endif
      __syncwarp();                                          // every lane of the warp is past its reads of the stage
      if (lane == 0) mbar_arrive(&s_bar[KC_STAGES + st]);   // this warp's MMAs no longer read the stage
    }
    // epilogue.  Fragment of m64nNk32: element e of a thread sits at row 16 wl + lane / 4 + 8 ((e >> 1) & 1) and column
    // 8 (e >> 2) + 2 (lane & 3) + (e & 1) of its instruction's 32 columns.  For one (c, h) the warp's values cover 8 aligned
    // target columns (one lane of a panel) and, over q, 16 aligned source rows: with V = 2 each q is one whole quad block
    // (row (lane & 3)), with V = 4 two consecutive q are (rows 2 (q & 1) + (lane & 3) / 2, even lanes).  The low bytes go
    // straight to the plane, the high-bit words are OR-reduced over the warp and written by lane 0.
    constexpr int QPQ = (V == 4) ? 2 : 1;   // fragment steps per quad
    constexpr int QB = FD_LOW_BYTES + 128 * HB;
    const size_t panel_stride = fd_quads(fd_rows) * QB;
    const int irel0 = src_base - row0;        // a multiple of 4
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int j = t * TC_TM + wl * 16 + (lane >> 2) + 8 * h;   // target column of the FD plane
      const int jp = j & (FD_PANEL - 1), c8 = j & 7;
      unsigned char *pbase = fdq + (size_t)(j >> 8) * panel_stride;
      unsigned char *hbase = pbase + FD_LOW_BYTES + (jp >> 3) * 4;   // word 0 of lane 0's panel lane, quad 0
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        unsigned hw[HB];
#pragma unroll
        for (int w = 0; w < HB; ++w) hw[w] = 0u;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          int best = max(acc[c][q * 4 + h * 2], acc[c][q * 4 + h * 2 + 1]);   // max dot = min Hamming
          if (V == 4) best = max(best, __shfl_xor_sync(0xffffffffu, best, 1));  // the other two variants sit in lane ^ 1
          // source row of this value, relative to the plane: quad (col0 + 32 c + 8 q) / (4 V), row u in the quad
          const int irel = irel0 + (col0 + c * TC_NCH + 8 * q + 2 * (lane & 3)) / V;
          const int u = irel & 3;
          if (!(V == 4 && (lane & 1)) && j < M && irel < nloc) {
            const unsigned ham = (unsigned)((bits - best) >> 1);
            pbase[(size_t)(irel >> 2) * QB + u * FD_PANEL + jp] = (unsigned char)ham;
            const int wd = fd_hi_word(HB, u, c8);
            const unsigned part = fd_hi_part(HB, u, c8, ham);
#pragma unroll
            for (int w = 0; w < HB; ++w) hw[w] |= (w == wd) ? part : 0u;
          }
          if (q % QPQ == QPQ - 1) {
            const int iq = irel >> 2;   // the warp's quad (lane 0's row is in it)
#pragma unroll
            for (int w = 0; w < HB; ++w) {
              const unsigned word = fd_lanes_or<32>(hw[w]);
              if (lane == 0 && j < M && iq * 4 < nloc) *reinterpret_cast<unsigned *>(hbase + (size_t)iq * QB + w * 128) = word;
              hw[w] = 0u;
            }
          }
        }
      }
    }
  }
}

}  // namespace

#if defined(GHICP_EMU_HOST)
#define GHICP_TC_OPT_IN_SMEM(kernel) (void)0
#else
#define GHICP_TC_OPT_IN_SMEM(kernel) cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)
#endif
template <int V, int TN, int HB>
static cudaError_t launch_tc(Ctx *c, const int8_t *T8, const int8_t *S8, int KP, int grid, size_t smem) {
  GHICP_TC_OPT_IN_SMEM((k_fd_bsc_tc<V, TN, HB>));
  GHICP_LAUNCH((k_fd_bsc_tc<V, TN, HB>), grid, TC_THREADS, smem, c->stream, T8, S8, reinterpret_cast<unsigned char *>(c->d_fd16), c->M, c->fd_rows, c->r0, c->nloc,
               c->bits, KP);
  return cudaGetLastError();
}

template <int V>
static cudaError_t launch_tc_hb(Ctx *c, const int8_t *T8, const int8_t *S8, int KP, int grid, size_t smem, int TN, int hb) {
  if (hb == 1) return TN == 256 ? launch_tc<V, 256, 1>(c, T8, S8, KP, grid, smem) : TN == 128 ? launch_tc<V, 128, 1>(c, T8, S8, KP, grid, smem)
                                                                                  : launch_tc<V, 64, 1>(c, T8, S8, KP, grid, smem);
  if (hb == 2) return TN == 256 ? launch_tc<V, 256, 2>(c, T8, S8, KP, grid, smem) : TN == 128 ? launch_tc<V, 128, 2>(c, T8, S8, KP, grid, smem)
                                                                                  : launch_tc<V, 64, 2>(c, T8, S8, KP, grid, smem);
  return TN == 256 ? launch_tc<V, 256, 4>(c, T8, S8, KP, grid, smem) : TN == 128 ? launch_tc<V, 128, 4>(c, T8, S8, KP, grid, smem)
                                                                     : launch_tc<V, 64, 4>(c, T8, S8, KP, grid, smem);
}

// Returns cudaErrorNotSupported when the shape does not fit this kernel (caller falls back to k_fd_bsc).
cudaError_t launch_fd_bsc_tc(Ctx *c) {
  const int V = (c->cfg.dof == 6) ? 4 : 2;
  const int KP = (c->bits + 31) / 32 * 32;
  if (c->V < V || c->nloc <= 0) return cudaErrorNotSupported;
  // the B tile narrows (256 / 128 / 64 rows) until it and the A ring fit the 227 KB a block may opt in to
  const size_t smem_max = 227 * 1024 - 128;   // less the kernel's static barriers
  const size_t ring_bytes = (size_t)KC_STAGES * TC_TM * KC_BYTES;
  int TN = 0;
  for (int cand : {256, 128, 64})
    if ((size_t)cand * KP + ring_bytes <= smem_max) { TN = cand; break; }
  if (TN == 0) return cudaErrorNotSupported;
  const size_t smem = (size_t)TN * KP + ring_bytes;
  DevBuf<int8_t> T8, S8;
  const int src_per_tile = TN / V;
  const int grid = (c->nloc + src_per_tile - 1) / src_per_tile;
  const int n_ttiles = (c->M + TC_TM - 1) / TC_TM;
  const size_t t_bytes = (size_t)n_ttiles * TC_TM * KP, s_bytes = (size_t)grid * TN * KP;
  CUDA_TRY(T8.alloc(t_bytes, c->stream));
  CUDA_TRY(S8.alloc(s_bytes, c->stream));
  {
    const long long tot = (long long)(t_bytes / 16);
    GHICP_LAUNCH(k_unpack_pm1, (unsigned)((tot + 255) / 256), 256, 0, c->stream, c->d_bt, 1, c->M, c->W64, c->bits, KP, TC_TM, 0, c->M, T8.get());
    const long long tos = (long long)(s_bytes / 16);
    GHICP_LAUNCH(k_unpack_pm1, (unsigned)((tos + 255) / 256), 256, 0, c->stream, c->d_bs, V, c->N, c->W64, c->bits, KP, TN, c->r0,
                 c->nloc * V, S8.get());
    c->launches += 2;
  }
  // the high-bit count of the plane is a template parameter, so the epilogue's bit positions are shifts by constants
  const int hb = fd_hb(c->bits);
  cudaError_t e;
  if (V == 4) e = launch_tc_hb<4>(c, T8.get(), S8.get(), KP, grid, smem, TN, hb);
  else e = launch_tc_hb<2>(c, T8.get(), S8.get(), KP, grid, smem, TN, hb);
  c->launches++;
  return e;
}

}  // namespace ghicp_b200
