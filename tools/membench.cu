// membench.cu — read-bandwidth ceilings for the access patterns k_stream can use on the FD plane.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o membench membench.cu && ./membench
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
#define CK(x) do{cudaError_t e=(x); if(e!=cudaSuccess){printf("%s: %s\n",#x,cudaGetErrorString(e)); return 1;}}while(0)

__global__ void k_linear(const uint4* p, size_t n, unsigned* out) {
  unsigned acc = 0;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
  for (; i + 3 * stride < n; i += 4 * stride) {
    uint4 a = p[i], b = p[i + stride], c = p[i + 2 * stride], d = p[i + 3 * stride];
    acc ^= a.x ^ b.y ^ c.z ^ d.w;
  }
  if (acc == 0x12345678u) out[0] = acc;
}
// per-warp sequential streams: warp w reads region [w*region, (w+1)*region) 512 B per step (like a panel)
template <int UNROLL>
__global__ void k_warpstream(const uint4* p, size_t region_u4, int nregions, unsigned* out) {
  const int lane = threadIdx.x & 31;
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  unsigned acc = 0;
  for (int r = gw; r < nregions; r += nw) {
    const uint4* q = p + (size_t)r * region_u4 + lane;
    for (size_t k = 0; k + 32 * UNROLL <= region_u4; k += 32 * UNROLL) {
      uint4 v[UNROLL];
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) v[u] = q[k + 32 * u];
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) acc ^= v[u].x ^ v[u].w;
    }
  }
  if (acc == 0x12345678u) out[0] = acc;
}
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
// per-warp TMA bulk ring: STAGE bytes per copy
template <int STAGE, int NST>
__global__ void k_tma(const unsigned char* p, size_t region_bytes, int nregions, unsigned* out) {
  extern __shared__ __align__(128) unsigned char ring[];
  __shared__ unsigned long long bar[32][NST];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  const int gw = blockIdx.x * wpb + warp, nw = gridDim.x * wpb;
  unsigned char* my = ring + (size_t)warp * NST * STAGE;
  if (lane == 0) { for (int s = 0; s < NST; ++s) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(smem_u32(&bar[warp][s]))); asm volatile("fence.mbarrier_init.release.cluster;"); }
  __syncthreads();
  unsigned acc = 0; unsigned phase_bits = 0; int it = 0;
  for (int r = gw; r < nregions; r += nw) {
    const unsigned char* src = p + (size_t)r * region_bytes;
    const int nb = (int)(region_bytes / STAGE);
    auto issue = [&](int k) { int s = (it + k) % NST; asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(&bar[warp][s])), "r"(STAGE) : "memory");
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" :: "r"(smem_u32(my + s * STAGE)), "l"(src + (size_t)k * STAGE), "r"(STAGE), "r"(smem_u32(&bar[warp][s])) : "memory"); };
    if (lane == 0) for (int k = 0; k < NST && k < nb; ++k) issue(k);
    for (int k = 0; k < nb; ++k) {
      int s = (it + k) % NST; unsigned par = (phase_bits >> s) & 1; unsigned ok;
      do { asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0,1,0,p; }" : "=r"(ok) : "r"(smem_u32(&bar[warp][s])), "r"(par) : "memory"); } while (!ok);
      phase_bits ^= (1u << s);
      for (int o = lane * 16; o < STAGE; o += 512) { uint4 v = *reinterpret_cast<const uint4*>(my + s * STAGE + o); acc ^= v.x ^ v.w; }
      __syncwarp();
      if (lane == 0 && k + NST < nb) { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); issue(k + NST); }
    }
    it += nb;
  }
  if (acc == 0x12345678u) out[0] = acc;
}
template <typename F> float timeit(F f, int rep = 5) {
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b); f(); cudaDeviceSynchronize();
  float best = 1e9; for (int i = 0; i < rep; ++i) { cudaEventRecord(a); f(); cudaEventRecord(b); cudaEventSynchronize(b); float ms; cudaEventElapsedTime(&ms, a, b); best = ms < best ? ms : best; }
  return best;
}
int main() {
  const size_t bytes = 5ull << 30; unsigned char* d; unsigned* out;
  CK(cudaMalloc(&d, bytes)); CK(cudaMalloc(&out, 4)); CK(cudaMemset(d, 1, bytes));
  const size_t n16 = bytes / 16;
  float ms = timeit([&] { k_linear<<<132 * 8, 256>>>((const uint4*)d, n16, out); });
  printf("linear grid-stride uint4 x4           : %.3f ms  %.0f GB/s\n", ms, bytes / ms / 1e6);
  const size_t region = 128 * 1024;  // 256 rows x 512 B, like one warp's sweep of a panel
  const int nregions = (int)(bytes / region);
  ms = timeit([&] { k_warpstream<4><<<132 * 2, 256>>>((const uint4*)d, region / 16, nregions, out); });
  printf("per-warp 128KB streams, LDG x4, 16w/SM: %.3f ms  %.0f GB/s\n", ms, bytes / ms / 1e6);
  ms = timeit([&] { k_warpstream<8><<<132 * 2, 256>>>((const uint4*)d, region / 16, nregions, out); });
  printf("per-warp 128KB streams, LDG x8, 16w/SM: %.3f ms  %.0f GB/s\n", ms, bytes / ms / 1e6);
  ms = timeit([&] { k_warpstream<8><<<132 * 4, 256>>>((const uint4*)d, region / 16, nregions, out); });
  printf("per-warp 128KB streams, LDG x8, 32w/SM: %.3f ms  %.0f GB/s\n", ms, bytes / ms / 1e6);
  cudaFuncSetAttribute(k_tma<2048, 6>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * 6 * 2048);
  ms = timeit([&] { k_tma<2048, 6><<<132 * 2, 256, 8 * 6 * 2048>>>(d, region, nregions, out); });
  printf("per-warp TMA bulk 2KB x6 stages, 16w/SM: %.3f ms  %.0f GB/s\n", ms, bytes / ms / 1e6);
  cudaFuncSetAttribute(k_tma<4096, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * 3 * 4096);
  ms = timeit([&] { k_tma<4096, 3><<<132 * 2, 256, 8 * 3 * 4096>>>(d, region, nregions, out); });
  printf("per-warp TMA bulk 4KB x3 stages, 16w/SM: %.3f ms  %.0f GB/s\n", ms, bytes / ms / 1e6);
  cudaFuncSetAttribute(k_tma<8192, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * 3 * 8192);
  ms = timeit([&] { k_tma<8192, 3><<<132 * 2, 128, 4 * 3 * 8192>>>(d, region, nregions, out); });
  printf("per-warp TMA bulk 8KB x3 stages,  8w/SM: %.3f ms  %.0f GB/s\n", ms, bytes / ms / 1e6);
  // strided 512 B segments (the old row-major plane): region = one segment, regions far apart
  ms = timeit([&] { k_warpstream<1><<<132 * 8, 256>>>((const uint4*)d, 32, (int)(bytes / 512), out); });
  printf("per-warp 512B segments round-robin     : %.3f ms  %.0f GB/s\n", ms, bytes / ms / 1e6);
  return 0;
}
