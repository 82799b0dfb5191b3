// The three approximate MUFU instructions of the FP32 correspondence filters against float64, on the device.
//   sqrt.approx.ftz.f32: every positive normal float32 (relative error; subnormal inputs are flushed, counted apart)
//   lg2.approx.ftz.f32 : every float32 in [1e-30, 1 + 2^-10] (absolute error, and absolute error / (1 + |log2 x|)): fd32
//                        and fd32 + FF_G of ghicp_fpfh.cu
//   ex2.approx.ftz.f32 : every float32 in [-2^-10, 100] (relative error): -ex * lg2(fd32) and -lg2(fd32), ex in (0, 1]
// Prints one line: "sqrt_rel <x> lg2_abs <x> lg2_model <x> ex2_rel <x> sqrt_sub_nonzero <n>".
#include <cmath>
#include <cstdio>
#include <cstring>

__device__ unsigned long long g_max[4];   // sqrt rel, lg2 abs, ex2 rel, lg2 abs / (1 + |log2 x|)
__device__ unsigned long long g_sub_nonzero;

__device__ __forceinline__ void note(int k, double e) {   // non-negative doubles order like their bits
  atomicMax(&g_max[k], (unsigned long long)__double_as_longlong(e));
}

__global__ void k_sweep(unsigned lo, unsigned hi, int op) {
  double worst = 0.0, worst_model = 0.0;
  unsigned long long subnz = 0;
  for (unsigned long long b = lo + (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; b <= hi;
       b += (unsigned long long)gridDim.x * blockDim.x) {
    const float x = __uint_as_float((unsigned)b);
    float r;
    if (op == 0) {
      asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
      if (fabsf(x) < 1.17549435e-38f) { subnz += r != 0.f; continue; }
      const double t = sqrt((double)x);
      worst = fmax(worst, fabs((double)r - t) / t);
    } else if (op == 1) {
      asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
      const double t = log2((double)x);
      worst = fmax(worst, fabs((double)r - t));
      worst_model = fmax(worst_model, fabs((double)r - t) / (1.0 + fabs(t)));
    } else {
      asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
      const double t = exp2((double)x);
      worst = fmax(worst, fabs((double)r - t) / t);
    }
  }
  note(op, worst);
  if (op == 1) note(3, worst_model);
  if (subnz) atomicAdd(&g_sub_nonzero, subnz);
}

static unsigned bits(float f) { unsigned u; std::memcpy(&u, &f, 4); return u; }

int main() {
  unsigned long long zero[4] = {0, 0, 0, 0}, z = 0;
  cudaMemcpyToSymbol(g_max, zero, sizeof(zero));
  cudaMemcpyToSymbol(g_sub_nonzero, &z, sizeof(z));
  k_sweep<<<132 * 16, 256>>>(1u, 0x7f7fffffu, 0);                              // every positive finite float32
  k_sweep<<<132 * 16, 256>>>(bits(1e-30f), bits(1.0f + 0x1p-10f), 1);
  k_sweep<<<132 * 16, 256>>>(0u, bits(100.0f), 2);                              // [0, 100]
  k_sweep<<<132 * 16, 256>>>(0x80000000u, bits(-0x1p-10f), 2);                 // [-2^-10, -0]
  unsigned long long out[4], sub;
  if (cudaMemcpyFromSymbol(out, g_max, sizeof(out)) != cudaSuccess ||
      cudaMemcpyFromSymbol(&sub, g_sub_nonzero, sizeof(sub)) != cudaSuccess) {
    std::fprintf(stderr, "CUDA error: %s\n", cudaGetErrorString(cudaGetLastError()));
    return 1;
  }
  double e[4];
  std::memcpy(e, out, sizeof(e));
  std::printf("sqrt_rel %.9e lg2_abs %.9e lg2_model %.9e ex2_rel %.9e sqrt_sub_nonzero %llu\n", e[0], e[1], e[3], e[2], sub);
  return 0;
}
