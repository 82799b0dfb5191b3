// cuda_runtime.h — HOST EMULATION SHIM (tests/harness/cuda_emu), found before the real CUDA header only by the
// kernel-logic harness builds (g++ -Itests/harness/cuda_emu -DGHICP_EMU_HOST).  It lets a .cu translation unit of
// the product compile as plain C++ and run its kernels on the CPU: every CUDA thread of a block is a ucontext fiber,
// __syncthreads() and the warp shuffles are rendezvous points between fibers (emu.h).  What this checks is the
// kernels' LOGIC (indexing, reductions, tie-breaks, arithmetic order) against the oracle without a GPU; code
// generation, memory ordering and performance are only checked by the -m gpu tests.  Test infrastructure only.
#pragma once
#include <math.h>
#include <stdlib.h>
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include "emu.h"
#include "emu_mbarrier.h"

#define __host__
#define __device__
#define __global__
#define __forceinline__ inline
#define __launch_bounds__(...)
#define __shared__ static
#define __align__(n) __attribute__((aligned(n)))

typedef int cudaError_t;
enum { cudaSuccess = 0, cudaErrorInvalidValue = 1, cudaErrorMemoryAllocation = 2, cudaErrorNotSupported = 801 };
typedef void *cudaStream_t;
typedef void *cudaEvent_t;
inline cudaError_t cudaGetLastError() { return cudaSuccess; }
enum cudaMemcpyKind { cudaMemcpyHostToDevice = 1, cudaMemcpyDeviceToHost = 2, cudaMemcpyDeviceToDevice = 3 };
enum cudaDeviceAttr { cudaDevAttrMultiProcessorCount = 16 };
inline cudaError_t cudaMemsetAsync(void *p, int v, size_t bytes, cudaStream_t) { memset(p, v, bytes); return cudaSuccess; }
inline cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t bytes, cudaMemcpyKind, cudaStream_t) { memmove(d, s, bytes); return cudaSuccess; }
inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaDeviceGetAttribute(int *v, cudaDeviceAttr, int) { *v = 2; return cudaSuccess; }   // "2 SMs": small cooperative grids
template <typename F> inline cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int *n, F, int, size_t) { *n = 1; return cudaSuccess; }
template <typename T> inline void __stcg(T *p, T v) { *p = v; }
// fresh "device" memory is POISONED (0xCD bytes: huge negative ints, -6.2e66 doubles): a kernel that reads what nobody wrote
// produces garbage here instead of the zeros a fresh page usually holds
inline void *emu_poisoned(size_t bytes) { void *q = malloc(bytes ? bytes : 1); if (q) memset(q, 0xCD, bytes ? bytes : 1); return q; }
// Test controls of the device allocations (tests/test_alloc_failures.py, through tests/harness/emu_library.cpp): the number of
// live ones, and a countdown that makes the k-th allocation from now fail (-1: none fails)
inline long long emu_live_allocs = 0;
inline long long emu_fail_countdown = -1;
inline void *emu_device_alloc(size_t bytes) {
  if (emu_fail_countdown >= 0 && emu_fail_countdown-- == 0) return nullptr;
  void *q = emu_poisoned(bytes);
  if (q) ++emu_live_allocs;
  return q;
}
inline void emu_device_free(void *p) {
  if (p) --emu_live_allocs;
  free(p);
}
template <typename T> inline cudaError_t cudaMallocAsync(T **p, size_t bytes, cudaStream_t) { *p = (T *)emu_device_alloc(bytes); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
inline cudaError_t cudaFreeAsync(void *p, cudaStream_t) { emu_device_free(p); return cudaSuccess; }
inline const char *cudaGetErrorString(cudaError_t e) { return e == cudaErrorNotSupported ? "operation not supported (emulation)" : "emulated"; }
// ---- the host-side runtime calls of ghicp_capi.cu (tests/harness/emu_library.cpp): device memory = the heap, one "device",
// streams and events are tokens, everything is synchronous
enum { cudaStreamNonBlocking = 1 };
inline cudaError_t cudaGetDeviceCount(int *n) { *n = 1; return cudaSuccess; }
inline cudaError_t cudaSetDevice(int d) { return d == 0 ? cudaSuccess : cudaErrorInvalidValue; }
inline cudaError_t cudaMalloc(void **p, size_t bytes) { *p = emu_device_alloc(bytes); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
inline cudaError_t cudaFree(void *p) { emu_device_free(p); return cudaSuccess; }
template <typename T> inline cudaError_t cudaMallocHost(T **p, size_t bytes) { *p = (T *)emu_poisoned(bytes); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
inline cudaError_t cudaFreeHost(void *p) { free(p); return cudaSuccess; }
// every host pointer is "pageable" here: the library's staging path is the one exercised
enum cudaMemoryType { cudaMemoryTypeUnregistered = 0, cudaMemoryTypeHost = 1, cudaMemoryTypeDevice = 2 };
struct cudaPointerAttributes { cudaMemoryType type; };
inline cudaError_t cudaPointerGetAttributes(cudaPointerAttributes *a, const void *) { a->type = cudaMemoryTypeUnregistered; return cudaSuccess; }
inline cudaError_t cudaMemcpy(void *d, const void *s, size_t bytes, cudaMemcpyKind) { memmove(d, s, bytes); return cudaSuccess; }
inline cudaError_t cudaMemset(void *p, int v, size_t bytes) { memset(p, v, bytes); return cudaSuccess; }
inline cudaError_t cudaMemGetInfo(size_t *free_b, size_t *total_b) { *free_b = (size_t)8 << 30; *total_b = (size_t)8 << 30; return cudaSuccess; }
inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned) { *s = nullptr; return cudaSuccess; }
inline cudaError_t cudaStreamDestroy(cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaEventCreate(cudaEvent_t *e) { *e = nullptr; return cudaSuccess; }
inline cudaError_t cudaEventDestroy(cudaEvent_t) { return cudaSuccess; }
inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t) { return cudaSuccess; }
inline cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t, cudaEvent_t) { *ms = 0.f; return cudaSuccess; }

struct float4 { float x, y, z, w; };
inline float4 make_float4(float x, float y, float z, float w) { float4 v; v.x = x; v.y = y; v.z = z; v.w = w; return v; }
struct uint2 { unsigned x, y; };
struct ulonglong2 { unsigned long long x, y; };
struct uint4 { unsigned x, y, z, w; };
inline uint4 make_uint4(unsigned x, unsigned y, unsigned z, unsigned w) { uint4 v; v.x = x; v.y = y; v.z = z; v.w = w; return v; }

#define threadIdx (emu::cur()->tidx)
#define blockIdx (emu::cur()->bidx)
#define blockDim (emu::g_bdim)
#define gridDim (emu::g_gdim)

inline void __syncthreads() { emu::syncthreads(); }
inline void __threadfence() {}   // one OS thread: program order is memory order
template <typename T>
inline T __shfl_xor_sync(unsigned, T v, int lane_mask) { return emu::shfl<T>(v, (emu::cur()->tidx.x & 31) ^ lane_mask); }
template <typename T>
inline T __shfl_up_sync(unsigned, T v, int delta) {
  const int lane = emu::cur()->tidx.x & 31;
  return emu::shfl<T>(v, lane >= delta ? lane - delta : lane);
}
template <typename T>
inline T atomicAdd(T *p, T v) { T old = *p; *p = old + v; return old; }   // one OS thread: fibers never preempt

template <typename T>
inline T atomicMin(T *p, T v) { T old = *p; if (v < old) *p = v; return old; }
template <typename T>
inline T atomicMax(T *p, T v) { T old = *p; if (v > old) *p = v; return old; }
inline unsigned __reduce_min_sync(unsigned, unsigned v) {
  unsigned all[32];
  emu::warp_all<unsigned>(v, all);
  unsigned m = all[0];
  for (int l = 1; l < 32; ++l) m = all[l] < m ? all[l] : m;
  return m;
}
inline unsigned __ballot_sync(unsigned, int pred) {
  unsigned all[32], m = 0;
  emu::warp_all<unsigned>(pred ? 1u : 0u, all);
  for (int l = 0; l < 32; ++l) m |= (all[l] & 1u) << l;
  return m;
}
inline int __popcll(unsigned long long v) { return __builtin_popcountll(v); }
inline int __popc(unsigned v) { return __builtin_popcount(v); }
inline void __syncwarp(unsigned = 0xffffffffu) { emu::shfl<int>(0, emu::cur()->tidx.x & 31); }   // a shuffle is a rendezvous of the warp's live lanes
template <typename T> inline T __shfl_sync(unsigned, T v, int src_lane) { return emu::shfl<T>(v, src_lane & 31); }
inline int __any_sync(unsigned, int pred) {
  unsigned all[32];
  emu::warp_all<unsigned>(pred ? 1u : 0u, all);
  for (int l = 0; l < 32; ++l) if (all[l] & 1u) return 1;
  return 0;
}
inline unsigned __reduce_add_sync(unsigned, unsigned v) {
  unsigned all[32], s = 0;
  emu::warp_all<unsigned>(v, all);
  for (int l = 0; l < 32; ++l) s += all[l];
  return s;
}
inline double __dsub_rn(double a, double b) { return a - b; }     // built with -ffp-contract=off: separately rounded
inline double __dadd_rn(double a, double b) { return a + b; }
inline double __dmul_rn(double a, double b) { return a * b; }
inline double __dsqrt_rn(double a) { return sqrt(a); }
inline float __fadd_rn(float a, float b) { return a + b; }
template <typename T> inline T __ldcg(const T *p) { return *p; }
inline int __ffs(unsigned v) { return v ? __builtin_ctz(v) + 1 : 0; }
inline unsigned __float_as_uint(float f) { unsigned u; memcpy(&u, &f, 4); return u; }
inline float __uint_as_float(unsigned u) { float f; memcpy(&f, &u, 4); return f; }
inline long long __double_as_longlong(double d) { long long l; memcpy(&l, &d, 8); return l; }
inline double __longlong_as_double(long long l) { double d; memcpy(&d, &l, 8); return d; }
inline long long __double2ll_rn(double x) { return llrint(x); }   // default rounding mode: to nearest even
inline float __double2float_ru(double x) {
  float f = (float)x;
  if ((double)f < x) f = nextafterf(f, INFINITY);
  return f;
}

inline int min(int a, int b) { return a < b ? a : b; }
inline int max(int a, int b) { return a > b ? a : b; }
inline long long min(long long a, long long b) { return a < b ? a : b; }
inline long long max(long long a, long long b) { return a > b ? a : b; }
