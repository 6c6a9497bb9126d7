// common.cuh -- shared helpers for the sam6d_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <math.h>

#define S6_API extern "C" __attribute__((visibility("default")))

#define S6_LAUNCH_CHECK()                              \
  do {                                                 \
    cudaError_t e__ = cudaGetLastError();              \
    if (e__ != cudaSuccess) return (int)e__;           \
  } while (0)

#define S6_CHECK(call)                                 \
  do {                                                 \
    cudaError_t e__ = (call);                          \
    if (e__ != cudaSuccess) return (int)e__;           \
  } while (0)

// argument errors are reported as negative codes (CUDA errors are positive)
#define S6_EINVAL (-22)
#define S6_REQUIRE(cond)                               \
  do {                                                 \
    if (!(cond)) return S6_EINVAL;                     \
  } while (0)

static inline cudaStream_t s6_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

// Programmatic dependent launch (PDL).  A step is ~280 launches, many of them 10-us kernels on 12608 token rows: with the
// launch attribute below the next grid is scheduled as soon as every CTA of the current one has started (s6_pdl_trigger at
// the top of the kernel), runs its prologue (barrier init, shared-memory set-up, descriptor prefetch) on free SMs and blocks in
// s6_pdl_wait until the predecessor has completed and flushed.  Every kernel launched this way calls s6_pdl_wait before its
// first global access that may depend on an earlier kernel; kernels launched the ordinary way are unaffected on either side.
__device__ __forceinline__ void s6_pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void s6_pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
template <typename... KArgs, typename... Args>
static inline cudaError_t s6_launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// (value, index) argmax with "first index wins ties" -- the torch.max / torch.topk convention
__device__ __forceinline__ void argmax_first(float& v, int& i, float v2, int i2) {
  if (v2 > v || (v2 == v && i2 < i)) { v = v2; i = i2; }
}
__device__ __forceinline__ void warp_argmax_first(float& v, int& i) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    float v2 = __shfl_xor_sync(0xffffffffu, v, o);
    int i2 = __shfl_xor_sync(0xffffffffu, i, o);
    argmax_first(v, i, v2, i2);
  }
}

__device__ __forceinline__ float ld_as_float(const float* p) { return *p; }
__device__ __forceinline__ float ld_as_float(const __nv_bfloat16* p) { return __bfloat162float(*p); }

// activation codes of the GEMM epilogues: 0 none, 1 ReLU, 2 GELU (exact erf form, nn.GELU default)
__device__ __forceinline__ float s6_act(float x, int act) {
  if (act == 1) return fmaxf(x, 0.f);
  if (act == 2) return 0.5f * x * (1.f + erff(x * 0.70710678118654752f));
  return x;
}

static inline int s6_cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// grid of a persistent kernel: min(work, per_sm x the SM count of the current device).  The device is queried on every call
// because the caller's current device can change between calls.
static inline cudaError_t s6_persistent_grid(long long work, int per_sm, int* grid) {
  int dev = 0, sms = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (e != cudaSuccess) return e;
  const long long cap = (long long)per_sm * sms;
  *grid = (int)(work < cap ? work : cap);
  return cudaSuccess;
}
