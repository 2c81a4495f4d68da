// Shared helpers for the sm_90a kernels of libdi_b200.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#define DI_OK 0
#define DI_ERR_ARG (-1)
#define DI_ERR_LAUNCH (-2)
#define DI_ERR_UNSUPPORTED (-3)

void di_set_error(const char* fmt, ...);

#define DI_CHECK_ARG(cond, ...)          \
  do {                                   \
    if (!(cond)) {                       \
      di_set_error(__VA_ARGS__);         \
      return DI_ERR_ARG;                 \
    }                                    \
  } while (0)

// Never synchronises: only picks up launch-configuration errors.
#define DI_CHECK_LAUNCH(name)                                             \
  do {                                                                    \
    cudaError_t e__ = cudaGetLastError();                                 \
    if (e__ != cudaSuccess) {                                             \
      di_set_error("%s: launch failed: %s", name, cudaGetErrorString(e__)); \
      return DI_ERR_LAUNCH;                                               \
    }                                                                     \
  } while (0)

static inline int di_cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) once per (call site, device): one process may drive several GPUs
struct DiSmemOnce {
  bool done[64];
};
template <class Kern>
static inline bool di_smem_once(DiSmemOnce& st, Kern kernel, int bytes) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return false;
  if (!st.done[dev]) {
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) != cudaSuccess) return false;
    st.done[dev] = true;
  }
  return true;
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

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

// Activation codes shared with the host side.
enum { DI_ACT_NONE = 0, DI_ACT_RELU = 1, DI_ACT_GELU = 2 };

// NOTE: call sites apply this inside a loop only under a warp-uniform `act`; for register tiles prefer one branch
// around the whole tile (see act_tile in gemm_tc.cu) so that the GELU polynomial is not if-converted per element.
__device__ __forceinline__ float di_gelu(float v) { return 0.5f * v * (1.f + erff(v * 0.70710678118654752440f)); }
__device__ __forceinline__ float di_act(float v, int act) {
  if (act == DI_ACT_RELU) return fmaxf(v, 0.f);
  if (act == DI_ACT_GELU) return 0.5f * v * (1.f + erff(v * 0.70710678118654752440f));
  return v;
}
