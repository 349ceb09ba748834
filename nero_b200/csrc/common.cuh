// Shared host/device helpers for libnero_b200.
#pragma once
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>
#include <cuda_bf16.h>

// Every k_*.cu defines the entry points of its kernels against these prototypes, inside extern "C": a definition whose
// parameters differ from its declaration does not compile.
#include "../../include/nero_b200.h"

#if defined(__CUDACC__)
#define NERO_HD __host__ __device__ __forceinline__
#else
#define NERO_HD inline
#endif

#define NERO_OK 0
#define NERO_ERR_ARG 1
#define NERO_ERR_CUDA 2

// Launch-error check used by every C-ABI entry point (no sync: errors of the launch itself only).
#define NERO_LAUNCH_CHECK()                                                     \
  do {                                                                          \
    cudaError_t e__ = cudaGetLastError();                                       \
    if (e__ != cudaSuccess) {                                                   \
      fprintf(stderr, "nero_b200: CUDA error %s at %s:%d\n", cudaGetErrorString(e__), __FILE__, __LINE__); \
      return NERO_ERR_CUDA;                                                     \
    }                                                                           \
  } while (0)

#define NERO_CUDA_TRY(expr)                                                     \
  do {                                                                          \
    cudaError_t e__ = (expr);                                                   \
    if (e__ != cudaSuccess) {                                                   \
      fprintf(stderr, "nero_b200: CUDA error %s at %s:%d\n", cudaGetErrorString(e__), __FILE__, __LINE__); \
      return NERO_ERR_CUDA;                                                     \
    }                                                                           \
  } while (0)

namespace nero {

constexpr int kNumSMs = 132;   // H100 SXM

// activation codes shared by the GEMM epilogues and the C ABI
enum Act : int { ACT_NONE = 0, ACT_SOFTPLUS100 = 1, ACT_RELU = 2, ACT_SIGMOID = 3, ACT_EXPCLAMP = 4 };

// GEMM epilogue modes
enum EpiMode : int {
  EPI_BIAS_ACT = 0,   // out = oscale * act(acc + bias)
  EPI_MUL_DACT = 1,   // out = oscale * dact(H) * acc (+ addend)            [input-gradient sweeps]
  EPI_TANGENT = 2,    // out = oscale * dact(H) * acc ; out2 = 100*(1-dact(H))*V*acc   [second-order sweep]
};

// softplus(beta=100) with torch's threshold (beta*x > 20 -> x)          network/field.py:124
NERO_HD float softplus100(float a) {
  float z = 100.0f * a;
  return z > 20.0f ? a : log1pf(expf(z)) * 0.01f;
}
// its derivative sigma(100 a) recovered from the stored activation h = softplus100(a): 1 - exp(-100 h)
NERO_HD float dsoftplus100_from_h(float h) {
  float z = 100.0f * h;
  return z > 20.0f ? 1.0f : -expm1f(-z);
}

NERO_HD float apply_act(float x, int act, float p) {
  switch (act) {
    case ACT_SOFTPLUS100: return softplus100(x);
    case ACT_RELU: return fmaxf(x, 0.0f);
    case ACT_SIGMOID: return 1.0f / (1.0f + expf(-x));
    case ACT_EXPCLAMP: return expf(fminf(x, p));
    default: return x;
  }
}
// derivative factor from the stored post-activation value h
NERO_HD float dact_from_h(float h, int act) {
  switch (act) {
    case ACT_SOFTPLUS100: return dsoftplus100_from_h(h);
    case ACT_RELU: return h > 0.0f ? 1.0f : 0.0f;
    default: return 1.0f;
  }
}

// split an fp32 into bf16 hi + bf16 lo (round-to-nearest both): x ~= hi + lo with ~2^-17 relative error
NERO_HD void split_bf16(float x, __nv_bfloat16& hi, __nv_bfloat16& lo) {
  hi = __float2bfloat16_rn(x);
  lo = __float2bfloat16_rn(x - __bfloat162float(hi));
}

// byte offset of element (row r, k index kk in [0,64)) inside one K-major SWIZZLE_128B operand tile
__host__ __device__ __forceinline__ uint32_t sw128_offset(uint32_t r, uint32_t kk) {
  return r * 128u + ((((kk >> 3) ^ (r & 7u)) << 4) | ((kk & 7u) << 1));
}
// byte offset of element (row r, k index kk in [0,32)) inside one K-major SWIZZLE_64B operand tile
__host__ __device__ __forceinline__ uint32_t sw64_offset(uint32_t r, uint32_t kk) {
  return r * 64u + ((((kk >> 3) ^ ((r >> 1) & 3u)) << 4) | ((kk & 7u) << 1));
}

}  // namespace nero
