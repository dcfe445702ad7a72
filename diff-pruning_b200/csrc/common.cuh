// common.cuh — shared helpers for libdpb200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "dpb200.h"

extern int g_dp_last_cuda_error;
// grid-stride kernels cap their grids at a multiple of the SM count (H100 SXM: 132)
constexpr int DP_NUM_SMS = 132;
extern long long g_dp_launch_count;

static inline int dp_check_launch() {
  ++g_dp_launch_count;
  cudaError_t e = cudaPeekAtLastError();
  if (e != cudaSuccess) {
    g_dp_last_cuda_error = (int)e;
    (void)cudaGetLastError();
    return DP_ERR_CUDA;
  }
  return DP_OK;
}

#define DP_REQUIRE(cond, code) \
  do {                         \
    if (!(cond)) return (code); \
  } while (0)

// a nullable fp32 view [rows][ld] that float4 accesses may use: 16-byte aligned base, row pitch a multiple of 4
static inline bool al16(const void* p, long long ld) { return p == nullptr || ((((uintptr_t)p) & 15) == 0 && (ld % 4) == 0); }

static inline int ilog2_exact(int v) {  // log2 if power of two, else -1
  if (v <= 0 || (v & (v - 1))) return -1;
  int l = 0;
  while ((1 << l) < v) ++l;
  return l;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// max |v| of the values a thread wrote -> the output tensor's amax slot (dp_amax semantics: atomicMax on the bit pattern of a
// non-negative float is order-independent, so slots are run-to-run identical); one atomic per converged warp
__device__ __forceinline__ void amax_commit(uint32_t* slot, float m) {
  const unsigned mask = __activemask();
  const uint32_t r = __reduce_max_sync(mask, __float_as_uint(m));
  if ((threadIdx.x & 31) == (unsigned)(__ffs(mask) - 1) && r) atomicMax(slot, r);
}
// 1 / (1 + exp(-x)): __frcp_rn is the correctly rounded reciprocal, i.e. the same bits as the IEEE division 1.0f / y, without the
// division's slow-path check
__device__ __forceinline__ float sigmoidf_acc(float x) { return __frcp_rn(1.0f + expf(-x)); }
