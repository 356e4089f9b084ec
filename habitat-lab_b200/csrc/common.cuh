// hb200 -- shared device/host helpers for the sm_90a DD-PPO learner kernels.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/hb200.h"

namespace hb200 {

// ---- error plumbing -----------------------------------------------------------
void set_last_error(const char* fmt, ...);

#define HB_CHECK_ARG(cond, ...)              \
  do {                                       \
    if (!(cond)) {                           \
      hb200::set_last_error(__VA_ARGS__);    \
      return HB200_ERR_INVALID_ARG;          \
    }                                        \
  } while (0)

#define HB_CUDA(expr)                                                          \
  do {                                                                         \
    cudaError_t _e = (expr);                                                   \
    if (_e != cudaSuccess) {                                                   \
      hb200::set_last_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr,       \
                            cudaGetErrorString(_e));                           \
      return HB200_ERR_CUDA;                                                   \
    }                                                                          \
  } while (0)

#define HB_LAUNCH_OK()                                                         \
  do {                                                                         \
    cudaError_t _e = cudaGetLastError();                                       \
    if (_e != cudaSuccess) {                                                   \
      hb200::set_last_error("%s:%d launch -> %s", __FILE__, __LINE__,          \
                            cudaGetErrorString(_e));                           \
      return HB200_ERR_CUDA;                                                   \
    }                                                                          \
  } while (0)

static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// ---- deterministic reductions ----------------------------------------------------------------------------------
// Gradients summed over frames / pixels / K splits are never accumulated with floating-point atomics (their order, and
// so the result's last bits, would change from run to run).  Kernels write one partial per block into a scratch
// buffer, and reduce_partials adds them in a fixed order.
// Per-stream scratch (tgemm.cu): one growing buffer per stream (per graph capture under capture), stream-ordered.
int stream_workspace(cudaStream_t st, size_t floats, int tiles, float** ws, int** tickets);
// dst[i] += sum over p = 0 .. nparts-1, in order of fixed chunks, of parts[p * ld + i] for i < count.
// tmp: min(nparts, kReduceChunks) * count floats of scratch.
constexpr int kReduceChunks = 32;
int reduce_partials(const float* parts, int nparts, long long ld, long long count, float* dst, float* tmp,
                    cudaStream_t st);
constexpr int kNumSMs = 132;  // H100 SXM

// ---- warp / block reductions ---------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// block-wide sum; result valid in thread 0 (and broadcast through smem slot 0)
template <typename T>
__device__ __forceinline__ T block_sum(T v, T* smem /* >= 32 */) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) smem[w] = v;
  __syncthreads();
  const int nw = (blockDim.x + 31) >> 5;
  T r = (threadIdx.x < nw) ? smem[threadIdx.x] : T(0);
  if (w == 0) {
    r = warp_sum(r);
    if (lane == 0) smem[0] = r;
  }
  __syncthreads();
  return smem[0];
}

// ---- bf16 pack helpers -----------------------------------------------------------
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}
__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y), c = unpack_bf16x2(u.z), d = unpack_bf16x2(u.w);
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint4 u;
  u.x = pack_bf16x2(f[0], f[1]); u.y = pack_bf16x2(f[2], f[3]);
  u.z = pack_bf16x2(f[4], f[5]); u.w = pack_bf16x2(f[6], f[7]);
  return u;
}

// ---- storage types -----------------------------------------------------------------
// FORWARD values (pooled input, conv outputs y, normalised activations a / o, packed weight images of the forward
// convs) are IEEE fp16: 11 significant bits -- the same significand as the TF32 operands the reference's cuDNN path
// multiplies -- at bf16's cost.  GRADIENTS (g, dy, gz) are bf16: they need fp32's exponent range (per-element
// magnitudes of 1e-8 are normal with a mean-over-4096-frames loss) and their rounding only perturbs the result
// linearly, while forward rounding flips ReLU / max-pool decisions (DESIGN.md section 3).
typedef __half act_t;
typedef __nv_bfloat16 grad_t;

// fp16 pack with saturation to +-65504 (one F2FP.SATFINITE instruction): an overflow must not become inf
__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
__device__ __forceinline__ float2 unpack_f16x2(uint32_t u) {
  __half2 v = *reinterpret_cast<__half2*>(&u);
  return __half22float2(v);
}
__device__ __forceinline__ void unpack8a(const uint4& u, float (&f)[8]) {
  float2 a = unpack_f16x2(u.x), b = unpack_f16x2(u.y), c = unpack_f16x2(u.z), d = unpack_f16x2(u.w);
  f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
}
__device__ __forceinline__ uint4 pack8a(const float (&f)[8]) {
  uint4 u;
  u.x = pack_f16x2(f[0], f[1]); u.y = pack_f16x2(f[2], f[3]);
  u.z = pack_f16x2(f[4], f[5]); u.w = pack_f16x2(f[6], f[7]);
  return u;
}

// 16-byte vector reduction to global memory (sm_90+): one L2 transaction for 4 floats
__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

}  // namespace hb200
