// hb200 -- fp32 SIMT GEMM with generic operand strides (linears, RNN projections, weight grads).
// C[M,N] = alpha * A[M,K] * B[K,N] (+bias[N]) (+C) (ReLU);  A(m,k) = a[m*a_ms + k*a_ks],
// B(k,n) = b[k*b_ks + n*b_ns].  128x128x8 tiles, 256 threads, 8x8 micro-tile per thread.
// The recurrent part of the policy stays in full fp32 so the masked-recurrence parity of
// test/test_rnn_state_encoder.py (tolerance 1e-3, TF32 off) holds.
#include "common.cuh"

namespace hb200 {
void count_launch(int n);

constexpr int BM = 128, BN = 128, BK = 8;

// load a BMxBK (A) or BKxBN (B) tile into smem laid out [k][mn]; 256 threads
// MODE 0: mn contiguous in memory (stride_mn == 1) -> float4 along mn
// MODE 1: k contiguous (stride_k == 1)             -> float4 along k, transposed store
// MODE 2: generic scalar
template <int MODE>
__device__ __forceinline__ void load_tile(const float* __restrict__ p, long long s_mn, long long s_k,
                                          int mn0, int k0, int MN, int K, float (*sm)[BM + 4]) {
  const int t = threadIdx.x;
  if (MODE == 0) {
    const int k = t >> 5, m4 = (t & 31) << 2;
    const int gk = k0 + k, gm = mn0 + m4;
    float4 v = make_float4(0, 0, 0, 0);
    if (gk < K) {
      const float* src = p + (long long)gk * s_k + gm;
      if (gm + 3 < MN && ((reinterpret_cast<uintptr_t>(src) & 15) == 0)) {
        v = *reinterpret_cast<const float4*>(src);
      } else {
        if (gm < MN) v.x = src[0];
        if (gm + 1 < MN) v.y = src[1];
        if (gm + 2 < MN) v.z = src[2];
        if (gm + 3 < MN) v.w = src[3];
      }
    }
    *reinterpret_cast<float4*>(&sm[k][m4]) = v;
  } else if (MODE == 1) {
    const int m = t >> 1, k4 = (t & 1) << 2;
    const int gm = mn0 + m, gk = k0 + k4;
    float4 v = make_float4(0, 0, 0, 0);
    if (gm < MN) {
      const float* src = p + (long long)gm * s_mn + gk;
      if (gk + 3 < K && ((reinterpret_cast<uintptr_t>(src) & 15) == 0)) {
        v = *reinterpret_cast<const float4*>(src);
      } else {
        if (gk < K) v.x = src[0];
        if (gk + 1 < K) v.y = src[1];
        if (gk + 2 < K) v.z = src[2];
        if (gk + 3 < K) v.w = src[3];
      }
    }
    sm[k4][m] = v.x; sm[k4 + 1][m] = v.y; sm[k4 + 2][m] = v.z; sm[k4 + 3][m] = v.w;
  } else {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int e = t + i * 256;
      const int k = e >> 7, m = e & 127;
      const int gk = k0 + k, gm = mn0 + m;
      sm[k][m] = (gk < K && gm < MN) ? p[(long long)gm * s_mn + (long long)gk * s_k] : 0.f;
    }
  }
}

template <int AMODE, int BMODE>
__global__ void __launch_bounds__(256)
sgemm_kernel(const float* __restrict__ a, long long a_ms, long long a_ks, const float* __restrict__ b,
             long long b_ks, long long b_ns, float* __restrict__ c, long long ldc,
             const float* __restrict__ bias, int M, int N, int K, float alpha, int accumulate, int relu,
             int k_per_split, float* __restrict__ ws) {
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN + 4];
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;  // 16 x 16 threads, 8x8 each
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  const int k_begin = blockIdx.z * k_per_split;
  const int k_end = min(K, k_begin + k_per_split);
  for (int k0 = k_begin; k0 < k_end; k0 += BK) {
    load_tile<AMODE>(a, a_ms, a_ks, m0, k0, M, k_end, As);
    load_tile<BMODE>(b, b_ns, b_ks, n0, k0, N, k_end, Bs);
    __syncthreads();
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float av[8], bv[8];
      const float4 a0 = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[k][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[k][64 + tx * 4]);
      av[0] = a0.x; av[1] = a0.y; av[2] = a0.z; av[3] = a0.w; av[4] = a1.x; av[5] = a1.y; av[6] = a1.z; av[7] = a1.w;
      bv[0] = b0.x; bv[1] = b0.y; bv[2] = b0.z; bv[3] = b0.w; bv[4] = b1.x; bv[5] = b1.y; bv[6] = b1.z; bv[7] = b1.w;
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (m >= M) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int n = n0 + (j < 4 ? tx * 4 + j : 64 + tx * 4 + (j - 4));
      if (n >= N) continue;
      float v = alpha * acc[i][j];
      if (gridDim.z > 1) {  // split-K: this split's partial, summed in split order by sgemm_split_sum_kernel
        ws[((size_t)blockIdx.z * M + m) * N + n] = v;
        continue;
      }
      float* dst = c + (long long)m * ldc + n;
      if (bias) v += bias[n];
      if (accumulate) v += *dst;
      if (relu) v = fmaxf(v, 0.f);
      *dst = v;
    }
  }
}
// C[m, n] += bias[n] + sum over z = 0 .. splits-1 of ws[z, m, n], always in that order (run-to-run identical)
__global__ void sgemm_split_sum_kernel(const float* __restrict__ ws, int splits, float* __restrict__ c, long long ldc,
                                       const float* __restrict__ bias, int M, int N) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)M * N) return;
  const int m = (int)(i / N), n = (int)(i - (long long)m * N);
  float v = ws[i];
  for (int z = 1; z < splits; ++z) v += ws[(size_t)z * M * N + i];
  if (bias) v += bias[n];
  c[(long long)m * ldc + n] += v;
}
}  // namespace hb200

using namespace hb200;

extern "C" int hb200_sgemm(const float* a, long long a_ms, long long a_ks, const float* b, long long b_ks,
                           long long b_ns, float* c, long long ldc, const float* bias, int m, int n, int k,
                           float alpha, int accumulate, int relu, hb200_stream_t stream) {
  HB_CHECK_ARG(a && b && c && m > 0 && n > 0 && k > 0, "sgemm: bad args");
  // split-K when the output tile grid cannot fill the GPU and the reduction is long (weight gradients:
  // K = frames).  Needs C to hold the value to accumulate into -> only in accumulate mode without ReLU.  The splits'
  // partials go to the stream's workspace and are added in split order (no float atomics: same result every run).
  int splits = 1;
  {
    const long long tiles = (long long)cdiv(n, BN) * cdiv(m, BM);
    if (accumulate && !relu && tiles < kNumSMs && k >= 1024) {
      splits = (int)((2 * kNumSMs + tiles - 1) / tiles);
      if (splits > k / 256) splits = k / 256;
      if (splits < 1) splits = 1;
    }
  }
  int k_per_split = ((cdiv(k, splits) + BK - 1) / BK) * BK;
  splits = cdiv(k, k_per_split);
  const int am = (a_ms == 1) ? 0 : (a_ks == 1 ? 1 : 2);
  const int bm = (b_ns == 1) ? 0 : (b_ks == 1 ? 1 : 2);
  dim3 grid(cdiv(n, BN), cdiv(m, BM), splits);
  cudaStream_t st = (cudaStream_t)stream;
  float* ws = nullptr;
  if (splits > 1) {
    int* tickets = nullptr;
    const int rc = stream_workspace(st, (size_t)splits * m * n, 0, &ws, &tickets);
    if (rc) return rc;
  }
#define HB_SG(AM, BMO) \
  sgemm_kernel<AM, BMO><<<grid, 256, 0, st>>>(a, a_ms, a_ks, b, b_ks, b_ns, c, ldc, bias, m, n, k, alpha, accumulate, relu, \
                                              k_per_split, ws)
  switch (am * 3 + bm) {
    case 0: HB_SG(0, 0); break;
    case 1: HB_SG(0, 1); break;
    case 2: HB_SG(0, 2); break;
    case 3: HB_SG(1, 0); break;
    case 4: HB_SG(1, 1); break;
    case 5: HB_SG(1, 2); break;
    case 6: HB_SG(2, 0); break;
    case 7: HB_SG(2, 1); break;
    default: HB_SG(2, 2); break;
  }
#undef HB_SG
  HB_LAUNCH_OK();
  count_launch(1);
  if (splits > 1) {
    sgemm_split_sum_kernel<<<cdiv((long long)m * n, 256), 256, 0, st>>>(ws, splits, c, ldc, bias, m, n);
    HB_LAUNCH_OK();
    count_launch(1);
  }
  return HB200_OK;
}
