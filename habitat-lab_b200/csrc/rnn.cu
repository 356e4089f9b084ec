// hb200 -- masked LSTM recurrence, one launch per (layer, time step), full fp32.
//   h_in = h_{t-1} * m_t ; c_in = c_{t-1} * m_t          (mask resets the state BEFORE the step,
//   gates = xproj_t + h_in W_hh^T                          HB/rl/models/rnn_state_encoder.py:301-316)
//   i,f,g,o = sig,sig,tanh,sig ; c = f*c_in + i*g ; h = o*tanh(c)
// The input projection (x W_ih^T + b_ih + b_hh) for ALL T*N frames is one hb200_sgemm call; only
// the truly sequential h W_hh^T part lives here.  This replaces the PackedSequence index
// machinery (rnn_state_encoder.py:35-277): a masked recurrence needs nothing but `masks`.
#include "common.cuh"
#include <stdlib.h>

namespace hb200 {
void count_launch(int n);

constexpr int kUnits = 4;  // hidden units per block -> 16 gate rows

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }

// grid = H / kUnits blocks, 256 threads (8 warps).  smem: W rows [16][H].
template <int NJ>  // H = 32 * NJ
__global__ void __launch_bounds__(256)
lstm_step_fwd_kernel(const float* __restrict__ xproj, const float* __restrict__ w_hh,
                     const float* __restrict__ b_hh, const uint8_t* __restrict__ masks, const float* __restrict__ h_prev,
                     long long hp_stride, const float* __restrict__ c_prev, long long cp_stride,
                     float* __restrict__ h, float* __restrict__ c, float* __restrict__ gates_out, int n) {
  constexpr int H = NJ * 32;
  extern __shared__ float sw[];  // [16][H]
  const int u0 = blockIdx.x * kUnits;
  for (int i = threadIdx.x; i < 16 * H; i += blockDim.x) {
    const int r = i / H, k = i - r * H;
    const int gate = r >> 2, u = r & 3;  // row r = gate*4 + u
    sw[i] = w_hh[((size_t)gate * H + u0 + u) * H + k];
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int s = warp; s < n; s += 8) {
    const float m = masks[s] ? 1.f : 0.f;
    float hv[NJ];
#pragma unroll
    for (int j = 0; j < NJ; ++j) hv[j] = h_prev[(size_t)s * hp_stride + lane + 32 * j] * m;
    float dot[16];
#pragma unroll
    for (int r = 0; r < 16; ++r) {
      float acc = 0.f;
#pragma unroll
      for (int j = 0; j < NJ; ++j) acc = fmaf(hv[j], sw[r * H + lane + 32 * j], acc);
      dot[r] = warp_sum(acc);
    }
    // lanes 0..3 finish one hidden unit each (static register indexing via select)
    float gi = 0, gf = 0, gg = 0, go = 0;
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (lane == u) { gi = dot[u]; gf = dot[4 + u]; gg = dot[8 + u]; go = dot[12 + u]; }
    if (lane < kUnits) {
      const int col = u0 + lane;
      const float* xp = xproj + (size_t)s * 4 * H;
      if (b_hh) { gi += b_hh[col]; gf += b_hh[H + col]; gg += b_hh[2 * H + col]; go += b_hh[3 * H + col]; }
      const float i_ = sigmoidf_(gi + xp[col]);
      const float f_ = sigmoidf_(gf + xp[H + col]);
      const float g_ = tanhf(gg + xp[2 * H + col]);
      const float o_ = sigmoidf_(go + xp[3 * H + col]);
      const float cin = c_prev[(size_t)s * cp_stride + col] * m;
      const float cn = f_ * cin + i_ * g_;
      const float hn = o_ * tanhf(cn);
      c[(size_t)s * H + col] = cn;
      h[(size_t)s * H + col] = hn;
      if (gates_out) {
        float* go_ = gates_out + (size_t)s * 4 * H;
        go_[col] = i_; go_[H + col] = f_; go_[2 * H + col] = g_; go_[3 * H + col] = o_;
      }
    }
  }
}

// pointwise part of the backward step; also zeroes dh_prev for the matmul kernel's atomics
__global__ void lstm_step_bwd_pointwise_kernel(const float* __restrict__ dh_out, const float* __restrict__ dh_rec,
                                               const float* __restrict__ dc_rec, const float* __restrict__ gates,
                                               const float* __restrict__ c, const float* __restrict__ c_prev,
                                               long long cp_stride, const uint8_t* __restrict__ masks,
                                               float* __restrict__ dgates, float* __restrict__ dh_prev,
                                               float* __restrict__ dc_prev, int n, int H) {
  const int total = n * H;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int s = i / H, k = i - s * H;
    const float m = masks[s] ? 1.f : 0.f;
    const float* gt = gates + (size_t)s * 4 * H;
    const float i_ = gt[k], f_ = gt[H + k], g_ = gt[2 * H + k], o_ = gt[3 * H + k];
    float dh = dh_out ? dh_out[i] : 0.f;
    if (dh_rec) dh += dh_rec[i];
    const float tc = tanhf(c[i]);
    float dc = dh * o_ * (1.f - tc * tc);
    if (dc_rec) dc += dc_rec[i];
    const float cin = c_prev[(size_t)s * cp_stride + k] * m;
    float* dg = dgates + (size_t)s * 4 * H;
    dg[k] = dc * g_ * i_ * (1.f - i_);
    dg[H + k] = dc * cin * f_ * (1.f - f_);
    dg[2 * H + k] = dc * i_ * (1.f - g_ * g_);
    dg[3 * H + k] = dh * tc * o_ * (1.f - o_);
    dc_prev[i] = dc * f_ * m;
    dh_prev[i] = 0.f;
  }
}

// dh_prev[s,k] += m_s * sum_{r in slab} dgates[s,r] * W_hh[r,k];  grid (H/32, R/rows_per_block)
template <int NS>  // sequences per warp
__global__ void __launch_bounds__(256)
lstm_step_bwd_matmul_kernel(const float* __restrict__ dgates, const float* __restrict__ w_hh,
                            const uint8_t* __restrict__ masks, float* __restrict__ dh_prev, int n, int H,
                            int rows_per_block) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int k = blockIdx.x * 32 + lane;
  const int r0 = blockIdx.y * rows_per_block, r1 = r0 + rows_per_block;
  const int R = 4 * H;
  for (int sb = warp * NS; sb < n; sb += 8 * NS) {
    float acc[NS];
#pragma unroll
    for (int q = 0; q < NS; ++q) acc[q] = 0.f;
    for (int r = r0; r < r1; ++r) {
      const float w = w_hh[(size_t)r * H + k];
#pragma unroll
      for (int q = 0; q < NS; ++q) {
        const int s = sb + q;
        if (s < n) acc[q] = fmaf(dgates[(size_t)s * R + r], w, acc[q]);
      }
    }
#pragma unroll
    for (int q = 0; q < NS; ++q) {
      const int s = sb + q;
      if (s < n && masks[s]) atomicAdd(&dh_prev[(size_t)s * H + k], acc[q]);
    }
  }
}
}  // namespace hb200

using namespace hb200;

extern "C" int hb200_lstm_step_fwd(const float* xproj, const float* w_hh, const float* b_hh, const uint8_t* masks,
                                   const float* h_prev, long long h_prev_stride, const float* c_prev,
                                   long long c_prev_stride, float* h, float* c, float* gates_out, int n,
                                   int hidden, hb200_stream_t stream) {
  HB_CHECK_ARG(xproj && w_hh && masks && h_prev && c_prev && h && c && n > 0, "lstm_step_fwd: bad args");
  HB_CHECK_ARG(hidden % 32 == 0 && hidden >= 32 && hidden <= 512 && hidden % kUnits == 0,
               "lstm_step_fwd: hidden=%d unsupported (multiple of 32, <= 512)", hidden);
  cudaStream_t st = (cudaStream_t)stream;
  const size_t smem = sizeof(float) * 16 * hidden;
  const int grid = hidden / kUnits;
#define HB_LSTM(NJ)                                                                                       \
  {                                                                                                       \
    auto kern = lstm_step_fwd_kernel<NJ>;                                                                 \
    if (smem > 48 * 1024) HB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    kern<<<grid, 256, smem, st>>>(xproj, w_hh, b_hh, masks, h_prev, h_prev_stride, c_prev, c_prev_stride, h, c,  \
                                  gates_out, n);                                                          \
  }
  switch (hidden / 32) {
    case 1: HB_LSTM(1); break;
    case 2: HB_LSTM(2); break;
    case 4: HB_LSTM(4); break;
    case 8: HB_LSTM(8); break;
    case 16: HB_LSTM(16); break;
    default:
      set_last_error("lstm_step_fwd: hidden=%d unsupported (32,64,128,256,512)", hidden);
      return HB200_ERR_UNSUPPORTED;
  }
#undef HB_LSTM
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

extern "C" int hb200_lstm_step_bwd(const float* dh_out, const float* dh_rec, const float* dc_rec,
                                   const float* gates, const float* c, const float* c_prev,
                                   long long c_prev_stride, const float* w_hh, const uint8_t* masks,
                                   float* dgates, float* dh_prev, float* dc_prev, int n, int hidden,
                                   hb200_stream_t stream) {
  HB_CHECK_ARG(gates && c && c_prev && w_hh && masks && dgates && dh_prev && dc_prev && n > 0,
               "lstm_step_bwd: bad args");
  HB_CHECK_ARG(hidden % 32 == 0, "lstm_step_bwd: hidden must be a multiple of 32");
  cudaStream_t st = (cudaStream_t)stream;
  const int total = n * hidden;
  lstm_step_bwd_pointwise_kernel<<<cdiv(total, 256), 256, 0, st>>>(dh_out, dh_rec, dc_rec, gates, c, c_prev,
                                                                   c_prev_stride, masks, dgates, dh_prev,
                                                                   dc_prev, n, hidden);
  HB_LAUNCH_OK();
  const int R = 4 * hidden;
  int rpb = 256;
  while (R % rpb) rpb >>= 1;
  dim3 grid(hidden / 32, R / rpb);
  lstm_step_bwd_matmul_kernel<4><<<grid, 256, 0, st>>>(dgates, w_hh, masks, dh_prev, n, hidden, rpb);
  HB_LAUNCH_OK();
  count_launch(2);
  return HB200_OK;
}

// =====================================================================================
// Persistent whole-sequence kernels: one cooperative launch per layer instead of T (forward)
// / 2T (backward) launches.  Each CTA keeps its slice of W_hh in shared memory for all T steps
// and the CTAs exchange h_t (forward) / dgates_t (backward) through L2 with one grid barrier per
// step.  Launched with cudaLaunchCooperativeKernel so all CTAs are co-resident.
// =====================================================================================
namespace hb200 {

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void grid_barrier(unsigned* counter, unsigned target) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(counter, 1u);
    // The launch is cooperative (all CTAs co-resident), so the wait always ends; the bound only turns a programming
    // error into a launch failure instead of a hung box.  It is WALL-CLOCK (globaltimer) and generous (30 s): time
    // slicing, MPS, a debugger or profiler replay may stretch a healthy barrier far beyond any cycle budget.
    unsigned long long t0 = 0, now;
    unsigned spins = 0;
    while (ld_acquire_u32(counter) < target) {
      if ((++spins & 0xFFFu) == 0) {
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
        if (t0 == 0) t0 = now;
        else if (now - t0 > 30000000000ull) __trap();
      }
    }
    __threadfence();
  }
  __syncthreads();
}

// transpose-reduce: every lane holds 16 partial sums v[r]; returns in lane l the full warp sum of
// row (l >> 1)  (16 shuffles instead of 16 x 5)
__device__ __forceinline__ float warp_reduce16(float (&v)[16], int lane) {
  float a[8];
  const bool b4 = lane & 16;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float send = b4 ? v[i] : v[i + 8];
    const float keep = b4 ? v[i + 8] : v[i];
    a[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
  }
  float b[4];
  const bool b3 = lane & 8;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float send = b3 ? a[i] : a[i + 4];
    const float keep = b3 ? a[i + 4] : a[i];
    b[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
  }
  float c[2];
  const bool b2 = lane & 4;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const float send = b2 ? b[i] : b[i + 2];
    const float keep = b2 ? b[i + 2] : b[i];
    c[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
  }
  const bool b1 = lane & 2;
  const float send = b1 ? c[0] : c[1];
  const float keep = b1 ? c[1] : c[0];
  float d = keep + __shfl_xor_sync(0xffffffffu, send, 2);
  d += __shfl_xor_sync(0xffffffffu, d, 1);
  return d;
}

constexpr int kSeqThreads = 1024;  // one warp per sequence (n <= 32 in one pass)

template <int NJ>
__global__ void __launch_bounds__(kSeqThreads)
lstm_seq_fwd_kernel(const float* __restrict__ xproj, const float* __restrict__ w_hh,
                    const float* __restrict__ b_hh, const uint8_t* __restrict__ masks,
                    const float* __restrict__ h0, long long h0_stride, const float* __restrict__ c0,
                    long long c0_stride, float* __restrict__ hs, float* __restrict__ cs,
                    float* __restrict__ gates_out, int T, int n, unsigned* counter) {
  constexpr int H = NJ * 32;
  extern __shared__ float sw[];  // [16][H]
  const int u0 = blockIdx.x * kUnits;
  for (int i = threadIdx.x; i < 16 * H; i += blockDim.x) {
    const int r = i / H, k = i - r * H;
    sw[i] = w_hh[((size_t)(r >> 2) * H + u0 + (r & 3)) * H + k];
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  // lane l finishes gate row (l >> 1): row = gate * 4 + unit
  const int row = lane >> 1, gate = row >> 2, unit = row & 3, col = u0 + unit;
  const float bias = b_hh ? b_hh[(size_t)gate * H + col] : 0.f;
  for (int t = 0; t < T; ++t) {
    const float* hp = t == 0 ? h0 : hs + (size_t)(t - 1) * n * H;
    const long long hps = t == 0 ? h0_stride : H;
    const float* cp = t == 0 ? c0 : cs + (size_t)(t - 1) * n * H;
    const long long cps = t == 0 ? c0_stride : H;
    for (int s = warp; s < n; s += nwarps) {
      const float m = masks[(size_t)t * n + s] ? 1.f : 0.f;
      float hv[NJ];
#pragma unroll
      for (int j = 0; j < NJ; ++j) hv[j] = __ldcg(hp + (size_t)s * hps + lane + 32 * j);
      const float xp = xproj[((size_t)t * n + s) * 4 * H + (size_t)gate * H + col];
      const float cprev = __ldcg(cp + (size_t)s * cps + col);
      float part[16];
#pragma unroll
      for (int r = 0; r < 16; ++r) {
        float acc = 0.f;
#pragma unroll
        for (int j = 0; j < NJ; ++j) acc = fmaf(hv[j], sw[r * H + lane + 32 * j], acc);
        part[r] = acc;
      }
      const float pre = warp_reduce16(part, lane) * m + bias + xp;  // (h*m) . w == m * (h . w)
      const float act = (gate == 2) ? tanhf(pre) : sigmoidf_(pre);
      // gather the four gates of this lane's unit: rows unit, 4+unit, 8+unit, 12+unit -> lanes 2*row
      const float i_ = __shfl_sync(0xffffffffu, act, 2 * unit);
      const float f_ = __shfl_sync(0xffffffffu, act, 2 * (4 + unit));
      const float g_ = __shfl_sync(0xffffffffu, act, 2 * (8 + unit));
      const float o_ = __shfl_sync(0xffffffffu, act, 2 * (12 + unit));
      if (lane < 8 && (lane & 1) == 0) {  // lanes 0,2,4,6 own units 0..3
        const float cn = f_ * (cprev * m) + i_ * g_;
        const size_t o = ((size_t)t * n + s) * H + col;
        cs[o] = cn;
        hs[o] = o_ * tanhf(cn);
        if (gates_out) {
          float* gp = gates_out + ((size_t)t * n + s) * 4 * H;
          gp[col] = i_; gp[H + col] = f_; gp[2 * H + col] = g_; gp[3 * H + col] = o_;
        }
      }
    }
    if (t + 1 < T) grid_barrier(counter, (unsigned)(t + 1) * gridDim.x);
  }
}

// backward through time for one layer.  CTA = 4 hidden units: pointwise for its units (dh_rec /
// dc_rec of those units never leave the CTA), publishes its 16 dgates columns, barrier, then its 4
// columns of dh_{t-1} = m_t * dgates_t W_hh  with W_hh^T[:, 4 cols] resident in shared memory.
__global__ void __launch_bounds__(kSeqThreads)
lstm_seq_bwd_kernel(const float* __restrict__ dh_out, const float* __restrict__ gates,
                    const float* __restrict__ cs, const float* __restrict__ c0, long long c0_stride,
                    const float* __restrict__ w_hh, const uint8_t* __restrict__ masks,
                    float* __restrict__ dgates, int T, int n, int H, unsigned* counter) {
  extern __shared__ __align__(16) float smem[];
  const int R = 4 * H;
  float* wt = smem;                 // [4][R]  (unit-major: conflict-free float4 reads along r)
  float* dh_rec = smem + 4 * R;     // [n][4]
  float* dc_rec = dh_rec + 4 * n;   // [n][4]
  const int u0 = blockIdx.x * kUnits;
  for (int i = threadIdx.x; i < 4 * R; i += blockDim.x) {
    const int u = i / R, r = i - u * R;
    wt[i] = w_hh[(size_t)r * H + u0 + u];
  }
  for (int i = threadIdx.x; i < 4 * n; i += blockDim.x) { dh_rec[i] = 0.f; dc_rec[i] = 0.f; }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  for (int t = T - 1; t >= 0; --t) {
    // ---- pointwise for own units
    for (int i = threadIdx.x; i < 4 * n; i += blockDim.x) {
      const int s = i >> 2, col = u0 + (i & 3);
      const size_t row = (size_t)t * n + s;
      const float m = masks[row] ? 1.f : 0.f;
      const float* gt = gates + row * R;
      const float i_ = gt[col], f_ = gt[H + col], g_ = gt[2 * H + col], o_ = gt[3 * H + col];
      const float dh = dh_out[row * H + col] + dh_rec[i];
      const float tc = tanhf(cs[row * H + col]);
      const float dc = dh * o_ * (1.f - tc * tc) + dc_rec[i];
      const float cin = (t == 0 ? c0[(size_t)s * c0_stride + col] : cs[(row - n) * H + col]) * m;
      float* dg = dgates + row * R;
      dg[col] = dc * g_ * i_ * (1.f - i_);
      dg[H + col] = dc * cin * f_ * (1.f - f_);
      dg[2 * H + col] = dc * i_ * (1.f - g_ * g_);
      dg[3 * H + col] = dh * tc * o_ * (1.f - o_);
      dc_rec[i] = dc * f_ * m;
    }
    if (t == 0) break;
    grid_barrier(counter, (unsigned)(T - t) * gridDim.x);
    // ---- dh_{t-1}[s, own 4 cols] = m_t[s] * sum_r dgates_t[s, r] * W_hh[r, col]; one warp per sequence
    for (int s = warp; s < n; s += nwarps) {
      const float4* dg4 = reinterpret_cast<const float4*>(dgates + ((size_t)t * n + s) * R);
      float a0 = 0, a1 = 0, a2 = 0, a3 = 0;
      for (int g0 = 0; g0 < R / 4; g0 += 32 * 4) {  // 4 independent 16-byte loads in flight per lane
        float4 d[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int g = g0 + q * 32 + lane;
          d[q] = (g < R / 4) ? __ldcg(dg4 + g) : make_float4(0, 0, 0, 0);
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int g = g0 + q * 32 + lane;
          if (g < R / 4) {
            const float4 w0 = *reinterpret_cast<const float4*>(wt + 0 * R + 4 * g);
            const float4 w1 = *reinterpret_cast<const float4*>(wt + 1 * R + 4 * g);
            const float4 w2 = *reinterpret_cast<const float4*>(wt + 2 * R + 4 * g);
            const float4 w3 = *reinterpret_cast<const float4*>(wt + 3 * R + 4 * g);
            a0 += d[q].x * w0.x + d[q].y * w0.y + d[q].z * w0.z + d[q].w * w0.w;
            a1 += d[q].x * w1.x + d[q].y * w1.y + d[q].z * w1.z + d[q].w * w1.w;
            a2 += d[q].x * w2.x + d[q].y * w2.y + d[q].z * w2.z + d[q].w * w2.w;
            a3 += d[q].x * w3.x + d[q].y * w3.y + d[q].z * w3.z + d[q].w * w3.w;
          }
        }
      }
      a0 = warp_sum(a0); a1 = warp_sum(a1); a2 = warp_sum(a2); a3 = warp_sum(a3);
      if (lane == 0) {
        const float m = masks[(size_t)t * n + s] ? 1.f : 0.f;
        dh_rec[4 * s] = a0 * m; dh_rec[4 * s + 1] = a1 * m; dh_rec[4 * s + 2] = a2 * m; dh_rec[4 * s + 3] = a3 * m;
      }
    }
    __syncthreads();
  }
}
}  // namespace hb200

// =====================================================================================
// v2 of the persistent LSTM kernels (hidden = 512): register-tiled recurrent mat-vecs.
// v1 gives every sequence its own warp, so each W_hh element is re-read from shared memory once per sequence and
// the step is bound by shared-memory bandwidth (1 LDS per FMA).  Here a warp owns an
// 8-sequence x 8-gate-row (forward) / 8-sequence x 4-column (backward) tile: one 16-byte LDS feeds 8 x 4 FMAs, the
// staged h_{t-1} block / the streamed dgates rows are shared by the whole tile, and the 64 (32) per-lane partial
// sums are finished with one transpose-reduce.
// =====================================================================================
namespace hb200 {

// lane l ends with the warp sums of v[2l], v[2l+1]
__device__ __forceinline__ void warp_reduce64(float (&v)[64], int lane, float& o0, float& o1) {
  float a[32], b[16], c[8], d[4], e[2];
  { const bool hi = lane & 16;
#pragma unroll
    for (int i = 0; i < 32; ++i) { const float send = hi ? v[i] : v[i + 32], keep = hi ? v[i + 32] : v[i];
                                   a[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16); } }
  { const bool hi = lane & 8;
#pragma unroll
    for (int i = 0; i < 16; ++i) { const float send = hi ? a[i] : a[i + 16], keep = hi ? a[i + 16] : a[i];
                                   b[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8); } }
  { const bool hi = lane & 4;
#pragma unroll
    for (int i = 0; i < 8; ++i) { const float send = hi ? b[i] : b[i + 8], keep = hi ? b[i + 8] : b[i];
                                  c[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4); } }
  { const bool hi = lane & 2;
#pragma unroll
    for (int i = 0; i < 4; ++i) { const float send = hi ? c[i] : c[i + 4], keep = hi ? c[i + 4] : c[i];
                                  d[i] = keep + __shfl_xor_sync(0xffffffffu, send, 2); } }
  { const bool hi = lane & 1;
#pragma unroll
    for (int i = 0; i < 2; ++i) { const float send = hi ? d[i] : d[i + 2], keep = hi ? d[i + 2] : d[i];
                                  e[i] = keep + __shfl_xor_sync(0xffffffffu, send, 1); } }
  o0 = e[0];
  o1 = e[1];
}
// lane l ends with the warp sum of v[l]
__device__ __forceinline__ float warp_reduce32(float (&v)[32], int lane) {
  float a[16], b[8], c[4], d[2];
  { const bool hi = lane & 16;
#pragma unroll
    for (int i = 0; i < 16; ++i) { const float send = hi ? v[i] : v[i + 16], keep = hi ? v[i + 16] : v[i];
                                   a[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16); } }
  { const bool hi = lane & 8;
#pragma unroll
    for (int i = 0; i < 8; ++i) { const float send = hi ? a[i] : a[i + 8], keep = hi ? a[i + 8] : a[i];
                                  b[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8); } }
  { const bool hi = lane & 4;
#pragma unroll
    for (int i = 0; i < 4; ++i) { const float send = hi ? b[i] : b[i + 4], keep = hi ? b[i + 4] : b[i];
                                  c[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4); } }
  { const bool hi = lane & 2;
#pragma unroll
    for (int i = 0; i < 2; ++i) { const float send = hi ? c[i] : c[i + 2], keep = hi ? c[i + 2] : c[i];
                                  d[i] = keep + __shfl_xor_sync(0xffffffffu, send, 2); } }
  const bool hi = lane & 1;
  const float send = hi ? d[0] : d[1], keep = hi ? d[1] : d[0];
  return keep + __shfl_xor_sync(0xffffffffu, send, 1);
}

constexpr int kV2Threads = 256;

template <int H>
__global__ void __launch_bounds__(kV2Threads)
lstm_seq_fwd_v2_kernel(const float* __restrict__ xproj, const float* __restrict__ w_hh,
                       const float* __restrict__ b_hh, const uint8_t* __restrict__ masks,
                       const float* __restrict__ h0, long long h0_stride, const float* __restrict__ c0,
                       long long c0_stride, float* __restrict__ hs, float* __restrict__ cs,
                       float* __restrict__ gates_out, int T, int n, unsigned* counter) {
  extern __shared__ __align__(16) float sm2[];
  float* sw = sm2;             // [16][H]   row = gate * 4 + unit
  float* sh = sw + 16 * H;     // [32][H]   h_{t-1} of the current block of 32 sequences
  float* spre = sh + 32 * H;   // [32][16]  recurrent pre-activation sums
  const int u0 = blockIdx.x * kUnits;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < 16 * H; i += kV2Threads) {
    const int r = i / H, k = i - r * H;
    sw[i] = w_hh[((size_t)(r >> 2) * H + u0 + (r & 3)) * H + k];
  }
  const int sg = warp & 3, rg = warp >> 2;           // 8-sequence group, 8-row group of this warp's tile
  const int ps = tid >> 2, pu = tid & 3, col = u0 + pu;  // pointwise role (threads 0..127)
  float bias[4] = {0.f, 0.f, 0.f, 0.f};
  if (b_hh && tid < 128) {
#pragma unroll
    for (int g = 0; g < 4; ++g) bias[g] = b_hh[(size_t)g * H + col];
  }
  __syncthreads();
  for (int t = 0; t < T; ++t) {
    asm volatile("" ::: "memory");  // keep step t+1's operand loads (xproj / masks rows) below this step's exit test
    const float* hp = t == 0 ? h0 : hs + (size_t)(t - 1) * n * H;
    const long long hps = t == 0 ? h0_stride : H;
    const float* cp = t == 0 ? c0 : cs + (size_t)(t - 1) * n * H;
    const long long cps = t == 0 ? c0_stride : H;
    for (int s0 = 0; s0 < n; s0 += 32) {
      const int ns = min(32, n - s0);
      // pointwise operands do not depend on the mat-vec: fetch them first
      float xp[4] = {0.f, 0.f, 0.f, 0.f}, cprev = 0.f, m = 0.f;
      const bool pw = tid < 128 && ps < ns;
      if (pw) {
        const size_t row = (size_t)t * n + s0 + ps;
        m = masks[row] ? 1.f : 0.f;
#pragma unroll
        for (int g = 0; g < 4; ++g) xp[g] = xproj[row * 4 * H + (size_t)g * H + col];
        cprev = __ldcg(cp + (size_t)(s0 + ps) * cps + col);   // written by this very thread one step ago
      }
      // stage h_{t-1} of the block (written by all CTAs in the previous step: L2 loads)
      float4* sh4 = reinterpret_cast<float4*>(sh);
      {
        constexpr int NV = 32 * (H / 4) / kV2Threads;  // 16 vectors per thread, all in flight at once
        float4 v[NV];
#pragma unroll
        for (int q = 0; q < NV; ++q) {
          const int i = tid + q * kV2Threads, row = i / (H / 4), c4 = i - row * (H / 4);
          v[q] = row < ns ? __ldcg(reinterpret_cast<const float4*>(hp + (size_t)(s0 + row) * hps) + c4)
                          : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int q = 0; q < NV; ++q) sh4[tid + q * kV2Threads] = v[q];
      }
      __syncthreads();
      float acc[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] = 0.f;
#pragma unroll 1
      for (int jj = 0; jj < H / 128; ++jj) {
        const int k = 4 * lane + 128 * jj;
        float4 wv[8];
#pragma unroll
        for (int r = 0; r < 8; ++r) wv[r] = *reinterpret_cast<const float4*>(sw + (rg * 8 + r) * H + k);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float4 hv = *reinterpret_cast<const float4*>(sh + (sg * 8 + i) * H + k);
#pragma unroll
          for (int r = 0; r < 8; ++r) {
            float a = acc[i * 8 + r];
            a = fmaf(hv.x, wv[r].x, a);
            a = fmaf(hv.y, wv[r].y, a);
            a = fmaf(hv.z, wv[r].z, a);
            a = fmaf(hv.w, wv[r].w, a);
            acc[i * 8 + r] = a;
          }
        }
      }
      float o0, o1;
      warp_reduce64(acc, lane, o0, o1);  // lane -> sequence (lane >> 2), rows 2 * (lane & 3) + {0, 1} of the tile
      *reinterpret_cast<float2*>(spre + (sg * 8 + (lane >> 2)) * 16 + rg * 8 + 2 * (lane & 3)) = make_float2(o0, o1);
      __syncthreads();
      if (pw) {
        const float* pr = spre + ps * 16 + pu;
        const float i_ = sigmoidf_(pr[0] * m + bias[0] + xp[0]);   // (h*m) . w == m * (h . w)
        const float f_ = sigmoidf_(pr[4] * m + bias[1] + xp[1]);
        const float g_ = tanhf(pr[8] * m + bias[2] + xp[2]);
        const float o_ = sigmoidf_(pr[12] * m + bias[3] + xp[3]);
        const float cn = f_ * (cprev * m) + i_ * g_;
        const size_t o = ((size_t)t * n + s0 + ps) * H + col;
        cs[o] = cn;
        hs[o] = o_ * tanhf(cn);
        if (gates_out) {
          float* gp = gates_out + ((size_t)t * n + s0 + ps) * 4 * H;
          gp[col] = i_; gp[H + col] = f_; gp[2 * H + col] = g_; gp[3 * H + col] = o_;
        }
      }
    }
    if (t + 1 < T) grid_barrier(counter, (unsigned)(t + 1) * gridDim.x);
  }
}

template <int H>
__global__ void __launch_bounds__(kV2Threads)
lstm_seq_bwd_v2_kernel(const float* __restrict__ dh_out, const float* __restrict__ gates,
                       const float* __restrict__ cs, const float* __restrict__ c0, long long c0_stride,
                       const float* __restrict__ w_hh, const uint8_t* __restrict__ masks,
                       float* __restrict__ dgates, int T, int n, unsigned* counter, float* __restrict__ carry,
                       int carry_in, int carry_out) {
  // carry [2][n][H] (dh, dc of the step before this launch's first one): lets a sequence be processed as several
  // launches over time chunks (last chunk first), so that two layers can run as a wavefront on two streams
  extern __shared__ __align__(16) float sm2[];
  constexpr int R = 4 * H;
  float* wt = sm2;                 // [4][R]  W_hh^T columns of this CTA's 4 units
  float* spart = wt + 4 * R;       // [2][32][4]  partial dh_rec of the two r-halves
  float* dh_rec = spart + 256;     // [n][4]
  float* dc_rec = dh_rec + 4 * n;  // [n][4]
  const int u0 = blockIdx.x * kUnits;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < 4 * R; i += kV2Threads) {
    const int u = i / R, r = i - u * R;
    wt[i] = w_hh[(size_t)r * H + u0 + u];
  }
  for (int i = tid; i < 4 * n; i += kV2Threads) {
    const size_t o = (size_t)(i >> 2) * H + u0 + (i & 3);
    dh_rec[i] = carry_in ? carry[o] : 0.f;
    dc_rec[i] = carry_in ? carry[(size_t)n * H + o] : 0.f;
  }
  __syncthreads();
  const int sg = warp & 3, rh = warp >> 2;  // 8-sequence group, half of the 4H gate rows
  for (int t = T - 1; t >= 0; --t) {
    // compiler barrier: without a grid barrier in the loop nvcc software-pipelines the read-only (LDG.CONSTANT)
    // operand loads of step t-1 above the exit test of step t and reads rows -n..-1 of gates / dh_out at t = 0
    asm volatile("" ::: "memory");
    // ---- pointwise for own units (identical to v1)
    for (int i = tid; i < 4 * n; i += kV2Threads) {
      const int s = i >> 2, col = u0 + (i & 3);
      const size_t row = (size_t)t * n + s;
      const float m = masks[row] ? 1.f : 0.f;
      const float* gt = gates + row * R;
      const float i_ = gt[col], f_ = gt[H + col], g_ = gt[2 * H + col], o_ = gt[3 * H + col];
      const float dh = dh_out[row * H + col] + dh_rec[i];
      const float tc = tanhf(cs[row * H + col]);
      const float dc = dh * o_ * (1.f - tc * tc) + dc_rec[i];
      const float cin = (t == 0 ? c0[(size_t)s * c0_stride + col] : cs[(row - n) * H + col]) * m;
      float* dg = dgates + row * R;
      dg[col] = dc * g_ * i_ * (1.f - i_);
      dg[H + col] = dc * cin * f_ * (1.f - f_);
      dg[2 * H + col] = dc * i_ * (1.f - g_ * g_);
      dg[3 * H + col] = dh * tc * o_ * (1.f - o_);
      dc_rec[i] = dc * f_ * m;
    }
    if (t == 0 && !carry_out) break;
    grid_barrier(counter, (unsigned)(T - t) * gridDim.x);
    asm volatile("" ::: "memory");
    // ---- dh_{t-1}[s, own 4 cols] = m_t[s] * sum_r dgates_t[s, r] * W_hh[r, col]
    for (int s0 = 0; s0 < n; s0 += 32) {
      float acc[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[i] = 0.f;
      const float* dgt = dgates + ((size_t)t * n + s0 + sg * 8) * R + rh * (R / 2) + 4 * lane;
      const int nrows = min(8, n - s0 - sg * 8);  // sequences of this tile that exist (<= 0: none)
#pragma unroll 2
      for (int jj = 0; jj < R / 2 / 128; ++jj) {
        float4 d[8];
#pragma unroll
        for (int i = 0; i < 8; ++i)
          d[i] = i < nrows ? __ldcg(reinterpret_cast<const float4*>(dgt + (size_t)i * R + jj * 128))
                           : make_float4(0.f, 0.f, 0.f, 0.f);
        const int r = rh * (R / 2) + jj * 128 + 4 * lane;
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const float4 w = *reinterpret_cast<const float4*>(wt + u * R + r);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            float a = acc[i * 4 + u];
            a = fmaf(d[i].x, w.x, a);
            a = fmaf(d[i].y, w.y, a);
            a = fmaf(d[i].z, w.z, a);
            a = fmaf(d[i].w, w.w, a);
            acc[i * 4 + u] = a;
          }
        }
      }
      const float v = warp_reduce32(acc, lane);  // lane -> sequence (lane >> 2), unit (lane & 3) of the tile
      spart[rh * 128 + sg * 32 + lane] = v;
      __syncthreads();
      if (tid < 128 && s0 + (tid >> 2) < n) {
        const int s = s0 + (tid >> 2);
        const float m = masks[(size_t)t * n + s] ? 1.f : 0.f;
        dh_rec[4 * s + (tid & 3)] = (spart[tid] + spart[128 + tid]) * m;
      }
      __syncthreads();
    }
    if (t == 0) {   // carry_out: hand the recurrent gradients to the launch that covers the earlier steps
      for (int i = tid; i < 4 * n; i += kV2Threads) {
        const size_t o = (size_t)(i >> 2) * H + u0 + (i & 3);
        carry[o] = dh_rec[i];
        carry[(size_t)n * H + o] = dc_rec[i];
      }
      break;
    }
  }
}
}  // namespace hb200

static int coop_check(const void* kern, int block, size_t smem, int grid) {
  int per_sm = 0;
  HB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, block, smem));
  int dev = 0, sms = 0;
  HB_CUDA(cudaGetDevice(&dev));
  HB_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  if (per_sm * sms < grid) {
    set_last_error("lstm_seq: %d CTAs cannot be co-resident (%d per SM x %d SMs)", grid, per_sm, sms);
    return HB200_ERR_UNSUPPORTED;
  }
  return HB200_OK;
}

extern "C" int hb200_lstm_seq_fwd(const float* xproj, const float* w_hh, const float* b_hh,
                                  const uint8_t* masks, const float* h0, long long h0_stride,
                                  const float* c0, long long c0_stride, float* hs, float* cs,
                                  float* gates_out, int t_steps, int n, int hidden, void* workspace,
                                  hb200_stream_t stream) {
  HB_CHECK_ARG(xproj && w_hh && masks && h0 && c0 && hs && cs && workspace && t_steps > 0 && n > 0,
               "lstm_seq_fwd: bad args");
  HB_CHECK_ARG(hidden == 32 || hidden == 64 || hidden == 128 || hidden == 256 || hidden == 512,
               "lstm_seq_fwd: hidden=%d unsupported (32,64,128,256,512)", hidden);
  cudaStream_t st = (cudaStream_t)stream;
  unsigned* counter = (unsigned*)workspace;
  HB_CUDA(cudaMemsetAsync(counter, 0, sizeof(unsigned), st));
  const int grid = hidden / kUnits;
  void* args[] = {(void*)&xproj, (void*)&w_hh, (void*)&b_hh, (void*)&masks, (void*)&h0, (void*)&h0_stride,
                  (void*)&c0, (void*)&c0_stride, (void*)&hs, (void*)&cs, (void*)&gates_out, (void*)&t_steps,
                  (void*)&n, (void*)&counter};
  static const bool use_v1 = getenv("HB200_LSTM_V1") != nullptr;
  if (hidden == 512 && !use_v1 && h0_stride % 4 == 0 && ((uintptr_t)h0 & 15) == 0 && ((uintptr_t)hs & 15) == 0) {
    const void* k2 = (const void*)lstm_seq_fwd_v2_kernel<512>;
    const size_t smem2 = sizeof(float) * (16 * 512 + 32 * 512 + 32 * 16);
    HB_CUDA(cudaFuncSetAttribute(k2, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2));
    int rc2 = coop_check(k2, kV2Threads, smem2, grid);
    if (rc2) return rc2;
    HB_CUDA(cudaLaunchCooperativeKernel(k2, dim3(grid), dim3(kV2Threads), args, smem2, st));
    count_launch(1);
    return HB200_OK;
  }
  const size_t smem = sizeof(float) * 16 * hidden;
  const void* kern = nullptr;
  switch (hidden / 32) {
    case 1: kern = (const void*)lstm_seq_fwd_kernel<1>; break;
    case 2: kern = (const void*)lstm_seq_fwd_kernel<2>; break;
    case 4: kern = (const void*)lstm_seq_fwd_kernel<4>; break;
    case 8: kern = (const void*)lstm_seq_fwd_kernel<8>; break;
    default: kern = (const void*)lstm_seq_fwd_kernel<16>; break;
  }
  if (smem > 48 * 1024) HB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int rc = coop_check(kern, kSeqThreads, smem, grid);
  if (rc) return rc;
  HB_CUDA(cudaLaunchCooperativeKernel(kern, dim3(grid), dim3(kSeqThreads), args, smem, st));
  count_launch(1);
  return HB200_OK;
}

static int lstm_seq_bwd_impl(const float* dh_out, const float* gates, const float* cs, const float* c0,
                             long long c0_stride, const float* w_hh, const uint8_t* masks, float* dgates,
                             int t_steps, int n, int hidden, void* workspace, float* carry, int carry_in,
                             int carry_out, hb200_stream_t stream) {
  HB_CHECK_ARG(dh_out && gates && cs && c0 && w_hh && masks && dgates && workspace && t_steps > 0 && n > 0,
               "lstm_seq_bwd: bad args");
  HB_CHECK_ARG(hidden % kUnits == 0 && hidden % 32 == 0, "lstm_seq_bwd: hidden must be a multiple of 32");
  // both kernels read the dgates rows of step t back with 16-byte loads for the dh_{t-1} mat-vec
  HB_CHECK_ARG(((uintptr_t)dgates & 15) == 0, "lstm_seq_bwd: dgates must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  unsigned* counter = (unsigned*)workspace;
  HB_CUDA(cudaMemsetAsync(counter, 0, sizeof(unsigned), st));
  const size_t smem = sizeof(float) * (16 * (size_t)hidden + 8 * (size_t)n);
  HB_CHECK_ARG(smem <= 200 * 1024, "lstm_seq_bwd: n=%d too large for one CTA's shared memory", n);
  const int grid = hidden / kUnits;
  static const bool use_v1 = getenv("HB200_LSTM_V1") != nullptr;
  if (hidden == 512 && !use_v1) {
    const void* k2 = (const void*)lstm_seq_bwd_v2_kernel<512>;
    const size_t smem2 = smem + sizeof(float) * 256;
    void* args2[] = {(void*)&dh_out, (void*)&gates, (void*)&cs, (void*)&c0, (void*)&c0_stride, (void*)&w_hh,
                     (void*)&masks, (void*)&dgates, (void*)&t_steps, (void*)&n, (void*)&counter,
                     (void*)&carry, (void*)&carry_in, (void*)&carry_out};
    if (smem2 > 48 * 1024) HB_CUDA(cudaFuncSetAttribute(k2, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2));
    int rc2 = coop_check(k2, kV2Threads, smem2, grid);
    if (rc2) return rc2;
    HB_CUDA(cudaLaunchCooperativeKernel(k2, dim3(grid), dim3(kV2Threads), args2, smem2, st));
    count_launch(1);
    return HB200_OK;
  }
  HB_CHECK_ARG(!carry_in && !carry_out, "lstm_seq_bwd: time chunks (carry) need hidden == 512");
  const void* kern = (const void*)lstm_seq_bwd_kernel;
  if (smem > 48 * 1024) HB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int rc = coop_check(kern, kSeqThreads, smem, grid);
  if (rc) return rc;
  void* args[] = {(void*)&dh_out, (void*)&gates, (void*)&cs, (void*)&c0, (void*)&c0_stride, (void*)&w_hh,
                  (void*)&masks, (void*)&dgates, (void*)&t_steps, (void*)&n, (void*)&hidden, (void*)&counter};
  HB_CUDA(cudaLaunchCooperativeKernel(kern, dim3(grid), dim3(kSeqThreads), args, smem, st));
  count_launch(1);
  return HB200_OK;
}

extern "C" int hb200_lstm_seq_bwd(const float* dh_out, const float* gates, const float* cs, const float* c0,
                                  long long c0_stride, const float* w_hh, const uint8_t* masks, float* dgates,
                                  int t_steps, int n, int hidden, void* workspace, hb200_stream_t stream) {
  return lstm_seq_bwd_impl(dh_out, gates, cs, c0, c0_stride, w_hh, masks, dgates, t_steps, n, hidden, workspace, nullptr,
                           0, 0, stream);
}
extern "C" int hb200_lstm_seq_bwd_chunk(const float* dh_out, const float* gates, const float* cs, const float* c0,
                                        long long c0_stride, const float* w_hh, const uint8_t* masks, float* dgates,
                                        int t_steps, int n, int hidden, void* workspace, float* carry, int carry_in,
                                        int carry_out, hb200_stream_t stream) {
  HB_CHECK_ARG(carry || (!carry_in && !carry_out), "lstm_seq_bwd_chunk: carry buffer missing");
  return lstm_seq_bwd_impl(dh_out, gates, cs, c0, c0_stride, w_hh, masks, dgates, t_steps, n, hidden, workspace, carry,
                           carry_in, carry_out, stream);
}

// =====================================================================================
// GRU (rnn_type GRU: PointNavBaselinePolicy / config #1, ObjectNav config #3), PyTorch gate order r,z,n:
//   r = sig(xr + Whr h + bhr)   z = sig(xz + Whz h + bhz)   n = tanh(xn + r * (Whn h + bhn))
//   h' = (1 - z) * n + z * h          with h = h_{t-1} * m_t  (mask resets before the step)
// xproj [T*n, 3H] = x W_ih^T + b_ih (one GEMM for all frames); same persistent cooperative structure as
// the LSTM kernels: one CTA = 4 hidden units (12 gate rows of W_hh in shared memory).
// saved [T,n,4H] = (r, z, n, hn_pre = Whn h + bhn) for the backward pass.
// =====================================================================================
namespace hb200 {

template <int NJ>
__global__ void __launch_bounds__(kSeqThreads)
gru_seq_fwd_kernel(const float* __restrict__ xproj, const float* __restrict__ w_hh,
                   const float* __restrict__ b_hh, const uint8_t* __restrict__ masks,
                   const float* __restrict__ h0, long long h0_stride, float* __restrict__ hs,
                   float* __restrict__ saved, int T, int n, unsigned* counter) {
  constexpr int H = NJ * 32;
  extern __shared__ float sw[];  // [16][H]: rows 0..11 = (gate, unit), rows 12..15 zero padding
  const int u0 = blockIdx.x * kUnits;
  for (int i = threadIdx.x; i < 16 * H; i += blockDim.x) {
    const int r = i / H, k = i - r * H;
    sw[i] = (r < 12) ? w_hh[((size_t)(r >> 2) * H + u0 + (r & 3)) * H + k] : 0.f;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int row = lane >> 1, gate = row >> 2, unit = row & 3, col = u0 + unit;
  const float bias = (b_hh && gate < 3) ? b_hh[(size_t)gate * H + col] : 0.f;
  for (int t = 0; t < T; ++t) {
    const float* hp = t == 0 ? h0 : hs + (size_t)(t - 1) * n * H;
    const long long hps = t == 0 ? h0_stride : H;
    for (int s = warp; s < n; s += nwarps) {
      const float m = masks[(size_t)t * n + s] ? 1.f : 0.f;
      float hv[NJ];
#pragma unroll
      for (int j = 0; j < NJ; ++j) hv[j] = __ldcg(hp + (size_t)s * hps + lane + 32 * j);
      const float xp = gate < 3 ? xproj[((size_t)t * n + s) * 3 * H + (size_t)gate * H + col] : 0.f;
      const float hprev = __ldcg(hp + (size_t)s * hps + col) * m;
      float part[16];
#pragma unroll
      for (int r = 0; r < 16; ++r) {
        float acc = 0.f;
#pragma unroll
        for (int j = 0; j < NJ; ++j) acc = fmaf(hv[j], sw[r * H + lane + 32 * j], acc);
        part[r] = acc;
      }
      const float hdot = warp_reduce16(part, lane) * m + bias;  // W_h* (h*m) + b_h*   for this lane's row
      // lanes 2*unit hold r-row, 2*(4+unit) z-row, 2*(8+unit) n-row
      const float hr = __shfl_sync(0xffffffffu, hdot, 2 * unit), xr = __shfl_sync(0xffffffffu, xp, 2 * unit);
      const float hz = __shfl_sync(0xffffffffu, hdot, 2 * (4 + unit)), xz = __shfl_sync(0xffffffffu, xp, 2 * (4 + unit));
      const float hn = __shfl_sync(0xffffffffu, hdot, 2 * (8 + unit)), xn = __shfl_sync(0xffffffffu, xp, 2 * (8 + unit));
      if (lane < 8 && (lane & 1) == 0) {
        const float r_ = sigmoidf_(xr + hr), z_ = sigmoidf_(xz + hz);
        const float n_ = tanhf(xn + r_ * hn);
        const size_t o = ((size_t)t * n + s) * H + col;
        hs[o] = (1.f - z_) * n_ + z_ * hprev;
        if (saved) {
          float* sp = saved + ((size_t)t * n + s) * 4 * H;
          sp[col] = r_; sp[H + col] = z_; sp[2 * H + col] = n_; sp[3 * H + col] = hn;
        }
      }
    }
    if (t + 1 < T) grid_barrier(counter, (unsigned)(t + 1) * gridDim.x);
  }
}

// dgx [T,n,3H] = d(xproj) = (dr_pre, dz_pre, dn_pre);  dgh [T,n,3H] = d(h-side pre-activations) =
// (dr_pre, dz_pre, dn_pre * r).  dh_{t-1} = m_t * (dh * z + dgh W_hh).
__global__ void __launch_bounds__(kSeqThreads)
gru_seq_bwd_kernel(const float* __restrict__ dh_out, const float* __restrict__ saved,
                   const float* __restrict__ hs, const float* __restrict__ h0, long long h0_stride,
                   const float* __restrict__ w_hh, const uint8_t* __restrict__ masks,
                   float* __restrict__ dgx, float* __restrict__ dgh, int T, int n, int H, unsigned* counter) {
  extern __shared__ __align__(16) float smem[];
  const int R = 3 * H;
  float* wt = smem;               // [4][R]
  float* dh_rec = smem + 4 * R;   // [n][4]
  const int u0 = blockIdx.x * kUnits;
  for (int i = threadIdx.x; i < 4 * R; i += blockDim.x) {
    const int u = i / R, r = i - u * R;
    wt[i] = w_hh[(size_t)r * H + u0 + u];
  }
  for (int i = threadIdx.x; i < 4 * n; i += blockDim.x) dh_rec[i] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  for (int t = T - 1; t >= 0; --t) {
    for (int i = threadIdx.x; i < 4 * n; i += blockDim.x) {
      const int s = i >> 2, col = u0 + (i & 3);
      const size_t row = (size_t)t * n + s;
      const float m = masks[row] ? 1.f : 0.f;
      const float* sp = saved + row * 4 * H;
      const float r_ = sp[col], z_ = sp[H + col], n_ = sp[2 * H + col], hn = sp[3 * H + col];
      const float hin = (t == 0 ? h0[(size_t)s * h0_stride + col] : hs[(row - n) * H + col]) * m;
      const float dh = dh_out[row * H + col] + dh_rec[i];
      const float dn_pre = dh * (1.f - z_) * (1.f - n_ * n_);
      const float dz_pre = dh * (hin - n_) * z_ * (1.f - z_);
      const float dr_pre = dn_pre * hn * r_ * (1.f - r_);
      float* gx = dgx + row * R;
      float* gh = dgh + row * R;
      gx[col] = dr_pre; gx[H + col] = dz_pre; gx[2 * H + col] = dn_pre;
      gh[col] = dr_pre; gh[H + col] = dz_pre; gh[2 * H + col] = dn_pre * r_;
      dh_rec[i] = dh * z_ * m;  // direct path; the W_hh path is added below
    }
    if (t == 0) break;
    grid_barrier(counter, (unsigned)(T - t) * gridDim.x);
    for (int s = warp; s < n; s += nwarps) {
      const float4* g4 = reinterpret_cast<const float4*>(dgh + ((size_t)t * n + s) * R);
      float a0 = 0, a1 = 0, a2 = 0, a3 = 0;
      for (int g0 = 0; g0 < R / 4; g0 += 32 * 4) {
        float4 d[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int g = g0 + q * 32 + lane;
          d[q] = (g < R / 4) ? __ldcg(g4 + g) : make_float4(0, 0, 0, 0);
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int g = g0 + q * 32 + lane;
          if (g < R / 4) {
            const float4 w0 = *reinterpret_cast<const float4*>(wt + 0 * R + 4 * g);
            const float4 w1 = *reinterpret_cast<const float4*>(wt + 1 * R + 4 * g);
            const float4 w2 = *reinterpret_cast<const float4*>(wt + 2 * R + 4 * g);
            const float4 w3 = *reinterpret_cast<const float4*>(wt + 3 * R + 4 * g);
            a0 += d[q].x * w0.x + d[q].y * w0.y + d[q].z * w0.z + d[q].w * w0.w;
            a1 += d[q].x * w1.x + d[q].y * w1.y + d[q].z * w1.z + d[q].w * w1.w;
            a2 += d[q].x * w2.x + d[q].y * w2.y + d[q].z * w2.z + d[q].w * w2.w;
            a3 += d[q].x * w3.x + d[q].y * w3.y + d[q].z * w3.z + d[q].w * w3.w;
          }
        }
      }
      a0 = warp_sum(a0); a1 = warp_sum(a1); a2 = warp_sum(a2); a3 = warp_sum(a3);
      if (lane == 0) {
        const float m = masks[(size_t)t * n + s] ? 1.f : 0.f;
        dh_rec[4 * s] += a0 * m; dh_rec[4 * s + 1] += a1 * m; dh_rec[4 * s + 2] += a2 * m; dh_rec[4 * s + 3] += a3 * m;
      }
    }
    __syncthreads();
  }
}
}  // namespace hb200

extern "C" int hb200_gru_seq_fwd(const float* xproj, const float* w_hh, const float* b_hh, const uint8_t* masks,
                                 const float* h0, long long h0_stride, float* hs, float* saved, int t_steps, int n,
                                 int hidden, void* workspace, hb200_stream_t stream) {
  HB_CHECK_ARG(xproj && w_hh && masks && h0 && hs && workspace && t_steps > 0 && n > 0, "gru_seq_fwd: bad args");
  HB_CHECK_ARG(hidden == 32 || hidden == 64 || hidden == 128 || hidden == 256 || hidden == 512,
               "gru_seq_fwd: hidden=%d unsupported (32,64,128,256,512)", hidden);
  cudaStream_t st = (cudaStream_t)stream;
  unsigned* counter = (unsigned*)workspace;
  HB_CUDA(cudaMemsetAsync(counter, 0, sizeof(unsigned), st));
  const size_t smem = sizeof(float) * 16 * hidden;
  const int grid = hidden / kUnits;
  void* args[] = {(void*)&xproj, (void*)&w_hh, (void*)&b_hh, (void*)&masks, (void*)&h0, (void*)&h0_stride,
                  (void*)&hs, (void*)&saved, (void*)&t_steps, (void*)&n, (void*)&counter};
  const void* kern = nullptr;
  switch (hidden / 32) {
    case 1: kern = (const void*)gru_seq_fwd_kernel<1>; break;
    case 2: kern = (const void*)gru_seq_fwd_kernel<2>; break;
    case 4: kern = (const void*)gru_seq_fwd_kernel<4>; break;
    case 8: kern = (const void*)gru_seq_fwd_kernel<8>; break;
    default: kern = (const void*)gru_seq_fwd_kernel<16>; break;
  }
  if (smem > 48 * 1024) HB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int rc = coop_check(kern, kSeqThreads, smem, grid);
  if (rc) return rc;
  HB_CUDA(cudaLaunchCooperativeKernel(kern, dim3(grid), dim3(kSeqThreads), args, smem, st));
  count_launch(1);
  return HB200_OK;
}

extern "C" int hb200_gru_seq_bwd(const float* dh_out, const float* saved, const float* hs, const float* h0,
                                 long long h0_stride, const float* w_hh, const uint8_t* masks, float* dgx, float* dgh,
                                 int t_steps, int n, int hidden, void* workspace, hb200_stream_t stream) {
  HB_CHECK_ARG(dh_out && saved && hs && h0 && w_hh && masks && dgx && dgh && workspace && t_steps > 0 && n > 0,
               "gru_seq_bwd: bad args");
  HB_CHECK_ARG(hidden % 32 == 0 && hidden % kUnits == 0, "gru_seq_bwd: hidden must be a multiple of 32");
  // the dh_{t-1} mat-vec reads the dgh rows of step t back with 16-byte loads
  HB_CHECK_ARG(((uintptr_t)dgh & 15) == 0, "gru_seq_bwd: dgh must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  unsigned* counter = (unsigned*)workspace;
  HB_CUDA(cudaMemsetAsync(counter, 0, sizeof(unsigned), st));
  const size_t smem = sizeof(float) * (12 * (size_t)hidden + 4 * (size_t)n);
  HB_CHECK_ARG(smem <= 200 * 1024, "gru_seq_bwd: n=%d too large for one CTA's shared memory", n);
  const int grid = hidden / kUnits;
  const void* kern = (const void*)gru_seq_bwd_kernel;
  if (smem > 48 * 1024) HB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  int rc = coop_check(kern, kSeqThreads, smem, grid);
  if (rc) return rc;
  void* args[] = {(void*)&dh_out, (void*)&saved, (void*)&hs, (void*)&h0, (void*)&h0_stride, (void*)&w_hh,
                  (void*)&masks, (void*)&dgx, (void*)&dgh, (void*)&t_steps, (void*)&n, (void*)&hidden, (void*)&counter};
  HB_CUDA(cudaLaunchCooperativeKernel(kern, dim3(grid), dim3(kSeqThreads), args, smem, st));
  count_launch(1);
  return HB200_OK;
}
