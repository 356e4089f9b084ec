// hb200 -- the HBM-/latency-bound PPO pieces: GAE return scan + advantages, advantage
// normalisation, action/value heads + clipped-surrogate/value/entropy loss (fwd+bwd),
// gradient-norm + clip + Adam on flat buffers.
#include <math.h>
#include <stdarg.h>

#include "common.cuh"

namespace hb200 {
static thread_local char g_err[512] = "";
static long long g_launches = 0;
void set_last_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
void count_launch(int n) { g_launches += n; }
}  // namespace hb200

using namespace hb200;

extern "C" const char* hb200_last_error(void) { return hb200::g_err; }
extern "C" int hb200_version(void) { return 100; }
extern "C" long long hb200_launch_count(void) { return hb200::g_launches; }

// =====================================================================================
// GAE  (HB/common/rollout_storage.py:174-205) + advantages (HB/rl/ppo/ppo.py:139-149)
// =====================================================================================
// The reference evaluates, per step and in fp32 with separate (unfused) ops:
//   delta = rewards[t] + gamma * V[t+1] * m[t+1] - V[t]
//   gae   = delta + gamma * tau * gae * m[t+1]          (gamma*tau folded in double by python)
//   R[t]  = gae + V[t]
// __fmul_rn/__fadd_rn keep nvcc from contracting to FMA so variant 1 is bit-exact with it.
__device__ __forceinline__ void acc_stats(float a, double& s, double& ss, double& cnt) {
  if (isfinite(a)) {
    s += (double)a;
    ss += (double)a * (double)a;
    cnt += 1.0;
  }
}

__global__ void gae_serial_kernel(const float* __restrict__ rewards, float* __restrict__ values,
                                  const uint8_t* __restrict__ masks,
                                  const float* __restrict__ next_value, float* __restrict__ returns,
                                  float* __restrict__ adv, double* __restrict__ stats, int T,
                                  int Talloc, int N, float gamma, float gt, int use_gae) {
  __shared__ double red[32];
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  double s = 0, ss = 0, cnt = 0;
  if (n < N) {
    const float nv = next_value[n];
    const bool want_adv = adv != nullptr;
    if (use_gae) {
      values[(size_t)T * N + n] = nv;
      float gae = 0.f, v_next = nv;
      // U time steps of loads are issued before the (serial, order-preserving) recurrence consumes them: the
      // chain is 4 dependent FP ops per step, the loads are what must be in flight.  Advantages come out of the
      // same pass: adv = fl(fl(gae + v) - v), exactly what `returns - value_preds` gives the reference.
      constexpr int U = 8;
      int t = T - 1;
      for (; t >= U - 1; t -= U) {
        float r[U], v[U];
        uint8_t mk[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const size_t i = (size_t)(t - u) * N + n;
          r[u] = rewards[i];
          v[u] = values[i];
          mk[u] = masks[i + N];
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const size_t i = (size_t)(t - u) * N + n;
          const float m = mk[u] ? 1.f : 0.f;
          const float delta = __fsub_rn(__fadd_rn(r[u], __fmul_rn(__fmul_rn(gamma, v_next), m)), v[u]);
          gae = __fadd_rn(delta, __fmul_rn(__fmul_rn(gt, gae), m));
          const float ret = __fadd_rn(gae, v[u]);
          returns[i] = ret;
          if (want_adv) {
            const float a = __fsub_rn(ret, v[u]);
            adv[i] = a;
            acc_stats(a, s, ss, cnt);
          }
          v_next = v[u];
        }
      }
      for (; t >= 0; --t) {
        const size_t i = (size_t)t * N + n;
        const float m = masks[i + N] ? 1.f : 0.f;
        const float r = rewards[i], v = values[i];
        const float delta = __fsub_rn(__fadd_rn(r, __fmul_rn(__fmul_rn(gamma, v_next), m)), v);
        gae = __fadd_rn(delta, __fmul_rn(__fmul_rn(gt, gae), m));
        const float ret = __fadd_rn(gae, v);
        returns[i] = ret;
        if (want_adv) {
          const float a = __fsub_rn(ret, v);
          adv[i] = a;
          acc_stats(a, s, ss, cnt);
        }
        v_next = v;
      }
      if (want_adv) {
        for (int t2 = T; t2 < Talloc; ++t2) {  // bootstrap row + stale rows of an early-ended rollout
          const size_t i = (size_t)t2 * N + n;
          const float a = __fsub_rn(returns[i], t2 == T ? nv : values[i]);
          adv[i] = a;
          acc_stats(a, s, ss, cnt);
        }
      }
    } else {
      returns[(size_t)T * N + n] = nv;
      float ret = nv;
      for (int t = T - 1; t >= 0; --t) {
        const size_t i = (size_t)t * N + n;
        const float m = masks[i + N] ? 1.f : 0.f;
        ret = __fadd_rn(__fmul_rn(__fmul_rn(gamma, ret), m), rewards[i]);
        returns[i] = ret;
      }
      if (want_adv) {
        for (int t = 0; t < Talloc; ++t) {
          const size_t i = (size_t)t * N + n;
          const float a = __fsub_rn(returns[i], values[i]);
          adv[i] = a;
          acc_stats(a, s, ss, cnt);
        }
      }
    }
  }
  if (adv != nullptr && stats != nullptr) {
    s = block_sum(s, red);
    ss = block_sum(ss, red);
    cnt = block_sum(cnt, red);
    if (threadIdx.x == 0) {
      atomicAdd(&stats[0], s);
      atomicAdd(&stats[1], ss);
      atomicAdd(&stats[2], cnt);
    }
  }
}

// warp-per-env: each lane folds a contiguous chunk of time steps into one affine map
// g_lo = A + Bc * g_in, a shuffle suffix-scan composes the maps across lanes, then every
// lane replays its chunk with the true incoming value.  (use_gae only; latency ~ T/32 + 5.)
__global__ void gae_warp_kernel(const float* __restrict__ rewards, float* __restrict__ values,
                                const uint8_t* __restrict__ masks,
                                const float* __restrict__ next_value, float* __restrict__ returns,
                                float* __restrict__ adv, double* __restrict__ stats, int T,
                                int Talloc, int N, float gamma, float gt) {
  __shared__ double red[32];
  const int lane = threadIdx.x & 31;
  const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  double s = 0, ss = 0, cnt = 0;
  if (n < N) {
    const float nv = next_value[n];
    if (lane == 0) values[(size_t)T * N + n] = nv;
    const int L = (T + 31) / 32;
    const int lo = lane * L, hi = min(T, lo + L) - 1;  // chunk [lo, hi]
    // fold chunk
    float A = 0.f, Bc = 1.f;
    for (int t = hi; t >= lo; --t) {
      const size_t i = (size_t)t * N + n;
      const float m = masks[i + N] ? 1.f : 0.f;
      const float v_next = (t + 1 == T) ? nv : values[i + N];
      const float delta = __fsub_rn(__fadd_rn(rewards[i], __fmul_rn(__fmul_rn(gamma, v_next), m)), values[i]);
      const float c = __fmul_rn(gt, m);
      A = fmaf(c, A, delta);
      Bc = c * Bc;
    }
    // inclusive suffix scan over lanes: (A,B)_l <- (A,B)_l o (A,B)_{l+o}
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float A2 = __shfl_down_sync(0xffffffffu, A, o);
      const float B2 = __shfl_down_sync(0xffffffffu, Bc, o);
      if (lane + o < 32) {
        A = fmaf(Bc, A2, A);
        Bc = Bc * B2;
      }
    }
    float g_in = __shfl_down_sync(0xffffffffu, A, 1);
    if (lane == 31) g_in = 0.f;
    // replay
    float gae = g_in;
    for (int t = hi; t >= lo; --t) {
      const size_t i = (size_t)t * N + n;
      const float m = masks[i + N] ? 1.f : 0.f;
      const float v = values[i];
      const float v_next = (t + 1 == T) ? nv : values[i + N];
      const float delta = __fsub_rn(__fadd_rn(rewards[i], __fmul_rn(__fmul_rn(gamma, v_next), m)), v);
      gae = __fadd_rn(delta, __fmul_rn(__fmul_rn(gt, gae), m));
      const float ret = __fadd_rn(gae, v);
      returns[i] = ret;
      if (adv != nullptr) {
        const float a = __fsub_rn(ret, v);
        adv[i] = a;
        acc_stats(a, s, ss, cnt);
      }
    }
    if (adv != nullptr) {
      for (int t = T + lane; t < Talloc; t += 32) {  // bootstrap + stale rows
        const size_t i = (size_t)t * N + n;
        const float v = (t == T) ? nv : values[i];
        const float a = __fsub_rn(returns[i], v);
        adv[i] = a;
        acc_stats(a, s, ss, cnt);
      }
    }
  }
  if (adv != nullptr && stats != nullptr) {
    s = block_sum(s, red);
    ss = block_sum(ss, red);
    cnt = block_sum(cnt, red);
    if (threadIdx.x == 0) {
      atomicAdd(&stats[0], s);
      atomicAdd(&stats[1], ss);
      atomicAdd(&stats[2], cnt);
    }
  }
}

extern "C" int hb200_gae_adv(const float* rewards, float* value_preds, const uint8_t* masks,
                             const float* next_value, float* returns, float* advantages,
                             double* stats, int t_cur, int t_alloc, int n_envs, float gamma,
                             float tau, int use_gae, int variant, hb200_stream_t stream) {
  HB_CHECK_ARG(rewards && value_preds && masks && next_value && returns, "gae: null pointer");
  HB_CHECK_ARG(t_cur >= 0 && t_cur < t_alloc && n_envs > 0, "gae: bad sizes t_cur=%d t_alloc=%d n=%d",
               t_cur, t_alloc, n_envs);
  cudaStream_t st = (cudaStream_t)stream;
  if (stats) HB_CUDA(cudaMemsetAsync(stats, 0, 4 * sizeof(double), st));
  const float gt = (float)((double)gamma * (double)tau);
  if (variant == 0) variant = (use_gae && n_envs < 8192 && t_cur >= 32) ? 2 : 1;
  if (!use_gae) variant = 1;
  if (variant == 1) {
    const int bs = 128;
    gae_serial_kernel<<<cdiv(n_envs, bs), bs, 0, st>>>(rewards, value_preds, masks, next_value,
                                                        returns, advantages, stats, t_cur, t_alloc,
                                                        n_envs, gamma, gt, use_gae);
  } else {
    const int wpb = 4;
    gae_warp_kernel<<<cdiv(n_envs, wpb), wpb * 32, 0, st>>>(rewards, value_preds, masks, next_value,
                                                            returns, advantages, stats, t_cur,
                                                            t_alloc, n_envs, gamma, gt);
  }
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

__global__ void adv_normalize_kernel(float* __restrict__ adv, long long n,
                                     const double* __restrict__ stats,
                                     const float* __restrict__ mean_var, int mode) {
  float mean, var;
  if (mode == 0) {
    const double s = stats[0], ss = stats[1], c = stats[2];
    const double m = s / c;
    mean = (float)m;
    var = (float)((ss - s * m) / (c - 1.0));  // unbiased, torch.var_mean default
  } else {
    mean = mean_var[0];
    var = mean_var[1];
  }
  const float inv = 1.0f / sqrtf(var + 1e-5f);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x)
    adv[i] = __fmul_rn(__fsub_rn(adv[i], mean), inv);
}

extern "C" int hb200_adv_normalize(float* advantages, long long n, const double* stats,
                                   const float* mean_var, int mode, hb200_stream_t stream) {
  HB_CHECK_ARG(advantages && n > 0, "adv_normalize: bad args");
  HB_CHECK_ARG((mode == 0 && stats) || (mode == 1 && mean_var), "adv_normalize: mode/pointer mismatch");
  const int bs = 256;
  const int grid = (int)min((long long)kNumSMs * 8, (n + bs - 1) / bs);
  adv_normalize_kernel<<<grid, bs, 0, (cudaStream_t)stream>>>(advantages, n, stats, mean_var, mode);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

// =====================================================================================
// heads + PPO loss  (HB/utils/common.py:64-96, HB/rl/ppo/policy.py:377-381,416-424,
//                    HB/rl/ppo/ppo.py:195-250,260-275)
// =====================================================================================
constexpr int kMaxA = 8;
struct LossPartial {  // one per block
  float vl, al, ent, vsum, rsum, nclip, vmin, vmax, rmin, rmax, pad0, pad1;
};

template <int NJ>
__global__ void __launch_bounds__(256)
ppo_loss_main_kernel(const float* __restrict__ feat, const float* __restrict__ w_act,
                     const float* __restrict__ b_act, const float* __restrict__ w_val,
                     const float* __restrict__ b_val, const int64_t* __restrict__ actions,
                     const float* __restrict__ old_lp, const float* __restrict__ advs,
                     const float* __restrict__ old_v, const float* __restrict__ rets,
                     const float* __restrict__ is_coeffs, int B, int A, float clip, float c_v,
                     float c_e, int use_clip_v, int compute_grads, float* __restrict__ values_o,
                     float* __restrict__ lp_o, float* __restrict__ ent_o, float* __restrict__ d_feat,
                     float* __restrict__ dl /* [B, A+1] */, LossPartial* __restrict__ partials) {
  constexpr int H = NJ * 32;
  extern __shared__ float sw[];  // [(A+1)][H]
  __shared__ LossPartial wpart[8];
  for (int i = threadIdx.x; i < (A + 1) * H; i += blockDim.x)
    sw[i] = (i < A * H) ? w_act[i] : w_val[i - A * H];
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nwarps = gridDim.x * (blockDim.x >> 5);
  const float invB = 1.0f / (float)B;
  LossPartial p = {0, 0, 0, 0, 0, 0, INFINITY, -INFINITY, INFINITY, -INFINITY, 0, 0};

  for (int f = blockIdx.x * (blockDim.x >> 5) + warp; f < B; f += nwarps) {
    float x[NJ];
#pragma unroll
    for (int j = 0; j < NJ; ++j) x[j] = feat[(size_t)f * H + lane + 32 * j];
    float z[kMaxA + 1];
#pragma unroll
    for (int a = 0; a <= kMaxA; ++a) {
      if (a <= A) {
        float acc = 0.f;
#pragma unroll
        for (int j = 0; j < NJ; ++j) acc = fmaf(x[j], sw[a * H + lane + 32 * j], acc);
        z[a] = warp_sum(acc);
      } else {
        z[a] = 0.f;
      }
    }
    // all lanes hold identical z[]; do the scalar math redundantly (no divergence)
    float mx = -INFINITY;
#pragma unroll
    for (int a = 0; a < kMaxA; ++a)
      if (a < A) { z[a] += b_act[a]; mx = fmaxf(mx, z[a]); }
    float v = b_val[0];
#pragma unroll
    for (int a = 0; a <= kMaxA; ++a)
      if (a == A) v += z[a];
    float se = 0.f;
#pragma unroll
    for (int a = 0; a < kMaxA; ++a)
      if (a < A) se += expf(z[a] - mx);
    const float lse = mx + logf(se);
    const int act = (int)actions[f];
    // an action outside [0, A) has no log-probability (torch's gather device-asserts): poison the frame with NaN so
    // the loss and every metric show it instead of silently using log_prob = 0
    float logp[kMaxA], prob[kMaxA], ent = 0.f, lp = (act >= 0 && act < A) ? 0.f : __int_as_float(0x7fc00000);
#pragma unroll
    for (int a = 0; a < kMaxA; ++a) {
      if (a < A) {
        logp[a] = z[a] - lse;
        prob[a] = expf(logp[a]);
        ent -= prob[a] * logp[a];
        if (a == act) lp = logp[a];
      } else { logp[a] = 0.f; prob[a] = 0.f; }
    }
    const float adv = advs[f], ov = old_v[f], ret = rets[f];
    const float isw = is_coeffs ? fminf(is_coeffs[f], 1.0f) : 1.0f;
    const float ratio = expf(lp - old_lp[f]);
    const float s1 = adv * ratio;
    const float s2 = adv * fminf(fmaxf(ratio, 1.0f - clip), 1.0f + clip);
    // fminf / fmaxf return the non-NaN operand: re-poison explicitly for an out-of-range action
    const float a_loss = (act >= 0 && act < A) ? -fminf(s1, s2) : __int_as_float(0x7fc00000);
    float v_used = v;
    bool v_live = true;
    if (use_clip_v) {
      const float delta = v - ov;
      v_live = fabsf(delta) < clip;
      if (!v_live) v_used = ov + fminf(fmaxf(delta, -clip), clip);
    }
    const float dv = v_used - ret;
    const float v_loss = 0.5f * dv * dv;

    if (lane == 0) {
      if (values_o) values_o[f] = v;
      if (lp_o) lp_o[f] = lp;
      if (ent_o) ent_o[f] = ent;
      p.vl += isw * v_loss; p.al += isw * a_loss; p.ent += isw * ent;
      p.vsum += v; p.rsum += ratio;
      p.nclip += (ratio > 1.0f + clip ? 1.f : 0.f) + (ratio < 1.0f - clip ? 1.f : 0.f);
      p.vmin = fminf(p.vmin, v); p.vmax = fmaxf(p.vmax, v);
      p.rmin = fminf(p.rmin, ratio); p.rmax = fmaxf(p.rmax, ratio);
    }
    if (compute_grads) {
      // d total / d lp, d total / d v, d total / d H(entropy)   (each already / B)
      const float g_lp = (s1 <= s2) ? (-adv * ratio) * isw * invB : 0.f;
      const float g_v = v_live ? c_v * dv * isw * invB : 0.f;
      const float g_h = -c_e * isw * invB;
      float dz[kMaxA + 1];
      dz[kMaxA] = 0.f;
#pragma unroll
      for (int a = 0; a < kMaxA; ++a)
        dz[a] = (a < A) ? (g_lp * ((a == act ? 1.f : 0.f) - prob[a]) - g_h * prob[a] * (logp[a] + ent)) : 0.f;
      float mine = 0.f;  // static register indexing only: select chains instead of dz[A], dz[lane]
#pragma unroll
      for (int a = 0; a <= kMaxA; ++a) {
        if (a == A) dz[a] = g_v;
        if (a == kMaxA && A < kMaxA) dz[a] = 0.f;
        if (lane == a) mine = dz[a];
      }
      if (lane <= A) dl[(size_t)f * (A + 1) + lane] = mine;
      // d_features = sum_a dz[a] * W[a,:]
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        float acc = 0.f;
#pragma unroll
        for (int a = 0; a <= kMaxA; ++a)
          if (a <= A) acc = fmaf(dz[a], sw[a * H + lane + 32 * j], acc);
        d_feat[(size_t)f * H + lane + 32 * j] = acc;
      }
    }
  }
  if (lane == 0) wpart[warp] = p;
  __syncthreads();
  if (threadIdx.x == 0) {
    LossPartial r = wpart[0];
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) {
      const LossPartial q = wpart[w];
      r.vl += q.vl; r.al += q.al; r.ent += q.ent; r.vsum += q.vsum; r.rsum += q.rsum; r.nclip += q.nclip;
      r.vmin = fminf(r.vmin, q.vmin); r.vmax = fmaxf(r.vmax, q.vmax);
      r.rmin = fminf(r.rmin, q.rmin); r.rmax = fmaxf(r.rmax, q.rmax);
    }
    partials[blockIdx.x] = r;
  }
}

// dW[a, col] = sum_b dl[b,a] * feat[b,col];  db[a] = sum_b dl[b,a]
// One partial row per frame slab (blockIdx.y): parts[y][a * H + col] and parts[y][A1 * H + a], summed in order by
// reduce_partials (no floating-point atomics: the result is the same every run).
__global__ void __launch_bounds__(256)
ppo_heads_wgrad_kernel(const float* __restrict__ feat, const float* __restrict__ dl, int B, int H,
                       int A1, float* __restrict__ parts) {
  float* prow = parts + (size_t)blockIdx.y * A1 * (H + 1);
  __shared__ float red[8][kMaxA + 1][33];
  const int col = blockIdx.x * 32 + (threadIdx.x & 31);
  const int slice = threadIdx.x >> 5;  // 8 slices of the frame range of this block
  const int per = (B + gridDim.y - 1) / gridDim.y;
  const int b0 = blockIdx.y * per, b1 = min(B, b0 + per);
  float acc[kMaxA + 1];
#pragma unroll
  for (int a = 0; a <= kMaxA; ++a) acc[a] = 0.f;
  float bacc = 0.f;  // bias grads: lane a of slice handles row a (col-block 0 only)
  for (int b = b0 + slice; b < b1; b += 8) {
    const float x = (col < H) ? feat[(size_t)b * H + col] : 0.f;
#pragma unroll
    for (int a = 0; a <= kMaxA; ++a)
      if (a < A1) acc[a] = fmaf(dl[(size_t)b * A1 + a], x, acc[a]);
    if (blockIdx.x == 0 && (threadIdx.x & 31) < A1) bacc += dl[(size_t)b * A1 + (threadIdx.x & 31)];
  }
  __shared__ float bred[8][32];   // bias partials of the 8 frame slices (block column 0)
#pragma unroll
  for (int a = 0; a <= kMaxA; ++a) red[slice][a][threadIdx.x & 31] = acc[a];
  bred[slice][threadIdx.x & 31] = bacc;
  __syncthreads();
  if (slice == 0 && col < H) {
#pragma unroll
    for (int a = 0; a <= kMaxA; ++a) {
      if (a < A1) {
        float s = 0.f;
        for (int w = 0; w < 8; ++w) s += red[w][a][threadIdx.x & 31];
        prow[(size_t)a * H + col] = s;
      }
    }
  }
  if (blockIdx.x == 0 && slice == 0 && (threadIdx.x & 31) < A1) {
    const int a = threadIdx.x & 31;
    float sb = 0.f;
    for (int w = 0; w < 8; ++w) sb += bred[w][a];
    prow[(size_t)A1 * H + a] = sb;
  }
}

__global__ void ppo_loss_finalize_kernel(const LossPartial* __restrict__ partials, int nblocks, int B,
                                         float c_v, float c_e, float* __restrict__ metrics) {
  if (threadIdx.x != 0) return;
  LossPartial r = partials[0];
  for (int i = 1; i < nblocks; ++i) {
    const LossPartial q = partials[i];
    r.vl += q.vl; r.al += q.al; r.ent += q.ent; r.vsum += q.vsum; r.rsum += q.rsum; r.nclip += q.nclip;
    r.vmin = fminf(r.vmin, q.vmin); r.vmax = fmaxf(r.vmax, q.vmax);
    r.rmin = fminf(r.rmin, q.rmin); r.rmax = fmaxf(r.rmax, q.rmax);
  }
  const float invB = 1.0f / (float)B;
  metrics[HB200_M_VALUE_LOSS] = r.vl * invB;
  metrics[HB200_M_ACTION_LOSS] = r.al * invB;
  metrics[HB200_M_DIST_ENTROPY] = r.ent * invB;
  metrics[HB200_M_VALUE_MIN] = r.vmin;
  metrics[HB200_M_VALUE_MEAN] = r.vsum * invB;
  metrics[HB200_M_VALUE_MAX] = r.vmax;
  metrics[HB200_M_RATIO_MIN] = r.rmin;
  metrics[HB200_M_RATIO_MEAN] = r.rsum * invB;
  metrics[HB200_M_RATIO_MAX] = r.rmax;
  metrics[HB200_M_FRAC_CLIPPED] = r.nclip * invB;
  metrics[HB200_M_TOTAL_LOSS] = c_v * r.vl * invB + r.al * invB - c_e * r.ent * invB;
  metrics[HB200_M_SPARE] = 0.f;
}

static int loss_grid(int B) { return min(cdiv(B, 8), kNumSMs * 2); }

extern "C" size_t hb200_ppo_loss_workspace_bytes(int batch, int hidden, int n_actions) {
  (void)hidden;
  return sizeof(LossPartial) * (size_t)(kNumSMs * 2) + sizeof(float) * (size_t)batch * (n_actions + 1) + 256;
}

extern "C" int hb200_ppo_loss(const float* features, const float* w_act, const float* b_act,
                              const float* w_val, const float* b_val, const int64_t* actions,
                              const float* old_log_probs, const float* advantages,
                              const float* old_values, const float* returns, const float* is_coeffs,
                              int batch, int hidden, int n_actions, float clip_param,
                              float value_loss_coef, float entropy_coef, int use_clipped_value_loss,
                              int compute_grads, float* values, float* log_probs, float* entropy,
                              float* d_features, float* d_w_act, float* d_b_act, float* d_w_val,
                              float* d_b_val, float* metrics, void* workspace,
                              hb200_stream_t stream) {
  HB_CHECK_ARG(features && w_act && b_act && w_val && b_val && actions && old_log_probs &&
                   advantages && old_values && returns && metrics && workspace,
               "ppo_loss: null pointer");
  HB_CHECK_ARG(batch > 0 && n_actions >= 1 && n_actions <= kMaxA, "ppo_loss: n_actions=%d unsupported (1..%d)",
               n_actions, kMaxA);
  HB_CHECK_ARG(hidden == 128 || hidden == 256 || hidden == 512 || hidden == 32 || hidden == 64,
               "ppo_loss: hidden=%d unsupported (32,64,128,256,512)", hidden);
  HB_CHECK_ARG(!compute_grads || (d_features && d_w_act && d_b_act && d_w_val && d_b_val),
               "ppo_loss: compute_grads needs gradient outputs");
  cudaStream_t st = (cudaStream_t)stream;
  LossPartial* partials = (LossPartial*)workspace;
  float* dl = (float*)((char*)workspace + ((sizeof(LossPartial) * (size_t)(kNumSMs * 2) + 255) / 256) * 256);
  const int grid = loss_grid(batch);
  const size_t smem = sizeof(float) * (size_t)(n_actions + 1) * hidden;
#define HB_LOSS_LAUNCH(NJ)                                                                       \
  ppo_loss_main_kernel<NJ><<<grid, 256, smem, st>>>(                                             \
      features, w_act, b_act, w_val, b_val, actions, old_log_probs, advantages, old_values,      \
      returns, is_coeffs, batch, n_actions, clip_param, value_loss_coef, entropy_coef,           \
      use_clipped_value_loss, compute_grads, values, log_probs, entropy, d_features, dl, partials)
  switch (hidden) {
    case 32: HB_LOSS_LAUNCH(1); break;
    case 64: HB_LOSS_LAUNCH(2); break;
    case 128: HB_LOSS_LAUNCH(4); break;
    case 256: HB_LOSS_LAUNCH(8); break;
    default: HB_LOSS_LAUNCH(16); break;
  }
#undef HB_LOSS_LAUNCH
  HB_LAUNCH_OK();
  ppo_loss_finalize_kernel<<<1, 32, 0, st>>>(partials, grid, batch, value_loss_coef, entropy_coef, metrics);
  HB_LAUNCH_OK();
  count_launch(2);
  if (compute_grads) {
    HB_CUDA(cudaMemsetAsync(d_w_act, 0, sizeof(float) * (size_t)n_actions * hidden, st));
    HB_CUDA(cudaMemsetAsync(d_b_act, 0, sizeof(float) * n_actions, st));
    HB_CUDA(cudaMemsetAsync(d_w_val, 0, sizeof(float) * hidden, st));
    HB_CUDA(cudaMemsetAsync(d_b_val, 0, sizeof(float), st));
    dim3 g(cdiv(hidden, 32), min(32, cdiv(batch, 64)));
    const int A1 = n_actions + 1;
    const long long row = (long long)A1 * (hidden + 1);   // one partial row per frame slab
    float* parts = nullptr;
    int* tickets = nullptr;
    int rc = stream_workspace(st, (size_t)(g.y + kReduceChunks) * row, 0, &parts, &tickets);
    if (rc) return rc;
    float* tmp = parts + (size_t)g.y * row;
    ppo_heads_wgrad_kernel<<<g, 256, 0, st>>>(features, dl, batch, hidden, A1, parts);
    HB_LAUNCH_OK();
    count_launch(1);
    const long long H = hidden;
    rc = reduce_partials(parts, g.y, row, (long long)n_actions * H, d_w_act, tmp, st);
    if (!rc) rc = reduce_partials(parts + (size_t)n_actions * H, g.y, row, H, d_w_val, tmp, st);
    if (!rc) rc = reduce_partials(parts + (size_t)A1 * H, g.y, row, n_actions, d_b_act, tmp, st);
    if (!rc) rc = reduce_partials(parts + (size_t)A1 * H + n_actions, g.y, row, 1, d_b_val, tmp, st);
    if (rc) return rc;
  }
  return HB200_OK;
}

// =====================================================================================
// clip_grad_norm_ + Adam  (HB/rl/ppo/ppo.py:112-137,257,347-371; torch.optim.Adam math)
// =====================================================================================
__global__ void sqnorm_partial_kernel(const float* __restrict__ g, long long n, float scale,
                                      double* __restrict__ partial) {
  __shared__ double red[32];
  double acc = 0;
  const long long n4 = n >> 2;
  const float4* g4 = reinterpret_cast<const float4*>(g);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    float4 v = g4[i];
    v.x *= scale; v.y *= scale; v.z *= scale; v.w *= scale;
    acc += (double)v.x * v.x + (double)v.y * v.y + (double)v.z * v.z + (double)v.w * v.w;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const float v = g[(n4 << 2) + threadIdx.x] * scale;
    acc += (double)v * v;
  }
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) partial[blockIdx.x] = acc;
}
__global__ void sqnorm_final_kernel(const double* __restrict__ partial, int nb, float* __restrict__ out) {
  __shared__ double red[32];
  double acc = 0;
  for (int i = threadIdx.x; i < nb; i += blockDim.x) acc += partial[i];
  acc = block_sum(acc, red);
  if (threadIdx.x == 0) out[0] = (float)acc;
}

__global__ void clip_adam_kernel(float* __restrict__ p, const float* __restrict__ g,
                                 float* __restrict__ m, float* __restrict__ v, long long n, float lr,
                                 float b1, float b2, float eps, float wd, float max_norm,
                                 float gscale, float bc1, float bc2_sqrt,
                                 const float* __restrict__ hyper, const float* __restrict__ sqnorm,
                                 float* __restrict__ grad_norm_out) {
  if (hyper) lr = hyper[0];
  const float total_norm = sqrtf(sqnorm[0]);
  if (blockIdx.x == 0 && threadIdx.x == 0 && grad_norm_out) grad_norm_out[0] = total_norm;
  float coef = gscale;
  if (max_norm > 0.f) coef *= fminf(max_norm / (total_norm + 1e-6f), 1.0f);
  const float step_size = lr / bc1;
  const long long n4 = n >> 2;
  float4* p4 = reinterpret_cast<float4*>(p);
  const float4* g4 = reinterpret_cast<const float4*>(g);
  float4* m4 = reinterpret_cast<float4*>(m);
  float4* v4 = reinterpret_cast<float4*>(v);
  auto upd = [&](float& pp, float gg, float& mm, float& vv) {
    gg *= coef;
    if (wd != 0.f) gg = fmaf(wd, pp, gg);
    mm = mm + (1.0f - b1) * (gg - mm);                 // exp_avg.lerp_(grad, 1-beta1)
    vv = fmaf(1.0f - b2, gg * gg, vv * b2);            // exp_avg_sq.mul_(b2).addcmul_(g,g,1-b2)
    const float denom = sqrtf(vv) / bc2_sqrt + eps;
    pp = pp - step_size * (mm / denom);                // param.addcdiv_(exp_avg, denom, -step_size)
  };
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4;
       i += (long long)gridDim.x * blockDim.x) {
    float4 pp = p4[i], gg = g4[i], mm = m4[i], vv = v4[i];
    upd(pp.x, gg.x, mm.x, vv.x); upd(pp.y, gg.y, mm.y, vv.y);
    upd(pp.z, gg.z, mm.z, vv.z); upd(pp.w, gg.w, mm.w, vv.w);
    p4[i] = pp; m4[i] = mm; v4[i] = vv;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {
    const long long i = (n4 << 2) + threadIdx.x;
    upd(p[i], g[i], m[i], v[i]);
  }
}

static const int kAdamGrid = kNumSMs * 8;
extern "C" size_t hb200_clip_adam_workspace_bytes(long long n) {
  (void)n;
  return sizeof(double) * kAdamGrid + 256;
}
extern "C" int hb200_grad_sqnorm(const float* grads, long long n, float grad_scale, float* sqnorm_out,
                                 void* workspace, hb200_stream_t stream) {
  HB_CHECK_ARG(grads && sqnorm_out && workspace && n > 0, "grad_sqnorm: bad args");
  HB_CHECK_ARG(((uintptr_t)grads & 15) == 0, "grad_sqnorm: grads must be 16B aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = (int)min((long long)kAdamGrid, (n / 4 + 255) / 256 + 1);
  sqnorm_partial_kernel<<<grid, 256, 0, st>>>(grads, n, grad_scale, (double*)workspace);
  HB_LAUNCH_OK();
  sqnorm_final_kernel<<<1, 256, 0, st>>>((const double*)workspace, grid, sqnorm_out);
  HB_LAUNCH_OK();
  count_launch(2);
  return HB200_OK;
}
extern "C" int hb200_clip_adam(float* params, const float* grads, float* exp_avg, float* exp_avg_sq,
                               long long n, float lr, float beta1, float beta2, float eps,
                               float weight_decay, float max_grad_norm, float grad_scale,
                               long long step, const float* hyper, float* grad_norm_out,
                               void* workspace, hb200_stream_t stream) {
  HB_CHECK_ARG(params && grads && exp_avg && exp_avg_sq && workspace && n > 0 && step >= 1,
               "clip_adam: bad args");
  HB_CHECK_ARG((((uintptr_t)params | (uintptr_t)grads | (uintptr_t)exp_avg | (uintptr_t)exp_avg_sq) & 15) == 0,
               "clip_adam: buffers must be 16B aligned");
  cudaStream_t st = (cudaStream_t)stream;
  float* sq = (float*)((char*)workspace + sizeof(double) * kAdamGrid);
  int rc = hb200_grad_sqnorm(grads, n, grad_scale, sq, workspace, stream);
  if (rc) return rc;
  const double bc1 = 1.0 - pow((double)beta1, (double)step);
  const double bc2 = 1.0 - pow((double)beta2, (double)step);
  const int grid = (int)min((long long)kAdamGrid, (n / 4 + 255) / 256 + 1);
  clip_adam_kernel<<<grid, 256, 0, st>>>(params, grads, exp_avg, exp_avg_sq, n, lr, beta1, beta2, eps,
                                         weight_decay, max_grad_norm, grad_scale, (float)bc1,
                                         (float)sqrt(bc2), hyper, sq, grad_norm_out);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}
