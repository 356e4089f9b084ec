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

// =====================================================================================
// VER: GAE over packed sequences (HB/rl/ver/ver_rollout_storage.py:430-568) + advantages
// =====================================================================================
// Step t of sequence s is frame select_inds[step_offset[t] + s]; sequences are sorted by length, longest first.
// One thread walks one sequence backwards, in fp64 with unfused operations in the reference's (numpy) order, so every
// return is the reference's float64 value rounded once to fp32: the results are bit-identical to it.  After a block
// barrier the same block writes advantages = returns - value_preds for every frame and sums the finite ones in a fixed
// order (one block: the statistics do not depend on scheduling).
constexpr int kVerGaeThreads = 1024;
__global__ void __launch_bounds__(kVerGaeThreads)
ver_gae_kernel(const float* __restrict__ rewards, const float* __restrict__ values, float* __restrict__ returns,
               const uint8_t* __restrict__ is_stale, const int32_t* __restrict__ select_inds,
               const int32_t* __restrict__ step_offset, const int32_t* __restrict__ seq_len,
               const int32_t* __restrict__ last_for_env, int n_frames, int n_seqs, double gamma, double gt,
               float* __restrict__ adv, double* __restrict__ stats) {
  __shared__ double red[32];
  for (int s = threadIdx.x; s < n_seqs; s += blockDim.x) {
    const bool env_last = last_for_env[s] != 0;
    double gae = 0.0, last_v = 0.0;
    for (int t = seq_len[s] - 1; t >= 0; --t) {
      const int i = select_inds[step_offset[t] + s];
      const double v = (double)values[i];
      const double delta = __dsub_rn(__dadd_rn((double)rewards[i], __dmul_rn(gamma, last_v)), v);
      gae = __dadd_rn(delta, __dmul_rn(gt, gae));
      const bool bootstrap = env_last && t == seq_len[s] - 1;
      if (bootstrap) gae = 0.0;   // the bootstrap step only provides last_v for the step before it
      const float old = returns[i];
      if (bootstrap) {
        returns[i] = __int_as_float(0x7fc00000);
      } else if (!is_stale[i] || !isfinite(old)) {
        returns[i] = (float)__dadd_rn(gae, v);
      }
      last_v = v;
    }
  }
  __syncthreads();
  double s = 0, ss = 0, cnt = 0, fin = 0;
  for (int i = threadIdx.x; i < n_frames; i += blockDim.x) {
    const float r = returns[i];
    const float a = __fsub_rn(r, values[i]);
    if (adv) adv[i] = a;
    acc_stats(a, s, ss, cnt);
    fin += isfinite(r) ? 1.0 : 0.0;
  }
  s = block_sum(s, red);
  ss = block_sum(ss, red);
  cnt = block_sum(cnt, red);
  fin = block_sum(fin, red);
  if (threadIdx.x == 0 && stats) {
    stats[0] = s;
    stats[1] = ss;
    stats[2] = cnt;
    stats[3] = fin;
  }
}

extern "C" int hb200_ver_gae(const float* rewards, const float* value_preds, float* returns, const uint8_t* is_stale,
                             const int32_t* seq_table, int n_frames, int n_seqs, int max_len, double gamma, double tau,
                             int use_gae, float* advantages, double* stats, int expected_finite,
                             hb200_stream_t stream) {
  HB_CHECK_ARG(rewards && value_preds && returns && is_stale && seq_table && stats, "ver_gae: null pointer");
  HB_CHECK_ARG(n_frames > 0 && n_seqs > 0 && n_seqs <= n_frames && max_len > 0 && max_len <= n_frames,
               "ver_gae: bad sizes n_frames=%d n_seqs=%d max_len=%d", n_frames, n_seqs, max_len);
  cudaStream_t st = (cudaStream_t)stream;
  const int32_t* select_inds = seq_table;
  const int32_t* step_offset = seq_table + n_frames;
  const int32_t* seq_len = step_offset + max_len;
  const int32_t* last_for_env = seq_len + n_seqs;
  // the reference evaluates `gamma * last_values` and `(tau * gamma) * gae` with python floats: double throughout
  const double g = gamma, gt = (use_gae ? tau : 1.0) * g;
  ver_gae_kernel<<<1, kVerGaeThreads, 0, st>>>(rewards, value_preds, returns, is_stale, select_inds, step_offset,
                                              seq_len, last_for_env, n_frames, n_seqs, g, gt, advantages, stats);
  HB_LAUNCH_OK();
  count_launch(1);
  if (expected_finite >= 0) {   // the reference's invariant: exactly T * N finite returns (one NaN bootstrap per env)
    double fin = 0;
    HB_CUDA(cudaMemcpyAsync(&fin, stats + 3, sizeof(double), cudaMemcpyDeviceToHost, st));
    HB_CUDA(cudaStreamSynchronize(st));
    if ((long long)fin != (long long)expected_finite) {
      set_last_error("ver_gae: %lld finite returns, expected %d (one bootstrap step per environment)",
                     (long long)fin, expected_finite);
      return HB200_ERR_INVALID_ARG;
    }
  }
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
__device__ __forceinline__ float clamp_nan(float x, float lo, float hi) { return min_nan(max_nan(x, lo), hi); }
struct LossPartial {  // one per block
  float vl, al, ent, vsum, rsum, nclip, vmin, vmax, rmin, rmax, pad0, pad1;
};

// (256, 2): loss_grid launches at most two blocks per SM, so each thread may use up to 128 registers (at the
// default heuristic ptxas capped some instantiations at 64 and spilled)
template <int NJ>
__global__ void __launch_bounds__(256, 2)
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
    // an action outside [0, A) has no log-probability (torch's gather device-asserts): lp = NaN poisons the frame's
    // loss, ratio metrics and gradients instead of silently using log_prob = 0
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
    const float isw = is_coeffs ? min_nan(is_coeffs[f], 1.0f) : 1.0f;
    const float ratio = expf(lp - old_lp[f]);
    const float s1 = adv * ratio;
    const float s2 = adv * clamp_nan(ratio, 1.0f - clip, 1.0f + clip);
    const float a_loss = -min_nan(s1, s2);
    float v_used = v;
    bool v_live = true;
    if (use_clip_v) {
      const float delta = v - ov;
      v_live = fabsf(delta) < clip;
      if (!v_live) v_used = ov + clamp_nan(delta, -clip, clip);
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
      p.vmin = min_nan(p.vmin, v); p.vmax = max_nan(p.vmax, v);
      p.rmin = min_nan(p.rmin, ratio); p.rmax = max_nan(p.rmax, ratio);
    }
    if (compute_grads) {
      // d total / d lp, d total / d v, d total / d H(entropy)   (each already / B).  torch.min's backward sends the
      // gradient to both operands when one is NaN, so a NaN s1 or s2 takes the unclipped (NaN) branch.
      const float g_lp = !(s1 > s2) ? (-adv * ratio) * isw * invB : 0.f;
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
      r.vmin = min_nan(r.vmin, q.vmin); r.vmax = max_nan(r.vmax, q.vmax);
      r.rmin = min_nan(r.rmin, q.rmin); r.rmax = max_nan(r.rmax, q.rmax);
    }
    partials[blockIdx.x] = r;
  }
}

// dW[a, col] = sum_b dl[b,a] * feat[b,col];  db[a] = sum_b dl[b,a]
// One partial row per frame slab (blockIdx.y): parts[y][a * H + col] and parts[y][A1 * H + a], summed in order by
// reduce_partials (no floating-point atomics: the result is the same every run).  (256, 4): up to 64 registers, where
// ptxas's default choice of 32 spilled the accumulators.
__global__ void __launch_bounds__(256, 4)
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
    r.vmin = min_nan(r.vmin, q.vmin); r.vmax = max_nan(r.vmax, q.vmax);
    r.rmin = min_nan(r.rmin, q.rmin); r.rmax = max_nan(r.rmax, q.rmax);
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
// Gaussian action head: act tail + PPO loss  (HB/utils/common.py:99-175 GaussianNet / CustomNormal,
//                                             HB/rl/ppo/policy.py:330-342, HB/rl/ppo/ppo.py:195-250)
// =====================================================================================
// One warp per frame.  mu_maybe_std = features @ W^T + b (A rows, plus A std rows without use_std_param) and the critic
// are length-H dot products reduced across the warp; lane a < A then owns action dimension a: its mean, standard
// deviation, log-probability and entropy term (and, in the loss, their gradients), and the per-frame sums over the
// action dimensions are warp sums.  Weights are read through the read-only cache: at most (2A + 1) x H floats.
constexpr int kMaxGaussA = 16;
constexpr float kHalfLog2Pi = 0.91893853320467274f;     // log(sqrt(2 pi))
constexpr float kEntConst = 1.4189385332046727f;        // 0.5 + log(sqrt(2 pi))

struct GaussFrame {
  float mu_pre, s0, s2, mu, std, v;   // lane a < A: pre-activation mean, raw std, std before softplus, mean, std; all: value
};

template <int NJ>
__device__ __forceinline__ GaussFrame gauss_frame(const float* __restrict__ xrow, const float* __restrict__ w_mu,
                                                  const float* __restrict__ b_mu, const float* __restrict__ std_p,
                                                  const float* __restrict__ w_val, const float* __restrict__ b_val,
                                                  int A, int flags, float lo, float hi, int lane) {
  constexpr int H = NJ * 32;
  float x[NJ];
#pragma unroll
  for (int j = 0; j < NJ; ++j) x[j] = xrow[lane + 32 * j];
  const bool std_param = flags & HB200_GAUSS_STD_PARAM;
  const int L = std_param ? A : 2 * A;
  GaussFrame g;
  g.mu_pre = 0.f;
  g.s0 = (std_param && lane < A) ? __ldg(std_p + lane) : 0.f;
  for (int o = 0; o < L; ++o) {
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < NJ; ++j) acc = fmaf(x[j], __ldg(w_mu + (size_t)o * H + lane + 32 * j), acc);
    const float z = warp_sum(acc) + __ldg(b_mu + o);
    if (o < A) {
      if (lane == o) g.mu_pre = z;
    } else if (lane == o - A) {
      g.s0 = z;
    }
  }
  float acc = 0.f;
#pragma unroll
  for (int j = 0; j < NJ; ++j) acc = fmaf(x[j], __ldg(w_val + lane + 32 * j), acc);
  g.v = warp_sum(acc) + __ldg(b_val);
  // GaussianNet.forward's order: tanh(mu); clamp(std); exp (log-std); softplus (threshold 20, as F.softplus)
  g.mu = (flags & HB200_GAUSS_TANH) ? tanhf(g.mu_pre) : g.mu_pre;
  float s = (flags & HB200_GAUSS_CLAMP_STD) ? clamp_nan(g.s0, lo, hi) : g.s0;
  if (flags & HB200_GAUSS_LOG_STD) s = expf(s);
  g.s2 = s;
  if (flags & HB200_GAUSS_SOFTPLUS) s = s > 20.f ? s : log1pf(expf(s));
  g.std = s;
  return g;
}

// Normal(mu, std).log_prob(x) as torch.distributions.Normal writes it
__device__ __forceinline__ float gauss_logp(float x, float mu, float std) {
  const float d = x - mu;
  return -(d * d) / (2.f * (std * std)) - logf(std) - kHalfLog2Pi;
}

template <int NJ>
__global__ void __launch_bounds__(256)
gaussian_act_kernel(const float* __restrict__ feat, const float* __restrict__ w_mu, const float* __restrict__ b_mu,
                    const float* __restrict__ std_p, const float* __restrict__ w_val, const float* __restrict__ b_val,
                    const float* __restrict__ eps, int B, int A, int flags, float lo, float hi,
                    float* __restrict__ actions, float* __restrict__ alp, float* __restrict__ values) {
  constexpr int H = NJ * 32;
  const int lane = threadIdx.x & 31;
  const int f = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (f >= B) return;
  const GaussFrame g = gauss_frame<NJ>(feat + (size_t)f * H, w_mu, b_mu, std_p, w_val, b_val, A, flags, lo, hi, lane);
  float lp = 0.f;
  if (lane < A) {
    // rsample: loc + eps * scale (two roundings, as torch evaluates it); deterministic: the mean
    const float a = eps ? __fadd_rn(g.mu, __fmul_rn(eps[(size_t)f * A + lane], g.std)) : g.mu;
    actions[(size_t)f * A + lane] = a;
    lp = gauss_logp(a, g.mu, g.std);
  }
  lp = warp_sum(lp);
  if (lane == 0) {
    alp[f] = lp;
    values[f] = g.v;
  }
}

extern "C" int hb200_gaussian_act(const float* features, const float* w_mu, const float* b_mu, const float* std_param,
                                  const float* w_val, const float* b_val, const float* eps, int batch, int hidden,
                                  int n_actions, int flags, float min_std, float max_std, float* actions,
                                  float* action_log_probs, float* values, hb200_stream_t stream) {
  HB_CHECK_ARG(features && w_mu && b_mu && w_val && b_val && actions && action_log_probs && values,
               "gaussian_act: null pointer");
  HB_CHECK_ARG(batch > 0 && n_actions >= 1 && n_actions <= kMaxGaussA, "gaussian_act: n_actions=%d unsupported (1..%d)",
               n_actions, kMaxGaussA);
  HB_CHECK_ARG(hidden == 32 || hidden == 64 || hidden == 128 || hidden == 256 || hidden == 512,
               "gaussian_act: hidden=%d unsupported (32,64,128,256,512)", hidden);
  HB_CHECK_ARG((flags & ~HB200_GAUSS_ALL_FLAGS) == 0, "gaussian_act: unknown flags 0x%x", flags);
  HB_CHECK_ARG(!(flags & HB200_GAUSS_STD_PARAM) == !std_param, "gaussian_act: std_param must be given iff use_std_param");
  cudaStream_t st = (cudaStream_t)stream;
  const int grid = cdiv(batch, 8);
#define HB_GACT_LAUNCH(NJ)                                                                                            \
  gaussian_act_kernel<NJ><<<grid, 256, 0, st>>>(features, w_mu, b_mu, std_param, w_val, b_val, eps, batch, n_actions, \
                                                flags, min_std, max_std, actions, action_log_probs, values)
  switch (hidden) {
    case 32: HB_GACT_LAUNCH(1); break;
    case 64: HB_GACT_LAUNCH(2); break;
    case 128: HB_GACT_LAUNCH(4); break;
    case 256: HB_GACT_LAUNCH(8); break;
    default: HB_GACT_LAUNCH(16); break;
  }
#undef HB_GACT_LAUNCH
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

// dl row of a frame (C = 2A + 1 columns): [0, L) d mu_maybe_std outputs (L = A with use_std_param, else 2A), L: d value,
// and with use_std_param [A + 1, 2A + 1): this frame's gradient of the std parameter.
template <int NJ>
__global__ void __launch_bounds__(256, 2)
gaussian_loss_main_kernel(const float* __restrict__ feat, const float* __restrict__ w_mu, const float* __restrict__ b_mu,
                          const float* __restrict__ std_p, const float* __restrict__ w_val,
                          const float* __restrict__ b_val, const float* __restrict__ actions,
                          const float* __restrict__ old_lp, const float* __restrict__ advs,
                          const float* __restrict__ old_v, const float* __restrict__ rets,
                          const float* __restrict__ is_coeffs, int B, int A, int flags, float lo, float hi, float clip,
                          float c_v, float c_e, int use_clip_v, int compute_grads, float* __restrict__ values_o,
                          float* __restrict__ lp_o, float* __restrict__ ent_o, float* __restrict__ d_feat,
                          float* __restrict__ dl, LossPartial* __restrict__ partials) {
  constexpr int H = NJ * 32;
  __shared__ LossPartial wpart[8];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int nwarps = gridDim.x * (blockDim.x >> 5);
  const float invB = 1.0f / (float)B;
  const bool std_param = flags & HB200_GAUSS_STD_PARAM;
  const int L = std_param ? A : 2 * A, C = 2 * A + 1;
  LossPartial p = {0, 0, 0, 0, 0, 0, INFINITY, -INFINITY, INFINITY, -INFINITY, 0, 0};

  for (int f = blockIdx.x * (blockDim.x >> 5) + warp; f < B; f += nwarps) {
    const GaussFrame g = gauss_frame<NJ>(feat + (size_t)f * H, w_mu, b_mu, std_p, w_val, b_val, A, flags, lo, hi, lane);
    const float xa = lane < A ? actions[(size_t)f * A + lane] : 0.f;
    const float lp = warp_sum(lane < A ? gauss_logp(xa, g.mu, g.std) : 0.f);
    const float ent = warp_sum(lane < A ? kEntConst + logf(g.std) : 0.f);
    const float v = g.v;
    const float adv = advs[f], ov = old_v[f], ret = rets[f];
    const float isw = is_coeffs ? min_nan(is_coeffs[f], 1.0f) : 1.0f;
    const float ratio = expf(lp - old_lp[f]);
    const float s1 = adv * ratio;
    const float s2 = adv * clamp_nan(ratio, 1.0f - clip, 1.0f + clip);
    const float a_loss = -min_nan(s1, s2);
    float v_used = v;
    bool v_live = true;
    if (use_clip_v) {
      const float delta = v - ov;
      v_live = fabsf(delta) < clip;
      if (!v_live) v_used = ov + clamp_nan(delta, -clip, clip);
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
      p.vmin = min_nan(p.vmin, v); p.vmax = max_nan(p.vmax, v);
      p.rmin = min_nan(p.rmin, ratio); p.rmax = max_nan(p.rmax, ratio);
    }
    if (compute_grads) {
      // as in ppo_loss_main_kernel: d total / d lp, d value, d entropy (each already / B)
      const float g_lp = !(s1 > s2) ? (-adv * ratio) * isw * invB : 0.f;
      const float g_v = v_live ? c_v * dv * isw * invB : 0.f;
      const float g_h = -c_e * isw * invB;
      float dmu_pre = 0.f, ds0 = 0.f;
      if (lane < A) {
        const float d = xa - g.mu, sd = g.std, var = sd * sd;
        const float dmu = g_lp * (d / var);
        // d log_prob / d std = d^2 / std^3 - 1 / std;  d entropy / d std = 1 / std
        float ds = g_lp * ((d * d) / (var * sd) - 1.f / sd) + g_h / sd;
        dmu_pre = (flags & HB200_GAUSS_TANH) ? dmu * (1.f - g.mu * g.mu) : dmu;
        if (flags & HB200_GAUSS_SOFTPLUS) {
          if (!(g.s2 > 20.f)) {
            const float z = expf(g.s2);
            ds = ds * z / (z + 1.f);
          }
        }
        if (flags & HB200_GAUSS_LOG_STD) ds = ds * g.s2;
        // clamp's backward passes the gradient where lo <= x <= hi (bounds included) and gives 0 elsewhere (NaN too)
        if ((flags & HB200_GAUSS_CLAMP_STD) && !(g.s0 >= lo && g.s0 <= hi)) ds = 0.f;
        ds0 = ds;
        float* row = dl + (size_t)f * C;
        row[lane] = dmu_pre;
        row[std_param ? A + 1 + lane : A + lane] = ds0;
      }
      if (lane == 0) dl[(size_t)f * C + L] = g_v;
      // d_features = sum_o dl_o W_o + g_v w_val, in row order
      float acc[NJ];
#pragma unroll
      for (int j = 0; j < NJ; ++j) acc[j] = 0.f;
      for (int o = 0; o < L; ++o) {
        const float dz = o < A ? __shfl_sync(0xffffffffu, dmu_pre, o) : __shfl_sync(0xffffffffu, ds0, o - A);
#pragma unroll
        for (int j = 0; j < NJ; ++j) acc[j] = fmaf(dz, __ldg(w_mu + (size_t)o * H + lane + 32 * j), acc[j]);
      }
#pragma unroll
      for (int j = 0; j < NJ; ++j) d_feat[(size_t)f * H + lane + 32 * j] = fmaf(g_v, __ldg(w_val + lane + 32 * j), acc[j]);
    }
  }
  if (lane == 0) wpart[warp] = p;
  __syncthreads();
  if (threadIdx.x == 0) {
    LossPartial r = wpart[0];
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) {
      const LossPartial q = wpart[w];
      r.vl += q.vl; r.al += q.al; r.ent += q.ent; r.vsum += q.vsum; r.rsum += q.rsum; r.nclip += q.nclip;
      r.vmin = min_nan(r.vmin, q.vmin); r.vmax = max_nan(r.vmax, q.vmax);
      r.rmin = min_nan(r.rmin, q.rmin); r.rmax = max_nan(r.rmax, q.rmax);
    }
    partials[blockIdx.x] = r;
  }
}

// Weight rows R = L + 1 (mu_maybe_std rows, then the critic): parts[y] = [dW (R x H) | column sums of dl (C = 2A + 1)]
// for frame slab y = blockIdx.y, summed over slabs in order by reduce_partials (no floating-point atomics).
constexpr int kMaxGaussRows = 2 * kMaxGaussA + 1;
__global__ void __launch_bounds__(256, 2)
gaussian_heads_wgrad_kernel(const float* __restrict__ feat, const float* __restrict__ dl, int B, int H, int R, int C,
                            float* __restrict__ parts) {
  float* prow = parts + (size_t)blockIdx.y * ((size_t)R * H + C);
  __shared__ float red[8][kMaxGaussRows][32];
  __shared__ float bred[8][64];
  const int lane = threadIdx.x & 31;
  const int col = blockIdx.x * 32 + lane;
  const int slice = threadIdx.x >> 5;
  const int per = (B + gridDim.y - 1) / gridDim.y;
  const int b0 = blockIdx.y * per, b1 = min(B, b0 + per);
  float acc[kMaxGaussRows];
#pragma unroll
  for (int r = 0; r < kMaxGaussRows; ++r) acc[r] = 0.f;
  float bacc0 = 0.f, bacc1 = 0.f;   // column sums of dl: columns lane and lane + 32 (block column 0 only)
  for (int b = b0 + slice; b < b1; b += 8) {
    const float x = (col < H) ? feat[(size_t)b * H + col] : 0.f;
    const float* drow = dl + (size_t)b * C;
#pragma unroll
    for (int r = 0; r < kMaxGaussRows; ++r)
      if (r < R) acc[r] = fmaf(drow[r], x, acc[r]);
    if (blockIdx.x == 0) {
      if (lane < C) bacc0 += drow[lane];
      if (lane + 32 < C) bacc1 += drow[lane + 32];
    }
  }
#pragma unroll
  for (int r = 0; r < kMaxGaussRows; ++r)
    if (r < R) red[slice][r][lane] = acc[r];
  bred[slice][lane] = bacc0;
  bred[slice][lane + 32] = bacc1;
  __syncthreads();
  if (slice == 0 && col < H) {
    for (int r = 0; r < R; ++r) {
      float s = 0.f;
      for (int w = 0; w < 8; ++w) s += red[w][r][lane];
      prow[(size_t)r * H + col] = s;
    }
  }
  if (blockIdx.x == 0 && slice < 2) {
    const int c = lane + 32 * slice;
    if (c < C) {
      float s = 0.f;
      for (int w = 0; w < 8; ++w) s += bred[w][c];
      prow[(size_t)R * H + c] = s;
    }
  }
}

extern "C" size_t hb200_gaussian_ppo_loss_workspace_bytes(int batch, int hidden, int n_actions) {
  (void)hidden;
  return sizeof(LossPartial) * (size_t)(kNumSMs * 2) + 256 + sizeof(float) * (size_t)batch * (2 * n_actions + 1);
}

extern "C" int hb200_gaussian_ppo_loss(const float* features, const float* w_mu, const float* b_mu,
                                       const float* std_param, const float* w_val, const float* b_val,
                                       const float* actions, const float* old_log_probs, const float* advantages,
                                       const float* old_values, const float* returns, const float* is_coeffs,
                                       int batch, int hidden, int n_actions, int flags, float min_std, float max_std,
                                       float clip_param, float value_loss_coef, float entropy_coef,
                                       int use_clipped_value_loss, int compute_grads, float* values, float* log_probs,
                                       float* entropy, float* d_features, float* d_w_mu, float* d_b_mu, float* d_std,
                                       float* d_w_val, float* d_b_val, float* metrics, void* workspace,
                                       hb200_stream_t stream) {
  HB_CHECK_ARG(features && w_mu && b_mu && w_val && b_val && actions && old_log_probs && advantages && old_values &&
                   returns && metrics && workspace,
               "gaussian_ppo_loss: null pointer");
  HB_CHECK_ARG(batch > 0 && n_actions >= 1 && n_actions <= kMaxGaussA,
               "gaussian_ppo_loss: n_actions=%d unsupported (1..%d)", n_actions, kMaxGaussA);
  HB_CHECK_ARG(hidden == 32 || hidden == 64 || hidden == 128 || hidden == 256 || hidden == 512,
               "gaussian_ppo_loss: hidden=%d unsupported (32,64,128,256,512)", hidden);
  HB_CHECK_ARG((flags & ~HB200_GAUSS_ALL_FLAGS) == 0, "gaussian_ppo_loss: unknown flags 0x%x", flags);
  const bool sp = flags & HB200_GAUSS_STD_PARAM;
  HB_CHECK_ARG(!sp == !std_param, "gaussian_ppo_loss: std_param must be given iff use_std_param");
  HB_CHECK_ARG(!compute_grads || (d_features && d_w_mu && d_b_mu && d_w_val && d_b_val && (!sp || d_std)),
               "gaussian_ppo_loss: compute_grads needs gradient outputs");
  cudaStream_t st = (cudaStream_t)stream;
  LossPartial* partials = (LossPartial*)workspace;
  float* dl = (float*)((char*)workspace + ((sizeof(LossPartial) * (size_t)(kNumSMs * 2) + 255) / 256) * 256);
  const int grid = loss_grid(batch);
#define HB_GLOSS_LAUNCH(NJ)                                                                                        \
  gaussian_loss_main_kernel<NJ><<<grid, 256, 0, st>>>(                                                             \
      features, w_mu, b_mu, std_param, w_val, b_val, actions, old_log_probs, advantages, old_values, returns,      \
      is_coeffs, batch, n_actions, flags, min_std, max_std, clip_param, value_loss_coef, entropy_coef,             \
      use_clipped_value_loss, compute_grads, values, log_probs, entropy, d_features, dl, partials)
  switch (hidden) {
    case 32: HB_GLOSS_LAUNCH(1); break;
    case 64: HB_GLOSS_LAUNCH(2); break;
    case 128: HB_GLOSS_LAUNCH(4); break;
    case 256: HB_GLOSS_LAUNCH(8); break;
    default: HB_GLOSS_LAUNCH(16); break;
  }
#undef HB_GLOSS_LAUNCH
  HB_LAUNCH_OK();
  ppo_loss_finalize_kernel<<<1, 32, 0, st>>>(partials, grid, batch, value_loss_coef, entropy_coef, metrics);
  HB_LAUNCH_OK();
  count_launch(2);
  if (compute_grads) {
    const int A = n_actions, L = sp ? A : 2 * A, R = L + 1, C = 2 * A + 1;
    const long long H = hidden;
    HB_CUDA(cudaMemsetAsync(d_w_mu, 0, sizeof(float) * (size_t)L * H, st));
    HB_CUDA(cudaMemsetAsync(d_b_mu, 0, sizeof(float) * L, st));
    HB_CUDA(cudaMemsetAsync(d_w_val, 0, sizeof(float) * H, st));
    HB_CUDA(cudaMemsetAsync(d_b_val, 0, sizeof(float), st));
    if (sp) HB_CUDA(cudaMemsetAsync(d_std, 0, sizeof(float) * A, st));
    dim3 g(cdiv(hidden, 32), min(32, cdiv(batch, 64)));
    const long long row = (long long)R * H + C;   // one partial row per frame slab
    float* parts = nullptr;
    int* tickets = nullptr;
    int rc = stream_workspace(st, (size_t)(g.y + kReduceChunks) * row, 0, &parts, &tickets);
    if (rc) return rc;
    float* tmp = parts + (size_t)g.y * row;
    gaussian_heads_wgrad_kernel<<<g, 256, 0, st>>>(features, dl, batch, hidden, R, C, parts);
    HB_LAUNCH_OK();
    count_launch(1);
    rc = reduce_partials(parts, g.y, row, (long long)L * H, d_w_mu, tmp, st);
    if (!rc) rc = reduce_partials(parts + (size_t)L * H, g.y, row, H, d_w_val, tmp, st);
    if (!rc) rc = reduce_partials(parts + (size_t)R * H, g.y, row, L, d_b_mu, tmp, st);
    if (!rc) rc = reduce_partials(parts + (size_t)R * H + L, g.y, row, 1, d_b_val, tmp, st);
    if (!rc && sp) rc = reduce_partials(parts + (size_t)R * H + A + 1, g.y, row, A, d_std, tmp, st);
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
  // a NaN norm makes every parameter NaN, as clip_grad_norm_ does (its clamp propagates NaN)
  if (max_norm > 0.f) coef *= min_nan(max_norm / (total_norm + 1e-6f), 1.0f);
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
