// hb200 -- HBM-bound passes around the conv stack (NHWC, 16-byte vectors; forward values fp16 = act_t, gradients
// bf16 = grad_t, see common.cuh):
// input prep (u8/f32 gather + 2x2 mean + running mean/var), GroupNorm apply / residual / maxpool,
// GroupNorm backward (reduce + apply), maxpool backward, dtype converts, goal/action embeddings.
#include "common.cuh"
#include "wgmma.cuh"
#include <cooperative_groups.h>

namespace hb200 {
namespace cg = cooperative_groups;
using wg::cp_async16;
using wg::cp_async_commit;
using wg::cp_async_wait;
using wg::smem_u32;
void count_launch(int n);

static inline int grid_for(long long n, int bs) {
  long long g = (n + bs - 1) / bs;
  const long long cap = (long long)kNumSMs * 16;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

// ======================================================================================
// input prep  (HB/rl/ddppo/policy/resnet_policy.py:255-271, running_mean_and_var.py:24-78)
// ======================================================================================
// one thread = 4 horizontally adjacent pooled pixels (8 input pixels x 2 rows)
template <bool HAS_RGB, bool HAS_DEPTH>
__device__ __forceinline__ void pooled4(const uint8_t* __restrict__ rgb, const float* __restrict__ depth,
                                        size_t row, int H, int W, int py, int px4, float rgb_scale,
                                        float (&out)[4][4]) {
  // out[pixel][channel]; channel order rgb(3) then depth(1)
#pragma unroll
  for (int p = 0; p < 4; ++p)
#pragma unroll
    for (int c = 0; c < 4; ++c) out[p][c] = 0.f;
  if (HAS_RGB) {
    const uint8_t* base = rgb + (row * H + 2 * py) * (size_t)W * 3 + (size_t)px4 * 8 * 3;
    uint8_t v[2][24];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const uint2* src = reinterpret_cast<const uint2*>(base + (size_t)r * W * 3);
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        const uint2 u = __ldg(src + q);
        *reinterpret_cast<uint2*>(&v[r][q * 8]) = u;
      }
    }
#pragma unroll
    for (int p = 0; p < 4; ++p)
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        // avg_pool2d sums the window row-major then divides (ATen); u8 is scaled first
        float s = __fmul_rn((float)v[0][(2 * p) * 3 + c], rgb_scale);
        s = __fadd_rn(s, __fmul_rn((float)v[0][(2 * p + 1) * 3 + c], rgb_scale));
        s = __fadd_rn(s, __fmul_rn((float)v[1][(2 * p) * 3 + c], rgb_scale));
        s = __fadd_rn(s, __fmul_rn((float)v[1][(2 * p + 1) * 3 + c], rgb_scale));
        out[p][c] = s * 0.25f;
      }
  }
  if (HAS_DEPTH) {
    const int dc = HAS_RGB ? 3 : 0;
    const float* base = depth + (row * H + 2 * py) * (size_t)W + (size_t)px4 * 8;
    float d[2][8];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float4* src = reinterpret_cast<const float4*>(base + (size_t)r * W);
      const float4 a = __ldg(src), b = __ldg(src + 1);
      d[r][0] = a.x; d[r][1] = a.y; d[r][2] = a.z; d[r][3] = a.w;
      d[r][4] = b.x; d[r][5] = b.y; d[r][6] = b.z; d[r][7] = b.w;
    }
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      float s = __fadd_rn(d[0][2 * p], d[0][2 * p + 1]);
      s = __fadd_rn(s, d[1][2 * p]);
      s = __fadd_rn(s, d[1][2 * p + 1]);
      out[p][dc] = s * 0.25f;
    }
  }
}

template <bool HAS_RGB, bool HAS_DEPTH>
__global__ void __launch_bounds__(256)
prep_stats_kernel(const uint8_t* __restrict__ rgb, const float* __restrict__ depth,
                  const int32_t* __restrict__ frame_rows, int B, int H, int W, float rgb_scale,
                  double* __restrict__ stats) {
  __shared__ double red[32];
  const int Hp = H / 2, Wq = W / 8;
  const long long total = (long long)B * Hp * Wq;
  float s[4] = {0, 0, 0, 0}, q[4] = {0, 0, 0, 0};
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int px4 = (int)(i % Wq);
    const long long t = i / Wq;
    const int py = (int)(t % Hp);
    const int f = (int)(t / Hp);
    float o[4][4];
    pooled4<HAS_RGB, HAS_DEPTH>(rgb, depth, (size_t)frame_rows[f], H, W, py, px4, rgb_scale, o);
#pragma unroll
    for (int p = 0; p < 4; ++p)
#pragma unroll
      for (int c = 0; c < 4; ++c) { s[c] += o[p][c]; q[c] = fmaf(o[p][c], o[p][c], q[c]); }
  }
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const double a = block_sum((double)s[c], red);
    const double b = block_sum((double)q[c], red);
    if (threadIdx.x == 0) { atomicAdd(&stats[c], a); atomicAdd(&stats[8 + c], b); }
  }
  // frame count (the reference's new_count = x.size(0), running_mean_and_var.py:27,36): written on the device -- no
  // pageable-host copy in the hot path, safe under stream capture
  if (blockIdx.x == 0 && threadIdx.x == 0) stats[16] = (double)B;
}

// S2D: write the pooled image space-to-depth'd, [B, Hp/2, Wp/2, 16] with channel = (dy*2+dx)*4 + c
// (c < 4), so the 7x7 stride-2 stem becomes a 4x4 stride-1 convolution (conv_halo.cu).
template <bool HAS_RGB, bool HAS_DEPTH, bool S2D>
__global__ void __launch_bounds__(256)
prep_apply_kernel(const uint8_t* __restrict__ rgb, const float* __restrict__ depth,
                  const int32_t* __restrict__ frame_rows, int B, int H, int W, float rgb_scale,
                  const float* __restrict__ scale_shift, act_t* __restrict__ out, grad_t* __restrict__ out2) {
  const int Hp = H / 2, Wq = W / 8;
  const long long total = (long long)B * Hp * Wq;
  float sc[4] = {1, 1, 1, 1}, sh[4] = {0, 0, 0, 0};
  if (scale_shift) {
#pragma unroll
    for (int c = 0; c < 4; ++c) { sc[c] = scale_shift[c]; sh[c] = scale_shift[8 + c]; }
  }
  const int C = (HAS_RGB ? 3 : 0) + (HAS_DEPTH ? 1 : 0);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int px4 = (int)(i % Wq);
    const long long t = i / Wq;
    const int py = (int)(t % Hp);
    const int f = (int)(t / Hp);
    float o[4][4];
    pooled4<HAS_RGB, HAS_DEPTH>(rgb, depth, (size_t)frame_rows[f], H, W, py, px4, rgb_scale, o);
    if (!S2D) {
      uint4* dst = reinterpret_cast<uint4*>(out + (((size_t)f * Hp + py) * (W / 2) + (size_t)px4 * 4) * 8);
#pragma unroll
      for (int p = 0; p < 4; ++p) {
        float v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
#pragma unroll
        for (int c = 0; c < 4; ++c)
          if (c < C) v[c] = fmaf(o[p][c], sc[c], sh[c]);
        dst[p] = pack8a(v);
        if (out2) reinterpret_cast<uint4*>(out2 + (((size_t)f * Hp + py) * (W / 2) + (size_t)px4 * 4) * 8)[p] = pack8(v);
      }
    } else {
      // pooled pixels (py, 4*px4 + p): s2d row i = py/2, dy = py&1; col j = 2*px4 + p/2, dx = p&1
      const int i2 = py >> 1, dy = py & 1;
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        float v[8];
#pragma unroll
        for (int dx = 0; dx < 2; ++dx)
#pragma unroll
          for (int c = 0; c < 4; ++c) v[dx * 4 + c] = (c < C) ? fmaf(o[2 * q + dx][c], sc[c], sh[c]) : 0.f;
        const size_t pix = ((size_t)f * (Hp / 2) + i2) * (W / 4) + (size_t)px4 * 2 + q;
        *reinterpret_cast<uint4*>(out + pix * 16 + dy * 8) = pack8a(v);
        if (out2) *reinterpret_cast<uint4*>(out2 + pix * 16 + dy * 8) = pack8(v);
      }
    }
  }
}

__global__ void prep_finalize_kernel(const double* __restrict__ stats, float* __restrict__ run_mean,
                                     float* __restrict__ run_var, float* __restrict__ run_count,
                                     float* __restrict__ scale_shift, int C, long long pix_per_frame,
                                     int update) {
  const int c = threadIdx.x;
  __shared__ float s_count;
  if (c == 0) s_count = run_count[0];
  __syncthreads();
  if (c < C) {
    float mean = run_mean[c], var = run_var[c];
    if (update) {
      const double frames = stats[16];
      const double n_el = frames * (double)pix_per_frame;
      const double nm = stats[c] / n_el;
      double nv = stats[8 + c] / n_el - nm * nm;
      if (nv < 0) nv = 0;
      const float count = s_count, new_count = (float)frames;
      const float new_mean = (float)nm, new_var = (float)nv;
      // parallel-variance merge, running_mean_and_var.py:50-66
      const float m_a = var * count, m_b = new_var * new_count;
      const float d = new_mean - mean;
      const float M2 = m_a + m_b + d * d * count * new_count / (count + new_count);
      var = M2 / (count + new_count);
      mean = (count * mean + new_count * new_mean) / (count + new_count);
      run_mean[c] = mean;
      run_var[c] = var;
    }
    const float inv = 1.0f / sqrtf(fmaxf(var, 1e-2f));
    scale_shift[c] = inv;
    scale_shift[8 + c] = -mean * inv;
  } else if (c < 8) {
    scale_shift[c] = 0.f;
    scale_shift[8 + c] = 0.f;
  }
  __syncthreads();
  if (c == 0 && update) run_count[0] = s_count + (float)stats[16];
}

// ======================================================================================
// GroupNorm helpers
// ======================================================================================
struct GnP {
  const double* stats;  // [B,G,2] sum, sumsq (double accumulators)
  const float* gamma;
  const float* beta;
  int C, G, lcpg;  // lcpg = log2(channels per group)
  float inv_m, eps;
};

// mean/rstd for the 8 channels starting at c0 of frame b
__device__ __forceinline__ void gn_coeffs(const GnP& p, int b, int c0, float (&mu)[8], float (&rs)[8]) {
  int prev = -1;
  float m = 0.f, r = 0.f;
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int g = (c0 + e) >> p.lcpg;
    if (g != prev) {
      const double2 st = *reinterpret_cast<const double2*>(p.stats + ((size_t)b * p.G + g) * 2);
      const double md = st.x * (double)p.inv_m;
      m = (float)md;
      const float var = max_nan((float)(st.y * (double)p.inv_m - md * md), 0.f);   // NaN statistics stay NaN
      r = rsqrtf(var + p.eps);
      prev = g;
    }
    mu[e] = m;
    rs[e] = r;
  }
}
__device__ __forceinline__ void load8f(const float* __restrict__ p, float (&f)[8]) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p));
  const float4 b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}

// The three per-layer GroupNorm passes below share one mapping: block = (frame, pixel slab),
// thread = (8-channel vector, pixel lane).  All per-channel / per-group coefficients are hoisted
// out of the pixel loop, so the inner loop is load - 8 FMAs - store: HBM-bound.
struct GnSlab {
  int b, vec, c0, pix0, pix1, npl, pl;
};
__device__ __forceinline__ GnSlab gn_slab(int C, int hw, int ppb) {
  GnSlab s;
  const int cv = C >> 3;
  const int slabs = (hw + ppb - 1) / ppb;
  s.b = blockIdx.x / slabs;
  const int slab = blockIdx.x - s.b * slabs;
  s.vec = threadIdx.x % cv;
  s.pl = threadIdx.x / cv;
  s.npl = blockDim.x / cv;
  s.c0 = s.vec << 3;
  s.pix0 = slab * ppb;
  s.pix1 = min(hw, s.pix0 + ppb);
  return s;
}

template <int OUT_F32>  // 0: bf16 NHWC, 1: f32 NHWC, 2: f32 flattened in (c, h, w) order (nn.Flatten of NCHW)
__global__ void __launch_bounds__(256)
gn_apply_kernel(const act_t* __restrict__ y, GnP p, void* __restrict__ out, grad_t* __restrict__ out2, int B, int hw,
                int relu, int ppb) {
  const GnSlab t = gn_slab(p.C, hw, ppb);
  const int cv = p.C >> 3;
  float mu[8], rs[8], ga[8], be[8], sc[8], sh[8];
  gn_coeffs(p, t.b, t.c0, mu, rs);
  load8f(p.gamma + t.c0, ga);
  load8f(p.beta + t.c0, be);
#pragma unroll
  for (int e = 0; e < 8; ++e) { sc[e] = rs[e] * ga[e]; sh[e] = fmaf(-mu[e], sc[e], be[e]); }
  for (int pix = t.pix0 + t.pl; pix < t.pix1; pix += t.npl) {
    const size_t i = ((size_t)t.b * hw + pix) * cv + t.vec;
    float x[8];
    unpack8a(reinterpret_cast<const uint4*>(y)[i], x);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float z = fmaf(x[e], sc[e], sh[e]);
      x[e] = relu ? max_nan(z, 0.f) : z;
    }
    if (OUT_F32 == 1) {
      float4* o = reinterpret_cast<float4*>(out) + 2 * i;
      o[0] = make_float4(x[0], x[1], x[2], x[3]);
      o[1] = make_float4(x[4], x[5], x[6], x[7]);
    } else if (OUT_F32 == 2) {
      float* o = reinterpret_cast<float*>(out) + (size_t)t.b * p.C * hw;
#pragma unroll
      for (int e = 0; e < 8; ++e) o[(size_t)(t.c0 + e) * hw + pix] = x[e];
    } else {
      reinterpret_cast<uint4*>(out)[i] = pack8a(x);
      if (out2) reinterpret_cast<uint4*>(out2)[i] = pack8(x);   // bf16 twin for the weight-gradient kernels
    }
  }
}

__global__ void __launch_bounds__(256)
gn_residual_relu_kernel(const act_t* __restrict__ y, GnP p, const act_t* __restrict__ res,
                        GnP rp, int res_is_prenorm, act_t* __restrict__ out, grad_t* __restrict__ out2, int B, int hw,
                        int ppb) {
  const GnSlab t = gn_slab(p.C, hw, ppb);
  const int cv = p.C >> 3;
  float mu[8], rs[8], ga[8], be[8], sc[8], sh[8], rsc[8], rsh[8];
  gn_coeffs(p, t.b, t.c0, mu, rs);
  load8f(p.gamma + t.c0, ga);
  load8f(p.beta + t.c0, be);
#pragma unroll
  for (int e = 0; e < 8; ++e) { sc[e] = rs[e] * ga[e]; sh[e] = fmaf(-mu[e], sc[e], be[e]); rsc[e] = 1.f; rsh[e] = 0.f; }
  if (res_is_prenorm) {
    gn_coeffs(rp, t.b, t.c0, mu, rs);
    load8f(rp.gamma + t.c0, ga);
    load8f(rp.beta + t.c0, be);
#pragma unroll
    for (int e = 0; e < 8; ++e) { rsc[e] = rs[e] * ga[e]; rsh[e] = fmaf(-mu[e], rsc[e], be[e]); }
  }
  for (int pix = t.pix0 + t.pl; pix < t.pix1; pix += t.npl) {
    const size_t i = ((size_t)t.b * hw + pix) * cv + t.vec;
    float x[8], r[8];
    unpack8a(reinterpret_cast<const uint4*>(y)[i], x);
    unpack8a(reinterpret_cast<const uint4*>(res)[i], r);
#pragma unroll
    for (int e = 0; e < 8; ++e) x[e] = max_nan(fmaf(x[e], sc[e], sh[e]) + fmaf(r[e], rsc[e], rsh[e]), 0.f);
    reinterpret_cast<uint4*>(out)[i] = pack8a(x);
    if (out2) reinterpret_cast<uint4*>(out2)[i] = pack8(x);
  }
}

__global__ void __launch_bounds__(256)
gn_relu_maxpool_kernel(const act_t* __restrict__ y, GnP p, act_t* __restrict__ out, grad_t* __restrict__ out2,
                       uint8_t* __restrict__ argmax, int B, int H, int W) {
  const int cv = p.C >> 3, Ho = (H + 1) / 2, Wo = (W + 1) / 2;   // MaxPool2d(3, 2, 1): floor((H + 2 - 3) / 2) + 1
  const long long total = (long long)B * Ho * Wo * cv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c0 = (int)(i % cv) << 3;
    long long t = i / cv;
    const int ox = (int)(t % Wo);
    t /= Wo;
    const int oy = (int)(t % Ho);
    const int b = (int)(t / Ho);
    float mu[8], rs[8], ga[8], be[8], best[8];
    int arg[8];
    gn_coeffs(p, b, c0, mu, rs);
    load8f(p.gamma + c0, ga);
    load8f(p.beta + c0, be);
#pragma unroll
    for (int e = 0; e < 8; ++e) { best[e] = -INFINITY; arg[e] = 0; }
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int iy = 2 * oy - 1 + r;
      if (iy < 0 || iy >= H) continue;
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        const int ix = 2 * ox - 1 + s;
        if (ix < 0 || ix >= W) continue;
        float x[8];
        unpack8a(*reinterpret_cast<const uint4*>(y + (((size_t)b * H + iy) * W + ix) * p.C + c0), x);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const float z = max_nan(fmaf((x[e] - mu[e]) * rs[e], ga[e], be[e]), 0.f);
          if (z > best[e] || z != z) { best[e] = z; arg[e] = r * 3 + s; }   // MaxPool2d: a NaN tap wins
        }
      }
    }
    reinterpret_cast<uint4*>(out)[i] = pack8a(best);
    if (out2) reinterpret_cast<uint4*>(out2)[i] = pack8(best);
    uint2 a;
    a.x = (uint32_t)arg[0] | ((uint32_t)arg[1] << 8) | ((uint32_t)arg[2] << 16) | ((uint32_t)arg[3] << 24);
    a.y = (uint32_t)arg[4] | ((uint32_t)arg[5] << 8) | ((uint32_t)arg[6] << 16) | ((uint32_t)arg[7] << 24);
    reinterpret_cast<uint2*>(argmax)[i] = a;
  }
}

// Row-slab variant: a CTA stages rows+1 input rows (one halo row above) in shared memory with cp.async and pools
// from there, so y crosses HBM once (plus 1/rows re-read of the halo row) in fully coalesced 16-byte copies.  The
// window maximum is taken on x * sign(rstd*gamma) (the affine map is monotonic per channel) and the affine + ReLU
// applied once per output.
__global__ void __launch_bounds__(256)
gn_relu_maxpool_slab_kernel(const act_t* __restrict__ y, GnP p, act_t* __restrict__ out, grad_t* __restrict__ out2,
                            uint8_t* __restrict__ argmax, int H, int W, int rows) {
  extern __shared__ __align__(16) uint8_t gsm[];
  uint4* sy = reinterpret_cast<uint4*>(gsm);
  const int cv = p.C >> 3, Ho = H >> 1, Wo = W >> 1, nslab = H / rows;
  const int b = blockIdx.x / nslab, slab = blockIdx.x - b * nslab;
  const int iy0 = slab * rows, yrow = W * cv;
  const int tid = threadIdx.x;
  {
    const int lr0 = iy0 == 0 ? 1 : 0;  // local row 0 is input row iy0-1 (absent for the first slab)
    const uint4* gy = reinterpret_cast<const uint4*>(y) + ((size_t)b * H + iy0 - 1 + lr0) * yrow;
    const uint32_t ay = smem_u32(sy) + lr0 * yrow * 16;
    const int n = (rows + 1 - lr0) * yrow;
    for (int i = tid; i < n; i += 256) cp_async16(ay + i * 16, gy + i, true);
    cp_async_commit();
  }
  const int vec = tid % cv, c0 = vec << 3;
  float sg[8], za[8], zd[8];
  {
    float mu[8], rs[8], ga[8], be[8];
    gn_coeffs(p, b, c0, mu, rs);
    load8f(p.gamma + c0, ga);
    load8f(p.beta + c0, be);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float zc = rs[e] * ga[e];
      // zc == 0: every tap's value is relu(beta); sg = 0 makes every x * sg equal, so the strict > below keeps the
      // first valid tap, as MaxPool2d does.  A NaN zc (NaN statistics) makes every tap NaN (sg = zc * 0 = NaN).
      sg[e] = zc < 0.f ? -1.f : (zc > 0.f ? 1.f : zc * 0.f);
      za[e] = fabsf(zc);
      zd[e] = fmaf(-mu[e], zc, be[e]);
    }
  }
  cp_async_wait<0>();
  __syncthreads();
  const int nout = (rows >> 1) * Wo * cv;
  uint4* o4 = reinterpret_cast<uint4*>(out) + ((size_t)b * Ho + (iy0 >> 1)) * Wo * cv;
  uint4* o4b = out2 ? reinterpret_cast<uint4*>(out2) + ((size_t)b * Ho + (iy0 >> 1)) * Wo * cv : nullptr;
  uint2* a2 = reinterpret_cast<uint2*>(argmax) + ((size_t)b * Ho + (iy0 >> 1)) * Wo * cv;
  for (int it = tid; it < nout; it += 256) {
    const int pos = it / cv, ol = pos / Wo, ox = pos - ol * Wo;
    float best[8];
    int arg[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) { best[e] = -INFINITY; arg[e] = 0; }
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int lr = 2 * ol + r;  // local row; input row iy0 - 1 + lr
      if (iy0 + lr < 1) continue;
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        const int ix = 2 * ox - 1 + s;
        if (ix < 0) continue;
        float x[8];
        unpack8a(sy[(lr * W + ix) * cv + vec], x);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const float xs = x[e] * sg[e];
          if (xs > best[e] || xs != xs) { best[e] = xs; arg[e] = r * 3 + s; }   // MaxPool2d: a NaN tap wins
        }
      }
    }
    float z[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) z[e] = max_nan(fmaf(best[e], za[e], zd[e]), 0.f);
    o4[it] = pack8a(z);
    if (o4b) o4b[it] = pack8(z);
    uint2 a;
    a.x = (uint32_t)arg[0] | ((uint32_t)arg[1] << 8) | ((uint32_t)arg[2] << 16) | ((uint32_t)arg[3] << 24);
    a.y = (uint32_t)arg[4] | ((uint32_t)arg[5] << 8) | ((uint32_t)arg[6] << 16) | ((uint32_t)arg[7] << 24);
    a2[it] = a;
  }
}

__global__ void __launch_bounds__(256)
maxpool_bwd_kernel(const grad_t* __restrict__ dout, const uint8_t* __restrict__ argmax,
                   grad_t* __restrict__ dz, int B, int H, int W, int C) {
  const int cv = C >> 3, Ho = (H + 1) / 2, Wo = (W + 1) / 2;
  const long long total = (long long)B * H * W * cv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c0 = (int)(i % cv) << 3;
    long long t = i / cv;
    const int ix = (int)(t % W);
    t /= W;
    const int iy = (int)(t % H);
    const int b = (int)(t / H);
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    // windows (oy,ox) with 2*o-1 <= i <= 2*o+1
    const int oy_lo = iy >> 1, oy_hi = (iy + 1) >> 1;
    const int ox_lo = ix >> 1, ox_hi = (ix + 1) >> 1;
    for (int oy = oy_lo; oy <= oy_hi; ++oy) {
      if (oy >= Ho) continue;
      const int r = iy - (2 * oy - 1);
      for (int ox = ox_lo; ox <= ox_hi; ++ox) {
        if (ox >= Wo) continue;
        const int s = ix - (2 * ox - 1);
        const int code = r * 3 + s;
        const size_t o = (((size_t)b * Ho + oy) * Wo + ox) * C + c0;
        const uint2 a = *reinterpret_cast<const uint2*>(argmax + o);
        float g[8];
        unpack8(*reinterpret_cast<const uint4*>(dout + o), g);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const int am = (int)(((e < 4 ? a.x : a.y) >> ((e & 3) * 8)) & 0xff);
          if (am == code) acc[e] += g[e];
        }
      }
    }
    reinterpret_cast<uint4*>(dz)[i] = pack8(acc);
  }
}

// ---- GroupNorm backward ----------------------------------------------------------------
// gz = g * mask;  per (frame, channel): a = sum gz, bb = sum gz*xhat
//   dbeta += a, dgamma += bb, sums[b,g] += (gamma*a, gamma*bb)
// dy = rstd * (gamma*gz - (S1 + xhat*S2)/m)
__device__ __forceinline__ void gn_masked_grad(int mask_mode, const float (&g)[8], const float (&z)[8],
                                               const float (&act)[8], float (&gz)[8]) {
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    float m = 1.f;
    if (mask_mode == 1) m = z[e] > 0.f ? 1.f : 0.f;
    if (mask_mode == 2) m = act[e] > 0.f ? 1.f : 0.f;
    gz[e] = g[e] * m;
  }
}

__global__ void __launch_bounds__(256)
gn_bwd_reduce_kernel(const grad_t* __restrict__ g, const act_t* __restrict__ act,
                     const act_t* __restrict__ y, GnP p, float* __restrict__ sums,
                     float* __restrict__ dgamma, float* __restrict__ dbeta, int B, int hw,
                     int pix_per_block, int mask_mode) {
  // block = (frame b, pixel slab); thread = (pixel lane, channel vector)
  __shared__ float sa[256][9], sb[256][9];
  const int cv = p.C >> 3;
  const int slabs = (hw + pix_per_block - 1) / pix_per_block;
  const int b = blockIdx.x / slabs, slab = blockIdx.x % slabs;
  const int vec = threadIdx.x % cv, pl = threadIdx.x / cv, npl = blockDim.x / cv;
  const int c0 = vec << 3;
  float mu[8], rs[8], ga[8], be[8], a[8], bb[8];
  gn_coeffs(p, b, c0, mu, rs);
  load8f(p.gamma + c0, ga);
  load8f(p.beta + c0, be);
#pragma unroll
  for (int e = 0; e < 8; ++e) { a[e] = 0.f; bb[e] = 0.f; }
  const int p1 = min(hw, (slab + 1) * pix_per_block);
  for (int pix = slab * pix_per_block + pl; pix < p1; pix += npl) {
    const size_t o = ((size_t)b * hw + pix) * cv + vec;
    float gg[8], x[8], z[8], ac[8], gz[8];
    unpack8(reinterpret_cast<const uint4*>(g)[o], gg);
    unpack8a(reinterpret_cast<const uint4*>(y)[o], x);
    if (mask_mode == 2) unpack8a(reinterpret_cast<const uint4*>(act)[o], ac);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      x[e] = (x[e] - mu[e]) * rs[e];
      z[e] = fmaf(x[e], ga[e], be[e]);
      if (mask_mode != 2) ac[e] = 0.f;
    }
    gn_masked_grad(mask_mode, gg, z, ac, gz);
#pragma unroll
    for (int e = 0; e < 8; ++e) { a[e] += gz[e]; bb[e] = fmaf(gz[e], x[e], bb[e]); }
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) { sa[threadIdx.x][e] = a[e]; sb[threadIdx.x][e] = bb[e]; }
  __syncthreads();
  // thread c (< C) finishes channel c
  for (int c = threadIdx.x; c < p.C; c += blockDim.x) {
    const int v = c >> 3, e = c & 7;
    float ta = 0.f, tb = 0.f;
    for (int q = 0; q < npl; ++q) { ta += sa[q * cv + v][e]; tb += sb[q * cv + v][e]; }
    atomicAdd(&dbeta[c], ta);
    atomicAdd(&dgamma[c], tb);
    const float gm = p.gamma[c];
    float* s = sums + ((size_t)b * p.G + (c >> p.lcpg)) * 2;
    atomicAdd(s, gm * ta);
    atomicAdd(s + 1, gm * tb);
  }
}

__global__ void __launch_bounds__(256)
gn_bwd_apply_kernel(const grad_t* __restrict__ g, const act_t* __restrict__ act,
                    const act_t* __restrict__ y, GnP p, const float* __restrict__ sums,
                    grad_t* __restrict__ dy, grad_t* __restrict__ gz_out, int B, int hw,
                    int mask_mode, int ppb) {
  const GnSlab t = gn_slab(p.C, hw, ppb);
  const int cv = p.C >> 3;
  float mu[8], rs[8], ga[8], be[8], k1[8], k2[8], k3[8];
  gn_coeffs(p, t.b, t.c0, mu, rs);
  load8f(p.gamma + t.c0, ga);
  load8f(p.beta + t.c0, be);
  // dy = rs*ga*gz - rs*inv_m*S1 - xhat * rs*inv_m*S2
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const float2 sm = *reinterpret_cast<const float2*>(sums + ((size_t)t.b * p.G + ((t.c0 + e) >> p.lcpg)) * 2);
    k1[e] = rs[e] * ga[e];
    k2[e] = rs[e] * p.inv_m * sm.x;
    k3[e] = rs[e] * p.inv_m * sm.y;
  }
  for (int pix = t.pix0 + t.pl; pix < t.pix1; pix += t.npl) {
    const size_t i = ((size_t)t.b * hw + pix) * cv + t.vec;
    float gg[8], x[8], z[8], ac[8], gz[8], o[8];
    unpack8(reinterpret_cast<const uint4*>(g)[i], gg);
    unpack8a(reinterpret_cast<const uint4*>(y)[i], x);
    if (mask_mode == 2) unpack8a(reinterpret_cast<const uint4*>(act)[i], ac);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      x[e] = (x[e] - mu[e]) * rs[e];
      z[e] = fmaf(x[e], ga[e], be[e]);
      if (mask_mode != 2) ac[e] = 0.f;
    }
    gn_masked_grad(mask_mode, gg, z, ac, gz);
#pragma unroll
    for (int e = 0; e < 8; ++e) o[e] = fmaf(k1[e], gz[e], -fmaf(x[e], k3[e], k2[e]));
    reinterpret_cast<uint4*>(dy)[i] = pack8(o);
    if (gz_out) reinterpret_cast<uint4*>(gz_out)[i] = pack8(gz);
  }
}

// GroupNorm (+ReLU) backward, frame held ON CHIP: a thread-block cluster owns one frame, each CTA of the cluster
// stages its pixel slice of g / y (/ act) in shared memory with cp.async (every thread later consumes exactly the
// 16-byte vectors it copied, so no block barrier is needed between copy and use), reduces the per-channel sums,
// exchanges them with its peers through distributed shared memory, then writes dy (/ gz) from the staged copy.
// HBM traffic is the algorithmic minimum (every operand read once, every result written once); slices are sized
// to <= 48 KB so 4+ CTAs are resident per SM and the copy / reduce / write phases of different frames overlap.

// Shared tail of the cluster GroupNorm-backward kernels: per-thread partial sums (a = sum gz, bx = sum gz*x over
// the thread's elements of channel vector `vec`) -> warp shuffle -> CTA -> cluster (DSMEM) -> the frame's row of the
// dgamma / dbeta partials [B][C] (cluster rank 0) -> per-group S1/S2 -> the per-channel dy coefficients c2, c3.  Ends with a cluster
// barrier ARRIVE; the caller must execute the matching WAIT before it exits.
__device__ __forceinline__ void gn_bwd_cluster_sums(cg::cluster_group& cluster, const GnP& p, int b, int CS, int rank,
                                                    int c0, float (&a)[8], float (&bx)[8], float* part, float* tot,
                                                    float* wred, float* gS, float* __restrict__ dgamma,
                                                    float* __restrict__ dbeta, float (&c2)[8], float (&c3)[8]) {
  const int C = p.C, G = p.G, cv = C >> 3;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // lanes l, l+cv, l+2cv, ... of a warp own the same channel vector
  for (int o = cv; o < 32; o <<= 1) {
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      a[e] += __shfl_xor_sync(0xffffffffu, a[e], o);
      bx[e] += __shfl_xor_sync(0xffffffffu, bx[e], o);
    }
  }
  if (lane < cv) {
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      wred[warp * 2 * C + c0 + e] = a[e];
      wred[warp * 2 * C + C + c0 + e] = bx[e];
    }
  }
  __syncthreads();
  for (int c = tid; c < 2 * C; c += 256) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += wred[w * 2 * C + c];
    part[c] = t;
  }
  cluster.sync();
  for (int c = tid; c < C; c += 256) {
    float ta = 0.f, tx = 0.f;
    for (int r = 0; r < CS; ++r) {
      const float* pr = cluster.map_shared_rank(part, r);
      ta += pr[c];
      tx += pr[C + c];
    }
    const double2 st = *reinterpret_cast<const double2*>(p.stats + ((size_t)b * G + (c >> p.lcpg)) * 2);
    const double md = st.x * (double)p.inv_m;
    const float m = (float)md;
    const float r = rsqrtf(max_nan((float)(st.y * (double)p.inv_m - md * md), 0.f) + p.eps);
    const float tb = r * (tx - m * ta);  // sum gz * xhat
    tot[c] = ta;
    tot[C + c] = tb;
    if (rank == 0) {   // this frame's row of the dgamma / dbeta partials (summed in order by reduce_partials)
      dbeta[(size_t)b * C + c] = ta;
      dgamma[(size_t)b * C + c] = tb;
    }
  }
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");  // peers may exit once all have read
  __syncthreads();
  const int cpg = 1 << p.lcpg;
  for (int gi = tid; gi < G; gi += 256) {
    float s1 = 0.f, s2 = 0.f;
    for (int c = gi * cpg; c < (gi + 1) * cpg; ++c) {
      const float gm = p.gamma[c];
      s1 = fmaf(gm, tot[c], s1);
      s2 = fmaf(gm, tot[C + c], s2);
    }
    gS[gi] = s1;
    gS[G + gi] = s2;
  }
  __syncthreads();
  // dy = zc*gz - xhat*k3 - k2  with xhat = (x - mu)*rs, k2 = rs*S1/m, k3 = rs*S2/m   ==  zc*gz + (x*c3 + c2)
  {
    float mu[8], rs[8];
    gn_coeffs(p, b, c0, mu, rs);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int gi = (c0 + e) >> p.lcpg;
      const float k2 = rs[e] * p.inv_m * gS[gi], k3 = rs[e] * p.inv_m * gS[G + gi];
      c3[e] = -rs[e] * k3;
      c2[e] = fmaf(mu[e] * rs[e], k3, -k2);
    }
  }
}

template <int MODE>
__global__ void __launch_bounds__(256, 4)
gn_bwd_cluster_kernel(const grad_t* __restrict__ g, const act_t* __restrict__ act,
                      const act_t* __restrict__ y, GnP p, float* __restrict__ dgamma,
                      float* __restrict__ dbeta, grad_t* __restrict__ dy,
                      grad_t* __restrict__ gz_out, int hw, int ppc) {
  extern __shared__ __align__(16) uint8_t gsm[];
  cg::cluster_group cluster = cg::this_cluster();
  const int CS = (int)cluster.num_blocks(), rank = (int)cluster.block_rank();
  const int b = blockIdx.x / CS;
  const int cv = p.C >> 3, C = p.C;
  const int pix0 = rank * ppc, pix1 = min(hw, pix0 + ppc);
  const int n = max(pix1 - pix0, 0) * cv, ncap = ppc * cv;
  uint4* sg = reinterpret_cast<uint4*>(gsm);
  uint4* sy = sg + ncap;
  uint4* sact = sy + ncap;
  float* part = reinterpret_cast<float*>(sy + (MODE == 2 ? 2 : 1) * ncap);  // [2C] this CTA's channel sums
  float* tot = part + 2 * C;                                                  // [2C] cluster totals
  float* wred = tot + 2 * C;                                                  // [8][2C]
  float* gS = wred + 16 * C;                                                  // [2G]
  const size_t base = ((size_t)b * hw + pix0) * cv;
  const int tid = threadIdx.x;
  {
    const uint4* gg = reinterpret_cast<const uint4*>(g) + base;
    const uint4* gy = reinterpret_cast<const uint4*>(y) + base;
    const uint4* ga = reinterpret_cast<const uint4*>(act) + base;
    const uint32_t ag = smem_u32(sg), ay = smem_u32(sy), aa = smem_u32(sact);
    for (int i = tid; i < n; i += 256) {
      cp_async16(ag + i * 16, gg + i, true);
      cp_async16(ay + i * 16, gy + i, true);
      if (MODE == 2) cp_async16(aa + i * 16, ga + i, true);
    }
    cp_async_commit();
  }
  const int vec = tid % cv, c0 = vec << 3;
  // z = x*zc + zd (only its sign is needed: the ReLU mask); zc = rstd*gamma is also the dy coefficient of gz
  float zc[8], zd[8];
  {
    float mu[8], rs[8], ga[8], be[8];
    gn_coeffs(p, b, c0, mu, rs);
    load8f(p.gamma + c0, ga);
    load8f(p.beta + c0, be);
#pragma unroll
    for (int e = 0; e < 8; ++e) { zc[e] = rs[e] * ga[e]; zd[e] = fmaf(-mu[e], zc[e], be[e]); }
  }
  cp_async_wait<0>();
  float a[8], bx[8];  // sum gz, sum gz*x (raw x; converted to sum gz*xhat per channel below)
#pragma unroll
  for (int e = 0; e < 8; ++e) { a[e] = 0.f; bx[e] = 0.f; }
  for (int i = tid; i < n; i += 256) {
    float gg[8], x[8], ac[8];
    unpack8(sg[i], gg);
    unpack8a(sy[i], x);
    if (MODE == 2) unpack8a(sact[i], ac);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      float gz = gg[e];
      if (MODE == 1) gz = fmaf(x[e], zc[e], zd[e]) > 0.f ? gz : 0.f;
      if (MODE == 2) gz = ac[e] > 0.f ? gz : 0.f;
      a[e] += gz;
      bx[e] = fmaf(gz, x[e], bx[e]);
    }
  }
  float c2[8], c3[8];
  gn_bwd_cluster_sums(cluster, p, b, CS, rank, c0, a, bx, part, tot, wred, gS, dgamma, dbeta, c2, c3);
  uint4* od = reinterpret_cast<uint4*>(dy) + base;
  uint4* oz = reinterpret_cast<uint4*>(gz_out) + base;
  for (int i = tid; i < n; i += 256) {
    float gg[8], x[8], ac[8], gz[8], o[8];
    unpack8(sg[i], gg);
    unpack8a(sy[i], x);
    if (MODE == 2) unpack8a(sact[i], ac);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      gz[e] = gg[e];
      if (MODE == 1) gz[e] = fmaf(x[e], zc[e], zd[e]) > 0.f ? gz[e] : 0.f;
      if (MODE == 2) gz[e] = ac[e] > 0.f ? gz[e] : 0.f;
      o[e] = fmaf(zc[e], gz[e], fmaf(x[e], c3[e], c2[e]));
    }
    od[i] = pack8(o);
    if (gz_out) oz[i] = pack8(gz);
  }
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// Stem backward: MaxPool(3,2,1) backward + ReLU backward + GroupNorm backward in one pass.  The full-resolution
// gradient of the pooled activation is never materialised: every CTA stages its rows of y plus the pooled-gradient /
// argmax rows that can route into them (R/2+1 pooled rows for R input rows), and evaluates
//   gz(iy,ix,c) = [z > 0] * sum over the <= 4 windows (oy,ox) containing (iy,ix) of [argmax(oy,ox,c) == tap] * dpool
// from shared memory in both phases.  Reference: resnet.py:244-252 (conv1 / GroupNorm / ReLU / MaxPool2d).
// gz += [argmax == code] * dpool for the 8 channels of one pooled window (o = its vector index in the staged rows)
__device__ __forceinline__ void pool_take(const uint4* __restrict__ sdp, const uint2* __restrict__ sarg, int o,
                                          uint32_t code, float (&gz)[8]) {
  const uint2 am = sarg[o];
  const uint4 dp = sdp[o];
  const uint32_t c4 = code * 0x01010101u;
  const uint32_t m0 = __vcmpeq4(am.x, c4), m1 = __vcmpeq4(am.y, c4);  // 0xff per matching channel
  const float2 f0 = unpack_bf16x2(dp.x & __byte_perm(m0, 0, 0x1100));
  const float2 f1 = unpack_bf16x2(dp.y & __byte_perm(m0, 0, 0x3322));
  const float2 f2 = unpack_bf16x2(dp.z & __byte_perm(m1, 0, 0x1100));
  const float2 f3 = unpack_bf16x2(dp.w & __byte_perm(m1, 0, 0x3322));
  gz[0] += f0.x; gz[1] += f0.y; gz[2] += f1.x; gz[3] += f1.y;
  gz[4] += f2.x; gz[5] += f2.y; gz[6] += f3.x; gz[7] += f3.y;
}

// Pooled gradient routed to input pixel (2k+DY, 2j+DX): the windows containing it and the tap it is in each are
// compile-time constants (row 2k: window k tap r=1; row 2k+1: window k tap 2 and window k+1 tap 0; same for columns).
// o00 = vector index of window (k, j) in the staged pooled rows; row_ok / col_ok: windows k+1 / j+1 exist.
template <int DY, int DX>
__device__ __forceinline__ void pool_route_px(const uint4* __restrict__ sdp, const uint2* __restrict__ sarg, int o00,
                                              int wrow, int cv, bool row_ok, bool col_ok, float (&gz)[8]) {
#pragma unroll
  for (int e = 0; e < 8; ++e) gz[e] = 0.f;
  constexpr int r0 = DY == 0 ? 1 : 2, s0 = DX == 0 ? 1 : 2;
  pool_take(sdp, sarg, o00, r0 * 3 + s0, gz);
  if (DX == 1 && col_ok) pool_take(sdp, sarg, o00 + cv, r0 * 3 + 0, gz);
  if (DY == 1 && row_ok) {
    pool_take(sdp, sarg, o00 + wrow, 0 * 3 + s0, gz);
    if (DX == 1 && col_ok) pool_take(sdp, sarg, o00 + wrow + cv, 0, gz);
  }
}

__global__ void __launch_bounds__(256, 3)
gn_pool_bwd_cluster_kernel(const grad_t* __restrict__ dpool, const uint8_t* __restrict__ argmax,
                           const act_t* __restrict__ y, GnP p, float* __restrict__ dgamma,
                           float* __restrict__ dbeta, grad_t* __restrict__ dy, int H, int W, int rows) {
  extern __shared__ __align__(16) uint8_t gsm[];
  cg::cluster_group cluster = cg::this_cluster();
  const int CS = (int)cluster.num_blocks(), rank = (int)cluster.block_rank();
  const int b = blockIdx.x / CS;
  const int cv = p.C >> 3, C = p.C, Ho = H >> 1, Wo = W >> 1;
  const int iy0 = rank * rows, oy0 = iy0 >> 1;           // rows is even
  const int prow = min(rows / 2 + 1, Ho - oy0);          // pooled rows that can route into this slice
  const int n = rows * W * cv, npool = prow * Wo * cv, pcap = (rows / 2 + 1) * Wo * cv;
  uint4* sy = reinterpret_cast<uint4*>(gsm);
  uint4* sdp = sy + n;
  uint2* sarg = reinterpret_cast<uint2*>(sdp + pcap);
  float* part = reinterpret_cast<float*>(sarg + pcap);
  float* tot = part + 2 * C;
  float* wred = tot + 2 * C;
  float* gS = wred + 16 * C;
  const size_t base = ((size_t)b * H + iy0) * W * cv;
  const int tid = threadIdx.x;
  {
    const uint4* gy = reinterpret_cast<const uint4*>(y) + base;
    const size_t pbase = ((size_t)b * Ho + oy0) * Wo * cv;
    const uint4* gd = reinterpret_cast<const uint4*>(dpool) + pbase;
    const uint4* gm = reinterpret_cast<const uint4*>(argmax + pbase * 8);
    const uint32_t ay = smem_u32(sy), ad = smem_u32(sdp), am = smem_u32(sarg);
    for (int i = tid; i < n; i += 256) cp_async16(ay + i * 16, gy + i, true);
    for (int i = tid; i < npool; i += 256) cp_async16(ad + i * 16, gd + i, true);
    for (int i = tid; i < npool / 2; i += 256) cp_async16(am + i * 16, gm + i, true);
    cp_async_commit();
  }
  const int vec = tid % cv, c0 = vec << 3;
  float zc[8], zd[8];
  {
    float mu[8], rs[8], ga[8], be[8];
    gn_coeffs(p, b, c0, mu, rs);
    load8f(p.gamma + c0, ga);
    load8f(p.beta + c0, be);
#pragma unroll
    for (int e = 0; e < 8; ++e) { zc[e] = rs[e] * ga[e]; zd[e] = fmaf(-mu[e], zc[e], be[e]); }
  }
  cp_async_wait<0>();
  __syncthreads();  // staged rows are consumed by other threads than the ones that copied them
  const int nblk = (rows >> 1) * Wo * cv;  // 2x2 input blocks x channel vectors; thread = (block, vec)
  const int wrow = Wo * cv;
  float a[8], bx[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) { a[e] = 0.f; bx[e] = 0.f; }
#define HB_POOL_PIXEL(DY, DX, BODY)                                                    \
  {                                                                                    \
    float gz[8], x[8];                                                                 \
    pool_route_px<DY, DX>(sdp, sarg, o00, wrow, cv, row_ok, col_ok, gz);               \
    const int yi = ((2 * kb + DY) * W + 2 * j + DX) * cv + vec;                        \
    unpack8a(sy[yi], x);                                                                \
    BODY                                                                               \
  }
  for (int it = tid; it < nblk; it += 256) {
    const int pos = it / cv, kb = pos / Wo, j = pos - kb * Wo;
    const int o00 = (kb * Wo + j) * cv + vec;
    const bool row_ok = oy0 + kb + 1 < Ho, col_ok = j + 1 < Wo;
#define HB_BODY1                                                                       \
  _Pragma("unroll") for (int e = 0; e < 8; ++e) {                                      \
    const float gm = fmaf(x[e], zc[e], zd[e]) > 0.f ? gz[e] : 0.f;                     \
    a[e] += gm;                                                                        \
    bx[e] = fmaf(gm, x[e], bx[e]);                                                     \
  }
    HB_POOL_PIXEL(0, 0, HB_BODY1)
    HB_POOL_PIXEL(0, 1, HB_BODY1)
    HB_POOL_PIXEL(1, 0, HB_BODY1)
    HB_POOL_PIXEL(1, 1, HB_BODY1)
#undef HB_BODY1
  }
  float c2[8], c3[8];
  gn_bwd_cluster_sums(cluster, p, b, CS, rank, c0, a, bx, part, tot, wred, gS, dgamma, dbeta, c2, c3);
  uint4* od = reinterpret_cast<uint4*>(dy) + base;
  for (int it = tid; it < nblk; it += 256) {
    const int pos = it / cv, kb = pos / Wo, j = pos - kb * Wo;
    const int o00 = (kb * Wo + j) * cv + vec;
    const bool row_ok = oy0 + kb + 1 < Ho, col_ok = j + 1 < Wo;
#define HB_BODY2                                                                       \
  float o[8];                                                                          \
  _Pragma("unroll") for (int e = 0; e < 8; ++e) {                                      \
    const float gm = fmaf(x[e], zc[e], zd[e]) > 0.f ? gz[e] : 0.f;                     \
    o[e] = fmaf(zc[e], gm, fmaf(x[e], c3[e], c2[e]));                                  \
  }                                                                                    \
  od[yi] = pack8(o);
    HB_POOL_PIXEL(0, 0, HB_BODY2)
    HB_POOL_PIXEL(0, 1, HB_BODY2)
    HB_POOL_PIXEL(1, 0, HB_BODY2)
    HB_POOL_PIXEL(1, 1, HB_BODY2)
#undef HB_BODY2
  }
#undef HB_POOL_PIXEL
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// One block per frame: phase 1 reduces (the frame's dgamma / dbeta partial row + per-group sums kept in shared memory),
// phase 2 re-reads the frame's g / y / act -- which phase 1 just pulled into L2 -- and writes dy (and
// gz).  Compared with gn_bwd_reduce + gn_bwd_apply this removes one full HBM read of every operand, the
// per-(frame,group) atomics and a launch + memset per layer.
__global__ void __launch_bounds__(256)
gn_bwd_fused_kernel(const grad_t* __restrict__ g, const act_t* __restrict__ act,
                    const act_t* __restrict__ y, GnP p, float* __restrict__ dgamma,
                    float* __restrict__ dbeta, grad_t* __restrict__ dy,
                    grad_t* __restrict__ gz_out, int B, int hw, int mask_mode) {
  __shared__ float sa[256][9], sb[256][9];
  extern __shared__ float dyn[];  // [C] gamma*a, [C] gamma*b, [G] S1, [G] S2
  float* ch_a = dyn;
  float* ch_b = dyn + p.C;
  float* gS1 = dyn + 2 * p.C;
  float* gS2 = gS1 + p.G;
  const int cv = p.C >> 3;
  const int b = blockIdx.x;
  const int vec = threadIdx.x % cv, pl = threadIdx.x / cv, npl = blockDim.x / cv;
  const int c0 = vec << 3;
  float mu[8], rs[8], ga[8], be[8], a[8], bb[8];
  gn_coeffs(p, b, c0, mu, rs);
  load8f(p.gamma + c0, ga);
  load8f(p.beta + c0, be);
#pragma unroll
  for (int e = 0; e < 8; ++e) { a[e] = 0.f; bb[e] = 0.f; }
  constexpr int UN = 4;  // pixels in flight per thread: 4 x (2..3) 16-byte loads issued before any use
  for (int pix = pl; pix < hw; pix += UN * npl) {
    uint4 G[UN], Y[UN], A[UN];
#pragma unroll
    for (int u = 0; u < UN; ++u) {
      const int pp = pix + u * npl;
      if (pp < hw) {
        const size_t o = ((size_t)b * hw + pp) * cv + vec;
        G[u] = reinterpret_cast<const uint4*>(g)[o];
        Y[u] = reinterpret_cast<const uint4*>(y)[o];
        if (mask_mode == 2) A[u] = reinterpret_cast<const uint4*>(act)[o];
      }
    }
#pragma unroll
    for (int u = 0; u < UN; ++u) {
      if (pix + u * npl >= hw) continue;
      float gg[8], x[8], z[8], ac[8], gz[8];
      unpack8(G[u], gg);
      unpack8a(Y[u], x);
      if (mask_mode == 2) unpack8a(A[u], ac);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        x[e] = (x[e] - mu[e]) * rs[e];
        z[e] = fmaf(x[e], ga[e], be[e]);
        if (mask_mode != 2) ac[e] = 0.f;
      }
      gn_masked_grad(mask_mode, gg, z, ac, gz);
#pragma unroll
      for (int e = 0; e < 8; ++e) { a[e] += gz[e]; bb[e] = fmaf(gz[e], x[e], bb[e]); }
    }
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) { sa[threadIdx.x][e] = a[e]; sb[threadIdx.x][e] = bb[e]; }
  __syncthreads();
  for (int c = threadIdx.x; c < p.C; c += blockDim.x) {
    const int v = c >> 3, e = c & 7;
    float ta = 0.f, tb = 0.f;
    for (int q = 0; q < npl; ++q) { ta += sa[q * cv + v][e]; tb += sb[q * cv + v][e]; }
    dbeta[(size_t)b * p.C + c] = ta;    // this frame's row of the partials
    dgamma[(size_t)b * p.C + c] = tb;
    const float gm = p.gamma[c];
    ch_a[c] = gm * ta;
    ch_b[c] = gm * tb;
  }
  __syncthreads();
  const int cpg = 1 << p.lcpg;
  for (int gi = threadIdx.x; gi < p.G; gi += blockDim.x) {
    float s1 = 0.f, s2 = 0.f;
    for (int c = gi * cpg; c < (gi + 1) * cpg; ++c) { s1 += ch_a[c]; s2 += ch_b[c]; }
    gS1[gi] = s1;
    gS2[gi] = s2;
  }
  __syncthreads();
  float k1[8], k2[8], k3[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int gi = (c0 + e) >> p.lcpg;
    k1[e] = rs[e] * ga[e];
    k2[e] = rs[e] * p.inv_m * gS1[gi];
    k3[e] = rs[e] * p.inv_m * gS2[gi];
  }
  for (int pix = pl; pix < hw; pix += UN * npl) {
    uint4 G[UN], Y[UN], A[UN];
#pragma unroll
    for (int u = 0; u < UN; ++u) {
      const int pp = pix + u * npl;
      if (pp < hw) {
        const size_t o = ((size_t)b * hw + pp) * cv + vec;
        G[u] = reinterpret_cast<const uint4*>(g)[o];
        Y[u] = reinterpret_cast<const uint4*>(y)[o];
        if (mask_mode == 2) A[u] = reinterpret_cast<const uint4*>(act)[o];
      }
    }
#pragma unroll
    for (int u = 0; u < UN; ++u) {
      const int pp = pix + u * npl;
      if (pp >= hw) continue;
      const size_t o = ((size_t)b * hw + pp) * cv + vec;
      float gg[8], x[8], z[8], ac[8], gz[8], out[8];
      unpack8(G[u], gg);
      unpack8a(Y[u], x);
      if (mask_mode == 2) unpack8a(A[u], ac);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        x[e] = (x[e] - mu[e]) * rs[e];
        z[e] = fmaf(x[e], ga[e], be[e]);
        if (mask_mode != 2) ac[e] = 0.f;
      }
      gn_masked_grad(mask_mode, gg, z, ac, gz);
#pragma unroll
      for (int e = 0; e < 8; ++e) out[e] = fmaf(k1[e], gz[e], -fmaf(x[e], k3[e], k2[e]));
      reinterpret_cast<uint4*>(dy)[o] = pack8(out);
      if (gz_out) reinterpret_cast<uint4*>(gz_out)[o] = pack8(gz);
    }
  }
}

// ---- converts ------------------------------------------------------------------------------
__global__ void bf16_to_f32_kernel(const __nv_bfloat16* __restrict__ x, float* __restrict__ o, long long n8) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n8;
       i += (long long)gridDim.x * blockDim.x) {
    float f[8];
    unpack8(reinterpret_cast<const uint4*>(x)[i], f);
    reinterpret_cast<float4*>(o)[2 * i] = make_float4(f[0], f[1], f[2], f[3]);
    reinterpret_cast<float4*>(o)[2 * i + 1] = make_float4(f[4], f[5], f[6], f[7]);
  }
}
__global__ void f16_to_bf16_kernel(const act_t* __restrict__ x, grad_t* __restrict__ o, long long n8) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n8;
       i += (long long)gridDim.x * blockDim.x) {
    float f[8];
    unpack8a(reinterpret_cast<const uint4*>(x)[i], f);
    reinterpret_cast<uint4*>(o)[i] = pack8(f);
  }
}
__global__ void f32_to_bf16_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ o, long long n8) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n8;
       i += (long long)gridDim.x * blockDim.x) {
    float f[8];
    load8f(x + 8 * i, f);
    reinterpret_cast<uint4*>(o)[i] = pack8(f);
  }
}

// ---- embeddings (HB/rl/ddppo/policy/resnet_policy.py:658-692, 747-761) ------------------
__global__ void embed_fwd_kernel(const float* __restrict__ goal, const int64_t* __restrict__ prev_actions,
                                 const uint8_t* __restrict__ masks, const int32_t* __restrict__ rows,
                                 const float* __restrict__ w_tgt, const float* __restrict__ b_tgt,
                                 const float* __restrict__ emb, float* __restrict__ out, int ld, int col0,
                                 int B) {
  const long long total = (long long)B * 64;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int f = (int)(i >> 6), j = (int)(i & 63);
    const size_t row = (size_t)rows[f];
    float v;
    if (j < 32) {
      const float r = goal[row * 2], th = goal[row * 2 + 1];
      v = b_tgt[j] + w_tgt[j * 3] * r + w_tgt[j * 3 + 1] * cosf(-th) + w_tgt[j * 3 + 2] * sinf(-th);
    } else {
      const int idx = masks[f] ? (int)prev_actions[f] + 1 : 0;
      v = emb[idx * 32 + (j - 32)];
    }
    out[(size_t)f * ld + col0 + j] = v;
  }
}
// One partial per (accumulator, chunk of kEmbedFrames frames), frames summed in order: deterministic.
constexpr int kEmbedFrames = 64;
__global__ void embed_bwd_kernel(const float* __restrict__ goal, const int64_t* __restrict__ prev_actions,
                                 const uint8_t* __restrict__ masks, const int32_t* __restrict__ rows,
                                 const float* __restrict__ d_out, int ld, int col0, int B, int n_emb,
                                 float* __restrict__ parts) {
  // accumulators: [0, 96) target-encoding weight (j, k), [96, 128) its bias, [128, 128 + 32 n_emb) action embedding
  const int nacc = 128 + n_emb * 32;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nacc) return;
  const int f0 = blockIdx.y * kEmbedFrames, f1 = min(B, f0 + kEmbedFrames);
  float v = 0.f;
  if (i < 128) {
    const int j = i < 96 ? i / 3 : i - 96, k = i < 96 ? i % 3 : 3;
    for (int f = f0; f < f1; ++f) {
      const float d = d_out[(size_t)f * ld + col0 + j];
      if (k == 3) { v += d; continue; }
      const size_t row = (size_t)rows[f];
      const float r = goal[row * 2], th = goal[row * 2 + 1];
      v += d * (k == 0 ? r : (k == 1 ? cosf(-th) : sinf(-th)));
    }
  } else {
    const int idx = (i - 128) >> 5, j = (i - 128) & 31;
    for (int f = f0; f < f1; ++f) {
      const int fi = masks[f] ? (int)prev_actions[f] + 1 : 0;
      if (fi == idx) v += d_out[(size_t)f * ld + col0 + 32 + j];
    }
  }
  parts[(size_t)blockIdx.y * nacc + i] = v;
}


// ---- generic 1-D sensors of PointNavResNetNet.forward (resnet_policy.py:658-763) -----------------------------
// feature transforms: 0 identity (gps, pointgoal, proximity, 1-D fuse keys), 1 polar-2D (r, cos(-t), sin(-t)),
// 2 polar-3D (r, cos(-t) sin(p), sin(-t) sin(p), cos(p)), 3 angle -> (cos, sin) (compass, heading)
__device__ __forceinline__ int sensor_features(const float* __restrict__ x, int in_dim, int transform, float (&f)[8]) {
  if (transform == 1) {
    f[0] = x[0]; f[1] = cosf(-x[1]); f[2] = sinf(-x[1]);
    return 3;
  }
  if (transform == 2) {
    const float vs = sinf(x[2]);
    f[0] = x[0]; f[1] = cosf(-x[1]) * vs; f[2] = sinf(-x[1]) * vs; f[3] = cosf(x[2]);
    return 4;
  }
  if (transform == 3) {
    f[0] = cosf(x[0]); f[1] = sinf(x[0]);
    return 2;
  }
  for (int k = 0; k < in_dim && k < 8; ++k) f[k] = x[k];
  return in_dim < 8 ? in_dim : 8;
}
// out[f, col0 + j] = b[j] + sum_k w[j, k] feat_k(x[row_f])   (w == nullptr: the features themselves, j < nfeat)
__global__ void sensor_linear_fwd_kernel(const float* __restrict__ x, int in_dim, const int32_t* __restrict__ rows,
                                         int B, int transform, const float* __restrict__ w, const float* __restrict__ b,
                                         float* __restrict__ out, int ld, int col0, int out_dim) {
  const long long total = (long long)B * out_dim;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int f = (int)(i / out_dim), j = (int)(i - (long long)f * out_dim);
    float ft[8];
    const int nf = sensor_features(x + (size_t)rows[f] * in_dim, in_dim, transform, ft);
    float v;
    if (w == nullptr) {
      v = ft[j];
    } else {
      v = b[j];
      for (int k = 0; k < nf; ++k) v = fmaf(w[j * nf + k], ft[k], v);
    }
    out[(size_t)f * ld + col0 + j] = v;
  }
}
// d_w[j, k] += sum_f d_out[f, col0 + j] feat_k ; d_b[j] += sum_f d_out[f, col0 + j]   (out_dim <= 64, nfeat <= 8)
// Thread i owns accumulator i of [d_w (out_dim x nf) | d_b (out_dim)] and walks the frames of chunk blockIdx.y in
// order; the per-chunk partials are added in order by reduce_partials (like embed_bwd: the same result every run).
__global__ void sensor_linear_bwd_kernel(const float* __restrict__ x, int in_dim, const int32_t* __restrict__ rows,
                                         int B, int transform, const float* __restrict__ d_out, int ld, int col0,
                                         int out_dim, int nf, float* __restrict__ parts) {
  const int nacc = out_dim * (nf + 1);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nacc) return;
  const bool bias = i >= out_dim * nf;
  const int j = bias ? i - out_dim * nf : i / nf, k = bias ? 0 : i - j * nf;
  const int f0 = blockIdx.y * kEmbedFrames, f1 = min(B, f0 + kEmbedFrames);
  float v = 0.f;
  for (int f = f0; f < f1; ++f) {
    const float d = d_out[(size_t)f * ld + col0 + j];
    if (bias) { v += d; continue; }
    float ft[8];
    sensor_features(x + (size_t)rows[f] * in_dim, in_dim, transform, ft);
    v = fmaf(d, ft[k], v);
  }
  parts[(size_t)blockIdx.y * nacc + i] = v;
}
// out[f, col0 + j] = table[index_f, j]; index from an int64 tensor through rows (objectgoal) or, with masks,
// masks[f] ? idx[f] + 1 : 0 (the previous-action embedding with its "start" token, resnet_policy.py:747-757)
__global__ void index_embed_fwd_kernel(const int64_t* __restrict__ idx, const int32_t* __restrict__ rows,
                                       const uint8_t* __restrict__ masks, int B, int n_rows_table,
                                       const float* __restrict__ table, int width, float* __restrict__ out, int ld,
                                       int col0) {
  const long long total = (long long)B * width;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int f = (int)(i / width), j = (int)(i - (long long)f * width);
    long long k = idx[rows ? (size_t)rows[f] : (size_t)f];
    if (masks) k = masks[f] ? k + 1 : 0;
    // an index outside the table has no embedding (torch device-asserts): poison the row
    out[(size_t)f * ld + col0 + j] = (k >= 0 && k < n_rows_table) ? table[k * width + j] : __int_as_float(0x7fc00000);
  }
}
// Thread i owns d_table element i (row i / width) and adds the frames of chunk blockIdx.y that index its row, in
// frame order; the per-chunk partials are added in order by reduce_partials.  Out-of-range indices add nothing.
__global__ void index_embed_bwd_kernel(const int64_t* __restrict__ idx, const int32_t* __restrict__ rows,
                                       const uint8_t* __restrict__ masks, int B, int n_rows_table, int width,
                                       const float* __restrict__ d_out, int ld, int col0, float* __restrict__ parts) {
  const long long nacc = (long long)n_rows_table * width;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= nacc) return;
  const long long row = i / width;
  const int j = (int)(i - row * width);
  const int f0 = blockIdx.y * kEmbedFrames, f1 = min(B, f0 + kEmbedFrames);
  float v = 0.f;
  for (int f = f0; f < f1; ++f) {
    long long k = idx[rows ? (size_t)rows[f] : (size_t)f];
    if (masks) k = masks[f] ? k + 1 : 0;
    if (k == row) v += d_out[(size_t)f * ld + col0 + j];
  }
  parts[(size_t)blockIdx.y * nacc + i] = v;
}

// Continuous previous action (resnet_policy.py:755-757): nn.Linear(A, 32) of masks * prev_actions.float().  The mask is
// a multiplication, as the reference's, so a NaN / inf previous action of a masked frame still gives NaN.
__global__ void prev_action_linear_fwd_kernel(const float* __restrict__ pa, const uint8_t* __restrict__ masks, int B,
                                              int A, const float* __restrict__ w, const float* __restrict__ b,
                                              float* __restrict__ out, int ld, int col0) {
  const long long total = (long long)B * 32;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int f = (int)(i >> 5), j = (int)(i & 31);
    const float m = masks[f] ? 1.f : 0.f;
    float v = b[j];
    for (int k = 0; k < A; ++k) v = fmaf(w[j * A + k], m * pa[(size_t)f * A + k], v);
    out[(size_t)f * ld + col0 + j] = v;
  }
}
// Thread i owns accumulator i of [d_w (32 x A) | d_b (32)] and walks the frames of chunk blockIdx.y in order; the
// per-chunk partials are added in order by reduce_partials.
__global__ void prev_action_linear_bwd_kernel(const float* __restrict__ pa, const uint8_t* __restrict__ masks, int B,
                                              int A, const float* __restrict__ d_out, int ld, int col0,
                                              float* __restrict__ parts) {
  const int nacc = 32 * (A + 1);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nacc) return;
  const bool bias = i >= 32 * A;
  const int j = bias ? i - 32 * A : i / A, k = bias ? 0 : i - j * A;
  const int f0 = blockIdx.y * kEmbedFrames, f1 = min(B, f0 + kEmbedFrames);
  float v = 0.f;
  for (int f = f0; f < f1; ++f) {
    const float d = d_out[(size_t)f * ld + col0 + j];
    if (bias) { v += d; continue; }
    v = fmaf(d, (masks[f] ? 1.f : 0.f) * pa[(size_t)f * A + k], v);
  }
  parts[(size_t)blockIdx.y * nacc + i] = v;
}

// ---- generic visual input prep: any mix of u8 / f32 / i32 HWC sensors, any H x W ----------------------------------
// (ResNetEncoder.forward, resnet_policy.py:255-271: per-key permute, u8 keys scaled by 1 / high, channel concat,
// avg_pool2d(2) -- the odd last row / column is dropped -- then RunningMeanAndVar.)  One thread per pooled pixel;
// the fast rgb-u8 + depth-f32 kernels above stay the path for the PointNav sensor set.
constexpr int kPrepMaxSrcs = 8;   // one channel each at most: the stem takes 8 input channels
struct PrepSrcs {
  const void* ptr[kPrepMaxSrcs];
  int dtype[kPrepMaxSrcs];     // 0 u8, 1 f32, 2 i32
  int channels[kPrepMaxSrcs];
  float scale[kPrepMaxSrcs];   // multiplied BEFORE pooling (u8: 1 / high)
  int n;
};
__device__ __forceinline__ float prep_load(const void* p, int dtype, size_t i) {
  if (dtype == 0) return (float)reinterpret_cast<const uint8_t*>(p)[i];
  if (dtype == 1) return reinterpret_cast<const float*>(p)[i];
  return (float)reinterpret_cast<const int32_t*>(p)[i];
}
template <bool STATS>
__global__ void __launch_bounds__(256)
prep_generic_kernel(PrepSrcs src, const int32_t* __restrict__ frame_rows, int B, int H, int W,
                    const float* __restrict__ scale_shift, act_t* __restrict__ out, grad_t* __restrict__ out2,
                    double* __restrict__ stats) {
  __shared__ double red[32];
  const int Hp = H / 2, Wp = W / 2;
  const long long total = (long long)B * Hp * Wp;
  float s[8] = {0, 0, 0, 0, 0, 0, 0, 0}, q[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int px = (int)(i % Wp);
    const long long t = i / Wp;
    const int py = (int)(t % Hp), f = (int)(t / Hp);
    const size_t row = (size_t)frame_rows[f];
    float v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    int c0 = 0;
    for (int k = 0; k < src.n; ++k) {
      const int C = src.channels[k];
      const size_t base = ((row * H + 2 * py) * (size_t)W + 2 * px) * C;
      for (int c = 0; c < C; ++c) {
        // avg_pool2d sums the window row-major then divides (ATen); scaled keys are scaled first
        float a = __fmul_rn(prep_load(src.ptr[k], src.dtype[k], base + c), src.scale[k]);
        a = __fadd_rn(a, __fmul_rn(prep_load(src.ptr[k], src.dtype[k], base + C + c), src.scale[k]));
        a = __fadd_rn(a, __fmul_rn(prep_load(src.ptr[k], src.dtype[k], base + (size_t)W * C + c), src.scale[k]));
        a = __fadd_rn(a, __fmul_rn(prep_load(src.ptr[k], src.dtype[k], base + (size_t)W * C + C + c), src.scale[k]));
        v[c0 + c] = a * 0.25f;
      }
      c0 += C;
    }
    if (STATS) {
#pragma unroll
      for (int c = 0; c < 8; ++c) { s[c] += v[c]; q[c] = fmaf(v[c], v[c], q[c]); }
    } else {
      float o[8];
#pragma unroll
      for (int c = 0; c < 8; ++c) o[c] = (c < c0) ? (scale_shift ? fmaf(v[c], scale_shift[c], scale_shift[8 + c]) : v[c]) : 0.f;
      reinterpret_cast<uint4*>(out)[i] = pack8a(o);
      if (out2) reinterpret_cast<uint4*>(out2)[i] = pack8(o);
    }
  }
  if (STATS) {
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const double a = block_sum((double)s[c], red);
      const double b = block_sum((double)q[c], red);
      if (threadIdx.x == 0) { atomicAdd(&stats[c], a); atomicAdd(&stats[8 + c], b); }
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) stats[16] = (double)B;
  }
}

// mask / shift helpers for the recurrent encoder
__global__ void rnn_shift_mask_kernel(const float* __restrict__ h_seq, const float* __restrict__ h0,
                                      long long h0_stride, const uint8_t* __restrict__ masks,
                                      float* __restrict__ h_in, int T, int n, int H) {
  const long long total = (long long)T * n * H;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(i % H);
    const long long tn = i / H;
    const int s = (int)(tn % n);
    const int t = (int)(tn / n);
    const float prev = (t == 0) ? h0[(size_t)s * h0_stride + k] : h_seq[i - (long long)n * H];
    h_in[i] = masks[tn] ? prev : 0.f;
  }
}
__global__ void __launch_bounds__(1024) colsum_kernel(const float* __restrict__ x, long long ld, float* __restrict__ out,
                                                      long long M, int N, int accumulate) {
  // block handles 32 columns; 32 x 32 threads stride the rows, 4 independent loads in flight per thread (the 8-row-group
  // version walked 512 dependent loads per thread); fixed summation order
  __shared__ float red[32][33];
  const int col = blockIdx.x * 32 + (threadIdx.x & 31), ry = threadIdx.x >> 5;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  if (col < N) {
    long long r = ry;
    for (; r + 96 < M; r += 128) {
      a0 += x[r * ld + col];
      a1 += x[(r + 32) * ld + col];
      a2 += x[(r + 64) * ld + col];
      a3 += x[(r + 96) * ld + col];
    }
    for (; r < M; r += 32) a0 += x[r * ld + col];
  }
  red[ry][threadIdx.x & 31] = (a0 + a1) + (a2 + a3);
  __syncthreads();
  if (ry == 0 && col < N) {
    float s = 0.f;
    for (int q = 0; q < 32; ++q) s += red[q][threadIdx.x & 31];
    out[col] = accumulate ? out[col] + s : s;
  }
}

// d[r, c] *= (y[r, c] > 0) for c < cols (ReLU backward on a column block of a wider matrix)
__global__ void relu_bwd_kernel(float* __restrict__ d, const float* __restrict__ y, long long ld_d,
                                long long ld_y, long long rows, int cols) {
  const long long total = rows * cols;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / cols;
    const int c = (int)(i - r * cols);
    if (!(y[r * ld_y + c] > 0.f)) d[r * ld_d + c] = 0.f;
  }
}
// x f32 [B, C*hw] in (c, h, w) order  ->  bf16 NHWC [B, hw, C]
__global__ void f32_chw_to_bf16_hwc_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ out,
                                           int B, int hw, int C) {
  const int cv = C >> 3;
  const long long total = (long long)B * hw * cv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c0 = (int)(i % cv) << 3;
    const long long t = i / cv;
    const int p = (int)(t % hw);
    const int b = (int)(t / hw);
    float f[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) f[e] = x[((size_t)b * C + c0 + e) * hw + p];
    reinterpret_cast<uint4*>(out)[i] = pack8(f);
  }
}
// logits/value heads only (actor path): logits [B,A], values [B]
__global__ void heads_fwd_kernel(const float* __restrict__ feat, const float* __restrict__ w_act,
                                 const float* __restrict__ b_act, const float* __restrict__ w_val,
                                 const float* __restrict__ b_val, int B, int H, int A,
                                 float* __restrict__ logits, float* __restrict__ values) {
  const int lane = threadIdx.x & 31;
  const int f = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (f >= B) return;
  for (int a = 0; a <= A; ++a) {
    const float* w = (a < A) ? w_act + (size_t)a * H : w_val;
    float acc = 0.f;
    for (int k = lane; k < H; k += 32) acc = fmaf(feat[(size_t)f * H + k], w[k], acc);
    acc = warp_sum(acc);
    if (lane == 0) {
      if (a < A) logits[(size_t)f * A + a] = acc + b_act[a];
      else values[f] = acc + b_val[0];
    }
  }
}

// actor step in one launch: both heads, log-softmax, and either the mode (uniform == nullptr) or an inverse-CDF draw
// from the caller's uniform [0,1) numbers: action = first index whose cumulative probability exceeds u.
// One warp per frame; lane 0 finishes the (tiny) per-action arithmetic.
__global__ void heads_act_kernel(const float* __restrict__ feat, const float* __restrict__ w_act,
                                 const float* __restrict__ b_act, const float* __restrict__ w_val,
                                 const float* __restrict__ b_val, const float* __restrict__ uniform, int B, int H, int A,
                                 float* __restrict__ logp, float* __restrict__ values, long long* __restrict__ actions,
                                 float* __restrict__ action_logp) {
  const int lane = threadIdx.x & 31;
  const int f = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (f >= B) return;
  float* lp = logp + (size_t)f * A;
  float mx = -INFINITY;
  // 8 output rows (actions, then the value head) per pass: 8 independent load streams per lane instead of one
  // dependent dot product after the other (this kernel is pure latency: 64 frames x 5 rows x 2 KB)
  for (int a0 = 0; a0 <= A; a0 += 8) {
    const float* w[8];
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int a = a0 + j;
      w[j] = (a < A) ? w_act + (size_t)a * H : w_val;   // rows past the value head re-read it (discarded)
      acc[j] = 0.f;
    }
#pragma unroll 4
    for (int k = lane; k < H; k += 32) {
      const float x = feat[(size_t)f * H + k];
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = fmaf(x, w[j][k], acc[j]);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float v = warp_sum(acc[j]);
      const int a = a0 + j;
      if (lane == 0 && a <= A) {
        if (a < A) {
          const float l = v + b_act[a];
          lp[a] = l;
          mx = fmaxf(mx, l);
        } else {
          values[f] = v + b_val[0];
        }
      }
    }
  }
  if (lane != 0) return;
  float se = 0.f;
  for (int a = 0; a < A; ++a) se += __expf(lp[a] - mx);
  const float lse = mx + __logf(se);
  int pick = 0;
  if (uniform) {
    const float u = uniform[f];
    float cum = 0.f;
    pick = -1;
    int last = 0;
    for (int a = 0; a < A; ++a) {
      const float l = lp[a] - lse;
      lp[a] = l;
      const float p = __expf(l);
      if (p > 0.f) last = a;
      cum += p;
      if (pick < 0 && u < cum) pick = a;
    }
    if (pick < 0) pick = last;   // u beyond the rounded total: the last action with non-zero probability
  } else {
    float best = -INFINITY;
    for (int a = 0; a < A; ++a) {
      const float l = lp[a] - lse;
      lp[a] = l;
      if (l > best) { best = l; pick = a; }   // first maximum, like argmax
    }
  }
  actions[f] = pick;
  action_logp[f] = lp[pick];
}

// block = (frame, slab of ppb pixels); 256 threads = (C/8 vectors) x (pixel lanes)
static int gn_slab_launch(int C, int hw, int B, int* ppb, int* grid) {
  const int cv = C / 8;
  HB_CHECK_ARG(cv >= 1 && cv <= 256 && 256 % cv == 0, "gn: C/8 = %d must divide 256", cv);
  const int npl = 256 / cv;
  int p = npl * 8;  // ~8 pixels per thread
  if (p > hw) p = hw;
  *ppb = p;
  *grid = B * ((hw + p - 1) / p);
  return HB200_OK;
}

// dst[c, r] = src[r, c]  (32x32 tiles through padded shared memory; both sides coalesced)
__global__ void transpose_f32_kernel(const float* __restrict__ src, long long ld_src, float* __restrict__ dst,
                                     long long ld_dst, int rows, int cols) {
  __shared__ float tile[32][33];
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  for (int i = ty; i < 32; i += 8) {
    const int r = r0 + i, c = c0 + tx;
    tile[i][tx] = (r < rows && c < cols) ? src[(long long)r * ld_src + c] : 0.f;
  }
  __syncthreads();
  for (int i = ty; i < 32; i += 8) {
    const int c = c0 + i, r = r0 + tx;
    if (c < cols && r < rows) dst[(long long)c * ld_dst + r] = tile[tx][i];
  }
}

// SimpleCNN input: rgb/255 and raw depth concatenated, NHWC bf16 padded to 8 channels, no pooling
// (simple_cnn.py:139-157).  One thread per pixel.
__global__ void prep_plain_kernel(const uint8_t* __restrict__ rgb, const float* __restrict__ depth,
                                  const int32_t* __restrict__ rows, long long npix_per_frame, int B, int c_rgb,
                                  int c_depth, act_t* __restrict__ out) {
  const long long total = (long long)B * npix_per_frame;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int f = (int)(i / npix_per_frame);
    const long long p = i - (long long)f * npix_per_frame;
    const size_t src = (size_t)rows[f] * npix_per_frame + p;
    float v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int c = 0; c < c_rgb; ++c) v[c] = (float)rgb[src * c_rgb + c] / 255.0f;
    for (int c = 0; c < c_depth; ++c) v[c_rgb + c] = depth[src * c_depth + c];
    reinterpret_cast<uint4*>(out)[i] = pack8a(v);
  }
}
// backward of (conv + bias) -> ReLU: dy = g * (out > 0); dbias[c] += sum dy   (out = post-ReLU activation)
// Each block writes its per-channel partial to parts[blockIdx.x][C]; reduce_partials adds them in block order.
__global__ void __launch_bounds__(256)
relu_bias_bwd_kernel(const grad_t* __restrict__ g, const act_t* __restrict__ out, int use_mask,
                     grad_t* __restrict__ dy, float* __restrict__ parts, long long npix, int C) {
  __shared__ float sacc[256][9];
  const int cv = C >> 3;
  const int vec = threadIdx.x % cv, pl = threadIdx.x / cv, npl = blockDim.x / cv;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (long long pix = (long long)blockIdx.x * npl + pl; pix < npix; pix += (long long)gridDim.x * npl) {
    const size_t o = (size_t)pix * cv + vec;
    float gg[8], oo[8];
    unpack8(reinterpret_cast<const uint4*>(g)[o], gg);
    if (use_mask) {
      unpack8a(reinterpret_cast<const uint4*>(out)[o], oo);
#pragma unroll
      for (int e = 0; e < 8; ++e) gg[e] = oo[e] > 0.f ? gg[e] : 0.f;
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] += gg[e];
    if (dy) reinterpret_cast<uint4*>(dy)[o] = pack8(gg);
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) sacc[threadIdx.x][e] = acc[e];
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float t = 0.f;
    for (int q = 0; q < npl; ++q) t += sacc[q * cv + (c >> 3)][c & 7];
    parts[(size_t)blockIdx.x * C + c] = t;
  }
}
// bf16 NHWC [B,hw,C] -> f32 [B, C*hw] flattened in (c,h,w) order (nn.Flatten of the NCHW map)
__global__ void bf16_hwc_to_f32_chw_kernel(const act_t* __restrict__ x, float* __restrict__ out, int B,
                                           int hw, int C) {
  const int cv = C >> 3;
  const long long total = (long long)B * hw * cv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int c0 = (int)(i % cv) << 3;
    const long long t = i / cv;
    const int p = (int)(t % hw);
    const int b = (int)(t / hw);
    float f[8];
    unpack8a(reinterpret_cast<const uint4*>(x)[i], f);
#pragma unroll
    for (int e = 0; e < 8; ++e) out[((size_t)b * C + c0 + e) * hw + p] = f[e];
  }
}

static int ilog2i(int v) {
  int l = 0;
  while ((1 << l) < v) ++l;
  return l;
}
static int make_gn(GnP& p, const double* stats, const float* gamma, const float* beta, int C, int G, int hw,
                   float eps) {
  HB_CHECK_ARG(stats && gamma && beta, "gn: null pointer");
  HB_CHECK_ARG(C % 8 == 0 && G > 0 && C % G == 0, "gn: C=%d G=%d unsupported", C, G);
  const int cpg = C / G;
  HB_CHECK_ARG((cpg & (cpg - 1)) == 0, "gn: channels per group (%d) must be a power of two", cpg);
  p.stats = stats; p.gamma = gamma; p.beta = beta; p.C = C; p.G = G; p.lcpg = ilog2i(cpg);
  p.inv_m = 1.0f / ((float)cpg * (float)hw);
  p.eps = eps;
  return HB200_OK;
}
// ---- deterministic reduction of block partials (common.cuh) ----------------------------------------------------
__global__ void reduce_partials_chunk_kernel(const float* __restrict__ parts, int nparts, long long ld, long long count,
                                             int per, float* __restrict__ tmp) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= count) return;
  const int p0 = blockIdx.y * per, p1 = min(nparts, p0 + per);
  float s = 0.f;
  for (int p = p0; p < p1; ++p) s += parts[(size_t)p * ld + i];
  tmp[(size_t)blockIdx.y * count + i] = s;
}
__global__ void reduce_partials_final_kernel(const float* __restrict__ tmp, int nchunks, long long count,
                                             float* __restrict__ dst) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= count) return;
  float s = 0.f;
  for (int k = 0; k < nchunks; ++k) s += tmp[(size_t)k * count + i];
  dst[i] += s;
}
int reduce_partials(const float* parts, int nparts, long long ld, long long count, float* dst, float* tmp,
                    cudaStream_t st) {
  if (nparts <= 0 || count <= 0) return HB200_OK;
  const int per = cdiv(nparts, kReduceChunks), nchunks = cdiv(nparts, per);
  const unsigned gx = (unsigned)cdiv(count, 256);
  reduce_partials_chunk_kernel<<<dim3(gx, nchunks), 256, 0, st>>>(parts, nparts, ld, count, per, tmp);
  reduce_partials_final_kernel<<<gx, 256, 0, st>>>(tmp, nchunks, count, dst);
  HB_LAUNCH_OK();
  count_launch(2);
  return HB200_OK;
}

// GroupNorm backward: per-frame rows of the dgamma / dbeta partials [B][C] + the reduction's scratch
static int gn_affine_grads_workspace(cudaStream_t st, int B, int C, float** part_g, float** part_b) {
  float* ws = nullptr;
  int* tickets = nullptr;
  const int rc = stream_workspace(st, (size_t)2 * B * C + (size_t)kReduceChunks * C, 0, &ws, &tickets);
  if (rc) return rc;
  *part_b = ws;
  *part_g = ws + (size_t)B * C;
  return HB200_OK;
}
static int gn_affine_grads_reduce(const float* part_g, const float* part_b, int B, int C, float* dgamma, float* dbeta,
                                  cudaStream_t st) {
  float* tmp = const_cast<float*>(part_b) + (size_t)2 * B * C;
  const int rc = reduce_partials(part_b, B, C, C, dbeta, tmp, st);
  if (rc) return rc;
  return reduce_partials(part_g, B, C, C, dgamma, tmp, st);
}

// ---- squeeze-excite block output (SEBottleneck, resnet.py:92-110, 155-180) ------------------------------------------
//   z = GN(y),  p = mean_hw(z),  h = relu(W1 p + b1),  s = sigmoid(W2 h + b2),  o = relu(s * z + r)
// p needs only per-channel sums of y: p = zc * mean_hw(y) + zd with zc = rstd * gamma, zd = beta - mu * zc.  In the
// backward, with gz = g * [o > 0], every per-frame quantity follows from three per-channel sums (sum gz, sum gz*y,
// sum y): ds = zc * sum(gz*y) + zd * sum(gz), a = ds * s * (1 - s), dh = (W2^T a) * [h > 0], dp = W1^T dh, and the
// GroupNorm backward runs on dz = s * gz + dp / hw, whose sums are s * sum(gz) + dp and s * sum(gz*y) + dp/hw * sum(y).
// One thread-block cluster owns a frame, like gn_bwd_cluster_kernel: each CTA stages its pixel slice in shared memory
// (slices too large to stage are re-read from global memory), the channel sums go threads -> CTA -> cluster ranks in a
// fixed order, and every CTA evaluates the excitation on the same totals in the same order, so all hold the same s.
struct SeP {
  const float *w1, *b1, *w2, *b2;  // excite.0 weight [cr, C], bias [cr]; excite.2 weight [C, cr], bias [C]
  const float *s_in, *h_in;        // backward: the forward's s [B, C] and h [B, cr]
  float *p, *h, *s;                // forward: squeeze [B, C], hidden [B, cr], scale [B, C]
  float *a, *dh;                   // backward: a = ds * s * (1 - s) [B, C], dh [B, cr]
  int cr;
};

// mean / rstd of channel c of frame b (the arithmetic of gn_coeffs)
__device__ __forceinline__ void gn_chan(const GnP& p, int b, int c, float& mu, float& rs) {
  const double2 st = *reinterpret_cast<const double2*>(p.stats + ((size_t)b * p.G + (c >> p.lcpg)) * 2);
  const double md = st.x * (double)p.inv_m;
  mu = (float)md;
  rs = rsqrtf(fmaxf((float)(st.y * (double)p.inv_m - md * md), 0.f) + p.eps);
}

// dst[c] = sum of v over the CTA's pixel lanes (thread = (vec = tid % cv, lane = tid / cv)), added in lane order
__device__ __forceinline__ void se_cta_chan_sum(const float (&v)[8], float (*sred)[9], float* dst, int C) {
  const int cv = C >> 3, npl = 256 / cv;
#pragma unroll
  for (int e = 0; e < 8; ++e) sred[threadIdx.x][e] = v[e];
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += 256) {
    float t = 0.f;
    for (int q = 0; q < npl; ++q) t += sred[q * cv + (c >> 3)][c & 7];
    dst[c] = t;
  }
  __syncthreads();
}

// tot[i] = sum over the cluster's CTAs, in rank order, of their part[i] (i < n).  Ends with a cluster barrier ARRIVE;
// the caller executes the matching WAIT before it exits, so no CTA leaves while a peer still reads its part.
__device__ __forceinline__ void se_cluster_total(cg::cluster_group& cluster, const float* part, float* tot, int n,
                                                 int CS) {
  cluster.sync();
  for (int i = threadIdx.x; i < n; i += 256) {
    float t = 0.f;
    for (int r = 0; r < CS; ++r) t += cluster.map_shared_rank(part, r)[i];
    tot[i] = t;
  }
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  __syncthreads();
}

__global__ void __launch_bounds__(256)
gn_se_residual_relu_kernel(const act_t* __restrict__ y, GnP p, const act_t* __restrict__ res, GnP rp,
                           int res_is_prenorm, SeP se, act_t* __restrict__ out, grad_t* __restrict__ out2, int hw,
                           int ppc, int staged) {
  extern __shared__ __align__(16) uint8_t gsm[];
  __shared__ float sred[256][9];
  cg::cluster_group cluster = cg::this_cluster();
  const int CS = (int)cluster.num_blocks(), rank = (int)cluster.block_rank();
  const int b = blockIdx.x / CS;
  const int C = p.C, cv = C >> 3, cr = se.cr, tid = threadIdx.x;
  const int pix0 = rank * ppc, pix1 = min(hw, pix0 + ppc);
  const int n = max(pix1 - pix0, 0) * cv;
  const size_t base = ((size_t)b * hw + pix0) * cv;
  const uint4* gy = reinterpret_cast<const uint4*>(y) + base;
  uint4* sy = reinterpret_cast<uint4*>(gsm);
  float* part = reinterpret_cast<float*>(gsm + (staged ? (size_t)ppc * C * 2 : 0));  // [C] this CTA's sums of y
  float* tot = part + C;                                                                // [C] the frame's sums
  float* pv = tot + C;                                                                  // [C] squeeze
  float* sv = pv + C;                                                                   // [C] scale
  float* hv = sv + C;                                                                   // [cr] hidden
  if (staged) {   // every thread later consumes exactly the vectors it copied: no block barrier before use
    const uint32_t ay = smem_u32(sy);
    for (int i = tid; i < n; i += 256) cp_async16(ay + i * 16, gy + i, true);
    cp_async_commit();
  }
  const uint4* src = staged ? sy : gy;
  const int vec = tid % cv, c0 = vec << 3;
  float zc[8], zd[8], rsc[8], rsh[8];
  {
    float mu[8], rs[8], ga[8], be[8];
    gn_coeffs(p, b, c0, mu, rs);
    load8f(p.gamma + c0, ga);
    load8f(p.beta + c0, be);
#pragma unroll
    for (int e = 0; e < 8; ++e) { zc[e] = rs[e] * ga[e]; zd[e] = fmaf(-mu[e], zc[e], be[e]); rsc[e] = 1.f; rsh[e] = 0.f; }
    if (res_is_prenorm) {
      gn_coeffs(rp, b, c0, mu, rs);
      load8f(rp.gamma + c0, ga);
      load8f(rp.beta + c0, be);
#pragma unroll
      for (int e = 0; e < 8; ++e) { rsc[e] = rs[e] * ga[e]; rsh[e] = fmaf(-mu[e], rsc[e], be[e]); }
    }
  }
  if (staged) cp_async_wait<0>();
  float acc[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) acc[e] = 0.f;
  for (int i = tid; i < n; i += 256) {
    float x[8];
    unpack8a(src[i], x);
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[e] += x[e];
  }
  se_cta_chan_sum(acc, sred, part, C);
  se_cluster_total(cluster, part, tot, C, CS);
  const float inv_hw = 1.f / (float)hw;
  for (int c = tid; c < C; c += 256) {
    float mu, rs;
    gn_chan(p, b, c, mu, rs);
    const float k = rs * p.gamma[c];
    pv[c] = fmaf(tot[c] * inv_hw, k, fmaf(-mu, k, p.beta[c]));
  }
  __syncthreads();
  // excite.0 + ReLU: one warp per hidden unit, lanes stride over C, fixed shuffle tree
  const int lane = tid & 31, warp = tid >> 5;
  for (int j = warp; j < cr; j += 8) {
    const float* w = se.w1 + (size_t)j * C;
    float t = 0.f;
    for (int c = lane; c < C; c += 32) t = fmaf(__ldg(w + c), pv[c], t);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    if (lane == 0) hv[j] = fmaxf(t + __ldg(se.b1 + j), 0.f);
  }
  __syncthreads();
  // excite.2 + sigmoid: one thread per channel, its weight row in order
  for (int c = tid; c < C; c += 256) {
    const float4* w = reinterpret_cast<const float4*>(se.w2 + (size_t)c * cr);
    float t = __ldg(se.b2 + c);
    for (int j = 0; j < cr; j += 4) {
      const float4 wv = __ldg(w + (j >> 2));
      t = fmaf(wv.x, hv[j], t);
      t = fmaf(wv.y, hv[j + 1], t);
      t = fmaf(wv.z, hv[j + 2], t);
      t = fmaf(wv.w, hv[j + 3], t);
    }
    sv[c] = 1.f / (1.f + expf(-t));
  }
  __syncthreads();
  if (rank == 0) {
    for (int c = tid; c < C; c += 256) {
      se.p[(size_t)b * C + c] = pv[c];
      se.s[(size_t)b * C + c] = sv[c];
    }
    for (int j = tid; j < cr; j += 256) se.h[(size_t)b * cr + j] = hv[j];
  }
  float sc[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) sc[e] = sv[c0 + e];
  const uint4* gr = reinterpret_cast<const uint4*>(res) + base;
  uint4* go = reinterpret_cast<uint4*>(out) + base;
  uint4* go2 = out2 ? reinterpret_cast<uint4*>(out2) + base : nullptr;
  for (int i = tid; i < n; i += 256) {
    float x[8], r[8];
    unpack8a(src[i], x);
    unpack8a(gr[i], r);
#pragma unroll
    for (int e = 0; e < 8; ++e) x[e] = fmaxf(fmaf(sc[e], fmaf(x[e], zc[e], zd[e]), fmaf(r[e], rsc[e], rsh[e])), 0.f);
    go[i] = pack8a(x);
    if (go2) go2[i] = pack8(x);
  }
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// Backward of gn_se_residual_relu_kernel's main branch: dy (grad wrt y), gz_out = g * [o > 0] (the residual branch's
// gradient), the frame's row of the dgamma / dbeta partials [B][C], and the excitation's a [B,C] / dh [B,cr] from which
// the caller forms the excitation weight gradients.
__global__ void __launch_bounds__(256)
gn_se_bwd_kernel(const grad_t* __restrict__ g, const act_t* __restrict__ act, const act_t* __restrict__ y, GnP p,
                 SeP se, float* __restrict__ dgamma, float* __restrict__ dbeta, grad_t* __restrict__ dy,
                 grad_t* __restrict__ gz_out, int hw, int ppc, int staged) {
  extern __shared__ __align__(16) uint8_t gsm[];
  __shared__ float sred[256][9];
  cg::cluster_group cluster = cg::this_cluster();
  const int CS = (int)cluster.num_blocks(), rank = (int)cluster.block_rank();
  const int b = blockIdx.x / CS;
  const int C = p.C, G = p.G, cv = C >> 3, cr = se.cr, tid = threadIdx.x;
  const int pix0 = rank * ppc, pix1 = min(hw, pix0 + ppc);
  const int n = max(pix1 - pix0, 0) * cv, ncap = staged ? ppc * cv : 0;
  const size_t base = ((size_t)b * hw + pix0) * cv;
  const uint4* gg = reinterpret_cast<const uint4*>(g) + base;
  const uint4* gy = reinterpret_cast<const uint4*>(y) + base;
  const uint4* ga = reinterpret_cast<const uint4*>(act) + base;
  uint4* sg = reinterpret_cast<uint4*>(gsm);
  uint4* sy = sg + ncap;
  uint4* sa = sy + ncap;
  float* part = reinterpret_cast<float*>(sa + ncap);  // [3C] this CTA's sum gz, sum gz*y, sum y
  float* tot = part + 3 * C;                           // [3C] the frame's
  float* av = tot + 3 * C;                             // [C] a
  float* dpv = av + C;                                 // [C] dp / hw
  float* t1 = dpv + C;                                 // [C] sum dz
  float* t2 = t1 + C;                                  // [C] sum dz * xhat
  float* red = t2 + C;                                 // [256] partial dot products of dh
  float* dhv = red + 256;                              // [cr]
  float* gS = dhv + cr;                                // [2G]
  if (staged) {
    const uint32_t ag = smem_u32(sg), ay = smem_u32(sy), aa = smem_u32(sa);
    for (int i = tid; i < n; i += 256) {
      cp_async16(ag + i * 16, gg + i, true);
      cp_async16(ay + i * 16, gy + i, true);
      cp_async16(aa + i * 16, ga + i, true);
    }
    cp_async_commit();
  }
  const uint4 *srg = staged ? sg : gg, *sry = staged ? sy : gy, *sra = staged ? sa : ga;
  const int vec = tid % cv, c0 = vec << 3;
  if (staged) cp_async_wait<0>();
  {
    float s1[8], s2[8], s3[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) { s1[e] = 0.f; s2[e] = 0.f; s3[e] = 0.f; }
    for (int i = tid; i < n; i += 256) {
      float gv[8], x[8], ac[8];
      unpack8(srg[i], gv);
      unpack8a(sry[i], x);
      unpack8a(sra[i], ac);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float gz = ac[e] > 0.f ? gv[e] : 0.f;
        s1[e] += gz;
        s2[e] = fmaf(gz, x[e], s2[e]);
        s3[e] += x[e];
      }
    }
    se_cta_chan_sum(s1, sred, part, C);
    se_cta_chan_sum(s2, sred, part + C, C);
    se_cta_chan_sum(s3, sred, part + 2 * C, C);
  }
  se_cluster_total(cluster, part, tot, 3 * C, CS);
  const float* sf = se.s_in + (size_t)b * C;
  for (int c = tid; c < C; c += 256) {
    float mu, rs;
    gn_chan(p, b, c, mu, rs);
    const float k = rs * p.gamma[c], kd = fmaf(-mu, k, p.beta[c]);
    const float ds = fmaf(k, tot[C + c], kd * tot[c]);   // sum_hw gz * z
    const float s = sf[c];
    const float a = ds * s * (1.f - s);
    av[c] = a;
    if (rank == 0) se.a[(size_t)b * C + c] = a;
  }
  __syncthreads();
  // dh = (W2^T a) * [h > 0]: thread (j, q) walks the q-th contiguous range of channels; ranges are added in order
  {
    const int j = tid % cr, q = tid / cr, per = C / (256 / cr);
    const float* w = se.w2 + j;
    float t = 0.f;
    for (int c = q * per; c < (q + 1) * per; ++c) t = fmaf(__ldg(w + (size_t)c * cr), av[c], t);
    red[tid] = t;
  }
  __syncthreads();
  if (tid < cr) {
    float t = 0.f;
    for (int q = 0; q < 256 / cr; ++q) t += red[q * cr + tid];
    t = se.h_in[(size_t)b * cr + tid] > 0.f ? t : 0.f;
    dhv[tid] = t;
    if (rank == 0) se.dh[(size_t)b * cr + tid] = t;
  }
  __syncthreads();
  const float inv_hw = 1.f / (float)hw;
  for (int c = tid; c < C; c += 256) {
    float dp = 0.f;
    for (int j = 0; j < cr; ++j) dp = fmaf(__ldg(se.w1 + (size_t)j * C + c), dhv[j], dp);
    const float s = sf[c];
    const float ta = fmaf(s, tot[c], dp);                              // sum dz
    const float tx = fmaf(s, tot[C + c], dp * inv_hw * tot[2 * C + c]);  // sum dz * y
    float mu, rs;
    gn_chan(p, b, c, mu, rs);
    const float tb = rs * (tx - mu * ta);                              // sum dz * xhat
    dpv[c] = dp * inv_hw;
    t1[c] = ta;
    t2[c] = tb;
    if (rank == 0) {   // this frame's row of the dgamma / dbeta partials (summed in order by reduce_partials)
      dbeta[(size_t)b * C + c] = ta;
      dgamma[(size_t)b * C + c] = tb;
    }
  }
  __syncthreads();
  const int cpg = 1 << p.lcpg;
  for (int gi = tid; gi < G; gi += 256) {
    float s1 = 0.f, s2 = 0.f;
    for (int c = gi * cpg; c < (gi + 1) * cpg; ++c) {
      const float gm = p.gamma[c];
      s1 = fmaf(gm, t1[c], s1);
      s2 = fmaf(gm, t2[c], s2);
    }
    gS[gi] = s1;
    gS[G + gi] = s2;
  }
  __syncthreads();
  // dy = zc*dz + (x*c3 + c2) as in gn_bwd_cluster_sums, with dz = s*gz + dp/hw
  float zc[8], c2[8], c3[8], sc[8], dq[8];
  {
    float mu[8], rs[8], gm[8];
    gn_coeffs(p, b, c0, mu, rs);
    load8f(p.gamma + c0, gm);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int gi = (c0 + e) >> p.lcpg;
      const float k2 = rs[e] * p.inv_m * gS[gi], k3 = rs[e] * p.inv_m * gS[G + gi];
      zc[e] = rs[e] * gm[e];
      c3[e] = -rs[e] * k3;
      c2[e] = fmaf(mu[e] * rs[e], k3, -k2);
      sc[e] = sf[c0 + e];
      dq[e] = dpv[c0 + e];
    }
  }
  uint4* od = reinterpret_cast<uint4*>(dy) + base;
  uint4* oz = gz_out ? reinterpret_cast<uint4*>(gz_out) + base : nullptr;
  for (int i = tid; i < n; i += 256) {
    float gv[8], x[8], ac[8], gz[8], o[8];
    unpack8(srg[i], gv);
    unpack8a(sry[i], x);
    unpack8a(sra[i], ac);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      gz[e] = ac[e] > 0.f ? gv[e] : 0.f;
      o[e] = fmaf(zc[e], fmaf(sc[e], gz[e], dq[e]), fmaf(x[e], c3[e], c2[e]));
    }
    od[i] = pack8(o);
    if (oz) oz[i] = pack8(gz);
  }
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// Cluster size (CTAs per frame) and pixels per CTA for the SE kernels: the smallest cluster whose staged slice of
// `ntens` 16-bit tensors is <= 48 KB (as in hb200_gn_bwd), up to the portable maximum of 8.  A slice that with the
// kernel's `extra` bytes of shared memory exceeds 200 KB is not staged (staged = 0: both passes read global memory).
static int se_launch(const void* kern, int batch, int hw, int C, int ntens, size_t extra, cudaStream_t st,
                     cudaLaunchConfig_t* cfg, cudaLaunchAttribute* at, int* ppc, int* staged) {
  int cs = 1;
  size_t slice = 0;
  for (;; cs *= 2) {
    *ppc = (hw + cs - 1) / cs;
    slice = (size_t)ntens * *ppc * C * 2;
    if (slice <= 48 * 1024 || cs == 8) break;
  }
  *staged = slice + extra <= 200 * 1024 ? 1 : 0;
  const size_t smem = (*staged ? slice : 0) + extra;
  HB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  *cfg = {};
  cfg->gridDim = dim3((unsigned)batch * cs);
  cfg->blockDim = dim3(256);
  cfg->dynamicSmemBytes = smem;
  cfg->stream = st;
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = cs; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  cfg->attrs = at;
  cfg->numAttrs = 1;
  return HB200_OK;
}

static int se_check(int C, int cr) {
  HB_CHECK_ARG(C / 8 >= 1 && C / 8 <= 256 && 256 % (C / 8) == 0, "gn_se: C/8 = %d must divide 256", C / 8);
  HB_CHECK_ARG(cr >= 4 && cr % 4 == 0 && 256 % cr == 0 && C % (256 / cr) == 0,
               "gn_se: reduced width %d must be a multiple of 4 dividing 256 (and 256/%d must divide C = %d)", cr, cr, C);
  return HB200_OK;
}

}  // namespace hb200

using namespace hb200;

// ---- C ABI ---------------------------------------------------------------------------------
static int prep_check(const uint8_t* rgb, const float* depth, const int32_t* rows, int B, int H, int W,
                      int c_rgb, int c_depth) {
  HB_CHECK_ARG(rows && B > 0, "prep: bad args");
  HB_CHECK_ARG((c_rgb == 3 && rgb) || (c_rgb == 0), "prep: c_rgb must be 0 or 3");
  HB_CHECK_ARG((c_depth == 1 && depth) || (c_depth == 0), "prep: c_depth must be 0 or 1");
  HB_CHECK_ARG(c_rgb + c_depth > 0, "prep: no visual channels");
  HB_CHECK_ARG(H % 2 == 0 && W % 8 == 0, "prep: H must be even and W a multiple of 8 (got %dx%d)", H, W);
  return HB200_OK;
}

extern "C" int hb200_prep_stats(const uint8_t* rgb, const float* depth, const int32_t* frame_rows,
                                int batch, int height, int width, int c_rgb, int c_depth,
                                float rgb_scale, double* stats_acc, hb200_stream_t stream) {
  int rc = prep_check(rgb, depth, frame_rows, batch, height, width, c_rgb, c_depth);
  if (rc) return rc;
  HB_CHECK_ARG(stats_acc, "prep_stats: null stats");
  cudaStream_t st = (cudaStream_t)stream;
  HB_CUDA(cudaMemsetAsync(stats_acc, 0, 17 * sizeof(double), st));
  const long long total = (long long)batch * (height / 2) * (width / 8);
  const int grid = grid_for(total, 256);
  if (c_rgb && c_depth) prep_stats_kernel<true, true><<<grid, 256, 0, st>>>(rgb, depth, frame_rows, batch, height, width, rgb_scale, stats_acc);
  else if (c_rgb) prep_stats_kernel<true, false><<<grid, 256, 0, st>>>(rgb, depth, frame_rows, batch, height, width, rgb_scale, stats_acc);
  else prep_stats_kernel<false, true><<<grid, 256, 0, st>>>(rgb, depth, frame_rows, batch, height, width, rgb_scale, stats_acc);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

extern "C" int hb200_prep_finalize(const double* stats_acc, float* run_mean, float* run_var,
                                   float* run_count, float* scale_shift, int channels,
                                   long long pixels_per_frame, int update, hb200_stream_t stream) {
  HB_CHECK_ARG(stats_acc && run_mean && run_var && run_count && scale_shift, "prep_finalize: null pointer");
  HB_CHECK_ARG(channels > 0 && channels <= 8, "prep_finalize: channels must be 1..8");
  prep_finalize_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(stats_acc, run_mean, run_var, run_count,
                                                            scale_shift, channels, pixels_per_frame, update);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

extern "C" int hb200_prep_apply(const uint8_t* rgb, const float* depth, const int32_t* frame_rows,
                                int batch, int height, int width, int c_rgb, int c_depth,
                                float rgb_scale, const float* scale_shift, hb200_f16* out, hb200_bf16* out_bf16,
                                int s2d, hb200_stream_t stream) {
  int rc = prep_check(rgb, depth, frame_rows, batch, height, width, c_rgb, c_depth);
  if (rc) return rc;
  HB_CHECK_ARG(out, "prep_apply: null out");
  cudaStream_t st = (cudaStream_t)stream;
  const long long total = (long long)batch * (height / 2) * (width / 8);
  const int grid = grid_for(total, 256);
  act_t* o = (act_t*)out;
  grad_t* o2 = (grad_t*)out_bf16;
  HB_CHECK_ARG(!s2d || (height % 4 == 0), "prep_apply: s2d needs H %% 4 == 0");
#define HB_PREP(R, D)                                                                                              \
  if (s2d) prep_apply_kernel<R, D, true><<<grid, 256, 0, st>>>(rgb, depth, frame_rows, batch, height, width, rgb_scale, scale_shift, o, o2); \
  else prep_apply_kernel<R, D, false><<<grid, 256, 0, st>>>(rgb, depth, frame_rows, batch, height, width, rgb_scale, scale_shift, o, o2)
  if (c_rgb && c_depth) { HB_PREP(true, true); }
  else if (c_rgb) { HB_PREP(true, false); }
  else { HB_PREP(false, true); }
#undef HB_PREP
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

extern "C" int hb200_gn_apply(const hb200_f16* y, const double* stats, const float* gamma,
                              const float* beta, void* out, hb200_bf16* out_bf16, int out_f32, int batch, int hw,
                              int channels, int groups, float eps, int relu, hb200_stream_t stream) {
  GnP p;
  int rc = make_gn(p, stats, gamma, beta, channels, groups, hw, eps);
  if (rc) return rc;
  HB_CHECK_ARG(y && out, "gn_apply: null pointer");
  HB_CHECK_ARG(!out_bf16 || out_f32 == 0, "gn_apply: the bf16 twin accompanies the fp16 output only");
  grad_t* o2 = (grad_t*)out_bf16;
  int ppb = 0, grid = 0;
  rc = gn_slab_launch(channels, hw, batch, &ppb, &grid);
  if (rc) return rc;
  if (out_f32 == 1)
    gn_apply_kernel<1><<<grid, 256, 0, (cudaStream_t)stream>>>((const act_t*)y, p, out, o2, batch, hw, relu, ppb);
  else if (out_f32 == 2)
    gn_apply_kernel<2><<<grid, 256, 0, (cudaStream_t)stream>>>((const act_t*)y, p, out, o2, batch, hw, relu, ppb);
  else
    gn_apply_kernel<0><<<grid, 256, 0, (cudaStream_t)stream>>>((const act_t*)y, p, out, o2, batch, hw, relu, ppb);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

extern "C" int hb200_gn_residual_relu(const hb200_f16* y, const double* stats, const float* gamma,
                                      const float* beta, const hb200_f16* res, const double* res_stats,
                                      const float* res_gamma, const float* res_beta, hb200_f16* out,
                                      hb200_bf16* out_bf16, int batch, int hw, int channels, int groups, float eps,
                                      hb200_stream_t stream) {
  GnP p, rp;
  int rc = make_gn(p, stats, gamma, beta, channels, groups, hw, eps);
  if (rc) return rc;
  HB_CHECK_ARG(y && res && out, "gn_residual_relu: null pointer");
  rp = p;
  if (res_stats) {
    rc = make_gn(rp, res_stats, res_gamma, res_beta, channels, groups, hw, eps);
    if (rc) return rc;
  }
  int ppb = 0, grid = 0;
  rc = gn_slab_launch(channels, hw, batch, &ppb, &grid);
  if (rc) return rc;
  gn_residual_relu_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(
      (const act_t*)y, p, (const act_t*)res, rp, res_stats ? 1 : 0, (act_t*)out, (grad_t*)out_bf16, batch, hw, ppb);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

extern "C" int hb200_gn_relu_maxpool(const hb200_f16* y, const double* stats, const float* gamma,
                                     const float* beta, hb200_f16* out, hb200_bf16* out_bf16, uint8_t* argmax,
                                     int batch, int h, int w, int channels, int groups, float eps,
                                     hb200_stream_t stream) {
  GnP p;
  int rc = make_gn(p, stats, gamma, beta, channels, groups, h * w, eps);
  if (rc) return rc;
  HB_CHECK_ARG(y && out && argmax && h > 0 && w > 0, "gn_relu_maxpool: bad args");
  if (h % 2 == 0 && w % 2 == 0) {
    // slab path: largest even row count <= 8 dividing h whose rows+1 staged rows fit in 64 KB
    const int cv = channels / 8;
    int rows = 0;
    for (int r = 8; r >= 2; r -= 2)
      if (h % r == 0 && (size_t)(r + 1) * w * channels * 2 <= 64 * 1024) { rows = r; break; }
    if (rows && cv <= 32 && 256 % cv == 0) {
      const size_t smem = (size_t)(rows + 1) * w * channels * 2;
      auto kern = gn_relu_maxpool_slab_kernel;
      HB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      kern<<<batch * (h / rows), 256, smem, (cudaStream_t)stream>>>((const act_t*)y, p, (act_t*)out,
                                                                    (grad_t*)out_bf16, argmax, h, w, rows);
      HB_LAUNCH_OK();
      count_launch(1);
      return HB200_OK;
    }
  }
  const long long total = (long long)batch * ((h + 1) / 2) * ((w + 1) / 2) * (channels / 8);
  gn_relu_maxpool_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(
      (const act_t*)y, p, (act_t*)out, (grad_t*)out_bf16, argmax, batch, h, w);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

extern "C" int hb200_maxpool_bwd(const hb200_bf16* dout, const uint8_t* argmax, hb200_bf16* dz,
                                 int batch, int h, int w, int channels, hb200_stream_t stream) {
  HB_CHECK_ARG(dout && argmax && dz && channels % 8 == 0 && h > 0 && w > 0, "maxpool_bwd: bad args");
  const long long total = (long long)batch * h * w * (channels / 8);
  maxpool_bwd_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(
      (const grad_t*)dout, argmax, (grad_t*)dz, batch, h, w, channels);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

extern "C" int hb200_gn_bwd_reduce(const hb200_bf16* g, const hb200_bf16* act, const hb200_bf16* y,
                                   const double* stats, const float* gamma, const float* beta,
                                   float* sums, float* dgamma, float* dbeta, int batch, int hw,
                                   int channels, int groups, float eps, int mask_mode,
                                   hb200_stream_t stream) {
  GnP p;
  int rc = make_gn(p, stats, gamma, beta, channels, groups, hw, eps);
  if (rc) return rc;
  HB_CHECK_ARG(g && y && sums && dgamma && dbeta, "gn_bwd_reduce: null pointer");
  HB_CHECK_ARG(mask_mode >= 0 && mask_mode <= 2 && (mask_mode != 2 || act), "gn_bwd_reduce: bad mask_mode");
  HB_CHECK_ARG(channels <= 2048 && 256 % (channels / 8) == 0, "gn_bwd_reduce: C/8 must divide 256");
  cudaStream_t st = (cudaStream_t)stream;
  HB_CUDA(cudaMemsetAsync(sums, 0, sizeof(float) * 2 * (size_t)batch * groups, st));
  const int npl = 256 / (channels / 8);
  int ppb = npl * 16;  // 16 pixels per thread
  if (ppb > hw) ppb = hw;
  const int slabs = (hw + ppb - 1) / ppb;
  gn_bwd_reduce_kernel<<<batch * slabs, 256, 0, st>>>((const grad_t*)g, (const act_t*)act,
                                                      (const act_t*)y, p, sums, dgamma, dbeta,
                                                      batch, hw, ppb, mask_mode);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

extern "C" int hb200_gn_bwd_apply(const hb200_bf16* g, const hb200_bf16* act, const hb200_bf16* y,
                                  const double* stats, const float* gamma, const float* beta,
                                  const float* sums, hb200_bf16* dy, hb200_bf16* gz_out, int batch,
                                  int hw, int channels, int groups, float eps, int mask_mode,
                                  hb200_stream_t stream) {
  GnP p;
  int rc = make_gn(p, stats, gamma, beta, channels, groups, hw, eps);
  if (rc) return rc;
  HB_CHECK_ARG(g && y && sums && dy, "gn_bwd_apply: null pointer");
  HB_CHECK_ARG(mask_mode >= 0 && mask_mode <= 2 && (mask_mode != 2 || act), "gn_bwd_apply: bad mask_mode");
  int ppb = 0, grid = 0;
  rc = gn_slab_launch(channels, hw, batch, &ppb, &grid);
  if (rc) return rc;
  gn_bwd_apply_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(
      (const grad_t*)g, (const act_t*)act, (const act_t*)y, p, sums,
      (grad_t*)dy, (grad_t*)gz_out, batch, hw, mask_mode, ppb);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

extern "C" int hb200_bf16_to_f32(const hb200_bf16* x, float* out, long long n, hb200_stream_t stream) {
  HB_CHECK_ARG(x && out && n > 0 && n % 8 == 0, "bf16_to_f32: n must be a positive multiple of 8");
  bf16_to_f32_kernel<<<grid_for(n / 8, 256), 256, 0, (cudaStream_t)stream>>>((const __nv_bfloat16*)x, out, n / 8);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}
extern "C" int hb200_f16_to_bf16(const hb200_f16* x, hb200_bf16* out, long long n, hb200_stream_t stream) {
  HB_CHECK_ARG(x && out && n % 8 == 0, "f16_to_bf16: n must be a multiple of 8");
  f16_to_bf16_kernel<<<grid_for(n / 8, 256), 256, 0, (cudaStream_t)stream>>>((const act_t*)x, (grad_t*)out, n / 8);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

extern "C" int hb200_f32_to_bf16(const float* x, hb200_bf16* out, long long n, hb200_stream_t stream) {
  HB_CHECK_ARG(x && out && n > 0 && n % 8 == 0, "f32_to_bf16: n must be a positive multiple of 8");
  f32_to_bf16_kernel<<<grid_for(n / 8, 256), 256, 0, (cudaStream_t)stream>>>(x, (__nv_bfloat16*)out, n / 8);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

extern "C" int hb200_embed_fwd(const float* goal, const int64_t* prev_actions, const uint8_t* masks,
                               const int32_t* frame_rows, const float* w_tgt, const float* b_tgt,
                               const float* emb_table, float* out, int ld, int col0, int batch,
                               hb200_stream_t stream) {
  HB_CHECK_ARG(goal && prev_actions && masks && frame_rows && w_tgt && b_tgt && emb_table && out && batch > 0,
               "embed_fwd: bad args");
  embed_fwd_kernel<<<grid_for((long long)batch * 64, 256), 256, 0, (cudaStream_t)stream>>>(
      goal, prev_actions, masks, frame_rows, w_tgt, b_tgt, emb_table, out, ld, col0, batch);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}
extern "C" int hb200_embed_bwd(const float* goal, const int64_t* prev_actions, const uint8_t* masks,
                               const int32_t* frame_rows, const float* d_out, int ld, int col0,
                               int batch, int n_emb, float* d_w_tgt, float* d_b_tgt, float* d_emb,
                               hb200_stream_t stream) {
  HB_CHECK_ARG(goal && prev_actions && masks && frame_rows && d_out && d_w_tgt && d_b_tgt && d_emb && batch > 0,
               "embed_bwd: bad args");
  HB_CHECK_ARG(n_emb > 0 && n_emb <= 64, "embed_bwd: n_emb out of range");
  cudaStream_t st = (cudaStream_t)stream;
  const int nacc = 128 + n_emb * 32, nparts = cdiv(batch, kEmbedFrames);
  float* parts = nullptr;
  int* tickets = nullptr;
  int rc = stream_workspace(st, (size_t)(nparts + kReduceChunks) * nacc, 0, &parts, &tickets);
  if (rc) return rc;
  float* tmp = parts + (size_t)nparts * nacc;
  embed_bwd_kernel<<<dim3(cdiv(nacc, 128), nparts), 128, 0, st>>>(goal, prev_actions, masks, frame_rows, d_out, ld,
                                                                   col0, batch, n_emb, parts);
  HB_LAUNCH_OK();
  count_launch(1);
  rc = reduce_partials(parts, nparts, nacc, 96, d_w_tgt, tmp, st);
  if (!rc) rc = reduce_partials(parts + 96, nparts, nacc, 32, d_b_tgt, tmp, st);
  if (!rc) rc = reduce_partials(parts + 128, nparts, nacc, (long long)n_emb * 32, d_emb, tmp, st);
  return rc;
}

extern "C" int hb200_sensor_linear_fwd(const float* x, int in_dim, const int32_t* frame_rows, int batch, int transform,
                                       const float* w, const float* b, float* out, int ld, int col0, int out_dim,
                                       hb200_stream_t stream) {
  HB_CHECK_ARG(x && frame_rows && out && batch > 0 && in_dim >= 1 && in_dim <= 8, "sensor_linear_fwd: bad args");
  HB_CHECK_ARG(transform >= 0 && transform <= 3 && out_dim >= 1 && out_dim <= 64, "sensor_linear_fwd: bad transform / width");
  HB_CHECK_ARG((w && b) || (!w && transform == 0 && out_dim == in_dim), "sensor_linear_fwd: raw copy needs identity features");
  sensor_linear_fwd_kernel<<<grid_for((long long)batch * out_dim, 256), 256, 0, (cudaStream_t)stream>>>(
      x, in_dim, frame_rows, batch, transform, w, b, out, ld, col0, out_dim);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

extern "C" int hb200_sensor_linear_bwd(const float* x, int in_dim, const int32_t* frame_rows, int batch, int transform,
                                       const float* d_out, int ld, int col0, int out_dim, float* d_w, float* d_b,
                                       hb200_stream_t stream) {
  HB_CHECK_ARG(x && frame_rows && d_out && d_w && d_b && batch > 0 && in_dim >= 1 && in_dim <= 8, "sensor_linear_bwd: bad args");
  HB_CHECK_ARG(transform >= 0 && transform <= 3 && out_dim >= 1 && out_dim <= 64, "sensor_linear_bwd: bad transform / width");
  const int nf = transform == 1 ? 3 : (transform == 2 ? 4 : (transform == 3 ? 2 : in_dim));   // sensor_features
  const int nacc = out_dim * (nf + 1), nparts = cdiv(batch, kEmbedFrames);
  HB_CHECK_ARG(nparts <= 65535, "sensor_linear_bwd: batch %d exceeds %d frames", batch, 65535 * kEmbedFrames);
  cudaStream_t st = (cudaStream_t)stream;
  float* parts = nullptr;
  int* tickets = nullptr;
  int rc = stream_workspace(st, (size_t)(nparts + kReduceChunks) * nacc, 0, &parts, &tickets);
  if (rc) return rc;
  float* tmp = parts + (size_t)nparts * nacc;
  sensor_linear_bwd_kernel<<<dim3(cdiv(nacc, 128), nparts), 128, 0, st>>>(x, in_dim, frame_rows, batch, transform, d_out,
                                                                          ld, col0, out_dim, nf, parts);
  HB_LAUNCH_OK();
  count_launch(1);
  rc = reduce_partials(parts, nparts, nacc, (long long)out_dim * nf, d_w, tmp, st);
  if (!rc) rc = reduce_partials(parts + (size_t)out_dim * nf, nparts, nacc, out_dim, d_b, tmp, st);
  return rc;
}

extern "C" int hb200_index_embed_fwd(const int64_t* idx, const int32_t* frame_rows, const uint8_t* masks, int batch,
                                     int table_rows, const float* table, int width, float* out, int ld, int col0,
                                     hb200_stream_t stream) {
  HB_CHECK_ARG(idx && table && out && batch > 0 && table_rows > 0 && width > 0, "index_embed_fwd: bad args");
  index_embed_fwd_kernel<<<grid_for((long long)batch * width, 256), 256, 0, (cudaStream_t)stream>>>(
      idx, frame_rows, masks, batch, table_rows, table, width, out, ld, col0);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

extern "C" int hb200_index_embed_bwd(const int64_t* idx, const int32_t* frame_rows, const uint8_t* masks, int batch,
                                     int table_rows, int width, const float* d_out, int ld, int col0, float* d_table,
                                     hb200_stream_t stream) {
  HB_CHECK_ARG(idx && d_out && d_table && batch > 0 && table_rows > 0 && width > 0, "index_embed_bwd: bad args");
  const long long nacc = (long long)table_rows * width;
  const int nparts = cdiv(batch, kEmbedFrames);
  HB_CHECK_ARG(nparts <= 65535, "index_embed_bwd: batch %d exceeds %d frames", batch, 65535 * kEmbedFrames);
  cudaStream_t st = (cudaStream_t)stream;
  float* parts = nullptr;
  int* tickets = nullptr;
  const int rc = stream_workspace(st, (size_t)(nparts + kReduceChunks) * nacc, 0, &parts, &tickets);
  if (rc) return rc;
  index_embed_bwd_kernel<<<dim3(cdiv(nacc, 128), nparts), 128, 0, st>>>(idx, frame_rows, masks, batch, table_rows, width,
                                                                        d_out, ld, col0, parts);
  HB_LAUNCH_OK();
  count_launch(1);
  return reduce_partials(parts, nparts, nacc, nacc, d_table, parts + (size_t)nparts * nacc, st);
}

extern "C" int hb200_prev_action_linear_fwd(const float* prev_actions, const uint8_t* masks, int batch, int n_actions,
                                            const float* w, const float* b, float* out, int ld, int col0,
                                            hb200_stream_t stream) {
  HB_CHECK_ARG(prev_actions && masks && w && b && out && batch > 0, "prev_action_linear_fwd: bad args");
  HB_CHECK_ARG(n_actions >= 1 && n_actions <= 64, "prev_action_linear_fwd: n_actions=%d unsupported (1..64)", n_actions);
  prev_action_linear_fwd_kernel<<<grid_for((long long)batch * 32, 256), 256, 0, (cudaStream_t)stream>>>(
      prev_actions, masks, batch, n_actions, w, b, out, ld, col0);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

extern "C" int hb200_prev_action_linear_bwd(const float* prev_actions, const uint8_t* masks, int batch, int n_actions,
                                            const float* d_out, int ld, int col0, float* d_w, float* d_b,
                                            hb200_stream_t stream) {
  HB_CHECK_ARG(prev_actions && masks && d_out && d_w && d_b && batch > 0, "prev_action_linear_bwd: bad args");
  HB_CHECK_ARG(n_actions >= 1 && n_actions <= 64, "prev_action_linear_bwd: n_actions=%d unsupported (1..64)", n_actions);
  const int nacc = 32 * (n_actions + 1), nparts = cdiv(batch, kEmbedFrames);
  HB_CHECK_ARG(nparts <= 65535, "prev_action_linear_bwd: batch %d exceeds %d frames", batch, 65535 * kEmbedFrames);
  cudaStream_t st = (cudaStream_t)stream;
  float* parts = nullptr;
  int* tickets = nullptr;
  int rc = stream_workspace(st, (size_t)(nparts + kReduceChunks) * nacc, 0, &parts, &tickets);
  if (rc) return rc;
  float* tmp = parts + (size_t)nparts * nacc;
  prev_action_linear_bwd_kernel<<<dim3(cdiv(nacc, 128), nparts), 128, 0, st>>>(prev_actions, masks, batch, n_actions,
                                                                               d_out, ld, col0, parts);
  HB_LAUNCH_OK();
  count_launch(1);
  rc = reduce_partials(parts, nparts, nacc, 32LL * n_actions, d_w, tmp, st);
  if (!rc) rc = reduce_partials(parts + 32 * n_actions, nparts, nacc, 32, d_b, tmp, st);
  return rc;
}

extern "C" int hb200_prep_generic(const void* const* h_srcs, const int* h_dtypes, const int* h_channels,
                                  const float* h_scales, int n_srcs, const int32_t* frame_rows, int batch, int height,
                                  int width, const float* scale_shift, hb200_f16* out, hb200_bf16* out_bf16,
                                  double* stats_acc, hb200_stream_t stream) {
  HB_CHECK_ARG(h_srcs && h_dtypes && h_channels && h_scales && n_srcs >= 1 && n_srcs <= kPrepMaxSrcs,
               "prep_generic: 1..%d sources", kPrepMaxSrcs);
  HB_CHECK_ARG(frame_rows && batch > 0 && height >= 2 && width >= 2, "prep_generic: bad shape");
  HB_CHECK_ARG((stats_acc != nullptr) != (out != nullptr), "prep_generic: pass either stats_acc (statistics pass) or out (apply pass)");
  PrepSrcs src;
  int ctot = 0;
  for (int k = 0; k < kPrepMaxSrcs; ++k) {
    src.ptr[k] = nullptr; src.dtype[k] = 0; src.channels[k] = 0; src.scale[k] = 1.f;
  }
  for (int k = 0; k < n_srcs; ++k) {
    HB_CHECK_ARG(h_srcs[k] && h_dtypes[k] >= 0 && h_dtypes[k] <= 2 && h_channels[k] >= 1, "prep_generic: bad source %d", k);
    src.ptr[k] = h_srcs[k]; src.dtype[k] = h_dtypes[k]; src.channels[k] = h_channels[k]; src.scale[k] = h_scales[k];
    ctot += h_channels[k];
  }
  HB_CHECK_ARG(ctot <= 8, "prep_generic: at most 8 input channels (got %d)", ctot);
  src.n = n_srcs;
  cudaStream_t st = (cudaStream_t)stream;
  const long long total = (long long)batch * (height / 2) * (width / 2);
  const int grid = grid_for(total, 256);
  if (stats_acc) {
    HB_CUDA(cudaMemsetAsync(stats_acc, 0, 17 * sizeof(double), st));
    prep_generic_kernel<true><<<grid, 256, 0, st>>>(src, frame_rows, batch, height, width, nullptr, nullptr, nullptr, stats_acc);
  } else {
    prep_generic_kernel<false><<<grid, 256, 0, st>>>(src, frame_rows, batch, height, width, scale_shift, (act_t*)out,
                                                     (grad_t*)out_bf16, nullptr);
  }
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}


extern "C" int hb200_rnn_shift_mask(const float* h_seq, const float* h0, long long h0_row_stride,
                                    const uint8_t* masks, float* h_in, int t_steps, int n, int hidden,
                                    hb200_stream_t stream) {
  HB_CHECK_ARG(h_seq && h0 && masks && h_in && t_steps > 0 && n > 0 && hidden > 0, "rnn_shift_mask: bad args");
  const long long total = (long long)t_steps * n * hidden;
  rnn_shift_mask_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(h_seq, h0, h0_row_stride, masks,
                                                                                 h_in, t_steps, n, hidden);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}
extern "C" int hb200_colsum(const float* x, long long ld, float* out, long long m, int n, int accumulate,
                            hb200_stream_t stream) {
  HB_CHECK_ARG(x && out && m > 0 && n > 0 && ld >= n, "colsum: bad args");
  colsum_kernel<<<(n + 31) / 32, 1024, 0, (cudaStream_t)stream>>>(x, ld, out, m, n, accumulate);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

extern "C" int hb200_relu_bwd(float* d, const float* y, long long ld_d, long long ld_y, long long rows,
                              int cols, hb200_stream_t stream) {
  HB_CHECK_ARG(d && y && rows > 0 && cols > 0, "relu_bwd: bad args");
  relu_bwd_kernel<<<grid_for(rows * cols, 256), 256, 0, (cudaStream_t)stream>>>(d, y, ld_d, ld_y, rows, cols);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}
extern "C" int hb200_f32_chw_to_bf16_hwc(const float* x, hb200_bf16* out, int batch, int hw, int channels,
                                         hb200_stream_t stream) {
  HB_CHECK_ARG(x && out && batch > 0 && hw > 0 && channels % 8 == 0, "f32_chw_to_bf16_hwc: bad args");
  const long long total = (long long)batch * hw * (channels / 8);
  f32_chw_to_bf16_hwc_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(x, (__nv_bfloat16*)out, batch, hw, channels);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}
extern "C" int hb200_heads_fwd(const float* features, const float* w_act, const float* b_act,
                               const float* w_val, const float* b_val, int batch, int hidden, int n_actions,
                               float* logits, float* values, hb200_stream_t stream) {
  HB_CHECK_ARG(features && w_act && b_act && w_val && b_val && logits && values && batch > 0, "heads_fwd: bad args");
  heads_fwd_kernel<<<cdiv(batch, 8), 256, 0, (cudaStream_t)stream>>>(features, w_act, b_act, w_val, b_val, batch,
                                                                      hidden, n_actions, logits, values);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

extern "C" int hb200_heads_act(const float* features, const float* w_act, const float* b_act, const float* w_val,
                               const float* b_val, const float* uniform, int batch, int hidden, int n_actions,
                               float* log_probs, float* values, long long* actions, float* action_log_probs,
                               hb200_stream_t stream) {
  HB_CHECK_ARG(features && w_act && b_act && w_val && b_val && log_probs && values && actions && action_log_probs &&
                   batch > 0 && n_actions > 0,
               "heads_act: bad args");
  heads_act_kernel<<<cdiv(batch, 8), 256, 0, (cudaStream_t)stream>>>(features, w_act, b_act, w_val, b_val, uniform, batch,
                                                                      hidden, n_actions, log_probs, values, actions,
                                                                      action_log_probs);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

extern "C" int hb200_gn_bwd(const hb200_bf16* g, const hb200_bf16* act, const hb200_bf16* y, const double* stats,
                            const float* gamma, const float* beta, float* dgamma, float* dbeta, hb200_bf16* dy,
                            hb200_bf16* gz_out, int batch, int hw, int channels, int groups, float eps,
                            int mask_mode, hb200_stream_t stream) {
  GnP p;
  int rc = make_gn(p, stats, gamma, beta, channels, groups, hw, eps);
  if (rc) return rc;
  HB_CHECK_ARG(g && y && dgamma && dbeta && dy, "gn_bwd: null pointer");
  HB_CHECK_ARG(mask_mode >= 0 && mask_mode <= 2 && (mask_mode != 2 || act), "gn_bwd: bad mask_mode");
  const int cv = channels / 8;
  HB_CHECK_ARG(cv >= 1 && cv <= 256 && 256 % cv == 0, "gn_bwd: C/8 = %d must divide 256", cv);
  float *part_g = nullptr, *part_b = nullptr;
  rc = gn_affine_grads_workspace((cudaStream_t)stream, batch, channels, &part_g, &part_b);
  if (rc) return rc;
  if (cv <= 32) {
    // cluster path: smallest cluster whose per-CTA slice is <= 48 KB (<= 200 KB at the portable maximum of 8)
    const int ntens = mask_mode == 2 ? 3 : 2;
    int cs = 1, ppc = hw;
    size_t slice = 0;
    for (;; cs *= 2) {
      ppc = (hw + cs - 1) / cs;
      slice = (size_t)ntens * ppc * channels * 2;
      if (slice <= 48 * 1024 || cs == 8) break;
    }
    const size_t smem = slice + sizeof(float) * (20 * (size_t)channels + 2 * (size_t)groups);
    if (smem <= 200 * 1024) {
      cudaLaunchConfig_t cfg = {};
      cfg.gridDim = dim3((unsigned)batch * cs);
      cfg.blockDim = dim3(256);
      cfg.dynamicSmemBytes = smem;
      cfg.stream = (cudaStream_t)stream;
      cudaLaunchAttribute at[1];
      at[0].id = cudaLaunchAttributeClusterDimension;
      at[0].val.clusterDim.x = cs; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
      cfg.attrs = at;
      cfg.numAttrs = 1;
      const grad_t* G_ = (const grad_t*)g;
      const act_t *A_ = (const act_t*)act, *Y_ = (const act_t*)y;
      grad_t *D_ = (grad_t*)dy, *Z_ = (grad_t*)gz_out;
#define HB_GNB_CASE(m)                                                                                       \
  {                                                                                                          \
    auto kern = gn_bwd_cluster_kernel<m>;                                                                    \
    HB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));             \
    HB_CUDA(cudaLaunchKernelEx(&cfg, kern, G_, A_, Y_, p, part_g, part_b, D_, Z_, hw, ppc));                 \
  }
      if (mask_mode == 0) HB_GNB_CASE(0) else if (mask_mode == 1) HB_GNB_CASE(1) else HB_GNB_CASE(2)
#undef HB_GNB_CASE
      count_launch(1);
      return gn_affine_grads_reduce(part_g, part_b, batch, channels, dgamma, dbeta, (cudaStream_t)stream);
    }
  }
  const size_t smem = sizeof(float) * (2 * (size_t)channels + 2 * (size_t)groups);
  gn_bwd_fused_kernel<<<batch, 256, smem, (cudaStream_t)stream>>>(
      (const grad_t*)g, (const act_t*)act, (const act_t*)y, p, part_g, part_b,
      (grad_t*)dy, (grad_t*)gz_out, batch, hw, mask_mode);
  HB_LAUNCH_OK();
  count_launch(1);
  return gn_affine_grads_reduce(part_g, part_b, batch, channels, dgamma, dbeta, (cudaStream_t)stream);
}

extern "C" int hb200_gn_se_residual_relu(const hb200_f16* y, const double* stats, const float* gamma,
                                         const float* beta, const hb200_f16* res, const double* res_stats,
                                         const float* res_gamma, const float* res_beta, const float* w1,
                                         const float* b1, const float* w2, const float* b2, float* p, float* h,
                                         float* s, hb200_f16* out, hb200_bf16* out_bf16, int batch, int hw,
                                         int channels, int groups, int reduced, float eps, hb200_stream_t stream) {
  GnP gp, rp;
  int rc = make_gn(gp, stats, gamma, beta, channels, groups, hw, eps);
  if (rc) return rc;
  HB_CHECK_ARG(y && res && out && w1 && b1 && w2 && b2 && p && h && s && batch > 0 && hw > 0,
               "gn_se_residual_relu: bad args");
  rc = se_check(channels, reduced);
  if (rc) return rc;
  rp = gp;
  if (res_stats) {
    rc = make_gn(rp, res_stats, res_gamma, res_beta, channels, groups, hw, eps);
    if (rc) return rc;
  }
  SeP se = {};
  se.w1 = w1; se.b1 = b1; se.w2 = w2; se.b2 = b2; se.p = p; se.h = h; se.s = s; se.cr = reduced;
  const size_t extra = sizeof(float) * (4 * (size_t)channels + reduced);
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute at[1];
  int ppc = 0, staged = 0;
  auto kern = gn_se_residual_relu_kernel;
  rc = se_launch((const void*)kern, batch, hw, channels, 1, extra, (cudaStream_t)stream, &cfg, at, &ppc, &staged);
  if (rc) return rc;
  HB_CUDA(cudaLaunchKernelEx(&cfg, kern, (const act_t*)y, gp, (const act_t*)res, rp, res_stats ? 1 : 0, se,
                             (act_t*)out, (grad_t*)out_bf16, hw, ppc, staged));
  count_launch(1);
  return HB200_OK;
}

extern "C" int hb200_gn_se_bwd(const hb200_bf16* g, const hb200_bf16* act, const hb200_bf16* y, const double* stats,
                               const float* gamma, const float* beta, const float* s, const float* h, const float* w1,
                               const float* w2, float* dgamma, float* dbeta, hb200_bf16* dy, hb200_bf16* gz_out,
                               float* a, float* dh, int batch, int hw, int channels, int groups, int reduced,
                               float eps, hb200_stream_t stream) {
  GnP gp;
  int rc = make_gn(gp, stats, gamma, beta, channels, groups, hw, eps);
  if (rc) return rc;
  HB_CHECK_ARG(g && act && y && s && h && w1 && w2 && dgamma && dbeta && dy && a && dh && batch > 0 && hw > 0,
               "gn_se_bwd: bad args");
  rc = se_check(channels, reduced);
  if (rc) return rc;
  float *part_g = nullptr, *part_b = nullptr;
  rc = gn_affine_grads_workspace((cudaStream_t)stream, batch, channels, &part_g, &part_b);
  if (rc) return rc;
  SeP se = {};
  se.w1 = w1; se.w2 = w2; se.s_in = s; se.h_in = h; se.a = a; se.dh = dh; se.cr = reduced;
  const size_t extra = sizeof(float) * (10 * (size_t)channels + 256 + reduced + 2 * (size_t)groups);
  cudaLaunchConfig_t cfg;
  cudaLaunchAttribute at[1];
  int ppc = 0, staged = 0;
  auto kern = gn_se_bwd_kernel;
  rc = se_launch((const void*)kern, batch, hw, channels, 3, extra, (cudaStream_t)stream, &cfg, at, &ppc, &staged);
  if (rc) return rc;
  HB_CUDA(cudaLaunchKernelEx(&cfg, kern, (const grad_t*)g, (const act_t*)act, (const act_t*)y, gp, se, part_g, part_b,
                             (grad_t*)dy, (grad_t*)gz_out, hw, ppc, staged));
  count_launch(1);
  return gn_affine_grads_reduce(part_g, part_b, batch, channels, dgamma, dbeta, (cudaStream_t)stream);
}

// rows per CTA for the fused stem backward: smallest cluster (1..8 CTAs per frame) whose slice fits; 0 = unsupported
static int gn_pool_bwd_plan(int h, int w, int channels, int groups, int* cs_out, size_t* smem_out) {
  const int cv = channels / 8;
  if (channels % 8 || cv < 1 || cv > 32 || 256 % cv || h % 2 || w % 2) return 0;
  for (int cs = 1; cs <= 8; cs *= 2) {
    if (h % (2 * cs)) continue;
    const int rows = h / cs;
    const size_t bytes = (size_t)rows * w * channels * 2 + (size_t)(rows / 2 + 1) * (w / 2) * channels * 3 +
                         sizeof(float) * (20 * (size_t)channels + 2 * (size_t)groups);
    if (bytes <= 50 * 1024 || (cs == 8 && bytes <= 200 * 1024)) {
      *cs_out = cs;
      *smem_out = bytes;
      return rows;
    }
  }
  return 0;
}

extern "C" int hb200_gn_relu_maxpool_bwd_supported(int h, int w, int channels, int groups) {
  int cs = 0;
  size_t smem = 0;
  return gn_pool_bwd_plan(h, w, channels, groups, &cs, &smem) > 0;
}

extern "C" int hb200_gn_relu_maxpool_bwd(const hb200_bf16* dpool, const uint8_t* argmax, const hb200_bf16* y,
                                         const double* stats, const float* gamma, const float* beta, float* dgamma,
                                         float* dbeta, hb200_bf16* dy, int batch, int h, int w, int channels,
                                         int groups, float eps, hb200_stream_t stream) {
  GnP p;
  int rc = make_gn(p, stats, gamma, beta, channels, groups, h * w, eps);
  if (rc) return rc;
  HB_CHECK_ARG(dpool && argmax && y && dgamma && dbeta && dy && batch > 0, "gn_relu_maxpool_bwd: null pointer");
  int cs = 0;
  size_t smem = 0;
  const int rows = gn_pool_bwd_plan(h, w, channels, groups, &cs, &smem);
  if (rows <= 0) {
    set_last_error("gn_relu_maxpool_bwd: unsupported shape %dx%dx%d (use maxpool_bwd + gn_bwd)", h, w, channels);
    return HB200_ERR_UNSUPPORTED;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)batch * cs);
  cfg.blockDim = dim3(256);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = (cudaStream_t)stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = cs; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  float *part_g = nullptr, *part_b = nullptr;
  rc = gn_affine_grads_workspace((cudaStream_t)stream, batch, channels, &part_g, &part_b);
  if (rc) return rc;
  auto kern = gn_pool_bwd_cluster_kernel;
  HB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  HB_CUDA(cudaLaunchKernelEx(&cfg, kern, (const grad_t*)dpool, argmax, (const act_t*)y, p, part_g, part_b,
                             (grad_t*)dy, h, w, rows));
  count_launch(1);
  return gn_affine_grads_reduce(part_g, part_b, batch, channels, dgamma, dbeta, (cudaStream_t)stream);
}

extern "C" int hb200_transpose_f32(const float* src, long long ld_src, float* dst, long long ld_dst, int rows,
                                   int cols, hb200_stream_t stream) {
  HB_CHECK_ARG(src && dst && rows > 0 && cols > 0 && ld_src >= cols && ld_dst >= rows, "transpose_f32: bad args");
  dim3 grid(cdiv(cols, 32), cdiv(rows, 32));
  transpose_f32_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(src, ld_src, dst, ld_dst, rows, cols);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

extern "C" int hb200_prep_plain(const uint8_t* rgb, const float* depth, const int32_t* frame_rows, int batch,
                                int height, int width, int c_rgb, int c_depth, hb200_bf16* out,
                                hb200_stream_t stream) {
  HB_CHECK_ARG(frame_rows && out && batch > 0 && c_rgb + c_depth > 0 && c_rgb + c_depth <= 8, "prep_plain: bad args");
  HB_CHECK_ARG((c_rgb == 0 || rgb) && (c_depth == 0 || depth), "prep_plain: missing sensor buffer");
  const long long total = (long long)batch * height * width;
  prep_plain_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>(rgb, depth, frame_rows,
                                                                            (long long)height * width, batch, c_rgb,
                                                                            c_depth, (act_t*)out);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}
extern "C" int hb200_relu_bias_bwd(const hb200_bf16* g, const hb200_bf16* out, hb200_bf16* dy, float* dbias,
                                   long long npix, int channels, hb200_stream_t stream) {
  HB_CHECK_ARG(g && dbias && npix > 0 && channels % 8 == 0 && 256 % (channels / 8) == 0, "relu_bias_bwd: bad args");
  int grid = (int)((npix + 255) / 256);
  if (grid > kNumSMs * 8) grid = kNumSMs * 8;
  if (grid < 1) grid = 1;
  cudaStream_t st = (cudaStream_t)stream;
  float* parts = nullptr;
  int* tickets = nullptr;
  const int rc = stream_workspace(st, (size_t)(grid + kReduceChunks) * channels, 0, &parts, &tickets);
  if (rc) return rc;
  relu_bias_bwd_kernel<<<grid, 256, 0, st>>>((const grad_t*)g, (const act_t*)out, out != nullptr, (grad_t*)dy, parts,
                                             npix, channels);
  HB_LAUNCH_OK();
  count_launch(1);
  return reduce_partials(parts, grid, channels, channels, dbias, parts + (size_t)grid * channels, st);
}
extern "C" int hb200_bf16_hwc_to_f32_chw(const hb200_bf16* x, float* out, int batch, int hw, int channels,
                                         hb200_stream_t stream) {
  HB_CHECK_ARG(x && out && batch > 0 && hw > 0 && channels % 8 == 0, "bf16_hwc_to_f32_chw: bad args");
  const long long total = (long long)batch * hw * (channels / 8);
  bf16_hwc_to_f32_chw_kernel<<<grid_for(total, 256), 256, 0, (cudaStream_t)stream>>>((const act_t*)x, out, batch, hw, channels);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

// ======================================================================================
// frozen-encoder learner: the minibatch's cached visual features (rollout rows frame_rows[f]) as one dense [B, F] matrix
// for the visual_fc GEMM (HB/rl/ddppo/policy/resnet_policy.py:631-645 reads observations["visual_features"])
// ======================================================================================
namespace hb200 {
__global__ void gather_rows_kernel(const float4* __restrict__ src, const int32_t* __restrict__ frame_rows,
                                   float4* __restrict__ out, int batch, long long vec_per_row) {
  const long long total = (long long)batch * vec_per_row;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long f = i / vec_per_row, j = i - f * vec_per_row;
    out[i] = __ldg(src + (long long)frame_rows[f] * vec_per_row + j);
  }
}
}  // namespace hb200

extern "C" int hb200_gather_rows(const float* src, const int32_t* frame_rows, float* out, int batch,
                                 long long row_elems, hb200_stream_t stream) {
  HB_CHECK_ARG(src && frame_rows && out && batch > 0 && row_elems > 0 && row_elems % 4 == 0 &&
               ((uintptr_t)src % 16) == 0 && ((uintptr_t)out % 16) == 0,
               "gather_rows: row_elems must be a positive multiple of 4 and both buffers 16-byte aligned");
  const long long vec = row_elems / 4;
  gather_rows_kernel<<<grid_for((long long)batch * vec, 256), 256, 0, (cudaStream_t)stream>>>(
      (const float4*)src, frame_rows, (float4*)out, batch, vec);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

// ======================================================================================
// VER learner: rows between the minibatch's frame order and the recurrence's time-major [T_max, S] layout
// ======================================================================================
namespace hb200 {
__global__ void gather_rows_pad_kernel(const float* __restrict__ src, long long ld_src, const int32_t* __restrict__ idx,
                                       float* __restrict__ out, long long ld_out, int rows, int cols) {
  const long long total = (long long)rows * cols;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / cols, c = i - r * cols;
    const int j = idx[r];
    out[r * ld_out + c] = j >= 0 ? __ldg(src + (long long)j * ld_src + c) : 0.f;
  }
}
}  // namespace hb200

extern "C" int hb200_gather_rows_pad(const float* src, long long ld_src, const int32_t* idx, float* out,
                                     long long ld_out, int rows, int cols, hb200_stream_t stream) {
  HB_CHECK_ARG(src && idx && out && rows > 0 && cols > 0 && ld_src >= cols && ld_out >= cols,
               "gather_rows_pad: bad args rows=%d cols=%d ld_src=%lld ld_out=%lld", rows, cols, ld_src, ld_out);
  gather_rows_pad_kernel<<<grid_for((long long)rows * cols, 256), 256, 0, (cudaStream_t)stream>>>(
      src, ld_src, idx, out, ld_out, rows, cols);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}
