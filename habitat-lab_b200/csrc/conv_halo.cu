// hb200 -- "halo" convolution kernels for the stride-1 layers that dominate the encoder's time
// (3x3 pad-1 convs of layer1/layer2, and the 7x7 stride-2 stem re-expressed as a 4x4 stride-1 conv
// over the space-to-depth input).
//
// The first-generation kernel (conv.cu) gathers an im2col tile per K chunk, so every input element
// crosses L2 -> shared memory 9 times (L2-bound, the tensor pipe mostly idle).  Here each CTA loads the
// (16+KH-1) x (8+KW-1) input halo of a 16x8 output tile ONCE into shared memory in the layout
//
//        offset(hy, cj, hx) = ((hy * C/8 + cj) * HW + hx) * 16 bytes        (16 B = 8 channels)
//
// and every filter tap is just a different wgmma shared-memory descriptor over that one buffer:
//   forward / dgrad (K-major A):  start = base + r*RP + s*16 + 2kk*P,  LBO = P (next 8 channels),
//                                 SBO = RP (next output row = next 8-pixel core-matrix group)
//   wgrad (MN-major A):           rows = (r, ci) with row-block stride P (because RP = C/8 * P the three
//                                 vertical taps are ONE affine M dimension), K = 16 pixels (2 tile rows)
// with P = HW*16, RP = (C/8)*P.  The no-swizzle descriptor mode is what makes this legal: shifting
// the start address by one pixel (16 B) keeps every core matrix 8 x 16 B contiguous.
//
// CTAs are persistent (weights stay resident across tiles); halo loads for tile i+1 (zero-filling
// cp.async or TMA: padding by predication / out-of-bounds fill) overlap the MMAs and the epilogue of tile i.
// One warpgroup owns the 128 x N accumulator of a tile in registers (wgmma.cuh).
#include <cuda.h>
#include <stdlib.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace hb200 {
void count_launch(int n);
using namespace wg;

constexpr int TH = 16, TW = 8;  // output tile: 16 rows x 8 cols = 128 pixels = MMA M

// transpose-reduce: each lane holds 16 partial sums v[i]; afterwards lane l holds the warp-wide sum of
// v[l >> 1] (16 shuffles).  Lanes 2i and 2i+1 hold the same value.
__device__ __forceinline__ float warp_reduce16(float (&v)[16], int lane) {
  float a[8], b[4], c[2];
  const bool b4 = lane & 16, b3 = lane & 8, b2 = lane & 4, b1 = lane & 2;
#pragma unroll
  for (int i = 0; i < 8; ++i) a[i] = (b4 ? v[i + 8] : v[i]) + __shfl_xor_sync(0xffffffffu, b4 ? v[i] : v[i + 8], 16);
#pragma unroll
  for (int i = 0; i < 4; ++i) b[i] = (b3 ? a[i + 4] : a[i]) + __shfl_xor_sync(0xffffffffu, b3 ? a[i] : a[i + 4], 8);
#pragma unroll
  for (int i = 0; i < 2; ++i) c[i] = (b2 ? b[i + 2] : b[i]) + __shfl_xor_sync(0xffffffffu, b2 ? b[i] : b[i + 2], 4);
  float d = (b1 ? c[1] : c[0]) + __shfl_xor_sync(0xffffffffu, b1 ? c[0] : c[1], 2);
  d += __shfl_xor_sync(0xffffffffu, d, 1);
  return d;
}

// lane l ends with the warp sum of v[l] (31 shuffles for 32 values)
__device__ __forceinline__ float halo_warp_reduce32(float (&v)[32], int lane) {
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

// GroupNorm sums of one 32-channel chunk of a 128-pixel tile (one warp = 32 pixels): per-pixel group partials first
// (channels of a group are adjacent), then ONE transpose-reduce over sums and squares together -- 31 shuffles for
// 2-channel groups, 16 for 4-channel groups, instead of two 16-value trees per chunk.
// stats_b = stats + b * groups * 2; ch0 = first channel of the chunk.
__device__ __forceinline__ void halo_gn_stats_chunk(const float (&acc)[32], int lane, int cpg, double* stats_b, int ch0) {
  if (cpg == 2) {
    float v[32];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      v[i] = acc[2 * i] + acc[2 * i + 1];
      v[16 + i] = acc[2 * i] * acc[2 * i] + acc[2 * i + 1] * acc[2 * i + 1];
    }
    const float t = halo_warp_reduce32(v, lane);   // lane < 16: sum of group lane; else sum of squares of group lane-16
    atomicAdd(stats_b + ((ch0 >> 1) + (lane & 15)) * 2 + (lane >> 4), (double)t);
  } else if (cpg == 4) {
    float v[16];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float a0 = acc[4 * i], a1 = acc[4 * i + 1], a2 = acc[4 * i + 2], a3 = acc[4 * i + 3];
      v[i] = (a0 + a1) + (a2 + a3);
      v[8 + i] = (a0 * a0 + a1 * a1) + (a2 * a2 + a3 * a3);
    }
    const float t = warp_reduce16(v, lane);        // lanes 2i, 2i+1 hold value i
    if ((lane & 1) == 0) {
      const int i = lane >> 1;
      atomicAdd(stats_b + ((ch0 >> 2) + (i & 7)) * 2 + (i >> 3), (double)t);
    }
  } else {
    float s2[16], q2[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      s2[i] = acc[2 * i] + acc[2 * i + 1];
      q2[i] = acc[2 * i] * acc[2 * i] + acc[2 * i + 1] * acc[2 * i + 1];
    }
    const float ts = warp_reduce16(s2, lane), tq = warp_reduce16(q2, lane);
    if ((lane & 1) == 0) {
      double* dst = stats_b + ((ch0 + lane) / cpg) * 2;
      atomicAdd(dst, (double)ts);
      atomicAdd(dst + 1, (double)tq);
    }
  }
}

struct HaloArgs {
  const __nv_bfloat16* x;      // [B,H,W,C] input of the conv (x for fwd, dy for dgrad)
  const __nv_bfloat16* wimg;   // [taps][C/8][N][8] weight image (K-major no-swizzle per tap)
  __nv_bfloat16* y;            // [B,H,W,N]
  const __nv_bfloat16* addend; // dgrad residual add, or nullptr
  double* stats;               // [B,G,2] or nullptr (double accumulators: run-to-run identical)
  int B, H, W, gn_groups, ntiles;
};

template <int C, int N, int KH, int KW, int PAD>
struct HaloCfg {
  static constexpr int CJ = C / 8;
  static constexpr int HH = TH + KH - 1, HWD = TW + KW - 1;
  static constexpr int P = HWD * 16;            // bytes between channel chunks
  static constexpr int RP = CJ * P;             // bytes between halo rows
  static constexpr int HALO_BYTES = HH * RP;
  static constexpr int W_BYTES = KH * KW * C * N * 2;
  // Halo stages per CTA.  Two stages let one CTA overlap the next tile's loads with the current MMAs, but for
  // C = N = 64 (72 KB of resident weights) that footprint (120 KB) leaves a single 128-thread CTA per SM: latency-bound.
  // One stage (97 KB) fits two CTAs per SM, which overlap each other instead.
  static constexpr int NBUF = (W_BYTES + 2 * HALO_BYTES > 110 * 1024) ? 1 : 2;
};

// issue the zero-filling loads of one halo tile (all 128 threads participate)
template <int C, int KH, int KW, int PAD, int ROWS>
__device__ __forceinline__ void load_halo(const __nv_bfloat16* __restrict__ x, uint32_t sdst, int b, int oh0,
                                          int ow0, int H, int W) {
  constexpr int CJ = C / 8, HWD = TW + KW - 1;
  constexpr int NV = ROWS * CJ * HWD;
  for (int v = threadIdx.x; v < NV; v += 128) {
    const int cj = v % CJ;  // channel chunk fastest: CJ consecutive threads read one pixel's C*2 contiguous bytes
    const int t = v / CJ;
    const int hx = t % HWD, hy = t / HWD;
    const int ih = oh0 - PAD + hy, iw = ow0 - PAD + hx;
    const bool ok = ih >= 0 && ih < H && iw >= 0 && iw < W;
    const __nv_bfloat16* g = ok ? x + (((size_t)b * H + ih) * W + iw) * C + cj * 8 : x;
    cp_async16(sdst + (uint32_t)(((hy * CJ + cj) * HWD + hx) * 16), g, ok);
  }
}

// Register-staged variant of load_halo for the weight-gradient kernels: coalesced LDG.128 (consecutive lanes walk the
// channel chunks of consecutive pixels of a halo row = contiguous global bytes) into registers, later STS.128 into the
// shifted-descriptor layout (bank-conflict free per 8-lane phase).  As LDGSTS the same copies cost 2 shared-memory
// wavefronts per lane; staged through registers they cost ~8x fewer LSU cycles, and the
// global latency hides behind the wait for the previous tile's MMAs.
template <int C, int KH, int KW, int PAD, int ROWS, int NTHR>
struct HaloRegs {
  static constexpr int CJ = C / 8, HWD = TW + KW - 1;
  static constexpr int NV = ROWS * CJ * HWD;
  static constexpr int PER = (NV + NTHR - 1) / NTHR;
  uint4 v[PER];
  __device__ __forceinline__ void load(const __nv_bfloat16* __restrict__ x, int lt, int b, int oh0, int ow0, int H, int W) {
#pragma unroll
    for (int i = 0; i < PER; ++i) {
      const int idx = lt + i * NTHR;
      uint4 r = make_uint4(0u, 0u, 0u, 0u);
      if (idx < NV) {
        const int cj = idx % CJ;
        const int t = idx / CJ;
        const int hx = t % HWD, hy = t / HWD;
        const int ih = oh0 - PAD + hy, iw = ow0 - PAD + hx;
        if (ih >= 0 && ih < H && iw >= 0 && iw < W)
          r = __ldg(reinterpret_cast<const uint4*>(x + (((size_t)b * H + ih) * W + iw) * C + cj * 8));
      }
      v[i] = r;
    }
  }
  __device__ __forceinline__ void store(uint32_t sdst, int lt) const {
#pragma unroll
    for (int i = 0; i < PER; ++i) {
      const int idx = lt + i * NTHR;
      if (idx < NV) {
        const int cj = idx % CJ;
        const int t = idx / CJ;
        const int hx = t % HWD, hy = t / HWD;
        asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(sdst + (uint32_t)(((hy * CJ + cj) * HWD + hx) * 16)),
                     "r"(v[i].x), "r"(v[i].y), "r"(v[i].z), "r"(v[i].w) : "memory");
      }
    }
  }
};

template <int C, int N, int KH, int KW, int PAD, int MODE>  // MODE 0: fwd (+stats), 1: dgrad (+addend)
__global__ void __launch_bounds__(128) conv_halo_kernel(const HaloArgs a) {
  using Cfg = HaloCfg<C, N, KH, KW, PAD>;
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __shared__ float stage_buf[kStageFloats];
  const uint32_t sbase = (smem_u32(smem_raw) + 127u) & ~127u;
  const uint32_t s_w = sbase;
  const uint32_t s_halo0 = s_w + Cfg::W_BYTES;
  const int tid = threadIdx.x, lane = tid & 31;

  // weights: resident for the CTA's whole life
  {
    const uint4* src = reinterpret_cast<const uint4*>(a.wimg);
    for (int v = tid; v < Cfg::W_BYTES / 16; v += 128) cp_async16(s_w + (uint32_t)v * 16, src + v, true);
  }
  const int tiles_x = a.W / TW, tiles_y = a.H / TH;
  const int tiles_per_img = tiles_x * tiles_y;
  auto tile_coords = [&](int tile, int& b, int& oh0, int& ow0) {
    b = tile / tiles_per_img;
    const int r = tile - b * tiles_per_img;
    oh0 = (r / tiles_x) * TH;
    ow0 = (r % tiles_x) * TW;
  };
  const int first = blockIdx.x, stride = gridDim.x;
  const int my_n = first < a.ntiles ? (a.ntiles - first + stride - 1) / stride : 0;
  if (my_n > 0) {
    int b, oh0, ow0;
    tile_coords(first, b, oh0, ow0);
    load_halo<C, KH, KW, PAD, Cfg::HH>(a.x, s_halo0, b, oh0, ow0, a.H, a.W);
  }
  cp_async_commit();  // group 0: weights + first halo
  // forward: fp16 input halo x fp16 weight image; dgrad: bf16 gradients x bf16 flipped / transposed image
  constexpr int kT = MODE == 0 ? kF16 : kBF16;
  float acc_t[N];

  const int py = tid >> 3, px = tid & 7;  // this thread's output pixel within the tile (epilogue)

  constexpr int NBUF = Cfg::NBUF;
  for (int it = 0; it < my_n; ++it) {
    if (NBUF == 2) {
      // prefetch the halo of tile it+1 into the stage tile it-1 used (its MMAs completed in the last iteration)
      if (it + 1 < my_n) {
        int b, oh0, ow0;
        tile_coords(first + (it + 1) * stride, b, oh0, ow0);
        load_halo<C, KH, KW, PAD, Cfg::HH>(a.x, s_halo0 + ((it + 1) & 1) * Cfg::HALO_BYTES, b, oh0, ow0, a.H, a.W);
      }
      cp_async_commit();
    }
    // halo of tile it has landed -> its MMAs
    if (NBUF == 2) cp_async_wait<1>(); else cp_async_wait<0>();
    fence_proxy_async_smem();
    __syncthreads();
    {
      const uint32_t sh = s_halo0 + (NBUF == 2 ? (it & 1) : 0) * Cfg::HALO_BYTES;
      wgmma_fence();
      uint32_t accum = 0;
#pragma unroll
      for (int r = 0; r < KH; ++r)
#pragma unroll
        for (int s = 0; s < KW; ++s)
#pragma unroll
          for (int kk = 0; kk < C / 16; ++kk) {
            const uint64_t da = make_smem_desc(sh + r * Cfg::RP + s * 16 + 2 * kk * Cfg::P, Cfg::P, Cfg::RP, kNoSwizzle);
            const uint64_t db = make_smem_desc(s_w + (r * KW + s) * (C * N * 2) + 2 * kk * (N * 16), N * 16, 128, kNoSwizzle);
            mma128<N, kT>(acc_t, da, 8 * Cfg::RP, db, accum);
            accum = 1;
          }
      wgmma_commit();
      wgmma_wait<0>();
      acc_fence(acc_t);
    }
    // single halo stage: the MMAs of tile it have consumed it -> the next tile loads during this epilogue
    if (NBUF == 1) {
      if (it + 1 < my_n) {
        int b, oh0, ow0;
        tile_coords(first + (it + 1) * stride, b, oh0, ow0);
        load_halo<C, KH, KW, PAD, Cfg::HH>(a.x, s_halo0, b, oh0, ow0, a.H, a.W);
      }
      cp_async_commit();
    }
    {   // epilogue of tile it
      int b, oh0, ow0;
      tile_coords(first + it * stride, b, oh0, ow0);
      const size_t pix = ((size_t)b * a.H + oh0 + py) * a.W + ow0 + px;
#pragma unroll
      for (int col0 = 0; col0 < N; col0 += 32) {
        float acc[32];
        acc_row32(acc_t, col0, stage_buf, acc);
        if (MODE == 0 && a.stats != nullptr) {
          // per (frame, group) sum / sum-of-squares of this 32-column slab over the warp's 32 pixels:
          // pairwise channel sums, then a transpose-reduce (16 + 16 shuffles instead of 2 x 16 x 5)
          const int cpg = N / a.gn_groups;
          float s2[16], q2[16];
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            s2[i] = acc[2 * i] + acc[2 * i + 1];
            q2[i] = acc[2 * i] * acc[2 * i] + acc[2 * i + 1] * acc[2 * i + 1];
          }
          const float ts = warp_reduce16(s2, lane), tq = warp_reduce16(q2, lane);  // lane l: channel pair l >> 1
          if ((lane & 1) == 0) {
            const int ch = col0 + lane;  // first channel of the pair
            double* dst = a.stats + ((size_t)b * a.gn_groups + ch / cpg) * 2;
            atomicAdd(dst, (double)ts);
            atomicAdd(dst + 1, (double)tq);
          }
        }
        const size_t o = pix * N + col0;
        if (MODE == 1 && a.addend != nullptr) {
          const uint4* ad = reinterpret_cast<const uint4*>(a.addend + o);
#pragma unroll
          for (int v = 0; v < 4; ++v) {
            float f[8];
            unpack8(ad[v], f);
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[v * 8 + e] += f[e];
          }
        }
        uint4* dst = reinterpret_cast<uint4*>(a.y + o);
#pragma unroll
        for (int v = 0; v < 4; ++v) {
          uint4 u;
          if (MODE == 0) {  // forward output y: fp16 (saturating)
            u.x = pack_f16x2(acc[v * 8 + 0], acc[v * 8 + 1]);
            u.y = pack_f16x2(acc[v * 8 + 2], acc[v * 8 + 3]);
            u.z = pack_f16x2(acc[v * 8 + 4], acc[v * 8 + 5]);
            u.w = pack_f16x2(acc[v * 8 + 6], acc[v * 8 + 7]);
          } else {          // data gradient: bf16
            u.x = pack_bf16x2(acc[v * 8 + 0], acc[v * 8 + 1]);
            u.y = pack_bf16x2(acc[v * 8 + 2], acc[v * 8 + 3]);
            u.z = pack_bf16x2(acc[v * 8 + 4], acc[v * 8 + 5]);
            u.w = pack_bf16x2(acc[v * 8 + 6], acc[v * 8 + 7]);
          }
          dst[v] = u;
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// weight gradient on the same halo buffer.  rows = (r, ci) [vertical taps form one affine M dim],
// one accumulator per horizontal tap s and per 128-row M tile; K = output pixels.
// ------------------------------------------------------------------------------------------
// ring depth of conv_halo_wgrad_kernel: 4 stages where they fit beside the 17 KB accumulator transpose buffer, else 3
constexpr int halo_wgrad_stages(int xmode, int c, int stage_bytes) {
  return (xmode != 0 && c >= 64) ? (4 * stage_bytes <= 200 * 1024 ? 4 : 3) : 2;
}

struct HaloWgradArgs {
  const __nv_bfloat16* x;   // [B,H,W,C]
  const __nv_bfloat16* dy;  // [B,H,W,N]
  float* dw;                // partials [blockIdx.x][(r*KW+s)*C + ci][N], summed in order by reduce_partials
  int B, H, W, ntiles;
};

// XMODE: how the x halo reaches shared memory.  0 = registers / cp.async (below).  1 = one 5-D TMA box over x viewed as
// [B, H, C/8, W, 8] (box = 8 channels x HWD pixels x C/8 chunks x halo rows = exactly the [row][chunk][pixel] layout the
// shifted descriptors read).  2 = the same over the 2x2 SPACE-TO-DEPTH view of a tensor with C/4 real channels: a
// 3x3 stride-2 pad-1 conv of x is a 2x2 stride-1 pad-1 conv of the view (csrc/conv_s2.cu), whose block row `by` is image
// rows 2by, 2by+1 -- the box simply covers twice the rows of the real tensor with (dx, c) as the chunk dimension.
template <int C, int N, int KH, int KW, int PAD, int XMODE = 0>
__global__ void __launch_bounds__(128)
conv_halo_wgrad_kernel(const HaloWgradArgs a, const __grid_constant__ CUtensorMap tmap_dy,
                       const __grid_constant__ CUtensorMap tmap_x) {
  constexpr int CJ = C / 8, HWD = TW + KW - 1;
  constexpr int P = HWD * 16, RP = CJ * P;
  constexpr int MT = (KH * CJ + 15) / 16;                  // 128-row M tiles over the (r, cj) row blocks
  constexpr int RMAX = (MT * 16 + CJ - 1) / CJ;            // vertical taps addressed incl. padding rows
  constexpr int HROWS = TH - 1 + RMAX;                     // halo rows that descriptors may touch
  constexpr int HROWS_LOAD = TH + KH - 1;                  // rows that hold real data
  constexpr int HALO_BYTES = HROWS * RP;
  constexpr int DY_BYTES = 128 * N * 2;                    // [pixel][N channels]: one swizzled row per pixel (TMA)
  constexpr int STAGE = (DY_BYTES + HALO_BYTES + 1023) / 1024 * 1024;   // dy tile first: swizzle atoms need 1024-byte alignment
  // Ring depth.  With the x halo AND the dy tile arriving by TMA, two stages expose the load latency of a tile once per
  // tile (its MMAs are much shorter): the wide configurations, one CTA per SM anyway (shared memory), prefetch NSW-1 tiles
  // ahead; the 32-channel layers and the stem keep two stages and more CTAs per SM instead.
  constexpr int NSW = halo_wgrad_stages(XMODE, C, STAGE);
  // accumulators (s, mt) of 128 rows x N: a CTA holds APC of them in registers (<= 128 columns), blockIdx.y picks the group
  constexpr int NACC = KW * MT;
  constexpr int APC = NACC * N <= 128 ? NACC : 128 / N;
  static_assert(NACC % APC == 0, "accumulator groups");
  static_assert(N == 32 || N == 64, "dy rows are 64 / 128 bytes: SWIZZLE_64B / SWIZZLE_128B");
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t dy_bar[NSW];
  __shared__ float stage_buf[kStageFloats];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const int tid = threadIdx.x;
  const int grp = blockIdx.y;
  const CUtensorMap* const tmap_p = &tmap_dy;   // param-space address (never through a by-reference lambda capture)
  const CUtensorMap* const tmap_xp = &tmap_x;

  if (tid == 0) {
#pragma unroll
    for (int i = 0; i < NSW; ++i) mbar_init(&dy_bar[i], 1);
    mbar_fence_init();
  }
  // the padding halo rows are read by the (discarded) padding M rows: keep them finite
  for (int st = 0; st < NSW; ++st)
    for (int v = tid; v < (HROWS - HROWS_LOAD) * RP / 16; v += 128) {
      const uint32_t addr = sbase + st * STAGE + DY_BYTES + HROWS_LOAD * RP + v * 16;
      asm volatile("st.shared.v4.b32 [%0], {%1,%1,%1,%1};" ::"r"(addr), "r"(0u) : "memory");
    }
  const int tiles_x = a.W / TW, tiles_y = a.H / TH, tiles_per_img = tiles_x * tiles_y;
  auto tile_coords = [&](int tile, int& b, int& oh0, int& ow0) {
    b = tile / tiles_per_img;
    const int r = tile - b * tiles_per_img;
    oh0 = (r / tiles_x) * TH;
    ow0 = (r % tiles_x) * TW;
  };
  // x halo: zero-filling cp.async into the shifted-descriptor layout (all threads).  dy tile: ONE TMA box (N channels x
  // 8 x 16 pixels) into the MN-major swizzled layout -- as LDGSTS it was a transpose (pixel-major tensor -> channel-chunk-
  // major rows), 2 shared-memory wavefronts per 16-byte copy, which made this kernel LSU-bound (see the small-image
  // kernel below).
  // Register staging pays while the halo is <= 8 vectors per thread (C <= 32, the stem); for C = 64 (12 vectors, 128
  // registers) the lost occupancy costs more than the LDGSTS wavefronts: cp.async there.
  constexpr bool kRegStage = XMODE == 0 && HROWS_LOAD * CJ * HWD <= 128 * 8;
  HaloRegs<C, KH, KW, PAD, kRegStage ? HROWS_LOAD : 1, 128> xr;   // the x halo of the NEXT tile, in flight in registers
  auto fetch_x = [&](int tile) {
    if (!kRegStage) return;
    int b, oh0, ow0;
    tile_coords(tile, b, oh0, ow0);
    xr.load(reinterpret_cast<const __nv_bfloat16*>(a.x), tid, b, oh0, ow0, a.H, a.W);
  };
  auto commit_tile = [&, tmap_p, tmap_xp](int tile, int st) {   // stage `st` is free: x halo -> smem, dy tile by TMA
    int b, oh0, ow0;
    tile_coords(tile, b, oh0, ow0);
    const uint32_t sd = sbase + st * STAGE;
    if (XMODE == 0) {
      if (kRegStage) xr.store(sd + DY_BYTES, tid);
      else load_halo<C, KH, KW, PAD, HROWS_LOAD>(a.x, sd + DY_BYTES, b, oh0, ow0, a.H, a.W);
    }
    if (tid == 0) {
      mbar_expect_tx(&dy_bar[st], (uint32_t)(DY_BYTES + (XMODE ? HROWS_LOAD * RP : 0)));
      tma_load_4d(sd, tmap_p, &dy_bar[st], 0, ow0, oh0, b);
      // coordinates (channel-in-chunk, pixel column, chunk, row, frame); space-to-depth: rows of the REAL tensor
      if (XMODE == 1) tma_load_5d(sd + DY_BYTES, tmap_xp, &dy_bar[st], 0, ow0 - PAD, 0, oh0 - PAD, b);
      if (XMODE == 2) tma_load_5d(sd + DY_BYTES, tmap_xp, &dy_bar[st], 0, ow0 - PAD, 0, 2 * (oh0 - PAD), b);
    }
  };
  const int first = blockIdx.x, stride = gridDim.x;
  const int my_n = first < a.ntiles ? (a.ntiles - first + stride - 1) / stride : 0;
  if (XMODE == 0 && my_n > 0) {
    fetch_x(first);
    commit_tile(first, 0);
  }
  cp_async_commit();
  fence_proxy_async_smem();
  __syncthreads();
  // A = bf16 twin of the forward activations (halo), B = output gradients (bf16); mixed fp16 x bf16 is not legal
  float acc_w[APC][N];
  auto mma_tile = [&](int it, uint32_t sd) {   // all 128 threads; returns with the MMAs complete
    const uint32_t sh = sd + DY_BYTES;
    wgmma_fence();
#pragma unroll
    for (int l = 0; l < APC; ++l) {
      const int ai = grp * APC + l, s = ai / MT, mt = ai % MT;
#pragma unroll
      for (int ks = 0; ks < TH / 2; ++ks) {
        // A: M = row blocks (stride P), K = 16 pixels = tile rows 2ks, 2ks+1 (stride RP)
        const uint64_t da = make_smem_desc(sh + 2 * ks * RP + s * 16 + mt * 16 * P, RP, P, kNoSwizzle);
        // B: MN-major swizzled rows (one pixel = N channels = 64 / 128 bytes); K16 = 2 groups of 8 rows
        const uint64_t db = make_smem_desc(sd + ks * (16 * N * 2), 0, 8 * N * 2, N == 64 ? kSwizzle128B : kSwizzle64B);
        mma128<N, kBF16, 1, 1>(acc_w[l], da, 8 * P, db, (it > 0 || ks > 0) ? 1u : 0u);
      }
    }
    wgmma_commit();
    wgmma_wait<0>();
  };

  if (XMODE != 0) {
    // both operands by TMA: thread 0 keeps NSW-1 tiles of loads ahead of the tensor core
    if (tid == 0)
      for (int p = 0; p < NSW - 1 && p < my_n; ++p) commit_tile(first + p * stride, p);
    for (int it = 0; it < my_n; ++it) {
      const int nxt = it + NSW - 1;   // its stage was read by the MMAs of tile it-1, complete
      if (tid == 0 && nxt < my_n) commit_tile(first + nxt * stride, nxt % NSW);
      mbar_wait(&dy_bar[it % NSW], (it / NSW) & 1);
      mma_tile(it, sbase + (it % NSW) * STAGE);
    }
  } else {
    for (int it = 0; it < my_n; ++it) {
      const bool more = it + 1 < my_n;
      if (more) fetch_x(first + (it + 1) * stride);                 // global loads in flight ...
      if (more) commit_tile(first + (it + 1) * stride, (it + 1) & 1);   // ... into the stage tile it-1 used
      cp_async_commit();
      cp_async_wait<1>();         // cp.async variant: this thread's copies of tile it (issued an iteration ago)
      fence_proxy_async_smem();   // st.shared / cp.async (generic proxy) -> wgmma (async proxy)
      __syncthreads();
      mbar_wait(&dy_bar[it & 1], (it >> 1) & 1);   // the TMA'd dy tile
      mma_tile(it, sbase + (it & 1) * STAGE);
    }
  }
  {   // a worker without tiles still writes its (zero) partial
#pragma unroll
    for (int l = 0; l < APC; ++l) {
      if (my_n == 0) {
#pragma unroll
        for (int j = 0; j < N; ++j) acc_w[l][j] = 0.f;
      }
      acc_fence(acc_w[l]);
      const int ai = grp * APC + l, s = ai / MT, mt = ai % MT;
      const int blk = mt * 16 + (tid >> 3);       // row block (r, cj)
      const int r = blk / CJ, cj = blk % CJ;
      const bool ok = r < KH;
      const size_t row = (size_t)(r * KW + s) * C + cj * 8 + (tid & 7);
#pragma unroll
      for (int col0 = 0; col0 < N; col0 += 32) {
        float rr[32];
        acc_row32(acc_w[l], col0, stage_buf, rr);
        if (ok) {
          float* dst = a.dw + ((size_t)blockIdx.x * (KH * KW * C) + row) * N + col0;
#pragma unroll
          for (int j = 0; j < 32; j += 4) *reinterpret_cast<float4*>(dst + j) = make_float4(rr[j], rr[j + 1], rr[j + 2], rr[j + 3]);
        }
      }
    }
  }
}


// ------------------------------------------------------------------------------------------
// weight gradient of the 3x3 pad-1 stride-1 convs on SMALL images (8x8: layer3, 4x4: layer4 / compression).
// The gather kernel (conv.cu) re-reads x once per tap and dy once per 128-row M tile through L2 (1.2 GB per launch
// for a 128->128 layer: L2-gather-bound, far below the tensor roofline).  Here the halo scheme of the kernel above
// is applied to a tile made of SEVERAL images: a 16x8 output tile = 16/IMG images stacked vertically, each with its
// own zero-padding rows in the halo buffer (and, for 4x4 images, 4 zero "virtual" pixels per 8-pixel row whose dy is
// zero), so x is loaded once per (channel slice) and every tap is a shifted descriptor.  Channels are sliced to keep
// the accumulator in registers: a CTA owns 32 input channels (the three vertical taps x 32 channels = 96 rows of
// one M = 128 tile), NS output channels and ONE horizontal tap s (a 128 x NS accumulator).
// grid = (tile workers, Ci/32 * Co/NS slices x 3 taps); results are accumulated into dw with vector red.add.
// ------------------------------------------------------------------------------------------
constexpr int kSmallWgradStages = 3;
struct HaloWgradSmallArgs {
  const grad_t* x;    // [B, IMG, IMG, Ci]  bf16 twin of the forward activation
  const grad_t* dy;   // [B, IMG, IMG, Co]  bf16
  float* dw;          // partials [blockIdx.x][(r*3+s)*Ci + ci][Co], summed in order by reduce_partials
  int B, Ci, Co, ntiles;
};

template <int NS, int IMG>
__global__ void __launch_bounds__(128)
conv_halo_wgrad_small_kernel(const HaloWgradSmallArgs a, const __grid_constant__ CUtensorMap tmap_dy) {
  constexpr int CJ = 4, KH = 3, KW = 3, HWD = TW + KW - 1;
  constexpr int P = HWD * 16, RP = CJ * P;
  constexpr int IPT = TH / IMG;                 // images per 16-row tile
  constexpr int RPI = IMG + 2;                  // halo rows per image (own top / bottom padding row)
  constexpr int HROWS_LOAD = IPT * RPI;
  constexpr int HROWS = (IPT - 1) * RPI + (IMG - 2) + 1 + 4;   // last K16 base row + second K8 row + 4 row blocks (M padding)
  constexpr int HROWS_A = HROWS > HROWS_LOAD ? HROWS : HROWS_LOAD;
  constexpr int HALO_BYTES = (HROWS_A * RP + 1023) / 1024 * 1024;   // the dy tile behind it must be 1024-byte aligned
  constexpr int NB = NS / 64;                   // 64-channel (128-byte) column blocks of the dy tile
  constexpr int DY_BYTES = NB * 128 * 128;      // [block][pixel][128 B], TMA SWIZZLE_128B
  constexpr int STAGE = HALO_BYTES + DY_BYTES;
  constexpr int NST = kSmallWgradStages;        // 3-deep ring: the loads of tile it+2 overlap the MMAs of tiles it, it+1
  static_assert(NS <= 128, "one 128 x NS accumulator per CTA");
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t dy_bar[NST];
  __shared__ float stage_buf[kStageFloats];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const int tid = threadIdx.x, warp = tid >> 5;
  const int nsl = a.Co / NS;
  const int s_tap = blockIdx.y % KW, slice = blockIdx.y / KW;   // horizontal tap of this CTA's accumulator
  const int c_off = (slice / nsl) * 32, n_off = (slice % nsl) * NS;
  const CUtensorMap* const tmap_p = &tmap_dy;   // param-space address (see conv_halo_tma_kernel)

  if (tid == 0) {
#pragma unroll
    for (int i = 0; i < NST; ++i) mbar_init(&dy_bar[i], 1);
    mbar_fence_init();
  }
  // rows beyond the loaded ones are read by the (discarded) padding M rows: keep them finite
  for (int st = 0; st < NST; ++st)
    for (int v = tid; v < (HROWS_A - HROWS_LOAD) * RP / 16; v += 128) {
      const uint32_t addr = sbase + st * STAGE + HROWS_LOAD * RP + v * 16;
      asm volatile("st.shared.v4.b32 [%0], {%1,%1,%1,%1};" ::"r"(addr), "r"(0u) : "memory");
    }
  // Operand traffic.  In an all-cp.async version every LDGSTS of the dy tile costs 64 shared-memory wavefronts
  // (ideal 8) -- a 16-byte copy only coalesces with its neighbours when 8 lanes are contiguous in BOTH global and
  // shared memory, and the MN-major no-swizzle layout ([channel chunk][pixel][16 B]) is a transpose of the pixel-major
  // tensor; 5700 LSU cycles per tile against 1536 tensor cycles.  The dy tile now arrives by TMA (box = 64 channels x
  // 8 x IMG x IPT pixels, hardware 128-byte swizzle = the MN-major SWIZZLE_128B operand layout; for 4x4 images the box
  // is 8 wide and the 4 out-of-range columns are the zero "virtual pixels"): zero LSU work, one thread.  Warps 1-3
  // keep loading the x halo with cp.async (its shifted-descriptor layout has no TMA box form).
  // x halo: LDG.128 into registers (4 lanes = the 64 bytes of one pixel's channel slice, consecutive pixels follow),
  // later STS.128 into the shifted-descriptor layout -- 8x fewer LSU cycles than the same copies as LDGSTS
  constexpr int XV = HROWS_LOAD * CJ * HWD, XPER = (XV + 95) / 96;
  uint4 xr[XPER];
  auto fetch_x = [&](int tile) {
    if (warp == 0) return;
    const int lt = tid - 32;
    const int b0 = tile * IPT;
#pragma unroll
    for (int i = 0; i < XPER; ++i) {
      const int v = lt + i * 96;
      uint4 r = make_uint4(0u, 0u, 0u, 0u);
      if (v < XV) {
        const int cj = v % CJ;
        const int t = v / CJ;
        const int hx = t % HWD, hy = t / HWD;
        const int j = hy / RPI, ih = hy - j * RPI - 1, iw = hx - 1;
        const int b = b0 + j;
        if (b < a.B && ih >= 0 && ih < IMG && iw >= 0 && iw < IMG)
          r = __ldg(reinterpret_cast<const uint4*>(a.x + ((((size_t)b * IMG + ih) * IMG + iw) * a.Ci + c_off + cj * 8)));
      }
      xr[i] = r;
    }
  };
  auto store_x = [&](int st) {
    if (warp == 0) return;
    const int lt = tid - 32;
    const uint32_t sh = sbase + st * STAGE;
#pragma unroll
    for (int i = 0; i < XPER; ++i) {
      const int v = lt + i * 96;
      if (v < XV) {
        const int cj = v % CJ;
        const int t = v / CJ;
        const int hx = t % HWD, hy = t / HWD;
        asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(sh + (uint32_t)(((hy * CJ + cj) * HWD + hx) * 16)),
                     "r"(xr[i].x), "r"(xr[i].y), "r"(xr[i].z), "r"(xr[i].w) : "memory");
      }
    }
  };
  auto load_dy = [&, tmap_p](int tile, int st) {   // thread 0 only
    const uint32_t sd = sbase + st * STAGE + HALO_BYTES;
    mbar_expect_tx(&dy_bar[st], (uint32_t)DY_BYTES);
#pragma unroll
    for (int nb = 0; nb < NB; ++nb)
      tma_load_4d(sd + (uint32_t)nb * (128 * 128), tmap_p, &dy_bar[st], n_off + nb * 64, 0, 0, tile * IPT);
  };
  const int first = blockIdx.x, stride = gridDim.x;
  const int my_n = first < a.ntiles ? (a.ntiles - first + stride - 1) / stride : 0;
  // prologue: tiles 0 .. NST-2 staged
#pragma unroll
  for (int i = 0; i < NST - 1; ++i) {
    if (i < my_n) {
      fetch_x(first + i * stride);
      store_x(i);
      if (tid == 0) load_dy(first + i * stride, i);
    }
  }
  fence_proxy_async_smem();
  __syncthreads();
  float acc_t[NS];

  for (int it = 0; it < my_n; ++it) {
    const int st = it % NST;
    const int nt = it + NST - 1;     // the tile that will refill the stage tile it-1 used
    if (nt < my_n) fetch_x(first + nt * stride);   // its x halo: global loads in flight from here on
    fence_proxy_async_smem();        // x halo of tile it was stored (st.shared) an iteration ago
    __syncthreads();
    mbar_wait(&dy_bar[st], (it / NST) & 1);   // the TMA'd dy tile
    {
      const uint32_t sh = sbase + st * STAGE;
      const uint32_t sd = sh + HALO_BYTES;
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < TH / 2; ++ks) {
        // K16 = tile rows 2ks, 2ks+1 (never straddle an image: IMG is even) -> halo rows hb, hb+1 (+ tap r in M)
        const int hb = ((2 * ks) / IMG) * RPI + (2 * ks) % IMG;
        const uint64_t da = make_smem_desc(sh + hb * RP + s_tap * 16, RP, P, kNoSwizzle);
        // B: MN-major, 128-byte swizzle: rows = pixels (K), 128 B = 64 channels; K16 = 2 groups of 8 rows (1024 B each);
        // LBO = next 64-channel block (128 rows x 128 B), SBO = next 8-row group
        const uint64_t db = make_smem_desc(sd + ks * 2048, 128 * 128, 1024, kSwizzle128B);
        mma128<NS, kBF16, 1, 1>(acc_t, da, 8 * P, db, (it > 0 || ks > 0) ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<0>();
    }
    // refill the stage tile it-1 used (its MMAs are complete) with tile it+NST-1
    if (nt < my_n) {
      store_x(nt % NST);
      if (tid == 0) load_dy(first + nt * stride, nt % NST);
    }
  }
  {   // a worker without tiles still writes its (zero) partial
    if (my_n == 0) {
#pragma unroll
      for (int j = 0; j < NS; ++j) acc_t[j] = 0.f;
    }
    acc_fence(acc_t);
    const int blk = tid >> 3;                  // row block (r, cj)
    const int r = blk / CJ, cj = blk % CJ;
    const bool ok = r < KH;
    const size_t row = (size_t)(r * KW + s_tap) * a.Ci + c_off + cj * 8 + (tid & 7);
#pragma unroll
    for (int col0 = 0; col0 < NS; col0 += 32) {
      float rr[32];
      acc_row32(acc_t, col0, stage_buf, rr);
      if (ok) {
        float* dst = a.dw + ((size_t)blockIdx.x * 9 * a.Ci + row) * a.Co + n_off + col0;
#pragma unroll
        for (int j = 0; j < 32; j += 4) *reinterpret_cast<float4*>(dst + j) = make_float4(rr[j], rr[j + 1], rr[j + 2], rr[j + 3]);
      }
    }
  }
}

// ---- weight image for the halo kernels: [tap][C/8][N][8] bf16 ---------------------------------
// mode 0 forward: img[t=(r,s)][ci][n=co] = W[co][ci][r][s]
// mode 1 dgrad  : img[t=(r,s)][k=co][n=ci] = W[co][ci][KH-1-r][KW-1-s]     (flipped taps, transposed)
// mode 2 stem   : 7x7 stride-2 conv as 4x4 stride-1 over space-to-depth input (channel = (dy*2+dx)*4 + c,
//                 c < 4 with zero padding above ci_real): img[(a,b)][(dy,dx,c)][co] = W[co][c][2a+dy-1][2b+dx-1]
__global__ void pack_halo_weight_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ img, int KH,
                                        int KW, int C, int N, int co, int ci_real, int mode) {
  const long long total = (long long)KH * KW * C * N;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const int e = (int)(i & 7);
    long long t = i >> 3;
    const int n = (int)(t % N);
    t /= N;
    const int cj = (int)(t % (C / 8));
    const int tap = (int)(t / (C / 8));
    const int r = tap / KW, s = tap % KW, k = cj * 8 + e;
    float v = 0.f;
    if (mode == 0) {
      if (k < ci_real) v = w[(((size_t)n * ci_real + k) * KH + r) * KW + s];
    } else if (mode == 1) {
      // here C = co (reduction), N = ci
      if (n < ci_real) v = w[(((size_t)k * ci_real + n) * KH + (KH - 1 - r)) * KW + (KW - 1 - s)];
    } else {
      const int dy = k >> 3, dx = (k >> 2) & 1, c = k & 3;
      const int fr = 2 * r + dy - 1, fs = 2 * s + dx - 1;  // 7x7 filter coordinates
      if (c < ci_real && fr >= 0 && fr < 7 && fs >= 0 && fs < 7) v = w[(((size_t)n * ci_real + c) * 7 + fr) * 7 + fs];
    }
    // forward / stem images multiply fp16 activations -> fp16; the dgrad image multiplies bf16 gradients -> bf16
    if (mode == 1) img[i] = __float2bfloat16(v);
    else reinterpret_cast<__half*>(img)[i] = __float2half_rn(v);
  }
}

// dw accumulator of the s2d stem [(a*4+b)*16 + (dy,dx,c)][co] -> OIHW 7x7 gradient
__global__ void unpack_stem_wgrad_kernel(const float* __restrict__ acc, float* __restrict__ dw, int co, int ci_real) {
  const int total = co * ci_real * 49;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int fs = i % 7, fr = (i / 7) % 7, c = (i / 49) % ci_real, o = i / (49 * ci_real);
    const int a = (fr + 1) >> 1, dy = (fr + 1) & 1, b = (fs + 1) >> 1, dx = (fs + 1) & 1;
    dw[i] = acc[((size_t)(a * 4 + b) * 16 + (dy * 2 + dx) * 4 + c) * co + o];
  }
}

// resident CTAs per SM from static limits (registers, shared memory); cached per kernel
// ------------------------------------------------------------------------------------------
// The same persistent forward / dgrad kernel with the halo loaded by TMA (HB200_NO_HALO_TMA=1 falls back to the cp.async
// kernel above).  One thread issues C/8
// `cp.async.bulk.tensor.4d` box copies per tile (box = {8 channels, halo width, halo height, 1 frame}; the conv
// padding is the TMA unit's out-of-bounds zero fill) that complete on an mbarrier, instead of ~6 predicated
// cp.async per thread -- the address / predicate arithmetic that makes conv_halo_kernel<32,32> issue-bound.
// The box lands as [cj][hy][hx][8 ch], so the K-major descriptors become
//   start = stage + 2kk*SLAB + r*HWD*16 + s*16,   LBO = SLAB (next 8 channels),   SBO = HWD*16 (next tile row).
// The warpgroup waits for the load on the stage's mbarrier before it issues the tile's MMAs.
// ------------------------------------------------------------------------------------------

template <int C, int N, int KH, int KW, int PAD, int MODE>
__global__ void __launch_bounds__(128)
conv_halo_tma_kernel(const HaloArgs a, const __grid_constant__ CUtensorMap tmap) {
  using Cfg = HaloCfg<C, N, KH, KW, PAD>;
  constexpr int CJ = Cfg::CJ, HH = Cfg::HH, HWD = Cfg::HWD;
  constexpr uint32_t SLAB = (uint32_t)((HH * HWD * 16 + 127) / 128 * 128);
  constexpr uint32_t STAGE = CJ * SLAB;
  // halo stages: two when they fit next to the resident weights with >= 2 CTAs per SM; ONE for C = N = 64 (72 KB of
  // weights): the load of tile it+1 then starts when the MMAs of tile it are done, and the second CTA on the SM covers
  // the gap -- like conv_halo_kernel, minus the 2880 LSU cycles per tile its cp.async halo gather costs
  constexpr int NB = (Cfg::W_BYTES + 2 * (int)STAGE > 110 * 1024) ? 1 : 2;
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t ld_bar[2];
  __shared__ float stage_buf[kStageFloats];
  const uint32_t sbase = (smem_u32(smem_raw) + 127u) & ~127u;
  const uint32_t s_w = sbase;
  const uint32_t s_halo0 = s_w + Cfg::W_BYTES;   // W_BYTES is a multiple of 128
  const int tid = threadIdx.x, lane = tid & 31;

  if (tid == 0) {
    mbar_init(&ld_bar[0], 1);
    mbar_init(&ld_bar[1], 1);
    mbar_fence_init();
  }
  {
    const uint4* src = reinterpret_cast<const uint4*>(a.wimg);
    for (int v = tid; v < Cfg::W_BYTES / 16; v += 128) cp_async16(s_w + (uint32_t)v * 16, src + v, true);
  }
  cp_async_commit();
  const int tiles_x = a.W / TW, tiles_y = a.H / TH;
  const int tiles_per_img = tiles_x * tiles_y;
  auto tile_coords = [&](int tile, int& b, int& oh0, int& ow0) {
    b = tile / tiles_per_img;
    const int r = tile - b * tiles_per_img;
    oh0 = (r / tiles_x) * TH;
    ow0 = (r % tiles_x) * TW;
  };
  // The descriptor must be addressed in PARAM space: `&tmap` evaluated here, in the kernel body.  Inside the lambda a
  // by-reference capture makes nvcc spill a thread-local copy of the 128-byte map and hand the TMA unit a stack
  // address (round-1 version: every tile loaded garbage).
  const CUtensorMap* const tmap_p = &tmap;
  auto issue_halo = [&, tmap_p](int tile, int stage) {   // thread 0 only
    int b, oh0, ow0;
    tile_coords(tile, b, oh0, ow0);
    mbar_expect_tx(&ld_bar[stage], (uint32_t)(CJ * HH * HWD * 16));
#pragma unroll
    for (int j = 0; j < CJ; ++j)
      tma_load_4d(s_halo0 + (uint32_t)stage * STAGE + (uint32_t)j * SLAB, tmap_p, &ld_bar[stage], j * 8, ow0 - PAD,
                  oh0 - PAD, b);
  };
  const int first = blockIdx.x, stride = gridDim.x;
  const int my_n = first < a.ntiles ? (a.ntiles - first + stride - 1) / stride : 0;
  __syncthreads();   // barriers initialised
  if (tid == 0 && my_n > 0) issue_halo(first, 0);
  cp_async_wait<0>();          // weights
  fence_proxy_async_smem();    // cp.async (generic proxy) -> wgmma (async proxy)
  __syncthreads();
  // forward: fp16 input halo x fp16 weight image; dgrad: bf16 gradients x bf16 flipped / transposed image
  constexpr int kT = MODE == 0 ? kF16 : kBF16;
  float acc_t[N];
  const int py = tid >> 3, px = tid & 7;

  for (int it = 0; it < my_n; ++it) {
    // two stages: tile it+1 loads into the stage tile it-1 used (its MMAs completed in the last iteration)
    if (NB == 2 && tid == 0 && it + 1 < my_n) issue_halo(first + (it + 1) * stride, (it + 1) & 1);
    mbar_wait(&ld_bar[NB == 2 ? (it & 1) : 0], NB == 2 ? ((it >> 1) & 1) : (it & 1));
    {
      const uint32_t sh = s_halo0 + (uint32_t)(NB == 2 ? (it & 1) : 0) * STAGE;
      wgmma_fence();
      uint32_t accum = 0;
#pragma unroll
      for (int r = 0; r < KH; ++r)
#pragma unroll
        for (int s = 0; s < KW; ++s)
#pragma unroll
          for (int kk = 0; kk < C / 16; ++kk) {
            const uint64_t da = make_smem_desc(sh + 2 * kk * SLAB + r * (HWD * 16) + s * 16, SLAB, HWD * 16, kNoSwizzle);
            const uint64_t db = make_smem_desc(s_w + (r * KW + s) * (C * N * 2) + 2 * kk * (N * 16), N * 16, 128, kNoSwizzle);
            mma128<N, kT>(acc_t, da, 8 * HWD * 16, db, accum);
            accum = 1;
          }
      wgmma_commit();
      wgmma_wait<0>();
      acc_fence(acc_t);
    }
    // single halo stage: the MMAs of tile it have consumed it -> the next tile loads during this epilogue
    if (NB == 1 && tid == 0 && it + 1 < my_n) issue_halo(first + (it + 1) * stride, 0);
    {   // epilogue of tile it
      int b, oh0, ow0;
      tile_coords(first + it * stride, b, oh0, ow0);
      const size_t pix = ((size_t)b * a.H + oh0 + py) * a.W + ow0 + px;
#pragma unroll
      for (int col0 = 0; col0 < N; col0 += 32) {
        float acc[32];
        acc_row32(acc_t, col0, stage_buf, acc);
        if (MODE == 0 && a.stats != nullptr)
          halo_gn_stats_chunk(acc, lane, N / a.gn_groups, a.stats + (size_t)b * a.gn_groups * 2, col0);
        const size_t o = pix * N + col0;
        if (MODE == 1 && a.addend != nullptr) {
          const uint4* ad = reinterpret_cast<const uint4*>(a.addend + o);
#pragma unroll
          for (int v = 0; v < 4; ++v) {
            float f[8];
            unpack8(ad[v], f);
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[v * 8 + e] += f[e];
          }
        }
        uint4* dst = reinterpret_cast<uint4*>(a.y + o);
#pragma unroll
        for (int v = 0; v < 4; ++v) {
          uint4 u;
          if (MODE == 0) {  // forward output y: fp16 (saturating)
            u.x = pack_f16x2(acc[v * 8 + 0], acc[v * 8 + 1]);
            u.y = pack_f16x2(acc[v * 8 + 2], acc[v * 8 + 3]);
            u.z = pack_f16x2(acc[v * 8 + 4], acc[v * 8 + 5]);
            u.w = pack_f16x2(acc[v * 8 + 6], acc[v * 8 + 7]);
          } else {          // data gradient: bf16
            u.x = pack_bf16x2(acc[v * 8 + 0], acc[v * 8 + 1]);
            u.y = pack_bf16x2(acc[v * 8 + 2], acc[v * 8 + 3]);
            u.z = pack_bf16x2(acc[v * 8 + 4], acc[v * 8 + 5]);
            u.w = pack_bf16x2(acc[v * 8 + 6], acc[v * 8 + 7]);
          }
          dst[v] = u;
        }
      }
    }
  }
}

template <int C, int N, int MODE>
__global__ void __launch_bounds__(128)
conv_halo_sw_kernel(const HaloArgs a, const __grid_constant__ CUtensorMap tmap) {
  // 3x3 stride-1 pad-1.  The halo is staged as KW = 3 copies of the tile rows, copy kx pre-shifted by kx pixels, each
  // copy [HH rows][8 pixels][C channels] in the 64- / 128-byte-swizzle K-major layout (one TMA box per copy: rows of
  // C*2 bytes instead of the 16-byte pieces of the no-swizzle slabs, whose rate -- not bytes -- bounds the slab-fed
  // kernels).  A filter tap (r, s) is then copy s shifted by r whole swizzle atoms: aligned descriptors only.
  using Cfg = HaloCfg<C, N, 3, 3, 1>;
  constexpr int KH = 3, KW = 3, PAD = 1, HH = Cfg::HH;
  constexpr uint32_t RB = C * 2;                 // bytes per pixel row of the operand: 64 (SWIZZLE_64B) or 128
  constexpr uint32_t ATOM = 8 * RB;              // 8 pixels = one output row of the tile = one swizzle atom
  constexpr uint32_t COPY = HH * ATOM;
  constexpr uint32_t STAGE = KW * COPY;
  constexpr int NB = (Cfg::W_BYTES + 2 * (int)STAGE > 200 * 1024) ? 1 : 2;
  constexpr int kSw = RB == 128 ? kSwizzle128B : kSwizzle64B;
  static_assert(RB == 64 || RB == 128, "conv_halo_sw: 32 or 64 channels");
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t ld_bar[2];
  __shared__ float stage_buf[kStageFloats];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;   // swizzle atoms: 1024-byte aligned
  const uint32_t s_w = sbase;
  const uint32_t s_halo0 = s_w + Cfg::W_BYTES;   // W_BYTES is a multiple of 128
  const int tid = threadIdx.x, lane = tid & 31;

  if (tid == 0) {
    mbar_init(&ld_bar[0], 1);
    mbar_init(&ld_bar[1], 1);
    mbar_fence_init();
  }
  {
    const uint4* src = reinterpret_cast<const uint4*>(a.wimg);
    for (int v = tid; v < Cfg::W_BYTES / 16; v += 128) cp_async16(s_w + (uint32_t)v * 16, src + v, true);
  }
  cp_async_commit();
  const int tiles_x = a.W / TW, tiles_y = a.H / TH;
  const int tiles_per_img = tiles_x * tiles_y;
  auto tile_coords = [&](int tile, int& b, int& oh0, int& ow0) {
    b = tile / tiles_per_img;
    const int r = tile - b * tiles_per_img;
    oh0 = (r / tiles_x) * TH;
    ow0 = (r % tiles_x) * TW;
  };
  // The descriptor must be addressed in PARAM space: `&tmap` evaluated here, in the kernel body.  Inside the lambda a
  // by-reference capture makes nvcc spill a thread-local copy of the 128-byte map and hand the TMA unit a stack
  // address (round-1 version: every tile loaded garbage).
  const CUtensorMap* const tmap_p = &tmap;
  auto issue_halo = [&, tmap_p](int tile, int stage) {   // thread 0 only
    int b, oh0, ow0;
    tile_coords(tile, b, oh0, ow0);
    mbar_expect_tx(&ld_bar[stage], STAGE);
#pragma unroll
    for (int kx = 0; kx < KW; ++kx)
      tma_load_4d(s_halo0 + (uint32_t)stage * STAGE + (uint32_t)kx * COPY, tmap_p, &ld_bar[stage], 0, ow0 - PAD + kx,
                  oh0 - PAD, b);
  };
  const int first = blockIdx.x, stride = gridDim.x;
  const int my_n = first < a.ntiles ? (a.ntiles - first + stride - 1) / stride : 0;
  __syncthreads();   // barriers initialised
  if (tid == 0 && my_n > 0) issue_halo(first, 0);
  cp_async_wait<0>();          // weights
  fence_proxy_async_smem();    // cp.async (generic proxy) -> wgmma (async proxy)
  __syncthreads();
  // forward: fp16 input halo x fp16 weight image; dgrad: bf16 gradients x bf16 flipped / transposed image
  constexpr int kT = MODE == 0 ? kF16 : kBF16;
  float acc_t[N];
  const int py = tid >> 3, px = tid & 7;

  for (int it = 0; it < my_n; ++it) {
    // two stages: tile it+1 loads into the stage tile it-1 used (its MMAs completed in the last iteration)
    if (NB == 2 && tid == 0 && it + 1 < my_n) issue_halo(first + (it + 1) * stride, (it + 1) & 1);
    mbar_wait(&ld_bar[NB == 2 ? (it & 1) : 0], NB == 2 ? ((it >> 1) & 1) : (it & 1));
    {
      const uint32_t sh = s_halo0 + (uint32_t)(NB == 2 ? (it & 1) : 0) * STAGE;
      wgmma_fence();
      uint32_t accum = 0;
#pragma unroll
      for (int r = 0; r < KH; ++r)
#pragma unroll
        for (int s = 0; s < KW; ++s)
#pragma unroll
          for (int kk = 0; kk < C / 16; ++kk) {
            const uint64_t da = make_smem_desc(sh + s * COPY + r * ATOM + kk * 32, 16, ATOM, (Layout)kSw);
            const uint64_t db = make_smem_desc(s_w + (r * KW + s) * (C * N * 2) + 2 * kk * (N * 16), N * 16, 128, kNoSwizzle);
            mma128<N, kT>(acc_t, da, 8 * ATOM, db, accum);
            accum = 1;
          }
      wgmma_commit();
      wgmma_wait<0>();
      acc_fence(acc_t);
    }
    // single halo stage: the MMAs of tile it have consumed it -> the next tile loads during this epilogue
    if (NB == 1 && tid == 0 && it + 1 < my_n) issue_halo(first + (it + 1) * stride, 0);
    {   // epilogue of tile it
      int b, oh0, ow0;
      tile_coords(first + it * stride, b, oh0, ow0);
      const size_t pix = ((size_t)b * a.H + oh0 + py) * a.W + ow0 + px;
#pragma unroll
      for (int col0 = 0; col0 < N; col0 += 32) {
        float acc[32];
        acc_row32(acc_t, col0, stage_buf, acc);
        if (MODE == 0 && a.stats != nullptr)
          halo_gn_stats_chunk(acc, lane, N / a.gn_groups, a.stats + (size_t)b * a.gn_groups * 2, col0);
        const size_t o = pix * N + col0;
        if (MODE == 1 && a.addend != nullptr) {
          const uint4* ad = reinterpret_cast<const uint4*>(a.addend + o);
#pragma unroll
          for (int v = 0; v < 4; ++v) {
            float f[8];
            unpack8(ad[v], f);
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[v * 8 + e] += f[e];
          }
        }
        uint4* dst = reinterpret_cast<uint4*>(a.y + o);
#pragma unroll
        for (int v = 0; v < 4; ++v) {
          uint4 u;
          if (MODE == 0) {  // forward output y: fp16 (saturating)
            u.x = pack_f16x2(acc[v * 8 + 0], acc[v * 8 + 1]);
            u.y = pack_f16x2(acc[v * 8 + 2], acc[v * 8 + 3]);
            u.z = pack_f16x2(acc[v * 8 + 4], acc[v * 8 + 5]);
            u.w = pack_f16x2(acc[v * 8 + 6], acc[v * 8 + 7]);
          } else {          // data gradient: bf16
            u.x = pack_bf16x2(acc[v * 8 + 0], acc[v * 8 + 1]);
            u.y = pack_bf16x2(acc[v * 8 + 2], acc[v * 8 + 3]);
            u.z = pack_bf16x2(acc[v * 8 + 4], acc[v * 8 + 5]);
            u.w = pack_bf16x2(acc[v * 8 + 6], acc[v * 8 + 7]);
          }
          dst[v] = u;
        }
      }
    }
  }
}


// ---- warp-specialised variant ---------------------------------------------------------------------------------------
// conv_halo_tma_kernel runs load -> MMA -> epilogue of consecutive tiles from one program order: with a single halo
// stage the TMA latency of tile it+1 is exposed after every tile, and only a second CTA of the SM hides it.  Here the
// loads run in their own warp and meet the consumers only at mbarriers:
//   warp 4 (one lane)  producer: halo stage ring, NS deep (as many as fit next to the resident weights)
//   warps 0-3          one warpgroup: waits full[stage], issues the tile's MMAs, releases the stage (empty[stage]) as
//                      soon as they complete, then GroupNorm sums / addend / pack / store while the producer loads ahead
// SW: stage the halo as KW pre-shifted copies of whole pixel rows in the swizzled K-major layout (conv_halo_sw_kernel)
// instead of 16-byte channel slabs: aligned operand reads for the MMAs at KW times the TMA bytes
template <int C, int N, int KH, int KW, int PAD, int MODE, int NS, bool SW = false>
__global__ void __launch_bounds__(160)
conv_halo_ws_kernel(const HaloArgs a, const __grid_constant__ CUtensorMap tmap) {
  using Cfg = HaloCfg<C, N, KH, KW, PAD>;
  constexpr int CJ = Cfg::CJ, HH = Cfg::HH, HWD = Cfg::HWD;
  constexpr uint32_t SLAB = (uint32_t)((HH * HWD * 16 + 127) / 128 * 128);
  constexpr uint32_t RB = C * 2, ATOM = 8 * RB, COPY = HH * ATOM;   // swizzled copies: pixel rows, 8-pixel atoms
  constexpr uint32_t STAGE = SW ? KW * COPY : CJ * SLAB;
  constexpr int kSw = RB == 128 ? kSwizzle128B : kSwizzle64B;
  static_assert(!SW || RB == 64 || RB == 128, "swizzled halo copies: 32 or 64 channels");
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[NS], empty_bar[NS];
  __shared__ float stage_buf[kStageFloats];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;   // swizzle atoms are 1024-byte aligned
  const uint32_t s_w = sbase;
  const uint32_t s_halo0 = s_w + Cfg::W_BYTES;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
#pragma unroll
    for (int i = 0; i < NS; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 1); }
    mbar_fence_init();
  }
  {
    const uint4* src = reinterpret_cast<const uint4*>(a.wimg);
    for (int v = tid; v < Cfg::W_BYTES / 16; v += blockDim.x) cp_async16(s_w + (uint32_t)v * 16, src + v, true);
  }
  cp_async_commit();
  cp_async_wait<0>();
  fence_proxy_async_smem();
  __syncthreads();
  const int tiles_x = a.W / TW, tiles_per_img = tiles_x * (a.H / TH);
  const int first = blockIdx.x, stride = gridDim.x;
  const int my_n = first < a.ntiles ? (a.ntiles - first + stride - 1) / stride : 0;
  const CUtensorMap* const tmap_p = &tmap;   // param-space address, taken in the kernel body

  if (warp == 4) {
    if (lane == 0) {
      for (int it = 0; it < my_n; ++it) {
        const int st = it % NS;
        if (it >= NS) mbar_wait(&empty_bar[st], ((it / NS) - 1) & 1);
        const int tile = first + it * stride;
        const int b = tile / tiles_per_img, r = tile - b * tiles_per_img;
        const int oh0 = (r / tiles_x) * TH, ow0 = (r % tiles_x) * TW;
        if constexpr (SW) {
          mbar_expect_tx(&full_bar[st], STAGE);
#pragma unroll
          for (int kx = 0; kx < KW; ++kx)
            tma_load_4d(s_halo0 + (uint32_t)st * STAGE + (uint32_t)kx * COPY, tmap_p, &full_bar[st], 0, ow0 - PAD + kx,
                        oh0 - PAD, b);
        } else {
          mbar_expect_tx(&full_bar[st], (uint32_t)(CJ * HH * HWD * 16));
#pragma unroll
          for (int j = 0; j < CJ; ++j)
            tma_load_4d(s_halo0 + (uint32_t)st * STAGE + (uint32_t)j * SLAB, tmap_p, &full_bar[st], j * 8, ow0 - PAD,
                        oh0 - PAD, b);
        }
      }
    }
    __syncwarp();
  } else {
    // forward: fp16 input halo x fp16 weight image; dgrad: bf16 gradients x bf16 flipped / transposed image
    constexpr int kT = MODE == 0 ? kF16 : kBF16;
    const int py = tid >> 3, px = tid & 7;
    float acc_t[N];
    for (int it = 0; it < my_n; ++it) {
      const int st = it % NS;
      const int tile = first + it * stride;
      const int b = tile / tiles_per_img, r = tile - b * tiles_per_img;
      const int oh0 = (r / tiles_x) * TH, ow0 = (r % tiles_x) * TW;
      mbar_wait(&full_bar[st], (it / NS) & 1);
      const uint32_t sh = s_halo0 + (uint32_t)st * STAGE;
      wgmma_fence();
      uint32_t accum = 0;
#pragma unroll
      for (int r = 0; r < KH; ++r)
#pragma unroll
        for (int s = 0; s < KW; ++s)
#pragma unroll
          for (int kk = 0; kk < C / 16; ++kk) {
            const uint64_t da = SW ? make_smem_desc(sh + s * COPY + r * ATOM + kk * 32, 16, ATOM, (Layout)kSw)
                                   : make_smem_desc(sh + 2 * kk * SLAB + r * (HWD * 16) + s * 16, SLAB, HWD * 16, kNoSwizzle);
            const uint64_t db = make_smem_desc(s_w + (r * KW + s) * (C * N * 2) + 2 * kk * (N * 16), N * 16, 128, kNoSwizzle);
            mma128<N, kT>(acc_t, da, SW ? 8 * ATOM : 8 * HWD * 16, db, accum);
            accum = 1;
          }
      wgmma_commit();
      wgmma_wait<0>();
      acc_fence(acc_t);
      if (tid == 0) mbar_arrive(&empty_bar[st]);   // the halo stage is free: the producer may refill it
      const size_t pix = ((size_t)b * a.H + oh0 + py) * a.W + ow0 + px;
#pragma unroll
      for (int col0 = 0; col0 < N; col0 += 32) {
        float acc_[32];
        acc_row32(acc_t, col0, stage_buf, acc_);
        if (MODE == 0 && a.stats != nullptr)
          halo_gn_stats_chunk(acc_, lane, N / a.gn_groups, a.stats + (size_t)b * a.gn_groups * 2, col0);
        const size_t o = pix * N + col0;
        if (MODE == 1 && a.addend != nullptr) {
          const uint4* ad = reinterpret_cast<const uint4*>(a.addend + o);
#pragma unroll
          for (int v = 0; v < 4; ++v) {
            float f[8];
            unpack8(ad[v], f);
#pragma unroll
            for (int e2 = 0; e2 < 8; ++e2) acc_[v * 8 + e2] += f[e2];
          }
        }
        uint4* dst = reinterpret_cast<uint4*>(a.y + o);
#pragma unroll
        for (int v = 0; v < 4; ++v) {
          uint4 u;
          if (MODE == 0) {
            u.x = pack_f16x2(acc_[v * 8 + 0], acc_[v * 8 + 1]);
            u.y = pack_f16x2(acc_[v * 8 + 2], acc_[v * 8 + 3]);
            u.z = pack_f16x2(acc_[v * 8 + 4], acc_[v * 8 + 5]);
            u.w = pack_f16x2(acc_[v * 8 + 6], acc_[v * 8 + 7]);
          } else {
            u.x = pack_bf16x2(acc_[v * 8 + 0], acc_[v * 8 + 1]);
            u.y = pack_bf16x2(acc_[v * 8 + 2], acc_[v * 8 + 3]);
            u.z = pack_bf16x2(acc_[v * 8 + 4], acc_[v * 8 + 5]);
            u.w = pack_bf16x2(acc_[v * 8 + 6], acc_[v * 8 + 7]);
          }
          dst[v] = u;
        }
      }
    }
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn halo_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
      q != cudaDriverEntryPointSuccess)
    return nullptr;
  fn = (EncodeTiledFn)p;
  return fn;
}

static int blocks_per_sm(const void* kern, size_t smem, int* cache) {
  if (*cache > 0) return *cache;
  cudaFuncAttributes fa;
  if (cudaFuncGetAttributes(&fa, kern) != cudaSuccess) return 1;
  const int regs = fa.numRegs > 0 ? fa.numRegs : 128;
  int by_regs = 65536 / (((regs + 7) / 8 * 8) * 128);
  int by_smem = (int)((227 * 1024) / (smem + fa.sharedSizeBytes + 1024));
  int n = by_regs < by_smem ? by_regs : by_smem;
  if (n > 16) n = 16;
  if (n < 1) n = 1;
  *cache = n;
  return n;
}

template <int C, int N, int KH, int KW, int PAD, int MODE>
static int launch_halo(const HaloArgs& a, cudaStream_t st) {
  using Cfg = HaloCfg<C, N, KH, KW, PAD>;
  const size_t smem = Cfg::W_BYTES + Cfg::NBUF * Cfg::HALO_BYTES + 256;
  auto kern = conv_halo_kernel<C, N, KH, KW, PAD, MODE>;
  static int cache = 0;
  if (cache == 0) HB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int per_sm = blocks_per_sm((const void*)kern, smem, &cache);
  int grid = kNumSMs * per_sm;
  if (grid > a.ntiles) grid = a.ntiles;
  kern<<<grid, 128, smem, st>>>(a);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

template <int C, int N, int KH, int KW, int PAD, int MODE>
static int launch_halo_tma(const HaloArgs& a, cudaStream_t st) {
  using Cfg = HaloCfg<C, N, KH, KW, PAD>;
  EncodeTiledFn enc = halo_encode_fn();
  if (!enc) {
    set_last_error("conv_halo (TMA): cuTensorMapEncodeTiled is not available from this driver");
    return HB200_ERR_UNSUPPORTED;
  }
  CUtensorMap tmap;
  const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)a.W, (cuuint64_t)a.H, (cuuint64_t)a.B};
  const cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)a.W * C * 2, (cuuint64_t)a.H * a.W * C * 2};
  const cuuint32_t box[4] = {8u, (cuuint32_t)Cfg::HWD, (cuuint32_t)Cfg::HH, 1u};
  const cuuint32_t estr[4] = {1u, 1u, 1u, 1u};
  const CUresult r = enc(&tmap, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, (void*)a.x, dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("conv_halo (TMA): cuTensorMapEncodeTiled failed (%d)", (int)r);
    return HB200_ERR_CUDA;
  }
  constexpr size_t slab = (size_t)((Cfg::HH * Cfg::HWD * 16 + 127) / 128 * 128);
  constexpr int nstage = (Cfg::W_BYTES + 2 * (int)(Cfg::CJ * slab) > 110 * 1024) ? 1 : 2;
  const size_t smem = Cfg::W_BYTES + nstage * Cfg::CJ * slab + 256;
  auto kern = conv_halo_tma_kernel<C, N, KH, KW, PAD, MODE>;
  static int cache = 0;
  if (cache == 0) HB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int per_sm = blocks_per_sm((const void*)kern, smem, &cache);
  int grid = kNumSMs * per_sm;
  if (grid > a.ntiles) grid = a.ntiles;
  kern<<<grid, 128, smem, st>>>(a, tmap);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

template <int C, int N, int KH, int KW, int PAD, int MODE, int NS, bool SW = false>
static int launch_halo_ws(const HaloArgs& a, cudaStream_t st) {
  using Cfg = HaloCfg<C, N, KH, KW, PAD>;
  EncodeTiledFn enc = halo_encode_fn();
  if (!enc) {
    set_last_error("conv_halo (TMA): cuTensorMapEncodeTiled is not available from this driver");
    return HB200_ERR_UNSUPPORTED;
  }
  CUtensorMap tmap;
  const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)a.W, (cuuint64_t)a.H, (cuuint64_t)a.B};
  const cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)a.W * C * 2, (cuuint64_t)a.H * a.W * C * 2};
  const cuuint32_t box_slab[4] = {8u, (cuuint32_t)Cfg::HWD, (cuuint32_t)Cfg::HH, 1u};
  const cuuint32_t box_rows[4] = {(cuuint32_t)C, (cuuint32_t)TW, (cuuint32_t)Cfg::HH, 1u};
  const cuuint32_t* box = SW ? box_rows : box_slab;
  const cuuint32_t estr[4] = {1u, 1u, 1u, 1u};
  const CUresult r = enc(&tmap, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, (void*)a.x, dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE,
                         !SW ? CU_TENSOR_MAP_SWIZZLE_NONE : (C == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B),
                         CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("conv_halo (TMA): cuTensorMapEncodeTiled failed (%d)", (int)r);
    return HB200_ERR_CUDA;
  }
  constexpr size_t slab = (size_t)((Cfg::HH * Cfg::HWD * 16 + 127) / 128 * 128);
  const size_t stage = SW ? (size_t)KW * Cfg::HH * 8 * C * 2 : Cfg::CJ * slab;
  const size_t smem = Cfg::W_BYTES + (size_t)NS * stage + 1024;
  auto kern = conv_halo_ws_kernel<C, N, KH, KW, PAD, MODE, NS, SW>;
  static int grid_cache = 0;
  if (grid_cache == 0) {
    HB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    // resident CTAs per SM from the static limits (registers of 160 threads, shared memory)
    cudaFuncAttributes fa;
    HB_CUDA(cudaFuncGetAttributes(&fa, (const void*)kern));
    const int regs = fa.numRegs > 0 ? fa.numRegs : 128;
    int per_sm = 65536 / (((regs + 7) / 8 * 8) * 160);
    const int by_smem = (int)((227 * 1024) / (smem + fa.sharedSizeBytes + 1024));
    if (by_smem < per_sm) per_sm = by_smem;
    if (per_sm < 1) per_sm = 1;
    grid_cache = kNumSMs * per_sm;
  }
  const int grid = grid_cache < a.ntiles ? grid_cache : a.ntiles;
  kern<<<grid, 160, smem, st>>>(a, tmap);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

template <int C, int N, int MODE>
static int launch_halo_sw(const HaloArgs& a, cudaStream_t st) {
  using Cfg = HaloCfg<C, N, 3, 3, 1>;
  EncodeTiledFn enc = halo_encode_fn();
  if (!enc) {
    set_last_error("conv_halo (swizzled TMA): cuTensorMapEncodeTiled is not available from this driver");
    return HB200_ERR_UNSUPPORTED;
  }
  CUtensorMap tmap;
  const cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)a.W, (cuuint64_t)a.H, (cuuint64_t)a.B};
  const cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)a.W * C * 2, (cuuint64_t)a.H * a.W * C * 2};
  const cuuint32_t box[4] = {(cuuint32_t)C, (cuuint32_t)TW, (cuuint32_t)Cfg::HH, 1u};   // whole pixels: C*2-byte rows
  const cuuint32_t estr[4] = {1u, 1u, 1u, 1u};
  const CUresult r = enc(&tmap, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, (void*)a.x, dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, C == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("conv_halo (swizzled TMA): cuTensorMapEncodeTiled failed (%d)", (int)r);
    return HB200_ERR_CUDA;
  }
  constexpr size_t stage = (size_t)3 * Cfg::HH * 8 * C * 2;
  constexpr int nstage = (Cfg::W_BYTES + 2 * (int)stage > 200 * 1024) ? 1 : 2;
  const size_t smem = Cfg::W_BYTES + nstage * stage + 1024;
  auto kern = conv_halo_sw_kernel<C, N, MODE>;
  static int cache = 0;
  if (cache == 0) HB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int per_sm = blocks_per_sm((const void*)kern, smem, &cache);
  int grid = kNumSMs * per_sm;
  if (grid > a.ntiles) grid = a.ntiles;
  kern<<<grid, 128, smem, st>>>(a, tmap);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

template <int C, int N, int KH, int KW, int PAD, int XMODE = 0>
static int launch_halo_wgrad(const HaloWgradArgs& a, cudaStream_t st) {
  constexpr int CJ = C / 8, HWD = TW + KW - 1, P = HWD * 16, RP = CJ * P;
  constexpr int MT = (KH * CJ + 15) / 16, RMAX = (MT * 16 + CJ - 1) / CJ, HROWS = TH - 1 + RMAX;
  constexpr int STAGE = (128 * N * 2 + HROWS * RP + 1023) / 1024 * 1024;
  constexpr int NSW = halo_wgrad_stages(XMODE, C, STAGE);
  const size_t smem = NSW * (size_t)STAGE + 1024 + 64;
  EncodeTiledFn enc = halo_encode_fn();
  if (!enc) {
    set_last_error("conv_halo_wgrad: cuTensorMapEncodeTiled is not available from this driver");
    return HB200_ERR_UNSUPPORTED;
  }
  // dy bf16 [B, H, W, N]: box = N channels (one swizzled 64- / 128-byte row per pixel) x 8 x 16 pixels of one frame
  CUtensorMap tmap;
  const cuuint64_t dims[4] = {(cuuint64_t)N, (cuuint64_t)a.W, (cuuint64_t)a.H, (cuuint64_t)a.B};
  const cuuint64_t strides[3] = {(cuuint64_t)N * 2, (cuuint64_t)a.W * N * 2, (cuuint64_t)a.H * a.W * N * 2};
  const cuuint32_t box[4] = {(cuuint32_t)N, (cuuint32_t)TW, (cuuint32_t)TH, 1u};
  const cuuint32_t estr[4] = {1u, 1u, 1u, 1u};
  const CUresult r = enc(&tmap, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, (void*)a.dy, dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, N == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("conv_halo_wgrad: cuTensorMapEncodeTiled failed (%d)", (int)r);
    return HB200_ERR_CUDA;
  }
  // x halo by TMA: x bf16 [B, Hx, Wx, Cx] seen as (8 | pixel column | chunk | row | frame).  XMODE 2: a.H, a.W are the
  // dims of the space-to-depth view; the real tensor has 2H x 2W pixels of C/4 channels, "pixel column" steps over
  // pixel PAIRS (2 * Cx * 2 bytes) and a row of the view's chunks = the (dx, c) run of one image row
  CUtensorMap tmap_x = tmap;
  if (XMODE != 0) {
    const int cx = XMODE == 2 ? C / 4 : C, hx = XMODE == 2 ? 2 * a.H : a.H, wx = XMODE == 2 ? 2 * a.W : a.W;
    const int chunks_per_row = XMODE == 2 ? CJ / 2 : CJ, col_bytes = (XMODE == 2 ? 2 : 1) * cx * 2;
    const cuuint64_t xd[5] = {8u, (cuuint64_t)a.W, (cuuint64_t)chunks_per_row, (cuuint64_t)hx, (cuuint64_t)a.B};
    const cuuint64_t xs[4] = {(cuuint64_t)col_bytes, 16u, (cuuint64_t)wx * cx * 2, (cuuint64_t)hx * wx * cx * 2};
    constexpr int HROWS_LOAD = TH + KH - 1;
    const cuuint32_t xb[5] = {8u, (cuuint32_t)HWD, (cuuint32_t)chunks_per_row,
                              (cuuint32_t)(XMODE == 2 ? 2 * HROWS_LOAD : HROWS_LOAD), 1u};
    const cuuint32_t xe[5] = {1u, 1u, 1u, 1u, 1u};
    const CUresult rx = enc(&tmap_x, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, (void*)a.x, xd, xs, xb, xe,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (rx != CUDA_SUCCESS) {
      set_last_error("conv_halo_wgrad: cuTensorMapEncodeTiled (x halo) failed (%d)", (int)rx);
      return HB200_ERR_CUDA;
    }
  }
  auto kern = conv_halo_wgrad_kernel<C, N, KH, KW, PAD, XMODE>;
  static int cache = 0;
  if (cache == 0) HB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  // accumulator groups (the kernel's APC): one grid row each, every row walks all tiles
  constexpr int nacc = KW * MT, ngrp = nacc * N <= 128 ? 1 : nacc / (128 / N);
  const int per_sm = blocks_per_sm((const void*)kern, smem, &cache);
  int grid = kNumSMs * per_sm / ngrp;
  if (grid < 1) grid = 1;
  if (grid > a.ntiles) grid = a.ntiles;
  // one partial per worker column, summed in worker order into the caller's accumulator (deterministic)
  const long long count = (long long)KH * KW * C * N;
  float* parts = nullptr;
  int* tickets = nullptr;
  int rc = stream_workspace(st, (size_t)(grid + (grid < kReduceChunks ? grid : kReduceChunks)) * count, 0, &parts, &tickets);
  if (rc) return rc;
  HaloWgradArgs ap = a;
  ap.dw = parts;
  kern<<<dim3(grid, ngrp), 128, smem, st>>>(ap, tmap, tmap_x);
  HB_LAUNCH_OK();
  count_launch(1);
  return reduce_partials(parts, grid, count, count, a.dw, parts + (size_t)grid * count, st);
}

template <int NS, int IMG>
static int launch_halo_wgrad_small(const HaloWgradSmallArgs& a, cudaStream_t st) {
  constexpr int RP = 4 * (TW + 2) * 16, IPT = TH / IMG, RPI = IMG + 2;
  constexpr int HROWS_LOAD = IPT * RPI, HROWS = (IPT - 1) * RPI + (IMG - 2) + 1 + 4;
  constexpr int HROWS_A = HROWS > HROWS_LOAD ? HROWS : HROWS_LOAD;
  constexpr int HALO_BYTES = (HROWS_A * RP + 1023) / 1024 * 1024;
  const size_t smem = kSmallWgradStages * (size_t)(HALO_BYTES + (NS / 64) * 128 * 128) + 1024 + 64;
  EncodeTiledFn enc = halo_encode_fn();
  if (!enc) {
    set_last_error("conv_halo_wgrad (small images): cuTensorMapEncodeTiled is not available from this driver");
    return HB200_ERR_UNSUPPORTED;
  }
  // dy bf16 [B, IMG, IMG, Co]: box = 64 channels (one 128-byte swizzled row per pixel) x 8 columns x IMG rows x IPT images;
  // columns / images past the tensor are zero-filled (the virtual pixels of 4x4 images, the ragged last tile)
  CUtensorMap tmap;
  const cuuint64_t dims[4] = {(cuuint64_t)a.Co, (cuuint64_t)IMG, (cuuint64_t)IMG, (cuuint64_t)a.B};
  const cuuint64_t strides[3] = {(cuuint64_t)a.Co * 2, (cuuint64_t)IMG * a.Co * 2, (cuuint64_t)IMG * IMG * a.Co * 2};
  const cuuint32_t box[4] = {64u, 8u, (cuuint32_t)IMG, (cuuint32_t)IPT};
  const cuuint32_t estr[4] = {1u, 1u, 1u, 1u};
  const CUresult r = enc(&tmap, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, (void*)a.dy, dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("conv_halo_wgrad (small images): cuTensorMapEncodeTiled failed (%d)", (int)r);
    return HB200_ERR_CUDA;
  }
  auto kern = conv_halo_wgrad_small_kernel<NS, IMG>;
  static bool attr = false;
  if (!attr) {
    HB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr = true;
  }
  const int slices = (a.Ci / 32) * (a.Co / NS) * 3;   // channel slices x the 3 horizontal taps (one accumulator each)
  int workers = 2 * kNumSMs / slices;
  if (workers < 1) workers = 1;
  if (workers > a.ntiles) workers = a.ntiles;
  // one partial per worker, summed in worker order into the caller's accumulator (deterministic)
  const long long count = 9LL * a.Ci * a.Co;
  float* parts = nullptr;
  int* tickets = nullptr;
  int rc = stream_workspace(st, (size_t)(workers + (workers < kReduceChunks ? workers : kReduceChunks)) * count, 0, &parts,
                            &tickets);
  if (rc) return rc;
  HaloWgradSmallArgs ap = a;
  ap.dw = parts;
  kern<<<dim3(workers, slices), 128, smem, st>>>(ap, tmap);
  HB_LAUNCH_OK();
  count_launch(1);
  return reduce_partials(parts, workers, count, count, a.dw, parts + (size_t)workers * count, st);
}
}  // namespace hb200

using namespace hb200;

// halo loads by TMA (default) or by the cp.async gather kernel (HB200_NO_HALO_TMA=1, or hb200_set_halo_tma(0) from tests)
static int g_halo_tma = getenv("HB200_NO_HALO_TMA") == nullptr ? 1 : 0;
static int g_wgrad_xtma = getenv("HB200_WGRAD_XTMA") ? atoi(getenv("HB200_WGRAD_XTMA")) : 1;
extern "C" int hb200_set_halo_tma(int enable) {
  g_halo_tma = enable;   // 0 cp.async gather, 1 best per layer (default), 2 swizzled rows, 3 warp-specialised slabs, 4 both, 5 plain TMA slabs
  return HB200_OK;
}
extern "C" int hb200_get_halo_tma(void) { return g_halo_tma; }

/* which (C, N, k) combinations have a halo instantiation */
extern "C" int hb200_conv_halo_supported(int c, int n, int k, int h, int w) {
  if (h % TH || w % TW) return 0;
  if (k == 3) return (c == 32 && n == 32) || (c == 64 && n == 64);
  if (k == 4) return c == 16 && n == 32;
  return 0;
}

/* weight-gradient variant: additionally the small-image layers (8x8 / 4x4, channels sliced 32 x 128) */
extern "C" int hb200_conv_halo_wgrad_supported(int c, int n, int k, int h, int w) {
  if (hb200_conv_halo_supported(c, n, k, h, w)) return 1;
  return k == 3 && c % 32 == 0 && n % 128 == 0 && h == w && (h == 8 || h == 4);
}

extern "C" int hb200_pack_halo_weight(const float* w_oihw, hb200_bf16* img, int co, int ci_real, int c, int n,
                                      int k, int mode, hb200_stream_t stream) {
  HB_CHECK_ARG(w_oihw && img && mode >= 0 && mode <= 2, "pack_halo_weight: bad args");
  const long long total = (long long)k * k * c * n;
  pack_halo_weight_kernel<<<(int)min((total + 255) / 256, (long long)kNumSMs * 4), 256, 0, (cudaStream_t)stream>>>(
      w_oihw, (__nv_bfloat16*)img, k, k, c, n, co, ci_real, mode);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

extern "C" int hb200_unpack_stem_wgrad(const float* dw_acc, float* dw_oihw, int co, int ci_real,
                                       hb200_stream_t stream) {
  HB_CHECK_ARG(dw_acc && dw_oihw && ci_real <= 4, "unpack_stem_wgrad: bad args");
  unpack_stem_wgrad_kernel<<<cdiv(co * ci_real * 49, 256), 256, 0, (cudaStream_t)stream>>>(dw_acc, dw_oihw, co, ci_real);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

/* x [B,H,W,C] -> y [B,H,W,N], stride-1 "same" conv, k = 3 (pad 1) or k = 4 (pad 2 top/left, 1 bottom/right:
 * the space-to-depth stem).  mode 0 forward (gn_stats optional), mode 1 dgrad (addend optional). */
extern "C" int hb200_conv_halo(const hb200_bf16* x, const hb200_bf16* wimg, hb200_bf16* y, const hb200_bf16* addend,
                               double* gn_stats, int gn_groups, int batch, int h, int w, int c, int n, int k,
                               int mode, hb200_stream_t stream) {
  HB_CHECK_ARG(x && wimg && y, "conv_halo: null pointer");
  HB_CHECK_ARG(hb200_conv_halo_supported(c, n, k, h, w), "conv_halo: unsupported shape C=%d N=%d k=%d %dx%d", c, n, k, h, w);
  if (gn_stats) HB_CHECK_ARG(gn_groups > 0 && n % gn_groups == 0 && n / gn_groups >= 2, "conv_halo: bad GroupNorm groups");
  HaloArgs a;
  a.x = (const __nv_bfloat16*)x; a.wimg = (const __nv_bfloat16*)wimg; a.y = (__nv_bfloat16*)y;
  a.addend = (const __nv_bfloat16*)addend; a.stats = gn_stats;
  a.B = batch; a.H = h; a.W = w; a.gn_groups = gn_groups > 0 ? gn_groups : 1;
  a.ntiles = batch * (h / TH) * (w / TW);
  cudaStream_t st = (cudaStream_t)stream;
  // TMA-fed halo for every halo layer (no per-thread address / predicate work); HB200_NO_HALO_TMA=1 disables
  const bool use_tma = g_halo_tma != 0;
  // Loader per layer (hb200_set_halo_tma): 1 = the default per layer below (compare with tools/halo_bench.py):
  //   64 / 32 channels: warp-specialised + swizzled pixel-row copies; the stem: warp-specialised slabs
  // 2 / 3 / 4 / 5 force swizzled copies / warp-specialised slabs / warp-specialised swizzled / plain slabs everywhere.
  if (g_halo_tma == 1 && k == 3 && c == 64)
    return mode == 0 ? launch_halo_ws<64, 64, 3, 3, 1, 0, 2, true>(a, st) : launch_halo_ws<64, 64, 3, 3, 1, 1, 2, true>(a, st);
  if (g_halo_tma == 1 && k == 3 && c == 32)   // 3 stages each: several CTAs per SM
    return mode == 0 ? launch_halo_ws<32, 32, 3, 3, 1, 0, 3, true>(a, st) : launch_halo_ws<32, 32, 3, 3, 1, 1, 3, true>(a, st);
  if (g_halo_tma == 1 && k == 4 && mode == 0) return launch_halo_ws<16, 32, 4, 4, 2, 0, 6>(a, st);
  if (g_halo_tma == 6 && k == 3 && c == 32)   // experiment: 2 stages, more CTAs per SM
    return mode == 0 ? launch_halo_ws<32, 32, 3, 3, 1, 0, 2, true>(a, st) : launch_halo_ws<32, 32, 3, 3, 1, 1, 2, true>(a, st);
  if (g_halo_tma == 4 && k == 3 && c == 32)
    return mode == 0 ? launch_halo_ws<32, 32, 3, 3, 1, 0, 3, true>(a, st) : launch_halo_ws<32, 32, 3, 3, 1, 1, 3, true>(a, st);
  if (g_halo_tma == 4 && k == 3 && c == 64)
    return mode == 0 ? launch_halo_ws<64, 64, 3, 3, 1, 0, 2, true>(a, st) : launch_halo_ws<64, 64, 3, 3, 1, 1, 2, true>(a, st);
  if (g_halo_tma == 3 && k == 3 && c == 32)
    return mode == 0 ? launch_halo_ws<32, 32, 3, 3, 1, 0, 4>(a, st) : launch_halo_ws<32, 32, 3, 3, 1, 1, 4>(a, st);
  if (g_halo_tma == 3 && k == 3 && c == 64)
    return mode == 0 ? launch_halo_ws<64, 64, 3, 3, 1, 0, 5>(a, st) : launch_halo_ws<64, 64, 3, 3, 1, 1, 5>(a, st);
  if (g_halo_tma == 3 && k == 4 && mode == 0) return launch_halo_ws<16, 32, 4, 4, 2, 0, 6>(a, st);
  if (g_halo_tma == 2 && k == 3 && c == 32)
    return mode == 0 ? launch_halo_sw<32, 32, 0>(a, st) : launch_halo_sw<32, 32, 1>(a, st);
  if (g_halo_tma == 2 && k == 3 && c == 64)
    return mode == 0 ? launch_halo_sw<64, 64, 0>(a, st) : launch_halo_sw<64, 64, 1>(a, st);
  if (use_tma && k == 3 && c == 32)
    return mode == 0 ? launch_halo_tma<32, 32, 3, 3, 1, 0>(a, st) : launch_halo_tma<32, 32, 3, 3, 1, 1>(a, st);
  if (use_tma && k == 4 && mode == 0) return launch_halo_tma<16, 32, 4, 4, 2, 0>(a, st);
  // 64-channel layers: single halo stage (72 KB of resident weights), the load replaces the cp.async gather's 1440
  // copies per tile
  if (use_tma && k == 3 && c == 64)
    return mode == 0 ? launch_halo_tma<64, 64, 3, 3, 1, 0>(a, st) : launch_halo_tma<64, 64, 3, 3, 1, 1>(a, st);
  if (k == 3 && c == 32) return mode == 0 ? launch_halo<32, 32, 3, 3, 1, 0>(a, st) : launch_halo<32, 32, 3, 3, 1, 1>(a, st);
  if (k == 3 && c == 64) return mode == 0 ? launch_halo<64, 64, 3, 3, 1, 0>(a, st) : launch_halo<64, 64, 3, 3, 1, 1>(a, st);
  HB_CHECK_ARG(mode == 0, "conv_halo: the stem has no data gradient");
  return launch_halo<16, 32, 4, 4, 2, 0>(a, st);
}

// accumulator of the space-to-depth weight gradient [((ky*2+kx)*4 + dy*2+dx) * ci + c][co] -> OIHW 3x3 gradient
__global__ void unpack_s2_wgrad_kernel(const float* __restrict__ acc, float* __restrict__ dw, int co, int ci) {
  const int total = co * ci * 9;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int s = i % 3, r = (i / 3) % 3, c = (i / 9) % ci, o = i / (9 * ci);
    const int ky = r == 0 ? 0 : 1, dy = r == 0 ? 1 : r - 1, kx = s == 0 ? 0 : 1, dx = s == 0 ? 1 : s - 1;
    dw[i] = acc[((size_t)((ky * 2 + kx) * 4 + dy * 2 + dx) * ci + c) * co + o];
  }
}

/* weight gradient of a 3x3 stride-2 pad-1 conv as the 2x2 stride-1 weight gradient over the space-to-depth view of x
 * (x halo: one 5-D TMA box per tile).  x bf16 [B,H,W,C] (the twin), dy bf16 [B,H/2,W/2,N]; dw_acc f32 [16*C][N]
 * pre-zeroed, rows ((ky*2+kx)*4 + dy*2+dx)*C + c; hb200_unpack_s2_wgrad extracts the 9 real taps. */
extern "C" int hb200_conv_s2_wgrad_supported(int c, int n, int h, int w) {
  return c == 32 && n == 64 && h % (2 * TH) == 0 && w % (2 * TW) == 0;
}
extern "C" int hb200_conv_s2_wgrad(const hb200_bf16* x, const hb200_bf16* dy, float* dw_acc, int batch, int h, int w,
                                   int c, int n, hb200_stream_t stream) {
  HB_CHECK_ARG(x && dy && dw_acc && batch > 0, "conv_s2_wgrad: null pointer");
  HB_CHECK_ARG(hb200_conv_s2_wgrad_supported(c, n, h, w), "conv_s2_wgrad: unsupported shape C=%d N=%d %dx%d", c, n, h, w);
  HaloWgradArgs a;
  a.x = (const __nv_bfloat16*)x; a.dy = (const __nv_bfloat16*)dy; a.dw = dw_acc;
  a.B = batch; a.H = h / 2; a.W = w / 2;
  a.ntiles = batch * (a.H / TH) * (a.W / TW);
  return launch_halo_wgrad<128, 64, 2, 2, 1, 2>(a, (cudaStream_t)stream);
}
extern "C" int hb200_unpack_s2_wgrad(const float* dw_acc, float* dw_oihw, int co, int ci, hb200_stream_t stream) {
  HB_CHECK_ARG(dw_acc && dw_oihw && co > 0 && ci > 0, "unpack_s2_wgrad: bad args");
  unpack_s2_wgrad_kernel<<<cdiv(co * ci * 9, 256), 256, 0, (cudaStream_t)stream>>>(dw_acc, dw_oihw, co, ci);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

extern "C" int hb200_conv_halo_wgrad(const hb200_bf16* x, const hb200_bf16* dy, float* dw_acc, int batch, int h,
                                     int w, int c, int n, int k, hb200_stream_t stream) {
  HB_CHECK_ARG(x && dy && dw_acc, "conv_halo_wgrad: null pointer");
  HB_CHECK_ARG(hb200_conv_halo_wgrad_supported(c, n, k, h, w), "conv_halo_wgrad: unsupported shape C=%d N=%d k=%d %dx%d", c, n, k, h, w);
  if (!hb200_conv_halo_supported(c, n, k, h, w)) {   // small images: several images per tile, sliced channels
    HaloWgradSmallArgs s;
    s.x = (const grad_t*)x; s.dy = (const grad_t*)dy; s.dw = dw_acc;
    s.B = batch; s.Ci = c; s.Co = n;
    const int ipt = TH / h;
    s.ntiles = (batch + ipt - 1) / ipt;
    return h == 8 ? launch_halo_wgrad_small<128, 8>(s, (cudaStream_t)stream) : launch_halo_wgrad_small<128, 4>(s, (cudaStream_t)stream);
  }
  HaloWgradArgs a;
  a.x = (const __nv_bfloat16*)x; a.dy = (const __nv_bfloat16*)dy; a.dw = dw_acc;
  a.B = batch; a.H = h; a.W = w;
  a.ntiles = batch * (h / TH) * (w / TW);
  cudaStream_t st = (cudaStream_t)stream;
  // x halo: 0 = registers (C <= 32) / cp.async, 1 = one 5-D TMA box per tile (HB200_WGRAD_XTMA / hb200_set_wgrad_xtma)
  if (g_wgrad_xtma) {
    if (k == 3 && c == 32) return launch_halo_wgrad<32, 32, 3, 3, 1, 1>(a, st);
    if (k == 3 && c == 64) return launch_halo_wgrad<64, 64, 3, 3, 1, 1>(a, st);
    return launch_halo_wgrad<16, 32, 4, 4, 2, 1>(a, st);
  }
  if (k == 3 && c == 32) return launch_halo_wgrad<32, 32, 3, 3, 1>(a, st);
  if (k == 3 && c == 64) return launch_halo_wgrad<64, 64, 3, 3, 1>(a, st);
  return launch_halo_wgrad<16, 32, 4, 4, 2>(a, st);
}
extern "C" int hb200_set_wgrad_xtma(int on) { g_wgrad_xtma = on ? 1 : 0; return HB200_OK; }
extern "C" int hb200_get_wgrad_xtma(void) { return g_wgrad_xtma; }
