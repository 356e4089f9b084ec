// hb200 -- "halo" convolution kernels for the stride-1 layers that dominate the encoder's time
// (3x3 pad-1 convs of layer1/layer2, and the 7x7 stride-2 stem re-expressed as a 4x4 stride-1 conv
// over the space-to-depth input).
//
// The first-generation kernel (conv.cu) gathers an im2col tile per K chunk, so every input element
// crosses L2 -> shared memory 9 times (L2-bound, the tensor pipe mostly idle).  Here each CTA loads the
// (16+KH-1) x (8+KW-1) input halo of a 16x8 output tile ONCE into shared memory, and every filter tap is just a
// different wgmma shared-memory descriptor over that one buffer (the forward / dgrad layouts are described at
// conv_halo_ws_kernel).  The weight gradient stores the halo as
//
//        offset(hy, cj, hx) = ((hy * C/8 + cj) * HW + hx) * 16 bytes        (16 B = 8 channels)
//
// and reads it MN-major: rows = (r, ci) with row-block stride P (because RP = C/8 * P the three vertical taps are ONE
// affine M dimension), K = 16 pixels (2 tile rows), with P = HW*16, RP = (C/8)*P.  The no-swizzle descriptor mode is
// what makes this legal: shifting the start address by one pixel (16 B) keeps every core matrix 8 x 16 B contiguous.
//
// CTAs are persistent (weights or accumulators stay resident across tiles); the halo of later tiles arrives by TMA
// (padding = the out-of-bounds zero fill) while the MMAs and the epilogue of earlier tiles run.
// A warpgroup owns the 128 x N accumulator of a tile in registers (wgmma.cuh).
#include <cuda.h>

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
  static constexpr int W_BYTES = KH * KW * C * N * 2;
};

// ------------------------------------------------------------------------------------------
// weight gradient on the same halo buffer.  rows = (r, ci) [vertical taps form one affine M dim],
// one accumulator per horizontal tap s and per 128-row M tile; K = output pixels.
// ------------------------------------------------------------------------------------------
// ring depth of conv_halo_wgrad_kernel: 4 stages where they fit beside the 17 KB accumulator transpose buffer, else 3
constexpr int halo_wgrad_stages(int c, int stage_bytes) {
  return c >= 64 ? (4 * stage_bytes <= 200 * 1024 ? 4 : 3) : 2;
}

struct HaloWgradArgs {
  const __nv_bfloat16* x;   // [B,H,W,C]
  const __nv_bfloat16* dy;  // [B,H,W,N]
  float* dw;                // partials [blockIdx.x][(r*KW+s)*C + ci][N], summed in order by reduce_partials
  int B, H, W, ntiles;
};

// XMODE: how the x halo reaches shared memory.  1 = one 5-D TMA box over x viewed as
// [B, H, C/8, W, 8] (box = 8 channels x HWD pixels x C/8 chunks x halo rows = exactly the [row][chunk][pixel] layout the
// shifted descriptors read).  2 = the same over the 2x2 SPACE-TO-DEPTH view of a tensor with C/4 real channels: a
// 3x3 stride-2 pad-1 conv of x is a 2x2 stride-1 pad-1 conv of the view (csrc/conv_s2.cu), whose block row `by` is image
// rows 2by, 2by+1 -- the box simply covers twice the rows of the real tensor with (dx, c) as the chunk dimension.
template <int C, int N, int KH, int KW, int PAD, int XMODE>
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
  constexpr int NSW = halo_wgrad_stages(C, STAGE);
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
  // dy tile: ONE TMA box (N channels x 8 x 16 pixels) into the MN-major swizzled layout -- as LDGSTS it was a transpose
  // (pixel-major tensor -> channel-chunk-major rows), 2 shared-memory wavefronts per 16-byte copy, which made this kernel
  // LSU-bound (see the small-image kernel below).
  auto commit_tile = [&, tmap_p, tmap_xp](int tile, int st) {   // stage `st` is free: x halo and dy tile by TMA
    int b, oh0, ow0;
    tile_coords(tile, b, oh0, ow0);
    const uint32_t sd = sbase + st * STAGE;
    if (tid == 0) {
      mbar_expect_tx(&dy_bar[st], (uint32_t)(DY_BYTES + HROWS_LOAD * RP));
      tma_load_4d(sd, tmap_p, &dy_bar[st], 0, ow0, oh0, b);
      // coordinates (channel-in-chunk, pixel column, chunk, row, frame); space-to-depth: rows of the REAL tensor
      if (XMODE == 1) tma_load_5d(sd + DY_BYTES, tmap_xp, &dy_bar[st], 0, ow0 - PAD, 0, oh0 - PAD, b);
      if (XMODE == 2) tma_load_5d(sd + DY_BYTES, tmap_xp, &dy_bar[st], 0, ow0 - PAD, 0, 2 * (oh0 - PAD), b);
    }
  };
  const int first = blockIdx.x, stride = gridDim.x;
  const int my_n = first < a.ntiles ? (a.ntiles - first + stride - 1) / stride : 0;
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

  // both operands by TMA: thread 0 keeps NSW-1 tiles of loads ahead of the tensor core
  if (tid == 0)
    for (int p = 0; p < NSW - 1 && p < my_n; ++p) commit_tile(first + p * stride, p);
  for (int it = 0; it < my_n; ++it) {
    const int nxt = it + NSW - 1;   // its stage was read by the MMAs of tile it-1, complete
    if (tid == 0 && nxt < my_n) commit_tile(first + nxt * stride, nxt % NSW);
    mbar_wait(&dy_bar[it % NSW], (it / NSW) & 1);
    mma_tile(it, sbase + (it % NSW) * STAGE);
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
// weight gradient of the 3x3 pad-1 stride-1 convs on SMALL images (8x8: layer3; 4x4: layer4 / compression; the
// Bottleneck / ResNeXt 3x3s and the compression of configs #3 / #4).  Per tap (r, s) it is a GEMM with M = input
// channels (no padding rows), N = output channels and K = output pixels.  A stage is one 16 x 8 output tile, i.e. 16 / IMG
// stacked images, and a K16 step is two of its 8-column rows, in this order: 16 real pixels (two rows of an 8x8 image),
// or two 4-pixel rows of a 4x4 image each followed by 4 columns of zero dy.  That is the K grouping, MMA order, tile ->
// worker assignment and partial layout of the halo tiling earlier versions used, so every fp32 addition is the same and
// the weight gradients are bit for bit what they were (a 4x4 image per K16 would halve the MMAs at 4x4, but round
// differently and change the training trajectory).
//   dy  [64-channel block][pixel][128 B]: TMA box {64 ch, 8 columns, IMG rows, images}, SWIZZLE_128B = the MN-major B
//       layout; columns 4..7 of a 4x4 image are outside the tensor and zero-filled.
//   x   [8-channel chunk][image][padded row][pixel][8 ch]: ONE 5-D TMA box of x viewed as (8 ch | column | row | frame |
//       chunk), columns starting at s - 1 and rows at -1.  The horizontal tap s is thereby pre-shifted into the copy, and
//       the out-of-bounds fill writes the zero columns of the padding, one zero row above and below every image, the
//       frames past B (ragged last tile) and the channels past Ci (a 32-channel last block).
//       A (MN-major, no swizzle) of tap (r, s) starts r rows into an image; its K8 halves start one row apart (LBO =
//       one row): an 8-pixel row, or a 4-pixel row followed by the next row's 4 pixels, which meet zero dy.  The
//       8-channel blocks of M sit at the uniform chunk stride (SBO).  The last 4x4 K8 half of a stage reads one row past
//       its chunk: the next chunk's zero padding row, or after the last chunk a gap zeroed once at the start (TMA never
//       writes it), so the products there are finite x 0.
// A CTA owns one (64-channel ci block, horizontal tap s, 128-column co block) slice.  Warp 12 is the producer (one
// thread issues the TMA into an NS-deep full / empty mbarrier ring); consumer warpgroup r = 0..2 owns tap (r, s) as a
// 64 x 128 register accumulator that persists over all of the worker's tiles, so one loaded stage feeds three taps.
// The consumers only issue MMAs and release stages (one wgmma group kept in flight across stage boundaries).  Tiles are
// strided statically over the workers (blockIdx.x); each worker writes its partial, summed in worker order by
// reduce_partials: the same result every run.
// ------------------------------------------------------------------------------------------
// 13 warps: three consumer warpgroups and the producer warp.  Accumulators are 64 x 128 (64 registers per thread): a
// 64 x 256 one spills and serialises the MMAs at the 152 registers 416 threads can have (setmaxnreg needs whole
// warpgroups, and ptxas allocates within the launch bound anyway).
constexpr int kWgradSmallThreads = 416;
constexpr int kWgradSmallCols = 128;   // output channels per CTA slice
struct WgradSmallArgs {
  float* dw;   // partials [blockIdx.x][(r*3+s)*Ci + ci][Co], summed in order by reduce_partials
  int Ci, Co, ntiles;
};

template <int IMG>
struct WgradSmallCfg {
  static constexpr int NIMG = TH / IMG;                       // images per stage: one 16 x 8 tile, 8 K16 steps
  static constexpr int ROWB = IMG * 16;                       // one padded row of one 8-channel chunk
  static constexpr int CHUNK = NIMG * (IMG + 2) * ROWB;       // one 8-channel chunk of the stage (A's SBO)
  static constexpr int XB = 8 * CHUNK;                        // 64 input channels
  static constexpr int DYBLK = TH * TW * 128;                 // one 64-channel block of dy: 128 pixels x 128 B
  static constexpr int DYB = kWgradSmallCols / 64 * DYBLK;
  static constexpr int GAP = 1024;                            // zeroed, behind x (the over-read above); keeps alignment
  static constexpr int STAGE = DYB + XB + GAP;                // dy first: its 1024-byte swizzle atoms stay aligned
  static constexpr int NS_FIT = (227 * 1024 - 1024 - 256) / STAGE;
  static constexpr int NS = NS_FIT < 8 ? NS_FIT : 8;
  static constexpr size_t SMEM = (size_t)NS * STAGE + 1024;
  static_assert(XB % 1024 == 0 && NS >= 3, "stage layout");
};

template <int IMG>
__global__ void __launch_bounds__(kWgradSmallThreads, 1)
conv_wgrad_small_ws_kernel(const WgradSmallArgs a, const __grid_constant__ CUtensorMap tmap_dy,
                           const __grid_constant__ CUtensorMap tmap_x) {
  using Cfg = WgradSmallCfg<IMG>;
  constexpr int NS = Cfg::NS, STAGE = Cfg::STAGE, NCO = kWgradSmallCols;
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[NS], empty_bar[NS];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const int tid = threadIdx.x, wg_id = tid >> 7, t = tid & 127;
  const int nci = (a.Ci + 63) / 64;
  const int s_tap = blockIdx.y % 3, cb = (blockIdx.y / 3) % nci, nb = blockIdx.y / (3 * nci);
  if (tid == 0) {
#pragma unroll
    for (int i = 0; i < NS; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 3);   // one arrival per consumer warpgroup
    }
    mbar_fence_init();
  }
  if (tid < NS * 8)   // the first 128 bytes of every stage's gap
    asm volatile("st.shared.v4.b32 [%0], {%1,%1,%1,%1};" ::"r"(sbase + (tid / 8) * STAGE + Cfg::DYB + Cfg::XB + (tid % 8) * 16),
                 "r"(0u) : "memory");
  fence_proxy_async_smem();   // st.shared (generic proxy) -> wgmma reads (async proxy)
  __syncthreads();
  const int first = blockIdx.x, stride = gridDim.x;
  const int my_n = first < a.ntiles ? (a.ntiles - first + stride - 1) / stride : 0;

  if (wg_id == 3) {
    if (t == 0) {
      const CUtensorMap* const pd = &tmap_dy;   // param-space addresses, taken in the kernel body
      const CUtensorMap* const px = &tmap_x;
      for (int it = 0; it < my_n; ++it) {
        const int st = it % NS;
        if (it >= NS) mbar_wait(&empty_bar[st], ((it / NS) - 1) & 1);
        const int b0 = (first + it * stride) * Cfg::NIMG;
        const uint32_t sd = sbase + (uint32_t)st * STAGE;
        mbar_expect_tx(&full_bar[st], (uint32_t)(Cfg::DYB + Cfg::XB));   // the gap is not loaded
#pragma unroll
        for (int j = 0; j < NCO / 64; ++j)
          tma_load_4d(sd + (uint32_t)j * Cfg::DYBLK, pd, &full_bar[st], nb * NCO + j * 64, 0, 0, b0);
        tma_load_5d(sd + Cfg::DYB, px, &full_bar[st], 0, s_tap - 1, -1, b0, cb * 8);
      }
    }
  } else {
    const int r = wg_id;   // vertical tap of this warpgroup's accumulator
    float acc[NCO / 2];
    for (int it = 0; it < my_n; ++it) {
      const int st = it % NS;
      mbar_wait(&full_bar[st], (it / NS) & 1);
      const uint32_t sd = sbase + (uint32_t)st * STAGE, sx = sd + Cfg::DYB;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < TH / 2; ++k) {
        // tile rows 2k, 2k+1 = image j, output rows oh0, oh0 + 1 (IMG is even: never straddles an image); tap r = r
        // rows further down
        const int j = (2 * k) / IMG, oh0 = (2 * k) % IMG;
        const uint64_t da = make_smem_desc(sx + (uint32_t)((j * (IMG + 2) + oh0 + r) * Cfg::ROWB), Cfg::ROWB, Cfg::CHUNK,
                                           kNoSwizzle);
        // B: MN-major, 128-byte swizzle: K16 = 2 groups of 8 pixel rows (SBO 1024 B), LBO = next 64-channel block
        const uint64_t db = make_smem_desc(sd + (uint32_t)k * 2048, Cfg::DYBLK, 1024, kSwizzle128B);
        Wgmma<NCO, kBF16>::template mma<1, 1>(acc, da, db, (it > 0 || k > 0) ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<1>();   // the MMAs of tile it-1 have read their stage: release it to the producer
      if (it > 0 && t == 0) mbar_arrive(&empty_bar[(it - 1) % NS]);
    }
    wgmma_wait<0>();
    if (my_n == 0) {   // a worker without tiles still writes its (zero) partial
#pragma unroll
      for (int i = 0; i < NCO / 2; ++i) acc[i] = 0.f;
    }
    acc_fence(acc);
    // fragment: rows 16w + l/4 (+8), columns 8i + 2(l%4) (+1); 4 lanes write one 32-byte sector
    const int w = t >> 5, l = t & 31;
    const int ci = cb * 64 + 16 * w + (l >> 2);
    float* const dst = a.dw + ((size_t)blockIdx.x * 9 * a.Ci + (size_t)(r * 3 + s_tap) * a.Ci + ci) * a.Co +
                       nb * NCO + 2 * (l & 3);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      if (ci + 8 * h < a.Ci) {
#pragma unroll
        for (int i = 0; i < NCO / 8; ++i)
          *reinterpret_cast<float2*>(dst + (size_t)(8 * h) * a.Co + 8 * i) = make_float2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
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

// ---- forward / dgrad: persistent, warp-specialised, halo by TMA ------------------------------------------------------
// One thread issues the halo's TMA box copies per tile (the conv padding is the TMA unit's out-of-bounds zero fill),
// which complete on an mbarrier.  A zero-filling cp.async gather needs ~6 predicated copies per thread per tile, and
// that address / predicate arithmetic made the 32-channel kernel issue-bound.  The halo lands in one of two layouts:
//   slabs (SW = false, the stem): C/8 boxes of {8 channels, halo width, halo height}, i.e. [cj][hy][hx][8 ch]; tap (r, s)
//        reads  start = stage + 2kk*SLAB + r*HWD*16 + s*16,  LBO = SLAB (next 8 channels),  SBO = HWD*16 (next tile row)
//   swizzled rows (SW = true, the 32- / 64-channel layers): KW copies of the tile rows, copy kx pre-shifted by kx
//        pixels, each [HH rows][8 pixels][C channels] in the 64- / 128-byte-swizzle K-major layout, one box per copy.
//        Its rows of C*2 bytes replace the 16-byte pieces of the slabs, whose rate -- not bytes -- bounds a slab-fed
//        kernel; tap (r, s) is copy s shifted by r whole swizzle atoms: aligned descriptors only, at KW times the bytes.
// With load -> MMA -> epilogue of consecutive tiles in one program order, the TMA latency of tile it+1 is exposed after
// every tile, and only a second CTA of the SM hides it.  Here the loads run in their own warp and meet the consumers
// only at mbarriers:
//   warp 8 (one lane)  producer: halo stage ring, NS deep
//   warps 0-3, 4-7     two consumer warpgroups; tile `it` of the CTA goes to warpgroup it & 1.  Each waits full[stage],
//                      issues the tile's MMAs, releases the stage (empty[stage]) as soon as they complete, then runs the
//                      GroupNorm sums / addend / pack / store while the other warpgroup's MMAs run on the next tile
// The accumulator lives in registers, so one warpgroup cannot overlap its own epilogue with MMAs: the second one is what
// keeps the tensor core busy.  Each warpgroup transposes through its own stage buffer (dynamic shared memory, after the
// halo ring) under its own named barrier (1 + warpgroup).
constexpr int kHaloWsThreads = 288;
template <int C, int N, int KH, int KW, int PAD, int MODE, int NS, bool SW = false>
__global__ void __launch_bounds__(kHaloWsThreads)
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
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;   // swizzle atoms are 1024-byte aligned
  const uint32_t s_w = sbase;
  const uint32_t s_halo0 = s_w + Cfg::W_BYTES;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  float* const stage_bufs = reinterpret_cast<float*>(smem_raw + (s_halo0 + NS * STAGE - smem_u32(smem_raw)));
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

  if (warp == 8) {
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
    const int wgi = warp >> 2, t = tid & 127;
    const int py = t >> 3, px = t & 7;
    float* const stage_buf = stage_bufs + wgi * kStageFloats;
    float acc_t[N];
    for (int it = wgi; it < my_n; it += 2) {
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
      if (t == 0) mbar_arrive(&empty_bar[st]);   // the halo stage is free: the producer may refill it
      const size_t pix = ((size_t)b * a.H + oh0 + py) * a.W + ow0 + px;
#pragma unroll
      for (int col0 = 0; col0 < N; col0 += 32) {
        float acc_[32];
        acc_row32(acc_t, col0, stage_buf, acc_, 1 + wgi);
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

static int blocks_per_sm(const void* kern, size_t smem, int* cache, int threads = 128) {
  if (*cache > 0) return *cache;
  cudaFuncAttributes fa;
  if (cudaFuncGetAttributes(&fa, kern) != cudaSuccess) return 1;
  const int regs = fa.numRegs > 0 ? fa.numRegs : 128;
  int by_regs = 65536 / (((regs + 7) / 8 * 8) * threads);
  int by_smem = (int)((227 * 1024) / (smem + fa.sharedSizeBytes + 1024));
  int n = by_regs < by_smem ? by_regs : by_smem;
  if (n > 16) n = 16;
  if (n < 1) n = 1;
  *cache = n;
  return n;
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
  // weights | NS halo stages | one transpose stage buffer per consumer warpgroup (+ 1024 for the alignment of the base)
  const size_t smem = Cfg::W_BYTES + (size_t)NS * stage + 2 * kStageFloats * sizeof(float) + 1024;
  auto kern = conv_halo_ws_kernel<C, N, KH, KW, PAD, MODE, NS, SW>;
  static int grid_cache = 0;
  if (grid_cache == 0) {
    HB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    // resident CTAs per SM from the static limits (registers of 288 threads, shared memory)
    cudaFuncAttributes fa;
    HB_CUDA(cudaFuncGetAttributes(&fa, (const void*)kern));
    const int regs = fa.numRegs > 0 ? fa.numRegs : 128;
    int per_sm = 65536 / (((regs + 7) / 8 * 8) * kHaloWsThreads);
    const int by_smem = (int)((227 * 1024) / (smem + fa.sharedSizeBytes + 1024));
    if (by_smem < per_sm) per_sm = by_smem;
    if (per_sm < 1) per_sm = 1;
    grid_cache = kNumSMs * per_sm;
  }
  const int grid = grid_cache < a.ntiles ? grid_cache : a.ntiles;
  kern<<<grid, kHaloWsThreads, smem, st>>>(a, tmap);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

template <int C, int N, int KH, int KW, int PAD, int XMODE>
static int launch_halo_wgrad(const HaloWgradArgs& a, cudaStream_t st) {
  constexpr int CJ = C / 8, HWD = TW + KW - 1, P = HWD * 16, RP = CJ * P;
  constexpr int MT = (KH * CJ + 15) / 16, RMAX = (MT * 16 + CJ - 1) / CJ, HROWS = TH - 1 + RMAX;
  constexpr int STAGE = (128 * N * 2 + HROWS * RP + 1023) / 1024 * 1024;
  constexpr int NSW = halo_wgrad_stages(C, STAGE);
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
  CUtensorMap tmap_x;
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

template <int IMG>
static int launch_wgrad_small(const grad_t* x, const grad_t* dy, float* dw, int B, int Ci, int Co, cudaStream_t st) {
  using Cfg = WgradSmallCfg<IMG>;
  EncodeTiledFn enc = halo_encode_fn();
  if (!enc) {
    set_last_error("conv_halo_wgrad (small images): cuTensorMapEncodeTiled is not available from this driver");
    return HB200_ERR_UNSUPPORTED;
  }
  // dy bf16 [B, IMG, IMG, Co]: box = 64 channels (one 128-byte swizzled row per pixel) x 8 columns x IMG rows x the
  // stage's images; columns / frames past the tensor are zero-filled (4x4 images, the ragged last tile)
  CUtensorMap tmap_dy, tmap_x;
  const cuuint64_t dims[4] = {(cuuint64_t)Co, (cuuint64_t)IMG, (cuuint64_t)IMG, (cuuint64_t)B};
  const cuuint64_t strides[3] = {(cuuint64_t)Co * 2, (cuuint64_t)IMG * Co * 2, (cuuint64_t)IMG * IMG * Co * 2};
  const cuuint32_t box[4] = {64u, (cuuint32_t)TW, (cuuint32_t)IMG, (cuuint32_t)Cfg::NIMG};
  const cuuint32_t estr[5] = {1u, 1u, 1u, 1u, 1u};
  CUresult r = enc(&tmap_dy, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, (void*)dy, dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("conv_halo_wgrad (small images): cuTensorMapEncodeTiled (dy) failed (%d)", (int)r);
    return HB200_ERR_CUDA;
  }
  // x bf16 [B, IMG, IMG, Ci] seen as (8 ch | column | row | frame | chunk): box = 8 ch x IMG columns x IMG + 2 rows x
  // the stage's images x 8 chunks, i.e. [chunk][image][padded row][pixel][8 ch] in shared memory
  const cuuint64_t xd[5] = {8u, (cuuint64_t)IMG, (cuuint64_t)IMG, (cuuint64_t)B, (cuuint64_t)(Ci / 8)};
  const cuuint64_t xs[4] = {(cuuint64_t)Ci * 2, (cuuint64_t)IMG * Ci * 2, (cuuint64_t)IMG * IMG * Ci * 2, 16u};
  const cuuint32_t xb[5] = {8u, (cuuint32_t)IMG, (cuuint32_t)(IMG + 2), (cuuint32_t)Cfg::NIMG, 8u};
  r = enc(&tmap_x, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, (void*)x, xd, xs, xb, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
          CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("conv_halo_wgrad (small images): cuTensorMapEncodeTiled (x) failed (%d)", (int)r);
    return HB200_ERR_CUDA;
  }
  auto kern = conv_wgrad_small_ws_kernel<IMG>;
  static int cache = 0;
  if (cache == 0) HB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Cfg::SMEM));
  // the grid is sized from the CTAs that fit per SM (registers of 416 threads, the stage ring): one here
  const int per_sm = blocks_per_sm((const void*)kern, Cfg::SMEM, &cache, kWgradSmallThreads);
  const int ntiles = (B + Cfg::NIMG - 1) / Cfg::NIMG;
  const int slices = (Ci + 63) / 64 * 3 * (Co / kWgradSmallCols);   // (ci block, horizontal tap, co block)
  int workers = kNumSMs * per_sm / slices;
  if (workers < 1) workers = 1;
  if (workers > ntiles) workers = ntiles;
  // one partial per worker, summed in worker order into the caller's accumulator (deterministic)
  const long long count = 9LL * Ci * Co;
  float* parts = nullptr;
  int* tickets = nullptr;
  int rc = stream_workspace(st, (size_t)(workers + (workers < kReduceChunks ? workers : kReduceChunks)) * count, 0, &parts,
                            &tickets);
  if (rc) return rc;
  WgradSmallArgs a;
  a.dw = parts; a.Ci = Ci; a.Co = Co; a.ntiles = ntiles;
  kern<<<dim3(workers, slices), kWgradSmallThreads, Cfg::SMEM, st>>>(a, tmap_dy, tmap_x);
  HB_LAUNCH_OK();
  count_launch(1);
  return reduce_partials(parts, workers, count, count, dw, parts + (size_t)workers * count, st);
}
}  // namespace hb200

using namespace hb200;

/* which (C, N, k) combinations have a halo instantiation */
extern "C" int hb200_conv_halo_supported(int c, int n, int k, int h, int w) {
  if (h % TH || w % TW) return 0;
  if (k == 3) return (c == 32 && n == 32) || (c == 64 && n == 64);
  if (k == 4) return c == 16 && n == 32;
  return 0;
}

/* weight-gradient variant: additionally the small-image layers (8x8 / 4x4, channels sliced 64 x 128) */
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
  if (k == 3 && c == 64)
    return mode == 0 ? launch_halo_ws<64, 64, 3, 3, 1, 0, 2, true>(a, st) : launch_halo_ws<64, 64, 3, 3, 1, 1, 2, true>(a, st);
  if (k == 3 && c == 32)   // one CTA per SM: 18 KB of weights, 6 halo stages, 2 transpose buffers
    return mode == 0 ? launch_halo_ws<32, 32, 3, 3, 1, 0, 6, true>(a, st) : launch_halo_ws<32, 32, 3, 3, 1, 1, 6, true>(a, st);
  HB_CHECK_ARG(mode == 0, "conv_halo: the stem has no data gradient");
  return launch_halo_ws<16, 32, 4, 4, 2, 0, 6>(a, st);
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
  if (!hb200_conv_halo_supported(c, n, k, h, w)) {   // small images: 16x8 tiles of stacked images, sliced channels
    const grad_t* xg = (const grad_t*)x;
    const grad_t* dyg = (const grad_t*)dy;
    cudaStream_t st = (cudaStream_t)stream;
    return h == 8 ? launch_wgrad_small<8>(xg, dyg, dw_acc, batch, c, n, st) : launch_wgrad_small<4>(xg, dyg, dw_acc, batch, c, n, st);
  }
  HaloWgradArgs a;
  a.x = (const __nv_bfloat16*)x; a.dy = (const __nv_bfloat16*)dy; a.dw = dw_acc;
  a.B = batch; a.H = h; a.W = w;
  a.ntiles = batch * (h / TH) * (w / TW);
  cudaStream_t st = (cudaStream_t)stream;
  if (k == 3 && c == 32) return launch_halo_wgrad<32, 32, 3, 3, 1, 1>(a, st);
  if (k == 3 && c == 64) return launch_halo_wgrad<64, 64, 3, 3, 1, 1>(a, st);
  return launch_halo_wgrad<16, 32, 4, 4, 2, 1>(a, st);
}
