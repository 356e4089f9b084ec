// hb200 -- the stride-2 block entry of the ResNet encoder (BasicBlock with a downsample branch,
// HB/rl/ddppo/policy/resnet.py:26-77 + :143-160) as ONE TMA-fed halo kernel launch per direction:
//
//   forward :  ya = conv3x3_s2_p1(x, Wa)   yb = conv1x1_s2(x, Wb)          x [B,H,W,C]  ->  ya, yb [B,H/2,W/2,NA|NB]
//   dgrad   :  dx = conv3x3_s2^T(dya, Wa) + conv1x1_s2^T(dyb, Wb)           (both branches read the same x)
//
// Stride 2 is removed by reading x as its 2x2 space-to-depth view xs [B,H/2,W/2,(dy,dx,c)]: input row 2*oy + r - 1 of
// filter row r is sub-row dy(r) of block row oy - 1 + ky(r) with (ky,dy) = (0,1), (1,0), (1,1) for r = 0, 1, 2 -- so a
// 3x3 stride-2 tap is a 2x2 stride-1 tap restricted to ONE (dy,dx) channel block, and the 1x1 stride-2 branch is the
// centre tap with its own output columns.  TMA loads the view straight from the NHWC tensor with a 5-D map
// (dims (dx,c) | bx | dy | by | b): no space-to-depth copy, no im2col, padding = out-of-range zero fill.
// Both branches share the halo tile and the accumulator: output columns [0,NA) | [NA,NA+NB).
//
// On the gather kernel (conv_igemm) these two convolutions of layer2.0 are 8192 / 32768 CTAs with 1-5 K chunks each at
// 4096 frames: fixed per-CTA costs dominate.
#include <cuda.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace hb200 {
void count_launch(int n);
using namespace wg;

namespace {
constexpr int S2_TH = 16, S2_TW = 8;  // tile: 16 x 8 output pixels (forward) / 2x2 input blocks (dgrad) = MMA M

__device__ __forceinline__ float s2_warp_reduce16(float (&v)[16], int lane) {
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
__device__ __forceinline__ float s2_warp_reduce32(float (&v)[32], int lane) {
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
__device__ __forceinline__ void s2_gn_stats_chunk(const float (&acc)[32], int lane, int cpg, double* stats_b, int ch0) {
  if (cpg == 2) {
    float v[32];
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      v[i] = acc[2 * i] + acc[2 * i + 1];
      v[16 + i] = acc[2 * i] * acc[2 * i] + acc[2 * i + 1] * acc[2 * i + 1];
    }
    const float t = s2_warp_reduce32(v, lane);   // lane < 16: sum of group lane; else sum of squares of group lane-16
    atomicAdd(stats_b + ((ch0 >> 1) + (lane & 15)) * 2 + (lane >> 4), (double)t);
  } else if (cpg == 4) {
    float v[16];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float a0 = acc[4 * i], a1 = acc[4 * i + 1], a2 = acc[4 * i + 2], a3 = acc[4 * i + 3];
      v[i] = (a0 + a1) + (a2 + a3);
      v[8 + i] = (a0 * a0 + a1 * a1) + (a2 * a2 + a3 * a3);
    }
    const float t = s2_warp_reduce16(v, lane);        // lanes 2i, 2i+1 hold value i
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
    const float ts = s2_warp_reduce16(s2, lane), tq = s2_warp_reduce16(q2, lane);
    if ((lane & 1) == 0) {
      double* dst = stats_b + ((ch0 + lane) / cpg) * 2;
      atomicAdd(dst, (double)ts);
      atomicAdd(dst + 1, (double)tq);
    }
  }
}

struct S2Args {
  const void* wimg;            // weight image (forward: fp16 [9][C/8][N][8]; dgrad: bf16 [9][N/8][C][8])
  void* ya; void* yb;          // forward outputs fp16 [B,Ho,Wo,NA] / [B,Ho,Wo,NB]; dgrad: ya = dx bf16 [B,H,W,C]
  const void* addend;          // dgrad: optional bf16 [B,H,W,C] added to dx
  double* stats_a; double* stats_b;   // forward: GroupNorm sums [B,G,2] per branch (optional)
  int B, Ho, Wo, groups_a, groups_b, ntiles;
};

// filter row / column r -> (halo shift k, sub-row d) of the space-to-depth view
__host__ __device__ constexpr int s2_k(int r) { return r == 0 ? 0 : 1; }
__host__ __device__ constexpr int s2_d(int r) { return r == 0 ? 1 : r - 1; }

// ---- forward / dgrad: warp-specialised, swizzled pixel-row copies ------------------------------------------------------
// A stage holds FOUR copies of the tile rows, each [17 rows][8 pixels][128 B] in the 128-byte-swizzle K-major layout, one
// TMA box each.  The 128-byte rows are 8x fewer TMA pieces than 8-channel slabs of 16 bytes, whose rate bounds a
// slab-fed kernel:
//   forward: copy (dy, kx) = sub-row dy of the space-to-depth view, pre-shifted by kx block columns; a filter tap (r, s) reads
//            copy (dy(r), kx(s)) shifted by ky(r) whole atoms, K offset dx(s) * 64 B inside the 128-byte (dx, c) row
//   dgrad:   copy (t, kx) = tensor t of (dya | dyb) pre-shifted by kx; K block kk of the 128 reduction channels reads
//            tensor kk / 4 at K offset (kk % 4) * 32 B
// B is the 3x3 weight image of the concatenated filters [NA + NB, C, 3, 3] (Wb sits in the centre tap).  The dgrad tile is
// 16 x 8 input BLOCKS (2x2 pixels each) over block rows by .. by+1 of the gradients (no top / left pad; bottom / right
// out-of-range = zero fill).  Output sub-pixel (dy,dx) of a block owns one accumulator and receives the filter taps with
// r = dy+1 (mod 2): r = 1 from output row by, r = 0 from by+1, r = 2 from by.  Its B = [tap][n/8][c][8] bf16
// (hb200_pack_halo_weight mode 1 stores it flipped: tap (2-r, 2-s)).
// Warp 4 is the producer over an NS-deep stage ring; warps 0-3 (one warpgroup) issue the MMAs of a tile, release its
// stage and run the epilogue while the producer already loads the following tiles.
template <int C, int NA, int NB, int MODE, int NS>
__global__ void __launch_bounds__(160) conv_s2_ws_kernel(const S2Args a, const __grid_constant__ CUtensorMap tmap_a,
                                                         const __grid_constant__ CUtensorMap tmap_b) {
  constexpr int N = NA + NB, HH = S2_TH + 1;
  constexpr int NQ = MODE == 0 ? 1 : 4, NW = MODE == 0 ? N : C;   // accumulators of one tile x their width
  constexpr int NACC = NQ * NW;
  constexpr uint32_t ATOM = 8 * 128, COPY = HH * ATOM, STAGE = 4 * COPY;
  constexpr uint32_t W_BYTES = 9 * C * N * 2;
  static_assert(C == 32 && NA == 64 && NB == 64, "conv_s2_ws: 128-byte rows = (dx, c) of 32 channels / 64-channel gradients");
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[NS], empty_bar[NS];
  __shared__ float stage_buf[kStageFloats];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t s_w = sbase, s_halo = s_w + W_BYTES;   // W_BYTES = 72 KB: the stages stay 1024-byte aligned
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid == 0) {
#pragma unroll
    for (int i = 0; i < NS; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 1); }
    mbar_fence_init();
  }
  {
    const uint4* src = reinterpret_cast<const uint4*>(a.wimg);
    for (int v = tid; v < (int)(W_BYTES / 16); v += blockDim.x) cp_async16(s_w + (uint32_t)v * 16, src + v, true);
  }
  cp_async_commit();
  cp_async_wait<0>();
  fence_proxy_async_smem();
  __syncthreads();
  const int tiles_x = a.Wo / S2_TW, tiles_per_img = tiles_x * (a.Ho / S2_TH);
  const int first = blockIdx.x, stride = gridDim.x;
  const int my_n = first < a.ntiles ? (a.ntiles - first + stride - 1) / stride : 0;
  const CUtensorMap* const pa = &tmap_a;   // param-space addresses, taken in the kernel body
  const CUtensorMap* const pb = &tmap_b;

  if (warp == 4) {
    if (lane == 0) {
      for (int it = 0; it < my_n; ++it) {
        const int st = it % NS;
        if (it >= NS) mbar_wait(&empty_bar[st], ((it / NS) - 1) & 1);
        const int tile = first + it * stride;
        const int b = tile / tiles_per_img, r = tile - b * tiles_per_img;
        const int oh0 = (r / tiles_x) * S2_TH, ow0 = (r % tiles_x) * S2_TW;
        const uint32_t sh = s_halo + (uint32_t)st * STAGE;
        mbar_expect_tx(&full_bar[st], STAGE);
#pragma unroll
        for (int q = 0; q < 4; ++q) {   // q = (dy | tensor) * 2 + kx
          if (MODE == 0) tma_load_5d(sh + q * COPY, pa, &full_bar[st], 0, ow0 - 1 + (q & 1), q >> 1, oh0 - 1, b);
          else tma_load_4d(sh + q * COPY, (q >> 1) ? pb : pa, &full_bar[st], 0, ow0 + (q & 1), oh0, b);
        }
      }
    }
    __syncwarp();
  } else {
    const int py = tid >> 3, px = tid & 7;
    float acc_q[NQ][NW];
    for (int it = 0; it < my_n; ++it) {
      const int st = it % NS;
      const int tile = first + it * stride;
      const int b = tile / tiles_per_img, r = tile - b * tiles_per_img;
      const int oh0 = (r / tiles_x) * S2_TH, ow0 = (r % tiles_x) * S2_TW;
      mbar_wait(&full_bar[st], (it / NS) & 1);
      const uint32_t sh = s_halo + (uint32_t)st * STAGE;
      wgmma_fence();
      if (MODE == 0) {
        uint32_t accum = 0;
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
          for (int s = 0; s < 3; ++s)
#pragma unroll
            for (int kk = 0; kk < C / 16; ++kk) {
              const uint64_t da = make_smem_desc(sh + (s2_d(r) * 2 + s2_k(s)) * COPY + s2_k(r) * ATOM + s2_d(s) * 64 + kk * 32,
                                                 16, ATOM, kSwizzle128B);
              const uint64_t db = make_smem_desc(s_w + (r * 3 + s) * (C * N * 2) + 2 * kk * (N * 16), N * 16, 128,
                                                 kNoSwizzle);
              mma128<NW, kF16>(acc_q[0], da, 8 * ATOM, db, accum);
              accum = 1;
            }
      } else {
#pragma unroll
        for (int dy = 0; dy < 2; ++dy)
#pragma unroll
          for (int dx = 0; dx < 2; ++dx) {
            uint32_t accum = 0;
#pragma unroll
            for (int r = 0; r < 3; ++r) {
              if (((dy + 1 - r) & 1) != 0) continue;
#pragma unroll
              for (int s = 0; s < 3; ++s) {
                if (((dx + 1 - s) & 1) != 0) continue;
                const int ky = (dy + 1 - r) / 2, kx = (dx + 1 - s) / 2;
                const int tap = (2 - r) * 3 + (2 - s);
#pragma unroll
                for (int kk = 0; kk < N / 16; ++kk) {
                  const uint64_t da = make_smem_desc(sh + ((kk / 4) * 2 + kx) * COPY + ky * ATOM + (kk % 4) * 32, 16, ATOM,
                                                     kSwizzle128B);
                  const uint64_t db = make_smem_desc(s_w + tap * (C * N * 2) + 2 * kk * (C * 16), C * 16, 128, kNoSwizzle);
                  mma128<NW, kBF16>(acc_q[(dy * 2 + dx) % NQ], da, 8 * ATOM, db, accum);
                  accum = 1;
                }
              }
            }
          }
      }
      wgmma_commit();
      wgmma_wait<0>();
#pragma unroll
      for (int q = 0; q < NQ; ++q) acc_fence(acc_q[q]);
      if (tid == 0) mbar_arrive(&empty_bar[st]);   // the producer may refill this stage now
#pragma unroll
      for (int col0 = 0; col0 < NACC; col0 += 32) {
        float v[32];
        acc_row32(acc_q[col0 / NW], col0 % NW, stage_buf, v);
        if (MODE == 0) {
          const size_t pix = ((size_t)b * a.Ho + oh0 + py) * a.Wo + ow0 + px;
          const bool second = col0 >= NA;
          double* stats = second ? a.stats_b : a.stats_a;
          if (stats != nullptr) {
            const int groups = second ? a.groups_b : a.groups_a;
            s2_gn_stats_chunk(v, lane, (second ? NB : NA) / groups, stats + (size_t)b * groups * 2, col0 - (second ? NA : 0));
          }
          __half* out = second ? reinterpret_cast<__half*>(a.yb) + pix * NB + (col0 - NA)
                               : reinterpret_cast<__half*>(a.ya) + pix * NA + col0;
          uint4* dst = reinterpret_cast<uint4*>(out);
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            uint4 u;
            u.x = pack_f16x2(v[q * 8 + 0], v[q * 8 + 1]);
            u.y = pack_f16x2(v[q * 8 + 2], v[q * 8 + 3]);
            u.z = pack_f16x2(v[q * 8 + 4], v[q * 8 + 5]);
            u.w = pack_f16x2(v[q * 8 + 6], v[q * 8 + 7]);
            dst[q] = u;
          }
        } else {
          const int H = 2 * a.Ho, W = 2 * a.Wo;
          const int q4 = col0 / C, c0 = col0 - q4 * C;
          const size_t o = ((((size_t)b * H + 2 * (oh0 + py) + (q4 >> 1)) * W) + 2 * (ow0 + px) + (q4 & 1)) * C + c0;
          if (a.addend != nullptr) {
            const uint4* ad = reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(a.addend) + o);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              float f[8];
              unpack8(ad[q], f);
#pragma unroll
              for (int e = 0; e < 8; ++e) v[q * 8 + e] += f[e];
            }
          }
          uint4* dst = reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(a.ya) + o);
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            uint4 u;
            u.x = pack_bf16x2(v[q * 8 + 0], v[q * 8 + 1]);
            u.y = pack_bf16x2(v[q * 8 + 2], v[q * 8 + 3]);
            u.z = pack_bf16x2(v[q * 8 + 4], v[q * 8 + 5]);
            u.w = pack_bf16x2(v[q * 8 + 6], v[q * 8 + 7]);
            dst[q] = u;
          }
        }
      }
    }
  }
}

typedef CUresult (*S2EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                               const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                               CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
S2EncodeFn s2_encode_fn() {
  static S2EncodeFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
      q != cudaDriverEntryPointSuccess)
    return nullptr;
  fn = (S2EncodeFn)p;
  return fn;
}

}  // namespace
}  // namespace hb200

using namespace hb200;

extern "C" int hb200_conv_s2_supported(int c, int na, int nb, int h, int w) {
  return c == 32 && na == 64 && nb == 64 && h % (2 * S2_TH) == 0 && w % (2 * S2_TW) == 0;
}

extern "C" int hb200_conv_s2_fwd(const hb200_f16* x, const hb200_f16* wimg, hb200_f16* ya, hb200_f16* yb,
                                 double* stats_a, int groups_a, double* stats_b, int groups_b, int batch, int h, int w,
                                 int c, int na, int nb, hb200_stream_t stream) {
  HB_CHECK_ARG(x && wimg && ya && yb && batch > 0, "conv_s2_fwd: null pointer");
  HB_CHECK_ARG(hb200_conv_s2_supported(c, na, nb, h, w), "conv_s2_fwd: unsupported shape C=%d N=%d+%d %dx%d", c, na, nb, h, w);
  if (stats_a) HB_CHECK_ARG(groups_a > 0 && na % groups_a == 0 && na / groups_a >= 2, "conv_s2_fwd: bad GroupNorm groups");
  if (stats_b) HB_CHECK_ARG(groups_b > 0 && nb % groups_b == 0 && nb / groups_b >= 2, "conv_s2_fwd: bad GroupNorm groups");
  S2EncodeFn enc = s2_encode_fn();
  if (!enc) {
    set_last_error("conv_s2_fwd: cuTensorMapEncodeTiled is not available from this driver");
    return HB200_ERR_UNSUPPORTED;
  }
  // space-to-depth view of x [B,H,W,C] (2-byte elements): ((dx,c) | bx | dy | by | b)
  CUtensorMap tmap;
  const cuuint64_t dims[5] = {(cuuint64_t)2 * c, (cuuint64_t)w / 2, 2, (cuuint64_t)h / 2, (cuuint64_t)batch};
  const cuuint64_t strides[4] = {(cuuint64_t)2 * c * 2, (cuuint64_t)w * c * 2, (cuuint64_t)2 * w * c * 2,
                                 (cuuint64_t)h * w * c * 2};
  // whole 128-byte (dx, c) rows of 8 block columns, swizzled (one box per (dy, kx) copy)
  const cuuint32_t box[5] = {(cuuint32_t)(2 * c), (cuuint32_t)S2_TW, 1u, (cuuint32_t)(S2_TH + 1), 1u};
  const cuuint32_t estr[5] = {1u, 1u, 1u, 1u, 1u};
  const CUresult r = enc(&tmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, (void*)x, dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("conv_s2_fwd: cuTensorMapEncodeTiled failed (%d)", (int)r);
    return HB200_ERR_CUDA;
  }
  S2Args a;
  a.wimg = wimg; a.ya = ya; a.yb = yb; a.addend = nullptr; a.stats_a = stats_a; a.stats_b = stats_b;
  a.groups_a = groups_a > 0 ? groups_a : 1; a.groups_b = groups_b > 0 ? groups_b : 1;
  a.B = batch; a.Ho = h / 2; a.Wo = w / 2;
  a.ntiles = batch * (a.Ho / S2_TH) * (a.Wo / S2_TW);
  constexpr int C = 32, NA = 64, NB = 64, N = NA + NB, NS = 2;
  const size_t smem = 9 * C * N * 2 + NS * (size_t)(4 * (S2_TH + 1) * 8 * 128) + 1024;
  auto kern = conv_s2_ws_kernel<C, NA, NB, 0, NS>;
  static bool attr = false;
  if (!attr) {
    HB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr = true;
  }
  const int grid = kNumSMs < a.ntiles ? kNumSMs : a.ntiles;   // 209 KB of shared memory: one CTA per SM
  kern<<<grid, 160, smem, (cudaStream_t)stream>>>(a, tmap, tmap);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

extern "C" int hb200_conv_s2_dgrad(const hb200_bf16* dya, const hb200_bf16* dyb, const hb200_bf16* wimg_t,
                                   const hb200_bf16* addend, hb200_bf16* dx, int batch, int h, int w, int c, int na,
                                   int nb, hb200_stream_t stream) {
  HB_CHECK_ARG(dya && dyb && wimg_t && dx && batch > 0, "conv_s2_dgrad: null pointer");
  HB_CHECK_ARG(hb200_conv_s2_supported(c, na, nb, h, w), "conv_s2_dgrad: unsupported shape C=%d N=%d+%d %dx%d", c, na, nb, h, w);
  S2EncodeFn enc = s2_encode_fn();
  if (!enc) {
    set_last_error("conv_s2_dgrad: cuTensorMapEncodeTiled is not available from this driver");
    return HB200_ERR_UNSUPPORTED;
  }
  const int ho = h / 2, wo = w / 2;
  CUtensorMap ta, tb;
  const cuuint32_t box[4] = {64u, (cuuint32_t)S2_TW, (cuuint32_t)(S2_TH + 1), 1u};   // 128-byte pixel rows, swizzled
  const cuuint32_t estr[4] = {1u, 1u, 1u, 1u};
  for (int which = 0; which < 2; ++which) {
    const int n = which ? nb : na;
    const cuuint64_t dims[4] = {(cuuint64_t)n, (cuuint64_t)wo, (cuuint64_t)ho, (cuuint64_t)batch};
    const cuuint64_t strides[3] = {(cuuint64_t)n * 2, (cuuint64_t)wo * n * 2, (cuuint64_t)ho * wo * n * 2};
    const CUresult r = enc(which ? &tb : &ta, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, (void*)(which ? dyb : dya), dims,
                           strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                           CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      set_last_error("conv_s2_dgrad: cuTensorMapEncodeTiled failed (%d)", (int)r);
      return HB200_ERR_CUDA;
    }
  }
  S2Args a;
  a.wimg = wimg_t; a.ya = dx; a.yb = nullptr; a.addend = addend; a.stats_a = nullptr; a.stats_b = nullptr;
  a.groups_a = a.groups_b = 1;
  a.B = batch; a.Ho = ho; a.Wo = wo;
  a.ntiles = batch * (ho / S2_TH) * (wo / S2_TW);
  constexpr int C = 32, NA = 64, NB = 64, N = NA + NB, NS = 2;
  const size_t smem = 9 * C * N * 2 + NS * (size_t)(4 * (S2_TH + 1) * 8 * 128) + 1024;
  auto kern = conv_s2_ws_kernel<C, NA, NB, 1, NS>;
  static bool attr = false;
  if (!attr) {
    HB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr = true;
  }
  const int grid = kNumSMs < a.ntiles ? kNumSMs : a.ntiles;
  kern<<<grid, 160, smem, (cudaStream_t)stream>>>(a, ta, tb);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}
