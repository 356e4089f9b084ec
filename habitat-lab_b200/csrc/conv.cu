// hb200 -- implicit-GEMM convolution (forward, data gradient, weight gradient) on wgmma.
//
// One CTA = one warpgroup = one 128-row accumulator tile held in registers.  The im2col A tile is gathered from the
// NHWC activation tensor straight into shared memory with zero-filling cp.async (padding and stride handled by
// predication, never materialised), the weight tile is a pre-packed shared-memory image copied verbatim, the
// warpgroup issues wgmma (fp16 x fp16 or bf16 x bf16 -> f32) and the epilogue reads the tile row by row through a
// shared-memory transpose, fusing the GroupNorm statistics (sum / sum of squares per frame x group) or the
// residual-gradient add.
//
//   forward : D[pixel, co]    = sum_{r,s,ci} X[pixel@(r,s), ci] * W[co, r,s,ci]     (K-major)
//   dgrad   : D[pixel, ci]    = sum_{r,s,co} dY[pixel@(r,s), co] * W[co, r,s,ci]    (K-major)
//   wgrad   : D[(r,s,ci), co] = sum_{pixel}  X[pixel@(r,s), ci] * dY[pixel, co]     (MN-major,
//             split over pixel slabs, fp32 atomics into the accumulator)
//
// Shared-memory operand layout of the conv kernels and their weight images (128-byte swizzle, K-major): 16-byte vector
// (row, k8) at (row>>3)*1024 + (row&7)*128 + ((k8 ^ (row&7)) << 4).  hb200_umma_gemm_probe pins it on hardware, together
// with the no-swizzle descriptor forms the halo kernels use (probe layout 0: "interleaved" core matrices, vector (row, k8)
// at k8 * rows*16 + row*16, LBO = rows*16, SBO = 128).
#include <cuda.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace hb200 {
void count_launch(int n);

using namespace wg;

constexpr int kStages = 3;
constexpr int kTileM = 128;
constexpr int kMaxBN = 128;  // N tile: a 128 x 128 fp32 accumulator is 128 registers per thread of the warpgroup
constexpr int kChunkK = 64;  // bf16 elements per K chunk (8 x 16-byte vectors)
constexpr int kMaxChunks = 512;  // K = taps * Ci up to 32768 (the 3x3 compression conv of ResNet50 has K = 9 * 1024)

template <int LAYOUT>
__device__ __forceinline__ uint32_t tile_off(int row, int k8, int rows_total) {
  if (LAYOUT == 0) return (uint32_t)(k8 * rows_total + row) << 4;
  return (uint32_t)((row >> 3) << 10) + (uint32_t)((row & 7) << 7) + (uint32_t)((k8 ^ (row & 7)) << 4);
}
template <int LAYOUT>
__device__ __forceinline__ uint64_t kmajor_desc(uint32_t base, int kk, int rows_total) {
  if (LAYOUT == 0)
    return make_smem_desc(base + (uint32_t)(kk * 2 * rows_total * 16), (uint32_t)rows_total * 16, 128, kNoSwizzle);
  return make_smem_desc(base + (uint32_t)(kk * 32), 16, 1024, kSwizzle128B);
}
// byte distance from row 0 to row 64 of a K-major operand (8 row groups of SBO bytes)
template <int LAYOUT>
constexpr uint32_t kmajor_hi() { return LAYOUT == 0 ? 8 * 128 : 8 * 1024; }

struct ConvArgs {
  const __nv_bfloat16* src;   // gathered activation tensor (x for fwd, dy for dgrad)
  const __nv_bfloat16* wimg;  // packed weight tile images
  __nv_bfloat16* out;
  const __nv_bfloat16* addend;
  double* stats;  // [B,G,2] sum / sum of squares, accumulated in double: order-independent after rounding
  int B, SH, SW, SC;  // gathered tensor dims (H, W, C), C power of two
  int OH, OW, OC;     // output grid and channels
  int kh, kw, stride, pad;
  int M, nchunks, cshift, gn_groups;
  const float* bias;  // forward only: per-output-channel bias (SimpleCNN), or nullptr
  int relu;           // forward only: ReLU in the epilogue
  int s2_classes;  // dgrad of a stride-2 conv: rows are grouped by output-pixel parity class (4 x M/4)
  int wbn;         // N tile the weight image was packed for (>= the kernel's BN: a CTA may take a row slice of a tile)
};

// NST = depth of the cp.async ring.  3 at the learner's sizes (several CTAs per SM hide the latency); the few-CTA launches
// of the actor are one dependent memory latency per chunk and get a deeper ring instead.
template <int BN, int MODE, int NST>
__global__ void __launch_bounds__(128) conv_igemm_kernel(const ConvArgs a) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  constexpr uint32_t kABytes = kTileM * kChunkK * 2;
  constexpr uint32_t kBBytes = BN * kChunkK * 2;
  constexpr uint32_t kStageBytes = kABytes + kBBytes;
  static_assert(BN <= kMaxBN, "conv: N tile");
  static_assert(NST * kStageBytes >= kStageFloats * sizeof(float), "conv: epilogue transpose buffer");
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  // the epilogue's transpose buffer reuses the operand ring: every load and MMA of the tile has completed by then.  A
  // separate 17 KB buffer would put a CTA just over half of the SM's shared memory (one CTA per SM instead of two, and
  // no second CTA's MMAs to run under this one's epilogue).
  float* const stage_buf = reinterpret_cast<float*>(smem_raw + (smem_base - smem_u32(smem_raw)));

  const int tid = threadIdx.x, lane = tid & 31;
  const int n0 = blockIdx.y * BN;
  __shared__ short chunk_ids[kMaxChunks];
  __shared__ int n_valid_s;
  // ---- row -> output pixel.  Stride-2 dgrad: tiles are grouped by the parity class (ph, pw) of the
  // output pixel, because a class only ever touches the filter taps with r = ph+pad (mod 2),
  // s = pw+pad (mod 2): the other ~3/4 of the K chunks are skipped instead of multiplied by zeros.
  int m, ob, op, oq, ph = 0, pw = 0;
  bool row_ok;
  if (MODE == 1 && a.s2_classes) {
    const int mq = a.M >> 2;                                   // rows per class
    const int tiles_per_class = (mq + kTileM - 1) / kTileM;
    const int cls = blockIdx.x / tiles_per_class;
    const int idx = (blockIdx.x - cls * tiles_per_class) * kTileM + tid;
    ph = cls >> 1; pw = cls & 1;
    row_ok = idx < mq;
    const int h2 = a.OH >> 1, w2 = a.OW >> 1;
    const int ii = row_ok ? idx : 0;
    ob = ii / (h2 * w2);
    const int rem = ii - ob * (h2 * w2);
    op = 2 * (rem / w2) + ph;
    oq = 2 * (rem % w2) + pw;
    m = (ob * a.OH + op) * a.OW + oq;
  } else {
    m = blockIdx.x * kTileM + tid;
    row_ok = m < a.M;
    const int hw = a.OH * a.OW;
    const int mm = row_ok ? m : 0;
    ob = mm / hw;
    const int rem = mm - ob * hw;
    op = rem / a.OW;
    oq = rem - op * a.OW;
  }
  // The 128-byte-swizzle layout gathers with a coalesced mapping -- 8 consecutive lanes fetch the 8 x 16 B of ONE
  // pixel's 64-channel run (one full 128-byte line) and write one swizzled smem row -- so every thread needs the
  // pixel coordinates of 8 other rows: publish them once per tile.
  __shared__ int4 row_info[kTileM];
  row_info[tid] = make_int4(ob, op, oq, row_ok ? 1 : 0);
  if (tid == 0) {
    int nv = 0;
    const int cpt = a.SC >> 6;  // 64-channel chunks per tap (>= 1 in class mode)
    for (int c = 0; c < a.nchunks && nv < kMaxChunks; ++c) {
      bool ok = true;
      if (MODE == 1 && a.s2_classes) {
        const int tap = c / cpt;
        const int r = tap / a.kw, sx = tap - r * a.kw;
        ok = tap < a.kh * a.kw && (((ph + a.pad - r) & 1) == 0) && (((pw + a.pad - sx) & 1) == 0);
      }
      if (ok) chunk_ids[nv++] = (short)c;
    }
    n_valid_s = nv;
  }

  __syncthreads();
  const int n_valid = n_valid_s;
  const int taps = a.kh * a.kw;
  // the image is [packed tile][chunk][wbn rows x 64]; in the 128B-swizzle layout a BN-row slice of a packed tile is a
  // contiguous run of whole 8-row groups, so a narrower CTA tile reads rows [n0 % wbn, +BN) of every chunk
  const int wbn = a.wbn;
  const __nv_bfloat16* wtile =
      a.wimg + (size_t)(n0 / wbn) * a.nchunks * ((size_t)wbn * kChunkK) + (size_t)(n0 % wbn) * kChunkK;

  // The 8 rows this thread gathers for (row = tid/8 + 16 i) never change -> their pixel origin lives in
  // registers (frame base, first input row / column of the window; an out-of-range row gets an origin no tap can reach).
  // Per chunk and row that leaves two adds, two unsigned range checks and the address (this loop was 440 warp
  // instructions per chunk and the whole cost of the few-CTA launches, where one warp per scheduler hides nothing).
  int rbase[8], rh[8], rw[8];
  uint32_t soff[8];
  const int jv = tid & 7;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int row = (tid >> 3) + 16 * i;
    const int4 ri = row_info[row];
    rbase[i] = ri.x * a.SH * a.SW;
    if (MODE == 0) {
      rh[i] = ri.w ? ri.y * a.stride - a.pad : -(1 << 20);
      rw[i] = ri.z * a.stride - a.pad;
    } else {
      rh[i] = ri.w ? ri.y + a.pad : -(1 << 20);
      rw[i] = ri.z + a.pad;
    }
    soff[i] = tile_off<1>(row, jv, kTileM);
  }
  const int inv_kw = 65536 / a.kw + 1;   // tap / kw == (tap * inv_kw) >> 16 for tap < 8192, kw <= 8

  auto load_chunk = [&](int chunk, int stage) {
    const uint32_t sa = smem_base + stage * kStageBytes;
    const uint32_t sb = sa + kABytes;
    const int k0 = (chunk * 8 + jv) << 3;
    const int tap = k0 >> a.cshift;
    const int c0 = k0 & (a.SC - 1);
    const int r = (tap * inv_kw) >> 16, s = tap - r * a.kw;
    const bool tap_ok = tap < taps;
    const __nv_bfloat16* srcc = a.src + c0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      int ih, iw;
      bool ok = tap_ok;
      if (MODE == 0) {
        ih = rh[i] + r;
        iw = rw[i] + s;
      } else {
        const int th = rh[i] - r, tw = rw[i] - s;
        if (a.stride == 1) {
          ih = th; iw = tw;
        } else if (a.stride == 2) {
          ih = th >> 1; iw = tw >> 1;
          ok = ok && (((th | tw) & 1) == 0);
        } else {
          ih = th / a.stride; iw = tw / a.stride;
          ok = ok && th >= 0 && tw >= 0 && (ih * a.stride == th) && (iw * a.stride == tw);
        }
      }
      ok = ok && (unsigned)ih < (unsigned)a.SH && (unsigned)iw < (unsigned)a.SW;
      const __nv_bfloat16* g = ok ? srcc + ((size_t)(rbase[i] + ih * a.SW + iw) << a.cshift) : a.src;
      cp_async16(sa + soff[i], g, ok);
    }
    const uint4* wsrc = reinterpret_cast<const uint4*>(wtile + (size_t)chunk * ((size_t)wbn * kChunkK));
#pragma unroll
    for (int i = 0; i < BN / 16; ++i) {
      const int v = tid + i * 128;
      cp_async16(sb + ((uint32_t)v << 4), wsrc + v, true);
    }
  };

  // forward: fp16 activations x fp16 weight image; dgrad: bf16 gradients x bf16 transposed weight image
  constexpr int kT = MODE == 0 ? kF16 : kBF16;
  float acc_t[BN];
  // ---- software pipeline: cp.async runs NST-1 chunks ahead of the tensor core ----
#pragma unroll
  for (int c = 0; c < NST - 1; ++c) {
    if (c < n_valid) load_chunk(chunk_ids[c], c);
    cp_async_commit();
  }
  for (int c = 0; c < n_valid; ++c) {
    const int stage = c % NST;
    cp_async_wait<NST - 2>();
    fence_proxy_async_smem();
    __syncthreads();
    {
      const uint32_t sa = smem_base + stage * kStageBytes;
      const uint32_t sb = sa + kABytes;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kChunkK / 16; ++kk)
        mma128<BN, kT>(acc_t, kmajor_desc<1>(sa, kk, kTileM), kmajor_hi<1>(), kmajor_desc<1>(sb, kk, BN),
                       (c > 0 || kk > 0) ? 1u : 0u);
      wgmma_commit();
    }
    const int nc = c + NST - 1;
    if (nc < n_valid) {
      wgmma_wait<1>();   // the MMAs of chunk c-1 have read stage nc % NST
      load_chunk(chunk_ids[nc], nc % NST);
    }
    cp_async_commit();
  }
  wgmma_wait<0>();   // (also: the ring is no longer read, stage_buf may overwrite it)
  acc_fence(acc_t);

  // ---- epilogue: registers -> (stats | + addend) -> fp16 / bf16 NHWC ----
  const int hw = a.OH * a.OW;
  int seg = 1;  // lanes of a warp that share a frame (power of two), else 1
  if ((hw & (hw - 1)) == 0) seg = hw < 32 ? hw : 32;
#pragma unroll
  for (int col0 = 0; col0 < BN; col0 += 32) {
    float acc[32];
    if (n_valid > 0) {
      acc_row32(acc_t, col0, stage_buf, acc);
    } else {
#pragma unroll
      for (int j = 0; j < 32; ++j) acc[j] = 0.f;
    }

    if (MODE == 0 && a.stats != nullptr) {
      const int cpg = a.OC / a.gn_groups;  // channels per group (power of two >= 2)
      float s2[16], q2[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        s2[i] = acc[2 * i] + acc[2 * i + 1];
        q2[i] = acc[2 * i] * acc[2 * i] + acc[2 * i + 1] * acc[2 * i + 1];
      }
      int lg = 0;  // log2(min(cpg,32)) - 1
      while ((2 << lg) < cpg && lg < 4) ++lg;
      // fixed inner trip count: bounded by (8 >> lvl) the loop stays rolled over dynamically indexed arrays (local memory)
#pragma unroll
      for (int lvl = 0; lvl < 4; ++lvl) {
        if (lvl < lg) {
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            if (i < (8 >> lvl)) {
              s2[i] = s2[2 * i] + s2[2 * i + 1];
              q2[i] = q2[2 * i] + q2[2 * i + 1];
            }
          }
        }
      }
      const int ng = 16 >> lg;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        if (off < seg) {
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            if (i < ng) {
              s2[i] += __shfl_xor_sync(0xffffffffu, s2[i], off);
              q2[i] += __shfl_xor_sync(0xffffffffu, q2[i], off);
            }
          }
        }
      }
      if (row_ok && (lane & (seg - 1)) == 0) {
        const int g0 = (n0 + col0) / cpg;
        double* dst = a.stats + ((size_t)ob * a.gn_groups + g0) * 2;
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          if (i < ng) {
            atomicAdd(dst + 2 * i, (double)s2[i]);
            atomicAdd(dst + 2 * i + 1, (double)q2[i]);
          }
        }
      }
    }
    if (MODE == 0 && a.bias != nullptr) {
#pragma unroll
      for (int j = 0; j < 32; ++j) acc[j] += __ldg(a.bias + n0 + col0 + j);
    }
    if (MODE == 0 && a.relu) {
#pragma unroll
      for (int j = 0; j < 32; ++j) acc[j] = fmaxf(acc[j], 0.f);
    }
    if (row_ok) {
      const size_t o = (size_t)m * a.OC + n0 + col0;
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
      uint4* dst = reinterpret_cast<uint4*>(a.out + o);
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

// ---- persistent, warp-specialised variant (learner-sized stride-1 forward and dgrad, gathered C % 64 == 0) ----------
// An overload of conv_igemm_kernel (template arguments MODE, SPLIT_N).  The gather kernel above issues its own gathers
// (address arithmetic and predicates for 8 rows per thread per chunk) between its MMAs, and its 128 x 128 tile reads
// 32 KB from L2 per 2.1 MFLOP.  Here:
//   warpgroup 0 (one thread)  producer: per K chunk (one filter tap x 64 channels) one TMA im2col box of the activation
//                             (forward) or gradient (dgrad) in the 128-byte-swizzle K-major layout (byte for byte
//                             what the gather kernel writes; padding is the TMA unit's zero fill) and one 16 KB bulk copy
//                             per 128 columns of the packed weight image, into a kWsStages-deep full / empty mbarrier ring
//   warpgroups 1, 2           consumers: both work on the same CTA tile and read the same stage, each with a 128 x 128
//                             fp32 accumulator.  SPLIT_N = false: tile 256 pixels x 128 channels, the consumers split M
//                             and share B; SPLIT_N = true (OC >= 256): 128 x 256, they split N and share A.  Either way
//                             a 48 KB stage feeds 4.2 MFLOP (85 FLOP per L2 byte, against 64 for the gather kernel)
// setmaxnreg moves registers from the producer warpgroup to the consumers.  Tiles are strided statically over a grid
// sized to the SMs.  Every output row sees the MMA sequence and operand bits of the gather kernel, and the epilogue
// below restates the gather kernel's: the results are bit-identical.  (One shared epilogue function changed the gather
// kernel's code generation and made its stride-2 parity-class dgrad 10-20 % slower, so each kernel keeps its own.)
// The im2col box walks output pixels in (frame, row, column) order, the kernel's row order: the map's bounding box
// spans the window origins (lower corner = the first origin, element strides = the conv stride), the instruction gives
// the first row's origin and the tap as the im2col offsets.  Stride-1 dgrad is a forward conv over dy with the flipped
// filter: origin lower corner -(k-1-pad), tap offsets (k-1-s, k-1-r), i.e. ih = oh + pad - r as in the gather.
constexpr int kWsThreads = 384;
constexpr int kWsStages = 4;          // 4 x 48 KB ring + 2 x 17 KB transpose buffers: 226 KB of the SM's 227
constexpr int kWsProducerRegs = 40;   // 128 x 40 + 256 x 232 = 64512 of the SM's 65536 registers
constexpr int kWsConsumerRegs = 232;

template <int MODE, bool SPLIT_N>
__global__ void __launch_bounds__(kWsThreads, 1)
conv_igemm_kernel(const ConvArgs a, const __grid_constant__ CUtensorMap tmap, int lo_w, int lo_h) {
  constexpr int BN = kMaxBN;
  extern __shared__ __align__(16) uint8_t smem_raw[];
  // epilogue: registers -> (stats | + addend) -> fp16 / bf16 NHWC, as in the gather kernel.  Thread t of the calling
  // warpgroup owns accumulator row t: output row `m` (pixel of frame `ob`, stored only if `row_ok`), columns
  // [n0, n0 + BN).  `stage_buf` / `bar`: the warpgroup's transpose buffer and named barrier.  (No bias / ReLU: those
  // launches stay on the gather kernel.)
  auto epilogue = [&](const float (&acc_t)[BN], int m, int ob, bool row_ok, int n0, float* stage_buf, int bar) {
    const int lane = threadIdx.x & 31;
    const int hw = a.OH * a.OW;
    int seg = 1;  // lanes of a warp that share a frame (power of two), else 1
    if ((hw & (hw - 1)) == 0) seg = hw < 32 ? hw : 32;
#pragma unroll
    for (int col0 = 0; col0 < BN; col0 += 32) {
      float acc[32];
      acc_row32(acc_t, col0, stage_buf, acc, bar);

      if (MODE == 0 && a.stats != nullptr) {
        const int cpg = a.OC / a.gn_groups;  // channels per group (power of two >= 2)
        float s2[16], q2[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          s2[i] = acc[2 * i] + acc[2 * i + 1];
          q2[i] = acc[2 * i] * acc[2 * i] + acc[2 * i + 1] * acc[2 * i + 1];
        }
        int lg = 0;  // log2(min(cpg,32)) - 1
        while ((2 << lg) < cpg && lg < 4) ++lg;
        // the gather kernel's pairwise tree, same additions in the same order.  The inner loop has a fixed trip count:
        // bounded by (8 >> lvl) it stays a rolled loop over dynamically indexed arrays, i.e. local memory, which at 226
        // KB of shared memory per SM has almost no L1 behind it
#pragma unroll
        for (int lvl = 0; lvl < 4; ++lvl) {
          if (lvl < lg) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              if (i < (8 >> lvl)) {
                s2[i] = s2[2 * i] + s2[2 * i + 1];
                q2[i] = q2[2 * i] + q2[2 * i + 1];
              }
            }
          }
        }
        const int ng = 16 >> lg;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
          if (off < seg) {
#pragma unroll
            for (int i = 0; i < 16; ++i) {
              if (i < ng) {
                s2[i] += __shfl_xor_sync(0xffffffffu, s2[i], off);
                q2[i] += __shfl_xor_sync(0xffffffffu, q2[i], off);
              }
            }
          }
        }
        if (row_ok && (lane & (seg - 1)) == 0) {
          const int g0 = (n0 + col0) / cpg;
          double* dst = a.stats + ((size_t)ob * a.gn_groups + g0) * 2;
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            if (i < ng) {
              atomicAdd(dst + 2 * i, (double)s2[i]);
              atomicAdd(dst + 2 * i + 1, (double)q2[i]);
            }
          }
        }
      }
      if (row_ok) {
        const size_t o = (size_t)m * a.OC + n0 + col0;
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
        uint4* dst = reinterpret_cast<uint4*>(a.out + o);
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
  };
  constexpr int MT = SPLIT_N ? 1 : 2, NT = SPLIT_N ? 2 : 1;   // 128-row / 128-column sub-tiles of a CTA tile
  constexpr uint32_t kSub = kTileM * kChunkK * 2;              // one 128-row K-major chunk: 16 KB
  constexpr uint32_t kABytes = MT * kSub, kStageBytes = (MT + NT) * kSub;
  __shared__ __align__(8) uint64_t full_bar[kWsStages], empty_bar[kWsStages];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;   // swizzle atoms are 1024-byte aligned
  float* const stage_bufs =
      reinterpret_cast<float*>(smem_raw + (sbase + kWsStages * kStageBytes - smem_u32(smem_raw)));
  const int tid = threadIdx.x, wg_id = tid >> 7;
  if (tid == 0) {
#pragma unroll
    for (int i = 0; i < kWsStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);   // one arrival per consumer warpgroup
    }
    mbar_fence_init();
  }
  __syncthreads();
  const int mtiles = (a.M + MT * kTileM - 1) / (MT * kTileM), ntiles = a.OC / (NT * kTileM);
  const int total = mtiles * ntiles;
  const int first = blockIdx.x, stride = gridDim.x;
  const int my_n = first < total ? (total - first + stride - 1) / stride : 0;
  const int hw = a.OH * a.OW;

  if (wg_id == 0) {
    setmaxnreg_dec<kWsProducerRegs>();
    if (tid == 0) {
      const CUtensorMap* const tmap_p = &tmap;   // param-space address, taken in the kernel body
      int it = 0;
      for (int i = 0; i < my_n; ++i) {
        const int tile = first + i * stride;
        const int mt = tile / ntiles, nt = tile - mt * ntiles;
        const int m0 = mt * MT * kTileM;
        const int ob = m0 / hw, rem = m0 - ob * hw;
        const int oh = rem / a.OW, ow = rem - oh * a.OW;
        const int w0 = ow * a.stride + lo_w, h0 = oh * a.stride + lo_h;   // the first row's window origin
        const __nv_bfloat16* wsrc = a.wimg + (size_t)nt * NT * a.nchunks * (kTileM * kChunkK);
        for (int c = 0; c < a.nchunks; ++c, ++it) {
          const int st = it % kWsStages;
          if (it >= kWsStages) mbar_wait(&empty_bar[st], ((it / kWsStages) - 1) & 1);
          const int k0 = c * kChunkK;
          const int tap = k0 >> a.cshift, c0 = k0 & (a.SC - 1);
          const int r = tap / a.kw, s = tap - r * a.kw;
          const int offw = MODE == 0 ? s : a.kw - 1 - s, offh = MODE == 0 ? r : a.kh - 1 - r;
          const uint32_t sa = sbase + (uint32_t)st * kStageBytes;
          mbar_expect_tx(&full_bar[st], kStageBytes);
          tma_load_im2col_4d(sa, tmap_p, &full_bar[st], c0, w0, h0, ob, (uint16_t)offw, (uint16_t)offh);
#pragma unroll
          for (int j = 0; j < NT; ++j)
            bulk_load_1d(sa + kABytes + j * kSub, wsrc + ((size_t)j * a.nchunks + c) * (kTileM * kChunkK), kSub,
                         &full_bar[st]);
        }
      }
    }
  } else {
    setmaxnreg_inc<kWsConsumerRegs>();
    // forward: fp16 activations x fp16 weight image; dgrad: bf16 gradients x bf16 transposed weight image
    constexpr int kT = MODE == 0 ? kF16 : kBF16;
    const int wgi = wg_id - 1, t = tid & 127;
    const uint32_t a_off = SPLIT_N ? 0u : (uint32_t)wgi * kSub;
    const uint32_t b_off = kABytes + (SPLIT_N ? (uint32_t)wgi * kSub : 0u);
    float* const stage_buf = stage_bufs + wgi * kStageFloats;
    float acc_t[kMaxBN];
    int it = 0;
    for (int i = 0; i < my_n; ++i) {
      const int tile = first + i * stride;
      const int mt = tile / ntiles, nt = tile - mt * ntiles;
      for (int c = 0; c < a.nchunks; ++c, ++it) {
        const int st = it % kWsStages;
        mbar_wait(&full_bar[st], (it / kWsStages) & 1);
        const uint32_t sa = sbase + (uint32_t)st * kStageBytes;
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < kChunkK / 16; ++kk)
          mma128<kMaxBN, kT>(acc_t, kmajor_desc<1>(sa + a_off, kk, kTileM), kmajor_hi<1>(),
                             kmajor_desc<1>(sa + b_off, kk, kMaxBN), (c > 0 || kk > 0) ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();   // the MMAs of chunk c-1 have read their stage: release it to the producer
        if (c > 0 && t == 0) mbar_arrive(&empty_bar[(it - 1) % kWsStages]);
      }
      wgmma_wait<0>();
      acc_fence(acc_t);
      if (t == 0) mbar_arrive(&empty_bar[(it - 1) % kWsStages]);
      const int m = mt * MT * kTileM + (SPLIT_N ? 0 : wgi * kTileM) + t;
      const bool row_ok = m < a.M;
      const int n0 = (nt * NT + (SPLIT_N ? wgi : 0)) * kTileM;
      epilogue(acc_t, m, (row_ok ? m : 0) / hw, row_ok, n0, stage_buf, 1 + wgi);
    }
  }
}

// ------------------------------------------------------------------------------------------
// weight gradient: rows = (tap, ci) (128 per CTA), cols = co, reduction over output pixels
// ------------------------------------------------------------------------------------------
struct WgradArgs {
  const __nv_bfloat16* x;
  const __nv_bfloat16* dy;
  float* dw;  // partials [split = blockIdx.z][(tap, ci)][Co], summed in split order by reduce_partials
  int B, Hi, Wi, Ci, Ho, Wo, Co, kh, kw, stride, pad;
  int P;       // output pixels B*Ho*Wo
  int KW;      // taps * Ci (valid rows)
  int chunks_per_split;
  int cshift;
};

template <int BN>
__global__ void __launch_bounds__(128) conv_wgrad_kernel(const WgradArgs a) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __shared__ float stage_buf[kStageFloats];
  constexpr uint32_t kABytes = kTileM * kChunkK * 2;
  constexpr uint32_t kBBytes = BN * kChunkK * 2;
  constexpr uint32_t kStageBytes = kABytes + kBBytes;
  constexpr uint32_t kLboA = (kTileM / 8) * 128, kLboB = (BN / 8) * 128;
  static_assert(BN <= kMaxBN, "conv_wgrad: N tile");
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;

  const int tid = threadIdx.x;
  const int row_base = blockIdx.x * kTileM;
  const int n0 = blockIdx.y * BN;
  const long long total_chunks = ((long long)a.P + kChunkK - 1) / kChunkK;
  const long long c_begin = (long long)blockIdx.z * a.chunks_per_split;
  long long c_end = c_begin + a.chunks_per_split;
  if (c_end > total_chunks) c_end = total_chunks;
  const int nchunks = (int)(c_end - c_begin);
  if (nchunks <= 0) return;

  const int kpix = tid & 63;    // pixel within the chunk handled by this thread
  const int half = tid >> 6;    // 0/1
  const int taps = a.kh * a.kw;
  const int hw = a.Ho * a.Wo;

  auto load_chunk = [&](int chunk, int stage) {
    const uint32_t sa = smem_base + stage * kStageBytes;
    const uint32_t sb = sa + kABytes;
    const long long pg = (c_begin + chunk) * kChunkK + kpix;
    const bool pix_ok = pg < a.P;
    int b = 0, oh = 0, ow = 0;
    if (pix_ok) {
      b = (int)(pg / hw);
      const int rem = (int)(pg - (long long)b * hw);
      oh = rem / a.Wo;
      ow = rem - oh * a.Wo;
    }
    const uint32_t koff = (uint32_t)(kpix >> 3) * 0 + (uint32_t)((kpix & 7) << 4);
    // A: rows (tap, ci) gathered from x
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int mb = half * 8 + i;
      const int row0 = row_base + mb * 8;
      const int tap = row0 >> a.cshift;
      const int c0 = row0 & (a.Ci - 1);
      const int r = tap / a.kw, s = tap - r * a.kw;
      const int ih = oh * a.stride - a.pad + r, iw = ow * a.stride - a.pad + s;
      const bool ok = pix_ok && tap < taps && ih >= 0 && ih < a.Hi && iw >= 0 && iw < a.Wi;
      const __nv_bfloat16* g = ok ? a.x + ((((size_t)b * a.Hi + ih) * a.Wi + iw) << a.cshift) + c0 : a.x;
      cp_async16(sa + (uint32_t)(kpix >> 3) * kLboA + (uint32_t)mb * 128 + koff, g, ok);
    }
    // B: cols co from dy
#pragma unroll
    for (int i = 0; i < BN / 16; ++i) {
      const int nb = half + 2 * i;
      const __nv_bfloat16* g = pix_ok ? a.dy + (size_t)pg * a.Co + n0 + nb * 8 : a.dy;
      cp_async16(sb + (uint32_t)(kpix >> 3) * kLboB + (uint32_t)nb * 128 + koff, g, pix_ok);
    }
  };

  // A = the bf16 twin of the forward activations, B = output gradients dy (bf16).  The tensor core has no mixed
  // fp16 x bf16 form, so the forward kernels write a bf16-rounded copy of x
  float acc_t[BN];
#pragma unroll
  for (int c = 0; c < kStages - 1; ++c) {
    if (c < nchunks) load_chunk(c, c);
    cp_async_commit();
  }
  for (int c = 0; c < nchunks; ++c) {
    const int stage = c % kStages;
    cp_async_wait<kStages - 2>();
    fence_proxy_async_smem();
    __syncthreads();
    {
      const uint32_t sa = smem_base + stage * kStageBytes;
      const uint32_t sb = sa + kABytes;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < kChunkK / 16; ++kk) {
        // MN-major, no swizzle: SBO = stride between 8-element MN blocks, LBO = between 8-k blocks
        const uint64_t da = make_smem_desc(sa + kk * 2 * kLboA, kLboA, 128, kNoSwizzle);
        const uint64_t db = make_smem_desc(sb + kk * 2 * kLboB, kLboB, 128, kNoSwizzle);
        mma128<BN, kBF16, 1, 1>(acc_t, da, 8 * 128, db, (c > 0 || kk > 0) ? 1u : 0u);
      }
      wgmma_commit();
    }
    const int nc = c + kStages - 1;
    if (nc < nchunks) {
      wgmma_wait<1>();   // the MMAs of chunk c-1 have read stage nc % kStages
      load_chunk(nc, nc % kStages);
    }
    cp_async_commit();
  }
  wgmma_wait<0>();
  acc_fence(acc_t);

  const int row = row_base + tid;
#pragma unroll
  for (int col0 = 0; col0 < BN; col0 += 32) {
    float r[32];
    acc_row32(acc_t, col0, stage_buf, r);
    if (row < a.KW) {
      float* dst = a.dw + ((size_t)blockIdx.z * a.KW + row) * a.Co + n0 + col0;
#pragma unroll
      for (int j = 0; j < 32; j += 4) *reinterpret_cast<float4*>(dst + j) = make_float4(r[j], r[j + 1], r[j + 2], r[j + 3]);
    }
  }
}

// ------------------------------------------------------------------------------------------
// minimal synchronous GEMM used to pin the descriptor encodings on hardware
// ------------------------------------------------------------------------------------------
template <int LAYOUT, int MNMAJOR, int N, int T>
__global__ void __launch_bounds__(128)
umma_probe_kernel(const __nv_bfloat16* __restrict__ A, const __nv_bfloat16* __restrict__ Bm,
                  float* __restrict__ D, int M, int K) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __shared__ float stage_buf[kStageFloats];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sa = smem_base, sb = smem_base + kTileM * kChunkK * 2;
  const int tid = threadIdx.x;
  const int m0 = blockIdx.x * kTileM;
  float acc_t[N];
  const int nchunks = K / kChunkK;
  for (int c = 0; c < nchunks; ++c) {
    if (!MNMAJOR) {
      // A [M,K] row-major, B [N,K] row-major
      for (int v = tid; v < kTileM * 8; v += 128) {
        const int row = v >> 3, j = v & 7;
        const uint4 val = *reinterpret_cast<const uint4*>(A + (size_t)(m0 + row) * K + c * kChunkK + j * 8);
        asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(sa + tile_off<LAYOUT>(row, j, kTileM)),
                     "r"(val.x), "r"(val.y), "r"(val.z), "r"(val.w) : "memory");
      }
      for (int v = tid; v < N * 8; v += 128) {
        const int row = v >> 3, j = v & 7;
        const uint4 val = *reinterpret_cast<const uint4*>(Bm + (size_t)row * K + c * kChunkK + j * 8);
        asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(sb + tile_off<LAYOUT>(row, j, N)),
                     "r"(val.x), "r"(val.y), "r"(val.z), "r"(val.w) : "memory");
      }
    } else {
      // A given as [K,M] (M contiguous), B as [K,N]
      const uint32_t lboA = (kTileM / 8) * 128, lboB = (uint32_t)(N / 8) * 128;
      for (int v = tid; v < kChunkK * (kTileM / 8); v += 128) {
        const int k = v / (kTileM / 8), mb = v % (kTileM / 8);
        const uint4 val = *reinterpret_cast<const uint4*>(A + (size_t)(c * kChunkK + k) * M + m0 + mb * 8);
        asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(sa + (k >> 3) * lboA + mb * 128 + ((k & 7) << 4)),
                     "r"(val.x), "r"(val.y), "r"(val.z), "r"(val.w) : "memory");
      }
      for (int v = tid; v < kChunkK * (N / 8); v += 128) {
        const int k = v / (N / 8), nb = v % (N / 8);
        const uint4 val = *reinterpret_cast<const uint4*>(Bm + (size_t)(c * kChunkK + k) * N + nb * 8);
        asm volatile("st.shared.v4.b32 [%0], {%1,%2,%3,%4};" ::"r"(sb + (k >> 3) * lboB + nb * 128 + ((k & 7) << 4)),
                     "r"(val.x), "r"(val.y), "r"(val.z), "r"(val.w) : "memory");
      }
    }
    fence_proxy_async_smem();
    __syncthreads();
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kChunkK / 16; ++kk) {
      uint64_t da, db;
      uint32_t a_hi;
      if (!MNMAJOR) {
        da = kmajor_desc<LAYOUT>(sa, kk, kTileM);
        db = kmajor_desc<LAYOUT>(sb, kk, N);
        a_hi = kmajor_hi<LAYOUT>();
      } else {
        const uint32_t lboA = (kTileM / 8) * 128, lboB = (uint32_t)(N / 8) * 128;
        da = make_smem_desc(sa + kk * 2 * lboA, lboA, 128, kNoSwizzle);
        db = make_smem_desc(sb + kk * 2 * lboB, lboB, 128, kNoSwizzle);
        a_hi = 8 * 128;
      }
      mma128<N, T, MNMAJOR, MNMAJOR>(acc_t, da, a_hi, db, (c > 0 || kk > 0) ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();  // fully synchronous: smem is reused next iteration
    __syncthreads();
  }
  acc_fence(acc_t);
  if (N >= 32) {
#pragma unroll
    for (int col0 = 0; col0 < N; col0 += 32) {
      float r[32];
      acc_row32(acc_t, col0, stage_buf, r);
      for (int j = 0; j < 32; ++j) D[(size_t)(m0 + tid) * N + col0 + j] = r[j];
    }
  } else {   // N = 16: straight from the fragment
    const int w = tid >> 5, l = tid & 31;
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int i = 0; i < N / 8; ++i) {
        const int row = m0 + h * 64 + 16 * w + (l >> 2), col = 8 * i + 2 * (l & 3);
        const float* f = &acc_t[h * (N / 2) + 4 * i];
        D[(size_t)row * N + col] = f[0];
        D[(size_t)row * N + col + 1] = f[1];
        D[(size_t)(row + 8) * N + col] = f[2];
        D[(size_t)(row + 8) * N + col + 1] = f[3];
      }
  }
}

// ------------------------------------------------------------------------------------------
// weight packing
// ------------------------------------------------------------------------------------------
// tile images [ntile][chunk][BN x 64 in the smem operand layout]
__global__ void pack_weight_kernel(const float* __restrict__ w, __nv_bfloat16* __restrict__ img,
                                   int rows /*N dim*/, int BN, int kc /*channels per tap*/,
                                   int kc_real, int taps, int kw, int nchunks, int transposed,
                                   int co, int ci_real) {
  // one thread per 16-byte vector of the image
  const long long nvec = (long long)(rows / BN) * nchunks * BN * 8;
  for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x; v < nvec;
       v += (long long)gridDim.x * blockDim.x) {
    const int per_tile = BN * 8;
    const long long t = v / per_tile;
    const int within = (int)(v - t * per_tile);
    const int ntile = (int)(t / nchunks), chunk = (int)(t - (long long)ntile * nchunks);
    // invert the 128-byte swizzle: find (row, k8) stored at vector slot `within`
    const int g = within >> 6, rr = (within >> 3) & 7, pos = within & 7;
    const int row = g * 8 + rr, k8 = pos ^ rr;
    const int n = ntile * BN + row;
    float f[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int k = chunk * kChunkK + k8 * 8 + e;
      const int tap = k / kc, c = k - tap * kc;
      float val = 0.f;
      if (tap < taps && c < kc_real) {
        const int r = tap / kw, s = tap - r * kw;
        const int kh = taps / kw;
        // forward:    n = co, c = ci : W[co][ci][r][s]
        // transposed: n = ci, c = co : W[co][ci][r][s]
        const int o = transposed ? c : n, i = transposed ? n : c;
        if (o < co && i < ci_real) val = w[(((size_t)o * ci_real + i) * kh + r) * kw + s];
      }
      f[e] = val;
    }
    // forward image: fp16 (multiplied with fp16 activations); transposed (dgrad) image: bf16 (with bf16 gradients)
    reinterpret_cast<uint4*>(img)[v] = transposed ? pack8(f) : pack8a(f);
  }
}

__global__ void unpack_wgrad_kernel(const float* __restrict__ acc, float* __restrict__ dw, int co,
                                    int ci_real, int ci_pad, int kh, int kw) {
  const long long n = (long long)co * ci_real * kh * kw;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    const int s = (int)(i % kw);
    long long t = i / kw;
    const int r = (int)(t % kh);
    t /= kh;
    const int ci = (int)(t % ci_real);
    const int o = (int)(t / ci_real);
    dw[i] = acc[((size_t)(r * kw + s) * ci_pad + ci) * co + o];
  }
}

static int ilog2(int v) {
  int l = 0;
  while ((1 << l) < v) ++l;
  return l;
}
static bool is_pow2(int v) { return v > 0 && (v & (v - 1)) == 0; }
static int pick_bn(int n) { return n >= kMaxBN ? kMaxBN : n; }

typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*,
                                   CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                   CUtensorMapFloatOOBfill);
static EncodeIm2colFn im2col_encode_fn() {
  static EncodeIm2colFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &p, cudaEnableDefault, &q) != cudaSuccess ||
      q != cudaDriverEntryPointSuccess)
    return nullptr;
  fn = (EncodeIm2colFn)p;
  return fn;
}

// window origins of the im2col traversal along one spatial dim: first = lower corner, then `step` apart, `n` of them.
// Forward: origin = o * stride - pad.  Stride-1 dgrad (forward conv over dy, flipped filter): origin = o - (k - 1 - pad)
static void im2col_corners(int src_dim, int n, int step, int lo, int* lower, int* upper) {
  *lower = lo;
  *upper = lo + (n - 1) * step - (src_dim - 1);   // the last origin, relative to the tensor's last element
}

template <int MODE, bool SPLIT_N>
static int launch_igemm_ws(const ConvArgs& a, cudaStream_t st) {
  constexpr int MT = SPLIT_N ? 1 : 2;
  EncodeIm2colFn enc = im2col_encode_fn();
  if (!enc) {
    set_last_error("conv (im2col TMA): cuTensorMapEncodeIm2col is not available from this driver");
    return HB200_ERR_UNSUPPORTED;
  }
  const int step = MODE == 0 ? a.stride : 1;
  const int lo_h = MODE == 0 ? -a.pad : -(a.kh - 1 - a.pad), lo_w = MODE == 0 ? -a.pad : -(a.kw - 1 - a.pad);
  int lower[2], upper[2];   // {W, H}
  im2col_corners(a.SW, a.OW, step, lo_w, &lower[0], &upper[0]);
  im2col_corners(a.SH, a.OH, step, lo_h, &lower[1], &upper[1]);
  CUtensorMap tmap;
  const cuuint64_t dims[4] = {(cuuint64_t)a.SC, (cuuint64_t)a.SW, (cuuint64_t)a.SH, (cuuint64_t)a.B};
  const cuuint64_t strides[3] = {(cuuint64_t)a.SC * 2, (cuuint64_t)a.SW * a.SC * 2, (cuuint64_t)a.SH * a.SW * a.SC * 2};
  const cuuint32_t estr[4] = {1u, (cuuint32_t)step, (cuuint32_t)step, 1u};
  const CUresult r = enc(&tmap, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, (void*)a.src, dims, strides, lower, upper,
                         (cuuint32_t)kChunkK, (cuuint32_t)(MT * kTileM), estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("conv (im2col TMA): cuTensorMapEncodeIm2col failed (%d)", (int)r);
    return HB200_ERR_CUDA;
  }
  // operand ring | one transpose buffer per consumer warpgroup (+ 1024 for the alignment of the base)
  const size_t smem = (size_t)kWsStages * 3 * kTileM * kChunkK * 2 + 2 * kStageFloats * sizeof(float) + 1024;
  auto kern = conv_igemm_kernel<MODE, SPLIT_N>;
  static int grid_cache = 0;
  if (grid_cache == 0) {
    HB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    // resident CTAs per SM from the static limits (registers of 384 threads, shared memory)
    cudaFuncAttributes fa;
    HB_CUDA(cudaFuncGetAttributes(&fa, (const void*)kern));
    const int regs = fa.numRegs > 0 ? fa.numRegs : 168;
    int per_sm = 65536 / (((regs + 7) / 8 * 8) * kWsThreads);
    const int by_smem = (int)((227 * 1024) / (smem + fa.sharedSizeBytes));
    if (by_smem < per_sm) per_sm = by_smem;
    if (per_sm < 1) per_sm = 1;
    grid_cache = kNumSMs * per_sm;
  }
  const int tiles = cdiv(a.M, MT * kTileM) * (a.OC / ((SPLIT_N ? 2 : 1) * kTileM));
  const int grid = grid_cache < tiles ? grid_cache : tiles;
  kern<<<grid, kWsThreads, smem, st>>>(a, tmap, lo_w, lo_h);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

template <int MODE>
static int launch_igemm(ConvArgs a, int BN, cudaStream_t st) {
  a.wbn = BN;
  // learner-sized stride-1 launches whose gathered tensor comes in whole 64-channel chunks: the persistent im2col TMA
  // variant.  "Learner-sized" = enough 128 x 128 tiles that the gather kernel would run them full width at two CTAs per
  // SM.  The gather kernel keeps the actor's few-tile launches, narrow gathers and stride 2: the dgrad has its parity
  // classes, and the stride-2 forwards (layer3 / layer4 entries) measured no faster on the im2col variant (it supports
  // them: element strides = the stride)
  if (BN == kMaxBN && a.SC % kChunkK == 0 && !a.s2_classes && a.stride == 1 &&
      a.bias == nullptr && !a.relu && 2LL * cdiv(a.M, kTileM) * (a.OC / kMaxBN) > kNumSMs) {
    if (a.OC >= 2 * kMaxBN) return launch_igemm_ws<MODE, true>(a, st);
    return launch_igemm_ws<MODE, false>(a, st);
  }
  // few output rows (the actor's 64-frame batches: 8 row tiles for the 4x4 layers): a 128-wide N tile leaves 16 CTAs on
  // 132 SMs, each walking the whole K serially.  Narrower N tiles (slices of the packed tile: whole 8-row groups of the
  // 128B-swizzle layout) multiply the CTA count; the activation rows are re-gathered per slice out of L2.
  const int mt = a.s2_classes ? 4 * cdiv(a.M / 4, kTileM) : cdiv(a.M, kTileM);
  while (BN > 32 && 2LL * mt * (a.OC / BN) <= kNumSMs) BN /= 2;
  // at most one CTA per SM: nothing else hides the gather latency -> deep ring (uses the whole shared memory)
  const bool deep = (long long)mt * (a.OC / BN) <= kNumSMs && a.nchunks > kStages;
  // the kernel walks a per-CTA list of K chunks held in shared memory: a longer reduction must fail loudly, never truncate
  HB_CHECK_ARG(a.nchunks <= kMaxChunks, "conv: K = kh*kw*C = %d exceeds %d", a.nchunks * kChunkK, kMaxChunks * kChunkK);
  dim3 grid(a.s2_classes ? 4 * cdiv(a.M / 4, kTileM) : cdiv(a.M, kTileM), a.OC / BN);
#define HB_CONV_CASE(bn, nst)                                                                   \
  {                                                                                             \
    const size_t smem = (size_t)(nst) * (kTileM * kChunkK * 2 + bn * kChunkK * 2) + 1024;       \
    auto kern = conv_igemm_kernel<bn, MODE, nst>;                                               \
    HB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    kern<<<grid, 128, smem, st>>>(a);                                                           \
  }
#define HB_CONV_BN(bn, nst_deep)                                \
  if (deep) HB_CONV_CASE(bn, nst_deep)                          \
  else HB_CONV_CASE(bn, kStages)
  switch (BN) {
    case 32: HB_CONV_BN(32, 8); break;
    case 64: HB_CONV_BN(64, 8); break;
    case 128: HB_CONV_BN(128, 6); break;
    default:
      set_last_error("conv: unsupported N tile %d", BN);
      return HB200_ERR_UNSUPPORTED;
  }
#undef HB_CONV_BN
#undef HB_CONV_CASE
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

static int check_shape(const hb200_conv_shape* s) {
  HB_CHECK_ARG(s, "conv: null shape");
  HB_CHECK_ARG(s->batch > 0 && s->hi > 0 && s->wi > 0 && s->kh > 0 && s->kw > 0 && s->stride > 0,
               "conv: bad shape");
  HB_CHECK_ARG(is_pow2(s->ci) && s->ci >= 8, "conv: Ci=%d must be a power of two >= 8", s->ci);
  HB_CHECK_ARG(is_pow2(s->co) && s->co >= 32, "conv: Co=%d must be a power of two >= 32", s->co);
  HB_CHECK_ARG(s->ho == (s->hi + 2 * s->pad - s->kh) / s->stride + 1 &&
                   s->wo == (s->wi + 2 * s->pad - s->kw) / s->stride + 1,
               "conv: output dims inconsistent");
  return HB200_OK;
}

}  // namespace hb200

using namespace hb200;

extern "C" int hb200_conv_fwd(const hb200_bf16* x, const hb200_bf16* w_packed, hb200_bf16* y,
                              double* gn_stats, int gn_groups, const hb200_conv_shape* s,
                              hb200_stream_t stream) {
  int rc = check_shape(s);
  if (rc) return rc;
  HB_CHECK_ARG(x && w_packed && y, "conv_fwd: null pointer");
  if (gn_stats) {
    HB_CHECK_ARG(gn_groups > 0 && s->co % gn_groups == 0 && is_pow2(s->co / gn_groups) && s->co / gn_groups >= 2,
                 "conv_fwd: channels per GroupNorm group must be a power of two >= 2");
  }
  ConvArgs a;
  a.src = (const __nv_bfloat16*)x; a.wimg = (const __nv_bfloat16*)w_packed; a.out = (__nv_bfloat16*)y;
  a.addend = nullptr; a.stats = gn_stats;
  a.B = s->batch; a.SH = s->hi; a.SW = s->wi; a.SC = s->ci;
  a.OH = s->ho; a.OW = s->wo; a.OC = s->co;
  a.kh = s->kh; a.kw = s->kw; a.stride = s->stride; a.pad = s->pad;
  a.M = s->batch * s->ho * s->wo;
  a.nchunks = cdiv((long long)s->kh * s->kw * s->ci, kChunkK);
  a.cshift = ilog2(s->ci);
  a.gn_groups = gn_groups > 0 ? gn_groups : 1;
  a.s2_classes = 0;
  a.bias = nullptr;
  a.relu = 0;
  return launch_igemm<0>(a, pick_bn(s->co), (cudaStream_t)stream);
}

/* forward with a per-channel bias and optional ReLU fused in the epilogue (SimpleCNN,
 * habitat-baselines/habitat_baselines/rl/models/simple_cnn.py:68-93); output dims may use pad 0 */
extern "C" int hb200_conv_bias_act_fwd(const hb200_bf16* x, const hb200_bf16* w_packed, const float* bias,
                                       hb200_bf16* y, int relu, const hb200_conv_shape* s, hb200_stream_t stream) {
  int rc = check_shape(s);
  if (rc) return rc;
  HB_CHECK_ARG(x && w_packed && y, "conv_bias_act_fwd: null pointer");
  ConvArgs a;
  a.src = (const __nv_bfloat16*)x; a.wimg = (const __nv_bfloat16*)w_packed; a.out = (__nv_bfloat16*)y;
  a.addend = nullptr; a.stats = nullptr; a.bias = bias; a.relu = relu;
  a.B = s->batch; a.SH = s->hi; a.SW = s->wi; a.SC = s->ci;
  a.OH = s->ho; a.OW = s->wo; a.OC = s->co;
  a.kh = s->kh; a.kw = s->kw; a.stride = s->stride; a.pad = s->pad;
  a.M = s->batch * s->ho * s->wo;
  a.nchunks = cdiv((long long)s->kh * s->kw * s->ci, kChunkK);
  a.cshift = ilog2(s->ci);
  a.gn_groups = 1;
  a.s2_classes = 0;
  return launch_igemm<0>(a, pick_bn(s->co), (cudaStream_t)stream);
}

extern "C" int hb200_conv_dgrad(const hb200_bf16* dy, const hb200_bf16* w_packed_t,
                                const hb200_bf16* addend, hb200_bf16* dx, const hb200_conv_shape* s,
                                hb200_stream_t stream) {
  int rc = check_shape(s);
  if (rc) return rc;
  HB_CHECK_ARG(dy && w_packed_t && dx, "conv_dgrad: null pointer");
  HB_CHECK_ARG(s->ci >= 32, "conv_dgrad: Ci=%d must be >= 32", s->ci);
  ConvArgs a;
  a.src = (const __nv_bfloat16*)dy; a.wimg = (const __nv_bfloat16*)w_packed_t; a.out = (__nv_bfloat16*)dx;
  a.addend = (const __nv_bfloat16*)addend; a.stats = nullptr;
  a.B = s->batch; a.SH = s->ho; a.SW = s->wo; a.SC = s->co;
  a.OH = s->hi; a.OW = s->wi; a.OC = s->ci;
  a.kh = s->kh; a.kw = s->kw; a.stride = s->stride; a.pad = s->pad;
  a.M = s->batch * s->hi * s->wi;
  a.nchunks = cdiv((long long)s->kh * s->kw * s->co, kChunkK);
  a.cshift = ilog2(s->co);
  a.gn_groups = 1;
  a.bias = nullptr;
  a.relu = 0;
  a.s2_classes = (s->stride == 2 && s->co >= 64 && (s->hi % 2 == 0) && (s->wi % 2 == 0)) ? 1 : 0;
  return launch_igemm<1>(a, pick_bn(s->ci), (cudaStream_t)stream);
}

extern "C" int hb200_conv_wgrad(const hb200_bf16* x, const hb200_bf16* dy, float* dw_acc,
                                const hb200_conv_shape* s, hb200_stream_t stream) {
  int rc = check_shape(s);
  if (rc) return rc;
  HB_CHECK_ARG(x && dy && dw_acc, "conv_wgrad: null pointer");
  WgradArgs a;
  a.x = (const __nv_bfloat16*)x; a.dy = (const __nv_bfloat16*)dy; a.dw = dw_acc;
  a.B = s->batch; a.Hi = s->hi; a.Wi = s->wi; a.Ci = s->ci; a.Ho = s->ho; a.Wo = s->wo; a.Co = s->co;
  a.kh = s->kh; a.kw = s->kw; a.stride = s->stride; a.pad = s->pad;
  a.P = s->batch * s->ho * s->wo;
  a.KW = s->kh * s->kw * s->ci;
  a.cshift = ilog2(s->ci);
  const int BN = pick_bn(s->co);
  const int mtiles = cdiv(a.KW, kTileM), ntiles = s->co / BN;
  const long long total_chunks = cdiv(a.P, kChunkK);
  // ~1.5 waves of CTAs: every extra split costs a full 128 x N tile of fp32 reductions into L2
  int nsplit = (kNumSMs * 3 / 2) / (mtiles * ntiles);
  if (nsplit < 1) nsplit = 1;
  if (nsplit > total_chunks) nsplit = (int)total_chunks;
  a.chunks_per_split = (int)((total_chunks + nsplit - 1) / nsplit);
  nsplit = (int)((total_chunks + a.chunks_per_split - 1) / a.chunks_per_split);
  dim3 grid(mtiles, ntiles, nsplit);
  const size_t smem = (size_t)kStages * (kTileM * kChunkK * 2 + BN * kChunkK * 2) + 1024;
  cudaStream_t st = (cudaStream_t)stream;
  // one partial per split, summed in split order into dw_acc (no floating-point atomics: deterministic)
  const long long count = (long long)a.KW * s->co;
  float* parts = nullptr;
  int* tickets = nullptr;
  rc = stream_workspace(st, (size_t)(nsplit + (nsplit < kReduceChunks ? nsplit : kReduceChunks)) * count, 0, &parts,
                        &tickets);
  if (rc) return rc;
  a.dw = parts;
#define HB_WG_CASE(bn)                                                                          \
  {                                                                                             \
    auto kern = conv_wgrad_kernel<bn>;                                                          \
    HB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    kern<<<grid, 128, smem, st>>>(a);                                                           \
  }
  switch (BN) {
    case 32: HB_WG_CASE(32); break;
    case 64: HB_WG_CASE(64); break;
    case 128: HB_WG_CASE(128); break;
    default:
      set_last_error("conv_wgrad: unsupported N tile %d", BN);
      return HB200_ERR_UNSUPPORTED;
  }
#undef HB_WG_CASE
  HB_LAUNCH_OK();
  count_launch(1);
  return reduce_partials(parts, nsplit, count, count, dw_acc, parts + (size_t)nsplit * count, st);
}

extern "C" int hb200_pack_conv_weight(const float* w_oihw, hb200_bf16* w_packed,
                                      hb200_bf16* w_packed_t, int co, int ci_real, int ci_pad, int kh,
                                      int kw, hb200_stream_t stream) {
  HB_CHECK_ARG(w_oihw && (w_packed || w_packed_t), "pack: null pointer");
  HB_CHECK_ARG(is_pow2(ci_pad) && ci_pad >= 8 && ci_pad >= ci_real && is_pow2(co) && co >= 32, "pack: bad dims");
  cudaStream_t st = (cudaStream_t)stream;
  const int taps = kh * kw;
  if (w_packed) {
    const int BN = pick_bn(co), nchunks = cdiv((long long)taps * ci_pad, kChunkK);
    const long long nvec = (long long)(co / BN) * nchunks * BN * 8;
    pack_weight_kernel<<<(int)min((nvec + 255) / 256, (long long)kNumSMs * 8), 256, 0, st>>>(
        w_oihw, (__nv_bfloat16*)w_packed, co, BN, ci_pad, ci_real, taps, kw, nchunks, 0, co, ci_real);
    HB_LAUNCH_OK();
    count_launch(1);
  }
  if (w_packed_t) {
    HB_CHECK_ARG(ci_pad >= 32, "pack: transposed pack needs Ci >= 32");
    const int BN = pick_bn(ci_pad), nchunks = cdiv((long long)taps * co, kChunkK);
    const long long nvec = (long long)(ci_pad / BN) * nchunks * BN * 8;
    pack_weight_kernel<<<(int)min((nvec + 255) / 256, (long long)kNumSMs * 8), 256, 0, st>>>(
        w_oihw, (__nv_bfloat16*)w_packed_t, ci_pad, BN, co, co, taps, kw, nchunks, 1, co, ci_real);
    HB_LAUNCH_OK();
    count_launch(1);
  }
  return HB200_OK;
}

extern "C" size_t hb200_packed_weight_elems(int n_rows, int k_channels, int kh, int kw) {
  const int nchunks = cdiv((long long)kh * kw * k_channels, kChunkK);
  return (size_t)n_rows * nchunks * kChunkK;
}

extern "C" int hb200_unpack_conv_wgrad(const float* dw_acc, float* dw_oihw, int co, int ci_real,
                                       int ci_pad, int kh, int kw, hb200_stream_t stream) {
  HB_CHECK_ARG(dw_acc && dw_oihw, "unpack: null pointer");
  const long long n = (long long)co * ci_real * kh * kw;
  unpack_wgrad_kernel<<<(int)min((n + 255) / 256, (long long)kNumSMs * 8), 256, 0, (cudaStream_t)stream>>>(
      dw_acc, dw_oihw, co, ci_real, ci_pad, kh, kw);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

extern "C" int hb200_umma_gemm_probe(const hb200_bf16* a, const hb200_bf16* b, float* d, int m, int n,
                                     int k, int layout, hb200_stream_t stream) {
  HB_CHECK_ARG(a && b && d, "probe: null pointer");
  HB_CHECK_ARG(m % 128 == 0 && (n == 16 || n == 32 || n == 64 || n == 128) && k % 64 == 0, "probe: bad dims");
  // bit 4 / bit 5 of `layout`: operand A / B holds IEEE fp16 instead of bf16; both operands must share one format
  const bool a_f16 = (layout & 16) != 0, b_f16 = (layout & 32) != 0;
  HB_CHECK_ARG(a_f16 == b_f16, "probe: the tensor core has no mixed fp16 x bf16 form");
  layout &= 15;
  HB_CHECK_ARG(layout >= 0 && layout <= 2, "probe: layout 0 (K-major no swizzle), 1 (K-major 128B), 2 (MN-major)");
  const size_t smem = (size_t)(kTileM + n) * kChunkK * 2 + 1024;
  cudaStream_t st = (cudaStream_t)stream;
  const __nv_bfloat16* A = (const __nv_bfloat16*)a;
  const __nv_bfloat16* B = (const __nv_bfloat16*)b;
#define HB_PROBE(L, MN, NN, T)                                                                  \
  {                                                                                             \
    auto kern = umma_probe_kernel<L, MN, NN, T>;                                                \
    HB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    kern<<<m / 128, 128, smem, st>>>(A, B, d, m, k);                                            \
  }
#define HB_PROBE_N(L, MN, T)                    \
  switch (n) {                                  \
    case 16: HB_PROBE(L, MN, 16, T); break;     \
    case 32: HB_PROBE(L, MN, 32, T); break;     \
    case 64: HB_PROBE(L, MN, 64, T); break;     \
    default: HB_PROBE(L, MN, 128, T); break;    \
  }
  if (layout == 0) {
    if (a_f16) HB_PROBE_N(0, 0, kF16) else HB_PROBE_N(0, 0, kBF16)
  } else if (layout == 1) {
    if (a_f16) HB_PROBE_N(1, 0, kF16) else HB_PROBE_N(1, 0, kBF16)
  } else {
    if (a_f16) HB_PROBE_N(0, 1, kF16) else HB_PROBE_N(0, 1, kBF16)
  }
#undef HB_PROBE_N
#undef HB_PROBE
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}
