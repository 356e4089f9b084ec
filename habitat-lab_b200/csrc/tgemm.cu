// hb200 -- TF32 tensor-core GEMM (wgmma .tf32) on fp32 operands for the dense layers:
// visual_fc, the LSTM input projections and their data / weight gradients.
//
//   C[M,N] (f32) (+)= A[M,K] * B[K,N] (+ bias[N]) (ReLU)
//   A(m,k) = a[m*a_ms + k*a_ks],  B(k,n) = b[k*b_ks + n*b_ns]   (one of the two strides of each == 1)
//
// Precision: operands are fp32 in memory; the tensor core reads them as TF32 (10-bit mantissa,
// the reference's own cuDNN-RNN precision on CUDA), accumulation is fp32 in the warpgroup's registers.
//
// wgmma reads tf32 operands K-major only: both operands are [rows][k] tiles in the 128-byte-swizzle layout, copied with
// 16-byte cp.async (4 floats) or one TMA box per operand and chunk.
// One MMA covers K = 8 (32 bytes); a chunk is K = 32 (4 MMAs); 3-stage cp.async ring as in conv.cu.
// Weight gradients (K = frames, tiny M x N tile grid) are split over K; the splits are summed in order (deterministic).
#include <cuda.h>
#include "common.cuh"
#include <stdlib.h>
#include <map>
#include <mutex>
#include "wgmma.cuh"

namespace hb200 {
void count_launch(int n);
using namespace wg;

constexpr int GT_M = 128, GT_K = 32, GT_STAGES = 3;

constexpr uint32_t GT_A_HI = 8 * 1024;   // rows 0 -> 64 of a swizzled K-major tile

struct TgemmArgs {
  const float* a; long long a_ms, a_ks;
  const float* b; long long b_ks, b_ns;
  float* c; long long ldc;
  const float* bias;
  int M, N, K, k_per_split, accumulate, relu;
  // deterministic split-K for skinny problems (the actor's 64-row batches): every split stores its partial tile to
  // ws[split][M][N]; the last CTA of a tile to arrive (ticket counter) sums the splits in order and runs the epilogue
  float* ws;
  int* tickets;
  int vec4;   // c, ldc (and bias) allow 16-byte accesses
};

// load one K-major [ROWS x 32] operand tile (rows = m or n, zero-filled out of range)
// vector = 4 consecutive k of one row; 8 vectors per row per chunk.  128-byte swizzle: 8 consecutive threads fetch the
// 8 x 16 B of one row (a full 128-byte line) and write one swizzled shared-memory row (conflict free).
__device__ __forceinline__ void tg_load(const float* __restrict__ p, long long s_mn, int mn0, int MN, int k0, int k_end,
                                        uint32_t sdst, int rows) {
  for (int v = threadIdx.x; v < rows * 8; v += 128) {
    const int row = v >> 3, k4 = v & 7;
    const int gm = mn0 + row, gk = k0 + k4 * 4;
    const bool ok = gm < MN && gk + 3 < k_end;
    const float* g = ok ? p + (long long)gm * s_mn + gk : p;
    cp_async16(sdst + (uint32_t)((row >> 3) << 10) + (uint32_t)((row & 7) << 7) + (uint32_t)((k4 ^ (row & 7)) << 4),
               g, ok);
  }
}

// accumulator tile -> C: shared by the cp.async and the TMA kernels.  Plain launches add bias / accumulate / ReLU
// here; split-K launches park their partial in the workspace for the ticketed reduction in split order (the same
// sum every run).
template <int BN>
__device__ __forceinline__ void tg_epilogue(const TgemmArgs& a, float (&acc_t)[BN], float* stage_buf, int m0, int n0) {
  const int tid = threadIdx.x;
  const int m = m0 + tid;
  acc_fence(acc_t);
  if (a.ws) {
    __shared__ int s_last;
    float* wrow = a.ws + ((size_t)blockIdx.z * a.M + m) * a.N + n0;
#pragma unroll
    for (int col0 = 0; col0 < BN; col0 += 32) {
      float r[32];
      acc_row32(acc_t, col0, stage_buf, r);
      if (m < a.M) {
#pragma unroll
        for (int j = 0; j < 32; j += 4) {
          if (n0 + col0 + j < a.N)   // N % 4 == 0
            __stcg(reinterpret_cast<float4*>(wrow + col0 + j), make_float4(r[j], r[j + 1], r[j + 2], r[j + 3]));
        }
      }
    }
    __threadfence();
    __syncthreads();
    const int tile = blockIdx.y * gridDim.x + blockIdx.x;
    if (tid == 0) s_last = (atomicAdd(&a.tickets[tile], 1) == (int)gridDim.z - 1);
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    const int rows = min(GT_M, a.M - m0), cols4 = min(BN, a.N - n0) >> 2;
    for (int i = tid; i < rows * cols4; i += 128) {
      const int r = i / cols4, c = (i - r * cols4) << 2;
      const size_t off = (size_t)(m0 + r) * a.N + n0 + c;
      float4 acc = __ldcg(reinterpret_cast<const float4*>(a.ws + off));
#pragma unroll 8
      for (int z = 1; z < (int)gridDim.z; ++z) {
        const float4 p = __ldcg(reinterpret_cast<const float4*>(a.ws + (size_t)z * a.M * a.N + off));
        acc.x += p.x; acc.y += p.y; acc.z += p.z; acc.w += p.w;
      }
      float v[4] = {acc.x, acc.y, acc.z, acc.w};
      float* dst = a.c + (long long)(m0 + r) * a.ldc + n0 + c;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (a.bias) v[j] += a.bias[n0 + c + j];
        if (a.accumulate) v[j] += dst[j];
        if (a.relu) v[j] = fmaxf(v[j], 0.f);
        dst[j] = v[j];
      }
    }
    if (tid == 0) a.tickets[tile] = 0;   // ready for the next launch on this stream
    return;
  }
#pragma unroll
  for (int col0 = 0; col0 < BN; col0 += 32) {
    float r[32];
    acc_row32(acc_t, col0, stage_buf, r);
    if (m < a.M && a.vec4) {   // (split-K launches always take the workspace path above)
      // one thread owns 128 contiguous bytes of its row: float4 stores (N % 4 == 0: a group of 4 is in or out)
      float* dst = a.c + (long long)m * a.ldc + n0 + col0;
#pragma unroll
      for (int j = 0; j < 32; j += 4) {
        const int n = n0 + col0 + j;
        if (n >= a.N) continue;
        float4 v = make_float4(r[j], r[j + 1], r[j + 2], r[j + 3]);
        if (a.bias) {
          const float4 b4 = *reinterpret_cast<const float4*>(a.bias + n);
          v.x += b4.x; v.y += b4.y; v.z += b4.z; v.w += b4.w;
        }
        if (a.accumulate) {
          const float4 o = *reinterpret_cast<const float4*>(dst + j);
          v.x += o.x; v.y += o.y; v.z += o.z; v.w += o.w;
        }
        if (a.relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
        *reinterpret_cast<float4*>(dst + j) = v;
      }
    } else if (m < a.M) {
      float* dst = a.c + (long long)m * a.ldc + n0 + col0;
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        const int n = n0 + col0 + j;
        if (n >= a.N) continue;
        float v = r[j];
        if (a.bias) v += a.bias[n];
        if (a.accumulate) v += dst[j];
        if (a.relu) v = fmaxf(v, 0.f);
        dst[j] = v;
      }
    }
  }
}

// NST = cp.async ring depth: 3 for the learner's many-CTA launches, deeper for the skinny (few CTAs, latency-bound) path
template <int BN, int NST = GT_STAGES>
__global__ void __launch_bounds__(128) tgemm_kernel(const TgemmArgs a) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __shared__ float stage_buf[kStageFloats];
  constexpr uint32_t kABytes = GT_M * GT_K * 4, kBBytes = BN * GT_K * 4, kStage = kABytes + kBBytes;
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;  // swizzle atoms are 1024-byte aligned
  const int m0 = blockIdx.y * GT_M, n0 = blockIdx.x * BN;
  const int k_begin = blockIdx.z * a.k_per_split;
  const int k_end = min(a.K, k_begin + a.k_per_split);
  const int nchunks = (k_end - k_begin + GT_K - 1) / GT_K;
  if (nchunks <= 0) return;
  float acc_t[BN];

  auto load_chunk = [&](int c, int st) {
    const uint32_t sa = sbase + st * kStage, sb = sa + kABytes;
    const int k0 = k_begin + c * GT_K;
    tg_load(a.a, a.a_ms, m0, a.M, k0, k_end, sa, GT_M);
    tg_load(a.b, a.b_ns, n0, a.N, k0, k_end, sb, BN);
  };
#pragma unroll
  for (int c = 0; c < NST - 1; ++c) {
    if (c < nchunks) load_chunk(c, c);
    cp_async_commit();
  }
  for (int c = 0; c < nchunks; ++c) {
    const int st = c % NST;
    cp_async_wait<NST - 2>();
    fence_proxy_async_smem();
    __syncthreads();
    {
      const uint32_t sa = sbase + st * kStage, sb = sa + kABytes;
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < GT_K / 8; ++kk)
        mma128<BN, kTF32>(acc_t, make_smem_desc(sa + kk * 32, 16, 1024, kSwizzle128B), GT_A_HI,
                          make_smem_desc(sb + kk * 32, 16, 1024, kSwizzle128B), (c > 0 || kk > 0) ? 1u : 0u);
      wgmma_commit();
    }
    const int nc = c + NST - 1;
    if (nc < nchunks) {
      wgmma_wait<1>();   // the MMAs of chunk c-1 have read stage nc % NST
      load_chunk(nc, nc % NST);
    }
    cp_async_commit();
  }
  wgmma_wait<0>();
  tg_epilogue<BN>(a, acc_t, stage_buf, m0, n0);
}

// ---- TMA-fed variant ---------------------------------------------------------------------------------------------------
// The cp.async kernel above spends far more issue slots per K chunk on 2048 LDGSTS + their addresses than the tensor core
// needs for the chunk: the LSU work, not the tensor core, bounds it.  Here one thread issues two TMA box loads per chunk ([32 k] x [128 | BN
// rows], SWIZZLE_128B = the K-major operand layout, out-of-range rows / k zero-filled by the TMA unit) into an NST-deep
// ring ordered by full (transaction-count) barriers; the warpgroup refills a stage once wgmma.wait_group says the
// MMAs that read it have completed.
template <int BN, int NST>
__global__ void __launch_bounds__(128) tgemm_tma_kernel(const TgemmArgs a, const __grid_constant__ CUtensorMap tmap_a,
                                                        const __grid_constant__ CUtensorMap tmap_b) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[NST];
  __shared__ float stage_buf[kStageFloats];
  constexpr uint32_t kABytes = GT_M * GT_K * 4, kBBytes = BN * GT_K * 4, kStage = kABytes + kBBytes;
  const CUtensorMap* const pa = &tmap_a;   // param-space addresses, taken in the kernel body
  const CUtensorMap* const pb = &tmap_b;
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const int tid = threadIdx.x;
  const int m0 = blockIdx.y * GT_M, n0 = blockIdx.x * BN;
  const int k_begin = blockIdx.z * a.k_per_split;
  const int k_end = min(a.K, k_begin + a.k_per_split);
  const int nchunks = (k_end - k_begin + GT_K - 1) / GT_K;
  if (nchunks <= 0) return;
  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < NST; ++s) mbar_init(&full_bar[s], 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (tid == 0) {
    for (int c = 0; c < NST && c < nchunks; ++c) {
      const uint32_t sa = sbase + c * kStage;
      mbar_expect_tx(&full_bar[c], kStage);
      tma_load_2d(sa, pa, &full_bar[c], k_begin + c * GT_K, m0);
      tma_load_2d(sa + kABytes, pb, &full_bar[c], k_begin + c * GT_K, n0);
    }
  }
  float acc_t[BN];
  for (int c = 0; c < nchunks; ++c) {
    const int st = c % NST;
    mbar_wait(&full_bar[st], (c / NST) & 1);
    const uint32_t sa = sbase + st * kStage, sb = sa + kABytes;
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < GT_K / 8; ++kk)
      mma128<BN, kTF32>(acc_t, make_smem_desc(sa + kk * 32, 16, 1024, kSwizzle128B), GT_A_HI,
                        make_smem_desc(sb + kk * 32, 16, 1024, kSwizzle128B), (c > 0 || kk > 0) ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<1>();   // the MMAs of chunk c-1 are done: refill its stage with chunk c-1+NST
    const int nc = c - 1 + NST;
    if (tid == 0 && c >= 1 && nc < nchunks) {
      const int ps = (c - 1) % NST;
      const uint32_t pa_s = sbase + ps * kStage;
      mbar_expect_tx(&full_bar[ps], kStage);
      tma_load_2d(pa_s, pa, &full_bar[ps], k_begin + nc * GT_K, m0);
      tma_load_2d(pa_s + kABytes, pb, &full_bar[ps], k_begin + nc * GT_K, n0);
    }
  }
  wgmma_wait<0>();
  tg_epilogue<BN>(a, acc_t, stage_buf, m0, n0);
}
}  // namespace hb200

using namespace hb200;

// per-stream scratch (split-K partials of the skinny path, the block partials of reduce_partials): one per stream (launches on a stream are ordered; two streams never share one),
// and one per CUDA-graph capture (keyed by the capture id: the graph keeps using its buffers after the capturing stream
// has gone back to the pool).  Under capture the allocation runs in relaxed capture mode -- cudaMalloc is not a stream
// operation -- and the ticket memset becomes the graph's first node (tickets are zero between launches anyway).
int hb200::stream_workspace(cudaStream_t st, size_t floats, int tiles, float** ws, int** tickets) {
  struct Ws { float* buf = nullptr; size_t cap = 0; int* tickets = nullptr; };
  static std::mutex mu;
  static std::map<unsigned long long, Ws> table;
  constexpr int kTickets = 1024;
  HB_CHECK_ARG(tiles <= kTickets, "tgemm: %d tiles exceed the ticket table", tiles);
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  unsigned long long cap_id = 0;
  HB_CUDA(cudaStreamGetCaptureInfo(st, &cs, &cap_id));
  const bool capturing = cs == cudaStreamCaptureStatusActive;
  const unsigned long long key = capturing ? ((1ull << 63) | cap_id) : (unsigned long long)(uintptr_t)st;
  std::lock_guard<std::mutex> lock(mu);
  Ws& w = table[key];
  cudaStreamCaptureMode mode = cudaStreamCaptureModeRelaxed;
  if (capturing) HB_CUDA(cudaThreadExchangeStreamCaptureMode(&mode));
  cudaError_t e = cudaSuccess;
  if (!w.tickets) {
    e = cudaMalloc(&w.tickets, kTickets * sizeof(int));
    if (e == cudaSuccess) e = cudaMemsetAsync(w.tickets, 0, kTickets * sizeof(int), st);
  }
  if (e == cudaSuccess && w.cap < floats) {
    if (w.buf && !capturing) {   // earlier launches of a capture keep their pointer: never freed there
      e = cudaStreamSynchronize(st);
      if (e == cudaSuccess) e = cudaFree(w.buf);
    }
    w.buf = nullptr; w.cap = 0;
    const size_t cap = floats < (size_t)(4 << 20) ? (size_t)(4 << 20) : floats;
    if (e == cudaSuccess) e = cudaMalloc(&w.buf, cap * sizeof(float));
    if (e == cudaSuccess) w.cap = cap;
  }
  if (capturing) cudaThreadExchangeStreamCaptureMode(&mode);
  HB_CUDA(e);
  *ws = w.buf; *tickets = w.tickets;
  return HB200_OK;
}

typedef CUresult (*TgEncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                               const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                               CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static TgEncodeFn tg_encode_fn() {
  static TgEncodeFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
      q != cudaDriverEntryPointSuccess)
    return nullptr;
  fn = (TgEncodeFn)p;
  return fn;
}
// row-major fp32 matrix [rows, k] with row pitch ld floats -> boxes of [box_rows] x [32 k] in the 128-byte swizzle
static int tg_tensor_map(CUtensorMap* tm, const float* p, long long rows, long long k, long long ld, int box_rows) {
  TgEncodeFn enc = tg_encode_fn();
  if (!enc) {
    set_last_error("tgemm: cuTensorMapEncodeTiled is not available from this driver");
    return HB200_ERR_UNSUPPORTED;
  }
  const cuuint64_t dims[2] = {(cuuint64_t)k, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)ld * 4};
  const cuuint32_t box[2] = {(cuuint32_t)GT_K, (cuuint32_t)box_rows};
  const cuuint32_t estr[2] = {1u, 1u};
  const CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)p, dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("tgemm: cuTensorMapEncodeTiled failed (%d)", (int)r);
    return HB200_ERR_CUDA;
  }
  return HB200_OK;
}
static int g_tgemm_tma = getenv("HB200_NO_TGEMM_TMA") ? 0 : 1;

template <int BN, int NST>
static int launch_tgemm_tma(const TgemmArgs& g, dim3 grid, cudaStream_t st) {
  CUtensorMap ta, tb;
  int rc = tg_tensor_map(&ta, g.a, g.M, g.K, g.a_ms, GT_M);
  if (rc) return rc;
  rc = tg_tensor_map(&tb, g.b, g.N, g.K, g.b_ns, BN);
  if (rc) return rc;
  const size_t smem = (size_t)NST * (GT_M * GT_K * 4 + BN * GT_K * 4) + 1024;
  auto kern = tgemm_tma_kernel<BN, NST>;
  HB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<grid, 128, smem, st>>>(g, ta, tb);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}

extern "C" int hb200_set_tgemm_tma(int on) { g_tgemm_tma = on ? 1 : 0; return HB200_OK; }
extern "C" int hb200_get_tgemm_tma(void) { return g_tgemm_tma; }

extern "C" int hb200_tgemm(const float* a, long long a_ms, long long a_ks, const float* b, long long b_ks,
                           long long b_ns, float* c, long long ldc, const float* bias, int m, int n, int k,
                           int accumulate, int relu, hb200_stream_t stream) {
  HB_CHECK_ARG(a && b && c && m > 0 && n > 0 && k > 0, "tgemm: bad args");
  // wgmma reads tf32 operands K-major only -> callers transpose
  HB_CHECK_ARG(a_ks == 1 && b_ks == 1, "tgemm: both operands must be K-major (a_ks == 1, b_ks == 1)");
  const int a_mn = (a_ks == 1) ? 0 : 1;   // k contiguous -> K-major
  const int b_mn = (b_ks == 1) ? 0 : 1;
  // 16-byte vector loads: leading dimensions / pointers must be multiples of 4 floats
  const long long lda = a_mn ? a_ks : a_ms, ldb = b_mn ? b_ks : b_ns;
  HB_CHECK_ARG(lda % 4 == 0 && ldb % 4 == 0 && ((uintptr_t)a & 15) == 0 && ((uintptr_t)b & 15) == 0,
               "tgemm: operands must be 16-byte aligned with leading dimensions that are multiples of 4");
  HB_CHECK_ARG(k % 4 == 0 && (!a_mn || m % 4 == 0) && (!b_mn || n % 4 == 0), "tgemm: k (and mn-major extents) must be multiples of 4");
  // N tile <= 128: a 128 x 128 fp32 accumulator is 128 registers per thread of the warpgroup
  int BN = n >= 128 ? 128 : (n >= 64 ? 64 : 32);
  {
    static const int forced = getenv("HB200_TGEMM_BN") ? atoi(getenv("HB200_TGEMM_BN")) : 0;
    if ((forced == 32 || forced == 64 || forced == 128) && forced <= BN) BN = forced;
  }
  HB_CHECK_ARG(n % 4 == 0, "tgemm: n must be a multiple of 4");
  TgemmArgs g;
  g.a = a; g.a_ms = a_ms; g.a_ks = a_ks; g.b = b; g.b_ks = b_ks; g.b_ns = b_ns; g.c = c; g.ldc = ldc; g.bias = bias;
  g.M = m; g.N = n; g.K = k; g.accumulate = accumulate; g.relu = relu;
  g.ws = nullptr; g.tickets = nullptr;
  g.vec4 = (ldc % 4 == 0 && ((uintptr_t)c & 15) == 0 && (!bias || ((uintptr_t)bias & 15) == 0)) ? 1 : 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (m <= GT_M && k >= 256 && cdiv(n, BN) < kNumSMs / 2 && !a_mn && !b_mn) {
    // one row tile (the actor: 64 frames): a handful of CTAs would each walk the whole K, one DRAM latency per
    // 32-wide chunk.  32-wide N tiles x K splits of >= 4 chunks put one CTA on every SM,
    // each with a deep cp.async ring; partial tiles meet in an L2-resident workspace and the last CTA of each tile
    // reduces them in split order (8 KB per split).
    BN = 32;
    constexpr int kDeep = 6;   // 6 x (16 KB + 4 KB) stages
    const int nt = cdiv(n, BN);
    int sp = kNumSMs / nt;
    if (sp > k / 128) sp = k / 128;
    if (sp > 32) sp = 32;
    if (sp < 1) sp = 1;
    const int kps = ((cdiv(k, sp) + GT_K - 1) / GT_K) * GT_K;
    sp = cdiv(k, kps);
    if (sp > 1) {
      int rc = stream_workspace(st, (size_t)sp * m * n, nt, &g.ws, &g.tickets);
      if (rc) return rc;
    }
    g.k_per_split = kps;
    dim3 grid(nt, 1, sp);
    if (g_tgemm_tma) return launch_tgemm_tma<32, kDeep>(g, grid, st);
    const size_t smem = (size_t)kDeep * (GT_M * GT_K * 4 + 32 * GT_K * 4) + 1024;
    auto kern = tgemm_kernel<32, kDeep>;
    HB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<grid, 128, smem, st>>>(g);
    HB_LAUNCH_OK();
    count_launch(1);
    return HB200_OK;
  }
  const long long tiles = (long long)cdiv(n, BN) * cdiv(m, GT_M);
  int splits = 1;
  if (accumulate && !relu && tiles < kNumSMs && k >= 1024) {
    splits = (int)((2 * kNumSMs + tiles - 1) / tiles);
    if (splits > k / 256) splits = k / 256;
    if (splits < 1) splits = 1;
  }
  g.k_per_split = ((cdiv(k, splits) + GT_K - 1) / GT_K) * GT_K;
  splits = cdiv(k, g.k_per_split);
  if (splits > 1) {   // partial tiles meet in the workspace and are summed in split order (deterministic)
    int rc = stream_workspace(st, (size_t)splits * m * n, (int)tiles, &g.ws, &g.tickets);
    if (rc) return rc;
  }
  dim3 grid(cdiv(n, BN), cdiv(m, GT_M), splits);
  if (g_tgemm_tma && !a_mn && !b_mn) {
    // ring depth: two CTAs per SM (3 x 32 KB stages) when there are enough tiles for that, else one CTA with a deep ring
    const long long ctas = (long long)grid.x * grid.y * grid.z;
    switch (BN) {
      case 32: return launch_tgemm_tma<32, 4>(g, grid, st);
      case 64: return launch_tgemm_tma<64, 4>(g, grid, st);
      default: return ctas > kNumSMs ? launch_tgemm_tma<128, 3>(g, grid, st) : launch_tgemm_tma<128, 6>(g, grid, st);
    }
  }
#define HB_TG(bn)                                                                                  \
  {                                                                                                \
    const size_t smem = (size_t)GT_STAGES * (GT_M * GT_K * 4 + bn * GT_K * 4) + 1024;              \
    auto kern = tgemm_kernel<bn>;                                                                  \
    HB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));   \
    kern<<<grid, 128, smem, st>>>(g);                                                              \
  }
  switch (BN) {
    case 32: HB_TG(32); break;
    case 64: HB_TG(64); break;
    default: HB_TG(128); break;
  }
#undef HB_TG
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}
