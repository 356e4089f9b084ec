// hb200 -- TMA halo load probe (pins the halo kernels' tensor-map encoding; not on the product path).
//
// Next step for the halo convolutions (NOTES_NEXT.md item 4): replace the per-thread zero-filling cp.async gather of the
// (TH+KH-1) x (TW+KW-1) input halo -- ~6 copies per thread, each with its own address and bounds predicate, the reason
// conv_halo_kernel<32,32> is issue-bound -- by C/8 `cp.async.bulk.tensor.4d` box copies issued by ONE thread: box =
// {8 channels, halo width, halo height, 1 frame} of the NHWC tensor, out-of-bounds rows / columns zero-filled by the TMA
// unit (that is the conv padding), completion signalled on an mbarrier.  The box lands as [hy][hx][8 ch] = one 16-byte
// vector per pixel, i.e. exactly one channel-chunk slab of the no-swizzle K-major operand layout the wgmma shared-
// memory descriptors address with LBO = slab stride (next 8 channels) and SBO = halo row pitch (next 8-pixel row group).
//
// This file only verifies the mechanism (driver entry point, tensor-map encoding, negative coordinates, expect_tx
// accounting): hb200_tma_halo_probe loads one halo tile and writes the staged slabs back to global memory.
#include <cuda.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace hb200 {
void count_launch(int n);
using namespace wg;

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_tiled_fn() {
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


// one CTA: stage the halo of one tile (C/8 slabs of hh x hwd x 16 B, each padded to a multiple of 128 B), copy it out
__global__ void __launch_bounds__(128)
tma_halo_probe_kernel(const __grid_constant__ CUtensorMap tmap, uint4* __restrict__ out, int cj, int hh, int hwd,
                      int b, int oh0, int ow0, int pad, int slab_bytes) {
  extern __shared__ __align__(128) uint8_t sm_raw[];
  __shared__ __align__(8) uint64_t bar;
  const uint32_t sbase = (smem_u32(sm_raw) + 127u) & ~127u;
  if (threadIdx.x == 0) {
    mbar_init(&bar, 1);
    mbar_fence_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_expect_tx(&bar, (uint32_t)(cj * hh * hwd * 16));
    for (int j = 0; j < cj; ++j) tma_load_4d(sbase + (uint32_t)(j * slab_bytes), &tmap, &bar, j * 8, ow0 - pad, oh0 - pad, b);
  }
  mbar_wait(&bar, 0);
  const uint8_t* base = sm_raw + (sbase - smem_u32(sm_raw));
  const int nvec = hh * hwd;
  for (int j = 0; j < cj; ++j)
    for (int v = threadIdx.x; v < nvec; v += blockDim.x)
      out[(size_t)j * nvec + v] = *reinterpret_cast<const uint4*>(base + (size_t)j * slab_bytes + (size_t)v * 16);
}
}  // namespace hb200

using namespace hb200;

extern "C" int hb200_tma_halo_probe(const hb200_bf16* x, hb200_bf16* out, int batch, int h, int w, int channels, int b,
                                    int oh0, int ow0, int halo_h, int halo_w, int pad, hb200_stream_t stream) {
  HB_CHECK_ARG(x && out && batch > 0 && h > 0 && w > 0 && channels >= 8 && channels % 8 == 0, "tma_halo_probe: bad tensor");
  HB_CHECK_ARG(halo_h >= 1 && halo_h <= 256 && halo_w >= 1 && halo_w <= 256 && b >= 0 && b < batch && pad >= 0,
               "tma_halo_probe: bad box");
  HB_CHECK_ARG(((uintptr_t)x & 15) == 0, "tma_halo_probe: tensor must be 16-byte aligned");
  EncodeTiledFn enc = encode_tiled_fn();
  if (!enc) {
    set_last_error("tma_halo_probe: cuTensorMapEncodeTiled is not available from this driver");
    return HB200_ERR_UNSUPPORTED;
  }
  CUtensorMap tmap;
  const cuuint64_t dims[4] = {(cuuint64_t)channels, (cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)batch};
  const cuuint64_t strides[3] = {(cuuint64_t)channels * 2, (cuuint64_t)w * channels * 2, (cuuint64_t)h * w * channels * 2};
  const cuuint32_t box[4] = {8u, (cuuint32_t)halo_w, (cuuint32_t)halo_h, 1u};
  const cuuint32_t estr[4] = {1u, 1u, 1u, 1u};
  const CUresult r = enc(&tmap, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, (void*)x, dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("tma_halo_probe: cuTensorMapEncodeTiled failed (%d)", (int)r);
    return HB200_ERR_CUDA;
  }
  const int cj = channels / 8;
  const int slab = (halo_h * halo_w * 16 + 127) / 128 * 128;
  const size_t smem = (size_t)cj * slab + 256;
  HB_CHECK_ARG(smem <= 200 * 1024, "tma_halo_probe: halo does not fit in shared memory");
  auto kern = tma_halo_probe_kernel;
  HB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<1, 128, smem, (cudaStream_t)stream>>>(tmap, reinterpret_cast<uint4*>(out), cj, halo_h, halo_w, b, oh0, ow0, pad, slab);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}
