// hb200 -- cube-map projection transforms (HB/common/obs_transformers.py CubeMap2Equirect, CubeMap2Fisheye,
// Equirect2CubeMap): one launch resamples every target of a batch from its input faces into its output images,
// straight into the caller's buffer (normally one time slot of the rollout storage).
//
// The host builds, once per transform, a table of one (x, y, input) float triple per output pixel: the input face
// assigned to the pixel (the first whose camera sees it, -1 for none) and the normalised align_corners sampling
// point in that face.  The reference samples all its inputs at every output pixel and sums the results; every input
// but the assigned one sits at grid value 2, which zero-padded bilinear sampling turns into an exact +0 on faces of
// 3 pixels or more, so reading the assigned face alone gives the same bits once +0.0f is added (the sum's only effect
// is -0 -> +0).
//
// Bit-exactness with the reference (torch on the CPU: grid_sample(img.float() [* in_zf], grid, align_corners=True,
// zeros) summed over inputs [* out_zf], .to(dtype)): x = (gx + 1) * ((W - 1) / 2), weights w = x - floor(x),
// e = 1 - w (likewise n, s for y), nw = s * e, ne = s * w, sw = n * e, se = n * w, and the value
// fma(v_se, se, fma(v_sw, sw, fma(v_ne, ne, v_nw * nw))), taps outside the face reading 0.  Every operation is an
// explicit round-to-nearest intrinsic, so no contraction can change the bits.  Results are converted back with
// truncation toward zero, as .to(dtype) does.
#include "common.cuh"

namespace hb200 {
void count_launch(int n);

namespace {

constexpr int kPrjMaxTargets = 8;
constexpr int kPrjMaxInputs = 6;
constexpr int kPrjMaxOutputs = 6;
constexpr int kPrjThreads = 256;
constexpr int kPrjBandRows = 2;   // output rows per CTA
enum { kDtU8 = 0, kDtF32 = 1, kDtI32 = 2 };

struct PrjTarget {
  const unsigned char* src[kPrjMaxInputs];  // [batch, Hi, Wi, C] per input face
  unsigned char* dst;                        // [batch, n_out, h, w, C]
  const float* table;                        // [n_out, h, w, 3]
  const float* in_zf;                        // [n_in, Hi, Wi] or null
  const float* out_zf;                       // [n_out, h, w] or null
  int dtype, n_in, n_out, Hi, Wi, C, h, w;
  int bands;        // ceil(h / kPrjBandRows)
  int first_block;  // first CTA of this target in the grid
};

struct PrjTable {
  PrjTarget t[kPrjMaxTargets];
  int n;
};

template <typename T> __device__ __forceinline__ float to_f(T v);
template <> __device__ __forceinline__ float to_f<unsigned char>(unsigned char v) { return (float)v; }
template <> __device__ __forceinline__ float to_f<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_f<int>(int v) { return __int2float_rn(v); }
template <typename T> __device__ __forceinline__ T from_f(float v);
template <> __device__ __forceinline__ unsigned char from_f<unsigned char>(float v) {
  return (unsigned char)__float2uint_rz(v);
}
template <> __device__ __forceinline__ float from_f<float>(float v) { return v; }
template <> __device__ __forceinline__ int from_f<int>(float v) { return __float2int_rz(v); }

template <typename T>
__device__ void run_project(const PrjTarget& k, int img, int oy0, int oy1) {
  const int b = img / k.n_out, o = img - b * k.n_out;
  const long long face_px = (long long)k.Hi * k.Wi;
  T* out = reinterpret_cast<T*>(k.dst) + (long long)img * k.h * k.w * k.C;
  const float* tab = k.table + (long long)o * k.h * k.w * 3;
  const float* ozf = k.out_zf ? k.out_zf + (long long)o * k.h * k.w : nullptr;
  const float sx = (float)(k.Wi - 1) / 2.f, sy = (float)(k.Hi - 1) / 2.f;  // exact: W - 1 < 2^24
  const float wmax = (float)k.Wi, hmax = (float)k.Hi;
  const int n = (oy1 - oy0) * k.w;
  for (int e = threadIdx.x; e < n; e += blockDim.x) {
    const long long p = (long long)oy0 * k.w + e;  // output pixel
    const float gx = __ldg(tab + 3 * p), gy = __ldg(tab + 3 * p + 1);
    const int f = (int)__ldg(tab + 3 * p + 2);
    T* dst = out + p * k.C;
    if (f < 0 || f >= k.n_in) {
      for (int c = 0; c < k.C; ++c) dst[c] = from_f<T>(0.f);
      continue;
    }
    const float x = __fmul_rn(__fadd_rn(gx, 1.f), sx), y = __fmul_rn(__fadd_rn(gy, 1.f), sy);
    const float xw = floorf(x), yn = floorf(y);
    const float w = __fsub_rn(x, xw), ea = __fsub_rn(1.f, w);
    const float nn = __fsub_rn(y, yn), s = __fsub_rn(1.f, nn);
    const float w_nw = __fmul_rn(s, ea), w_ne = __fmul_rn(s, w), w_sw = __fmul_rn(nn, ea), w_se = __fmul_rn(nn, w);
    // taps inside the face (float compares first, so no out-of-range float reaches an int conversion)
    const bool in_x0 = xw > -1.f && xw < wmax, in_x1 = xw > -2.f && xw < wmax - 1.f;
    const bool in_y0 = yn > -1.f && yn < hmax, in_y1 = yn > -2.f && yn < hmax - 1.f;
    const int ix = in_x0 || in_x1 ? (int)xw : 0, iy = in_y0 || in_y1 ? (int)yn : 0;
    const long long q_nw = (long long)iy * k.Wi + ix;
    const bool t_nw = in_y0 && in_x0, t_ne = in_y0 && in_x1, t_sw = in_y1 && in_x0, t_se = in_y1 && in_x1;
    const T* face = reinterpret_cast<const T*>(k.src[f]) + (long long)b * face_px * k.C;
    const float* izf = k.in_zf ? k.in_zf + (long long)f * face_px : nullptr;
    const float z_out = ozf ? __ldg(ozf + p) : 1.f;
    auto tap = [&](bool inside, long long q, int c) -> float {
      if (!inside) return 0.f;
      const float v = to_f<T>(__ldg(face + q * k.C + c));
      return izf ? __fmul_rn(v, __ldg(izf + q)) : v;
    };
    for (int c = 0; c < k.C; ++c) {
      const float v_nw = tap(t_nw, q_nw, c), v_ne = tap(t_ne, q_nw + 1, c);
      const float v_sw = tap(t_sw, q_nw + k.Wi, c), v_se = tap(t_se, q_nw + k.Wi + 1, c);
      float acc = __fmaf_rn(v_se, w_se, __fmaf_rn(v_sw, w_sw, __fmaf_rn(v_ne, w_ne, __fmul_rn(v_nw, w_nw))));
      acc = __fadd_rn(acc, 0.f);
      if (ozf) acc = __fmul_rn(acc, z_out);
      dst[c] = from_f<T>(acc);
    }
  }
}

// grid: for each target, batch x n_out x bands CTAs (target-major); each CTA owns kPrjBandRows rows of one image
__global__ void __launch_bounds__(kPrjThreads) obs_project_kernel(const __grid_constant__ PrjTable tt) {
  int ti = 0;
  while (ti + 1 < tt.n && (int)blockIdx.x >= tt.t[ti + 1].first_block) ++ti;
  const PrjTarget& k = tt.t[ti];
  const int local = blockIdx.x - k.first_block;
  const int img = local / k.bands, band = local - img * k.bands;
  const int oy0 = band * kPrjBandRows, oy1 = min(oy0 + kPrjBandRows, k.h);
  if (k.dtype == kDtU8) run_project<unsigned char>(k, img, oy0, oy1);
  else if (k.dtype == kDtF32) run_project<float>(k, img, oy0, oy1);
  else run_project<int>(k, img, oy0, oy1);
}

}  // namespace
}  // namespace hb200

using namespace hb200;

extern "C" int hb200_obs_project(const void* const* src, void* const* dst, const float* const* table,
                                 const float* const* in_zf, const float* const* out_zf, const int32_t* desc,
                                 int n_targets, int batch, hb200_stream_t stream) {
  HB_CHECK_ARG(src && dst && table && in_zf && out_zf && desc, "obs_project: null argument");
  HB_CHECK_ARG(n_targets >= 1 && n_targets <= kPrjMaxTargets, "obs_project: n_targets = %d (1..%d)", n_targets,
               kPrjMaxTargets);
  HB_CHECK_ARG(batch >= 1, "obs_project: batch = %d", batch);
  PrjTable tt{};
  tt.n = n_targets;
  long long blocks = 0;
  for (int i = 0; i < n_targets; ++i) {
    const int32_t* d = desc + 8 * i;
    PrjTarget& k = tt.t[i];
    k.dtype = d[0]; k.n_in = d[1]; k.n_out = d[2]; k.Hi = d[3]; k.Wi = d[4]; k.C = d[5]; k.h = d[6]; k.w = d[7];
    HB_CHECK_ARG(k.dtype >= kDtU8 && k.dtype <= kDtI32, "obs_project: target %d: dtype %d", i, k.dtype);
    HB_CHECK_ARG(k.n_in >= 1 && k.n_in <= kPrjMaxInputs && k.n_out >= 1 && k.n_out <= kPrjMaxOutputs,
                 "obs_project: target %d: %d inputs, %d outputs (1..6 each)", i, k.n_in, k.n_out);
    HB_CHECK_ARG(k.Hi >= 3 && k.Wi >= 3, "obs_project: target %d: input faces of %dx%d (at least 3x3)", i, k.Hi,
                 k.Wi);
    HB_CHECK_ARG(k.C >= 1 && k.h >= 1 && k.w >= 1, "obs_project: target %d: bad sizes", i);
    const int esize = k.dtype == kDtU8 ? 1 : 4;
    HB_CHECK_ARG((long long)k.Hi * k.Wi * k.C * batch < (1LL << 40) &&
                 (long long)k.h * k.w * k.C * k.n_out * batch < (1LL << 40) && k.Hi < (1 << 24) && k.Wi < (1 << 24),
                 "obs_project: target %d: tensor too large", i);
    for (int j = 0; j < k.n_in; ++j) {
      k.src[j] = static_cast<const unsigned char*>(src[kPrjMaxInputs * i + j]);
      HB_CHECK_ARG(k.src[j] && (uintptr_t)k.src[j] % esize == 0,
                   "obs_project: target %d: input %d null or not aligned to its element size", i, j);
    }
    k.dst = static_cast<unsigned char*>(dst[i]);
    k.table = table[i];
    k.in_zf = in_zf[i];
    k.out_zf = out_zf[i];
    HB_CHECK_ARG(k.dst && (uintptr_t)k.dst % esize == 0, "obs_project: target %d: output null or misaligned", i);
    HB_CHECK_ARG(k.table && (uintptr_t)k.table % 4 == 0, "obs_project: target %d: table null or misaligned", i);
    HB_CHECK_ARG((uintptr_t)k.in_zf % 4 == 0 && (uintptr_t)k.out_zf % 4 == 0,
                 "obs_project: target %d: z-factor plane misaligned", i);
    k.bands = (k.h + kPrjBandRows - 1) / kPrjBandRows;
    k.first_block = (int)blocks;
    blocks += (long long)batch * k.n_out * k.bands;
  }
  HB_CHECK_ARG(blocks < (1LL << 31), "obs_project: grid too large");
  obs_project_kernel<<<(unsigned)blocks, kPrjThreads, 0, (cudaStream_t)stream>>>(tt);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}
