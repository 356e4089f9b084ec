// hb200 -- observation transforms (HB/common/obs_transformers.py ResizeShortestEdge + CenterCropper,
// HB/utils/common.py image_resize_shortest_edge / center_crop): one launch resamples every image key of a batch
// and writes only the pixels of an output window, straight into the caller's buffer (normally one time slot of
// the rollout storage).  The resampled image outside the window is never formed.
//
// Bit-exactness with the reference (torch on the CPU, F.interpolate(img.float(), size, mode).to(img.dtype)):
//  - area (adaptive average pooling): bin [start, end) with start = (i*H)/Hr and end = ceil((i+1)*H/Hr) in integer
//    arithmetic; one fp32 running sum from 0, rows outer and columns inner, then (sum / kh) / kw.  Every add and
//    divide is an explicit IEEE round-to-nearest intrinsic, so no contraction or reordering can change the bits.
//  - nearest: src = min(floor(float(i) * (float(H) / Hr)), H - 1), the value taken through float and back.
//  - copy: the window's bytes, for any element size.
// Results are converted back with truncation toward zero, as the reference's .to(dtype) does.
#include <initializer_list>

#include "common.cuh"

namespace hb200 {
void count_launch(int n);

namespace {

constexpr int kObsMaxKeys = 8;
constexpr int kObsThreads = 256;
constexpr int kObsBandRows = 8;              // output rows per CTA: neighbouring rows share their boundary input row
constexpr int kObsSmemBudget = 48 * 1024;    // staged input rows per CTA; larger needs fall back to direct loads
enum { kDtU8 = 0, kDtF32 = 1, kDtI32 = 2 };
enum { kModeArea = 0, kModeNearest = 1, kModeCopy = 2 };

struct ObsKey {
  const unsigned char* src;
  unsigned char* dst;
  int dtype, mode, H, W, C, Hr, Wr, y0, x0, h, w;
  int esize;           // bytes per element
  int bands;           // ceil(h / kObsBandRows)
  int first_block;     // first CTA of this key in the grid
  int vec;             // load width in bytes (16, 4 or 1): divides the base address, the row pitch and (copy) offsets
  int slots;           // area: staged input rows (>= the largest bin height); 0 = read global memory directly
  int seg_off;         // area staged: byte offset in an input row of the first staged byte (multiple of vec)
  int seg_bytes;       // area staged: bytes staged per row (multiple of vec), slot pitch rounded up to 16
  int slot_pitch;
  float nearest_scale; // float(H) / Hr, as torch computes it
};

struct ObsTable {
  ObsKey k[kObsMaxKeys];
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

// copy unit u (vec bytes) of g to s; both vec-aligned
__device__ __forceinline__ void copy_unit(unsigned char* s, const unsigned char* g, int u, int vec) {
  if (vec == 16) reinterpret_cast<uint4*>(s)[u] = __ldg(reinterpret_cast<const uint4*>(g) + u);
  else if (vec == 4) reinterpret_cast<uint32_t*>(s)[u] = __ldg(reinterpret_cast<const uint32_t*>(g) + u);
  else s[u] = __ldg(g + u);
}

// One output row of an area key.  Row r of the input is at row(r); element (iw, c) at row(r)[iw * C + c].
template <typename T, typename RowFn>
__device__ __forceinline__ void area_row(const ObsKey& k, int i, T* out, RowFn row) {
  const int rs = i * k.H / k.Hr;
  const int re = ((i + 1) * k.H + k.Hr - 1) / k.Hr;
  const float kh = (float)(re - rs);
  const int n = k.w * k.C;
  for (int e = threadIdx.x; e < n; e += blockDim.x) {
    const int ox = e / k.C, c = e - ox * k.C;
    const int j = k.x0 + ox;
    const int cs = j * k.W / k.Wr;
    const int ce = ((j + 1) * k.W + k.Wr - 1) / k.Wr;
    float s = 0.f;
    for (int r = rs; r < re; ++r) {
      const T* p = row(r) + (long long)cs * k.C + c;
      for (int iw = cs; iw < ce; ++iw, p += k.C) s = __fadd_rn(s, to_f<T>(*p));
    }
    out[e] = from_f<T>(__fdiv_rn(__fdiv_rn(s, kh), (float)(ce - cs)));
  }
}

template <typename T>
__device__ void run_area(const ObsKey& k, int b, int oy0, int oy1, unsigned char* smem) {
  const T* img = reinterpret_cast<const T*>(k.src) + (long long)b * k.H * k.W * k.C;
  T* out = reinterpret_cast<T*>(k.dst) + (long long)b * k.h * k.w * k.C;
  const long long pitch = (long long)k.W * k.C;
  if (k.slots == 0) {
    for (int oy = oy0; oy < oy1; ++oy)
      area_row<T>(k, k.y0 + oy, out + (long long)oy * k.w * k.C, [=](int r) { return img + r * pitch; });
    return;
  }
  // staged: input rows live in a ring of `slots` smem rows (slot r % slots), each loaded once per CTA
  const unsigned char* gimg = reinterpret_cast<const unsigned char*>(img);
  const long long pitch_b = pitch * k.esize;
  const int units = k.seg_bytes / k.vec;
  int loaded = (k.y0 + oy0) * k.H / k.Hr;  // next input row to stage
  for (int oy = oy0; oy < oy1; ++oy) {
    const int i = k.y0 + oy;
    const int re = ((i + 1) * k.H + k.Hr - 1) / k.Hr;
    __syncthreads();  // the previous row's reads are done before its slots are overwritten
    const int nr = re - loaded;
    for (int q = threadIdx.x; q < nr * units; q += blockDim.x) {
      const int rr = q / units, u = q - rr * units;
      const int r = loaded + rr;
      copy_unit(smem + (r % k.slots) * k.slot_pitch, gimg + r * pitch_b + k.seg_off, u, k.vec);
    }
    if (nr > 0) loaded = re;
    __syncthreads();
    // element (iw, c) of row r is at byte (iw * C + c) * esize - seg_off of its slot
    area_row<T>(k, i, out + (long long)oy * k.w * k.C, [=](int r) {
      return reinterpret_cast<const T*>(smem + (r % k.slots) * k.slot_pitch - k.seg_off);
    });
  }
}

template <typename T>
__device__ void run_nearest(const ObsKey& k, int b, int oy0, int oy1) {
  const T* img = reinterpret_cast<const T*>(k.src) + (long long)b * k.H * k.W * k.C;
  T* out = reinterpret_cast<T*>(k.dst) + (long long)b * k.h * k.w * k.C;
  const float sw = __fdiv_rn((float)k.W, (float)k.Wr);
  const int n = k.w * k.C;
  for (int oy = oy0; oy < oy1; ++oy) {
    const int sy = min((int)floorf(__fmul_rn((float)(k.y0 + oy), k.nearest_scale)), k.H - 1);
    const T* src = img + (long long)sy * k.W * k.C;
    T* dst = out + (long long)oy * n;
    for (int e = threadIdx.x; e < n; e += blockDim.x) {
      const int ox = e / k.C, c = e - ox * k.C;
      const int sx = min((int)floorf(__fmul_rn((float)(k.x0 + ox), sw)), k.W - 1);
      dst[e] = from_f<T>(to_f<T>(__ldg(src + (long long)sx * k.C + c)));
    }
  }
}

__device__ void run_copy(const ObsKey& k, int b, int oy0, int oy1) {
  const long long row_b = (long long)k.W * k.C * k.esize;
  const int units = k.w * k.C * k.esize / k.vec;
  for (int oy = oy0; oy < oy1; ++oy) {
    const unsigned char* src = k.src + ((long long)b * k.H + k.y0 + oy) * row_b + (long long)k.x0 * k.C * k.esize;
    unsigned char* dst = k.dst + ((long long)b * k.h + oy) * units * (long long)k.vec;
    for (int u = threadIdx.x; u < units; u += blockDim.x) copy_unit(dst, src, u, k.vec);
  }
}

// grid: for each key, batch x bands CTAs (key-major); each CTA owns kObsBandRows output rows of one image
__global__ void __launch_bounds__(kObsThreads, 1) obs_resample_kernel(const __grid_constant__ ObsTable t) {
  extern __shared__ __align__(16) unsigned char smem[];
  int ki = 0;
  while (ki + 1 < t.n && (int)blockIdx.x >= t.k[ki + 1].first_block) ++ki;
  const ObsKey& k = t.k[ki];
  const int local = blockIdx.x - k.first_block;
  const int b = local / k.bands, band = local - b * k.bands;
  const int oy0 = band * kObsBandRows, oy1 = min(oy0 + kObsBandRows, k.h);
  if (k.mode == kModeCopy) {
    run_copy(k, b, oy0, oy1);
  } else if (k.mode == kModeArea) {
    if (k.dtype == kDtU8) run_area<unsigned char>(k, b, oy0, oy1, smem);
    else if (k.dtype == kDtF32) run_area<float>(k, b, oy0, oy1, smem);
    else run_area<int>(k, b, oy0, oy1, smem);
  } else {
    if (k.dtype == kDtU8) run_nearest<unsigned char>(k, b, oy0, oy1);
    else if (k.dtype == kDtF32) run_nearest<float>(k, b, oy0, oy1);
    else run_nearest<int>(k, b, oy0, oy1);
  }
}

int widest_vec(std::initializer_list<long long> vals) {
  for (int v : {16, 4}) {
    bool ok = true;
    for (long long x : vals) ok = ok && (x % v == 0);
    if (ok) return v;
  }
  return 1;
}

}  // namespace
}  // namespace hb200

using namespace hb200;

extern "C" int hb200_obs_resample(const void* const* src, void* const* dst, const int32_t* desc, int n_keys,
                                  int batch, hb200_stream_t stream) {
  HB_CHECK_ARG(src && dst && desc, "obs_resample: null argument");
  HB_CHECK_ARG(n_keys >= 1 && n_keys <= kObsMaxKeys, "obs_resample: n_keys = %d (1..%d)", n_keys, kObsMaxKeys);
  HB_CHECK_ARG(batch >= 1, "obs_resample: batch = %d", batch);
  ObsTable t{};
  t.n = n_keys;
  long long blocks = 0;
  int smem = 0;
  for (int i = 0; i < n_keys; ++i) {
    const int32_t* d = desc + 11 * i;
    ObsKey& k = t.k[i];
    k.src = static_cast<const unsigned char*>(src[i]);
    k.dst = static_cast<unsigned char*>(dst[i]);
    k.dtype = d[0]; k.mode = d[1]; k.H = d[2]; k.W = d[3]; k.C = d[4]; k.Hr = d[5]; k.Wr = d[6];
    k.y0 = d[7]; k.x0 = d[8]; k.h = d[9]; k.w = d[10];
    HB_CHECK_ARG(k.src && k.dst, "obs_resample: key %d: null pointer", i);
    HB_CHECK_ARG(k.dtype >= kDtU8 && k.dtype <= kDtI32, "obs_resample: key %d: dtype %d", i, k.dtype);
    HB_CHECK_ARG(k.mode >= kModeArea && k.mode <= kModeCopy, "obs_resample: key %d: mode %d", i, k.mode);
    HB_CHECK_ARG(k.H >= 1 && k.W >= 1 && k.C >= 1 && k.Hr >= 1 && k.Wr >= 1, "obs_resample: key %d: bad sizes", i);
    HB_CHECK_ARG(k.mode != kModeCopy || (k.Hr == k.H && k.Wr == k.W), "obs_resample: key %d: copy needs Hr=H, Wr=W",
                 i);
    HB_CHECK_ARG(k.h >= 1 && k.w >= 1 && k.y0 >= 0 && k.x0 >= 0 && k.y0 + k.h <= k.Hr && k.x0 + k.w <= k.Wr,
                 "obs_resample: key %d: window (%d, %d, %d, %d) outside the %dx%d resampled image", i, k.y0, k.x0,
                 k.h, k.w, k.Hr, k.Wr);
    k.esize = k.dtype == kDtU8 ? 1 : 4;
    const long long pitch_b = (long long)k.W * k.C * k.esize;
    // bin bounds are computed in 32-bit integers: (Hr + 1) * H and (Wr + 1) * W must fit
    HB_CHECK_ARG((long long)(k.Hr + 1) * k.H < (1LL << 31) && (long long)(k.Wr + 1) * k.W < (1LL << 31),
                 "obs_resample: key %d: sizes too large", i);
    HB_CHECK_ARG(pitch_b * k.H * batch < (1LL << 40) && (long long)k.w * k.C * k.esize < (1LL << 30),
                 "obs_resample: key %d: tensor too large", i);
    HB_CHECK_ARG((uintptr_t)k.src % k.esize == 0 && (uintptr_t)k.dst % k.esize == 0,
                 "obs_resample: key %d: pointer not aligned to its element size", i);
    k.bands = (k.h + kObsBandRows - 1) / kObsBandRows;
    k.first_block = (int)blocks;
    blocks += (long long)batch * k.bands;
    if (k.mode == kModeCopy) {
      k.vec = widest_vec({(long long)(uintptr_t)k.src, (long long)(uintptr_t)k.dst, pitch_b,
                          (long long)k.x0 * k.C * k.esize, (long long)k.w * k.C * k.esize});
    } else if (k.mode == kModeNearest) {
      k.nearest_scale = (float)k.H / (float)k.Hr;
    } else {
      k.vec = widest_vec({(long long)(uintptr_t)k.src, pitch_b});
      int kh = 0;
      for (int y = k.y0; y < k.y0 + k.h; ++y) {
        const int rs = (int)(((long long)y * k.H) / k.Hr);
        const int re = (int)(((long long)(y + 1) * k.H + k.Hr - 1) / k.Hr);
        kh = re - rs > kh ? re - rs : kh;
      }
      const long long c0 = ((long long)k.x0 * k.W) / k.Wr;
      const long long c1 = ((long long)(k.x0 + k.w) * k.W + k.Wr - 1) / k.Wr;
      const long long b0 = c0 * k.C * k.esize / k.vec * k.vec;
      const long long b1 = (c1 * k.C * k.esize + k.vec - 1) / k.vec * k.vec;
      const long long slot_pitch = (b1 - b0 + 15) / 16 * 16;
      if (kh * slot_pitch <= kObsSmemBudget) {
        k.slots = kh;
        k.seg_off = (int)b0;
        k.seg_bytes = (int)(b1 - b0);
        k.slot_pitch = (int)slot_pitch;
        smem = (int)(kh * slot_pitch) > smem ? (int)(kh * slot_pitch) : smem;
      }
    }
  }
  HB_CHECK_ARG(blocks < (1LL << 31), "obs_resample: grid too large");
  obs_resample_kernel<<<(unsigned)blocks, kObsThreads, smem, (cudaStream_t)stream>>>(t);
  HB_LAUNCH_OK();
  count_launch(1);
  return HB200_OK;
}
