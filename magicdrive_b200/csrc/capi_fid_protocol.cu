// FID evaluation protocol (include/magicdrive_b200.h: mdb_resample_u8, mdb_jpeg_roundtrip_u8): the 8-bit image steps the
// reference's FID chain applies between the pipeline's views and Inception -- an antialiased bicubic resize with a zero pad
// or a crop, and a JPEG save and load -- restated as integer arithmetic so that the results equal Pillow's byte for byte.
// oracle/fid_protocol.py is the same arithmetic in numpy.  Everything here is integer except the fp32 -> uint8 rounding of
// the input, which uses explicitly rounded operations.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/magicdrive_b200.h"
#include "common_host.h"
#include "jpeg_fdct.cuh"

namespace {

constexpr int kPrecisionBits = 22;  // fraction bits of the resample weights

// ------------------------------------------------------------------------------------------------------------- resample
// A source image of n x h x w RGB pixels: uint8 NHWC, or fp32 [0, 1] NHWC / NCHW rounded as numpy_to_pil does,
// (x * 255).round() in fp32 with ties to even.
struct SrcU8 {
  const uint8_t* p;
  int h, w;
  __device__ __forceinline__ int at(int img, int y, int x, int c) const {
    return p[((static_cast<long long>(img) * h + y) * w + x) * 3 + c];
  }
};
struct SrcF32 {
  const float* p;
  int h, w, nhwc;
  __device__ __forceinline__ int at(int img, int y, int x, int c) const {
    const long long hw = static_cast<long long>(h) * w;
    const long long off = nhwc ? ((img * hw + static_cast<long long>(y) * w + x) * 3 + c)
                               : ((static_cast<long long>(img) * 3 + c) * hw + static_cast<long long>(y) * w + x);
    const float v = rintf(__fmul_rn(__ldg(p + off), 255.f));
    return static_cast<int>(fminf(fmaxf(v, 0.f), 255.f));
  }
};

__device__ __forceinline__ uint8_t clip_weighted(int acc) {
  const int v = acc >> kPrecisionBits;
  return static_cast<uint8_t>(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// Horizontal pass: tmp[img, y, j] = resampled column crop_left + j of input row y, for y < h and j < cw.
// coef row i: [first input column, tap count, weights...] (stride taps + 2).
template <typename Src>
__global__ void resample_h_kernel(Src src, int n, const int* __restrict__ coef, int taps, int crop_left, int cw,
                                  uint8_t* __restrict__ tmp) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long long>(n) * src.h * cw) return;
  const int j = static_cast<int>(i % cw);
  const int y = static_cast<int>((i / cw) % src.h);
  const int img = static_cast<int>(i / (static_cast<long long>(cw) * src.h));
  const int* k = coef + static_cast<long long>(crop_left + j) * (taps + 2);
  const int x0 = __ldg(k), cnt = __ldg(k + 1);
  int acc[3] = {1 << (kPrecisionBits - 1), 1 << (kPrecisionBits - 1), 1 << (kPrecisionBits - 1)};
  for (int t = 0; t < cnt; ++t) {
    const int wt = __ldg(k + 2 + t);
#pragma unroll
    for (int c = 0; c < 3; ++c) acc[c] += src.at(img, y, x0 + t, c) * wt;
  }
  uint8_t* o = tmp + i * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) o[c] = clip_weighted(acc[c]);
}

// Vertical pass (or a plain copy when coef is null) and placement: canvas pixel (top + i, left + j) takes row crop_top + i,
// column j of the source (columns already cropped), every other canvas pixel is zero.
template <typename Src>
__global__ void resample_v_place_kernel(Src src, int n, const int* __restrict__ coef, int taps, int crop_top, int ch,
                                        int cw, uint8_t* __restrict__ out, int oh, int ow, int top, int left) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long long>(n) * oh * ow) return;
  const int ox = static_cast<int>(i % ow);
  const int oy = static_cast<int>((i / ow) % oh);
  const int img = static_cast<int>(i / (static_cast<long long>(ow) * oh));
  uint8_t* o = out + i * 3;
  const int r = oy - top, j = ox - left;
  if (r < 0 || r >= ch || j < 0 || j >= cw) {
    o[0] = o[1] = o[2] = 0;
    return;
  }
  if (!coef) {
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = static_cast<uint8_t>(src.at(img, crop_top + r, j, c));
    return;
  }
  const int* k = coef + static_cast<long long>(crop_top + r) * (taps + 2);
  const int y0 = __ldg(k), cnt = __ldg(k + 1);
  int acc[3] = {1 << (kPrecisionBits - 1), 1 << (kPrecisionBits - 1), 1 << (kPrecisionBits - 1)};
  for (int t = 0; t < cnt; ++t) {
    const int wt = __ldg(k + 2 + t);
#pragma unroll
    for (int c = 0; c < 3; ++c) acc[c] += src.at(img, y0 + t, j, c) * wt;
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) o[c] = clip_weighted(acc[c]);
}

// Source view shifted right by `x0` columns: the vertical pass reads the input directly when the width is unchanged.
template <typename Src>
struct Shifted {
  Src s;
  int x0;
  __device__ __forceinline__ int at(int img, int y, int x, int c) const { return s.at(img, y, x + x0, c); }
};

inline unsigned blocks_for(long long total, int threads) { return static_cast<unsigned>((total + threads - 1) / threads); }

template <typename Src>
int launch_resample(Src src, int n, const int* coef_w, int taps_w, const int* coef_h, int taps_h, int crop_top,
                    int crop_left, int ch, int cw, uint8_t* tmp, uint8_t* out, int oh, int ow, int top, int left,
                    cudaStream_t st) {
  const int threads = 256;
  const long long total = static_cast<long long>(n) * oh * ow;
  if (coef_w) {
    resample_h_kernel<Src><<<blocks_for(static_cast<long long>(n) * src.h * cw, threads), threads, 0, st>>>(
        src, n, coef_w, taps_w, crop_left, cw, tmp);
    MDB_CHECK_LAUNCH("resample_h_kernel");
    SrcU8 t{tmp, src.h, cw};
    resample_v_place_kernel<SrcU8><<<blocks_for(total, threads), threads, 0, st>>>(t, n, coef_h, taps_h, crop_top, ch, cw,
                                                                                   out, oh, ow, top, left);
  } else {
    Shifted<Src> s{src, crop_left};
    resample_v_place_kernel<Shifted<Src>><<<blocks_for(total, threads), threads, 0, st>>>(s, n, coef_h, taps_h, crop_top,
                                                                                          ch, cw, out, oh, ow, top, left);
  }
  MDB_CHECK_LAUNCH("resample_v_place_kernel");
  return MDB_OK;
}

// ----------------------------------------------------------------------------------------------------------------- JPEG
template <int kShift>
__device__ __forceinline__ void idct8(int* p, int s) {
  const int e = (p[2 * s] + p[6 * s]) * F0541;
  const int t2 = e - p[6 * s] * F1847, t3 = e + p[2 * s] * F0765;
  const int t0 = (p[0] + p[4 * s]) * (1 << kConstBits), t1 = (p[0] - p[4 * s]) * (1 << kConstBits);
  const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  const int o0 = p[7 * s], o1 = p[5 * s], o2 = p[3 * s], o3 = p[s];
  const int z5 = (o0 + o2 + o1 + o3) * F1175;
  const int z1 = -(o0 + o3) * F0899, z2 = -(o1 + o2) * F2562;
  const int z3 = -(o0 + o2) * F1961 + z5, z4 = -(o1 + o3) * F0390 + z5;
  const int a0 = o0 * F0298 + z1 + z3, a1 = o1 * F2053 + z2 + z4;
  const int a2 = o2 * F3072 + z2 + z3, a3 = o3 * F1501 + z1 + z4;
  p[0] = descale(t10 + a3, kShift);
  p[7 * s] = descale(t10 - a3, kShift);
  p[s] = descale(t11 + a2, kShift);
  p[6 * s] = descale(t11 - a2, kShift);
  p[2 * s] = descale(t12 + a1, kShift);
  p[5 * s] = descale(t12 - a1, kShift);
  p[3 * s] = descale(t13 + a0, kShift);
  p[4 * s] = descale(t13 - a0, kShift);
}

// centred inverse-DCT output -> sample: wrapped modulo 1024 into [-512, 511], then x + 128 clipped to 0..255
__device__ __forceinline__ uint8_t range_limit(int x) {
  x = ((x + 512) & 1023) - 512;
  x += 128;
  return static_cast<uint8_t>(x < 0 ? 0 : (x > 255 ? 255 : x));
}

// One CTA per 16 x 16 MCU of one image: colour conversion, chroma averaging, and for each of the six 8 x 8 blocks the
// forward DCT, quantisation, dequantisation and inverse DCT.  Writes the decoder's reconstructed planes: Y [hp, wp] and
// Cb, Cr [hp / 2, wp / 2] per image (hp, wp: h, w rounded up to 16).
__global__ void __launch_bounds__(256) jpeg_code_mcu_kernel(const uint8_t* __restrict__ x, int h, int w, QuantTables qt,
                                                            uint8_t* __restrict__ planes) {
  __shared__ int blk[6][64];  // Y00, Y01, Y10, Y11, Cb, Cr
  const int mcus_x = (w + 15) >> 4;
  const int my = blockIdx.x / mcus_x, mx = blockIdx.x % mcus_x, img = blockIdx.y;
  const int hp = ((h + 15) >> 4) << 4, wp = ((w + 15) >> 4) << 4;
  const int t = threadIdx.x;
  load_mcu(x, h, w, img, my, mx, blk);
  __syncthreads();
  const int b = t >> 3, k = t & 7;  // 48 threads: block b, row / column k
  if (t < 48) fdct8<true>(&blk[b][k * 8], 1);
  __syncthreads();
  if (t < 48) {
    int* col = &blk[b][k];
    fdct8<false>(col, 8);
    const int* q = qt.q[b < 4 ? 0 : 1];
#pragma unroll
    for (int r = 0; r < 8; ++r) {  // quantise (round half away from zero), dequantise
      const int v = col[8 * r], qq = q[8 * r + k], d = qq * 8;
      const int a = ((v < 0 ? -v : v) + (d >> 1)) / d;
      col[8 * r] = (v < 0 ? -a : a) * qq;
    }
    idct8<kConstBits - kPass1Bits>(col, 8);
  }
  __syncthreads();
  if (t < 48) {
    int* row = &blk[b][k * 8];
    idct8<kConstBits + kPass1Bits + 3>(row, 1);
    const long long ysz = static_cast<long long>(hp) * wp, csz = ysz / 4;
    uint8_t* dst;
    if (b < 4) {
      dst = planes + img * ysz * 3 / 2 + static_cast<long long>(my * 16 + (b >> 1) * 8 + k) * wp + mx * 16 + (b & 1) * 8;
    } else {
      dst = planes + img * ysz * 3 / 2 + ysz + (b - 4) * csz + static_cast<long long>(my * 8 + k) * (wp / 2) + mx * 8;
    }
    uint32_t lo = 0, hi = 0;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      lo |= static_cast<uint32_t>(range_limit(row[c])) << (8 * c);
      hi |= static_cast<uint32_t>(range_limit(row[c + 4])) << (8 * c);
    }
    *reinterpret_cast<uint2*>(dst) = make_uint2(lo, hi);
  }
}

// YCbCr -> RGB in 16 fraction bits, from lookup values nearest to 1.402 Cr, 1.772 Cb and -0.34414 Cb - 0.71414 Cr
constexpr int kCrR = 91881, kCbB = 116130, kCbG = 22554, kCrG = 46802;  // FIX(1.402), FIX(1.772), FIX(0.34414), FIX(0.71414)
__device__ __forceinline__ uint8_t clamp255(int v) { return static_cast<uint8_t>(v < 0 ? 0 : (v > 255 ? 255 : v)); }

// One thread per output pixel: triangle ("fancy") 2x upsampling of the chroma, 3/4 of the nearest chroma sample and 1/4 of
// the next nearest in each direction with the edges replicated, rounded with 8 (even outputs) or 7 (odd) before >> 4;
// chroma planes of 1 or 2 samples per row are replicated instead.  Then the colour conversion.
__global__ void jpeg_color_kernel(const uint8_t* __restrict__ planes, int n, int h, int w, uint8_t* __restrict__ out) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long long>(n) * h * w) return;
  const int xx = static_cast<int>(i % w);
  const int yy = static_cast<int>((i / w) % h);
  const int img = static_cast<int>(i / (static_cast<long long>(w) * h));
  const int hp = ((h + 15) >> 4) << 4, wp = ((w + 15) >> 4) << 4;
  const int hc = (h + 1) >> 1, wc = (w + 1) >> 1, cld = wp / 2;
  const long long ysz = static_cast<long long>(hp) * wp;
  const uint8_t* yp = planes + img * ysz * 3 / 2;
  const uint8_t* cp[2] = {yp + ysz, yp + ysz + ysz / 4};
  const int cy = yy >> 1, cx = xx >> 1;
  int c[2];
  if (wc <= 2) {
#pragma unroll
    for (int p = 0; p < 2; ++p) c[p] = cp[p][cy * cld + cx];
  } else {
    const int fy = min(max((yy & 1) ? cy + 1 : cy - 1, 0), hc - 1);
    const int fx = min(max((xx & 1) ? cx + 1 : cx - 1, 0), wc - 1);
    const int bias = (xx & 1) ? 7 : 8;
#pragma unroll
    for (int p = 0; p < 2; ++p) {
      const uint8_t* near = cp[p] + cy * cld;
      const uint8_t* far = cp[p] + fy * cld;
      const int s0 = 3 * near[cx] + far[cx], s1 = 3 * near[fx] + far[fx];
      c[p] = (3 * s0 + s1 + bias) >> 4;
    }
  }
  const int y = yp[static_cast<long long>(yy) * wp + xx];
  const int cb = c[0] - 128, cr = c[1] - 128;
  uint8_t* o = out + i * 3;
  o[0] = clamp255(y + ((kCrR * cr + kHalf) >> 16));
  o[1] = clamp255(y + ((-kCbG * cb - kCrG * cr + kHalf) >> 16));
  o[2] = clamp255(y + ((kCbB * cb + kHalf) >> 16));
}

}  // namespace

extern "C" int mdb_resample_u8(const void* x, int x_is_f32, int x_is_nhwc, int n, int h, int w, const int* coef_w,
                               int taps_w, int rw, const int* coef_h, int taps_h, int rh, int crop_top, int crop_left,
                               int crop_h, int crop_w, void* tmp, void* out, int out_h, int out_w, int top, int left,
                               void* stream) {
  if (!x || !out) return mdb::set_error(MDB_ERR_INVALID, "mdb_resample_u8: null pointer");
  if (n <= 0 || h <= 0 || w <= 0 || rh <= 0 || rw <= 0 || out_h <= 0 || out_w <= 0)
    return mdb::set_error(MDB_ERR_INVALID, "mdb_resample_u8: bad shape");
  if (!x_is_f32 && !x_is_nhwc) return mdb::set_error(MDB_ERR_UNSUPPORTED, "mdb_resample_u8: uint8 input must be NHWC");
  if ((coef_w == nullptr) != (rw == w) || (coef_h == nullptr) != (rh == h) || (coef_w && taps_w <= 0) ||
      (coef_h && taps_h <= 0))
    return mdb::set_error(MDB_ERR_INVALID,
                          "mdb_resample_u8: coefficients are required exactly for the changed sizes (%dx%d -> %dx%d)", h, w,
                          rh, rw);
  if (crop_h <= 0 || crop_w <= 0 || crop_top < 0 || crop_left < 0 || crop_top + crop_h > rh || crop_left + crop_w > rw)
    return mdb::set_error(MDB_ERR_INVALID, "mdb_resample_u8: crop (%d, %d, %dx%d) outside the %dx%d resize", crop_top,
                          crop_left, crop_h, crop_w, rh, rw);
  if (top < 0 || left < 0 || top + crop_h > out_h || left + crop_w > out_w)
    return mdb::set_error(MDB_ERR_INVALID, "mdb_resample_u8: window %dx%d at (%d, %d) outside the %dx%d canvas", crop_h,
                          crop_w, top, left, out_h, out_w);
  if (coef_w && !tmp) return mdb::set_error(MDB_ERR_INVALID, "mdb_resample_u8: a width change needs tmp");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  uint8_t* t = static_cast<uint8_t*>(tmp);
  uint8_t* o = static_cast<uint8_t*>(out);
  if (x_is_f32)
    return launch_resample(SrcF32{static_cast<const float*>(x), h, w, x_is_nhwc}, n, coef_w, taps_w, coef_h, taps_h,
                           crop_top, crop_left, crop_h, crop_w, t, o, out_h, out_w, top, left, st);
  return launch_resample(SrcU8{static_cast<const uint8_t*>(x), h, w}, n, coef_w, taps_w, coef_h, taps_h, crop_top,
                         crop_left, crop_h, crop_w, t, o, out_h, out_w, top, left, st);
}

extern "C" int mdb_jpeg_roundtrip_u8(const void* x, int n, int h, int w, int quality, void* planes, void* out,
                                     void* stream) {
  if (!x || !planes || !out) return mdb::set_error(MDB_ERR_INVALID, "mdb_jpeg_roundtrip_u8: null pointer");
  if (n <= 0 || h <= 0 || w <= 0) return mdb::set_error(MDB_ERR_INVALID, "mdb_jpeg_roundtrip_u8: bad shape");
  if (quality < 1 || quality > 100)
    return mdb::set_error(MDB_ERR_INVALID, "mdb_jpeg_roundtrip_u8: quality %d outside 1..100", quality);
  if (reinterpret_cast<uintptr_t>(planes) & 7)
    return mdb::set_error(MDB_ERR_INVALID, "mdb_jpeg_roundtrip_u8: planes must be 8-byte aligned");
  if (static_cast<long long>((h + 15) / 16) * ((w + 15) / 16) > 0x7fffffffLL || n > 65535)
    return mdb::set_error(MDB_ERR_UNSUPPORTED, "mdb_jpeg_roundtrip_u8: too many MCUs or images");
  const QuantTables qt = quant_tables(quality);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const dim3 grid(((h + 15) / 16) * ((w + 15) / 16), n);
  jpeg_code_mcu_kernel<<<grid, 256, 0, st>>>(static_cast<const uint8_t*>(x), h, w, qt, static_cast<uint8_t*>(planes));
  MDB_CHECK_LAUNCH("jpeg_code_mcu_kernel");
  const long long total = static_cast<long long>(n) * h * w;
  jpeg_color_kernel<<<blocks_for(total, 256), 256, 0, st>>>(static_cast<const uint8_t*>(planes), n, h, w,
                                                            static_cast<uint8_t*>(out));
  MDB_CHECK_LAUNCH("jpeg_color_kernel");
  return MDB_OK;
}
