// The forward half of the baseline JPEG codec shared by the FID protocol's round trip (capi_fid_protocol.cu) and the
// encoder (capi_jpeg.cu): IJG libjpeg's colour conversion, 4:2:0 chroma sums, islow forward DCT and quantisation tables.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace {

// Integer Loeffler-Ligtenberg-Moschytz 8-point DCT pair: 13 fraction bits in the rotations, 2 extra bits kept between
// the passes.  The forward output is 8x the orthonormal DCT; the inverse output carries 3 more bits that its second pass
// removes.
constexpr int kConstBits = 13, kPass1Bits = 2;
constexpr int F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633;
constexpr int F1501 = 12299, F1847 = 15137, F1961 = 16069, F2053 = 16819, F2562 = 20995, F3072 = 25172;

__device__ __forceinline__ int descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }

// forward transform of 8 values at p[0], p[s], ..., p[7 s]; the first pass keeps the even outputs exact (shifted left),
// the second rounds them away
template <bool kFirst>
__device__ __forceinline__ void fdct8(int* p, int s) {
  constexpr int odd = kFirst ? kConstBits - kPass1Bits : kConstBits + kPass1Bits;
  const int t0 = p[0] + p[7 * s], t7 = p[0] - p[7 * s];
  const int t1 = p[s] + p[6 * s], t6 = p[s] - p[6 * s];
  const int t2 = p[2 * s] + p[5 * s], t5 = p[2 * s] - p[5 * s];
  const int t3 = p[3 * s] + p[4 * s], t4 = p[3 * s] - p[4 * s];
  const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  if (kFirst) {
    p[0] = (t10 + t11) * (1 << kPass1Bits);
    p[4 * s] = (t10 - t11) * (1 << kPass1Bits);
  } else {
    p[0] = descale(t10 + t11, kPass1Bits);
    p[4 * s] = descale(t10 - t11, kPass1Bits);
  }
  const int e = (t12 + t13) * F0541;
  p[2 * s] = descale(e + t13 * F0765, odd);
  p[6 * s] = descale(e - t12 * F1847, odd);
  const int z5 = (t4 + t6 + t5 + t7) * F1175;
  const int z1 = -(t4 + t7) * F0899, z2 = -(t5 + t6) * F2562;
  const int z3 = -(t4 + t6) * F1961 + z5, z4 = -(t5 + t7) * F0390 + z5;
  p[7 * s] = descale(t4 * F0298 + z1 + z3, odd);
  p[5 * s] = descale(t5 * F2053 + z2 + z4, odd);
  p[3 * s] = descale(t6 * F3072 + z2 + z3, odd);
  p[s] = descale(t7 * F1501 + z1 + z4, odd);
}

// BT.601 RGB -> YCbCr in 16 fraction bits; Cb and Cr round with 1/2 - 2^-16 so that they never exceed 255
constexpr int kRY = 19595, kGY = 38470, kBY = 7471, kRCb = 11059, kGCb = 21709, kHalf = 32768;  // FIX(0.299) ...
constexpr int kGCr = 27439, kBCr = 5329, kHalfC = 32768;                                         // FIX(0.41869) ...
__device__ __forceinline__ void rgb_ycc(int r, int g, int b, int* y, int* cb, int* cr) {
  *y = (kRY * r + kGY * g + kBY * b + kHalf) >> 16;
  *cb = (-kRCb * r - kGCb * g + kHalfC * b + (128 << 16) + kHalf - 1) >> 16;
  *cr = (kHalfC * r - kGCr * g - kBCr * b + (128 << 16) + kHalf - 1) >> 16;
}

struct QuantTables {
  int q[2][64];  // luma, chroma; natural order
};

// ITU-T T.81 Annex K.1, natural order
constexpr unsigned char kStdLuma[64] = {16, 11, 10, 16, 24,  40,  51,  61,  12, 12, 14, 19, 26,  58,  60,  55,
                                        14, 13, 16, 24, 40,  57,  69,  56,  14, 17, 22, 29, 51,  87,  80,  62,
                                        18, 22, 37, 56, 68,  109, 103, 77,  24, 35, 55, 64, 81,  104, 113, 92,
                                        49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
constexpr unsigned char kStdChroma[64] = {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99,
                                          24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99, 99, 99, 99, 99,
                                          99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
                                          99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99};

// The 16 x 16 MCU (my, mx) of image img of x (uint8 RGB [n, h, w, 3]) as centred samples, one per thread of 256:
// blk[0..3] the luma blocks Y00, Y01, Y10, Y11, blk[4], blk[5] the 8 x 8 Cb, Cr blocks.
__device__ __forceinline__ void load_mcu(const uint8_t* __restrict__ x, int h, int w, int img, int my, int mx,
                                         int (*blk)[64]) {
  const int hc = (h + 1) >> 1;
  const uint8_t* src = x + static_cast<long long>(img) * h * w * 3;
  const int t = threadIdx.x;
  auto pixel = [&](int yy, int xx, int* r, int* g, int* b) {
    const uint8_t* p = src + (static_cast<long long>(yy) * w + xx) * 3;
    *r = p[0], *g = p[1], *b = p[2];
  };
  {  // luma: the last row and column replicated
    const int py = t >> 4, px = t & 15;
    int r, g, b, y, cb, cr;
    pixel(min(my * 16 + py, h - 1), min(mx * 16 + px, w - 1), &r, &g, &b);
    rgb_ycc(r, g, b, &y, &cb, &cr);
    blk[(py >> 3) * 2 + (px >> 3)][(py & 7) * 8 + (px & 7)] = y - 128;
  }
  if (t < 64) {  // chroma: 2 x 2 sums of full-resolution samples (columns replicated, rows replicated to an even count),
                 // bias 1, 2, 1, 2 along the row; chroma rows past the image replicate the last chroma row
    const int cy = t >> 3, cx = t & 7;
    const int gy = min(my * 8 + cy, hc - 1), gx = mx * 8 + cx;
    int scb = 0, scr = 0;
#pragma unroll
    for (int d = 0; d < 4; ++d) {
      int r, g, b, y, cb, cr;
      pixel(min(2 * gy + (d >> 1), h - 1), min(2 * gx + (d & 1), w - 1), &r, &g, &b);
      rgb_ycc(r, g, b, &y, &cb, &cr);
      scb += cb, scr += cr;
    }
    const int bias = (gx & 1) ? 2 : 1;
    blk[4][t] = ((scb + bias) >> 2) - 128;
    blk[5][t] = ((scr + bias) >> 2) - 128;
  }
}

// quality 1..100 -> the standard tables scaled as libjpeg's jpeg_quality_scaling and clamped to the baseline 1..255
inline QuantTables quant_tables(int quality) {
  QuantTables qt;
  const int scale = quality < 50 ? 5000 / quality : 200 - 2 * quality;
  for (int i = 0; i < 64; ++i) {
    const int l = (kStdLuma[i] * scale + 50) / 100, c = (kStdChroma[i] * scale + 50) / 100;
    qt.q[0][i] = l < 1 ? 1 : (l > 255 ? 255 : l);
    qt.q[1][i] = c < 1 ? 1 : (c > 255 ? 255 : c);
  }
  return qt;
}

}  // namespace
