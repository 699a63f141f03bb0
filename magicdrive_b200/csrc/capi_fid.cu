// FID Inception helpers (include/magicdrive_b200.h: mdb_pool2d, mdb_fid_input): the pooling layers of the FID
// InceptionV3 and its input step (8-bit rounding, bilinear resize to 299x299, 2x - 1).  Its convolutions run on
// mdb_gemm_conv.  Compiled WITHOUT --use_fast_math: the resize and the averages follow ATen's fp32 arithmetic.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>

#include "../../include/magicdrive_b200.h"
#include "common_host.h"

namespace {

// one thread per (output pixel, 8 channels): 16-byte loads and stores
__global__ void pool2d_kernel(const uint4* __restrict__ x, int ldx8, int n, int h, int w, int c8, int avg, int k,
                              int stride, int pad, uint4* __restrict__ o, int ldo8, int ho, int wo) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  const long long total = static_cast<long long>(n) * ho * wo * c8;
  if (i >= total) return;
  const int cv = static_cast<int>(i % c8);
  long long p = i / c8;
  const int ow = static_cast<int>(p % wo);
  p /= wo;
  const int oh = static_cast<int>(p % ho);
  const int img = static_cast<int>(p / ho);
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = avg ? 0.f : -INFINITY;
  int count = 0;
  const int h0 = oh * stride - pad, w0 = ow * stride - pad;
  for (int r = 0; r < k; ++r) {
    const int ih = h0 + r;
    if (ih < 0 || ih >= h) continue;
    for (int s = 0; s < k; ++s) {
      const int iw = w0 + s;
      if (iw < 0 || iw >= w) continue;
      const uint4 v = __ldg(x + ((static_cast<long long>(img) * h + ih) * w + iw) * ldx8 + cv);
      const __nv_bfloat162* hv = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __bfloat1622float2(hv[j]);
        if (avg) {
          acc[2 * j] += f.x, acc[2 * j + 1] += f.y;
        } else {
          acc[2 * j] = fmaxf(acc[2 * j], f.x), acc[2 * j + 1] = fmaxf(acc[2 * j + 1], f.y);
        }
      }
      ++count;
    }
  }
  if (avg) {
    const float inv = 1.0f / static_cast<float>(count);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] *= inv;
  }
  uint4 r;
  __nv_bfloat162* hr = reinterpret_cast<__nv_bfloat162*>(&r);
#pragma unroll
  for (int j = 0; j < 4; ++j) hr[j] = __floats2bfloat162_rn(acc[2 * j], acc[2 * j + 1]);
  o[(static_cast<long long>(img) * ho + oh) * wo * ldo8 + static_cast<long long>(ow) * ldo8 + cv] = r;
}

// global average pool: one thread per (image, 8 channels), pixels summed in order in fp32
__global__ void global_avgpool_kernel(const uint4* __restrict__ x, int ldx8, int n, int hw, int c8, float* __restrict__ o,
                                      int ldo) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * c8) return;
  const int cv = i % c8, img = i / c8;
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  for (int p = 0; p < hw; ++p) {
    const uint4 v = __ldg(x + (static_cast<long long>(img) * hw + p) * ldx8 + cv);
    const __nv_bfloat162* hv = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = __bfloat1622float2(hv[j]);
      acc[2 * j] += f.x, acc[2 * j + 1] += f.y;
    }
  }
  const float inv = 1.0f / static_cast<float>(hw);
  float4* dst = reinterpret_cast<float4*>(o + static_cast<long long>(img) * ldo + 8 * cv);
  dst[0] = make_float4(acc[0] * inv, acc[1] * inv, acc[2] * inv, acc[3] * inv);
  dst[1] = make_float4(acc[4] * inv, acc[5] * inv, acc[6] * inv, acc[7] * inv);
}

template <typename T>
__device__ __forceinline__ float ldf(const T* p);
template <>
__device__ __forceinline__ float ldf<float>(const float* p) { return __ldg(p); }
template <>
__device__ __forceinline__ float ldf<__nv_bfloat16>(const __nv_bfloat16* p) { return __bfloat162float(*p); }

// ATen's upsample_bilinear2d source index (align_corners=False): max(scale * (dst + 0.5) - 0.5, 0), scale = in / out
__device__ __forceinline__ void src_index(int dst, int in, int out, int* i0, int* i1, float* l1) {
  const float scale = static_cast<float>(in) / static_cast<float>(out);
  const float real = fmaxf(scale * (static_cast<float>(dst) + 0.5f) - 0.5f, 0.f);
  const int i = static_cast<int>(real);
  *i0 = i;
  *i1 = i + (i < in - 1 ? 1 : 0);
  *l1 = real - static_cast<float>(i);
}

// one thread per output pixel: 3 channels in, 8 bf16 channels out (3..7 zero)
template <typename T>
__global__ void fid_input_kernel(const T* __restrict__ x, int nhwc, int n, int h, int w, int quantize, int normalize,
                                 uint4* __restrict__ o, int ho, int wo) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long long>(n) * ho * wo) return;
  const int ow = static_cast<int>(i % wo);
  const int oh = static_cast<int>((i / wo) % ho);
  const int img = static_cast<int>(i / (static_cast<long long>(wo) * ho));
  int h0, h1, w0, w1;
  float lh, lw;
  src_index(oh, h, ho, &h0, &h1, &lh);
  src_index(ow, w, wo, &w0, &w1, &lw);
  const long long hw = static_cast<long long>(h) * w;
  auto at = [&](int ch, int ih, int iw) {
    const long long off = nhwc ? ((img * hw + static_cast<long long>(ih) * w + iw) * 3 + ch)
                               : ((static_cast<long long>(img) * 3 + ch) * hw + static_cast<long long>(ih) * w + iw);
    float v = ldf(x + off);
    if (quantize) v = fminf(fmaxf(rintf(v * 255.f), 0.f), 255.f) / 255.f;
    return v;
  };
  float res[3];
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    // the order of ATen's CPU kernel: h0l * (w0l * x00 + w1l * x01) + h1l * (w0l * x10 + w1l * x11)
    const float top = (1.f - lw) * at(ch, h0, w0) + lw * at(ch, h0, w1);
    const float bot = (1.f - lw) * at(ch, h1, w0) + lw * at(ch, h1, w1);
    const float v = (1.f - lh) * top + lh * bot;
    res[ch] = normalize ? 2.f * v - 1.f : v;
  }
  uint4 r;
  __nv_bfloat162* hr = reinterpret_cast<__nv_bfloat162*>(&r);
  hr[0] = __floats2bfloat162_rn(res[0], res[1]);
  hr[1] = __floats2bfloat162_rn(res[2], 0.f);
  hr[2] = __floats2bfloat162_rn(0.f, 0.f);
  hr[3] = hr[2];
  o[i] = r;
}

inline unsigned blocks_for(long long total, int threads) { return static_cast<unsigned>((total + threads - 1) / threads); }

}  // namespace

extern "C" int mdb_pool2d(const void* x, int ldx, int n, int h, int w, int c, int mode, int k, int stride, int pad,
                          void* out, int ldo, int ho, int wo, void* stream) {
  if (!x || !out) return mdb::set_error(MDB_ERR_INVALID, "mdb_pool2d: null pointer");
  if (c <= 0 || c % 8 || ldx % 8 || ldo % 8 || ldx < c || ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(out)) & 15))
    return mdb::set_error(MDB_ERR_UNSUPPORTED, "mdb_pool2d: c, ldx, ldo must be multiples of 8 and pointers 16-byte aligned");
  if (n <= 0 || h <= 0 || w <= 0) return mdb::set_error(MDB_ERR_INVALID, "mdb_pool2d: bad shape");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int threads = 256;
  if (mode == 2) {
    if (ldo < c) return mdb::set_error(MDB_ERR_INVALID, "mdb_pool2d: ldo < c");
    global_avgpool_kernel<<<blocks_for((long long)n * (c / 8), threads), threads, 0, st>>>(
        static_cast<const uint4*>(x), ldx / 8, n, h * w, c / 8, static_cast<float*>(out), ldo);
    MDB_CHECK_LAUNCH("global_avgpool_kernel");
    return MDB_OK;
  }
  if (mode != 0 && mode != 1) return mdb::set_error(MDB_ERR_INVALID, "mdb_pool2d: mode must be 0, 1 or 2");
  if (k <= 0 || stride <= 0 || pad < 0 || pad > k / 2 || ho <= 0 || wo <= 0 || ldo < c ||
      (ho - 1) * stride - pad + k > h + pad || (wo - 1) * stride - pad + k > w + pad)
    return mdb::set_error(MDB_ERR_INVALID, "mdb_pool2d: bad window (k=%d stride=%d pad=%d %dx%d -> %dx%d)", k, stride, pad, h,
                          w, ho, wo);
  const long long total = (long long)n * ho * wo * (c / 8);
  pool2d_kernel<<<blocks_for(total, threads), threads, 0, st>>>(static_cast<const uint4*>(x), ldx / 8, n, h, w, c / 8,
                                                                 mode == 1, k, stride, pad, static_cast<uint4*>(out), ldo / 8,
                                                                 ho, wo);
  MDB_CHECK_LAUNCH("pool2d_kernel");
  return MDB_OK;
}

extern "C" int mdb_fid_input(const void* x, int x_is_f32, int x_is_nhwc, int n, int h, int w, int quantize, int normalize,
                             void* out, int ho, int wo, void* stream) {
  if (!x || !out) return mdb::set_error(MDB_ERR_INVALID, "mdb_fid_input: null pointer");
  if (n <= 0 || h <= 0 || w <= 0 || ho <= 0 || wo <= 0) return mdb::set_error(MDB_ERR_INVALID, "mdb_fid_input: bad shape");
  if (reinterpret_cast<uintptr_t>(out) & 15) return mdb::set_error(MDB_ERR_INVALID, "mdb_fid_input: out must be 16-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int threads = 256;
  const long long total = (long long)n * ho * wo;
  if (x_is_f32)
    fid_input_kernel<float><<<blocks_for(total, threads), threads, 0, st>>>(static_cast<const float*>(x), x_is_nhwc, n, h, w,
                                                                            quantize, normalize, static_cast<uint4*>(out), ho, wo);
  else
    fid_input_kernel<__nv_bfloat16><<<blocks_for(total, threads), threads, 0, st>>>(
        static_cast<const __nv_bfloat16*>(x), x_is_nhwc, n, h, w, quantize, normalize, static_cast<uint4*>(out), ho, wo);
  MDB_CHECK_LAUNCH("fid_input_kernel");
  return MDB_OK;
}
