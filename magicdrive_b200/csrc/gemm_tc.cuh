// Operand scheme and shared definitions of the tensor-core GEMM / implicit-GEMM convolution for sm_90a
// (gemm_wgmma.cuh: persistent warp-specialised kernel, TMA producer + two wgmma consumer warpgroups, on single CTAs
// with split-K or on 2-CTA clusters that share each weight tile through TMA multicast).
//
//   D[pixel, n] = sum_{tap, c}  A[pixel shifted by tap, c] * W[n, tap*C + c]      (+ epilogue)
//
// * A is an NHWC bf16 activation tensor.  M tile mt is the 128 consecutive output pixels [128 mt, 128 mt + 128) of the
//   flattened (image, row, column) order, whatever the image and row boundaries, so only the last tile has idle rows.
//   - Convolutions (taps > 1, stride or padding): a 4-D (C, W, H, N) TMA map in im2col mode.  Each filter tap loads the
//     tile's 128 pixels shifted by (s, r); the TMA walks across row and image ends, zero-fills the halo and the pixels
//     past the last image, and steps by the stride through the map's element strides.  No im2col buffer exists.
//   - 1x1 / stride-1 launches (plain GEMMs): a 2-D [pixels, C] tiled map with row stride lda.
//   Two A sources are supported (the K loop runs over source 0's channels then source 1's): this is how
//   channel-concatenated inputs (UNet skip connections) are consumed without materialising the concat.
// * W is a bf16 [N, K] (K-major) matrix behind a 2-D tensor map, K ordered (tap, channel).
// * Both operands land in shared memory with the 128-byte swizzle and are consumed by wgmma
//   (per consumer warpgroup M=64, N=BLOCK_N, K=16, bf16 x bf16 -> fp32 in registers).
#pragma once
#include "ptx.cuh"

namespace mdb {

// EPI_QUICK_GELU is mdb_gemm_desc.epi_mode 2 (internal 2 is the split-K partial store), EPI_RELU is epi_mode 3
enum EpiMode : int { EPI_LINEAR = 0, EPI_GEGLU = 1, EPI_PARTIAL_F32 = 2, EPI_QUICK_GELU = 3, EPI_RELU = 4 };

struct GemmParams {
  // output pixel grid
  int n_img, h_out, w_out;
  int n_out;  // GEMM N (for GEGLU: the packed 2x width)
  // filter
  int taps_h, taps_w, stride, pad_h, pad_w;
  int cblocks0, cblocks1;  // 64-channel blocks of A source 0 / 1 (the last one partial, zero-filled, if C % 64 != 0)
  int im2col;              // A maps: 1 = 4-D im2col (convolutions), 0 = 2-D [pixels, C] (1x1)
  int m_tiles, n_tiles, splits;  // tiles = m_tiles * n_tiles * splits (m fastest); m_tiles = ceil(pixels / 128)
  int m_groups;                  // ceil(m_tiles / CTAS): M tiles are walked in groups of one per CTA of a cluster
  int kb_per_split;
  // epilogue
  int epi_mode;
  int out_is_f32;
  const float* bias;     // [n_out] or nullptr
  const float* rowbias;  // [n_img][rowbias_ld] or nullptr (time-embedding shift, per image)
  int rowbias_ld;
  const __nv_bfloat16* residual;  // [pixels][ldr] or nullptr
  int ldr;
  void* out;  // bf16 or fp32 [pixels][ldo]
  int ldo;
  float out_scale;
  float* partial;  // [splits][pixels][n_out] fp32 workspace (EPI_PARTIAL_F32)
  // LayerNorm folded into this GEMM (consumer side): out = rstd * scale * (acc - mean * colsum_n) + c_n
  const float* ln_stats;   // [pixels][ln_parts][2] partial (sum, sum sq) of the A rows, or nullptr
  int ln_parts;
  float ln_inv_c, ln_eps;
  const float* ln_colsum;  // [n_out] sum_k W'[n, k]
  // row statistics of this GEMM's output (producer side): [pixels][n_tiles][2] partial (sum, sum sq) of the values as
  // stored (bf16-rounded for bf16 outputs), or nullptr
  float* stats_out;
};

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;
constexpr int kABytes = kBlockM * kBlockK * 2;  // 16 KiB

// Exact-form GELU 0.5 x (1 + erf(x / sqrt 2)) with erf from Abramowitz-Stegun 7.1.26 (|error| <= 1.5e-7 plus the
// ~1e-7 relative error of the approximate rcp / ex2 units: far below the bf16 output rounding).  2 MUFU + 11 FP32 ops;
// erff() costs ~30 instructions and made the GEGLU epilogue instruction-bound (38 instr / output element).
__device__ __forceinline__ float gelu_erf(float x) {
  const float ax = fabsf(x) * 0.70710678118654752440f;
  float t, e;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, ax, 1.0f)));
  float poly = fmaf(t, 1.061405429f, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  poly *= t;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-1.4426950408889634f * ax * ax));
  const float erf_abs = fmaf(-poly, e, 1.0f);
  const float hx = 0.5f * x;
  return fmaf(hx, copysignf(erf_abs, x), hx);
}

// CLIP's quick_gelu x * sigmoid(1.702 x) (transformers activations.py QuickGELUActivation).  For x << 0 the exponential
// overflows to +inf and the result is -0, the limit.
__device__ __forceinline__ float quick_gelu(float x) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-1.702f * 1.4426950408889634f * x));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
  return x * r;
}

// Deterministic split-K finalisation: sum the fp32 partials in split order, then the same linear epilogue (+ ReLU).
template <bool RELU = false>
__global__ void splitk_finalize_kernel(const float* __restrict__ partial, int splits, long long pixels, int n_out,
                                       int hw_out, const float* __restrict__ bias, const float* __restrict__ rowbias,
                                       int rowbias_ld, const __nv_bfloat16* __restrict__ residual, int ldr,
                                       void* __restrict__ out, int ldo, int out_is_f32, float out_scale) {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const long long idx = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 4;
  if (idx >= pixels * n_out) return;
  const long long pix = idx / n_out;
  const int col = static_cast<int>(idx - pix * n_out);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int s = 0; s < splits; ++s) {
    const float4 t = *reinterpret_cast<const float4*>(partial + (static_cast<long long>(s) * pixels + pix) * n_out + col);
    acc.x += t.x, acc.y += t.y, acc.z += t.z, acc.w += t.w;
  }
  float f[4] = {acc.x, acc.y, acc.z, acc.w};
  if (bias)
    for (int j = 0; j < 4; ++j) f[j] += bias[col + j];
  if (rowbias) {
    const long long img = pix / hw_out;
    for (int j = 0; j < 4; ++j) f[j] += rowbias[img * rowbias_ld + col + j];
  }
  for (int j = 0; j < 4; ++j) f[j] *= out_scale;
  if (residual)
    for (int j = 0; j < 4; ++j) f[j] += __bfloat162float(residual[pix * ldr + col + j]);
  if constexpr (RELU)
    for (int j = 0; j < 4; ++j) f[j] = fmaxf(f[j], 0.f);
  if (out_is_f32) {
    *reinterpret_cast<float4*>(static_cast<float*>(out) + pix * ldo + col) = make_float4(f[0], f[1], f[2], f[3]);
  } else {
    uint2 o = make_uint2(pack_bf16(f[0], f[1]), pack_bf16(f[2], f[3]));
    *reinterpret_cast<uint2*>(static_cast<__nv_bfloat16*>(out) + pix * ldo + col) = o;
  }
}

}  // namespace mdb
