// C-ABI launcher for the wgmma GEMM / implicit-GEMM convolution (include/magicdrive_b200.h: mdb_gemm_conv).
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <mutex>

#include "../../include/magicdrive_b200.h"
#define MDB_NEED_TENSORMAP
#include "common_host.h"
#include "gemm_wgmma.cuh"

using namespace mdb;

namespace {

// A operand of a convolution: 4-D (C, W, H, N) im2col map, innermost first; pixel stride = ld elements.  The bounding box
// of filter-tap-(0, 0) positions runs from -pad to (extent - 1 + pad + pad_end - (taps - 1)) in each spatial dimension,
// walked with the stride: exactly h_out x w_out positions per image.
// operand element type of a descriptor (mdb_gemm_desc.operand_dtype: 0 bf16, 1 f16)
CUtensorMapDataType operand_type(const mdb_gemm_desc* d) {
  return d->operand_dtype == 1 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
}

bool make_im2col_map(CUtensorMap* m, const void* ptr, int c, int ld, const mdb_gemm_desc* d) {
  EncodeIm2colFn enc = get_encode_im2col();
  if (!enc) return false;
  const int n = d->n_img, h = d->h_in, w = d->w_in;
  cuuint64_t dims[4] = {(cuuint64_t)c, (cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)n};
  cuuint64_t strides[3] = {(cuuint64_t)ld * 2, (cuuint64_t)w * ld * 2, (cuuint64_t)h * w * ld * 2};
  int lower[2] = {-d->pad_w, -d->pad_h};
  int upper[2] = {d->pad_w + d->pad_w_end - (d->taps_w - 1), d->pad_h + d->pad_h_end - (d->taps_h - 1)};
  cuuint32_t estr[4] = {1u, (cuuint32_t)d->stride, (cuuint32_t)d->stride, 1u};
  CUresult r = enc(m, operand_type(d), 4, const_cast<void*>(ptr), dims, strides, lower, upper, 64u,
                   (cuuint32_t)kBlockM, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS;
}

// A operand of a 1x1 / stride-1 launch: 2-D [pixels, C] map, row stride ld elements.
bool make_rows_map(CUtensorMap* m, const void* ptr, int c, int ld, long long pixels, CUtensorMapDataType dt) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return false;
  cuuint64_t dims[2] = {(cuuint64_t)c, (cuuint64_t)pixels};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  cuuint32_t box[2] = {64u, (cuuint32_t)kBlockM};
  cuuint32_t estr[2] = {1u, 1u};
  CUresult r = enc(m, dt, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS;
}

bool make_act_map(CUtensorMap* m, const void* ptr, int c, int ld, const mdb_gemm_desc* d, bool im2col) {
  return im2col ? make_im2col_map(m, ptr, c, ld, d)
                : make_rows_map(m, ptr, c, ld, (long long)d->n_img * d->h_out * d->w_out, operand_type(d));
}

bool make_w_map(CUtensorMap* m, const void* ptr, int n_out, int k, int block_n, CUtensorMapDataType dt) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return false;
  cuuint64_t dims[2] = {(cuuint64_t)k, (cuuint64_t)n_out};
  cuuint64_t strides[1] = {(cuuint64_t)k * 2};
  cuuint32_t box[2] = {64u, (cuuint32_t)block_n};
  cuuint32_t estr[2] = {1u, 1u};
  CUresult r = enc(m, dt, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS;
}

struct Plan {
  int m_tiles;  // ceil(pixels / 128): tiles of consecutive output pixels
  int ctas, m_groups;  // CTAs per cluster (1, or 2 = CTA pairs) and M-tile groups walked by one cluster
  int block_n, n_tiles, splits, kb_per_split, kb_total;
};

int num_sms() {
  static int sms = 0;
  if (!sms) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
  }
  return sms;
}

// 64-wide K blocks per filter tap of a source with c channels: the last one is partial when c % 64 != 0 (the TMA
// zero-fills the channels past c, and the weights hold zeros in the same K columns)
inline int cblocks(int c) { return (c + kBlockK - 1) / kBlockK; }

int validate(const mdb_gemm_desc* d) {
  if (!d || !d->a0 || !d->w || !d->out) return set_error(MDB_ERR_INVALID, "mdb_gemm_conv: null pointer");
  if (d->c0 <= 0 || d->c0 % 8 || d->c1 < 0 || d->c1 % 8)
    return set_error(MDB_ERR_UNSUPPORTED, "mdb_gemm_conv: channel counts must be multiples of 8 (c0=%d c1=%d)", d->c0,
                     d->c1);
  if (d->c1 > 0 && !d->a1) return set_error(MDB_ERR_INVALID, "mdb_gemm_conv: c1>0 but a1 is null");
  if (d->lda0 % 8 || (d->c1 > 0 && d->lda1 % 8) || d->ldo % 8 || (d->residual && d->ldr % 8))
    return set_error(MDB_ERR_UNSUPPORTED, "mdb_gemm_conv: leading dimensions must be multiples of 8");
  if (d->n_out % 8) return set_error(MDB_ERR_UNSUPPORTED, "mdb_gemm_conv: n_out must be a multiple of 8");
  if (d->stride != 1 && d->stride != 2) return set_error(MDB_ERR_UNSUPPORTED, "mdb_gemm_conv: stride must be 1 or 2");
  if (d->kernel_variant != 0 && (d->kernel_variant < 2 || d->kernel_variant > 4))
    return set_error(MDB_ERR_INVALID, "mdb_gemm_conv: kernel_variant must be 0, 2, 3 or 4");
  if (d->n_img <= 0 || d->h_out <= 0 || d->w_out <= 0 || d->taps_h <= 0 || d->taps_w <= 0)
    return set_error(MDB_ERR_INVALID, "mdb_gemm_conv: bad shape");
  if ((reinterpret_cast<uintptr_t>(d->a0) | reinterpret_cast<uintptr_t>(d->a1) | reinterpret_cast<uintptr_t>(d->w) |
       reinterpret_cast<uintptr_t>(d->out) | reinterpret_cast<uintptr_t>(d->residual)) & 15)
    return set_error(MDB_ERR_INVALID, "mdb_gemm_conv: pointers must be 16-byte aligned");
  if (d->epi_mode == 1 && (d->n_out % 256 || d->residual || d->rowbias || d->out_is_f32 || d->stats_out))
    return set_error(MDB_ERR_UNSUPPORTED, "mdb_gemm_conv: GEGLU epilogue needs n_out %% 256 == 0 and a plain bf16 output "
                                          "(no residual, per-image shift or row statistics)");
  if (d->epi_mode == 2 && (d->residual || d->rowbias || d->out_is_f32 || d->stats_out))
    return set_error(MDB_ERR_UNSUPPORTED, "mdb_gemm_conv: quick-GELU epilogue needs a plain bf16 output "
                                          "(no residual, per-image shift or row statistics)");
  if (d->epi_mode == 3 && (d->residual || d->rowbias || d->out_is_f32 || d->stats_out))
    return set_error(MDB_ERR_UNSUPPORTED, "mdb_gemm_conv: ReLU epilogue needs a plain bf16 output "
                                          "(no residual, per-image shift or row statistics)");
  if (d->epi_mode < 0 || d->epi_mode > 3)
    return set_error(MDB_ERR_INVALID, "mdb_gemm_conv: epi_mode must be 0, 1, 2 or 3");
  if (d->operand_dtype != 0 && d->operand_dtype != 1)
    return set_error(MDB_ERR_INVALID, "mdb_gemm_conv: operand_dtype must be 0 (bf16) or 1 (f16)");
  if (d->operand_dtype == 1 && (d->epi_mode == 2 || d->epi_mode == 3 || d->kernel_variant == 3))
    return set_error(MDB_ERR_UNSUPPORTED, "mdb_gemm_conv: f16 operands take the linear and GEGLU epilogues on single CTAs "
                                          "(no quick-GELU, ReLU or CTA pairs)");
  if (d->pad_h_end < 0 || d->pad_w_end < 0)
    return set_error(MDB_ERR_INVALID, "mdb_gemm_conv: end padding must not be negative (pad_h_end=%d pad_w_end=%d)",
                     d->pad_h_end, d->pad_w_end);
  // im2col bounding-box corners of a 4-D map are signed 8-bit and the per-tap offsets unsigned 8-bit
  const int corners[4] = {-d->pad_w, -d->pad_h, d->pad_w + d->pad_w_end - (d->taps_w - 1),
                          d->pad_h + d->pad_h_end - (d->taps_h - 1)};
  for (int i = 0; i < 4; ++i)
    if (corners[i] < -128 || corners[i] > 127 || d->taps_h > 256 || d->taps_w > 256)
      return set_error(MDB_ERR_UNSUPPORTED,
                       "mdb_gemm_conv: filter %dx%d with padding %dx%d (end %dx%d) exceeds the TMA im2col limits",
                       d->taps_h, d->taps_w, d->pad_h, d->pad_w, d->pad_h_end, d->pad_w_end);
  return MDB_OK;
}

// Tile width / split-K plan for `ctas` CTAs per cluster.
void plan_for(const mdb_gemm_desc* d, int ctas, bool allow_split, Plan* pl) {
  const int m_tiles = (int)(((long long)d->n_img * d->h_out * d->w_out + kBlockM - 1) / kBlockM);
  pl->m_tiles = m_tiles;
  pl->ctas = ctas;
  pl->m_groups = (m_tiles + ctas - 1) / ctas;
  pl->kb_total = d->taps_h * d->taps_w * (cblocks(d->c0) + cblocks(d->c1));
  const int sms = num_sms();
  const int clusters = sms / ctas;
  int bn_choice = 0;
  if (d->epi_mode == 1) {
    bn_choice = 256;
  } else if (d->force_block_n) {
    bn_choice = d->force_block_n;
  } else {
    const int cands[4] = {256, 160, 128, 64};
    double best = 1e30;
    for (int i = 0; i < 4; ++i) {
      const int bn = cands[i];
      if (bn == 64 && d->n_out >= 128) continue;  // 64-wide tiles re-read A too often
      const int nt = (d->n_out + bn - 1) / bn;
      const long long groups = (long long)pl->m_groups * nt;
      const long long waves = (groups + clusters - 1) / clusters;
      // cost ~ waves * (MMA time ~ bn, floored by the A-side cost) ; prefer big tiles on ties
      const double cost = (double)waves * (bn < 96 ? 96 : bn) * 1.0 + (double)waves * 6.0;
      if (cost < best - 1e-9) best = cost, bn_choice = bn;
    }
  }
  pl->block_n = bn_choice;
  pl->n_tiles = (d->n_out + bn_choice - 1) / bn_choice;
  // split-K when the grid cannot fill the machine and K is deep
  int splits = 1;
  const long long ctas_total = (long long)m_tiles * pl->n_tiles;
  if (!allow_split) {
    splits = 1;
  } else if (d->force_splits > 0) {
    splits = d->force_splits;
  } else if ((d->epi_mode == 0 || d->epi_mode == 3) && !d->ln_stats && !d->stats_out && d->workspace && ctas_total * 2 <= sms && pl->kb_total >= 16) {
    splits = (int)(sms / ctas_total);
    if (splits > pl->kb_total / 8) splits = pl->kb_total / 8;
    if (splits > 16) splits = 16;
    if (splits < 1) splits = 1;
  }
  if (splits > pl->kb_total) splits = pl->kb_total;
  if (splits > 1) {
    const size_t need = (size_t)splits * d->n_img * d->h_out * d->w_out * d->n_out * sizeof(float);
    const bool linear = d->epi_mode == 0 || d->epi_mode == 3;  // the finalize pass applies the linear epilogue (+ ReLU)
    if (!d->workspace || d->workspace_bytes < need || !linear || d->ln_stats || d->stats_out) splits = 1;
  }
  pl->kb_per_split = (pl->kb_total + splits - 1) / splits;
  pl->splits = (pl->kb_total + pl->kb_per_split - 1) / pl->kb_per_split;  // no empty split
}

// kernel_variant: 0 / 2 = single CTAs (split-K allowed), 3 = CTA pairs, 4 = single CTAs without split-K.  Single CTAs are the
// default because they measured faster on H100: the whole denoising step takes 18.4 ms with them and 25.6 ms with CTA pairs
// (bench.py, H100 SXM).
void make_plan(const mdb_gemm_desc* d, Plan* pl) {
  if (d->kernel_variant == 3) return plan_for(d, 2, false, pl);
  plan_for(d, 1, d->kernel_variant != 4, pl);
}

template <int BN, int CTAS, bool RELU, bool F16>
int launch(const CUtensorMap& tA0, const CUtensorMap& tA1, const CUtensorMap& tB, const GemmParams& gp, cudaStream_t st) {
  using Cfg = WgGemmCfg<BN, CTAS>;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(gemm_wgmma_kernel<BN, CTAS, RELU, F16>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         Cfg::kSmemBytes);
    if (e != cudaSuccess) return set_error(MDB_ERR_CUDA, "cudaFuncSetAttribute: %s", cudaGetErrorString(e));
    attr_set = true;
  }
  const long long total = (long long)gp.m_groups * gp.n_tiles * gp.splits;  // tiles per cluster walk
  const int clusters_max = num_sms() / CTAS;
  const int clusters = (int)(total < clusters_max ? total : clusters_max);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(clusters * CTAS);
  cfg.blockDim = dim3(Cfg::kThreads);
  cfg.dynamicSmemBytes = Cfg::kSmemBytes;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = CTAS;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  add_pdl_attr(cfg, attr, 1);
  cudaError_t e = cudaLaunchKernelEx(&cfg, gemm_wgmma_kernel<BN, CTAS, RELU, F16>, tA0, tA1, tB, gp);
  if (e == cudaSuccess) e = cudaGetLastError();
  if (e != cudaSuccess) return set_error(MDB_ERR_CUDA, "gemm_wgmma_kernel<%d,%d> launch: %s", BN, CTAS, cudaGetErrorString(e));
  return MDB_OK;
}

template <int CTAS, bool RELU = false, bool F16 = false>
int launch_bn(int block_n, const CUtensorMap& tA0, const CUtensorMap& tA1, const CUtensorMap& tB, const GemmParams& gp,
              cudaStream_t st) {
  if constexpr (!F16) {  // f16 launches never take the ReLU epilogue (validate)
    if (!RELU && gp.epi_mode == EPI_RELU) return launch_bn<CTAS, true>(block_n, tA0, tA1, tB, gp, st);
  }
  switch (block_n) {
    case 256: return launch<256, CTAS, RELU, F16>(tA0, tA1, tB, gp, st);
    case 160: return launch<160, CTAS, RELU, F16>(tA0, tA1, tB, gp, st);
    case 128: return launch<128, CTAS, RELU, F16>(tA0, tA1, tB, gp, st);
    case 64: return launch<64, CTAS, RELU, F16>(tA0, tA1, tB, gp, st);
    default: return set_error(MDB_ERR_UNSUPPORTED, "mdb_gemm_conv: unsupported block_n %d", block_n);
  }
}

}  // namespace

extern "C" int mdb_gemm_conv_launches(const mdb_gemm_desc* d) {
  if (validate(d) != MDB_OK) return MDB_ERR_INVALID;
  Plan pl;
  make_plan(d, &pl);
  return pl.splits > 1 ? 2 : 1;
}

extern "C" int mdb_gemm_conv_stats_parts(const mdb_gemm_desc* d) {
  if (validate(d) != MDB_OK) return MDB_ERR_INVALID;
  Plan pl;
  make_plan(d, &pl);
  return pl.n_tiles;  // one (sum, sum sq) slot per row and N tile
}

extern "C" int mdb_gemm_conv_plan(const mdb_gemm_desc* d, int* plan) {
  if (validate(d) != MDB_OK) return MDB_ERR_INVALID;
  Plan pl;
  make_plan(d, &pl);
  const long long walk = (long long)pl.m_groups * pl.n_tiles * pl.splits;
  const int clusters = num_sms() / pl.ctas;
  plan[0] = pl.block_n;
  plan[1] = pl.m_tiles;
  plan[2] = pl.n_tiles;
  plan[3] = pl.splits;
  plan[4] = (int)((walk + clusters - 1) / clusters);
  return MDB_OK;
}

extern "C" int mdb_gemm_conv(const mdb_gemm_desc* d, void* stream) {
  int rc = validate(d);
  if (rc != MDB_OK) return rc;
  if (d->ln_stats && (d->taps_h != 1 || d->taps_w != 1 || !d->ln_colsum || d->ln_parts <= 0))
    return set_error(MDB_ERR_INVALID, "mdb_gemm_conv: a folded LayerNorm needs a 1x1 GEMM, ln_colsum and ln_parts");
  Plan pl;
  make_plan(d, &pl);
  if (d->epi_mode == 1 && pl.block_n != 256) return set_error(MDB_ERR_UNSUPPORTED, "GEGLU needs block_n 256");
  cudaStream_t st = static_cast<cudaStream_t>(stream);

  // output pixel p reads input pixel p unless the filter, stride, padding or output size say otherwise
  const bool im2col = d->taps_h != 1 || d->taps_w != 1 || d->stride != 1 || d->pad_h || d->pad_w || d->pad_h_end ||
                      d->pad_w_end || d->h_in != d->h_out || d->w_in != d->w_out;
  CUtensorMap tA0, tA1, tB;
  if (!make_act_map(&tA0, d->a0, d->c0, d->lda0, d, im2col))
    return set_error(MDB_ERR_CUDA, "cuTensorMapEncode%s(A0) failed (c=%d ld=%d n=%d h=%d w=%d taps=%dx%d pad=%dx%d s=%d)",
                     im2col ? "Im2col" : "Tiled", d->c0, d->lda0, d->n_img, d->h_in, d->w_in, d->taps_h, d->taps_w,
                     d->pad_h, d->pad_w, d->stride);
  if (d->c1 > 0) {
    if (!make_act_map(&tA1, d->a1, d->c1, d->lda1, d, im2col))
      return set_error(MDB_ERR_CUDA, "cuTensorMapEncode%s(A1) failed", im2col ? "Im2col" : "Tiled");
  } else {
    tA1 = tA0;
  }
  const int ktot = d->taps_h * d->taps_w * kBlockK * (cblocks(d->c0) + cblocks(d->c1));
  if (!make_w_map(&tB, d->w, d->n_out, ktot, pl.block_n / pl.ctas, operand_type(d)))
    return set_error(MDB_ERR_CUDA, "cuTensorMapEncodeTiled(W) failed (n=%d k=%d)", d->n_out, ktot);

  GemmParams gp;
  memset(&gp, 0, sizeof(gp));
  gp.n_img = d->n_img, gp.h_out = d->h_out, gp.w_out = d->w_out, gp.n_out = d->n_out;
  gp.taps_h = d->taps_h, gp.taps_w = d->taps_w, gp.stride = d->stride, gp.pad_h = d->pad_h, gp.pad_w = d->pad_w;
  gp.cblocks0 = cblocks(d->c0), gp.cblocks1 = cblocks(d->c1);
  gp.im2col = im2col;
  gp.m_tiles = pl.m_tiles, gp.n_tiles = pl.n_tiles, gp.splits = pl.splits;
  gp.m_groups = pl.m_groups;
  gp.kb_per_split = pl.kb_per_split;
  gp.epi_mode = pl.splits > 1      ? EPI_PARTIAL_F32
                : d->epi_mode == 2 ? EPI_QUICK_GELU
                : d->epi_mode == 3 ? EPI_RELU
                                   : d->epi_mode;
  gp.out_is_f32 = d->out_is_f32;
  gp.bias = d->bias, gp.rowbias = d->rowbias, gp.rowbias_ld = d->rowbias_ld;
  gp.residual = d->residual, gp.ldr = d->ldr;
  gp.out = d->out, gp.ldo = d->ldo, gp.out_scale = d->out_scale;
  gp.partial = static_cast<float*>(d->workspace);
  gp.ln_stats = d->ln_stats, gp.ln_parts = d->ln_parts, gp.ln_eps = d->ln_eps, gp.ln_colsum = d->ln_colsum;
  gp.ln_inv_c = 1.0f / (float)(d->c0 + d->c1);
  gp.stats_out = d->stats_out;

  const bool f16 = d->operand_dtype == 1;
  rc = pl.ctas == 2 ? launch_bn<2>(pl.block_n, tA0, tA1, tB, gp, st)
       : f16        ? launch_bn<1, false, true>(pl.block_n, tA0, tA1, tB, gp, st)
                    : launch_bn<1>(pl.block_n, tA0, tA1, tB, gp, st);
  if (rc != MDB_OK) return rc;
  if (pl.splits > 1) {
    const long long pixels = (long long)d->n_img * d->h_out * d->w_out;
    const long long total4 = pixels * d->n_out / 4;
    const int threads = 256;
    const int blocks = (int)((total4 + threads - 1) / threads);
    cudaError_t e =
        f16 ? launch_pdl(splitk_finalize_kernel<false, true>, dim3(blocks), dim3(threads), 0, st,
                         static_cast<const float*>(d->workspace), pl.splits, pixels, d->n_out, d->h_out * d->w_out, d->bias,
                         d->rowbias, d->rowbias_ld, static_cast<const __half*>(d->residual), d->ldr, d->out, d->ldo,
                         d->out_is_f32, d->out_scale)
            : launch_pdl(d->epi_mode == 3 ? splitk_finalize_kernel<true> : splitk_finalize_kernel<false>, dim3(blocks),
                         dim3(threads), 0, st, static_cast<const float*>(d->workspace), pl.splits, pixels, d->n_out,
                         d->h_out * d->w_out, d->bias, d->rowbias, d->rowbias_ld,
                         static_cast<const __nv_bfloat16*>(d->residual), d->ldr, d->out, d->ldo, d->out_is_f32,
                         d->out_scale);
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) return set_error(MDB_ERR_CUDA, "splitk_finalize launch: %s", cudaGetErrorString(e));
  }
  return MDB_OK;
}
