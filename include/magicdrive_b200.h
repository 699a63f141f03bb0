/*
 * magicdrive_b200 — C ABI of the multi-view denoising hot path (CUDA kernels for sm_90a, NVIDIA H100).
 *
 * Every entry point takes raw device pointers, sizes, strides and a cudaStream_t (as void*), returns 0 on
 * success or a negative status, and never allocates, synchronises or takes ownership.  mdb_last_error()
 * returns a thread-local message for the last failure.  Activations are bf16, channel-innermost (NHWC for
 * feature maps == [tokens, channels] for transformer blocks); accumulation is fp32.  Models with fp16 parameters run
 * the denoising step in f16: mdb_gemm_desc.operand_dtype and the *_f16 entry points below, each the f16 twin of the bf16
 * entry point it follows, with the same signature and checks.
 *
 * The reference has no native boundary of its own for this path except one op: xformers'
 * efficient_attention_forward_cutlass (third_party/xformers/xformers/csrc/attention/attention.cpp:27,
 * attention_forward_generic.cu:330-334).  Everything else it runs is a torch.nn call; each function below
 * names the reference call site (file:line in the MagicDrive source tree) it replaces.
 */
#ifndef MAGICDRIVE_B200_H
#define MAGICDRIVE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MDB_OK 0
#define MDB_ERR_INVALID (-1)
#define MDB_ERR_CUDA (-2)
#define MDB_ERR_UNSUPPORTED (-3)

const char* mdb_last_error(void);

/* Programmatic dependent launch for the launches that follow (process-wide flag, returns the previous value): the next
 * kernel's launch latency and prologue overlap the tail of its stream predecessor.  Switch it on only around
 * single-stream regions (the UNet up path); the environment variable MDB_PDL=0|1 overrides the flag. */
int mdb_set_pdl(int on);
int mdb_version(void);
/* 1 if a CUDA device of compute capability 9.0 (sm_90a) is usable, else 0 (never raises). */
int mdb_device_ok(void);

/* ------------------------------------------------------------------------------------------------
 * mdb_gemm_conv: tensor-core (wgmma) GEMM / implicit-GEMM convolution with fused epilogue.
 *   out[pix, n] = scale * ( sum_{r,s,c} A[pix*stride + (r,s) - pad, c] * W[n, (r*taps_w+s)*C + c]
 *                           + bias[n] + rowbias[img(pix), n] ) + residual[pix, n]
 *   epi_mode 1 (GEGLU): W/bias are packed per 256-column tile as [128 value | 128 gate] and
 *   out[pix, j] = value_j * gelu(gate_j) with n_out/2 output columns.
 * Channel counts c0, c1 are multiples of 8.  The K loop runs over 64-channel blocks per filter tap; when c % 64 != 0 the
 * last block of each tap is partial (channels past c read as zeros), so W is packed per tap at the width rounded up to 64:
 *   W[n, tap*K64 + c] with K64 = 64*ceil(c0/64) + 64*ceil(c1/64), source 1 starting at column 64*ceil(c0/64), zeros in
 *   the gaps.  For channel counts that are multiples of 64 this is the plain (tap, channel) layout.
 * Filters are taps_h x taps_w with padding pad_h / pad_w (1x7, 7x1, 5x5, ...); the TMA im2col limits apply:
 * -128 <= -pad and pad + pad_end - (taps - 1) <= 127 per dimension, else MDB_ERR_UNSUPPORTED.
 * pad_h_end / pad_w_end add zero rows below and zero columns right of the image on top of pad_h / pad_w (0 = symmetric
 * padding), so h_out = (h_in + pad_h + pad_h_end - taps_h) / stride + 1: Downsample2D(padding=0) of the VAE encoder,
 * F.pad(x, (0, 1, 0, 1)) then a 3x3 stride-2 conv (diffusers/models/resnet.py:199,215-217), is pad 0 with end pad 1.
 * Negative end pads are MDB_ERR_INVALID.
 * Replaces: nn.Conv2d 3x3/1x1 in ResnetBlock2D (diffusers/models/resnet.py:537,560,586), Downsample2D
 * (resnet.py:199), Upsample2D.conv (resnet.py:129), Transformer2DModel.proj_in/proj_out
 * (transformer_2d.py:149,205), Attention.to_q/to_k/to_v/to_out (attention_processor.py:141-156),
 * GEGLU.proj + FeedForward out (attention.py:270,226), connector (magicdrive/networks/blocks.py:83),
 * ControlNet zero convs (magicdrive/networks/unet_addon_rawbox.py:221-272).
 * A may be split over two sources along channels (torch.cat skip connections, unet_2d_blocks.py:1984,2086).
 * ------------------------------------------------------------------------------------------------ */
typedef struct {
  const void* a0;      /* bf16 [n_img, h_in, w_in, lda0] using the first c0 channels */
  const void* a1;      /* optional second source (NULL if c1 == 0) */
  int c0, lda0, c1, lda1;
  int n_img, h_in, w_in;
  const void* w;       /* bf16 [n_out, taps_h*taps_w*K64] (K64 = c0+c1 rounded up per source to 64, see above) */
  int n_out;
  int taps_h, taps_w, stride, pad_h, pad_w;
  int h_out, w_out;
  const float* bias;    /* [n_out] or NULL */
  const float* rowbias; /* [n_img, rowbias_ld] or NULL */
  int rowbias_ld;
  const void* residual; /* bf16 [pixels, ldr] or NULL */
  int ldr;
  void* out;            /* bf16 (or fp32 if out_is_f32) [pixels, ldo] */
  int ldo;
  int out_is_f32;
  float out_scale;
  int epi_mode;         /* 0 linear, 1 GEGLU, 2 quick-GELU: out = y * sigmoid(1.702 y) on y = the linear epilogue's value
                         * (CLIP MLP fc1, transformers models/clip/modeling_clip.py CLIPMLP); never split-K, no residual,
                         * rowbias, stats_out or fp32 output; 3 ReLU: out = max(0, v) on v = the linear epilogue's value
                         * (bias, out_scale), for a BatchNorm folded into W / bias followed by ReLU (torchvision Inception3
                         * BasicConv2d); plain bf16 output only (no residual, rowbias, stats_out or fp32 output); split-K
                         * applies it in the finalize pass.  ReLU launches run their own kernel instantiations. */
  void* workspace;      /* split-K scratch (may be NULL => no split-K) */
  size_t workspace_bytes;
  int force_block_n;    /* 0 = auto; test hook */
  int force_splits;     /* 0 = auto; test hook */
  int kernel_variant;   /* 0 = auto (single CTAs, split-K where the planner wants it); 2 = the same; 3 = CTA pairs: 2-CTA
                         * clusters on consecutive M tiles, each CTA TMA-loads half of the weight tile and multicasts it to
                         * both (no split-K); 4 = single CTAs without split-K; test / A-B hook */
  /* LayerNorm folded into the GEMM (attention.py:85,104,120; blocks.py:67-71): A is the RAW tensor x, W was
   * pre-multiplied by gamma (W' = W * gamma), bias holds c_n = sum_k beta_k W[n,k] + b_n, and the epilogue applies
   *   out = rstd_row * (acc - mean_row * ln_colsum[n]) + c_n
   * with mean/rstd from the per-row partial sums the PRODUCER of x wrote (stats_out of that call). */
  const float* ln_stats;   /* fp32 [pixels, ln_parts, 2] partial (sum, sum of squares) of the rows of A, or NULL */
  int ln_parts;
  float ln_eps;
  const float* ln_colsum;  /* fp32 [n_out]: sum_k W'[n, k] */
  /* Producer side: fp32 [pixels, mdb_gemm_conv_stats_parts(d), 2] receiving partial (sum, sum of squares) of every output
   * row (after bias / residual) over the columns of one N tile per slot, taken from the stored values (bf16-rounded for
   * bf16 outputs), or NULL. */
  float* stats_out;
  int pad_h_end, pad_w_end;  /* extra zero rows below / columns right of the image (see above); 0 = symmetric padding */
  /* Element type of a0, a1, w, residual and a non-fp32 out: 0 = bf16 (every field above says bf16), 1 = f16 (models with
   * fp16 parameters).  f16 launches take the linear and GEGLU epilogues, split-K included, on single CTAs; quick-GELU,
   * ReLU and kernel_variant 3 are MDB_ERR_UNSUPPORTED.  Row statistics are then taken from the f16-rounded values. */
  int operand_dtype;
} mdb_gemm_desc;

int mdb_gemm_conv(const mdb_gemm_desc* d, void* stream);
/* Number of kernels mdb_gemm_conv would launch for this descriptor (1, or 2 with split-K). */
int mdb_gemm_conv_launches(const mdb_gemm_desc* d);
/* Partial-sum slots per output row that mdb_gemm_conv writes to stats_out for this descriptor (depends on the tiling the
 * planner picks); negative status if the descriptor cannot emit row statistics. */
int mdb_gemm_conv_stats_parts(const mdb_gemm_desc* d);
/* The planner's tiling for this descriptor, for profiling tools: plan[0..4] = block_n, M tiles, N tiles, K splits,
 * waves of the persistent grid. */
int mdb_gemm_conv_plan(const mdb_gemm_desc* d, int* plan);

/* ------------------------------------------------------------------------------------------------
 * FID Inception helpers (magicdrive/misc/inception.py InceptionV3 with fid_inception_v3(), inception.py:129-163, 197-341).
 * mdb_pool2d over NHWC bf16 [n, h, w, ldx] using the first c channels (c, ldx, ldo multiples of 8, 16-byte aligned
 * pointers), writing into the first c columns of out [n*ho*wo, ldo] -- a column slice of a wider buffer, so the Inception
 * blocks' torch.cat is never materialised:
 *   mode 0: max over the k x k window at stride, padding ignored (F.max_pool2d / nn.MaxPool2d, inception.py:89,98,337);
 *   mode 1: average over the window's in-image pixels (F.avg_pool2d count_include_pad=False, inception.py:241,269,302);
 *   mode 2: global average of each image into fp32 out [n, ldo] (nn.AdaptiveAvgPool2d(1), inception.py:122);
 *           k, stride, pad, ho, wo are ignored.
 * mdb_fid_input: a [0, 1] image batch, fp32 or bf16, NCHW [n, 3, h, w] or (x_is_nhwc) NHWC [n, h, w, 3] -> bf16 NHWC
 * [n, ho, wo, 8] with channels 3..7 zero (the K-padded A operand of Conv2d_1a_3x3 on mdb_gemm_conv, c0 = 8):
 *   quantize: x = rint(255 x) / 255 clamped to [0, 1], the 8-bit levels a saved PNG holds (diffusers pil_utils.py:41);
 *   bilinear resize to ho x wo with F.interpolate(align_corners=False) semantics, no antialias (inception.py:146-150)
 *   (ho == h and wo == w is the identity); normalize: 2x - 1 (inception.py:152-153).
 * ------------------------------------------------------------------------------------------------ */
int mdb_pool2d(const void* x, int ldx, int n, int h, int w, int c, int mode, int k, int stride, int pad, void* out,
               int ldo, int ho, int wo, void* stream);
int mdb_fid_input(const void* x, int x_is_f32, int x_is_nhwc, int n, int h, int w, int quantize, int normalize, void* out,
                  int ho, int wo, void* stream);
/* The same with f16 in place of bf16: x fp32 or f16, out f16.  The conv_in operand of an fp16 VAE's encoder
 * (AutoencoderKL.encode); without quantize, resize or normalize each value is x rounded to f16 once. */
int mdb_fid_input_f16(const void* x, int x_is_f32, int x_is_nhwc, int n, int h, int w, int quantize, int normalize,
                      void* out, int ho, int wo, void* stream);

/* ------------------------------------------------------------------------------------------------
 * FID evaluation protocol (perception/data_prepare/val_set_gen.py:29-43, 103-116; tools/fid_score.py:361-368, 474-482):
 * the 8-bit steps between the pipeline's views and Inception, equal byte for byte to Pillow's.
 * mdb_resample_u8: Pillow's bicubic resample (Image.resize(..., BICUBIC), a = -0.5, support widened by the scale when
 *   downsampling) of n images h x w -> rh x rw, RGB.  x: uint8 NHWC, or (x_is_f32) fp32 [0, 1] NHWC / NCHW rounded to
 *   uint8 first as (x * 255).round() (diffusers numpy_to_pil).  coef_w / coef_h: int32 [rw, taps_w + 2] / [rh, taps_h + 2],
 *   row i = [first input index, tap count, 22-bit fixed-point weights...]; a pass is run exactly when its size changes and
 *   its coefficients must then be given (NULL otherwise).  The horizontal pass runs first and is rounded and clipped to
 *   uint8 (tmp: uint8 [n, h, crop_w, 3], needed when the width changes).  Of the resized image, the window rows
 *   [crop_top, crop_top + crop_h) x columns [crop_left, crop_left + crop_w) is written at (top, left) of out, uint8 NHWC
 *   [n, out_h, out_w, 3]; every other out pixel is 0 (a zero pad).
 * mdb_jpeg_roundtrip_u8: uint8 NHWC RGB [n, h, w, 3] -> the image a baseline JPEG at `quality` (1..100, the standard
 *   tables scaled as IJG libjpeg does) with 4:2:0 chroma decodes to, as Pillow saves and loads it by default (quality 75):
 *   integer DCTs, triangle chroma upsampling.  The entropy coder is lossless and is skipped.  planes: 8-byte aligned
 *   scratch of n * hp * wp * 3 / 2 bytes (hp, wp: h, w rounded up to 16).  out may be x.
 * ------------------------------------------------------------------------------------------------ */
int mdb_resample_u8(const void* x, int x_is_f32, int x_is_nhwc, int n, int h, int w, const int* coef_w, int taps_w,
                    int rw, const int* coef_h, int taps_h, int rh, int crop_top, int crop_left, int crop_h, int crop_w,
                    void* tmp, void* out, int out_h, int out_w, int top, int left, void* stream);
int mdb_jpeg_roundtrip_u8(const void* x, int n, int h, int w, int quality, void* planes, void* out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * JPEG files of generated views (perception/data_prepare/val_set_gen.py:29-43, copy_save_image's PIL save).
 * mdb_jpeg_encode_u8: uint8 NHWC RGB [n, h, w, 3] (n in 1..65535, h and w in 1..65535) -> the files
 *   PIL.Image.fromarray(x[i]).save(f, "JPEG", quality=quality) writes, byte for byte: baseline, 4:2:0, the standard
 *   quantisation tables scaled as in mdb_jpeg_roundtrip_u8 and the standard Huffman tables, no restart interval.  Each
 *   file is the MDB_JPEG_HEADER_BYTES-byte header, the entropy-coded data and EOI.  The files are written back to back in
 *   `out` (out_bytes bytes).  meta: 8-byte aligned device int64 [n, 3], per image (entropy-coded bytes before stuffing,
 *   file length, offset of the file in out); the length is -1 when the scratch was too small to count it, the offset -1
 *   when the files were not written (scratch or out too small: nothing is written to out then, and meta says what is
 *   needed).  scratch: 256-byte aligned, scratch_bytes >= mdb_jpeg_scratch_bytes(n, h, w, chunks) for `chunks` 4 KiB
 *   chunks of entropy-coded data, each image taking ceil(entropy-coded bytes / 4096) of them (at least n are required).
 *   Arguments are checked before any launch; the lengths are known only on the device, so the caller reads meta.
 * mdb_jpeg_scratch_bytes: that scratch size, or -1 for bad arguments.
 * ------------------------------------------------------------------------------------------------ */
#define MDB_JPEG_HEADER_BYTES 623
long long mdb_jpeg_scratch_bytes(int n, int h, int w, long long chunks);
int mdb_jpeg_encode_u8(const void* x, int n, int h, int w, int quality, void* scratch, long long scratch_bytes, void* out,
                       long long out_bytes, long long* meta, void* stream);

/* Direct (CUDA-core) convolution for tiny channel counts: conv_in 4->320 (unet_2d_condition.py:231),
 * conv_out 320->4 (:503), BEV map encoder (magicdrive/networks/map_embedder.py:66-76).
 * x: [n, h, w, cin] bf16 or fp32; w: fp32 [kh, kw, cin, cout] (output channel innermost: coalesced across a warp);
 * out bf16/fp32 [n, ho, wo, cout] (+= residual). */
int mdb_conv_direct(const void* x, int x_is_f32, int n, int h, int w, int cin, const float* wgt, const float* bias,
                    int cout, int kh, int kw, int stride_h, int stride_w, int pad_h, int pad_w, int ho, int wo,
                    int silu, const void* residual, void* out, int out_is_f32, void* stream);
/* The same with f16 in place of bf16: x f16 or fp32, out (and residual) f16 or fp32.  The decoder conv_in of an fp16 VAE
 * (fp32 latents in, the f16 feature map out); the weights stay fp32. */
int mdb_conv_direct_f16(const void* x, int x_is_f32, int n, int h, int w, int cin, const float* wgt, const float* bias,
                        int cout, int kh, int kw, int stride_h, int stride_w, int pad_h, int pad_w, int ho, int wo,
                        int silu, const void* residual, void* out, int out_is_f32, void* stream);

/* GroupNorm (+SiLU) over NHWC, optionally over the channel-concat of two sources; writes one normalised tensor.
 * Replaces nn.GroupNorm + SiLU (resnet.py:535,556,598,630; transformer_2d.py:145; unet_2d_condition.py:492).
 * stats_ws: fp32 [max(n_img, 160) * groups * 2] scratch (per-image or per-CTA-run group partials). */
int mdb_groupnorm(const void* x0, int c0, int ld0, const void* x1, int c1, int ld1, int n_img, int hw, int groups,
                  float eps, const float* gamma, const float* beta, int silu, void* out, int ldo, float* stats_ws,
                  void* stream);
/* The same over f16 sources and output (fp32 statistics). */
int mdb_groupnorm_f16(const void* x0, int c0, int ld0, const void* x1, int c1, int ld1, int n_img, int hw, int groups,
                      float eps, const float* gamma, const float* beta, int silu, void* out, int ldo, float* stats_ws,
                      void* stream);

/* LayerNorm over the last dim of [rows, C] bf16 (attention.py:85,104,120; blocks.py:67-71). */
int mdb_layernorm(const void* x, long long rows, int c, int ldx, const float* gamma, const float* beta, float eps,
                  void* out, int ldo, void* stream);

/* Row softmax of fp32 scores into bf16 probabilities: out[r, j] = softmax_j(s[r, :cols]) for j < cols and 0 for
 * cols <= j < cols_out (K padding of the following P.V GEMM).  Used by the VAE decoder's single-head 512-wide attention
 * (unet_2d_blocks.py:433-446; attention_processor.py:1252), whose QK^T and PV products run on mdb_gemm_conv. */
int mdb_softmax_rows(const float* s, int lds, long long rows, int cols, void* out, int ldo, int cols_out, void* stream);
/* The same with f16 probabilities (the mid-block attention of an fp16 VAE). */
int mdb_softmax_rows_f16(const float* s, int lds, long long rows, int cols, void* out, int ldo, int cols_out,
                         void* stream);

/* Fused multi-head attention forward, softmax(Q K^T * scale) V, bf16 in/out, fp32 softmax.
 * q: [b, Lq, heads*d] with row stride ldq; k, v: [b_kv, Lk, heads*d] with row strides ldk, ldv; out like q (ldo).
 * kv_index: device int32 [b * n_sets] of K/V batch indices (< b_kv) or NULL (then n_sets == 1, b_kv == b and batch i attends
 * to K/V batch i).  b_kv > b is the view-sharded case: K/V of all views were all-gathered, queries are local.
 * With n_sets in 1..MDB_ATT_MAX_SETS the kernel computes
 *   out[b] = sum over s with kv_index[b*n_sets + s] >= 0, in order s = 0, 1, ..., of bf16(attn(q[b], kv[kv_index[b*n_sets + s]]))
 * (each set's output rounded to bf16 before it is added; a row with no entry >= 0 is written as zeros).  An entry -1 is an
 * empty slot: nothing is loaded for it, so [a, -1, b] gives bitwise the result of [a, b].  This is the cross-view "add" mode
 * (magicdrive/networks/blocks.py:112-121, 213-217) for any camera rig, without duplicating tokens per (view, neighbour)
 * pair.  Replaces xformers efficient_attention_forward_cutlass / F.scaled_dot_product_attention
 * (attention_processor.py:1165-1171, 1252). */
#define MDB_ATT_MAX_SETS 8
int mdb_attention(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv, void* out, int ldo, int b,
                  int b_kv, int heads, int lq, int lk, int d, const int* kv_index, int n_sets, float scale, void* stream);

/* The same with the K/V batches spread over n_src (1..3) buffers: k[i] / v[i] are [b_kv[i], Lk, heads*d] with row strides
 * ldk[i] / ldv[i]; kv_index entries are (source << 24) | batch index inside that source.  This is how the view-sharded mode
 * consumes its ring neighbours' K/V without gathering them: source 1 / 2 are the neighbour GPUs' K/V buffers, mapped through
 * NVLink peer memory (the TMA loads go over NVLink tile by tile, overlapping the local QK^T / PV work). */
int mdb_attention_multi(const void* q, int ldq, int n_src, const void* const* k, const int* ldk, const void* const* v,
                        const int* ldv, const int* b_kv, void* out, int ldo, int b, int heads, int lq, int lk, int d,
                        const int* kv_index, int n_sets, float scale, void* stream);

/* mdb_attention_multi with a per-query-batch key count: kv_len is a device int32 [b] array or NULL (= lk for every batch).
 * Keys at or beyond kv_len[b] take no weight and key tiles past it are not loaded.  The kernel clamps each entry to [0, lk]
 * (a batch with 0 keys contributes nothing, like an empty slot).  This is the cross-view "concat" mode
 * (blocks.py:122-133) when views have different neighbour counts: their neighbours' tokens are gathered into
 * [b, lk, heads*d] with kv_len[b] = neighbours * tokens.
 * With one set and lk <= 256 it is also the conditioning cross-attention of a denoiser whose K/V buffers are sized for a box
 * capacity (lk = 1 + 77 + capacity, kv_len[b] = 1 + 77 + boxes of the scene, changed between replays of a captured graph):
 * such a launch may walk several query tiles per CTA with up to a ring of key tiles (4 x 128 keys for d <= 64, 4 x 64 for
 * d = 80, 3 x 64 for d = 160) kept in shared memory, or stream them where kv_len[b] needs more.  For every kv_len[b] the
 * output is bitwise that of the launch with lk = kv_len[b].  Rows at or past kv_len[b] that share the last walked key tile
 * with counted keys are loaded and weighted 0: they must hold finite values. */
int mdb_attention_varlen(const void* q, int ldq, int n_src, const void* const* k, const int* ldk, const void* const* v,
                         const int* ldv, const int* b_kv, void* out, int ldo, int b, int heads, int lq, int lk, int d,
                         const int* kv_index, int n_sets, const int* kv_len, float scale, void* stream);
/* The same with f16 q, k, v and output (kv_len may be NULL): P is packed to f16 for the P V product and each set's output
 * is rounded to f16 before the sum.  One key-tile width (the default of MDB_ATTN_KERNEL); the same head dims. */
int mdb_attention_varlen_f16(const void* q, int ldq, int n_src, const void* const* k, const int* ldk, const void* const* v,
                             const int* ldv, const int* b_kv, void* out, int ldo, int b, int heads, int lq, int lk, int d,
                             const int* kv_index, int n_sets, const int* kv_len, float scale, void* stream);

/* Causal self-attention of the CLIP text encoder (transformers models/clip/modeling_clip.py CLIPAttention.forward with the
 * causal_attention_mask of CLIPTextTransformer.forward): as mdb_attention with one set, b_kv == b and no kv_index, and key j
 * visible to query i iff j <= i.  Requires lq == lk (MDB_ERR_INVALID otherwise).  Key tiles wholly above a query tile's
 * diagonal are neither loaded nor computed.  Same head dims and MDB_ATTN_KERNEL variants as mdb_attention. */
int mdb_attention_causal(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv, void* out, int ldo, int b,
                         int heads, int lq, int lk, int d, float scale, void* stream);

/* CLIP token + position embedding (modeling_clip.py CLIPTextEmbeddings.forward): for row r = s * len + p of n_seq sequences
 * of len tokens, out[r, :dim] = bf16(tok[ids[r]] + pos[p]) and stats_out[r] = (sum, sum of squares) of that bf16 row: the
 * fp32 [rows, 1, 2] row statistics a GEMM with a folded LayerNorm reads (ln_parts = 1).  ids: device int32, or int64 if
 * ids_are_i64; an id outside [0, vocab) gives a NaN row (and NaN statistics) and is never used as an address.
 * tok_table_bf16 [vocab, dim], pos_table_bf16 [>= len, dim]; dim and ldo multiples of 8. */
int mdb_clip_embed(const void* ids, int ids_are_i64, int n_seq, int len, const void* tok_table_bf16, int vocab,
                   const void* pos_table_bf16, int dim, void* out_bf16, int ldo, float* stats_out, void* stream);

/* out = a + b (bf16), n elements (unet_2d_condition_multiview.py:464-473, 487-488). */
int mdb_add(const void* a, const void* b, void* out, long long n, void* stream);
/* out = a + b (f16), the sum taken in fp32 and rounded once. */
int mdb_add_f16(const void* a, const void* b, void* out, long long n, void* stream);

/* Nearest-neighbour resize NHWC, src index = floor(dst * in / out) (resnet.py:156-159).  A copy of 2-byte elements:
 * bf16 and f16 maps alike. */
int mdb_upsample_nearest(const void* x, int n, int h, int w, int c, void* out, int ho, int wo, void* stream);
/* nn.AdaptiveAvgPool2d((ho, wo)) over an NHWC fp32 map, optionally followed by SiLU: the pooling block of
 * BEVControlNetConditioningEmbeddingPlus (magicdrive/networks/map_embedder.py:118, forward :66-76 applies SiLU after every
 * block, the pool included).  Step-invariant (once per scene). */
int mdb_adaptive_avgpool(const float* x, int n, int h, int w, int c, float* out, int ho, int wo, int silu, void* stream);

/* Skinny linear for tiny M (time embedding MLP, time_emb_proj, camera / box encoders):
 * out[m, n] = act(in)[m, :] . W[n, :] + b[n], W bf16 [n, k] (ldw), in/out fp32.  pre_silu applies SiLU to the input,
 * post_silu to the output (embeddings.py:192-201; resnet.py:615-616; bbox_embedder.py:145-152). */
int mdb_linear_small(const float* in, int m, int k, int ldi, const void* w, int ldw, const float* bias, int n,
                     int pre_silu, int post_silu, float* out, int ldo, void* stream);
/* The same with f16 weights (the time-embedding MLP and camera / box encoders of fp16 models). */
int mdb_linear_small_f16(const float* in, int m, int k, int ldi, const void* w, int ldw, const float* bias, int n,
                         int pre_silu, int post_silu, float* out, int ldo, void* stream);

/* Sinusoidal timestep embedding, flip_sin_to_cos, freq_shift (embeddings.py:24-64).  t: fp32 [m] on device. */
int mdb_timestep_embedding(const float* t, int m, int dim, int flip_sin_to_cos, float freq_shift, float* out,
                           void* stream);

/* NeRF Fourier features [x, sin(2^k x), cos(2^k x)]_{k<num_freqs} on the last dim d of fp32 [rows, d]
 * (magicdrive/networks/embedder.py:15-40). out fp32 [rows, d*(1+2*num_freqs)]. */
int mdb_fourier_embed(const float* x, long long rows, int d, int num_freqs, float* out, void* stream);

/* dtype conversions / layout: NCHW fp32|bf16 <-> NHWC bf16 (pipeline boundary, pipeline_bev_controlnet.py:409-411). */
int mdb_nchw_to_nhwc(const void* x, int x_is_f32, int n, int c, int h, int w, void* out_bf16, void* stream);
int mdb_nhwc_to_nchw(const void* x_bf16, int n, int c, int h, int w, void* out, int out_is_f32, void* stream);
int mdb_f32_to_bf16(const float* x, void* out, long long n, void* stream);
int mdb_bf16_to_f32(const void* x, float* out, long long n, void* stream);
/* fp32 -> f16 (round to nearest even; overflow to inf) and f16 -> fp32 (exact). */
int mdb_f32_to_f16(const float* x, void* out, long long n, void* stream);
int mdb_f16_to_f32(const void* x, float* out, long long n, void* stream);

/* Latents [pix, cin] (fp32 or bf16) -> bf16 [repeat*pix, cpad] with channels >= cin zeroed: the K-padded A operand
 * that lets conv_in (unet_2d_condition.py:231, 4 -> 320 channels) run on the tensor-core path; repeat = 2 duplicates
 * the batch for classifier-free guidance (pipeline_bev_controlnet.py:352-354). */
int mdb_pack_latents(const void* x, int x_is_f32, long long pix, int cin, int cpad, int repeat, void* out, void* stream);
/* The same with an f16 output; x is fp32, or f16 when x_is_f32 == 0. */
int mdb_pack_latents_f16(const void* x, int x_is_f32, long long pix, int cin, int cpad, int repeat, void* out, void* stream);

/* Classifier-free guidance + DDIM (eta = 0) update fused (pipeline_bev_controlnet.py:426-436;
 * scheduling_ddim.py:325-445).  eps: fp32 [(2 if cfg else 1) * n/c pixels, eps_ld] (uncond half first), c channels
 * used per pixel.  coef: device fp32[2] = {sqrt(abar_prev/abar_t), sqrt(1-abar_prev) - sqrt(abar_prev*(1-abar_t)/abar_t)}
 * so x_prev = c0*x + c1*eps.  latents: fp32 [n/c, c] updated in place. */
int mdb_cfg_ddim_step(const float* eps, int eps_ld, int c, int cfg, float guidance, const float* coef, float* latents,
                      long long n, void* stream);

/* Classifier-free guidance + one UniPCMultistepScheduler step fused (the reference's default sampler,
 * magicdrive/misc/test_utils.py:129; scheduling_unipc_multistep.py:518-600 with solver_order 2, bh2, predict_x0,
 * epsilon prediction).  eps as in mdb_cfg_ddim_step.  latents, last_sample, m0, m1: fp32 [n/c, c], all updated in
 * place (sample, sample before the last predictor, newest and previous x0 prediction; zero them before step 0).
 * coef: device fp32[12] for this step = {a0, a1, c0, c1, c2, c3, p0, p1, p2, use_corrector, 0, 0}:
 *   x0 = a0 x + a1 eps;  xc = use_corrector ? c0 last + c1 m0 + c2 m1 + c3 x0 : x;  x' = p0 xc + p1 x0 + p2 m0. */
int mdb_cfg_unipc_step(const float* eps, int eps_ld, int c, int cfg, float guidance, const float* coef, float* latents,
                       float* last_sample, float* m0, float* m1, long long n, void* stream);

/* Given-view generation (magicdrive/pipeline/pipeline_bev_controlnet_given_view.py:263-296, 379-389): for every view v
 * with view_mask[v] != 0, rows [v*rows_per_view, (v+1)*rows_per_view) of dst (fp32, row stride dst_ld, c channels used)
 * become coef[0]*a + coef[1]*b; a, b: fp32 [n_views*rows_per_view, c] contiguous, a may be NULL (term dropped);
 * coef: device fp32[2].  Used to re-noise pinned views (scheduler.add_noise) and to replace their predicted noise. */
int mdb_pin_views(float* dst, int dst_ld, const float* a, const float* b, int c, const float* coef, const int* view_mask,
                  long long rows_per_view, int n_views, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Input preparation (the step before the path; magicdrive/dataset/utils.py:120-352, demo/helper.py:386-466).
 * mdb_prepare_boxes: for every (scene, camera view) keep the boxes that have at least one corner in front of the camera
 * (z > 0 in the frame img_aug @ lidar2camera; the TEST uses the box shifted down by dz/2 exactly like the reference's
 * box_center_shift), compacted in their original order, as 8 corners (mmdet3d order) of the ORIGINAL box.
 *   boxes: fp32 [sum n_s, box_dim] rows (x, y, z, dx, dy, dz, yaw, ...), bottom-centred; labels: int64 [sum n_s];
 *   box_offsets: int32 [n_scenes + 1]; lidar2camera, img_aug (may be NULL): fp32 [n_scenes, n_views, 4, 4];
 *   out_boxes fp32 [n_scenes, n_views, capacity, 8, 3] (0-padded), out_classes int64 [.., capacity] (-1 padded),
 *   out_masks uint8 [.., capacity], out_counts int32 [n_scenes, n_views] (visible boxes, may exceed capacity: overflow is dropped).
 * mdb_camera_param: out fp32 [n, 3, 7] = [K[:3,:3] | (lidar2camera^-1)[:3]] for n = scenes * views rigid transforms
 * (dataset/utils.py:294-297). */
int mdb_prepare_boxes(const float* boxes, int box_dim, const long long* labels, const int* box_offsets, int n_scenes,
                      const float* lidar2camera, const float* img_aug, int n_views, int capacity, float* out_boxes,
                      long long* out_classes, unsigned char* out_masks, int* out_counts, void* stream);
int mdb_camera_param(const float* intrinsics, const float* lidar2camera, int n, float* out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * 3D-box overlays (demo/helper.py:197-307: visualize_camera, show_box_on_views, draw_box_on_imgs with thickness 1):
 * each view with its boxes drawn as OpenCV draws them, byte for byte.
 * mdb_project_boxes: per (scene, view), the boxes whose 8 corners (of the box shifted down by dz/2, mmdet3d order, fp32)
 *   all lie in front of the camera (z > 0 in float64 after `transform`), ordered far to near by their smallest z (a
 *   stable order: exact ties keep box order, which numpy's argsort does not promise beyond 16 boxes).
 *   boxes: fp32 [sum n_s, box_dim >= 7] (x, y, z, dx, dy, dz, yaw, ...), bottom-centred; sincos: fp32 [sum n_s, 2],
 *   sin and cos of each yaw as the caller computes them; labels: int64 [sum n_s]; box_offsets: int32 [n_scenes + 1];
 *   transforms: fp32 [n_scenes, n_views, 4, 4] (img_aug @ lidar2image).  capacity >= every scene's box count, <= 4096.
 *   endpoints: int32 [n_scenes, n_views, capacity, 8, 2], the corners' x / z, y / z (z clipped to [1e-5, 1e5]) truncated
 *   toward zero; colors: int32 [.., capacity], the box's label; counts: int32 [n_scenes, n_views], the boxes drawn;
 *   status: int32 [n_scenes, n_views], 0, 1 when an endpoint falls outside int32 (cv2 refuses it), 2 when the scene has
 *   more boxes than capacity.  Slots past counts are not written.
 * mdb_draw_box_edges_aa: for n_images = n_scenes * n_views views h x w, the 12 edges of each drawn box, in box order and
 *   the fixed edge order, each as cv2.line(img, p0, p1, palette[colors], 1, cv2.LINE_AA) on the RGB image.  images:
 *   uint8 [n_images, h, w, 3], or (images_is_f32) fp32 [0, 1] rounded as (x * 255).round(); out: uint8 [n_images, h, w,
 *   3], may be a uint8 `images`.  transparent_bg: images is ignored, the boxes are drawn on black and out is uint8
 *   [n_images, h, w, 4] with alpha 255 where any channel is non-zero.  palette: uint8 [n_colors, 3].  When any status is
 *   non-zero nothing is written.  h, w <= 32767.
 * ------------------------------------------------------------------------------------------------ */
int mdb_project_boxes(const float* boxes, int box_dim, const float* sincos, const long long* labels, const int* box_offsets,
                      int n_scenes, const float* transforms, int n_views, int capacity, int* endpoints, int* colors,
                      int* counts, int* status, void* stream);
int mdb_draw_box_edges_aa(const void* images, int images_is_f32, int n_images, int h, int w, const int* endpoints,
                          const int* colors, const int* counts, const int* status, int capacity,
                          const unsigned char* palette, int n_colors, int transparent_bg, void* out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Map images and view mosaics (magicdrive/misc/test_utils.py:258-321 run_one_batch; runner/map_visualizer.py:106-211
 * render_static, render_dynamic, visualize_map; runner/img_utils.py:5-40 concat_6_views, img_m11_to_01): the pixels of
 * the reference's `{n}_map.png`, `{n}_ori.png` and view mosaics, byte for byte.
 * mdb_render_bev_map: maps [n_maps, channels, h, w], fp32 or (maps_is_f32 = 0) uint8 / bool, every value 0 or 1; pixel
 *   (y, x) of map m is coloured from maps[m, :, y, x].  Channels [0, n_static) are the static layers, coloured as the
 *   active class with the highest priority[c] (the first such channel on ties); channels [n_static, n_static + n_dynamic)
 *   the dynamic layers, coloured as the first one set.  out: uint8 [n_maps, h, w, 3], dynamic over static over
 *   (200, 200, 200).  colors: uint8 [n_static + n_dynamic, 4], RGB and 1 where the class has a colour; a static class
 *   without a STATIC_PRIORITY rank has priority -1.  info: int64 [n_maps, 4] = {class mask of semantic_used: every active
 *   static class, and with n_dynamic > 0 the dynamic argmax of every pixel (channel n_static where none is set); status,
 *   bit 0 set when a value is neither 0 nor 1; the smallest (pixel << 6 | class), pixel = y * w + x, where an active
 *   static class has priority -1 (the first such channel of the pixel); the smallest (pixel << 6 | class) where the
 *   static class chosen at a pixel (under a dynamic layer or not) has colour flag 0}; an error word is all ones when the
 *   error never arises.  n_static + n_dynamic in 1..64, <= channels; h, w <= 32767.
 * mdb_place_map_u8: resized uint8 [n_maps, s, s, 3] -> per map m, Image.rotate(90) of it (np.rot90) with a legend pasted
 *   to its right or below it.  desc: int64 [n_maps, 5] = {legend address (uint8 [lh, lw, 3]), lh, lw, 1 = right (lh == s:
 *   image s x (s + lw)) or 0 = below (lw == s: image (s + lh) x s), byte offset of the image in out}.  max_pixels: the
 *   largest image's pixel count.
 * mdb_concat_views_u8: views uint8 [n_scenes, n_views, h, w, c], c = 3 or 4 -> out [n_scenes, 2h, max(3, n_views - 3) w,
 *   c], views 0..2 on the first row and 3.. on the second (n_views >= 5), or with oneline [n_scenes, h, n_views w, c]
 *   (n_views >= 2).  Uncovered pixels are black, alpha 255.
 * mdb_m11_to_u8: x fp32 [n, 3, h, w] in [-1, 1] -> out uint8 [n, h, w, 3], ((x * 0.5 + 0.5) * 255) with each operation
 *   rounded to fp32, truncated toward zero.
 * ------------------------------------------------------------------------------------------------ */
int mdb_render_bev_map(const void* maps, int maps_is_f32, int n_maps, int channels, int h, int w, int n_static,
                       int n_dynamic, const int* priority, const unsigned char* colors, unsigned char* out, long long* info,
                       void* stream);
int mdb_place_map_u8(const unsigned char* resized, int n_maps, int s, const long long* desc, long long max_pixels,
                     unsigned char* out, void* stream);
int mdb_concat_views_u8(const unsigned char* views, int n_scenes, int n_views, int h, int w, int c, int oneline,
                        unsigned char* out, void* stream);
int mdb_m11_to_u8(const float* x, int n, int h, int w, unsigned char* out, void* stream);

/* Barrier between the `world` GPUs of a sharding group over NVLink peer memory, as one stream operation (graph-capturable).
 * flag_ptrs_dev: device array of `world` pointers, entry i = GPU i's symmetric uint32[n_channels * world] flag array as mapped
 * into THIS GPU's address space; epoch_dev: this GPU's uint32[n_channels] counter; timed_out_dev: int set to 1 if a peer did
 * not arrive within timeout_cycles SM cycles (0 = wait for ever).  Everything the peers wrote before their call is visible to
 * the kernels launched after this one (the view-sharded cross-view attention reads the neighbours' K/V right after it). */
int mdb_peer_barrier(void* const* flag_ptrs_dev, int rank, int world, int channel, int n_channels, void* epoch_dev,
                     long long timeout_cycles, int* timed_out_dev, void* stream);

#ifdef __cplusplus
}
#endif
#endif
