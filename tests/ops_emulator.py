"""TEST INFRASTRUCTURE ONLY — a torch restatement of every operator in magicdrive_b200/ops.py that launches a kernel, following
the semantics the C header documents (include/magicdrive_b200.h), so that the HOST side of the product (weight packing in
engine._Weights / params.py, layer sequencing in engine.py, the module wrappers, the denoiser, the text encoder, the VAE
encoder, the FID Inception) can be executed and checked against the oracle in the build container, which has no GPU.  It is
never imported by the package; `install(monkeypatch)` swaps it in for the duration of one test.  What it cannot check is
the CUDA code itself: that is tests/test_*_gpu.py.

Every function takes exactly the arguments of its ops.py counterpart (tests/test_ops_emulator_cpu.py holds them equal), and
rejects the argument combinations the library rejects.  The pure-Python wrappers of ops.py (`linear`, `workspace_slot`, the
route of `attention` to `attention_multi`) are not restated: the real ones run over these operators.

Arithmetic is fp32 from the (bf16-rounded) packed weights; activations are NOT rounded to bf16 (`ROUND_ACTIVATIONS`
switches that on), so a host-logic mistake shows up at 1e-5, not inside bf16 noise.  `compute(torch.float64)` switches the
arithmetic to float64 (tests/launch_census.py takes its GEMM references from gemm_conv that way, on the operands' device)."""
import contextlib
import math

import torch
import torch.nn.functional as F

from magicdrive_b200 import ops

ROUND_ACTIVATIONS = False
COMPUTE = torch.float32  # the type every restatement computes in


@contextlib.contextmanager
def compute(dtype):
    """Run the enclosed restatements in `dtype` arithmetic (float64: a reference for the kernels)."""
    global COMPUTE
    old, COMPUTE = COMPUTE, dtype
    try:
        yield
    finally:
        COMPUTE = old


def _f(x):
    return x.to(COMPUTE)


def _act(x):
    """Output of a device operator: a fresh contiguous buffer (optionally with the device's bf16 rounding)."""
    return _f(x.to(torch.bfloat16) if ROUND_ACTIVATIONS else x).contiguous()


def _write(out, res, ld=None):
    """The operator's result, or `res` written into the first columns of `out` (row stride `ld`) and `out` returned."""
    if out is None:
        return res
    assert out.dim() == 2 and out.stride(0) == (out.stride(0) if ld is None else ld), (out.shape, out.stride(), ld)
    out[:, :res.shape[1]] = res
    return out


def _k64_filter(w, n_out, kh, kw, c0, c1):
    """The [n_out, c0 + c1, kh, kw] filter held in the header's K64 layout W[n, tap*K64 + c] (each source's channels
    rounded up to 64, source 1 from column 64*ceil(c0/64)); the gaps must hold zeros."""
    p0, p1 = -(-c0 // 64) * 64, -(-c1 // 64) * 64
    assert w.shape == (n_out, kh * kw * (p0 + p1)), (tuple(w.shape), n_out, kh, kw, c0, c1)
    wt = w.to(COMPUTE).reshape(n_out, kh, kw, p0 + p1)
    assert not wt[..., c0:p0].any() and not wt[..., p0 + c1:].any(), "the K64 gaps must hold zeros"
    return torch.cat([wt[..., :c0], wt[..., p0:p0 + c1]], -1).permute(0, 3, 1, 2)


def gemm_conv(a0, w, *, n_img, h_in, w_in, c0, lda0, n_out, taps=1, stride=1, pad=0, h_out=None, w_out=None, a1=None,
              c1=0, lda1=0, bias=None, rowbias=None, residual=None, ldr=0, out=None, ldo=None, out_f32=False,
              out_scale=1.0, geglu=False, force_block_n=0, force_splits=0, allow_split_k=True, kernel_variant=0,
              ln=None, ln_colsum=None, ln_eps=1e-5, emit_stats=False, quick_gelu=False, relu=False, taps_h=None,
              taps_w=None, pad_h=None, pad_w=None, pad_h_end=0, pad_w_end=0):
    """mdb_gemm_conv.  force_block_n, force_splits, allow_split_k and kernel_variant choose the tiling, not the result."""
    kh, kw = (taps if taps_h is None else taps_h), (taps if taps_w is None else taps_w)
    ph, pw = (pad if pad_h is None else pad_h), (pad if pad_w is None else pad_w)
    # the descriptors the library rejects
    assert c0 > 0 and c0 % 8 == 0 and c1 >= 0 and c1 % 8 == 0 and n_out % 8 == 0, (c0, c1, n_out)
    assert lda0 % 8 == 0 and (c1 == 0 or (a1 is not None and lda1 % 8 == 0)), (lda0, c1, lda1)
    assert residual is None or ldr % 8 == 0, ldr
    assert stride in (1, 2) and kernel_variant in (0, 2, 3, 4), (stride, kernel_variant)
    assert pad_h_end >= 0 and pad_w_end >= 0, "negative end padding is rejected"
    for p, p_end, t in ((ph, pad_h_end, kh), (pw, pad_w_end, kw)):
        assert t > 0 and -128 <= -p and p + p_end - (t - 1) <= 127, "beyond the TMA im2col limits"
    assert geglu + quick_gelu + relu <= 1, "one activation epilogue per launch"
    if geglu or quick_gelu or relu:
        assert residual is None and rowbias is None and not out_f32 and not emit_stats, \
            "GEGLU / quick-GELU / ReLU epilogues write a plain bf16 output"
    assert not geglu or n_out % 256 == 0, n_out
    assert ln is None or (kh == kw == 1 and ln_colsum is not None and ln.parts > 0), "a folded LayerNorm needs a 1x1 GEMM"

    if h_out is None:
        h_out = (h_in + 2 * ph + pad_h_end - kh) // stride + 1
    if w_out is None:
        w_out = (w_in + 2 * pw + pad_w_end - kw) // stride + 1
    pix_in = n_img * h_in * w_in
    assert a0.shape[0] == pix_in and a0.stride(0) == lda0, (a0.shape, a0.stride(), lda0)
    x = a0[:, :c0].to(COMPUTE)
    if c1:
        assert a1.shape[0] == pix_in and a1.stride(0) == lda1, (a1.shape, a1.stride(), lda1)
        x = torch.cat([x, a1[:, :c1].to(COMPUTE)], 1)
    cin = c0 + c1
    x = x.reshape(n_img, h_in, w_in, cin).permute(0, 3, 1, 2)
    if pad_h_end or pad_w_end:
        x = F.pad(x, (0, pad_w_end, 0, pad_h_end))
    acc = F.conv2d(x, _k64_filter(w, n_out, kh, kw, c0, c1), stride=stride, padding=(ph, pw))
    assert acc.shape[2:] == (h_out, w_out), (acc.shape, h_out, w_out)
    acc = acc.permute(0, 2, 3, 1).reshape(n_img * h_out * w_out, n_out)
    if ln is not None:  # folded LayerNorm: rstd * (acc - mean * colsum) with the producer's row statistics
        assert ln.data.shape[0] == acc.shape[0]
        tot = ln.data.to(COMPUTE).sum(1)
        mean = tot[:, 0:1] / cin
        var = (tot[:, 1:2] / cin - mean * mean).clamp_min(0)
        acc = torch.rsqrt(var + ln_eps) * (acc - mean * ln_colsum.to(COMPUTE)[None, :])
    if bias is not None:
        acc = acc + bias.to(COMPUTE)
    if rowbias is not None:
        rb = rowbias.to(COMPUTE)
        rb = rb.expand(n_img, -1) if rb.shape[0] == 1 else rb
        assert rb.shape[0] == n_img, (rowbias.shape, n_img)
        acc = acc + rb[:, :n_out].repeat_interleave(h_out * w_out, 0)
    acc = acc * out_scale
    if geglu:  # 256-column tiles of [128 value | 128 gate]
        t = acc.reshape(acc.shape[0], n_out // 256, 2, 128)
        res = (t[:, :, 0] * F.gelu(t[:, :, 1])).reshape(acc.shape[0], n_out // 2)
    elif quick_gelu:
        res = acc * torch.sigmoid(1.702 * acc)
    elif relu:
        res = F.relu(acc)
    else:
        res = acc
    if residual is not None:
        r2 = residual.reshape(-1, residual.shape[-1])  # the device reads it as [pixels, ldr] through a raw pointer
        assert r2.shape[0] == res.shape[0] and r2.stride(0) == ldr, (residual.shape, ldr)
        res = res + r2[:, :res.shape[1]].to(COMPUTE)
    res = res.contiguous() if out_f32 else _act(res)
    assert out is None or (out.stride(0) if ldo is None else ldo) % 8 == 0, ldo
    res_out = _write(out, res, ldo)
    if not emit_stats:
        return res_out
    # two partial slots per row, like a launch of the device kernel with two N tiles; the device accumulates the values it
    # stores (already bf16-rounded when ROUND_ACTIVATIONS)
    half = res.shape[1] // 2
    parts = torch.stack([torch.stack([res[:, :half].sum(1), (res[:, :half] ** 2).sum(1)], -1),
                         torch.stack([res[:, half:].sum(1), (res[:, half:] ** 2).sum(1)], -1)], 1)
    return res_out, ops.RowStats(parts.contiguous(), 2)


def conv_direct(x, wgt, bias, *, n, h, w, cin, cout, k, stride=(1, 1), pad=(1, 1), silu=False, residual=None,
                out_f32=False):
    assert wgt.shape == (k, k, cin, cout)
    y = F.conv2d(x.to(COMPUTE).reshape(n, h, w, cin).permute(0, 3, 1, 2), wgt.to(COMPUTE).permute(3, 2, 0, 1), bias.to(COMPUTE),
                 stride=stride, padding=pad)
    if silu:
        y = F.silu(y)
    y = y.permute(0, 2, 3, 1)
    if residual is not None:
        y = y + residual.to(COMPUTE).reshape(y.shape)
    return (y if out_f32 else _act(y)).contiguous()


def groupnorm(x0, c0, ld0, n_img, hw, gamma, beta, eps, silu, x1=None, c1=0, ld1=0, groups=32):
    assert x0.stride(0) == ld0
    x = x0[:, :c0].to(COMPUTE)
    if c1:
        assert x1.stride(0) == ld1
        x = torch.cat([x, x1[:, :c1].to(COMPUTE)], 1)
    c = c0 + c1
    y = F.group_norm(x.reshape(n_img, hw, c).permute(0, 2, 1), groups, gamma.to(COMPUTE), beta.to(COMPUTE), eps)
    if silu:
        y = F.silu(y)
    return _act(y.permute(0, 2, 1).reshape(n_img * hw, c))


def layernorm(x, gamma, beta, eps=1e-5):
    return _act(F.layer_norm(x.to(COMPUTE), (x.shape[1],), gamma.to(COMPUTE), beta.to(COMPUTE), eps))


def softmax_rows(s, cols, cols_out):
    p = torch.softmax(s[:, :cols].to(COMPUTE), -1)
    return _act(F.pad(p, (0, cols_out - cols)))


def _heads(t, ld, batches, length, heads, d):
    """[batches * length, >= heads * d] rows with stride ld -> [batches, heads, length, d]."""
    assert t.stride(0) == ld, (t.stride(), ld)
    return t[:, :heads * d].to(COMPUTE).reshape(batches, length, heads, d).transpose(1, 2)


def attention_multi(q, sources, *, b, heads, lq, lk, d, ldq, scale, kv_index, n_sets=1, out=None, kv_len=None):
    """mdb_attention_multi / mdb_attention_varlen: kv_index entries are (source << 24) | batch, -1 an empty slot that adds
    nothing (a row without a present set is zero); kv_len[b] (clamped to [0, lk]) cuts query batch b's keys, and a batch
    with 0 keys adds nothing either.  Each set's output is rounded to bf16 before the sum, in slot order."""
    assert 1 <= len(sources) <= 3 and 1 <= n_sets <= 8, (len(sources), n_sets)
    qh = _heads(q, ldq, b, lq, heads, d)
    ks, vs, first = [], [], [0]
    for s_ in sources:
        k, v, ldk, b_kv = s_[:4]
        ks.append(_heads(k, ldk, b_kv, lk, heads, d))
        vs.append(_heads(v, s_[4] if len(s_) > 4 else ldk, b_kv, lk, heads, d))
        first.append(first[-1] + b_kv)
    kh, vh = torch.cat(ks), torch.cat(vs)
    idx = kv_index.reshape(b, n_sets).long().cpu()
    src, batch = idx >> 24, idx & 0xFFFFFF
    assert bool(((idx < 0) | (src < len(sources))).all())
    flat = torch.tensor(first)[src.clamp(0, len(sources) - 1)] + batch
    n_keys = torch.full((b,), lk) if kv_len is None else kv_len.long().cpu().clamp(0, lk)
    key_mask = torch.where(torch.arange(lk)[None] < n_keys[:, None], 0.0, -math.inf)[:, None, None, :]
    res = torch.zeros(b, heads, lq, d)
    for s in range(n_sets):
        present = ((idx[:, s] >= 0) & (n_keys > 0))[:, None, None, None]
        sel = torch.where(idx[:, s] >= 0, flat[:, s], 0)
        o = torch.softmax(qh @ kh[sel].transpose(-1, -2) * scale + key_mask, -1) @ vh[sel]
        res = res + torch.where(present, _act(o), 0.0)
    return _write(out, _act(res.transpose(1, 2).reshape(b * lq, heads * d)))


def attention(q, k, v, *, b, heads, lq, lk, d, ldq, ldk, ldv, scale, kv_index=None, n_sets=1, out=None, b_kv=None,
              kv_len=None):
    """mdb_attention (mdb_attention_varlen with kv_len): attention_multi with one source, whose entries are batch indices."""
    b_kv = b if b_kv is None else b_kv
    if kv_index is None:
        assert n_sets == 1 and b_kv == b
        kv_index = torch.arange(b, dtype=torch.int32)
    return attention_multi(q, [(k, v, ldk, b_kv, ldv)], b=b, heads=heads, lq=lq, lk=lk, d=d, ldq=ldq, scale=scale,
                           kv_index=kv_index, n_sets=n_sets, out=out, kv_len=kv_len)


def attention_causal(q, k, v, *, b, heads, l, d, ldq, ldk, ldv, scale, out=None):
    qh, kh, vh = (_heads(t, ld, b, l, heads, d) for t, ld in ((q, ldq), (k, ldk), (v, ldv)))
    mask = torch.full((l, l), -math.inf).triu(1)
    o = torch.softmax(qh @ kh.transpose(-1, -2) * scale + mask, -1) @ vh
    return _write(out, _act(o.transpose(1, 2).reshape(b * l, heads * d)))


def clip_embed(ids, tok, pos, out=None):
    """bf16(tok[id] + pos[p]) per token (NaN rows for ids outside the vocabulary) and the rows' (sum, sum of squares) from
    the stored values, one part."""
    n_seq, ln = ids.shape
    assert ids.dtype in (torch.int32, torch.int64) and pos.shape[0] >= ln
    bad = (ids < 0) | (ids >= tok.shape[0])
    x = tok.to(COMPUTE)[ids.clamp(0, tok.shape[0] - 1).long()] + pos.to(COMPUTE)[:ln][None]
    x = _act(torch.where(bad[..., None], torch.full_like(x, math.nan), x).reshape(n_seq * ln, -1))
    stats = torch.stack([x.sum(1), (x * x).sum(1)], -1)[:, None]
    return _write(out, x), ops.RowStats(stats.contiguous(), 1)


def add(a, b):
    return _act(a.to(COMPUTE) + b.to(COMPUTE))


def nearest_index(n_in, n_out):
    """ATen's nearest source index: min(floor(dst * scale), n_in - 1) with scale = n_in / n_out and the product in float32.
    Not the exact floor(dst * n_in / n_out): at 26 -> 44, output row 22 reads row 12, not 13."""
    scale = torch.tensor(n_in, dtype=torch.float32) / torch.tensor(n_out, dtype=torch.float32)
    return (torch.arange(n_out, dtype=torch.float32) * scale).floor().long().clamp_max(n_in - 1)


def upsample_nearest(x, n, h, w, c, ho, wo):
    xi = x.to(COMPUTE).reshape(n, h, w, c)
    return xi[:, nearest_index(h, ho)][:, :, nearest_index(w, wo)].reshape(n * ho * wo, c).contiguous()


def adaptive_avgpool(x, n, h, w, c, ho, wo, silu=False):
    y = F.adaptive_avg_pool2d(x.to(COMPUTE).reshape(n, h, w, c).permute(0, 3, 1, 2), (ho, wo))
    y = F.silu(y) if silu else y
    return y.permute(0, 2, 3, 1).contiguous()


def pool2d(x, *, n, h, w, c, mode, k=3, stride=1, pad=0, ldx=None, out=None, ldo=None):
    assert x.stride(0) == (c if ldx is None else ldx)
    xi = x[:, :c].to(COMPUTE).reshape(n, h, w, c).permute(0, 3, 1, 2)
    if mode == ops.POOL_GLOBAL_AVG:  # fp32 output
        return _write(out, xi.mean((2, 3)), ldo)
    assert mode in (ops.POOL_MAX, ops.POOL_AVG), mode
    y = F.max_pool2d(xi, k, stride, pad) if mode == ops.POOL_MAX else F.avg_pool2d(xi, k, stride, pad,
                                                                                  count_include_pad=False)
    return _write(out, _act(y.permute(0, 2, 3, 1).reshape(-1, c)), ldo)


def fid_input(x, *, nhwc, quantize, normalize, size=None):
    x = (x.permute(0, 3, 1, 2) if nhwc else x).to(COMPUTE)
    assert x.shape[1] == 3
    if quantize:
        x = torch.round(x * 255).clamp(0, 255) / 255
    if size is not None and tuple(size) != tuple(x.shape[2:]):
        x = F.interpolate(x, size=size, mode="bilinear", align_corners=False)
    if normalize:
        x = 2 * x - 1
    return _act(F.pad(x.permute(0, 2, 3, 1), (0, 5)).reshape(-1, 8))


def linear_small(x, w, bias=None, pre_silu=False, post_silu=False):
    h = F.silu(x.to(COMPUTE)) if pre_silu else x.to(COMPUTE)
    y = h @ w.to(COMPUTE).t()
    if bias is not None:
        y = y + bias.to(COMPUTE)
    return F.silu(y) if post_silu else y


def timestep_embedding(t, dim, flip_sin_to_cos=True, freq_shift=0.0):
    half = dim // 2
    freqs = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float32) / (half - freq_shift))
    arg = t.to(COMPUTE)[:, None] * freqs[None]
    emb = torch.cat([torch.sin(arg), torch.cos(arg)], -1)
    return torch.cat([emb[:, half:], emb[:, :half]], -1) if flip_sin_to_cos else emb


def fourier_embed(x, num_freqs):
    outs = [x.to(COMPUTE)]
    for k in range(num_freqs):
        outs += [torch.sin(x.to(COMPUTE) * 2.0 ** k), torch.cos(x.to(COMPUTE) * 2.0 ** k)]
    return torch.cat(outs, -1)


def nchw_to_nhwc(x):
    n, c, h, w = x.shape
    return _act(x.to(COMPUTE).permute(0, 2, 3, 1).reshape(n * h * w, c))


def nhwc_to_nchw(x, n, c, h, w, dtype=torch.float32):
    return x.to(COMPUTE).reshape(n, h, w, -1)[..., :c].permute(0, 3, 1, 2).contiguous().to(dtype)


def f32_to_bf16(x):
    return _act(x)


def pack_latents(x, cpad=64, repeat=1):
    return _act(F.pad(x.to(COMPUTE), (0, cpad - x.shape[1]))).repeat(repeat, 1)


def _cfg_combine(eps, cfg, guidance, c, npix):
    e = eps[:, :c].to(COMPUTE)
    return e[:npix] + guidance * (e[npix:] - e[:npix]) if cfg else e


def cfg_ddim_step(eps, latents, coef, cfg, guidance, c=4):
    latents.copy_(coef[0] * latents + coef[1] * _cfg_combine(eps, cfg, guidance, c, latents.shape[0]))
    return latents


def cfg_unipc_step(eps, latents, last_sample, m0, m1, coef, cfg, guidance, c=4):
    e, x = _cfg_combine(eps, cfg, guidance, c, latents.shape[0]), latents.clone()
    x0 = coef[0] * x + coef[1] * e
    xc = coef[2] * last_sample + coef[3] * m0 + coef[4] * m1 + coef[5] * x0 if coef[9] != 0 else x
    latents.copy_(coef[6] * xc + coef[7] * x0 + coef[8] * m0)
    last_sample.copy_(xc)
    m1.copy_(m0)
    m0.copy_(x0)
    return latents


def pin_views(dst, a, b, coef, view_mask, rows_per_view, c=4):
    assert dst.shape[0] == view_mask.numel() * rows_per_view
    sel = view_mask.bool().repeat_interleave(rows_per_view)
    dst[sel, :c] = (coef[0] * a[sel] if a is not None else 0) + coef[1] * b[sel]
    return dst


EMULATED = ["gemm_conv", "conv_direct", "groupnorm", "layernorm", "softmax_rows", "attention", "attention_multi",
            "attention_causal", "clip_embed", "add", "upsample_nearest", "adaptive_avgpool", "pool2d", "fid_input",
            "linear_small", "timestep_embedding", "fourier_embed", "nchw_to_nhwc", "nhwc_to_nchw", "f32_to_bf16",
            "cfg_ddim_step", "cfg_unipc_step", "pin_views", "pack_latents"]


def install(monkeypatch):
    """Swap every operator of magicdrive_b200.ops for its torch restatement and let the modules build their engines on the
    CPU.  The fold precision (engine._Weights.fold_dtype) is each test's own choice."""
    from magicdrive_b200 import engine, models
    for name in EMULATED:
        assert hasattr(ops, name), name
        monkeypatch.setattr(ops, name, globals()[name])
    monkeypatch.setattr(models._B200Module, "_get_engine",
                        lambda self, cls_: self.__dict__.setdefault("_eng", cls_(self.arch_cfg, dict(self.state_dict()), self.device)))
    real = models.AutoencoderKL.encoder_engine

    def encoder_engine(self):  # the same checks, with the engine built on the CPU
        if self._encoder_missing or self._enc_engine is not None:
            return real(self)
        self._enc_engine = engine.VaeEncoderEngine(self.arch_cfg, dict(self.state_dict()), self.device)
        return self._enc_engine

    monkeypatch.setattr(models.AutoencoderKL, "encoder_engine", encoder_engine)
