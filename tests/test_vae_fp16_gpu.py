"""An AutoencoderKL with fp16 parameters decodes and encodes in fp16 on the device.

Kernels, under guard bands against float64 (tests/test_kernel_edges_gpu.py's Guarded): mdb_softmax_rows_f16 and
mdb_conv_direct_f16 within one f16 ulp, mdb_fid_input_f16 bitwise torch's rounding, and each way the VAE calls the f16 GEMM
that the denoising step does not (fp32 output with a scale, the end-padded stride-2 convolution, the c0 = 8 K tail).

Models: test_fp16_model_gpu.py's two criteria on every decode and encode output,
  rel-L2(ours fp16 vs fp32 truth) <= 1.0 x rel-L2(reference arithmetic in fp16 vs fp32 truth) + 1e-4, and
  rel-L2(ours fp16) <= 0.5 x rel-L2(ours bf16) + 1e-5  (the arithmetic really is fp16),
where the truth is the fp32 oracle or the reference-run fixture and "reference arithmetic in fp16" is the oracle run with
fp16 weights and activations through torch's CUDA kernels."""
import math
import os
from dataclasses import asdict

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from magicdrive_b200 import arch, ops, vae_f16_ops
from magicdrive_b200.models import AutoencoderKL, BEVControlNetModel, UNet2DConditionModelMultiview
from magicdrive_b200.pipeline import BEVControlNetDenoiser
from oracle import torch_oracle as O  # checker only
from oracle import vae_encode as OV  # checker only
from oracle.make_golden_vae_encode import full_state_dict, images, vae_config
from tests.common import GOLDEN, golden, record, rel_l2, tiny_configs, tiny_state_dicts, to_dev
from tests.test_kernel_edges_gpu import CONV_DIRECT, Guarded, _close_f16, _close_f32, _gen, _randn
from tests.test_vae_encode_gpu import END_PAD

pytestmark = pytest.mark.gpu
DEV = "cuda"
F16, BF16, F32, F64 = torch.float16, torch.bfloat16, torch.float32, torch.float64


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _within_one_ulp(out, ref, what):
    """Every element within one f16 ulp of the float64 reference (the ulp floored at 2^-24 in the subnormal range)."""
    ref = ref.to(F64)
    err = (out.to(F64) - ref).abs()
    ulp = torch.exp2(torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** -14))) - 10)
    bad = (err > ulp).nonzero()
    assert bad.shape[0] == 0, f"{what}: {bad.shape[0]} elements off, first at {tuple(bad[0].tolist())}, " \
                              f"max err / ulp {(err / ulp).max().item():.3f}"


# ------------------------------------------------------------------------------------------------ softmax_rows f16
# row lengths around every 64-column pad up to the 512 wide K blocks, and the mid-block token counts of the VAE at
# 224x400 (28x50), 272x736 (34x92) and 424x800 (53x100)
SOFTMAX_COLS = [1, 2, 63, 64, 65, 127, 128, 129, 191, 192, 193, 255, 256, 257, 511, 512, 513, 1400, 3128, 5300]
SCORES = ["unit", "spread_1e4", "dominant"]


def _scores(rows, cols, lds, regime, g):
    s = _randn(rows, lds, g=g)
    if regime == "unit":
        return s * 3
    if regime == "spread_1e4":  # scores over +-1e4: most keys underflow to 0, a few rows keep several close keys
        s = (torch.rand(rows, lds, device=DEV, generator=g) * 2 - 1) * 1e4
        s[::3, : cols // 2] = s[::3, :1] + _randn(rows, lds, g=g)[::3, : cols // 2]  # near-ties at the top of some rows
        return s
    s = s * 2  # one dominant key per row, at a row-dependent column
    idx = torch.arange(rows, device=DEV) * 7 % cols
    s[torch.arange(rows, device=DEV), idx] = 40.0
    return s


@pytest.mark.parametrize("regime", SCORES)
@pytest.mark.parametrize("cols", SOFTMAX_COLS)
def test_softmax_rows_f16(cuda_lib, cols, regime):
    rows, cols_out = 37, (cols + 63) // 64 * 64
    lds = cols_out + 8
    s = _scores(rows, cols, lds, regime, _gen(cols))
    out = Guarded(rows, cols_out, F16)
    rc = cuda_lib.mdb_softmax_rows_f16(s.data_ptr(), lds, rows, cols, out.out.data_ptr(), cols_out, cols_out, _stream())
    assert rc == 0, cuda_lib.mdb_last_error()
    out.check(f"softmax {cols} {regime}")
    assert not out.out[:, cols:].any(), "padded key columns must be 0"
    ref = torch.softmax(s[:, :cols].to(F64), -1)
    _within_one_ulp(out.out[:, :cols], ref, f"softmax {cols} {regime}")


def test_softmax_rows_f16_wrapper(cuda_lib):
    s = _randn(5, 200, g=_gen(1))
    p16, pbf = vae_f16_ops.softmax_rows_f16(s, 130, 192), ops.softmax_rows(s, 130, 192)
    assert p16.dtype == F16 and pbf.dtype == BF16 and p16.shape == pbf.shape == (5, 192)
    _within_one_ulp(p16[:, :130], torch.softmax(s[:, :130].to(F64), -1), "wrapper")


# ------------------------------------------------------------------------------------------------ conv_direct f16
CONV_DIRECT_F16 = {
    **CONV_DIRECT,
    "vae_conv_in_224x400": (6, 28, 50, 4, 512, 3, (1, 1), (1, 1), False, True, False, False),
    "vae_conv_in_424x800": (6, 53, 100, 4, 512, 3, (1, 1), (1, 1), False, True, False, False),
    "vae_conv_in_small_odd": (2, 9, 13, 4, 64, 3, (1, 1), (1, 1), False, True, False, False),
}


@pytest.mark.parametrize("case", list(CONV_DIRECT_F16))
def test_conv_direct_f16(cuda_lib, case):
    n, h, w, cin, cout, k, stride, pad, silu, in_f32, out_f32, with_res = CONV_DIRECT_F16[case]
    g = _gen(12)
    x = _randn(n, h, w, cin, g=g)
    if not in_f32:
        x = x.to(F16)
    wt = _randn(k, k, cin, cout, g=g, scale=1 / math.sqrt(k * k * cin))
    b = _randn(cout, g=g)
    ho, wo = (h + 2 * pad[0] - k) // stride[0] + 1, (w + 2 * pad[1] - k) // stride[1] + 1
    odt = F32 if out_f32 else F16
    res = _randn(n * ho * wo, cout, g=g).to(odt) if with_res else None
    out = Guarded(n * ho * wo, cout, odt)
    rc = cuda_lib.mdb_conv_direct_f16(x.data_ptr(), int(in_f32), n, h, w, cin, wt.data_ptr(), b.data_ptr(), cout, k, k,
                                      stride[0], stride[1], pad[0], pad[1], ho, wo, int(silu),
                                      res.data_ptr() if with_res else None, out.out.data_ptr(), int(out_f32), _stream())
    assert rc == 0, cuda_lib.mdb_last_error()
    out.check(case)
    ref = F.conv2d(x.to(F64).permute(0, 3, 1, 2), wt.to(F64).permute(3, 2, 0, 1), b.to(F64), stride=stride, padding=pad)
    ref = (F.silu(ref) if silu else ref).permute(0, 2, 3, 1).reshape(n * ho * wo, cout)
    if with_res:
        ref = ref + res.to(F64)
    (_close_f32 if out_f32 else _close_f16)(out.out, ref, case)


# ------------------------------------------------------------------------------------------------ fid_input f16
@pytest.mark.parametrize("nhwc", [False, True], ids=["nchw", "nhwc"])
@pytest.mark.parametrize("in_dt", [F32, F16], ids=["f32", "f16"])
@pytest.mark.parametrize("n,h,w", [(1, 1, 1), (3, 7, 13), (2, 50, 70), (6, 224, 400), (1, 27, 45)])
def test_fid_input_f16_is_torchs_rounding(cuda_lib, n, h, w, in_dt, nhwc):
    g = _gen(h * w)
    x = (torch.rand(n, h, w, 3, device=DEV, generator=g) * 2 - 1) * torch.exp2(_randn(n, h, w, 3, g=g).round().clamp(-16, 8))
    x = x.to(in_dt)
    xin = x if nhwc else x.permute(0, 3, 1, 2).contiguous()
    out = Guarded(n * h * w, 8, F16)
    rc = cuda_lib.mdb_fid_input_f16(xin.data_ptr(), int(in_dt == F32), int(nhwc), n, h, w, 0, 0, out.out.data_ptr(), h, w,
                                    _stream())
    assert rc == 0, cuda_lib.mdb_last_error()
    out.check("fid_input_f16")
    expect = x.reshape(-1, 3).to(F16)
    assert torch.equal(out.out[:, :3].view(torch.int16), expect.view(torch.int16)), "not bitwise x.to(torch.float16)"
    assert not out.out[:, 3:].view(torch.int16).any()
    a = vae_f16_ops.fid_input_f16(xin, nhwc=nhwc, quantize=False, normalize=False)
    assert torch.equal(a.view(torch.int16), out.out.view(torch.int16))


# ------------------------------------------------------------------------------------------------ the VAE's f16 GEMMs
def _f16(x):
    return x.to(F16)


def _k64(wt):
    """[co, kh, kw, c] -> [co, kh * kw * K64] zero-padded channels (params.pack_conv_weight_k64)."""
    co, kh, kw, c = wt.shape
    k64 = (c + 63) // 64 * 64
    wm = torch.zeros((co, kh, kw, k64), dtype=wt.dtype, device=DEV)
    wm[..., :c] = wt
    return wm.reshape(co, -1)


# name: (rows L, keys padded lp): the mid-block score GEMM S = Q K^T / sqrt(512), fp32 out, at the VAE's token counts
SCORE_CASES = {"224x400": (1400, 1408), "272x736": (3128, 3136), "424x800": (5300, 5312), "odd_130": (130, 192),
               "odd_7": (7, 64)}


@pytest.mark.parametrize("case", list(SCORE_CASES))
def test_f16_gemm_scores_out_f32_with_scale(cuda_lib, case):
    L, lp = SCORE_CASES[case]
    C, g = 512, _gen(L)
    q, k = _f16(_randn(L, C, g=g)), _f16(_randn(lp, C, g=g))
    out = Guarded(L, lp, F32)
    ops.linear(q, k, out_f32=True, out_scale=C ** -0.5, out=out.out, ldo=lp)
    out.check(case)
    _close_f32(out.out, (q.to(F64) @ k.to(F64).t()) * C ** -0.5, case)


# name: (n, h, w, c0, n_out, out_scale, bias + 1): conv_out of the decoder (to_unit_range: 0.5 (acc + b + 1)) and the
# encoder's conv_out.quant_conv fold, fp32 out, 3x3
CONV_OUT_CASES = {
    "dec_224x400": (6, 224, 400, 128, 8, 0.5, True),
    "dec_small_odd_c32": (2, 72, 104, 32, 8, 0.5, True),
    "dec_odd_c64": (3, 26, 27, 64, 8, 1.0, False),
    "enc_28x50": (6, 28, 50, 512, 8, 1.0, False),
    "enc_53x100": (6, 53, 100, 512, 8, 1.0, False),
    "enc_odd": (2, 6, 8, 64, 8, 1.0, False),
}


@pytest.mark.parametrize("case", list(CONV_OUT_CASES))
def test_f16_conv_out_f32_with_scale(cuda_lib, case):
    n, h, w, c0, co, scale, plus1 = CONV_OUT_CASES[case]
    g = _gen(c0 + h)
    a = _f16(_randn(n * h * w, c0, g=g))
    wt = _f16(_randn(co, 3, 3, c0, g=g, scale=1 / math.sqrt(9 * c0)))
    b = _randn(co, g=g) + (1.0 if plus1 else 0.0)
    out = Guarded(n * h * w, co, F32)
    ops.gemm_conv(a, _k64(wt), n_img=n, h_in=h, w_in=w, c0=c0, lda0=c0, n_out=co, taps=3, pad=1, bias=b, out_f32=True,
                  out_scale=scale, out=out.out, ldo=co)
    out.check(case)
    x = a.to(F64).view(n, h, w, c0).permute(0, 3, 1, 2)
    ref = F.conv2d(x, wt.to(F64).permute(0, 3, 1, 2), padding=1).permute(0, 2, 3, 1).reshape(-1, co) + b.to(F64)
    _close_f32(out.out, ref * scale, case)


@pytest.mark.parametrize("case", list(END_PAD))
def test_f16_end_padded_conv(cuda_lib, case):
    """Downsample2D(padding=0) as one stride-2 convolution with end padding, and the c0 = 8 / 32 K tails, in f16."""
    n, h, w, c0, co, ph, pw, eh, ew, stride = END_PAD[case]
    g = _gen(len(case))
    ho, wo = (h + 2 * ph + eh - 3) // stride + 1, (w + 2 * pw + ew - 3) // stride + 1
    a = _f16(_randn(n * h * w, c0, g=g))
    wt = _f16(_randn(co, 3, 3, c0, g=g, scale=1 / math.sqrt(9 * c0)))
    b = _randn(co, g=g)
    out = Guarded(n * ho * wo, co, F16)
    ops.gemm_conv(a, _k64(wt), n_img=n, h_in=h, w_in=w, c0=c0, lda0=c0, n_out=co, taps=3, stride=stride, pad_h=ph, pad_w=pw,
                  pad_h_end=eh, pad_w_end=ew, bias=b, out=out.out, ldo=co)
    out.check(case)
    x = F.pad(a.to(F64).view(n, h, w, c0).permute(0, 3, 1, 2), (pw, pw + ew, ph, ph + eh))
    ref = F.conv2d(x, wt.to(F64).permute(0, 3, 1, 2), stride=stride).permute(0, 2, 3, 1).reshape(-1, co) + b.to(F64)
    _close_f16(out.out, ref, case)


@pytest.mark.parametrize("n,h,w", [(6, 224, 400), (2, 50, 70), (3, 27, 45)])
def test_f16_conv_in_c8_tail(cuda_lib, n, h, w):
    """The encoder's conv_in on the 8-channel RGB operand: one partial K block per tap."""
    g = _gen(h)
    x = images(n, h, w, h).to(DEV)
    a = vae_f16_ops.fid_input_f16(x, nhwc=False, quantize=False, normalize=False)
    wt = torch.zeros((128, 3, 3, 8), dtype=F16, device=DEV)
    wt[..., :3] = _f16(_randn(128, 3, 3, 3, g=g, scale=0.2))
    b = _randn(128, g=g)
    out = Guarded(n * h * w, 128, F16)
    ops.gemm_conv(a, _k64(wt), n_img=n, h_in=h, w_in=w, c0=8, lda0=8, n_out=128, taps=3, pad=1, bias=b, out=out.out, ldo=128)
    out.check("conv_in c8")
    xr = x.to(F16).to(F64)
    ref = F.conv2d(xr, wt[..., :3].to(F64).permute(0, 3, 1, 2), padding=1).permute(0, 2, 3, 1).reshape(-1, 128) + b.to(F64)
    _close_f16(out.out, ref, "conv_in c8")


# ------------------------------------------------------------------------------------------------ argument checks
def _refused(fn):
    before = ops.launch_count()
    with pytest.raises(TypeError):
        fn()
    torch.cuda.synchronize()
    assert ops.launch_count() == before


def test_dtype_mismatches_raise_before_any_launch(cuda_lib):
    s = torch.zeros(4, 64, device=DEV)
    _refused(lambda: vae_f16_ops.softmax_rows_f16(s.half(), 64, 64))
    _refused(lambda: vae_f16_ops.softmax_rows_f16(s.bfloat16(), 64, 64))
    x, wd, b = torch.zeros(1, 5, 6, 4, device=DEV), torch.zeros(3, 3, 4, 16, device=DEV), torch.zeros(16, device=DEV)
    kw = dict(n=1, h=5, w=6, cin=4, cout=16, k=3)
    conv = vae_f16_ops.conv_direct_f16
    _refused(lambda: conv(x.bfloat16(), wd, b, **kw))
    _refused(lambda: conv(x, wd.half(), b, **kw))
    _refused(lambda: conv(x, wd, b.half(), **kw))
    _refused(lambda: conv(x, wd, b, residual=torch.zeros(1, 5, 6, 16, device=DEV, dtype=BF16), **kw))
    _refused(lambda: conv(x, wd, b, out_f32=True, residual=torch.zeros(1, 5, 6, 16, device=DEV, dtype=F16), **kw))
    _refused(lambda: vae_f16_ops.fid_input_f16(torch.zeros(1, 3, 4, 4, device=DEV, dtype=BF16), nhwc=False,
                                               quantize=False, normalize=False))
    a, wm = torch.zeros(64, 64, device=DEV, dtype=F16), torch.zeros(64, 64, device=DEV, dtype=BF16)
    out = Guarded(64, 64, F32)
    _refused(lambda: ops.linear(a, wm, out_f32=True, out=out.out, ldo=64))
    _refused(lambda: ops.linear(a, wm.half(), out_f32=False, out=out.out, ldo=64))
    assert bool((out.buf.view(out.itype) == out.fill).all()), "a refused call wrote to the given output"


# ------------------------------------------------------------------------------------------------ models: decode
def _check(name, ours16, ours_bf, truth, yard):
    for t in (ours16, ours_bf):
        assert torch.isfinite(t.float()).all(), f"{name}: inf or NaN"
    e16, ebf, eref = rel_l2(ours16, truth), rel_l2(ours_bf, truth), rel_l2(yard, truth)
    record(f"[parity vae fp16] {name}: rel-L2 ours fp16 {e16:.3e}  reference-fp16 {eref:.3e}  ours bf16 {ebf:.3e}")
    assert e16 <= eref + 1e-4, (name, e16, eref)
    assert e16 <= 0.5 * ebf + 1e-5, (name, e16, ebf)


def _u8(img):
    """numpy_to_pil's rounding of [0, 1] images: (images * 255).round().astype("uint8")."""
    return (img.float().cpu().numpy() * 255).round().astype(np.uint8)


def _both(cfg, sd):
    vaes = {}
    for dt in (F16, BF16):
        vae = AutoencoderKL(**asdict(cfg))
        vae.load_state_dict(sd)
        vaes[dt] = vae.to(DEV, dt)
    return vaes


SD15 = arch.VaeConfig()
DECODE_CASES = {  # name: (config, n, latent h, latent w)
    "small_odd_5x9": (vae_config(), 3, 5, 9),
    "small_odd_11x7": (vae_config(), 2, 11, 7),
    "sd15_224x400": (SD15, 6, 28, 50),
    "sd15_272x736": (SD15, 1, 34, 92),
    "sd15_424x800": (SD15, 6, 53, 100),
}
U8_SLACK = 2e-3  # fraction of 8-bit values by which ours may exceed the fp16 yardstick's differing fraction


@torch.no_grad()
@pytest.mark.parametrize("case", list(DECODE_CASES))
def test_decode_fp16(cuda_lib, case):
    cfg, n, h, w = DECODE_CASES[case]
    sd = arch.synthetic_state_dict(arch.vae_decoder_param_shapes(cfg), 61)
    vaes = _both(cfg, sd)
    lat = torch.randn(1, n, 4, h, w, generator=torch.Generator().manual_seed(h * w)).to(DEV)
    z = lat[0] / cfg.scaling_factor
    s32 = {k: v.to(DEV) for k, v in sd.items()}
    s16 = {k: v.to(DEV, F16) for k, v in sd.items()}
    truth = O.vae_decode(s32, cfg, z)
    yard = O.vae_decode(s16, cfg, z.half()).float()
    out = {dt: v.decode(z.to(dt)).sample for dt, v in vaes.items()}
    assert vaes[F16].engine().dtype == F16 and out[F16].dtype == F16 and out[F16].shape == truth.shape
    _check(f"decode {case}", out[F16], out[BF16], truth, yard)
    del truth, yard, out
    torch.cuda.empty_cache()
    imgs = {dt: v.decode_latents(lat) for dt, v in vaes.items()}
    truth_i = O.decode_latents(s32, cfg, lat)
    yard_i = O.decode_latents(s16, cfg, lat.half()).float()
    assert imgs[F16].dtype == F32 and imgs[F16].shape == truth_i.shape and 0 <= imgs[F16].min() and imgs[F16].max() <= 1
    _check(f"decode_latents {case}", imgs[F16], imgs[BF16], truth_i, yard_i)
    t8 = _u8(truth_i)
    frac = {k: float((_u8(v) != t8).mean()) for k, v in (("fp16", imgs[F16]), ("bf16", imgs[BF16]), ("ref-fp16", yard_i))}
    record(f"[parity vae fp16] 8-bit views {case}: fraction differing from the fp32 oracle: ours fp16 {frac['fp16']:.4%}, "
           f"ours bf16 {frac['bf16']:.4%}, reference-fp16 {frac['ref-fp16']:.4%}")
    assert frac["fp16"] <= frac["ref-fp16"] + U8_SLACK, frac


@torch.no_grad()
def test_decode_fp16_vs_reference_fixture(cuda_lib):
    g = golden("vae_decode.pt")
    cfg = arch.VaeConfig(block_out_channels=tuple(g["block_out_channels"]))
    sd = arch.synthetic_state_dict(arch.vae_decoder_param_shapes(cfg), g["seed"])
    vaes = _both(cfg, sd)
    z = g["z"].to(DEV)
    out = {dt: v.decode(z.to(dt)).sample for dt, v in vaes.items()}
    yard = O.vae_decode({k: v.to(DEV, F16) for k, v in sd.items()}, cfg, z.half()).float()
    _check("decode fixture", out[F16], out[BF16], g["sample"], yard)


# ------------------------------------------------------------------------------------------------ models: encode
def _latent_size(x):
    for _ in range(3):
        x = (x - 2) // 2 + 1
    return x


ENCODE_CASES = {  # name: (config, n, H, W)
    "small_50x70": (vae_config(), 2, 50, 70),
    "small_27x45": (vae_config(), 3, 27, 45),
    "sd15_224x400": (SD15, 6, 224, 400),
    "sd15_272x736": (SD15, 1, 272, 736),
    "sd15_424x800": (SD15, 6, 424, 800),
}


@torch.no_grad()
@pytest.mark.parametrize("case", list(ENCODE_CASES))
def test_encode_fp16(cuda_lib, case):
    cfg, n, h, w = ENCODE_CASES[case]
    sd = full_state_dict(cfg, 17)
    vaes = _both(cfg, sd)
    s32 = {k: v.to(DEV) for k, v in sd.items()}
    x = images(n, h, w, 5).to(DEV)
    truth = OV.vae_encode_moments(s32, cfg, x)
    yard = OV.vae_encode_moments(s32, cfg, x, dtype=F16).float()
    dist = {dt: v.encode(x.to(dt)).latent_dist for dt, v in vaes.items()}
    m16 = dist[F16].parameters
    assert vaes[F16].encoder_engine().dtype == F16 and m16.dtype == F16
    assert m16.shape == (n, 8, _latent_size(h), _latent_size(w))
    _check(f"encode {case} moments", m16, dist[BF16].parameters, truth, yard)
    _check(f"encode {case} mean", dist[F16].mean, dist[BF16].mean, truth[:, :4], yard[:, :4])
    del truth, yard, dist
    torch.cuda.empty_cache()
    pix = x.reshape(1, n, 3, h, w)
    lat = {dt: v.encode_latents(pix) for dt, v in vaes.items()}
    assert lat[F16].dtype == F32
    _check(f"encode_latents {case}", lat[F16], lat[BF16], OV.encode_latents(s32, cfg, pix),
           OV.encode_latents(s32, cfg, pix, dtype=F16).float())


@torch.no_grad()
@pytest.mark.parametrize("case", ["odd", "even"])
def test_encode_fp16_vs_reference_fixture(cuda_lib, case):
    fx = torch.load(os.path.join(GOLDEN, "vae_encode.pt"), map_location="cpu", weights_only=False)
    cfg = arch.VaeConfig(block_out_channels=tuple(fx["block_out_channels"]))
    sd = full_state_dict(cfg, fx["seed"])
    vaes = _both(cfg, sd)
    c = fx["cases"][case]
    x = c["x"].to(DEV)
    dist = {dt: v.encode(x.to(dt)).latent_dist for dt, v in vaes.items()}
    yard = OV.vae_encode_moments({k: v.to(DEV) for k, v in sd.items()}, cfg, x, dtype=F16).float()
    _check(f"encode fixture {case} moments", dist[F16].parameters, dist[BF16].parameters, c["moments"], yard)
    _check(f"encode fixture {case} mean", dist[F16].mean, dist[BF16].mean, c["mean"], yard[:, :4])


# ------------------------------------------------------------------------------------------------ graphs and .to()
# 64 / 128 channels: GroupNorm(32) runs its deterministic single-kernel path (see test_vae_encode_gpu.py)
DET = arch.VaeConfig(block_out_channels=(64, 128, 128, 128))


@torch.no_grad()
def test_graph_replay_is_bitwise_the_eager_call(cuda_lib):
    vae = _both(DET, full_state_dict(DET, 23))[F16]
    lat = torch.randn(1, 6, 4, 10, 13, generator=torch.Generator().manual_seed(4)).to(DEV)
    pix = images(6, 80, 104, 8).reshape(1, 6, 3, 80, 104).to(DEV)
    first_d, first_e = vae.decode_latents(lat), vae.encode_latents(pix)  # capture
    replay_d, replay_e = vae.decode_latents(lat), vae.encode_latents(pix)
    vae.use_cuda_graph = False
    eager_d, eager_e = vae.decode_latents(lat), vae.encode_latents(pix)
    assert torch.equal(first_d, replay_d) and torch.equal(replay_d, eager_d)
    assert torch.equal(first_e, replay_e) and torch.equal(replay_e, eager_e)


def _fresh(vae):
    """A newly built module with `vae`'s current parameters, in their dtype."""
    sd = {k: v.detach().clone() for k, v in vae.state_dict().items()}
    m = AutoencoderKL(**asdict(DET))
    m.load_state_dict({k: v.float() for k, v in sd.items()})
    return m.to(DEV, next(iter(sd.values())).dtype)


@torch.no_grad()
def test_to_bf16_and_back_equals_a_fresh_module(cuda_lib):
    """Engines and captured graphs follow .to(): after each dtype change the results are those of a module built fresh with
    the same parameters (bf16 <-> fp16 rounds the parameters, so each step is compared with its own fresh module)."""
    lat = torch.randn(1, 6, 4, 10, 13, generator=torch.Generator().manual_seed(5)).to(DEV)
    pix = images(6, 80, 104, 9).reshape(1, 6, 3, 80, 104).to(DEV)
    vae = _both(DET, full_state_dict(DET, 29))[F16]
    d16, e16 = vae.decode_latents(lat), vae.encode_latents(pix)  # graphs captured in fp16
    vae.to(BF16)
    dbf, ebf = vae.decode_latents(lat), vae.encode_latents(pix)
    assert vae.engine().dtype == vae.encoder_engine().dtype == BF16 and not torch.equal(dbf, d16)
    fresh = _fresh(vae)
    assert torch.equal(dbf, fresh.decode_latents(lat)) and torch.equal(ebf, fresh.encode_latents(pix))
    vae.to(F16)
    d, e = vae.decode_latents(lat), vae.encode_latents(pix)
    assert vae.engine().dtype == vae.encoder_engine().dtype == F16 and not torch.equal(d, dbf)
    fresh = _fresh(vae)
    assert torch.equal(d, fresh.decode_latents(lat)) and torch.equal(e, fresh.encode_latents(pix))


# ------------------------------------------------------------------------------------------------ with the denoiser
@torch.no_grad()
def test_sd15_unipc_loop_to_images_with_fp16_vae(cuda_lib):
    """3 UniPC CFG steps of the fp16 UNet / ControlNet at 224x400 (CUDA graph, two-stream overlap) decoded by an fp16 VAE
    through output_type="pt", against the fp32 oracle chain (loop, then decode_latents)."""
    from magicdrive_b200.synthetic import synthetic_inputs
    ucfg, ccfg = arch.UNetConfig(), arch.ControlNetConfig()
    usd = arch.synthetic_state_dict(arch.unet_param_shapes(ucfg), 11)
    csd = arch.synthetic_state_dict(arch.controlnet_param_shapes(ccfg), 12)
    vsd = arch.synthetic_state_dict(arch.vae_decoder_param_shapes(SD15), 13)
    inp = synthetic_inputs(1, 6, 28, 50, n_box=20, map_hw=200, seed=0)
    vaes = _both(SD15, vsd)
    un = UNet2DConditionModelMultiview(**asdict(ucfg))
    cn = BEVControlNetModel(**asdict(ccfg))
    un.load_state_dict(usd)
    cn.load_state_dict(csd)
    pipe = BEVControlNetDenoiser(un.to(DEV, F16), cn.to(DEV, F16), use_cuda_graph=True, overlap_controlnet=True,
                                 scheduler="unipc", vae=vaes[F16])
    kw = dict(image=inp["bev_map"], camera_param=inp["camera_param"], prompt_embeds=inp["prompt_embeds"],
              negative_prompt_embeds=inp["negative_prompt_embeds"], latents=inp["latents"], num_inference_steps=3,
              guidance_scale=2.0, bev_controlnet_kwargs={"bboxes_3d_data": inp["bboxes_3d_data"]})
    ours = pipe(output_type="pt", **kw)
    lat = pipe(output_type="latent", **kw)
    mixed = vaes[BF16].decode_latents(lat)  # the same latents through the bf16 VAE
    assert ours.dtype == F32 and ours.shape == (1, 6, 224, 400, 3) and torch.isfinite(ours).all()
    assert torch.equal(ours, vaes[F16].decode_latents(lat))
    del pipe, un, cn
    torch.cuda.empty_cache()
    di = to_dev(inp, DEV)

    def chain(dt):
        d = to_dev(di, DEV, dt)
        us, cs, vs = ({k: v.to(DEV, dt) for k, v in s.items()} for s in (usd, csd, vsd))
        lat_ = O.denoise_loop(us, cs, ucfg, ccfg, d["latents"], d["prompt_embeds"], d["negative_prompt_embeds"],
                              d["camera_param"], d["bboxes_3d_data"], d["bev_map"], 3, 2.0, scheduler="unipc")
        return O.decode_latents(vs, SD15, lat_.to(dt)).float()
    truth = chain(F32)
    yard = chain(F16)
    e, em, ey = rel_l2(ours, truth), rel_l2(mixed, truth), rel_l2(yard, truth)
    record(f"[parity vae fp16] 224x400 UniPC loop + decode: rel-L2 fp16 VAE {e:.3e}, bf16 VAE on the same latents {em:.3e}, "
           f"reference-fp16 chain {ey:.3e}")
    assert e < em and e <= ey + 1e-4, (e, em, ey)


PINNED = (0, 3)


@torch.no_grad()
@pytest.mark.parametrize("step_dtype", [F16, BF16], ids=["fp16-step", "bf16-step"])
def test_given_view_from_fp16_encoded_images(cuda_lib, step_dtype):
    """Images -> an fp16 VAE's encode_latents -> BEVControlNetDenoiser(conditional_latents=...) at the tiny config, 3 CFG
    steps.  Yardstick as in test_vae_encode_gpu.py: the denoiser's own error (fed the fp32 oracle's latents) plus how far the
    oracle's chain moves when fed the fp16 oracle's latents."""
    inp = golden("tiny_pipeline.pt")["inputs"]
    ucfg, ccfg = tiny_configs()
    usd, csd = tiny_state_dicts(7)
    un, cn = UNet2DConditionModelMultiview(**asdict(ucfg)), BEVControlNetModel(**asdict(ccfg))
    un.load_state_dict(usd)
    cn.load_state_dict(csd)
    if step_dtype == F16:
        un, cn = un.half(), cn.half()
    pipe = BEVControlNetDenoiser(un.to(DEV), cn.to(DEV), use_cuda_graph=True, scheduler="ddim")
    cfg = vae_config()
    vsd = full_state_dict(cfg, 29)
    vae = _both(cfg, vsd)[F16]
    pix = images(6, 80, 104, 12).reshape(1, 6, 3, 80, 104)
    pin = lambda lat: [[lat[0, j] if j in PINNED else None for j in range(6)]]
    kw = dict(image=inp["bev_map"], camera_param=inp["camera_param"], prompt_embeds=inp["prompt_embeds"],
              negative_prompt_embeds=inp["negative_prompt_embeds"], latents=inp["latents"], num_inference_steps=3,
              guidance_scale=2.0, bev_controlnet_kwargs={"bboxes_3d_data": inp["bboxes_3d_data"]})
    ours = pipe(conditional_latents=pin(vae.encode_latents(pix.to(DEV, F16))), **kw)
    cpu_vsd = {k: v.cpu() for k, v in vsd.items()}
    lat32 = OV.encode_latents(cpu_vsd, cfg, pix)
    lat16 = OV.encode_latents({k: v.to(DEV) for k, v in vsd.items()}, cfg, pix.to(DEV), dtype=F16).float().cpu()
    chain = lambda lat: O.denoise_loop(usd, csd, ucfg, ccfg, inp["latents"], inp["prompt_embeds"], inp["negative_prompt_embeds"],
                                       inp["camera_param"], inp["bboxes_3d_data"], inp["bev_map"], 3, 2.0,
                                       conditional_latents=pin(lat))
    truth = chain(lat32)
    e = rel_l2(ours, truth)
    e_den = rel_l2(pipe(conditional_latents=pin(lat32.to(DEV)), **kw), truth)
    e_enc = rel_l2(chain(lat16), truth)
    record(f"[parity vae fp16] given view from fp16-encoded images ({step_dtype} step): rel-L2 {e:.3e}; denoiser alone "
           f"{e_den:.3e}, fp16 encode in the oracle {e_enc:.3e}")
    assert ours.shape == truth.shape and torch.isfinite(ours).all() and e <= e_den + e_enc + 5e-4
