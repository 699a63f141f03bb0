"""The step's small operators and the device input preparation against float64 or exact references, under guard bands.

Covers the entry points of csrc/capi_pointwise.cu and csrc/capi_inputprep.cu that run on every call or every step: the
latent update the denoiser returns (cfg_ddim_step, cfg_unipc_step, pin_views), the time embedding and the skinny linear
layers behind it (timestep_embedding, linear_small), the camera and box tokens (fourier_embed, camera_param,
prepare_boxes), and the layout / dtype changes at the module boundary (nchw_to_nhwc, nhwc_to_nchw, pack_latents,
upsample_nearest, add, f32_to_bf16, bf16_to_f32).

Criteria, per element:
* copies, conversions, the bf16 add and the nearest resize are bitwise equal to torch (NaN compared as NaN);
* guidance + scheduler updates and pin_views: |err| <= 2^-21 * sum|terms| of the header's formula evaluated in float64 from the
  same fp32 inputs;
* the embeddings: |err| <= 2^-21 * max(1, |arg|) against the reference formula in float64 (2^-20 for the timestep
  embedding, whose exponent is itself rounded to fp32);
* linear_small: |err| <= 2^-20 * (sum|h w| + |b|) against float64 from the bf16 weights and fp32 inputs;
* camera_param: K and R^T bitwise, -R^T t within 2^-21 * sum|R t|;
* prepare_boxes: masks, classes and counts exact, corners at rtol 1e-5 / atol 2e-5 against oracle/input_prep.py.

Every output sits in a buffer pre-filled with a bit pattern no kernel produces (test_kernel_edges_gpu.Guarded): guard rows
before and after, guard columns on both sides wherever the ABI takes a row stride, NaN in the unused pad channels of
in-place buffers.  Every guard must be bitwise unchanged and no output element may still hold the fill.  Argument checks
must return their status and leave the guarded output untouched.

Also here: programmatic dependent launch on against off, bitwise, and the CPU emulator of these operators
(tests/ops_emulator.py) against the kernels."""
import math
import os
from dataclasses import asdict

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from magicdrive_b200 import _lib, ops  # noqa: E402
from oracle import input_prep as OP  # noqa: E402  (checker only)
from tests.common import record  # noqa: E402
from tests.test_kernel_edges_gpu import _FILL, BF16, F16, F32, F64, G, _bf, _gen, with_dt  # noqa: E402
from tests.test_kernel_edges_gpu import Guarded as _Guarded  # noqa: E402
from tests.test_kernel_edges_gpu import _close, _close_f32  # noqa: E402

I32, I64, U8 = torch.int32, torch.int64, torch.uint8
INVALID, UNSUPPORTED = -1, -3
_FILL_INT = {I32: (I32, 0x5AA5A55A), I64: (I64, 0x5AA5A55A5AA5A55A), U8: (U8, 0xA5)}  # values no kernel here writes
_BITS = {BF16: torch.int16, F16: torch.int16, F32: torch.int32}
WORST = {}  # operator -> largest measured |err| / bound


def _attn_close(out, ref, n_sets=1):
    """Kernel against the emulator (both from the same stored inputs): xformers' tolerances, bf16 atol 2e-2 / rtol 5e-3
    (3e-2 with several sets), fp16 atol 4e-3 / rtol 4e-4.  The kernel against float64 is held to the error model of
    tests/attention_model.py (test_attention_bounds_gpu.py)."""
    if out.dtype == F16:
        torch.testing.assert_close(out.to(F64), ref, atol=4e-3, rtol=4e-4)
    else:
        torch.testing.assert_close(out.to(F64), ref, atol=2e-2 if n_sets == 1 else 3e-2, rtol=5e-3)


class Guarded(_Guarded):
    """test_kernel_edges_gpu.Guarded, also for int32 / int64 / uint8 outputs."""

    def __init__(self, rows, cols, dtype=F32, ld=None, col0=0):
        if dtype in _FILL:
            super().__init__(rows, cols, dtype, ld, col0)
            return
        self.rows, self.cols, self.col0, self.ld = rows, cols, col0, ld or cols
        assert col0 + cols <= self.ld
        self.itype, self.fill = _FILL_INT[dtype]
        self.buf = torch.full((rows + 2 * G, self.ld), self.fill, dtype=dtype, device="cuda")
        self.out = self.buf[G:G + rows, col0:col0 + cols]

    def untouched(self, what=""):
        torch.cuda.synchronize()
        assert bool((self.buf.view(self.itype) == self.fill).all()), f"{what}: a rejected call wrote to its output"


def _inplace(values, ld=None):
    """A guarded fp32 buffer whose interior holds `values` (an in-place operand; NaN in pad columns when ld > cols)."""
    gd = Guarded(values.shape[0], values.shape[1], F32, ld=ld)
    gd.out.copy_(values)
    return gd


def _st():
    return torch.cuda.current_stream().cuda_stream


def _lib_ok(rc, what):
    assert rc == 0, f"{what} returned {rc}: {_lib.lib().mdb_last_error()}"


def _same(out, ref, what=""):
    """Bitwise equal, NaN compared as NaN."""
    assert out.dtype == ref.dtype and out.shape == ref.shape, (what, out.dtype, ref.dtype, out.shape, ref.shape)
    it = _BITS[out.dtype]
    ok = (out.view(it) == ref.view(it)) | (out.isnan() & ref.isnan())
    bad = (~ok).nonzero()
    assert bad.shape[0] == 0, f"{what}: {bad.shape[0]} elements differ, first at {tuple(bad[0].tolist())}: " \
                              f"{out[tuple(bad[0].tolist())].item()!r} vs {ref[tuple(bad[0].tolist())].item()!r}"


def _within(op, out, ref, bound, what=""):
    """|out - ref| <= bound elementwise (NaN fails); records the largest ratio for `op`."""
    err = (out.to(F64) - ref).abs()
    bad = (~(err <= bound)).nonzero()
    ratio = (err / bound.clamp_min(1e-300)).max().item()
    WORST[op] = max(WORST.get(op, 0.0), ratio)
    assert bad.shape[0] == 0, f"{what}: {bad.shape[0]} elements off, first at {tuple(bad[0].tolist())}: " \
                              f"err {err[tuple(bad[0].tolist())].item():.3e} bound {bound[tuple(bad[0].tolist())].item():.3e}"


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    for op, r in sorted(WORST.items()):
        record(f"[bound] {op}: max |err| / bound = {r:.3f}", "small_ops_gpu_latest.txt")


# ------------------------------------------------------------------------------------------------------ add
@pytest.mark.parametrize("n", [8, 8 * 1001, 12 * 28 * 50 * 320])
def test_add_bitwise(cuda_lib, n):
    g = _gen(1)
    a = _bf(torch.randn(n, device="cuda", generator=g) * 4)
    b = _bf(torch.randn(n, device="cuda", generator=g) * 4)
    inf, big = float("inf"), 3.3895e38
    # 0 + -0, -0 + -0, inf + -inf, -inf + 1, NaN + 2, overflow to ±inf, two subnormals
    a[:8] = torch.tensor([0.0, -0.0, inf, -inf, float("nan"), big, -big, 1e-40], dtype=BF16, device="cuda")
    b[:8] = torch.tensor([-0.0, -0.0, -inf, 1.0, 2.0, big, -big, 1e-40], dtype=BF16, device="cuda")
    out = Guarded(n // 8, 8, BF16)
    _lib_ok(cuda_lib.mdb_add(a.data_ptr(), b.data_ptr(), out.out.data_ptr(), n, _st()), "mdb_add")
    out.check("add")
    _same(out.out.reshape(-1), (a.float() + b.float()).to(BF16), "add")


# ------------------------------------------------------------------------------------------------------ upsample
# (n, h, w, c, ho, wo): the UNet's up-path pairs of the 224x400, 272x736 and 424x800 pyramids at their channel counts, the VAE
# decoder's 2x steps, and sizes where floor(j * h / ho) and ATen's float-scale index differ (26 -> 44: output row 22)
UPSAMPLE = [
    (2, 4, 7, 1280, 7, 13), (2, 7, 13, 1280, 14, 25), (2, 14, 25, 640, 28, 50),
    (2, 5, 12, 1280, 9, 23), (2, 9, 23, 1280, 17, 46), (1, 17, 46, 640, 34, 92),
    (1, 7, 13, 1280, 14, 25), (1, 14, 25, 1280, 27, 50), (1, 27, 50, 640, 53, 100),
    (1, 28, 50, 512, 56, 100), (1, 56, 100, 512, 112, 200), (1, 112, 200, 256, 224, 400), (1, 53, 100, 128, 106, 200),
    (3, 26, 26, 8, 44, 44), (2, 13, 26, 16, 22, 44), (1, 3, 5, 8, 7, 11),
]


@pytest.mark.parametrize("n,h,w,c,ho,wo", UPSAMPLE)
def test_upsample_nearest_bitwise(cuda_lib, n, h, w, c, ho, wo):
    x = _bf(torch.randn(n, h, w, c, device="cuda", generator=_gen(2)))
    out = Guarded(n * ho * wo, c, BF16)
    _lib_ok(cuda_lib.mdb_upsample_nearest(x.data_ptr(), n, h, w, c, out.out.data_ptr(), ho, wo, _st()), "upsample")
    out.check("upsample")
    ref = F.interpolate(x.permute(0, 3, 1, 2).float(), size=(ho, wo), mode="nearest").permute(0, 2, 3, 1)
    _same(out.out, ref.reshape(-1, c).to(BF16), "upsample")


# ------------------------------------------------------------------------------------------------------ layout
LAYOUT = [(c, n, h, w) for c in (3, 4, 8, 33) for (n, h, w) in ((2, 28, 50), (3, 5, 7))] + \
         [(320, 2, 28, 50), (320, 12, 7, 13), (1280, 2, 7, 13), (1280, 1, 14, 25), (640, 2, 27, 50)]


@pytest.mark.parametrize("x_dtype", [F32, BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("c,n,h,w", LAYOUT)
def test_nchw_to_nhwc_bitwise(cuda_lib, c, n, h, w, x_dtype):
    x = (torch.randn(n, c, h, w, device="cuda", generator=_gen(3)) * 3).to(x_dtype)
    out = Guarded(n * h * w, c, BF16)
    _lib_ok(cuda_lib.mdb_nchw_to_nhwc(x.data_ptr(), int(x_dtype == F32), n, c, h, w, out.out.data_ptr(), _st()), "nchw_to_nhwc")
    out.check("nchw_to_nhwc")
    _same(out.out, x.permute(0, 2, 3, 1).reshape(-1, c).to(BF16), "nchw_to_nhwc")


# + the FID Inception block outputs (64 x 73x73, 192 x 35x35, 768 x 17x17 for a 299x299 input)
@pytest.mark.parametrize("out_dtype", [F32, BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("c,n,h,w", LAYOUT + [(64, 2, 73, 73), (192, 2, 35, 35), (768, 2, 17, 17)])
def test_nhwc_to_nchw_bitwise(cuda_lib, c, n, h, w, out_dtype):
    x = _bf(torch.randn(n * h * w, c, device="cuda", generator=_gen(4)) * 3)
    out = Guarded(n * c, h * w, out_dtype)
    _lib_ok(cuda_lib.mdb_nhwc_to_nchw(x.data_ptr(), n, c, h, w, out.out.data_ptr(), int(out_dtype == F32), _st()),
            "nhwc_to_nchw")
    out.check("nhwc_to_nchw")
    _same(out.out, x.view(n, h * w, c).permute(0, 2, 1).reshape(n * c, h * w).to(out_dtype), "nhwc_to_nchw")


@pytest.mark.parametrize("repeat", [1, 2])
@pytest.mark.parametrize("x_dtype", [F32, BF16, F16], ids=["f32", "bf16", "f16"])
@pytest.mark.parametrize("pix", [12 * 28 * 50, 1001])
def test_pack_latents_bitwise(cuda_lib, pix, x_dtype, repeat):
    """mdb_pack_latents from fp32 / bf16, and mdb_pack_latents_f16 (an fp16 model's conv_in operand) from an f16 source,
    which it copies without a conversion (its fp32 source is test_fp16_kernels_gpu.py's)."""
    cin, cpad = 4, 64
    x = (torch.randn(pix, cin, device="cuda", generator=_gen(5)) * 3).to(x_dtype)
    odt = F16 if x_dtype == F16 else BF16
    fn = cuda_lib.mdb_pack_latents_f16 if x_dtype == F16 else cuda_lib.mdb_pack_latents
    out = Guarded(repeat * pix, cpad, odt)
    _lib_ok(fn(x.data_ptr(), int(x_dtype == F32), pix, cin, cpad, repeat, out.out.data_ptr(), _st()), "pack_latents")
    out.check("pack_latents")
    _same(out.out, F.pad(x.to(odt), (0, cpad - cin)).repeat(repeat, 1), "pack_latents")


# ------------------------------------------------------------------------------------------------------ conversions
def _bf16_patterns():
    """All 65536 bf16 bit patterns (±0, subnormals, ±inf, every NaN payload) as a bf16 tensor."""
    return torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(BF16)


def test_bf16_to_f32_exhaustive(cuda_lib):
    x = _bf16_patterns().cuda()
    out = Guarded(x.numel(), 1, F32)
    _lib_ok(cuda_lib.mdb_bf16_to_f32(x.data_ptr(), out.out.data_ptr(), x.numel(), _st()), "bf16_to_f32")
    out.check("bf16_to_f32")
    _same(out.out.reshape(-1), x.float(), "bf16_to_f32")


def test_f32_to_bf16_round_to_nearest_even(cuda_lib):
    """Every bf16 pattern widened with low halves 0, 1, 0x7FFF, 0x8000 (a tie), 0x8001 and 0xFFFF: exact values, ties to
    even in both directions, rounding across binade edges and into inf, subnormals, ±0, ±inf and NaNs whose payload sits in
    the low half only; plus random fp32 values.  Reference: torch's CPU conversion (round to nearest even)."""
    hi = _bf16_patterns().view(torch.int16).to(torch.int32) << 16
    lows = torch.tensor([0, 1, 0x7FFF, 0x8000, 0x8001, 0xFFFF], dtype=torch.int32)
    bits = (hi[:, None] | lows[None, :]).reshape(-1)
    rnd = torch.randn(100003, generator=torch.Generator().manual_seed(6)) * torch.logspace(-40, 38, 100003).float()
    x = torch.cat([bits.view(F32), rnd]).cuda()
    out = Guarded(x.numel(), 1, BF16)
    _lib_ok(cuda_lib.mdb_f32_to_bf16(x.data_ptr(), out.out.data_ptr(), x.numel(), _st()), "f32_to_bf16")
    out.check("f32_to_bf16")
    _same(out.out.reshape(-1), x.cpu().to(BF16).cuda(), "f32_to_bf16")


# ------------------------------------------------------------------------------------------------------ guidance + schedulers
def _combine(eu, ec, cfg, gd):
    """(e, sum|terms| of e) in float64: e = eu + g (ec - eu) with guidance, else eu."""
    if not cfg:
        return eu, eu.abs()
    return eu + gd * (ec - eu), eu.abs() + gd * (ec.abs() + eu.abs())


CFG = [(False, 1.0), (True, 1.0), (True, 2.5), (True, 7.5)]
CFG_IDS = ["nocfg", "g1", "g2.5", "g7.5"]
SIZES = {"424x800x12": 12 * 53 * 100, "small": 6 * 10 * 13 + 1}


@pytest.mark.parametrize("size", list(SIZES))
@pytest.mark.parametrize("eps_ld", [4, 8])
@pytest.mark.parametrize("cfg,guidance", CFG, ids=CFG_IDS)
def test_cfg_ddim_step(cuda_lib, cfg, guidance, eps_ld, size):
    from magicdrive_b200.pipeline import DDIMSchedule
    npix, c = SIZES[size], 4
    g = _gen(7)
    sch = DDIMSchedule()
    sch.set_timesteps(20)
    coef = torch.tensor(sch.coefs[13], dtype=F32, device="cuda")
    eps = _inplace(torch.randn((2 if cfg else 1) * npix, c, device="cuda", generator=g), ld=eps_ld)
    lat = _inplace(torch.randn(npix, c, device="cuda", generator=g) * 5)
    x0 = lat.out.to(F64)
    _lib_ok(cuda_lib.mdb_cfg_ddim_step(eps.out.data_ptr(), eps_ld, c, int(cfg), guidance, coef.data_ptr(), lat.out.data_ptr(),
                                       npix * c, _st()), "cfg_ddim_step")
    lat.check("latents")
    eps.check("eps")
    e64 = eps.out.to(F64)
    e, ea = _combine(e64[:npix], e64[npix:], cfg, guidance)
    c0, c1 = coef.to(F64).tolist()
    ref = c0 * x0 + c1 * e
    _within("cfg_ddim_step", lat.out, ref, 2.0 ** -21 * (abs(c0) * x0.abs() + abs(c1) * ea), "ddim")


@pytest.mark.parametrize("size", list(SIZES))
@pytest.mark.parametrize("eps_ld", [4, 8])
@pytest.mark.parametrize("cfg,guidance", CFG, ids=CFG_IDS)
def test_cfg_unipc_step_full_schedule(cuda_lib, cfg, guidance, eps_ld, size):
    """A whole 20-step UniPC coefficient sequence (the corrector off at step 0, on after): each step against float64 of the
    header's formula on the fp32 state the previous step left."""
    from magicdrive_b200.pipeline import UniPCSchedule
    npix, c = SIZES[size], 4
    g = _gen(8)
    sch = UniPCSchedule()
    sch.set_timesteps(20)
    lat = _inplace(torch.randn(npix, c, device="cuda", generator=g) * 14)
    last, m0, m1 = (_inplace(torch.zeros(npix, c, device="cuda")) for _ in range(3))
    seen = set()
    for i, cf in enumerate(sch.coefs):
        coef = torch.tensor(cf, dtype=F32, device="cuda")
        k = coef.to(F64).tolist()
        seen.add(k[9] != 0)
        eps = _inplace(torch.randn((2 if cfg else 1) * npix, c, device="cuda", generator=g), ld=eps_ld)
        x, la, h0, h1 = (t.out.to(F64) for t in (lat, last, m0, m1))
        h0_bits = m0.out.clone()
        _lib_ok(cuda_lib.mdb_cfg_unipc_step(eps.out.data_ptr(), eps_ld, c, int(cfg), guidance, coef.data_ptr(),
                                            lat.out.data_ptr(), last.out.data_ptr(), m0.out.data_ptr(), m1.out.data_ptr(),
                                            npix * c, _st()), "cfg_unipc_step")
        for name, t in (("latents", lat), ("last", last), ("m0", m0), ("m1", m1), ("eps", eps)):
            t.check(f"step {i} {name}")
        e64 = eps.out.to(F64)
        ref = _unipc_ref(k, x, la, h0, h1, e64[:npix], e64[npix:], cfg, guidance)
        for name, t in (("latents", lat), ("last", last), ("m0", m0)):
            _within("cfg_unipc_step", t.out, *ref[name], f"step {i} {name}")
        _same(m1.out, h0_bits, f"step {i} m1")  # the history shift is a copy
    assert seen == {False, True}


def _unipc_ref(k, x, last, h0, h1, eu, ec, cfg, gd):
    """The header's UniPC step in float64: {output: (value, 2^-21 * sum|terms|)} for the new latents, last and m0
    (m1 becomes h0)."""
    e, ea = _combine(eu, ec, cfg, gd)
    x0 = k[0] * x + k[1] * e
    x0a = abs(k[0]) * x.abs() + abs(k[1]) * ea
    if k[9] != 0:
        xc = k[2] * last + k[3] * h0 + k[4] * h1 + k[5] * x0
        xca = abs(k[2]) * last.abs() + abs(k[3]) * h0.abs() + abs(k[4]) * h1.abs() + abs(k[5]) * x0a
    else:
        xc, xca = x, x.abs()
    new = k[6] * xc + k[7] * x0 + k[8] * h0
    newa = abs(k[6]) * xca + abs(k[7]) * x0a + abs(k[8]) * h0.abs()
    b = 2.0 ** -21
    return {"latents": (new, b * newa), "last": (xc, b * xca), "m0": (x0, b * x0a)}


@pytest.mark.parametrize("rows_per_view", [130, 53 * 100])
@pytest.mark.parametrize("with_a", [True, False], ids=["a", "a_null"])
@pytest.mark.parametrize("views", ["all", "none", "alternate", "some"])
def test_pin_views(cuda_lib, views, with_a, rows_per_view):
    n_views, c, ld = 12, 4, 8
    mask = {"all": [1] * 12, "none": [0] * 12, "alternate": [1, 0] * 6, "some": [1, 0, 0, 1, 0, 0, 0, 1, 0, 0, 0, 1]}[views]
    g = _gen(9)
    rows = n_views * rows_per_view
    dst = _inplace(torch.randn(rows, c, device="cuda", generator=g), ld=ld)
    before = dst.out.clone()
    a = torch.randn(rows, c, device="cuda", generator=g) if with_a else None
    b = torch.randn(rows, c, device="cuda", generator=g)
    coef = torch.tensor([0.7316, -1.2904] if with_a else [0.0, 1.0], dtype=F32, device="cuda")
    m = torch.tensor(mask, dtype=I32, device="cuda")
    _lib_ok(cuda_lib.mdb_pin_views(dst.out.data_ptr(), ld, a.data_ptr() if with_a else None, b.data_ptr(), c, coef.data_ptr(),
                                   m.data_ptr(), rows_per_view, n_views, _st()), "pin_views")
    dst.check("pin_views")
    sel = m.bool().repeat_interleave(rows_per_view)
    k0, k1 = coef.to(F64).tolist()
    ref = k1 * b.to(F64) + (k0 * a.to(F64) if with_a else 0)
    bound = 2.0 ** -21 * (abs(k1) * b.to(F64).abs() + (abs(k0) * a.to(F64).abs() if with_a else 0))
    if sel.any():
        _within("pin_views", dst.out[sel], ref[sel], bound[sel], "pinned rows")
    _same(dst.out[~sel], before[~sel], "rows of unpinned views")


# ------------------------------------------------------------------------------------------------------ embeddings
@pytest.mark.parametrize("freq_shift", [0.0, 1.0])
@pytest.mark.parametrize("flip", [1, 0])
@pytest.mark.parametrize("dim", [320, 321, 2])
def test_timestep_embedding(cuda_lib, dim, flip, freq_shift):
    """get_timestep_embedding (embeddings.py:24-64) in float64; odd dim pads a zero column.  Bound 2^-20 * max(1, |arg|):
    the exponent -ln(10^4) j / (half - shift) is rounded to fp32 (as in the reference), so arg carries a relative error of a
    few 2^-24 times |exponent| (up to 9.2); measured 1.13 * 2^-21 * |arg| at t = 999 on H100."""
    if dim == 2 and freq_shift == 1.0:
        pytest.skip("half - freq_shift = 0: the formula itself divides by zero")
    t = torch.tensor([0.0, 1.0, 500.0, 981.0, 999.0], device="cuda")
    m, half = t.numel(), dim // 2
    out = Guarded(m, dim, F32)
    _lib_ok(cuda_lib.mdb_timestep_embedding(t.data_ptr(), m, dim, flip, freq_shift, out.out.data_ptr(), _st()), "timestep")
    out.check("timestep_embedding")
    j = torch.arange(half, dtype=F64, device="cuda")
    arg = t.to(F64)[:, None] * torch.exp(-math.log(10000.0) * j / (half - freq_shift))[None]
    s, co = torch.sin(arg), torch.cos(arg)
    ref = torch.cat([co, s] if flip else [s, co], -1)
    a = arg.abs().clamp_min(1.0).repeat(1, 2)
    if dim % 2:
        ref, a = F.pad(ref, (0, 1)), F.pad(a, (0, 1), value=1.0)
        assert bool((out.out[:, -1] == 0).all())
    _within("timestep_embedding", out.out, ref, 2.0 ** -20 * a, f"dim {dim} flip {flip} shift {freq_shift}")


@pytest.mark.parametrize("num_freqs", [4, 8])
def test_fourier_embed(cuda_lib, num_freqs):
    """Embedder (embedder.py:15-40) on box corners up to ±60 m: [x, sin(2^k x), cos(2^k x)] in float64."""
    rows, d = 1201, 3
    x = (torch.rand(rows, d, device="cuda", generator=_gen(10)) * 120 - 60)
    x[0] = torch.tensor([0.0, 60.0, -60.0])
    out = Guarded(rows, d * (1 + 2 * num_freqs), F32)
    _lib_ok(cuda_lib.mdb_fourier_embed(x.data_ptr(), rows, d, num_freqs, out.out.data_ptr(), _st()), "fourier")
    out.check("fourier_embed")
    x64 = x.to(F64)
    parts, bounds = [x64], [torch.zeros_like(x64)]
    for k in range(num_freqs):
        arg = x64 * 2.0 ** k
        parts += [torch.sin(arg), torch.cos(arg)]
        bounds += [2.0 ** -21 * arg.abs().clamp_min(1.0)] * 2
    _same(out.out[:, :d], x, "fourier identity part")
    _within("fourier_embed", out.out[:, d:], torch.cat(parts[1:], -1), torch.cat(bounds[1:], -1), f"{num_freqs} freqs")


# ------------------------------------------------------------------------------------------------------ linear_small
TEMB_TOTAL = 2 * 320 + 2 * 640 + 6 * 1280  # SD-1.5 UNet: one time_emb_proj slice per encoder + mid resnet (UNetEngine.temb_total)
# (m, n, k, ldw - k, ldi - k, ldo - n, bias, pre_silu, post_silu): every m around the 16-row chunk and the 64-CTA row loop
LINEAR_SMALL = [
    (1, 1280, 320, 0, 0, 0, True, False, True),            # time MLP linear_1
    (1, 1280, 1280, 0, 0, 0, True, False, False),          # time MLP linear_2
    (12, TEMB_TOTAL, 1280, 0, 0, 0, True, True, False),    # concatenated time_emb_proj
    (15, 33, 189, 3, 5, 7, False, False, False),
    (16, 4, 8, 3, 0, 7, True, True, True),
    (17, 768, 189, 0, 5, 7, True, False, True),            # cam2token-like
    (1023, 1, 320, 3, 5, 7, True, True, False),
    (1024, 768, 3200, 0, 5, 7, False, True, True),         # k at the shared-memory limit
    (1025, 33, 1280, 0, 5, 7, True, False, False),
    (2100, 768, 189, 0, 0, 7, True, False, True),          # box encoder: 6 views x 350 padded boxes
    (2100, 1280, 3200, 3, 5, 7, True, True, True),
]


@pytest.mark.parametrize("wdt,m,n,k,dw,di,do,bias,pre,post", with_dt(LINEAR_SMALL))
def test_linear_small(cuda_lib, wdt, m, n, k, dw, di, do, bias, pre, post):
    """fp32 activations times bf16 weights (mdb_linear_small) or f16 weights (mdb_linear_small_f16, fp16 models).  The
    bound is one of fp32 arithmetic on the weights as stored, so it holds for either weight type."""
    g = _gen(11)
    ldw, ldi, ldo = k + dw, k + di, n + do
    xin = torch.randn(m, ldi, device="cuda", generator=g) * 2
    wbuf = (torch.randn(n, ldw, device="cuda", generator=g) / math.sqrt(k)).to(wdt)
    b = torch.randn(n, device="cuda", generator=g) if bias else None
    out = Guarded(m, n, F32, ld=ldo, col0=do // 2)  # guard columns on both sides when ldo > n
    fn = cuda_lib.mdb_linear_small_f16 if wdt == F16 else cuda_lib.mdb_linear_small
    rc = fn(xin.data_ptr(), m, k, ldi, wbuf.data_ptr(), ldw, b.data_ptr() if bias else None, n, int(pre), int(post),
            out.out.data_ptr(), ldo, _st())
    _lib_ok(rc, "linear_small")
    out.check(f"linear_small m={m} n={n} k={k}")
    y, bound = _linear_small_ref(xin[:, :k], wbuf[:, :k], b, pre, post)
    _within("linear_small", out.out, y, bound, f"m={m} n={n} k={k}")


def _linear_small_ref(x, w, b, pre, post):
    """float64 act(x) W^T + b and its bound 2^-20 (sum|h w| + |b|); after a post-SiLU (1.1-Lipschitz) the bound is scaled
    by 1.1 and gains 2^-21 |result| for the SiLU's own fp32 evaluation."""
    h, w = x.to(F64), w.to(F64)
    if pre:
        h = F.silu(h)
    y, mag = h @ w.t(), h.abs() @ w.abs().t()
    if b is not None:
        y, mag = y + b.to(F64), mag + b.to(F64).abs()
    bound = 2.0 ** -20 * mag
    if post:
        y = F.silu(y)
        bound = 1.1 * bound + 2.0 ** -21 * y.abs()
    return y, bound


# ------------------------------------------------------------------------------------------------------ camera_param
def _rigid(n, g, scale=20.0):
    """n random rigid transforms [R | t] as fp32 4x4 (det R = +1)."""
    q, r = torch.linalg.qr(torch.randn(n, 3, 3, generator=g, dtype=F64))
    q = q * torch.sign(torch.diagonal(r, dim1=1, dim2=2))[:, None, :]
    q[torch.linalg.det(q) < 0, :, 0] *= -1
    m = torch.eye(4, dtype=F64).repeat(n, 1, 1)
    m[:, :3, :3] = q
    m[:, :3, 3] = torch.randn(n, 3, generator=g, dtype=F64) * scale
    return m.float()


@pytest.mark.parametrize("n", [1, 6, 300])
def test_camera_param(cuda_lib, n):
    g = torch.Generator().manual_seed(12)
    K = torch.randn(n, 4, 4, generator=g) * 500
    M = _rigid(n, g)
    Kd, Md = K.cuda(), M.cuda()
    out = Guarded(n, 21, F32)
    _lib_ok(cuda_lib.mdb_camera_param(Kd.data_ptr(), Md.data_ptr(), n, out.out.data_ptr(), _st()), "camera_param")
    out.check("camera_param")
    o = out.out.view(n, 3, 7)
    _same(o[:, :, :3], Kd[:, :3, :3], "K")
    _same(o[:, :, 3:6], Md[:, :3, :3].transpose(1, 2).contiguous(), "R^T")
    R, t = M[:, :3, :3].to(F64).cuda(), M[:, :3, 3:].to(F64).cuda()
    ref = -(R.transpose(1, 2) @ t)
    bound = 2.0 ** -21 * (R.abs().transpose(1, 2) @ t.abs())
    _within("camera_param", o[:, :, 6:], ref, bound, "-R^T t")
    # the oracle restatement agrees (same float64 rigid inverse, rounded to fp32)
    torch.testing.assert_close(o.cpu(), OP.camera_param(K, M), rtol=1e-6, atol=1e-5)


# ------------------------------------------------------------------------------------------------------ prepare_boxes
N_VIEWS = 6
SCENE_BOXES = [1, 127, 0, 128, 300, 129]  # the 128-box passes carry their running count; an empty scene in the middle
MARGIN = 1e-2


def _depth_max(boxes, trans):
    """Largest camera-frame depth over the 8 corners of each box re-interpreted with a gravity-centre origin (the
    reference's visibility test) and of the box as given: float64 [n_views, n] each."""
    sh = boxes.clone()
    sh[:, 2] -= 0.5 * sh[:, 5]
    out = []
    for bx in (sh, boxes):
        cs = OP.corners(bx.to(F64))
        homo = torch.cat([cs, torch.ones(*cs.shape[:2], 1, dtype=F64)], -1)
        out.append(torch.einsum("nkj,vj->vnk", homo, trans[:, 2].to(F64)).amax(-1))
    return out


def _make_scenes(box_dim):
    """Boxes around tilted cameras, each at least MARGIN from the visibility boundary in every view of its scene."""
    g = torch.Generator().manual_seed(13)
    l2c = _rigid(len(SCENE_BOXES) * N_VIEWS, g, scale=2.0).view(len(SCENE_BOXES), N_VIEWS, 4, 4)
    aug = torch.eye(4).repeat(len(SCENE_BOXES), N_VIEWS, 1, 1)
    aug[..., 0, 0] = aug[..., 1, 1] = 0.5 + 0.1 * torch.rand(len(SCENE_BOXES), N_VIEWS, generator=g)
    aug[..., :2, 3] = torch.randn(len(SCENE_BOXES), N_VIEWS, 2, generator=g) * 30
    aug[..., 2, :] += torch.randn(len(SCENE_BOXES), N_VIEWS, 4, generator=g) * torch.tensor([0.02, 0.02, 0.1, 0.3])
    boxes, labels, flips = [], [], [0, 0]
    for s, nb in enumerate(SCENE_BOXES):
        trans = (aug[s] @ l2c[s])  # fp32, as the reference multiplies them
        cand = torch.cat([torch.randn(4000, 2, generator=g) * 6, torch.randn(4000, 1, generator=g) * 2,
                          0.5 + 4 * torch.rand(4000, 2, generator=g), 0.5 + 3 * torch.rand(4000, 1, generator=g),
                          (torch.rand(4000, 1, generator=g) * 2 - 1) * math.pi,
                          torch.randn(4000, box_dim - 7, generator=g)], 1)
        shifted, plain = _depth_max(cand, trans)
        keep = (shifted.abs() >= MARGIN).all(0) & (plain.abs() >= MARGIN).all(0)
        idx = keep.nonzero()[:, 0][:nb]
        assert idx.numel() == nb
        flips[0] += int(((shifted[:, idx] > 0) & (plain[:, idx] <= 0)).sum())
        flips[1] += int(((shifted[:, idx] <= 0) & (plain[:, idx] > 0)).sum())
        boxes.append(cand[idx])
        labels.append(torch.randint(0, 10, (nb,), generator=g))
    return boxes, labels, l2c, aug, flips


@pytest.fixture(scope="module")
def box_scenes():
    return {d: _make_scenes(d) for d in (9, 7)}


def _run_prepare(lib, boxes, labels, l2c, aug, capacity, box_dim, use_aug=True):
    S = len(boxes)
    off = torch.tensor([0] + np.cumsum([b.shape[0] for b in boxes]).tolist(), dtype=I32).cuda()
    bx = torch.cat(boxes).contiguous().cuda()
    lb = torch.cat(labels).cuda()
    l2c_d, aug_d = l2c.contiguous().cuda(), aug.contiguous().cuda()
    ob = Guarded(S * N_VIEWS * capacity, 24, F32)
    oc = Guarded(S * N_VIEWS, capacity, I64)
    om = Guarded(S * N_VIEWS, capacity, U8)
    cnt = Guarded(S, N_VIEWS, I32)
    _lib_ok(lib.mdb_prepare_boxes(bx.data_ptr(), box_dim, lb.data_ptr(), off.data_ptr(), S, l2c_d.data_ptr(),
                                  aug_d.data_ptr() if use_aug else None, N_VIEWS, capacity, ob.out.data_ptr(),
                                  oc.out.data_ptr(), om.out.data_ptr(), cnt.out.data_ptr(), _st()), "prepare_boxes")
    for name, t in (("boxes", ob), ("classes", oc), ("masks", om), ("counts", cnt)):
        t.check(f"prepare_boxes {name}")
    return ob, oc, om, cnt


@pytest.mark.parametrize("capacity", [300, 40, 1])
@pytest.mark.parametrize("box_dim", [9, 7])
def test_prepare_boxes(cuda_lib, box_scenes, box_dim, capacity):
    """Against oracle/input_prep.py scene by scene; below the visible count the oracle's list is truncated in order and the
    counts still report every visible box."""
    boxes, labels, l2c, aug, flips = box_scenes[box_dim]
    assert flips[0] > 0 and flips[1] > 0, flips  # boxes only the gravity-centre shift makes visible, and the reverse
    ob, oc, om, cnt = _run_prepare(cuda_lib, boxes, labels, l2c, aug, capacity, box_dim)
    S = len(boxes)
    got_b = ob.out.view(S, N_VIEWS, capacity, 8, 3).cpu()
    got_c, got_m = oc.out.view(S, N_VIEWS, capacity).cpu(), om.out.view(S, N_VIEWS, capacity).cpu()
    got_n = cnt.out.cpu()
    for s in range(S):
        want_b, want_c = torch.zeros(N_VIEWS, capacity, 8, 3), -torch.ones(N_VIEWS, capacity, dtype=I64)
        want_m, want_n = torch.zeros(N_VIEWS, capacity, dtype=U8), torch.zeros(N_VIEWS, dtype=I32)
        r = OP.preprocess_bbox(boxes[s], labels[s], l2c[s], aug[s]) if boxes[s].shape[0] else None
        if r is not None:
            L = min(capacity, r["masks"].shape[1])
            want_b[:, :L], want_c[:, :L], want_m[:, :L] = r["bboxes"][:, :L], r["classes"][:, :L], r["masks"][:, :L].to(U8)
            want_n = r["masks"].sum(-1).to(I32)
        what = f"scene {s} ({boxes[s].shape[0]} boxes) capacity {capacity}"
        assert torch.equal(got_n[s], want_n), (what, got_n[s].tolist(), want_n.tolist())
        assert torch.equal(got_m[s], want_m), what
        assert torch.equal(got_c[s], want_c), what
        assert bool((got_b[s][want_m == 0] == 0).all()), what
        torch.testing.assert_close(got_b[s], want_b, rtol=1e-5, atol=2e-5, msg=what)
    assert int(got_n.max()) > 128  # one view of the 300-box scene sees more boxes than one pass compacts


def test_prepare_boxes_without_img_aug_is_identity_aug(cuda_lib, box_scenes):
    boxes, labels, l2c, _, _ = box_scenes[9]
    eye = torch.eye(4).repeat(len(boxes), N_VIEWS, 1, 1)
    a = _run_prepare(cuda_lib, boxes, labels, l2c, eye, 300, 9, use_aug=True)
    b = _run_prepare(cuda_lib, boxes, labels, l2c, eye, 300, 9, use_aug=False)
    for x, y in zip(a, b):
        assert torch.equal(x.buf.view(x.itype), y.buf.view(y.itype))


# ------------------------------------------------------------------------------------------------------ argument checks
def test_argument_checks_reject_and_write_nothing(cuda_lib):
    L, st = cuda_lib, _st()
    x = torch.zeros(4096, device="cuda")
    p = x.data_ptr()
    o32 = Guarded(64, 64, F32)
    o16 = Guarded(64, 64, BF16)
    op = o32.out.data_ptr()

    def rejects(rc, want, what, *outs):
        assert rc == want, f"{what}: returned {rc}, expected {want} ({L.mdb_last_error()})"
        assert L.mdb_last_error(), what
        for o in outs or (o32, o16):
            o.untouched(what)

    o16p = o16.out.data_ptr()
    rejects(L.mdb_add(p, p, o16p, 12, st), UNSUPPORTED, "add n % 8")
    rejects(L.mdb_add(None, p, o16p, 16, st), INVALID, "add null a")
    rejects(L.mdb_add(p, p, None, 16, st), INVALID, "add null out")
    rejects(L.mdb_upsample_nearest(p, 1, 2, 2, 12, o16p, 4, 4, st), UNSUPPORTED, "upsample c % 8")
    rejects(L.mdb_upsample_nearest(None, 1, 2, 2, 8, o16p, 4, 4, st), INVALID, "upsample null x")
    rejects(L.mdb_nchw_to_nhwc(None, 1, 1, 4, 2, 2, o16p, st), INVALID, "nchw_to_nhwc null x")
    rejects(L.mdb_nchw_to_nhwc(p, 1, 1, 4, 2, 2, None, st), INVALID, "nchw_to_nhwc null out")
    rejects(L.mdb_nhwc_to_nchw(None, 1, 4, 2, 2, op, 1, st), INVALID, "nhwc_to_nchw null x")
    rejects(L.mdb_nhwc_to_nchw(p, 1, 4, 2, 2, None, 1, st), INVALID, "nhwc_to_nchw null out")
    rejects(L.mdb_f32_to_bf16(None, o16p, 16, st), INVALID, "f32_to_bf16 null x")
    rejects(L.mdb_f32_to_bf16(p, None, 16, st), INVALID, "f32_to_bf16 null out")
    rejects(L.mdb_bf16_to_f32(None, op, 16, st), INVALID, "bf16_to_f32 null x")
    rejects(L.mdb_bf16_to_f32(p, None, 16, st), INVALID, "bf16_to_f32 null out")
    rejects(L.mdb_timestep_embedding(None, 2, 320, 1, 0.0, op, st), INVALID, "timestep null t")
    rejects(L.mdb_timestep_embedding(p, 2, 320, 1, 0.0, None, st), INVALID, "timestep null out")
    rejects(L.mdb_fourier_embed(None, 4, 3, 4, op, st), INVALID, "fourier null x")
    rejects(L.mdb_fourier_embed(p, 4, 3, 4, None, st), INVALID, "fourier null out")
    rejects(L.mdb_linear_small(p, 4, 3201, 3201, p, 3201, None, 8, 0, 0, op, 8, st), UNSUPPORTED, "linear_small k = 3201")
    rejects(L.mdb_linear_small(None, 4, 8, 8, p, 8, None, 8, 0, 0, op, 8, st), INVALID, "linear_small null in")
    rejects(L.mdb_linear_small(p, 4, 8, 8, None, 8, None, 8, 0, 0, op, 8, st), INVALID, "linear_small null w")
    rejects(L.mdb_linear_small(p, 4, 8, 8, p, 8, None, 8, 0, 0, None, 8, st), INVALID, "linear_small null out")
    rejects(L.mdb_pack_latents(p, 1, 16, 4, 3, 1, o16p, st), INVALID, "pack_latents cpad < cin")
    rejects(L.mdb_pack_latents(p, 1, 16, 4, 64, 0, o16p, st), INVALID, "pack_latents repeat 0")
    rejects(L.mdb_pack_latents(None, 1, 16, 4, 64, 1, o16p, st), INVALID, "pack_latents null x")
    # in-place operators: the latents / dst buffers are the guarded outputs
    lat = _inplace(torch.ones(64, 4, device="cuda"))
    hist = [_inplace(torch.ones(64, 4, device="cuda")) for _ in range(3)]
    bits = [t.buf.clone() for t in [lat] + hist]

    def unchanged(what):
        torch.cuda.synchronize()
        for t, b in zip([lat] + hist, bits):
            assert torch.equal(t.buf.view(torch.int32), b.view(torch.int32)), what

    lp, hp = lat.out.data_ptr(), [h.out.data_ptr() for h in hist]
    for eps_ld, c, n, what in ((3, 4, 256, "eps_ld < c"), (8, 4, 254, "n % c"), (8, 0, 256, "c = 0")):
        assert L.mdb_cfg_ddim_step(p, eps_ld, c, 1, 2.0, p, lp, n, st) == INVALID, "ddim " + what
        unchanged("ddim " + what)
        assert L.mdb_cfg_unipc_step(p, eps_ld, c, 1, 2.0, p, lp, *hp, n, st) == INVALID, "unipc " + what
        unchanged("unipc " + what)
    assert L.mdb_cfg_ddim_step(None, 8, 4, 1, 2.0, p, lp, 256, st) == INVALID
    assert L.mdb_cfg_ddim_step(p, 8, 4, 1, 2.0, None, lp, 256, st) == INVALID
    for i in range(3):
        ptrs = list(hp)
        ptrs[i] = None
        assert L.mdb_cfg_unipc_step(p, 8, 4, 1, 2.0, p, lp, *ptrs, 256, st) == INVALID
    assert L.mdb_cfg_unipc_step(p, 8, 4, 1, 2.0, p, None, *hp, 256, st) == INVALID
    mask = torch.ones(4, dtype=I32, device="cuda")
    mp = mask.data_ptr()
    for args, what in (((lp, 3, p, p, 4, p, mp, 16, 4), "dst_ld < c"), ((lp, 4, p, p, 0, p, mp, 16, 4), "c = 0"),
                       ((lp, 4, p, p, 4, p, mp, 0, 4), "rows_per_view = 0"), ((lp, 4, p, p, 4, p, mp, 16, 0), "n_views = 0"),
                       ((None, 4, p, p, 4, p, mp, 16, 4), "null dst"), ((lp, 4, p, None, 4, p, mp, 16, 4), "null b"),
                       ((lp, 4, p, p, 4, None, mp, 16, 4), "null coef"), ((lp, 4, p, p, 4, p, None, 16, 4), "null mask")):
        assert L.mdb_pin_views(*args, st) == INVALID, "pin_views " + what
        unchanged("pin_views " + what)
    # input preparation
    off = torch.tensor([0, 2], dtype=I32, device="cuda")
    lab = torch.zeros(2, dtype=I64, device="cuda")
    ob, oc, om, cnt = Guarded(24, 24, F32), Guarded(6, 4, I64), Guarded(6, 4, U8), Guarded(1, 6, I32)
    outs = (ob.out.data_ptr(), oc.out.data_ptr(), om.out.data_ptr(), cnt.out.data_ptr())
    good = [p, 9, lab.data_ptr(), off.data_ptr(), 1, p, None, 6, 4, *outs]
    for i, v, what in ((1, 6, "box_dim 6"), (4, 0, "no scenes"), (7, 0, "no views"), (8, 0, "capacity 0"),
                       (0, None, "null boxes"), (2, None, "null labels"), (3, None, "null offsets"), (5, None, "null lidar2camera"),
                       (9, None, "null out_boxes"), (10, None, "null out_classes"), (11, None, "null out_masks"),
                       (12, None, "null out_counts")):
        args = list(good)
        args[i] = v
        rejects(L.mdb_prepare_boxes(*args, st), INVALID, "prepare_boxes " + what, ob, oc, om, cnt)
    rejects(L.mdb_camera_param(p, p, 0, op, st), INVALID, "camera_param n = 0")
    rejects(L.mdb_camera_param(None, p, 1, op, st), INVALID, "camera_param null intrinsics")
    rejects(L.mdb_camera_param(p, None, 1, op, st), INVALID, "camera_param null lidar2camera")
    rejects(L.mdb_camera_param(p, p, 1, None, st), INVALID, "camera_param null out")


# ------------------------------------------------------------------------------------------------------ PDL on vs off
def _pdl_chain(monkeypatch):
    """One chain over the kernels that launch with programmatic dependent launch, with add / upsample_nearest (launched
    without it) placed between them in both orders; returns every output."""
    g = _gen(14)
    n, h, w, c, heads, d = 2, 14, 25, 320, 8, 40
    m = n * h * w
    x = _bf(torch.randn(m, c, device="cuda", generator=g))
    w1 = _bf(torch.randn(c, c, device="cuda", generator=g) / math.sqrt(c))
    b1 = torch.randn(c, device="cuda", generator=g)
    gamma, beta = 1 + 0.1 * torch.randn(c, device="cuda", generator=g), 0.1 * torch.randn(c, device="cuda", generator=g)
    w2 = torch.randn(c, c, device="cuda", generator=g) / math.sqrt(c)
    w2g = _bf(w2 * gamma)
    colsum, c2 = w2g.float().sum(1), w2 @ beta
    w3 = _bf(torch.randn(c, 4 * c, device="cuda", generator=g) / math.sqrt(4 * c))
    ids = torch.randint(0, 1000, (2, 77), device="cuda", generator=g, dtype=I32)
    tok, pos = _bf(torch.randn(1000, c, device="cuda", generator=g)), _bf(torch.randn(77, c, device="cuda", generator=g))
    outs = []
    y, st = ops.linear(x, w1, bias=b1, residual=x, emit_stats=True)                  # GEMM writing row statistics
    z = ops.linear(y, w2g, bias=c2, ln=st, ln_colsum=colsum)                          # folded LayerNorm GEMM
    s = ops.add(z, y)                                                                 # PDL -> add -> upsample -> PDL
    u = ops.upsample_nearest(s, n, h, w, c, 2 * h, 2 * w)
    monkeypatch.setenv("MDB_GN_ROWS", "0")
    g1 = ops.groupnorm(u, c, c, n, 4 * h * w, gamma, beta, 1e-5, True)                # gn_fused<true>
    monkeypatch.setenv("MDB_GN_ROWS", "1")
    g2 = ops.groupnorm(g1, c, c, n, 4 * h * w, gamma, beta, 1e-5, False)              # gn_rows
    monkeypatch.delenv("MDB_GN_ROWS")
    u2 = ops.upsample_nearest(z, n, h, w, c, 2 * h, 2 * w)                            # PDL -> upsample -> add -> PDL
    s2 = ops.add(u2, g2)
    a = ops.attention(s2, s2, s2, b=n, heads=heads, lq=4 * h * w, lk=4 * h * w, d=d, ldq=c, ldk=c, ldv=c, scale=d ** -0.5)
    ln = ops.layernorm(a, gamma, beta)
    sk = ops.linear(ln.view(m, 4 * c), w3, bias=b1, force_splits=4)                  # split-K + finalize
    e, est = ops.clip_embed(ids, tok, pos)
    f = ops.linear(e, w2g, bias=c2, ln=est, ln_colsum=colsum)
    ca = ops.attention_causal(f, f, f, b=2, heads=heads, l=77, d=d, ldq=c, ldk=c, ldv=c, scale=d ** -0.5)
    outs += [y, st.data, z, s, u, g1, g2, u2, s2, a, ln, sk, e, est.data, f, ca]
    torch.cuda.synchronize()
    return outs


def test_pdl_on_matches_pdl_off_bitwise(cuda_lib, monkeypatch):
    """Every kernel launched with PDL executes griddepcontrol.wait before it touches global memory; a missing wait shows up
    as a race against its predecessor.  One run each way: a pass is evidence, not proof."""
    if "MDB_PDL" in os.environ:
        pytest.skip("MDB_PDL in the environment overrides mdb_set_pdl for the whole process")
    with ops.pdl_region(False):
        off = _pdl_chain(monkeypatch)
    with ops.pdl_region(True):
        assert cuda_lib.mdb_set_pdl(1) == 1  # the region switched it on
        on = _pdl_chain(monkeypatch)
    assert cuda_lib.mdb_set_pdl(0) == 0
    for i, (a, b) in enumerate(zip(off, on)):
        it = _BITS[a.dtype]
        assert torch.equal(a.view(it), b.view(it)), f"output {i} differs with PDL on"


@torch.no_grad()
def test_pdl_decoder_pipeline_bitwise(cuda_lib, monkeypatch):
    """The tiny three-step CFG pipeline with the UNet up path under PDL (MDB_PDL_DECODER=1) against the same with it off."""
    if "MDB_PDL" in os.environ:
        pytest.skip("MDB_PDL in the environment overrides mdb_set_pdl for the whole process")
    from magicdrive_b200.models import BEVControlNetModel, UNet2DConditionModelMultiview
    from magicdrive_b200.pipeline import BEVControlNetDenoiser
    from tests.common import golden, tiny_configs, tiny_state_dicts
    gd = golden("tiny_pipeline.pt")
    ucfg, ccfg = tiny_configs()
    usd, csd = tiny_state_dicts(gd["seed"])
    inp = gd["inputs"]
    outs = []
    for flag in ("0", "1"):
        monkeypatch.setenv("MDB_PDL_DECODER", flag)
        un, cn = UNet2DConditionModelMultiview(**asdict(ucfg)), BEVControlNetModel(**asdict(ccfg))
        un.load_state_dict(usd)
        cn.load_state_dict(csd)
        pipe = BEVControlNetDenoiser(un.to("cuda"), cn.to("cuda"), use_cuda_graph=True)
        assert pipe.pdl_decoder == (flag == "1")
        outs.append(pipe(image=inp["bev_map"], camera_param=inp["camera_param"], prompt_embeds=inp["prompt_embeds"],
                         negative_prompt_embeds=inp["negative_prompt_embeds"], latents=inp["latents"],
                         num_inference_steps=gd["steps"], guidance_scale=gd["guidance"],
                         bev_controlnet_kwargs={"bboxes_3d_data": inp["bboxes_3d_data"]}))
    _same(outs[1], outs[0], "MDB_PDL_DECODER=1 against 0")


# ------------------------------------------------------------------------------------------------------ emulator vs kernels
def test_ops_emulator_agrees_with_the_kernels(cuda_lib, monkeypatch):
    """tests/ops_emulator.py (the CPU restatement the host tests run on) against the kernels, with its bf16 rounding of
    activations on, for every operator of this file it restates and one case per semantic of the GEMM, attention and FID /
    text-encoder operators: bitwise where the kernel is exact, else within the operator's bound above, one bf16 rounding
    step for the GEMM (test_kernel_edges_gpu._close) and xformers' bf16 tolerance for attention."""
    from tests import ops_emulator as E
    monkeypatch.setattr(E, "ROUND_ACTIVATIONS", True)
    g = _gen(15)
    cpu = lambda t: None if t is None else t.cpu()  # noqa: E731
    assert {"add", "upsample_nearest", "nchw_to_nhwc", "nhwc_to_nchw", "f32_to_bf16", "pack_latents", "cfg_ddim_step",
            "cfg_unipc_step", "pin_views", "timestep_embedding", "fourier_embed", "linear_small", "gemm_conv", "attention",
            "attention_multi", "attention_causal", "pool2d", "fid_input", "clip_embed"} <= set(E.EMULATED)

    def same(dev, emu, what):
        _same(dev.cpu().to(emu.dtype).reshape(emu.shape), emu, f"emulator {what}")

    a, b = _bf(torch.randn(700, 320, device="cuda", generator=g)), _bf(torch.randn(700, 320, device="cuda", generator=g))
    same(ops.add(a, b), E.add(cpu(a), cpu(b)), "add")
    for (n, h, w, c, ho, wo) in UPSAMPLE[:3] + UPSAMPLE[-3:]:
        x = _bf(torch.randn(n * h * w, c, device="cuda", generator=g))
        same(ops.upsample_nearest(x, n, h, w, c, ho, wo), E.upsample_nearest(cpu(x), n, h, w, c, ho, wo), f"upsample {h}x{w}")
    for dt in (F32, BF16):
        x = torch.randn(3, 33, 5, 7, device="cuda", generator=g).to(dt)
        same(ops.nchw_to_nhwc(x), E.nchw_to_nhwc(cpu(x)), "nchw_to_nhwc")
        xh = _bf(torch.randn(3 * 35, 33, device="cuda", generator=g))
        same(ops.nhwc_to_nchw(xh, 3, 33, 5, 7, dt), E.nhwc_to_nchw(cpu(xh), 3, 33, 5, 7, dt), "nhwc_to_nchw")
        xl = torch.randn(1001, 4, device="cuda", generator=g).to(dt)
        same(ops.pack_latents(xl, 64, 2), E.pack_latents(cpu(xl), 64, 2), "pack_latents")
    xf = torch.randn(5000, device="cuda", generator=g) * 1e3
    same(ops.f32_to_bf16(xf), E.f32_to_bf16(cpu(xf)), "f32_to_bf16")

    # guidance + scheduler updates and pin_views: within 2^-21 * sum|terms|
    npix, c = 6 * 10 * 13, 4
    eps = torch.randn(2 * npix, 8, device="cuda", generator=g)
    lat = torch.randn(npix, c, device="cuda", generator=g) * 5
    coef = torch.tensor([1.0123, -0.2345], device="cuda")
    dev, emu = ops.cfg_ddim_step(eps, lat.clone(), coef, True, 7.5, c), E.cfg_ddim_step(cpu(eps), cpu(lat), cpu(coef), True, 7.5, c)
    e, ea = _combine(eps[:npix, :c].to(F64), eps[npix:, :c].to(F64), True, 7.5)
    _within("emulator cfg_ddim_step", emu, dev.cpu().to(F64), (2.0 ** -21 * (1.0123 * lat.to(F64).abs() + 0.2345 * ea)).cpu(), "ddim")
    uc = torch.tensor([0.9, -0.4, 0.3, 0.5, -0.2, 0.4, 1.1, -0.3, 0.2, 1.0, 0, 0], device="cuda")
    st = [torch.randn(npix, c, device="cuda", generator=g) for _ in range(3)]
    dstate = [lat.clone()] + [t.clone() for t in st]
    estate = [cpu(lat).clone()] + [cpu(t).clone() for t in st]
    ref = _unipc_ref(uc.to(F64).tolist(), *(t.to(F64) for t in [lat] + st), eps[:npix, :c].to(F64), eps[npix:, :c].to(F64),
                     True, 2.5)
    ops.cfg_unipc_step(eps, *dstate, uc, True, 2.5, c)
    E.cfg_unipc_step(cpu(eps), *estate, cpu(uc), True, 2.5, c)
    for name, dv, ev in zip(("latents", "last", "m0"), dstate, estate):
        _within("emulator cfg_unipc_step", ev, dv.cpu().to(F64), ref[name][1].cpu(), f"unipc {name}")
    _same(estate[3], dstate[3].cpu(), "emulator unipc m1")
    mask = torch.tensor([1, 0, 1, 1, 0, 0], dtype=I32, device="cuda")
    dst = torch.randn(6 * 130, 8, device="cuda", generator=g)
    pa, pb = torch.randn(6 * 130, c, device="cuda", generator=g), torch.randn(6 * 130, c, device="cuda", generator=g)
    pc = torch.tensor([0.7316, -1.2904], device="cuda")
    dv = ops.pin_views(dst.clone(), pa, pb, pc, mask, 130, c)
    ev = E.pin_views(cpu(dst).clone(), cpu(pa), cpu(pb), cpu(pc), cpu(mask), 130, c)
    pbound = 2.0 ** -21 * (0.7316 * F.pad(pa.abs(), (0, 4)) + 1.2904 * F.pad(pb.abs(), (0, 4))).to(F64).cpu()
    _within("emulator pin_views", ev, dv.cpu().to(F64), pbound, "pin_views")

    # embeddings: within 2^-21 * max(1, |arg|); linear_small within 2^-20 * (sum|h w| + |b|)
    t = torch.tensor([0.0, 1.0, 500.0, 981.0, 999.0], device="cuda")
    for dim, flip, shift in ((320, True, 0.0), (320, False, 1.0)):
        arg = t.to(F64)[:, None] * torch.exp(-math.log(10000.0) * torch.arange(dim // 2, dtype=F64, device="cuda") /
                                            (dim // 2 - shift))
        _within("emulator timestep_embedding", E.timestep_embedding(cpu(t), dim, flip, shift),
                ops.timestep_embedding(t, dim, flip, shift).cpu().to(F64), 2.0 ** -21 * arg.abs().clamp_min(1).repeat(1, 2).cpu(),
                f"timestep dim {dim}")
    xs = torch.rand(300, 3, device="cuda", generator=g) * 120 - 60
    fb = torch.cat([torch.ones_like(xs)] + [(xs * 2.0 ** k).abs().clamp_min(1).to(F32) for k in range(4) for _ in (0, 1)], -1)
    _within("emulator fourier_embed", E.fourier_embed(cpu(xs), 4), ops.fourier_embed(xs, 4).cpu().to(F64),
            2.0 ** -21 * fb.to(F64).cpu(), "fourier")
    h = torch.randn(37, 189, device="cuda", generator=g)
    wl = _bf(torch.randn(768, 189, device="cuda", generator=g) / math.sqrt(189))
    bl = torch.randn(768, device="cuda", generator=g)
    _, bound = _linear_small_ref(h, wl, bl, True, True)
    _within("emulator linear_small", E.linear_small(cpu(h), cpu(wl), cpu(bl), True, True),
            ops.linear_small(h, wl, bl, True, True).cpu().to(F64), bound.cpu(), "linear_small")

    # gemm_conv: two sources with K tails (80 + 40 channels), a 1x7 filter and ReLU into a column slice; end padding
    from magicdrive_b200.params import pack_conv_weight_k64
    x0, x1 = _bf(torch.randn(2 * 9 * 11, 88, device="cuda", generator=g)), _bf(torch.randn(2 * 9 * 11, 40, device="cuda", generator=g))
    wk = pack_conv_weight_k64(torch.randn(64, 120, 1, 7, device="cuda", generator=g) / math.sqrt(840), [80, 40])
    bk = torch.randn(64, device="cuda", generator=g)
    conv = dict(n_img=2, h_in=9, w_in=11, c0=80, lda0=88, c1=40, lda1=40, n_out=64, taps_h=1, taps_w=7, pad_h=0, pad_w=3,
                relu=True)
    dev = ops.gemm_conv(x0, wk, a1=x1, bias=bk, out=torch.zeros(198, 80, dtype=BF16, device="cuda")[:, 8:72], ldo=80, **conv)
    emu = E.gemm_conv(cpu(x0), cpu(wk), a1=cpu(x1), bias=cpu(bk), out=torch.zeros(198, 80)[:, 8:72], ldo=80, **conv)
    _close(dev, emu.cuda(), "emulator gemm_conv 1x7 two sources relu")
    xe = _bf(torch.randn(2 * 13 * 17, 64, device="cuda", generator=g))
    we = pack_conv_weight_k64(torch.randn(96, 64, 3, 3, device="cuda", generator=g) / 24)
    conv = dict(n_img=2, h_in=13, w_in=17, c0=64, lda0=64, n_out=96, taps=3, stride=2, pad=0, pad_h_end=1, pad_w_end=1)
    be = torch.randn(96, device="cuda", generator=g)
    _close(ops.gemm_conv(xe, we, bias=be, **conv), E.gemm_conv(cpu(xe), cpu(we), bias=cpu(be), **conv).cuda(),
           "emulator gemm_conv end padding")
    # row statistics of an fp32 producer (bias + residual), then a folded LayerNorm with quick-GELU reading them
    m, k, n = 300, 320, 320
    xa, res = _bf(torch.randn(m, k, device="cuda", generator=g)), _bf(torch.randn(m, n, device="cuda", generator=g) + 16)
    wp, bp = _bf(torch.randn(n, k, device="cuda", generator=g) / math.sqrt(k)), torch.randn(n, device="cuda", generator=g)
    prod = dict(n_img=1, h_in=1, w_in=m, c0=k, lda0=k, n_out=n, ldr=n, out_f32=True, emit_stats=True)
    dx, dst_ = ops.gemm_conv(xa, wp, bias=bp, residual=res, **prod)
    ex, est = E.gemm_conv(cpu(xa), cpu(wp), bias=cpu(bp), residual=cpu(res), **prod)
    _close_f32(dx, ex.cuda(), "emulator gemm_conv fp32 producer")
    stored = dx.to(F64)
    bound = 3e-5 * torch.stack([stored.abs().sum(1), (stored * stored).sum(1)], -1)
    _within("emulator gemm_conv row statistics", est.data.sum(1).cuda(), dst_.data.sum(1).to(F64), bound, "row statistics")
    xb, wg = _bf(dx), _bf(torch.randn(512, n, device="cuda", generator=g) / math.sqrt(n))
    cs, cb = wg.float().sum(1), torch.randn(512, device="cuda", generator=g)
    cons = dict(n_img=1, h_in=1, w_in=m, c0=n, lda0=n, n_out=512, ln_eps=1e-5, quick_gelu=True)
    _close(ops.gemm_conv(xb, wg, bias=cb, ln=dst_, ln_colsum=cs, **cons),
           E.gemm_conv(cpu(xb), cpu(wg), bias=cpu(cb), ln=ops.RowStats(cpu(dst_.data), dst_.parts), ln_colsum=cpu(cs),
                       **cons).cuda(), "emulator gemm_conv folded LayerNorm + quick-GELU")

    # attention: an empty slot and per-batch key counts (one batch without keys); two K/V sources; causal
    heads, d, lq, lk = 2, 64, 70, 90
    c = heads * d
    q = _bf(torch.randn(3 * lq, c, device="cuda", generator=g))
    kv = _bf(torch.randn(4 * lk, 2 * c, device="cuda", generator=g))
    kv2 = _bf(torch.randn(2 * lk, 2 * c, device="cuda", generator=g))
    idx = torch.tensor([[0, -1], [-1, 2], [3, 1]], dtype=I32, device="cuda")
    kv_len = torch.tensor([90, 37, 0], dtype=I32, device="cuda")
    att = dict(b=3, heads=heads, lq=lq, lk=lk, d=d, ldq=c, scale=d ** -0.5, n_sets=2)
    dev = ops.attention(q, kv[:, :c], kv[:, c:], b_kv=4, ldk=2 * c, ldv=2 * c, kv_index=idx, kv_len=kv_len, **att)
    emu = E.attention(cpu(q), cpu(kv)[:, :c], cpu(kv)[:, c:], b_kv=4, ldk=2 * c, ldv=2 * c, kv_index=cpu(idx),
                      kv_len=cpu(kv_len), **att)
    _attn_close(dev, emu.cuda().to(F64), 2)
    assert not dev[2 * lq:].any() and not emu[2 * lq:].any()
    idx2 = torch.tensor([[1 << 24, 3], [2, (1 << 24) | 1], [-1, 1 << 24]], dtype=I32, device="cuda")
    srcs = lambda t, t2: [(t[:, :c], t[:, c:], 2 * c, 4), (t2[:, :c], t2[:, c:], 2 * c, 2)]  # noqa: E731
    dev = ops.attention_multi(q, srcs(kv, kv2), kv_index=idx2, **att)
    _attn_close(dev, E.attention_multi(cpu(q), srcs(cpu(kv), cpu(kv2)), kv_index=cpu(idx2), **att).cuda().to(F64), 2)
    qkv = _bf(torch.randn(2 * 77, 3 * c, device="cuda", generator=g))
    causal = dict(b=2, heads=heads, l=77, d=d, ldq=3 * c, ldk=3 * c, ldv=3 * c, scale=d ** -0.5)
    dev = ops.attention_causal(qkv[:, :c], qkv[:, c:2 * c], qkv[:, 2 * c:], **causal)
    qc = cpu(qkv)
    _attn_close(dev, E.attention_causal(qc[:, :c], qc[:, c:2 * c], qc[:, 2 * c:], **causal).cuda().to(F64))

    # FID pools (max bitwise) and input step; CLIP embedding (bitwise, statistics within 3e-5 * sum|x|, sum x^2)
    xp = _bf(torch.randn(2 * 17 * 17, 96, device="cuda", generator=g))
    pool = dict(n=2, h=17, w=17, c=80, ldx=96)
    for mode, k_, s_, p_ in ((ops.POOL_MAX, 3, 2, 0), (ops.POOL_AVG, 3, 1, 1), (ops.POOL_GLOBAL_AVG, 3, 1, 0)):
        dev, emu = ops.pool2d(xp, mode=mode, k=k_, stride=s_, pad=p_, **pool), E.pool2d(cpu(xp), mode=mode, k=k_, stride=s_, pad=p_, **pool)
        if mode == ops.POOL_MAX:
            same(dev, emu, "pool2d max")
        else:
            _close(dev, emu.cuda(), f"emulator pool2d mode {mode}")
    img = torch.rand(2, 3, 60, 90, device="cuda", generator=g)
    dev = ops.fid_input(img, nhwc=False, quantize=True, normalize=True, size=(75, 97))
    emu = E.fid_input(cpu(img), nhwc=False, quantize=True, normalize=True, size=(75, 97))
    assert (dev.cpu().to(F64) - emu.to(F64)).abs().max().item() <= 2.0 ** -8 * emu.abs().max().item() + 1e-6
    tok, pos = _bf(torch.randn(500, 768, device="cuda", generator=g)), _bf(torch.randn(77, 768, device="cuda", generator=g))
    ids = torch.randint(0, 500, (2, 77), dtype=I32, device="cuda", generator=g)
    ids[1, 3] = 500  # outside the vocabulary: a NaN row
    (dx, dst_), (ex, est) = ops.clip_embed(ids, tok, pos), E.clip_embed(cpu(ids), cpu(tok), cpu(pos))
    same(dx, ex, "clip_embed")
    ok = ~dx.isnan().any(1)
    stored = dx[ok].to(F64)
    bound = 3e-5 * torch.stack([stored.abs().sum(1), (stored * stored).sum(1)], -1)
    _within("emulator clip_embed statistics", est.data[:, 0][ok.cpu()].cuda(), dst_.data[:, 0][ok].to(F64), bound, "clip_embed")
