"""Kernel parity at the launch shapes the engines issue and at the edges where tiled kernels go wrong: M / N tails, several
images per tile, split-K finalisation, strided inputs and outputs, multi-source attention, long sequences, every GroupNorm
kernel, the direct convolution and the adaptive pool.

The GEMM, attention and GroupNorm kernels have f16 twins (the denoising step of a model with fp16 parameters) that share
their bodies through Act<F16> (csrc/ptx.cuh); those tests take the element type `dt` (bf16 | f16, `with_dt`) and run both at
the same edges, the f16 cases under ids that start with "f16-".  The VAE decoder's GEMM launches run in both types too (an
fp16 VAE computes in f16); the direct convolution and the adaptive pool are bf16 / fp32 here (the f16 direct convolution is
test_vae_fp16_gpu.py's).

Every reference is computed in float64 on the GPU from the same bf16- (or f16-) rounded inputs.  Every output is written
into a larger buffer pre-filled with a NaN bit pattern: at least one full 128-row M tile of guard rows before and after the
output, and guard columns on both sides whenever the row stride exceeds the written width.  After each call every guard
element must be bitwise unchanged and no interior element may still hold the fill pattern."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from magicdrive_b200 import ops  # noqa: E402
from tests.attention_model import attention_model, check_model  # noqa: E402

BF16, F16, F32, F64 = torch.bfloat16, torch.float16, torch.float32, torch.float64
G = 128  # guard rows before and after every output: one full GEMM M tile
_FILL = {BF16: (torch.int16, 0x7FA5), F16: (torch.int16, 0x7E5A), F32: (torch.int32, 0x7FA5A5A5)}  # NaNs no kernel produces


# ---------------------------------------------------------------------------------------------------------- helpers
def with_dt(values, ids=None, f16=None):
    """pytest params (dt, *value) for the element types of the kernels with f16 twins: every value in bf16 under the id it
    has without `dt` (so the bf16 cases keep the ids they had before the f16 twins existed), then in f16 under "f16-" + that
    id, for every value or only those whose id is in `f16`."""
    values = [v if isinstance(v, tuple) else (v,) for v in values]
    ids = ids or ["-".join(str(x) for x in v) for v in values]
    return ([pytest.param(BF16, *v, id=i) for v, i in zip(values, ids)] +
            [pytest.param(F16, *v, id=f"f16-{i}") for v, i in zip(values, ids) if f16 is None or i in f16])


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _bf(x):
    return x.to(BF16)


def _randn(*shape, g, scale=1.0):
    return torch.randn(*shape, device="cuda", generator=g) * scale


class Guarded:
    """A [rows, cols] output at column `col0` of a [G + rows + G, ld] buffer filled with a NaN bit pattern."""

    def __init__(self, rows, cols, dtype=BF16, ld=None, col0=0, device="cuda"):
        self.rows, self.cols, self.col0, self.ld = rows, cols, col0, ld or cols
        assert col0 + cols <= self.ld
        self.itype, self.fill = _FILL[dtype]
        self.buf = torch.empty((rows + 2 * G, self.ld), dtype=dtype, device=device)
        self.buf.view(self.itype).fill_(self.fill)
        self.out = self.buf[G:G + rows, col0:col0 + cols]

    def check(self, what=""):
        if self.buf.is_cuda:
            torch.cuda.synchronize()
        bits = self.buf.view(self.itype)
        outside = torch.ones_like(bits, dtype=torch.bool)
        outside[G:G + self.rows, self.col0:self.col0 + self.cols] = False
        hit = ((bits != self.fill) & outside).nonzero()
        assert hit.shape[0] == 0, f"{what}: {hit.shape[0]} guard elements overwritten, first at (row, col) " \
                                  f"{(hit[0, 0].item() - G, hit[0, 1].item() - self.col0)} relative to the output"
        left = (self.out.view(self.itype) == self.fill).sum().item()
        assert left == 0, f"{what}: {left} output elements never written"


def _tol_bf16(ref, ref_max=None):
    """_close_bf16's elementwise tolerance for a float64 reference; ref_max = max |ref| over the whole output (default: over
    `ref`), so that an output checked in pieces is held to the tolerance of the whole."""
    return ref.abs() * 2.0 ** -7 + 2e-3 * (ref.abs().max() if ref_max is None else ref_max)


def _tol_f16(ref, ref_max=None):
    """_close_f16's elementwise tolerance: one f16 ulp of ref plus 1e-4 of max |ref| (ref_max as in _tol_bf16)."""
    ulp = torch.exp2(torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** -14))) - 10)
    return ulp + 1e-4 * (ref.abs().max() if ref_max is None else ref_max)


def _tol_f32(ref, ref_max=None):
    """_close_f32's tolerance, one value for every element: 3e-5 of max |ref| (ref_max as in _tol_bf16)."""
    return 3e-5 * (ref.abs().max() if ref_max is None else ref_max)


def _close_bf16(out, ref, what=""):
    """Every element within one bf16 rounding step of the reference plus accumulation-order slack (test_gemm_pair_gpu.py)."""
    ref = ref.to(F64)
    err = (out.to(F64) - ref).abs()
    tol = _tol_bf16(ref)
    bad = (err > tol).nonzero()
    assert bad.shape[0] == 0, f"{what}: {bad.shape[0]} elements off, first at {tuple(bad[0].tolist())}, " \
                              f"max err {err.max().item():.3e} (max |ref| {ref.abs().max().item():.3e})"


def _close_f16(out, ref, what=""):
    """Every element within one f16 ulp of the float64 reference (the ulp floored at 2^-24 in the subnormal range), plus 1e-4
    of the largest |ref| for the fp32 accumulation order.  Every f16 store rounds an fp32 value to nearest even (Act<true> in
    csrc/ptx.cuh), so a store at any coarser precision (bf16's 8 bits) fails it."""
    ref = ref.to(F64)
    err = (out.to(F64) - ref).abs()
    tol = _tol_f16(ref)
    bad = (err > tol).nonzero()
    assert bad.shape[0] == 0, f"{what}: {bad.shape[0]} elements off, first at {tuple(bad[0].tolist())}, " \
                              f"max err {err.max().item():.3e} (max |ref| {ref.abs().max().item():.3e})"


def _close_f32(out, ref, what=""):
    ref = ref.to(F64)
    err = (out.to(F64) - ref).abs()
    tol = _tol_f32(ref)
    bad = (err > tol).nonzero()
    assert bad.shape[0] == 0, f"{what}: {bad.shape[0]} elements off, first at {tuple(bad[0].tolist())}, " \
                              f"max err {err.max().item():.3e} (tolerance {tol.item():.3e})"


def _close(out, ref, what=""):
    {F32: _close_f32, BF16: _close_bf16, F16: _close_f16}[out.dtype](out, ref, what)


def _conv_ref(srcs, n, h, w, wmat, taps, stride=1, pad=0):
    """float64 convolution of NHWC [pixels, c] sources (channel-concatenated) with a [co, taps*taps*cin] (tap, channel)
    weight matrix -> [pixels_out, co]."""
    x = torch.cat([s.to(F64) for s in srcs], 1).view(n, h, w, -1).permute(0, 3, 1, 2)
    co, ci = wmat.shape[0], x.shape[1]
    wt = wmat.to(F64).view(co, taps, taps, ci).permute(0, 3, 1, 2)
    y = F.conv2d(x, wt, stride=stride, padding=pad)
    return y.permute(0, 2, 3, 1).reshape(-1, co)


def _kernels_launched(fn):
    """Names of the CUDA kernels `fn` launches."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return " | ".join(e.key for e in prof.key_averages())


# ----------------------------------------------------------------------------------------------- GEMM / implicit conv
VARIANTS = [0, 4]  # 0 = the planner's choice (split-K allowed), 4 = single CTAs without split-K
VARIANT_IDS = ["planner", "nosplit"]


def _run_conv(*, n, h, w, c0, co, taps=1, stride=1, pad=0, lda0=None, c1=0, bias=True, rowbias=None, residual=False,
              out_f32=False, out_scale=1.0, ldo=None, col0=0, variant=0, seed=0, a0=None, dt=BF16, **kw):
    """One guarded gemm_conv launch on random `dt` (bf16 | f16) operands, checked against float64; returns (Guarded, ref)."""
    g = _gen(seed)
    ho = (h + 2 * pad - taps) // stride + 1
    wo = (w + 2 * pad - taps) // stride + 1
    pix_in, pix = n * h * w, n * ho * wo
    lda0 = lda0 or c0
    if a0 is None:
        a0 = _randn(pix_in, lda0, g=g).to(dt)[:, :c0]
    a1 = _randn(pix_in, c1, g=g).to(dt) if c1 else None
    k = taps * taps * (c0 + c1)
    wm = _randn(co, k, g=g, scale=1 / math.sqrt(k)).to(dt)
    b = _randn(co, g=g) if bias else None
    rb = None
    if rowbias == "image":  # per-image shift, a column slice of a wider table (temb_all[:, off:off + cout])
        rb = _randn(n, co + 72, g=g)[:, 40:40 + co]
    elif rowbias == "shared":  # one row for every image
        rb = _randn(1, co, g=g)
    res = _randn(pix, co, g=g).to(dt) if residual else None
    out = Guarded(pix, co, F32 if out_f32 else dt, ld=ldo, col0=col0)
    ops.gemm_conv(a0, wm, n_img=n, h_in=h, w_in=w, c0=c0, lda0=lda0, a1=a1, c1=c1, lda1=c1, n_out=co, taps=taps,
                  stride=stride, pad=pad, bias=b, rowbias=rb, residual=res, ldr=co, out=out.out, ldo=out.ld,
                  out_f32=out_f32, out_scale=out_scale, kernel_variant=variant, **kw)
    ref = _conv_ref([a0] + ([a1] if c1 else []), n, h, w, wm, taps, stride, pad)
    if b is not None:
        ref = ref + b.to(F64)
    if rb is not None:
        ref = ref + rb.to(F64).repeat_interleave(ho * wo, 0) if rb.shape[0] > 1 else ref + rb.to(F64)
    ref = ref * out_scale
    if res is not None:
        ref = ref + res.to(F64)
    return out, ref


# (n, h, w, c0, co, taps, stride, pad, extras): launches of the UNet / ControlNet / VAE decoder at their real shapes
PRODUCT_CONVS = {
    # conv_in: latents zero-padded to one 64-wide K block per tap, + the BEV-map embedding as residual (ControlNet)
    "conv_in": (12, 28, 50, 64, 320, 3, 1, 1, dict(residual=True)),
    # conv_out: 8 padded output channels in fp32 (an N tail far below any block width)
    "conv_out": (12, 28, 50, 320, 8, 3, 1, 1, dict(out_f32=True)),
    # VAE decoder conv_out with the image / 2 + 0.5 epilogue scale
    "vae_conv_out": (1, 224, 400, 128, 8, 3, 1, 1, dict(out_f32=True, out_scale=0.5)),
    "vae_mid_conv": (6, 28, 50, 512, 512, 3, 1, 1, dict(residual=True)),
    "vae_up_56x100": (6, 56, 100, 512, 512, 3, 1, 1, {}),
    "vae_conv1_112x200": (2, 112, 200, 512, 256, 3, 1, 1, {}),
    "vae_shortcut_112x200": (2, 112, 200, 512, 256, 1, 1, 0, {}),
    "vae_conv2_224x400": (2, 224, 400, 128, 128, 3, 1, 1, dict(residual=True)),
    "vae_shortcut_224x400": (1, 224, 400, 256, 128, 1, 1, 0, {}),
    "downsample_s2": (12, 28, 50, 320, 320, 3, 2, 1, {}),
}
# all of them in both element types: the UNet / ControlNet, and the VAE decoder, which computes in f16 when its parameters
# are fp16 (AutoencoderKL.engine)
PRODUCT_F16 = ("conv_in", "conv_out", "vae_conv_out", "vae_mid_conv", "vae_up_56x100", "vae_conv1_112x200",
               "vae_shortcut_112x200", "vae_conv2_224x400", "vae_shortcut_224x400", "downsample_s2")


@pytest.mark.parametrize("variant", VARIANTS, ids=VARIANT_IDS)
@pytest.mark.parametrize("dt,case", with_dt(list(PRODUCT_CONVS), f16=PRODUCT_F16))
def test_gemm_product_convs(cuda_lib, dt, case, variant):
    n, h, w, c0, co, taps, stride, pad, extra = PRODUCT_CONVS[case]
    out, ref = _run_conv(n=n, h=h, w=w, c0=c0, co=co, taps=taps, stride=stride, pad=pad, variant=variant, seed=1, dt=dt,
                         **extra)
    out.check(case)
    _close(out.out, ref, case)


@pytest.mark.parametrize("dt,variant", with_dt(VARIANTS, ids=VARIANT_IDS))
def test_gemm_vae_attention(cuda_lib, dt, variant):
    """The three GEMMs of the VAE mid-block attention (engine.py VaeDecoderEngine._attention) for the second of two
    28x50 images: S = q k^T (fp32, n_out = ldo = lp), V^T = W_v X^T (n_out = lp) and O = P V + b_v (K = lp), in both
    element types (an fp16 VAE runs them in f16)."""
    g = _gen(2)
    n, L, C = 2, 1400, 512
    lp = (L + 63) // 64 * 64
    i = 1
    q = _randn(n * L, C, g=g).to(dt)
    kbuf = torch.zeros(n * L + lp - L, C, dtype=dt, device="cuda")
    kbuf[: n * L] = _randn(n * L, C, g=g).to(dt)
    s = Guarded(L, lp, F32)
    ops.linear(q[i * L:(i + 1) * L], kbuf[i * L: i * L + lp], out_f32=True, out_scale=C ** -0.5, out=s.out, ldo=lp,
               kernel_variant=variant)
    s.check("scores")
    _close_f32(s.out, (q[i * L:(i + 1) * L].to(F64) @ kbuf[i * L: i * L + lp].to(F64).t()) * C ** -0.5, "scores")
    wv = _randn(C, C, g=g, scale=C ** -0.5).to(dt)
    t = _randn(n * L + lp - L, C, g=g).to(dt)
    vt = Guarded(C, lp, dt)
    ops.linear(wv, t[i * L: i * L + lp], out=vt.out, ldo=lp, kernel_variant=variant)
    vt.check("V^T")
    _close(vt.out, wv.to(F64) @ t[i * L: i * L + lp].to(F64).t(), "V^T")
    p = torch.softmax(_randn(L, lp, g=g, scale=3.0), -1).to(dt)
    bv = _randn(C, g=g)
    o = Guarded(L, C, dt)
    ops.linear(p, vt.out, bias=bv, out=o.out, ldo=C, kernel_variant=variant)
    o.check("P V")
    _close(o.out, p.to(F64) @ vt.out.to(F64).t() + bv.to(F64), "P V")


# (n, h, w, taps, stride): pixel counts 128k - 1, 128k + 1 and < 128, and last tiles that span several images
M_TAILS = [
    (1, 1, 127, 1, 1), (1, 1, 129, 1, 1), (3, 5, 17, 1, 1), (1, 1, 1025, 1, 1), (2, 5, 9, 1, 1), (13, 3, 13, 1, 1),
    (3, 5, 17, 3, 1), (1, 3, 43, 3, 1), (2, 5, 9, 3, 1), (7, 4, 7, 3, 1), (13, 3, 13, 3, 1), (1, 1, 257, 3, 1),
    (3, 9, 19, 3, 2), (5, 4, 7, 3, 2),
]


@pytest.mark.parametrize("variant", VARIANTS, ids=VARIANT_IDS)
@pytest.mark.parametrize("dt,n,h,w,taps,stride", with_dt(M_TAILS))
def test_gemm_m_tails(cuda_lib, dt, n, h, w, taps, stride, variant):
    pad = taps // 2
    out, ref = _run_conv(n=n, h=h, w=w, c0=128, co=192, taps=taps, stride=stride, pad=pad, rowbias="image",
                         residual=True, variant=variant, seed=3, dt=dt)
    out.check()
    _close(out.out, ref)


@pytest.mark.parametrize("variant", VARIANTS, ids=VARIANT_IDS)
@pytest.mark.parametrize("stats", [False, True], ids=["plain", "stats"])
@pytest.mark.parametrize("bn", [64, 128, 160, 256])
@pytest.mark.parametrize("dt,n_out", with_dt([8, 40, 136, 264, 520]))  # a tail past every block width
def test_gemm_n_tails(cuda_lib, dt, n_out, bn, stats, variant):
    g = _gen(4)
    m, k = 1000, 320
    x = _randn(m, k, g=g).to(dt)
    w = _randn(n_out, k, g=g, scale=1 / math.sqrt(k)).to(dt)
    b = _randn(n_out, g=g)
    r = _randn(m, n_out, g=g).to(dt)
    out = Guarded(m, n_out, dt)
    res = ops.linear(x, w, bias=b, residual=r, out=out.out, ldo=n_out, force_block_n=bn, kernel_variant=variant,
                     emit_stats=stats)
    out.check()
    ref = x.to(F64) @ w.to(F64).t() + b.to(F64) + r.to(F64)
    _close(out.out, ref)
    if stats:
        st = res[1]
        assert st.parts == (n_out + bn - 1) // bn and st.data.shape == (m, st.parts, 2)
        s = st.data.to(F64).sum(1)
        # the statistics are taken from the values as stored, after their rounding to bf16 / f16
        stored = out.out.to(F64)
        torch.testing.assert_close(s[:, 0], stored.sum(1), rtol=0, atol=2e-3)
        torch.testing.assert_close(s[:, 1], (stored ** 2).sum(1), rtol=1e-5, atol=2e-3)


@pytest.mark.parametrize("variant", VARIANTS, ids=VARIANT_IDS)
@pytest.mark.parametrize("rowbias", ["image", "shared"])
@pytest.mark.parametrize("dt,splits", with_dt([2, 3, 7]))
def test_gemm_split_k_epilogue(cuda_lib, dt, splits, rowbias, variant):
    """Split-K finalisation with the UNet resnet's epilogue: bf16 / f16 output + bias + time-embedding shift (per image, or
    one row for all) + scale + residual; the result is bitwise reproducible."""
    kw = dict(n=3, h=14, w=25, c0=640, co=640, taps=3, pad=1, rowbias=rowbias, residual=True, out_scale=0.75,
              force_splits=splits, variant=variant, seed=5, dt=dt)
    out, ref = _run_conv(**kw)
    out.check()
    _close(out.out, ref)
    again, _ = _run_conv(**kw)
    assert torch.equal(out.out.view(torch.int16), again.out.view(torch.int16))


@pytest.mark.parametrize("variant", VARIANTS, ids=VARIANT_IDS)
@pytest.mark.parametrize("dt,taps,stride", with_dt([(3, 1), (1, 1), (3, 2)]))
def test_gemm_strided_sources_and_output(cuda_lib, dt, taps, stride, variant):
    """Source 0 a channel slice of a wider buffer (lda0 > c0), a second concatenated source, output into a column slice."""
    out, ref = _run_conv(n=3, h=14, w=25, c0=320, lda0=448, c1=192, co=320, taps=taps, stride=stride, pad=taps // 2,
                         residual=True, ldo=512, col0=128, variant=variant, seed=6, dt=dt)
    out.check()
    _close(out.out, ref)


# ------------------------------------------------------------------------------------------------------ attention
ATTN_KERNELS = ["tc2", "tc2d", "tc"]  # key-tile width: per head dim (default) | 64 keys | 128 keys
# MDB_ATTN_KERNEL is a bf16 A/B switch: the f16 kernels have the default key-tile width only (capi_attention.cu)
ATTN_DT_KERNELS = with_dt(ATTN_KERNELS, f16=("tc2",))
HEADS = {32: 2, 40: 8, 64: 2, 80: 4, 160: 2}


def _attn_ref(q, kv_of, b, heads, lq, d, scale, n_sets=1, chunk=512, dt=BF16):
    """The float64 attention and its error model (tests/attention_model.py); kv_of(i, s) -> (k, v) [lk, >= heads*d] of
    query batch i, set s."""
    return attention_model(q, lambda i: [kv_of(i, s) for s in range(n_sets)], b, heads, lq, d, scale, dt, chunk=chunk)


def _attn_close(out, model):
    """Both criteria of the error model of the kernel's roundings (tests/attention_model.py)."""
    check_model(out, model)


def _kv_index(entries):
    return torch.tensor([[(s << 24) | j for s, j in row] for row in entries], dtype=torch.int32, device="cuda")


@pytest.mark.parametrize("n_sets", [1, 2])
@pytest.mark.parametrize("d", list(HEADS))
@pytest.mark.parametrize("dt,kernel", ATTN_DT_KERNELS)
def test_attention_multi_source(cuda_lib, monkeypatch, dt, kernel, d, n_sets):
    """K/V in three buffers (batch counts 6 / 3 / 3, row strides 2C / 2C / 3C), the view-sharded cross-view layout; kv_index
    entries (source << 24) | batch reach every source."""
    monkeypatch.setenv("MDB_ATTN_KERNEL", kernel)
    g = _gen(7)
    heads = HEADS[d]
    c = heads * d
    b, lq, lk = 4, 201, 333
    scale = d ** -0.5
    q = _randn(b * lq, c, g=g).to(dt)
    b0 = _randn(6 * lk, 2 * c, g=g).to(dt)
    b1 = _randn(3 * lk, 2 * c, g=g).to(dt)
    b2 = _randn(3 * lk, 3 * c, g=g).to(dt)
    srcs = [(b0[:, :c], b0[:, c:], 2 * c, 6), (b1[:, :c], b1[:, c:], 2 * c, 3), (b2[:, c:2 * c], b2[:, 2 * c:], 3 * c, 3)]
    if n_sets == 1:
        entries = [[(2, 1)], [(0, 5)], [(1, 2)], [(2, 0)]]
    else:
        entries = [[(0, 5), (2, 2)], [(1, 0), (0, 0)], [(2, 0), (1, 2)], [(0, 3), (2, 1)]]
    idx = _kv_index(entries)
    out = Guarded(b * lq, c, dt, ld=c + 16, col0=8)
    ops.attention_multi(q, srcs, b=b, heads=heads, lq=lq, lk=lk, d=d, ldq=c, scale=scale, kv_index=idx, n_sets=n_sets,
                        out=out.out)
    out.check("multi-source")

    def kv_of(i, s):
        src, j = entries[i][s]
        k, v = srcs[src][:2]
        return k[j * lk:(j + 1) * lk], v[j * lk:(j + 1) * lk]

    _attn_close(out.out, _attn_ref(q, kv_of, b, heads, lq, d, scale, n_sets, dt=dt))

    # entries that all name source 0: bit for bit the single-buffer call
    e0 = [[(0, (3 * i + s) % 6) for s in range(n_sets)] for i in range(b)]
    multi0 = Guarded(b * lq, c, dt)
    ops.attention_multi(q, srcs, b=b, heads=heads, lq=lq, lk=lk, d=d, ldq=c, scale=scale, kv_index=_kv_index(e0),
                        n_sets=n_sets, out=multi0.out)
    single0 = ops.attention(q, b0[:, :c], b0[:, c:], b=b, b_kv=6, heads=heads, lq=lq, lk=lk, d=d, ldq=c, ldk=2 * c,
                            ldv=2 * c, scale=scale, kv_index=_kv_index(e0), n_sets=n_sets)
    multi0.check("source 0")
    assert torch.equal(multi0.out, single0)

    # three sources that are row ranges of one buffer: bit for bit the single-source call on the whole buffer
    big = _randn(12 * lk, 2 * c, g=g).to(dt)
    first = [0, 6, 9]
    slices = [(big[f * lk:(f + nb) * lk, :c], big[f * lk:(f + nb) * lk, c:], 2 * c, nb) for f, nb in zip(first, [6, 3, 3])]
    split = Guarded(b * lq, c, dt)
    ops.attention_multi(q, slices, b=b, heads=heads, lq=lq, lk=lk, d=d, ldq=c, scale=scale, kv_index=idx, n_sets=n_sets,
                        out=split.out)
    flat = torch.tensor([[first[s] + j for s, j in row] for row in entries], dtype=torch.int32, device="cuda")
    whole = ops.attention(q, big[:, :c], big[:, c:], b=b, b_kv=12, heads=heads, lq=lq, lk=lk, d=d, ldq=c, ldk=2 * c,
                          ldv=2 * c, scale=scale, kv_index=flat, n_sets=n_sets)
    split.check("row-range sources")
    assert torch.equal(split.out, whole)


@pytest.mark.parametrize("d", [40, 64])
@pytest.mark.parametrize("dt,kernel", ATTN_DT_KERNELS)
def test_attention_kv_batches_differ(cuda_lib, monkeypatch, dt, kernel, d):
    """b_kv != b through kv_index with one set; queries read from a fused-QKV-style wide buffer."""
    monkeypatch.setenv("MDB_ATTN_KERNEL", kernel)
    g = _gen(8)
    heads = HEADS[d]
    c = heads * d
    b, b_kv, lq, lk = 5, 3, 333, 200
    qbuf = _randn(b * lq, 3 * c, g=g).to(dt)
    q = qbuf[:, c:2 * c]
    kv = _randn(b_kv * lk, 2 * c, g=g).to(dt)
    sel = [2, 0, 1, 1, 2]
    idx = torch.tensor(sel, dtype=torch.int32, device="cuda")[:, None].contiguous()
    out = Guarded(b * lq, c, dt, ld=c + 64, col0=32)
    ops.attention(q, kv, kv[:, c:], b=b, b_kv=b_kv, heads=heads, lq=lq, lk=lk, d=d, ldq=3 * c, ldk=2 * c, ldv=2 * c,
                  scale=d ** -0.5, kv_index=idx, out=out.out)
    out.check()
    ref = _attn_ref(q, lambda i, s: (kv[sel[i] * lk:(sel[i] + 1) * lk, :c], kv[sel[i] * lk:(sel[i] + 1) * lk, c:]),
                    b, heads, lq, d, d ** -0.5, dt=dt)
    _attn_close(out.out, ref)


def test_attention_multi_q_with_kv_index(cuda_lib, monkeypatch):
    """One K/V tile (lk <= 128) and more query tiles than SMs with kv_index and b_kv != b: multi-Q mode, against float64
    and bit for bit against one query tile per CTA."""
    _multi_q_with_kv_index(monkeypatch, BF16)


def test_attention_multi_q_with_kv_index_f16(cuda_lib, monkeypatch):
    """test_attention_multi_q_with_kv_index for the f16 kernels."""
    _multi_q_with_kv_index(monkeypatch, F16)


def _multi_q_with_kv_index(monkeypatch, dt):
    monkeypatch.delenv("MDB_ATTN_KERNEL", raising=False)
    g = _gen(9)
    b, b_kv, heads, d, lq, lk = 6, 2, 8, 40, 1400, 77
    c = heads * d
    assert b * heads * ((lq + 127) // 128) > torch.cuda.get_device_properties(0).multi_processor_count
    q = _randn(b * lq, c, g=g).to(dt)
    kv = _randn(b_kv * lk, 2 * c, g=g).to(dt)
    sel = [1, 0, 1, 1, 0, 0]
    idx = torch.tensor(sel, dtype=torch.int32, device="cuda")[:, None].contiguous()
    outs = []
    for multiq in ("1", "0"):
        monkeypatch.setenv("MDB_ATTN_MULTIQ", multiq)
        o = Guarded(b * lq, c, dt, ld=c + 8, col0=8)
        ops.attention(q, kv, kv[:, c:], b=b, b_kv=b_kv, heads=heads, lq=lq, lk=lk, d=d, ldq=c, ldk=2 * c, ldv=2 * c,
                      scale=d ** -0.5, kv_index=idx, out=o.out)
        o.check(f"MDB_ATTN_MULTIQ={multiq}")
        outs.append(o.out)
    ref = _attn_ref(q, lambda i, s: (kv[sel[i] * lk:(sel[i] + 1) * lk, :c], kv[sel[i] * lk:(sel[i] + 1) * lk, c:]),
                    b, heads, lq, d, d ** -0.5, dt=dt)
    _attn_close(outs[0], ref)
    assert torch.equal(outs[0], outs[1])


@pytest.mark.parametrize("dt,b,heads,d,l", with_dt([(2, 8, 40, 8400), (6, 8, 40, 5300)]))
def test_attention_long_self(cuda_lib, monkeypatch, dt, b, heads, d, l):
    """The 'self' cross-view mode: one attention over the tokens of all six views (6 x 1400 at 224x400), and the
    424x800 level's 5300-token self-attention; fused-QKV input, output into a column slice."""
    monkeypatch.delenv("MDB_ATTN_KERNEL", raising=False)
    g = _gen(10)
    c = heads * d
    qkv = _randn(b * l, 3 * c, g=g).to(dt)
    out = Guarded(b * l, c, dt, ld=c + 16, col0=8)
    ops.attention(qkv, qkv[:, c:], qkv[:, 2 * c:], b=b, heads=heads, lq=l, lk=l, d=d, ldq=3 * c, ldk=3 * c, ldv=3 * c,
                  scale=d ** -0.5, out=out.out)
    out.check()
    ref = _attn_ref(qkv, lambda i, s: (qkv[i * l:(i + 1) * l, c:2 * c], qkv[i * l:(i + 1) * l, 2 * c:]), b, heads, l, d,
                    d ** -0.5, dt=dt)
    _attn_close(out.out, ref)


# ------------------------------------------------------------------------------------------------------ GroupNorm
# (n, hw, c0, pad, c1): pad = extra row stride of source 0 (a channel slice); c1 = second concatenated source
GN_SLAB = {  # the slab kernels: one CTA per (image, group)
    "vae_224x400": (1, 89600, 128, 0, 0),
    "vae_112x200": (1, 22400, 256, 0, 0),
    "vae_56x100": (2, 5600, 512, 0, 0),
    "skip_1280+640": (2, 1400, 1280, 0, 640),
    "skip_1280+1280": (2, 1400, 1280, 0, 1280),
    "level_53x100": (2, 5300, 320, 0, 0),
    "ld0>c0": (2, 1400, 320, 64, 0),
    "skip_640+320": (3, 350, 640, 0, 320),
}
GN_ROWS = {  # the pixel-major cluster kernel
    "28x50_8cta": (2, 1400, 320, 0, 0),
    "ld0>c0": (2, 1400, 320, 64, 0),
    "4x7_skip_1280+1280": (3, 28, 1280, 0, 1280),
    "14x25_16cta": (2, 350, 1280, 0, 1280),  # only a 16-CTA cluster holds this image
}
GN_CASES = ([(f"fused-{k}", v, {"MDB_GN_ROWS": "0"}, "gn_fused_kernel") for k, v in GN_SLAB.items()] +
            [(f"two-{k}", v, {"MDB_GN_ROWS": "0", "MDB_GN_TWO_KERNEL": "1"}, "gn_stats_kernel") for k, v in GN_SLAB.items()] +
            [(f"rows-{k}", v, {"MDB_GN_ROWS": "1"}, "gn_rows_kernel") for k, v in GN_ROWS.items()] +
            [("rows16-28x50", (2, 1400, 320, 0, 0), {"MDB_GN_ROWS": "1", "MDB_GN_ROWS_CLUSTER": "16"}, "gn_rows_kernel"),
             ("rows16-14x25", (2, 350, 640, 0, 320), {"MDB_GN_ROWS": "1", "MDB_GN_ROWS_CLUSTER": "16"}, "gn_rows_kernel"),
             # three channels per group: only the statistics + apply pair takes odd groups
             ("odd-c96", (2, 1400, 96, 0, 0), {"MDB_GN_ROWS": "0"}, "gn_stats_kernel"),
             ("odd-c96-ld0>c0", (2, 1400, 96, 32, 0), {"MDB_GN_ROWS": "0"}, "gn_stats_kernel")])


GN_F16_NAMES = {"gn_rows_kernel": "gn_rows_f16_kernel", "gn_stats_kernel": "gn_stats_f16_kernel",
                "gn_fused_kernel": "gn_fused_kernel"}  # gn_fused_kernel is one template for both element types


@pytest.mark.parametrize("offset", [0, 16, 64, 256])
@pytest.mark.parametrize("dt,case,shape,env,kernel", with_dt(GN_CASES, ids=[c[0] for c in GN_CASES]))
def test_groupnorm_kernels(cuda_lib, monkeypatch, dt, case, shape, env, kernel, offset):
    """Each GroupNorm kernel, forced through its environment knobs, on inputs whose group means sit `offset` standard
    deviations away from zero; output into a column slice.  At 256 standard deviations a variance taken as
    E[x^2] - mean^2 in fp32 is off by several percent on these group sizes; at 64 the error still hides in the bf16 output.
    f16 (mdb_groupnorm_f16): one f16 ulp of float64 (_close_f16).  At 256 standard deviations the f16 inputs sit around 128,
    where their spacing is 1/8 of a standard deviation; the reference normalises the same stored values."""
    for k in ("MDB_GN_ROWS", "MDB_GN_ROWS_CLUSTER", "MDB_GN_TWO_KERNEL"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    n, hw, c0, pad, c1 = shape
    c, groups = c0 + c1, 32
    vae = case.split("-", 1)[1].startswith("vae")
    eps, silu = (1e-6, True) if vae else (1e-5, not case.endswith("ld0>c0"))
    g = _gen(11)
    sigma = 0.5
    chan = _randn(c, g=g, scale=0.25 * sigma)  # per-channel means around the offset

    def make(rows, cols, ch):
        return (_randn(rows, cols, g=g, scale=sigma) + offset * sigma + ch).to(dt)

    x0 = make(n * hw, c0 + pad, torch.cat([chan[:c0], torch.zeros(pad, device="cuda")]))[:, :c0]
    x1 = make(n * hw, c1, chan[c0:]) if c1 else None
    gamma = _randn(c, g=g)
    beta = _randn(c, g=g)
    out = Guarded(n * hw, c, dt, ld=c + 16, col0=8)
    stats = torch.empty(max(n, 160) * groups * 2, dtype=F32, device="cuda")
    fn = cuda_lib.mdb_groupnorm_f16 if dt == F16 else cuda_lib.mdb_groupnorm
    names = {k: GN_F16_NAMES[k] if dt == F16 else k for k in GN_F16_NAMES}

    def run():
        rc = fn(x0.data_ptr(), c0, c0 + pad, x1.data_ptr() if c1 else None, c1, c1, n, hw, groups, eps, gamma.data_ptr(),
                beta.data_ptr(), int(silu), out.out.data_ptr(), out.ld, stats.data_ptr(),
                torch.cuda.current_stream().cuda_stream)
        assert rc == 0, cuda_lib.mdb_last_error()

    # the profiler now and then drops a kernel's record: profile again when no GroupNorm kernel shows up at all
    for _ in range(3):
        launched = _kernels_launched(run)
        if any(k in launched for k in names.values()):
            break
    assert names[kernel] in launched, launched
    out.check(case)
    full = x0.to(F64) if x1 is None else torch.cat([x0.to(F64), x1.to(F64)], 1)
    ref = F.group_norm(full.view(n, hw, c).permute(0, 2, 1), groups, gamma.to(F64), beta.to(F64), eps)
    if silu:
        ref = F.silu(ref)
    _close(out.out, ref.permute(0, 2, 1).reshape(n * hw, c), case)


# ----------------------------------------------------------------------------------------- conv_direct, adaptive pool
# (n, h, w, cin, cout, k, stride, pad, silu, in_f32, out_f32, residual)
CONV_DIRECT = {
    "vae_post_quant": (6, 28, 50, 4, 4, 1, (1, 1), (0, 0), False, True, True, False),
    "vae_conv_in": (2, 28, 50, 4, 512, 3, (1, 1), (1, 1), False, True, False, False),
    # BEVControlNetConditioningEmbedding at a 200x200 map (arch.map_encoder_layers)
    "cond_conv_in": (1, 200, 200, 8, 16, 3, (1, 1), (1, 1), True, True, True, False),
    "cond_s2": (1, 200, 200, 16, 32, 3, (2, 2), (2, 1), True, True, True, False),
    "cond_96": (1, 52, 50, 96, 96, 3, (1, 1), (2, 1), True, True, True, False),
    "cond_s21": (1, 54, 50, 96, 256, 3, (2, 1), (2, 1), True, True, True, False),
    "cond_conv_out": (1, 28, 50, 256, 320, 3, (1, 1), (1, 1), False, True, False, False),
    "bf16_in": (2, 28, 50, 64, 32, 3, (2, 1), (2, 1), True, False, False, False),
    "residual_f32": (2, 25, 27, 32, 24, 3, (1, 1), (1, 1), True, True, True, True),
    "residual_bf16": (2, 28, 50, 4, 64, 3, (1, 1), (1, 1), False, True, False, True),
}


@pytest.mark.parametrize("case", list(CONV_DIRECT))
def test_conv_direct(cuda_lib, case):
    n, h, w, cin, cout, k, stride, pad, silu, in_f32, out_f32, with_res = CONV_DIRECT[case]
    g = _gen(12)
    x = _randn(n, h, w, cin, g=g)
    if not in_f32:
        x = _bf(x)
    wt = _randn(k, k, cin, cout, g=g, scale=1 / math.sqrt(k * k * cin))  # [kh][kw][cin][cout]
    b = _randn(cout, g=g)
    ho = (h + 2 * pad[0] - k) // stride[0] + 1
    wo = (w + 2 * pad[1] - k) // stride[1] + 1
    odt = F32 if out_f32 else BF16
    res = _randn(n * ho * wo, cout, g=g).to(odt) if with_res else None
    out = Guarded(n * ho * wo, cout, odt)
    rc = cuda_lib.mdb_conv_direct(x.data_ptr(), int(in_f32), n, h, w, cin, wt.data_ptr(), b.data_ptr(), cout, k, k,
                                  stride[0], stride[1], pad[0], pad[1], ho, wo, int(silu),
                                  res.data_ptr() if with_res else None, out.out.data_ptr(), int(out_f32),
                                  torch.cuda.current_stream().cuda_stream)
    assert rc == 0, cuda_lib.mdb_last_error()
    out.check(case)
    ref = F.conv2d(x.to(F64).permute(0, 3, 1, 2), wt.to(F64).permute(3, 2, 0, 1), b.to(F64), stride=stride, padding=pad)
    if silu:
        ref = F.silu(ref)
    ref = ref.permute(0, 2, 3, 1).reshape(n * ho * wo, cout)
    if with_res:
        ref = ref + res.to(F64)
    _close(out.out, ref, case)


@pytest.mark.parametrize("silu", [False, True])
@pytest.mark.parametrize("n,h,w,c,ho,wo", [
    (2, 13, 17, 24, 5, 7), (2, 7, 9, 24, 3, 13), (1, 4, 5, 8, 9, 11),  # non-divisible both ways; output larger than input
    (1, 50, 50, 96, 28, 50), (2, 50, 50, 96, 34, 92),  # the map embedder's pool onto the 224x400 / 272x736 latent grids
])
def test_adaptive_avgpool(cuda_lib, n, h, w, c, ho, wo, silu):
    g = _gen(13)
    x = _randn(n, h, w, c, g=g, scale=2.0)
    out = Guarded(n * ho * wo, c, F32)
    rc = cuda_lib.mdb_adaptive_avgpool(x.data_ptr(), n, h, w, c, out.out.data_ptr(), ho, wo, int(silu),
                                       torch.cuda.current_stream().cuda_stream)
    assert rc == 0, cuda_lib.mdb_last_error()
    out.check()
    ref = F.adaptive_avg_pool2d(x.to(F64).permute(0, 3, 1, 2), (ho, wo))
    if silu:
        ref = F.silu(ref)
    _close_f32(out.out, ref.permute(0, 2, 3, 1).reshape(n * ho * wo, c))
