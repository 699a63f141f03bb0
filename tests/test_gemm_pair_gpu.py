"""GPU parity of the wgmma GEMM / implicit-GEMM conv with bf16 output (bias / per-image shift / residual / scale, GEGLU,
row statistics, folded LayerNorm) against plain torch fp32 on the same bf16-rounded inputs.  kernel_variant 3 = CTA pairs
(2-CTA clusters sharing each weight tile through TMA multicast), 4 = the same kernel on single CTAs without split-K,
2 = single CTAs with split-K allowed (yardstick: all must agree with torch equally well)."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from magicdrive_b200 import ops  # noqa: E402
from magicdrive_b200.params import pack_geglu  # noqa: E402


def _bf(x):
    return x.to(torch.bfloat16)


def _rel(a, b):
    return ((a.float() - b.float()).abs().max() / (b.float().abs().max() + 1e-6)).item()


def _close_bf16(out, ref, what=""):
    """Every element within one bf16 rounding step of the fp32 reference (plus accumulation-order slack)."""
    err = (out.float() - ref.float()).abs()
    tol = ref.float().abs() * 2.0 ** -7 + 2e-3 * ref.float().abs().max()
    bad = (err > tol).sum().item()
    assert bad == 0, f"{what}: {bad} elements off, max err {err.max().item():.3e}, rel {_rel(out, ref):.3e}"


def _nhwc(x):
    n, c, h, w = x.shape
    return x.permute(0, 2, 3, 1).reshape(n * h * w, c).contiguous()


def _conv_weight(wt):
    co, ci, kh, kw = wt.shape
    return wt.permute(0, 2, 3, 1).reshape(co, kh * kw * ci).contiguous()


VARIANTS = [3, 4]
VARIANT_IDS = ["pair", "single"]


@pytest.mark.parametrize("variant", VARIANTS, ids=VARIANT_IDS)
@pytest.mark.parametrize("bn", [0, 64, 128, 160, 256])
@pytest.mark.parametrize("m,k,n", [(1000, 320, 320), (128, 64, 640), (336, 1280, 1280), (16800, 320, 960), (129, 128, 32),
                                   (4200, 640, 640)])
def test_gemm_plain(cuda_lib, bn, m, k, n, variant):
    g = torch.Generator(device="cuda").manual_seed(1)
    x = _bf(torch.randn(m, k, device="cuda", generator=g))
    w = _bf(torch.randn(n, k, device="cuda", generator=g) / math.sqrt(k))
    b = torch.randn(n, device="cuda", generator=g)
    r = _bf(torch.randn(m, n, device="cuda", generator=g))
    ref = x.float() @ w.float().t() + b
    out = ops.linear(x, w, bias=b, force_block_n=bn, kernel_variant=variant)
    torch.cuda.synchronize()
    _close_bf16(out, ref, "bias only")
    out = ops.linear(x, w, bias=b, residual=r, force_block_n=bn, kernel_variant=variant)
    _close_bf16(out, ref + r.float(), "bias + residual")
    out = ops.linear(x, w, residual=r, out_scale=0.25, force_block_n=bn, kernel_variant=variant)
    _close_bf16(out, 0.25 * (x.float() @ w.float().t()) + r.float(), "scale + residual")


@pytest.mark.parametrize("variant", VARIANTS, ids=VARIANT_IDS)
def test_gemm_repeated_launches_are_identical(cuda_lib, variant):
    """Ring / staging-buffer phases must come back to the same state: bit-identical results over many launches."""
    g = torch.Generator(device="cuda").manual_seed(11)
    m, k, n = 16800, 320, 320
    x = _bf(torch.randn(m, k, device="cuda", generator=g))
    w = _bf(torch.randn(n, k, device="cuda", generator=g) / math.sqrt(k))
    r = _bf(torch.randn(m, n, device="cuda", generator=g))
    first = ops.linear(x, w, residual=r, kernel_variant=variant).clone()
    for _ in range(10):
        again = ops.linear(x, w, residual=r, kernel_variant=variant)
        assert torch.equal(first, again)
    base = ops.linear(x, w, residual=r, kernel_variant=2)
    assert (first.float() - base.float()).abs().max().item() <= 2.0 ** -6 * base.float().abs().max().item()


@pytest.mark.parametrize("variant", VARIANTS, ids=VARIANT_IDS)
def test_gemm_strided_views(cuda_lib, variant):
    g = torch.Generator(device="cuda").manual_seed(3)
    m, k, n = 700, 320, 320
    big = _bf(torch.randn(m, 3 * k, device="cuda", generator=g))
    x = big[:, k:2 * k]
    w = _bf(torch.randn(n, k, device="cuda", generator=g) / math.sqrt(k))
    rbig = _bf(torch.randn(m, 2 * n, device="cuda", generator=g))
    outbuf = torch.zeros(m, 2 * n, dtype=torch.bfloat16, device="cuda")
    ops.linear(x, w, residual=rbig[:, :n], out=outbuf[:, n:], ldo=2 * n, kernel_variant=variant)
    ref = x.float() @ w.float().t() + rbig[:, :n].float()
    _close_bf16(outbuf[:, n:], ref)
    assert outbuf[:, :n].abs().max().item() == 0


@pytest.mark.parametrize("n,h,w,ci,co,stride", [
    (3, 28, 50, 320, 320, 1), (2, 14, 25, 640, 1280, 1), (3, 7, 13, 1280, 640, 1),
    (2, 28, 50, 320, 320, 2), (3, 14, 25, 640, 640, 2), (5, 7, 13, 1280, 1280, 2), (1, 53, 100, 320, 320, 1),
    (12, 28, 50, 320, 320, 1), (12, 14, 25, 640, 640, 1),
])
@pytest.mark.parametrize("variant", VARIANTS, ids=VARIANT_IDS)
def test_conv3x3(cuda_lib, n, h, w, ci, co, stride, variant):
    g = torch.Generator(device="cuda").manual_seed(4)
    x = _bf(torch.randn(n, ci, h, w, device="cuda", generator=g))
    wt = _bf(torch.randn(co, ci, 3, 3, device="cuda", generator=g) / math.sqrt(9 * ci))
    b = torch.randn(co, device="cuda", generator=g)
    temb = torch.randn(n, co, device="cuda", generator=g)
    ref = F.conv2d(x.float(), wt.float(), b, stride=stride, padding=1) + temb[:, :, None, None]
    ho, wo = ref.shape[-2:]
    res = _bf(torch.randn(n, co, ho, wo, device="cuda", generator=g))
    out = ops.gemm_conv(_nhwc(x), _conv_weight(wt), n_img=n, h_in=h, w_in=w, c0=ci, lda0=ci, n_out=co, taps=3,
                        stride=stride, pad=1, bias=b, rowbias=temb, residual=_nhwc(res), ldr=co, kernel_variant=variant)
    assert out.shape == (n * ho * wo, co)
    _close_bf16(out, _nhwc(ref + res.float()))


@pytest.mark.parametrize("variant", VARIANTS, ids=VARIANT_IDS)
def test_conv3x3_small_images_many_per_tile(cuda_lib, variant):
    """4x7 level: several images per 128-row tile (and, for pairs, a cluster whose second tile lies past the last image)."""
    g = torch.Generator(device="cuda").manual_seed(8)
    n, h, w, ci, co = 5, 4, 7, 1280, 1280
    x = _bf(torch.randn(n, ci, h, w, device="cuda", generator=g))
    wt = _bf(torch.randn(co, ci, 3, 3, device="cuda", generator=g) / math.sqrt(9 * ci))
    b = torch.randn(co, device="cuda", generator=g)
    ref = F.conv2d(x.float(), wt.float(), b, padding=1)
    out = ops.gemm_conv(_nhwc(x), _conv_weight(wt), n_img=n, h_in=h, w_in=w, c0=ci, lda0=ci, n_out=co, taps=3, pad=1,
                        bias=b, kernel_variant=variant, allow_split_k=False)
    _close_bf16(out, _nhwc(ref))


@pytest.mark.parametrize("variant", VARIANTS, ids=VARIANT_IDS)
def test_conv3x3_two_sources_residual(cuda_lib, variant):
    g = torch.Generator(device="cuda").manual_seed(5)
    n, h, w, c0, c1, co = 2, 14, 25, 640, 320, 640
    xa = _bf(torch.randn(n, c0, h, w, device="cuda", generator=g))
    xb = _bf(torch.randn(n, c1, h, w, device="cuda", generator=g))
    wt = _bf(torch.randn(co, c0 + c1, 3, 3, device="cuda", generator=g) / math.sqrt(9 * (c0 + c1)))
    res = _bf(torch.randn(n, co, h, w, device="cuda", generator=g))
    ref = F.conv2d(torch.cat([xa, xb], 1).float(), wt.float(), None, padding=1) + res.float()
    out = ops.gemm_conv(_nhwc(xa), _conv_weight(wt), n_img=n, h_in=h, w_in=w, c0=c0, lda0=c0, a1=_nhwc(xb), c1=c1,
                        lda1=c1, n_out=co, taps=3, pad=1, residual=_nhwc(res), ldr=co, kernel_variant=variant)
    _close_bf16(out, _nhwc(ref))


@pytest.mark.parametrize("variant", VARIANTS, ids=VARIANT_IDS)
@pytest.mark.parametrize("m,c", [(777, 320), (16800, 320), (1092, 1280)])
def test_geglu(cuda_lib, variant, m, c):
    g = torch.Generator(device="cuda").manual_seed(6)
    x = _bf(torch.randn(m, c, device="cuda", generator=g))
    w = _bf(torch.randn(8 * c, c, device="cuda", generator=g) / math.sqrt(c))
    b = torch.randn(8 * c, device="cuda", generator=g)
    h = x.float() @ w.float().t() + b
    val, gate = h.chunk(2, dim=-1)
    ref = val * F.gelu(gate)
    wp, bp = pack_geglu(w, b)
    out = ops.linear(x, wp, bias=bp, geglu=True, kernel_variant=variant)
    assert out.shape == (m, 4 * c)
    assert _rel(out, ref) < 8e-3, _rel(out, ref)


@pytest.mark.parametrize("variant", VARIANTS, ids=VARIANT_IDS)
@pytest.mark.parametrize("m,c,n", [(1000, 320, 960), (16800, 320, 320), (4200, 640, 1920), (1092, 1280, 1280), (336, 1280, 3840),
                                   (1, 320, 960), (129, 320, 960),  # a single row, one row past a tile
                                   (77, 768, 2304), (154, 768, 2304), (924, 768, 3072)])  # the text encoder's
def test_row_stats_and_folded_layernorm(cuda_lib, variant, m, c, n):
    """producer GEMM emits (sum, sum sq) of its bf16 output rows; consumer GEMM applies LayerNorm through its epilogue."""
    g = torch.Generator(device="cuda").manual_seed(9)
    x0 = _bf(torch.randn(m, c, device="cuda", generator=g))
    w0 = _bf(torch.randn(c, c, device="cuda", generator=g) / math.sqrt(c))
    b0 = torch.randn(c, device="cuda", generator=g) * 0.5 + 0.3  # non-zero row mean
    r0 = _bf(torch.randn(m, c, device="cuda", generator=g))
    x, st = ops.linear(x0, w0, bias=b0, residual=r0, kernel_variant=variant, emit_stats=True)
    torch.cuda.synchronize()
    # the statistics describe the values as stored (bf16-rounded): those are what the consumer multiplies
    s = st.data.double().sum(1)
    xf = x0.float() @ w0.float().t() + b0 + r0.float()  # the row values before rounding (fp32 reference of the producer)
    assert (xf - x.float()).abs().max().item() < 0.05
    xs = x.double()
    e_s, e_ss = (s[:, 0] - xs.sum(-1)).abs(), (s[:, 1] - (xs ** 2).sum(-1)).abs()
    # 3e-5 of sum |x| / sum x^2 (test_clip_embed's bound), and never looser than 2e-2 on the sum
    assert (e_s <= (3e-5 * xs.abs().sum(-1)).clamp(max=2e-2)).all(), e_s.max().item()
    assert (e_ss <= 3e-5 * (xs ** 2).sum(-1)).all(), e_ss.max().item()
    gamma = torch.randn(c, device="cuda", generator=g) * 0.3 + 1.0
    beta = torch.randn(c, device="cuda", generator=g) * 0.2
    w = torch.randn(n, c, device="cuda", generator=g) / math.sqrt(c)
    b = torch.randn(n, device="cuda", generator=g)
    ref = F.layer_norm(x.float(), (c,), gamma, beta, 1e-5) @ w.t() + b
    wg = _bf(w * gamma[None, :])
    colsum = wg.float().sum(1)
    cn = w @ beta + b
    out = ops.linear(x, wg, bias=cn, ln=st, ln_colsum=colsum, ln_eps=1e-5, kernel_variant=variant)
    # yardstick: the unfused path (LayerNorm rounded to bf16, then the GEMM with bf16 weights)
    unf = ops.linear(ops.layernorm(x, gamma, beta), _bf(w), bias=b, kernel_variant=2)
    e_fold, e_unf = _rel(out, ref), _rel(unf, ref)
    assert e_fold < max(1.5 * e_unf, 8e-3), (e_fold, e_unf)


@pytest.mark.parametrize("variant", VARIANTS, ids=VARIANT_IDS)
def test_folded_layernorm_geglu(cuda_lib, variant):
    g = torch.Generator(device="cuda").manual_seed(10)
    m, c = 4200, 640
    x0 = _bf(torch.randn(m, c, device="cuda", generator=g))
    w0 = _bf(torch.randn(c, c, device="cuda", generator=g) / math.sqrt(c))
    x, st = ops.linear(x0, w0, kernel_variant=variant, emit_stats=True)
    gamma = torch.randn(c, device="cuda", generator=g) * 0.3 + 1.0
    beta = torch.randn(c, device="cuda", generator=g) * 0.2
    w = torch.randn(8 * c, c, device="cuda", generator=g) / math.sqrt(c)
    b = torch.randn(8 * c, device="cuda", generator=g)
    h = F.layer_norm(x.float(), (c,), gamma, beta, 1e-5) @ w.t() + b
    val, gate = h.chunk(2, dim=-1)
    ref = val * F.gelu(gate)
    wg = _bf(w * gamma[None, :])
    wp, bp = pack_geglu(wg, w @ beta + b)
    _, cs = pack_geglu(wg, wg.float().sum(1))  # column sums in the packed row order
    out = ops.linear(x, wp, bias=bp, geglu=True, ln=st, ln_colsum=cs, kernel_variant=variant)
    assert _rel(out, ref) < 1e-2, _rel(out, ref)
