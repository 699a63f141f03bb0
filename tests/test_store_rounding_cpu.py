"""tests/store_rounding.py on a CPU simulation of one GEMM launch, and on the edges of the bracket.

The simulation has the step's resnet shape class (M 4096, K 2880 = 3x3x320, N 320) with bias, out_scale 0.75 and a
residual: torch's fp32 matmul stands in for the tensor cores, then come the kernel's fp32 epilogue (the bias times the scale,
one fma with the accumulator, the residual add) and a round-to-nearest store.  The correct store passes the twin
comparison, the fp32 bound and the store statistics; each one-line epilogue slip below leaves elements outside the bracket,
while every bf16 slip passes the absolute-slack criterion of test_kernel_edges_gpu._close_bf16.  That is why
test_store_rounding_gpu.py exists."""
import math

import pytest
import torch

from tests import store_rounding as sr
from tests.test_kernel_edges_gpu import _tol_bf16

BF16, F16, F32, F64 = torch.bfloat16, torch.float16, torch.float32, torch.float64
M, K, N, SCALE, SPLITS = 4096, 2880, 320, 0.75, 3


def _round_toward_zero(x, dt):
    """fp32 -> dt truncated toward zero (normal range)."""
    x = x.to(F64)
    u = sr.ulp(x, dt)
    return (torch.sign(x) * torch.floor(x.abs() / u) * u).to(dt)


def _epilogue(acc, b, r):
    """The kernel's single-CTA epilogue in fp32: fma(scale, acc, bias * scale) + residual."""
    cbs = (b * SCALE).float()
    v = (acc.double() * SCALE + cbs.double()).float()  # one rounding: an fma
    return v + r.float()


@pytest.fixture(scope="module", params=[BF16, F16], ids=["bf16", "f16"])
def sim(request):
    dt = request.param
    g = torch.Generator().manual_seed(0)
    x = torch.randn(M, K, generator=g).to(dt)
    w = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(dt)
    b = torch.randn(N, generator=g)
    r = torch.randn(M, N, generator=g).to(dt)
    call = dict(a0=x, w=w, n_img=1, h_in=1, w_in=M, c0=K, lda0=K, n_out=N, bias=b, residual=r, ldr=N, out_scale=SCALE)
    v, delta = sr.gemm_model(call)
    _, delta_split = sr.gemm_model(call, splits=SPLITS)
    acc = x.float() @ w.float().t()
    f32 = _epilogue(acc, b, r)
    seg = K // SPLITS
    partial_bf16 = sum((x[:, i * seg:(i + 1) * seg].float() @ w[:, i * seg:(i + 1) * seg].float().t()).to(BF16).float()
                       for i in range(SPLITS))
    stores = {
        "correct": f32.to(dt),
        "round toward zero": _round_toward_zero(f32, dt),
        "residual added to the rounded GEMM value": (_epilogue(acc, b, torch.zeros_like(r)).to(dt).float() + r.float()).to(dt),
        "bias rounded to the storage type": _epilogue(acc, b.to(dt).float(), r).to(dt),
        "split-K partials carried in bf16": _epilogue(partial_bf16, b, r).to(dt),
        "out_scale off by 1 + 2^-10": ((acc.double() * SCALE * (1 + 2 ** -10) + (b * SCALE).double()).float()
                                       + r.float()).to(dt),
    }
    return dt, v, delta, delta_split, f32, stores


MUTANTS = ["round toward zero", "residual added to the rounded GEMM value", "bias rounded to the storage type",
           "split-K partials carried in bf16", "out_scale off by 1 + 2^-10"]
F16_MUTANTS = ["round toward zero", "bias rounded to the storage type"]


def test_correct_store_passes(sim):
    dt, v, delta, _, f32, stores = sim
    out = stores["correct"]
    assert torch.equal(out.view(torch.int16), f32.to(dt).view(torch.int16))  # (a) the twin, bitwise
    ratio = sr.check_f32(f32, v, delta, "fp32 value")  # (c)
    sr.check_bracket(out, v, delta, "correct store")
    mean, rms, n = sr.check_stats(out, v, "correct store")
    print(f"[store] {dt}: fp32 |out - v| / bound {ratio:.3f}; store mean {mean:+.4f} rms {rms:.4f} ulp over {n}")
    assert abs(rms - 1 / math.sqrt(12)) < 0.01


@pytest.mark.parametrize("mutant", MUTANTS)
def test_mutant_leaves_the_bracket(sim, mutant):
    dt, v, delta, delta_split, _, stores = sim
    if dt == F16 and mutant not in F16_MUTANTS:
        pytest.skip("the f16 table is truncation and a rounded bias")
    d = delta_split if mutant.startswith("split-K") else delta
    frac = sr.outside(stores[mutant], v, d).double().mean().item()
    print(f"[store] {dt} {mutant}: {100 * frac:.1f} % of the elements outside the bracket")
    assert frac > 0.05, f"{mutant}: only {100 * frac:.2f} % outside"
    with pytest.raises(AssertionError):
        sr.check_bracket(stores[mutant], v, d, mutant)


@pytest.mark.parametrize("mutant", MUTANTS)
def test_mutant_passes_the_absolute_slack_criterion(sim, mutant):
    """The criterion of test_kernel_edges_gpu._close_bf16 lets every bf16 slip through: its worst err / tol stays < 1."""
    dt, v, _, _, _, stores = sim
    if dt != BF16:
        pytest.skip("_close_bf16 is the bf16 criterion")
    ratio = ((stores[mutant].to(F64) - v).abs() / _tol_bf16(v)).max().item()
    print(f"[store] {mutant}: err / tol of _close_bf16 {ratio:.2f}")
    assert ratio < 1.0


def test_truncation_fails_the_statistics(sim):
    dt, v, _, _, _, stores = sim
    mean, rms, _ = sr.store_stats(stores["round toward zero"], v)
    assert mean < -0.4, mean
    with pytest.raises(AssertionError):
        sr.check_stats(stores["round toward zero"], v)


def test_double_rounding_fails_the_statistics(sim):
    """Storing a value already rounded to the storage type plus an independent term: a second rounding, rms about 0.41."""
    dt, v, _, _, _, stores = sim
    _, rms, _ = sr.store_stats(stores["residual added to the rounded GEMM value"], v)
    assert rms > sr.RMS_MAX, rms


# ------------------------------------------------------------------------------------------------- bracket edges
def _t(*x):
    return torch.tensor(x, dtype=F64)


def test_ulp():
    assert sr.ulp(_t(1.0, 1.5, -2.0), BF16).tolist() == [2 ** -7, 2 ** -7, 2 ** -6]
    assert sr.ulp(_t(1.0, 65504.0), F16).tolist() == [2 ** -10, 32.0]
    # subnormals and zero: the smallest step of the type
    assert sr.ulp(_t(0.0, 2 ** -20, 2 ** -14 - 2 ** -24, 2 ** -14), F16).tolist() == [2 ** -24] * 4
    assert sr.ulp(_t(0.0, 1e-40), BF16).tolist() == [2 ** -133] * 2


@pytest.mark.parametrize("dt,tie,even,odd", [(BF16, 1 + 2 ** -8, 1.0, 1 + 2 ** -7), (F16, 1 + 2 ** -11, 1.0, 1 + 2 ** -10),
                                              (BF16, 1 + 3 * 2 ** -8, 1 + 2 ** -6, 1 + 2 ** -7),
                                              (F16, -(1 + 3 * 2 ** -11), -(1 + 2 ** -9), -(1 + 2 ** -10))],
                         ids=["bf16-even-below", "f16-even-below", "bf16-even-above", "f16-negative-even-above"])
def test_exact_ties_round_to_even(dt, tie, even, odd):
    """With δ = 0 a tie has a one-point bracket: the even neighbour."""
    lo, hi = sr.bracket(_t(tie), _t(0.0), dt)
    assert lo.item() == hi.item() == even
    assert not sr.outside(torch.tensor([even], dtype=dt), _t(tie), _t(0.0)).item()
    assert sr.outside(torch.tensor([odd], dtype=dt), _t(tie), _t(0.0)).item()


def test_f16_subnormal_boundary():
    # halfway between the largest subnormal 2^-14 - 2^-24 and the smallest normal 2^-14: even is 2^-14
    v = _t(2 ** -14 - 2 ** -25)
    lo, hi = sr.bracket(v, _t(0.0), F16)
    assert lo.item() == hi.item() == 2 ** -14
    assert sr.outside(torch.tensor([2 ** -14 - 2 ** -24], dtype=F16), v, _t(0.0)).item()
    # inside the subnormal range the step is 2^-24: 3.4 steps rounds to 3
    lo, hi = sr.bracket(_t(3.4 * 2 ** -24), _t(0.0), F16)
    assert lo.item() == hi.item() == 3 * 2 ** -24
    # a bracket reaching across the boundary keeps both neighbours
    lo, hi = sr.bracket(v, _t(0.75 * 2 ** -24), F16)
    assert (lo.item(), hi.item()) == (2 ** -14 - 2 ** -24, 2 ** -14)


def test_signed_zeros():
    for dt in (BF16, F16):
        for v in (0.0, -0.0, 1e-60, -1e-60):
            for z in (0.0, -0.0):
                assert not sr.outside(torch.tensor([z], dtype=dt), _t(v), _t(0.0)).item()
        assert sr.outside(torch.tensor([2 ** -24], dtype=F16), _t(0.0), _t(0.0)).item()


def test_f16_overflow_to_inf():
    # 65520 is halfway between 65504 and 2^16: round to nearest even gives 2^16, which is +inf in f16
    for v, want in ((65520.0, math.inf), (-65520.0, -math.inf), (65519.99, 65504.0), (1e6, math.inf)):
        lo, hi = sr.bracket(_t(v), _t(0.0), F16)
        assert lo.item() == hi.item() == want, (v, lo, hi)
    assert sr.outside(torch.tensor([65504.0], dtype=F16), _t(65520.0), _t(0.0)).item()
    assert not sr.outside(torch.tensor([math.inf], dtype=F16), _t(65520.0), _t(0.0)).item()
    # a bracket straddling the overflow threshold admits both
    assert not sr.outside(torch.tensor([65504.0, math.inf], dtype=F16), _t(65520.0, 65520.0), _t(1.0, 1.0)).any()


def test_nan_is_outside():
    for dt in (BF16, F16):
        assert sr.outside(torch.tensor([math.nan], dtype=dt), _t(1.0), _t(1.0)).item()


def test_activation_bounds_cover_an_fp32_evaluation():
    """gelu_eps / quick_gelu_eps hold for the kernel's formulas evaluated in fp32 with exact exp2 and reciprocal (the
    approximate units' own error is inside the derivation's 2^-22 terms)."""
    x = torch.linspace(-12, 12, 200001, dtype=F32)
    ax = x.abs() * 0.70710678118654752440
    t = 1.0 / (0.3275911 * ax + 1.0)
    poly = t * 1.061405429 - 1.453152027
    for c in (1.421413741, -0.284496736, 0.254829592):
        poly = poly * t + c
    poly = poly * t
    e = torch.exp2(-1.4426950408889634 * ax * ax)
    g = 0.5 * x * (1.0 + torch.copysign(1.0 - poly * e, x))
    ref = torch.nn.functional.gelu(x.double())
    assert ((g.double() - ref).abs() <= sr.gelu_eps(x)).all()
    e = torch.exp2(torch.tensor(-1.702, dtype=F32) * 1.4426950408889634 * x)
    q = x * (1.0 / (1.0 + e))
    assert ((q.double() - x.double() * torch.sigmoid(1.702 * x.double())).abs() <= sr.quick_gelu_eps(x)).all()
