"""GEMM / implicit-GEMM convolution stores held bit for bit to the fp32 result of the same launch, that result held to a
float64 error model, and the other bf16 / f16 stores held to round-to-nearest statistics (tests/store_rounding.py).

(a) Twins.  Every storage-type launch here goes through ops.gemm_conv, whose calls a spy captures; each one is launched
    again with an fp32 output on the identical operands and descriptor (same `force_block_n`, `force_splits`, kernel variant,
    row statistics and column-slice layout, so the planner picks the same tiling: asserted through mdb_gemm_conv_plan).  The
    stored output must equal `twin.to(dt)` bitwise.  A residual that aliases the output is read by the twin from an untouched
    copy.  The twin's output is guard-banded too and must be fully written.
(b) Activation epilogues.  ReLU: bitwise max(0, twin).to(bf16).  quick-GELU and GEGLU: inside the bracket around f(twin)
    evaluated in float64, widened by the approximation error of the kernel's quick_gelu / gelu_erf (store_rounding.py).
    The twin of an activation launch is a linear launch without split-K (the activation epilogues never split) over the same
    weights and block width; for GEGLU it is the [128 value | 128 gate] weight at block width 256, its columns mapped to
    value and gate.
(c) Every fp32 twin without a folded LayerNorm within δ of the float64 value (store_rounding.gemm_model), with the plan's
    split count.  The folded LayerNorm keeps test_layernorm_fold_gpu.py's criterion: its statistics add errors the model
    does not describe.
(d) The bf16 / f16 stores without an fp32 twin (GroupNorm, LayerNorm, the row softmax, the direct convolution): signed
    mean and rms of the store error in ulps over >= 10^4 normal-range elements, a statistical criterion by design.

The worst ratio per family is printed through tests/common.record."""
import inspect
import math
import re
from collections import defaultdict

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from magicdrive_b200 import ops, vae_f16_ops  # noqa: E402
from tests import store_rounding as sr  # noqa: E402
from tests.common import record  # noqa: E402
from tests.launch_census import _2d, _window  # noqa: E402
from tests.test_kernel_edges_gpu import (BF16, F16, F32, F64, M_TAILS, PRODUCT_CONVS, Guarded, _gen, _randn,  # noqa: E402
                                         _run_conv)
from tests.test_layernorm_fold_gpu import CONSUMER_CALLS, OFFSETS, _consumer_rows, _fold_weights, _split_stats  # noqa: E402

WORST = defaultdict(float)  # family -> worst ratio


@pytest.fixture(scope="module", autouse=True)
def _record_worst():
    yield
    for fam, r in sorted(WORST.items()):
        record(f"[store] {fam}: worst {r:.3g}")


def _note(family, ratio):
    WORST[family] = max(WORST[family], ratio)


def dt_variants(values, ids=None):
    """pytest params (dt, variant, *value): bf16 at kernel variants 0 (planner), 4 (single CTAs, no split-K) and 3 (CTA
    pairs); f16 at 0 and 4 (the f16 kernels have no CTA pairs)."""
    values = [v if isinstance(v, tuple) else (v,) for v in values]
    ids = ids or ["-".join(str(x) for x in v) for v in values]
    names = {0: "planner", 4: "nosplit", 3: "pair"}
    out = []
    for dt, variants in ((BF16, (0, 4, 3)), (F16, (0, 4))):
        for var in variants:
            out += [pytest.param(dt, var, *v, id=f"{'f16-' if dt == F16 else ''}{i}-{names[var]}") for v, i in zip(values, ids)]
    return out


# ------------------------------------------------------------------------------------------------------- twins
_GEMM_SIG = inspect.signature(ops.gemm_conv)


def _planned(fn, a):
    """fn(**a) with the planner's tiling read back: (result, [block_n, m_tiles, n_tiles, splits, waves])."""
    ops._profile = []  # ops.gemm_conv asks the planner for its tiling only while profiling
    try:
        res = fn(**a)
        info = ops._profile[-1][4]
    finally:
        ops._profile = None
    return res, [int(x) for x in re.findall(r"BN=(\d+) tiles=(\d+)x(\d+)x(\d+) waves=(\d+)", info)[0]]


def _strided_copy(t, ld):
    """A copy of the 2-D view t with row stride ld."""
    buf = torch.empty((t.shape[0], ld), dtype=t.dtype, device=t.device)[:, :t.shape[1]]
    buf.copy_(t)
    return buf


class Twin:
    """One captured storage-type launch (its arguments by name, plan and output window) and its fp32 twin."""

    def __init__(self, a, plan, twin, twin_plan, residual):
        self.a, self.plan, self.twin, self.twin_plan = a, plan, twin, twin_plan
        self.residual = residual  # what the launch read as residual (a copy taken before it, when it aliased the output)
        rows, cols, ld = _window("gemm_conv", a)
        self.out = _2d(a["out"], rows, cols, ld)


def twins(monkeypatch, run):
    """Run `run()` with ops.gemm_conv spied on; returns (run's result, [Twin per call])."""
    real = ops.gemm_conv
    got = []

    def spy(*args, **kw):
        b = _GEMM_SIG.bind(*args, **kw)
        b.apply_defaults()
        a = dict(b.arguments)
        assert a["out"] is not None, "the twin needs the launch's output window"
        res_in = a["residual"]
        if res_in is not None and res_in.data_ptr() == a["out"].data_ptr():
            res_in = _strided_copy(res_in, a["ldr"])
        res, plan = _planned(real, a)
        rows, cols, ld = _window("gemm_conv", a)
        o = a["out"]
        col0 = o.storage_offset() % ld if ld > cols else 0
        width = a["n_out"] if a["geglu"] else cols
        tw = Guarded(rows, width, F32, ld=max(ld, width) if not a["geglu"] else width, col0=col0 if not a["geglu"] else 0)
        t = dict(a, out=tw.out, ldo=tw.ld, out_f32=True, residual=res_in, geglu=False, quick_gelu=False, relu=False)
        if a["geglu"] or a["quick_gelu"]:
            t["allow_split_k"] = False  # these epilogues never split
        if a["geglu"]:
            t["force_block_n"] = 256
        _, tplan = _planned(real, t)
        tw.check("fp32 twin")
        got.append(Twin(a, plan, tw, tplan, res_in))
        return res

    monkeypatch.setattr(ops, "gemm_conv", spy)
    try:
        r = run()
    finally:
        monkeypatch.setattr(ops, "gemm_conv", real)
    torch.cuda.synchronize()
    assert got, "run() launched no GEMM"
    return r, got


def _bits(t):
    return t.contiguous().view(torch.int16)


def check_twin(tw, family, model=True):
    """(a) bitwise, and (c) the twin within the model's δ (unless model=False)."""
    assert tw.plan[:4] == tw.twin_plan[:4], f"the fp32 twin planned {tw.twin_plan}, the launch {tw.plan}"
    want = tw.twin.out.to(tw.out.dtype)
    diff = (_bits(tw.out) != _bits(want)).nonzero()
    assert diff.shape[0] == 0, (f"{diff.shape[0]} stored elements differ from the fp32 twin rounded to nearest, first at "
                                f"{tuple(diff[0].tolist())}: {tw.out[tuple(diff[0])].item()!r} vs fp32 "
                                f"{tw.twin.out[tuple(diff[0])].item()!r} (plan {tw.plan})")
    if model:
        fp32_model(tw, family)


def fp32_model(tw, family):
    a = dict(tw.a, residual=tw.residual, geglu=False, quick_gelu=False, relu=False)  # the twin's linear epilogue
    if tw.residual is not None:
        a["ldr"] = tw.residual.stride(0)
    v, d = sr.gemm_model(a, splits=tw.plan[3])
    _note(f"fp32 |out - v| / delta, {family}", sr.check_f32(tw.twin.out, v, d, f"fp32 twin ({family}, plan {tw.plan})"))


# ------------------------------------------------------------------------------------------ (a) + (c) linear epilogue
@pytest.mark.parametrize("dt,variant,case", dt_variants(list(PRODUCT_CONVS)))
def test_product_convs(cuda_lib, monkeypatch, dt, variant, case):
    n, h, w, c0, co, taps, stride, pad, extra = PRODUCT_CONVS[case]
    extra = {k: v for k, v in extra.items() if k != "out_f32"}  # conv_out / vae_conv_out: the fp32 launch is the twin
    (out, _), tws = twins(monkeypatch, lambda: _run_conv(n=n, h=h, w=w, c0=c0, co=co, taps=taps, stride=stride, pad=pad,
                                                         variant=variant, seed=1, dt=dt, **extra))
    out.check(case)
    check_twin(tws[0], "product convolutions")


@pytest.mark.parametrize("dt,variant,n,h,w,taps,stride", dt_variants(M_TAILS))
def test_m_tails(cuda_lib, monkeypatch, dt, variant, n, h, w, taps, stride):
    (out, _), tws = twins(monkeypatch, lambda: _run_conv(n=n, h=h, w=w, c0=128, co=192, taps=taps, stride=stride,
                                                         pad=taps // 2, rowbias="image", residual=True, variant=variant,
                                                         seed=3, dt=dt))
    out.check()
    check_twin(tws[0], "M tails")


@pytest.mark.parametrize("stats", [False, True], ids=["plain", "stats"])
@pytest.mark.parametrize("bn", [64, 128, 160, 256])
@pytest.mark.parametrize("dt,variant,n_out", dt_variants([8, 40, 136, 264, 520]))
def test_n_tails(cuda_lib, monkeypatch, dt, variant, n_out, bn, stats):
    g = _gen(4)
    m, k = 1000, 320
    x = _randn(m, k, g=g).to(dt)
    w = _randn(n_out, k, g=g, scale=1 / math.sqrt(k)).to(dt)
    b = _randn(n_out, g=g)
    r = _randn(m, n_out, g=g).to(dt)
    out = Guarded(m, n_out, dt)
    _, tws = twins(monkeypatch, lambda: ops.linear(x, w, bias=b, residual=r, out=out.out, ldo=n_out, force_block_n=bn,
                                                   kernel_variant=variant, emit_stats=stats))
    out.check()
    check_twin(tws[0], "N tails")


@pytest.mark.parametrize("rowbias", ["image", "shared"])
@pytest.mark.parametrize("dt,splits", [pytest.param(BF16, s, id=str(s)) for s in (2, 3, 7)] +
                         [pytest.param(F16, s, id=f"f16-{s}") for s in (2, 3, 7)])
def test_split_k(cuda_lib, monkeypatch, dt, splits, rowbias):
    (out, _), tws = twins(monkeypatch, lambda: _run_conv(n=3, h=14, w=25, c0=640, co=640, taps=3, pad=1, rowbias=rowbias,
                                                         residual=True, out_scale=0.75, force_splits=splits, seed=5, dt=dt))
    out.check()
    assert tws[0].plan[3] == splits, tws[0].plan
    check_twin(tws[0], "split-K")


@pytest.mark.parametrize("dt,variant,taps,stride", dt_variants([(3, 1), (1, 1), (3, 2)]))
def test_strided_sources_column_slice(cuda_lib, monkeypatch, dt, variant, taps, stride):
    (out, _), tws = twins(monkeypatch, lambda: _run_conv(n=3, h=14, w=25, c0=320, lda0=448, c1=192, co=320, taps=taps,
                                                         stride=stride, pad=taps // 2, residual=True, ldo=512, col0=128,
                                                         variant=variant, seed=6, dt=dt))
    out.check()
    check_twin(tws[0], "strided sources, column slice")


# (dt, variant, force_splits): single CTAs, CTA pairs, and a split-K launch whose finalise reads the residual it overwrites
ALIAS = [(BF16, 4, 0), (BF16, 3, 0), (BF16, 0, 3), (F16, 4, 0), (F16, 0, 3)]


@pytest.mark.parametrize("dt,variant,splits", ALIAS, ids=["nosplit", "pair", "split3", "f16-nosplit", "f16-split3"])
def test_residual_aliases_output(cuda_lib, monkeypatch, dt, variant, splits):
    """out = (conv(x) + bias) * 0.75 + out: the residual is the output itself, in a column slice of a wider buffer."""
    g = _gen(7)
    n, h, w, c, co = 3, 14, 25, 640, 640
    pix = n * h * w
    x = _randn(pix, c, g=g).to(dt)
    wm = _randn(co, 9 * c, g=g, scale=1 / math.sqrt(9 * c)).to(dt)
    b = _randn(co, g=g)
    out = Guarded(pix, co, dt, ld=co + 64, col0=32)
    out.out.copy_(_randn(pix, co, g=g))
    _, tws = twins(monkeypatch, lambda: ops.gemm_conv(x, wm, n_img=n, h_in=h, w_in=w, c0=c, lda0=c, n_out=co, taps=3, pad=1,
                                                      bias=b, residual=out.out, ldr=out.ld, out=out.out, ldo=out.ld,
                                                      out_scale=0.75, force_splits=splits, kernel_variant=variant))
    out.check()
    assert tws[0].plan[3] == max(splits, 1), tws[0].plan
    check_twin(tws[0], "residual aliasing the output")


@pytest.mark.parametrize("offset", OFFSETS)
@pytest.mark.parametrize("dt,variant", dt_variants([()], ids=["fold"]))
def test_folded_layernorm(cuda_lib, monkeypatch, dt, variant, offset):
    """The linear consumer of a folded LayerNorm (test_layernorm_fold_gpu.py's rows, statistics and weights): bitwise
    against its fp32 twin; the fp32 value is not held to the model (see the module docstring)."""
    g = _gen(50)
    m, c, n = 300, 320, 960
    wg, colsum, cvec = _fold_weights(n, c, g)
    wg = wg.to(dt)
    colsum = wg.float().sum(1)
    for parts, bn, eps, slice_ in CONSUMER_CALLS:
        x = _consumer_rows(m, c, offset, eps, g).to(dt)
        stats = _split_stats(x, parts, g)
        out = Guarded(m, n, dt, ld=n + 16 if slice_ else None, col0=8 if slice_ else 0)
        _, tws = twins(monkeypatch, lambda: ops.linear(x, wg, bias=cvec, out=out.out, ldo=out.ld, force_block_n=bn,
                                                       kernel_variant=variant, ln=ops.RowStats(stats, parts),
                                                       ln_colsum=colsum, ln_eps=eps))
        out.check(f"parts={parts} bn={bn}")
        check_twin(tws[0], "folded LayerNorm", model=False)


# ----------------------------------------------------------------------------------------------- (c) fp32 launches
def test_vae_attention_fp32(cuda_lib, monkeypatch):
    """The VAE mid-block attention's fp32-output launches (test_kernel_edges_gpu.test_gemm_vae_attention): the scores
    S = q k^T scale with n_out = ldo = lp, and P V + b_v from probabilities, in both types."""
    L, C = 1400, 512
    lp = (L + 63) // 64 * 64
    for dt in (BF16, F16):
        g = _gen(2)
        q = _randn(L, C, g=g).to(dt)
        kbuf = torch.zeros(lp, C, dtype=dt, device="cuda")
        kbuf[:L] = _randn(L, C, g=g).to(dt)
        p = torch.softmax(_randn(L, lp, g=g, scale=3.0), -1).to(dt)
        vt = _randn(C, lp, g=g).to(dt)
        bv = _randn(C, g=g)
        s, o = Guarded(L, lp, dt), Guarded(L, C, dt)
        _, tws = twins(monkeypatch, lambda: (ops.linear(q, kbuf, out_scale=C ** -0.5, out=s.out, ldo=lp),
                                             ops.linear(p, vt, bias=bv, out=o.out, ldo=C)))
        s.check("scores")
        o.check("P V")
        assert len(tws) == 2
        for tw in tws:
            check_twin(tw, "VAE attention")


# K from one 64-wide block to the deepest product launch (3x3 over 2560 channels)
DEPTHS = [(1, 64), (1, 320), (3, 320), (3, 1280), (3, 2560)]


@pytest.mark.parametrize("nonneg", [False, True], ids=["signed", "nonneg"])
@pytest.mark.parametrize("dt,variant,taps,c", dt_variants(DEPTHS))
def test_depth(cuda_lib, monkeypatch, dt, variant, taps, c, nonneg):
    """12 images of 4x7 pixels (the 1280-channel level's grid) into 320 channels.  nonneg: both operands >= 0, so every
    product of a dot product has the same sign and a truncating accumulator would drift instead of cancelling."""
    g = _gen(8)
    n, h, w, co = 12, 4, 7, 320
    k = taps * taps * c
    x = _randn(n * h * w, c, g=g)
    wm = _randn(co, k, g=g, scale=1 / math.sqrt(k))
    if nonneg:
        x, wm = x.abs(), wm.abs()
    x, wm = x.to(dt), wm.to(dt)
    b = _randn(co, g=g)
    out = Guarded(n * h * w, co, dt)
    _, tws = twins(monkeypatch, lambda: ops.gemm_conv(x, wm, n_img=n, h_in=h, w_in=w, c0=c, lda0=c, n_out=co, taps=taps,
                                                      pad=taps // 2, bias=b, out=out.out, ldo=co, kernel_variant=variant))
    out.check()
    check_twin(tws[0], f"K {k}" + (" nonnegative" if nonneg else ""))


# ------------------------------------------------------------------------------------------------ (b) activations
RELU_SHAPES = {  # (n, h, w, c0, co, taps, force_splits): Inception-like convolutions with BatchNorm folded, then ReLU
    "3x3_17x17": (2, 17, 17, 192, 160, 3, 0),
    "1x1_8x8": (2, 8, 8, 768, 192, 1, 0),
    "3x3_8x8_split3": (2, 8, 8, 384, 192, 3, 3),
}


RELU_CASES = [(c, v) for c in RELU_SHAPES for v in (0, 3) if not (v == 3 and RELU_SHAPES[c][6])]  # pairs never split


@pytest.mark.parametrize("bn", [0, 64, 128, 160, 256], ids=["planner", "bn64", "bn128", "bn160", "bn256"])
@pytest.mark.parametrize("case,variant", RELU_CASES, ids=[f"{c}-{'pair' if v == 3 else 'planner'}" for c, v in RELU_CASES])
def test_relu(cuda_lib, monkeypatch, case, variant, bn):
    n, h, w, c0, co, taps, splits = RELU_SHAPES[case]
    (out, _), tws = twins(monkeypatch, lambda: _run_conv(n=n, h=h, w=w, c0=c0, co=co, taps=taps, pad=taps // 2, relu=True,
                                                         force_block_n=bn, force_splits=splits, variant=variant, seed=9))
    out.check(case)
    tw = tws[0]
    assert tw.plan[:4] == tw.twin_plan[:4], (tw.plan, tw.twin_plan)
    want = tw.twin.out.clamp_min(0.0).to(BF16)
    bad = (_bits(tw.out) != _bits(want)).sum().item()
    assert bad == 0, f"{bad} ReLU outputs differ from max(0, fp32 twin) rounded to nearest"
    fp32_model(tw, "ReLU twins")


def _act_bracket(out, f, eps, family):
    """out inside [RN(f - eps), RN(f + eps)]; notes the worst |out - f| / (eps + ulp(f) / 2)."""
    sr.check_bracket(out, f, eps, family)
    r = ((out.to(F64) - f).abs() / (eps + sr.ulp(f, out.dtype) / 2)).max().item()
    _note(f"|out - f| / (eps + ulp / 2), {family}", r)


@pytest.mark.parametrize("bn", [0, 64, 128, 160, 256], ids=["planner", "bn64", "bn128", "bn160", "bn256"])
@pytest.mark.parametrize("variant", [0, 3, 4], ids=["planner", "pair", "nosplit"])
def test_quick_gelu(cuda_lib, monkeypatch, variant, bn):
    """CLIP's fc1 on two 77-token captions: [154, 768] x [3072, 768] with bias, scaled up so the negative tail is reached."""
    g = _gen(10)
    m, k, n = 154, 768, 3072
    x = _randn(m, k, g=g).to(BF16)
    w = _randn(n, k, g=g, scale=3 / math.sqrt(k)).to(BF16)
    b = _randn(n, g=g)
    out = Guarded(m, n, BF16)
    _, tws = twins(monkeypatch, lambda: ops.linear(x, w, bias=b, out=out.out, ldo=n, quick_gelu=True, force_block_n=bn,
                                                   kernel_variant=variant))
    out.check()
    tw = tws[0]
    assert tw.plan[:4] == tw.twin_plan[:4], (tw.plan, tw.twin_plan)
    v = tw.twin.out.to(F64)
    _act_bracket(tw.out, v * torch.sigmoid(1.702 * v), sr.quick_gelu_eps(tw.twin.out), "quick-GELU")
    fp32_model(tw, "activation twins")


@pytest.mark.parametrize("dt,variant", dt_variants([()], ids=["geglu"]))
def test_geglu(cuda_lib, monkeypatch, dt, variant):
    """The UNet's GEGLU projection (1000 tokens, C 320, inner 1280) on a weight already in [128 value | 128 gate] order."""
    g = _gen(11)
    m, k, inner = 1000, 320, 1280
    x = _randn(m, k, g=g).to(dt)
    w = _randn(2 * inner, k, g=g, scale=2 / math.sqrt(k)).to(dt)
    b = _randn(2 * inner, g=g)
    out = Guarded(m, inner, dt)
    _, tws = twins(monkeypatch, lambda: ops.linear(x, w, bias=b, out=out.out, ldo=inner, geglu=True,
                                                   kernel_variant=variant))
    out.check()
    tw = tws[0]
    assert tw.plan[0] == tw.twin_plan[0] == 256 and tw.plan[1:4] == tw.twin_plan[1:4], (tw.plan, tw.twin_plan)
    t = tw.twin.out.view(m, inner // 128, 2, 128)
    a32, g32 = t[:, :, 0].reshape(m, inner), t[:, :, 1].reshape(m, inner)
    a, gt = a32.to(F64), g32.to(F64)
    f = a * F.gelu(gt)
    eps = a.abs() * sr.gelu_eps(g32) + 2.0 ** -23 * f.abs()
    _act_bracket(tw.out, f, eps, "GEGLU")
    tail = (gt < -3) & (f.abs() > 0)
    if tail.any():
        rel = ((tw.out.to(F64) - f).abs() / f.abs())[tail].max().item()
        _note("GEGLU relative error against exact erf GELU, gate < -3", rel)
    fp32_model(tw, "activation twins")


# ------------------------------------------------------------------------------------------------ (d) statistics
def _stats(out, ref, family):
    mean, rms, cnt = sr.check_stats(out, ref, family)
    _note(f"|store mean| (ulp), {family}", abs(mean))
    _note(f"store rms (ulp), {family}", rms)
    return mean, rms, cnt


@pytest.mark.parametrize("rows", ["0", "1"], ids=["slab", "rows"])
@pytest.mark.parametrize("dt", [BF16, F16], ids=["bf16", "f16"])
def test_groupnorm_statistics(cuda_lib, monkeypatch, dt, rows):
    """The GroupNorm kernels (slab and pixel-major cluster) with SiLU on N(0, 1) groups."""
    for k in ("MDB_GN_ROWS", "MDB_GN_ROWS_CLUSTER", "MDB_GN_TWO_KERNEL"):
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("MDB_GN_ROWS", rows)
    g = _gen(12)
    n, hw, c = 2, 1400, 320
    x = _randn(n * hw, c, g=g).to(dt)
    gamma, beta = _randn(c, g=g), _randn(c, g=g)
    out = ops.groupnorm(x, c, c, n, hw, gamma, beta, 1e-5, True)
    ref = F.silu(F.group_norm(x.to(F64).view(n, hw, c).permute(0, 2, 1), 32, gamma.to(F64), beta.to(F64), 1e-5))
    _stats(out, ref.permute(0, 2, 1).reshape(n * hw, c), f"GroupNorm {dt}")


def test_layernorm_statistics(cuda_lib):
    g = _gen(13)
    x = _randn(2000, 768, g=g).to(BF16)
    gamma, beta = _randn(768, g=g), _randn(768, g=g)
    out = ops.layernorm(x, gamma, beta)
    _stats(out, F.layer_norm(x.to(F64), (768,), gamma.to(F64), beta.to(F64), 1e-5), "LayerNorm")


@pytest.mark.parametrize("dt", [BF16, F16], ids=["bf16", "f16"])
def test_softmax_rows_statistics(cuda_lib, dt):
    g = _gen(14)
    rows, cols, cols_out = 700, 1400, 1408
    s = _randn(rows, cols, g=g, scale=3.0)
    out = (ops.softmax_rows if dt == BF16 else vae_f16_ops.softmax_rows_f16)(s, cols, cols_out)
    assert not out[:, cols:].any()
    _stats(out[:, :cols], torch.softmax(s.to(F64), -1), f"softmax_rows {dt}")


@pytest.mark.parametrize("dt", [BF16, F16], ids=["bf16", "f16"])
def test_conv_direct_statistics(cuda_lib, dt):
    """The VAE decoder's conv_in (4 -> 512 channels, 3x3) from fp32 latents."""
    g = _gen(15)
    n, h, w, cin, cout = 2, 28, 50, 4, 512
    x = _randn(n, h, w, cin, g=g)
    wt = _randn(3, 3, cin, cout, g=g, scale=1 / math.sqrt(9 * cin))
    b = _randn(cout, g=g)
    fn = ops.conv_direct if dt == BF16 else vae_f16_ops.conv_direct_f16
    out = fn(x, wt, b, n=n, h=h, w=w, cin=cin, cout=cout, k=3)
    assert out.dtype == dt
    ref = F.conv2d(x.to(F64).permute(0, 3, 1, 2), wt.to(F64).permute(3, 2, 0, 1), b.to(F64), padding=1)
    _stats(out.reshape(-1, cout), ref.permute(0, 2, 3, 1).reshape(-1, cout), f"conv_direct {dt}")
