"""The attention error model (tests/attention_model.py) held to the kernel's arithmetic on the CPU.

`_restate` is a tile-by-tile fp32 restatement of the consumer loop of csrc/attention_wgmma.cuh for one head: S from the stored
q, k in fp32, keys at or past the batch's key count and (causal) above the diagonal at -inf, a running row max, corr =
exp2(m - m_new), P = exp2(S·c - m) packed to the storage type (f16 with its subnormals), l summed from the unrounded p,
O = O·corr + P V in fp32, each set's O / l rounded to the storage type and added to the stored partial sum, which is rounded
again.  Key tiles are 64 or 128 wide, as the kernel's.  The unmutated restatement meets both criteria with its worst row
within ROW_MAX of the modelled σ in every score regime of the GPU tests; each value-only mutation of the loop exceeds τ,
at shapes where the xformers tolerance the attention tests used before passes it.

Two mutations stay out of the model's reach, and the tests below say so: P truncated instead of rounded (a bias of u/2 per
element, inside the u²/3 variance the model allows for a rounding; see test_truncated_p_is_out_of_reach), and a set's
output added without its own rounding (one rounding fewer than the model counts: the output is more accurate, not less).
The second is caught instead by composing the per-set outputs with the kernel's rounding order, bit for bit
(test_set_rounding_is_caught_by_composition here, test_sets_compose_bitwise on the GPU)."""
import math

import pytest
import torch

from tests.attention_model import TAU, attention_model, model_ratios

BF16, F16, F32, F64 = torch.bfloat16, torch.float16, torch.float32, torch.float64
LOG2E = 1.4426950408889634
# σ bounds each column's error variance; the rms over d columns of one row is an estimate of it, and the worst of 128 rows
# sits near 1 (0.54-1.05 over the regimes and shapes below, the maximum at 8400 keys with unit scores in bf16)
ROW_MAX = 1.1


def _restate(q, k, v, scale, bn, dt, lkb=None, causal=False, mutation=None, rows=None):
    """fp32 restatement of one set of one head: q [lq, d], k / v [lk, d] in `dt`; `rows`: the query row index of each q row
    (causal).  Returns the fp32 O / l before the store."""
    lk = k.shape[0]
    lkb = lk if lkb is None else lkb
    lq = q.shape[0]
    rows = torch.arange(lq) if rows is None else rows
    sc = torch.tensor(scale * LOG2E, dtype=F32)
    s_all = q.float() @ k.float().t()
    nt = (lkb + bn - 1) // bn
    if causal:
        nt = min(nt, (int(rows.max()) // bn) + 1)
    m = torch.full((lq, 1), -math.inf, dtype=F32)
    l = torch.zeros(lq, 1, dtype=F32)
    o = torch.zeros(lq, q.shape[1], dtype=F32)
    for j in range(nt):
        kb = j * bn
        keys = torch.arange(kb, kb + bn)
        s = torch.full((lq, bn), 0.0, dtype=F32)
        n = min(bn, lk - kb)
        s[:, :n] = s_all[:, kb:kb + n]  # keys past lk: TMA zero fill
        cut = lkb - 1 if mutation == "lkb-1" else lkb
        s = s.masked_fill((keys >= cut)[None, :], -math.inf)
        if mutation == "last-tile" and nt > 1 and j == nt - 1:
            s = torch.full_like(s, -math.inf)
        if causal:
            hide = keys[None, :] >= rows[:, None] if mutation == "causal>=" else keys[None, :] > rows[:, None]
            s = s.masked_fill(hide, -math.inf)
        m_new = torch.maximum(m, s.amax(1, keepdim=True) * sc)
        corr = torch.exp2(m - m_new)
        m = m_new
        p = torch.exp2(s * sc - m)
        if mutation == "truncate":
            pb = p.to(dt).float()
            pb = torch.where(pb > p, torch.nextafter(pb.to(dt), torch.zeros((), dtype=dt)).float(), pb)
        else:
            pb = p.to(dt).float()
        l = l + p.sum(1, keepdim=True) if mutation == "l-no-corr" else l * corr + p.sum(1, keepdim=True)
        vt = torch.zeros(bn, v.shape[1], dtype=F32)
        vt[:n] = v[kb:kb + n].float()
        o = o * corr + pb @ vt
    return o / l


def _store(sets_out, dt, mutation=None):
    """The kernel's store of several sets: the first rounded, each next one rounded, added in fp32 to the stored partial sum
    and rounded again."""
    acc = sets_out[0].to(dt)
    for o in sets_out[1:]:
        f = o if mutation == "unrounded-set" else o.to(dt).float()
        acc = (f + acc.float()).to(dt)
    return acc


def _xformers_passes(out, ref, n_sets=1):
    """The tolerance the attention tests held the kernel to before the model (xformers' own: bf16 atol 2e-2 / rtol 5e-3,
    3e-2 with several sets; fp16 atol 4e-3 / rtol 4e-4)."""
    if out.dtype == F16:
        atol, rtol = 4e-3, 4e-4
    else:
        atol, rtol = (2e-2 if n_sets == 1 else 3e-2), 5e-3
    return bool(((out.to(F64) - ref).abs() <= atol + rtol * ref.abs()).all())


# score regimes of tests/test_attention_bounds_gpu.py: q, k, v for lq rows, lk keys, head dim d
def _regime(name, lq, lk, d, dt, g):
    q = torch.randn(lq, d, generator=g)
    k = torch.randn(lk, d, generator=g)
    v = torch.randn(lk, d, generator=g)
    ramp = torch.arange(lk, dtype=F32) / max(lk - 1, 1)
    if name == "peaked":
        q = q * 3
    elif name == "late-max":  # the row max in the last key tile: every tile raises it and runs corr < 1
        q[:, 0] = 3.0
        k[:, 0] = 4.0 * math.sqrt(d) * ramp
    elif name == "early-max":  # tile 0 dominates: corr = 1 afterwards
        q[:, 0] = 3.0
        k[:, 0] = 4.0 * math.sqrt(d) * (1 - ramp)
    elif name == "wide":  # scores spread over about ±100 in log2 units: most p underflow, f16 P goes subnormal
        q = q * 25
    elif name == "v-offset":
        v = v + 20
    elif name == "v-1e3":
        v = v * 250 + 1000
    return q.to(dt), k.to(dt), v.to(dt)


REGIMES = ["unit", "peaked", "late-max", "early-max", "wide", "v-offset"]


def _model(q, k, v, scale, dt, lkb=None, causal=False, sets=1):
    lkb = k.shape[0] if lkb is None else lkb
    kvs = [(k[:lkb], v[:lkb])] * sets
    return attention_model(q, lambda i: kvs, 1, 1, q.shape[0], q.shape[1], scale, dt, causal=causal)


def _run(q, k, v, bn, dt, mutation=None, lkb=None, causal=False):
    d = q.shape[1]
    return _restate(q, k, v, d ** -0.5, bn, dt, lkb=lkb, causal=causal, mutation=mutation).to(dt)


# (lk, d, key-tile width): the 8400-token self-attention at d = 40 (128-key tiles), 1400 keys at d = 80 (64-key tiles),
# a key tail below one tile at each width and a single key
SHAPES = [(8400, 40, 128), (1400, 80, 64), (333, 64, 128), (98, 160, 64), (1, 32, 128), (127, 40, 128), (65, 80, 64)]


@pytest.mark.parametrize("dt", [BF16, F16], ids=["bf16", "f16"])
@pytest.mark.parametrize("regime", REGIMES + ["v-1e3"])
@pytest.mark.parametrize("lk,d,bn", SHAPES, ids=[f"lk{s[0]}-d{s[1]}-bn{s[2]}" for s in SHAPES])
def test_restatement_meets_the_model(lk, d, bn, regime, dt):
    if regime == "v-1e3" and dt != F16:
        pytest.skip("|V| near 1e3 is an f16 range case")
    g = torch.Generator().manual_seed(lk + d)
    q, k, v = _regime(regime, 128, lk, d, dt, g)
    out = _run(q, k, v, bn, dt)
    elem, row, nonzero = model_ratios(out, _model(q, k, v, d ** -0.5, dt))
    assert nonzero == 0 and elem <= 1.0 and row <= ROW_MAX, (elem, row)


@pytest.mark.parametrize("dt", [BF16, F16], ids=["bf16", "f16"])
@pytest.mark.parametrize("lkb", [1, 63, 64, 65, 200])
def test_restatement_kv_len(dt, lkb):
    """Keys past the batch's count filled with 1e4 take no weight."""
    g = torch.Generator().manual_seed(lkb)
    lk, d = 256, 64
    q, k, v = _regime("unit", 128, lk, d, dt, g)
    k[lkb:], v[lkb:] = 1e4, 1e4
    out = _run(q, k, v, 64, dt, lkb=lkb)
    elem, row, nonzero = model_ratios(out, _model(q, k, v, d ** -0.5, dt, lkb=lkb))
    assert nonzero == 0 and elem <= 1.0 and row <= ROW_MAX, (elem, row)


@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("l", [77, 300, 1000])
def test_restatement_causal(l, bn):
    g = torch.Generator().manual_seed(l)
    d = 64
    q, k, v = _regime("peaked", l, l, d, BF16, g)
    out = _restate(q, k, v, d ** -0.5, bn, BF16, causal=True).to(BF16)
    elem, row, _ = model_ratios(out, _model(q, k, v, d ** -0.5, BF16, causal=True))
    assert elem <= 1.0 and row <= ROW_MAX, (elem, row)


@pytest.mark.parametrize("dt", [BF16, F16], ids=["bf16", "f16"])
@pytest.mark.parametrize("n_sets", [2, 3, 8])
def test_restatement_sets(dt, n_sets):
    """Several sets (the cross-view add mode): per-set and partial-sum roundings inside the model."""
    g = torch.Generator().manual_seed(n_sets)
    lk, d = 333, 40
    q, _, _ = _regime("unit", 128, lk, d, dt, g)
    kvs = [_regime("v-offset" if s % 2 else "unit", 1, lk, d, dt, g)[1:] for s in range(n_sets)]
    out = _store([_restate(q, k, v, d ** -0.5, 128, dt) for k, v in kvs], dt)
    m = attention_model(q, lambda i: kvs, 1, 1, 128, d, d ** -0.5, dt)
    elem, row, _ = model_ratios(out, m)
    assert elem <= 1.0 and row <= ROW_MAX, (elem, row)


# (mutation, lk, d, bn, dt, xformers passes it): the mutations of the consumer loop that change values only, at shapes
# where the xformers tolerance does not see them (True) or does (False); every one exceeds tau under the model
MUTATIONS = [
    ("last-tile", 8400, 40, 128, True),
    ("last-tile", 1400, 80, 64, False),
    ("lkb-1", 8400, 40, 128, True),
    ("lkb-1", 1400, 80, 64, True),
    ("l-no-corr", 8400, 40, 128, False),
    ("l-no-corr", 1400, 80, 64, False),
]


@pytest.mark.parametrize("mutation,lk,d,bn,xformers", MUTATIONS, ids=[f"{m[0]}-lk{m[1]}-d{m[2]}" for m in MUTATIONS])
def test_mutations_exceed_tau(mutation, lk, d, bn, xformers):
    g = torch.Generator().manual_seed(lk + d)
    q, k, v = _regime("unit", 128, lk, d, BF16, g)
    out = _run(q, k, v, bn, BF16, mutation=mutation)
    m = _model(q, k, v, d ** -0.5, BF16)
    _, row, _ = model_ratios(out, m)
    assert row > TAU, row
    assert _xformers_passes(out, m.ref) == xformers


@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("l", [77, 300])
def test_causal_off_by_one_exceeds_tau(l, bn):
    """`>=` for `>` in the causal mask: every row loses its diagonal key (row 0, left with none, is NaN)."""
    g = torch.Generator().manual_seed(l)
    d = 64
    q, k, v = _regime("unit", l, l, d, BF16, g)
    out = _restate(q, k, v, d ** -0.5, bn, BF16, causal=True, mutation="causal>=").to(BF16)
    m = _model(q, k, v, d ** -0.5, BF16, causal=True)
    assert torch.isnan(out[0]).all()
    out[0] = m.ref[0].to(BF16)  # the other rows alone
    _, row, _ = model_ratios(out, m)
    assert row > TAU, row


def test_truncated_p_is_out_of_reach():
    """P packed by truncation biases every P element by u/2 on average: the worst row reaches 1.2-1.5 of the modelled σ
    against the unmutated 0.8-1.0, but not τ = 2; a τ between the two would leave the GPU kernel, whose worst row over
    thousands of rows and heads is not that of 128 restated rows, no margin."""
    g = torch.Generator().manual_seed(1)
    for lk, d, bn in [(8400, 40, 128), (1400, 80, 64)]:
        q, k, v = _regime("unit", 128, lk, d, BF16, g)
        m = _model(q, k, v, d ** -0.5, BF16)
        _, good, _ = model_ratios(_run(q, k, v, bn, BF16), m)
        _, trunc, _ = model_ratios(_run(q, k, v, bn, BF16, mutation="truncate"), m)
        assert good < trunc < TAU, (good, trunc)


@pytest.mark.parametrize("dt", [BF16, F16], ids=["bf16", "f16"])
def test_set_rounding_is_caught_by_composition(dt):
    """A set's output added without its own rounding stays inside the model (one rounding fewer than it counts), but the
    stored sum is then not the per-set outputs composed in the kernel's rounding order, which the GPU test checks bit for
    bit against one launch per set."""
    g = torch.Generator().manual_seed(5)
    lk, d, n_sets = 333, 40, 3
    q, _, _ = _regime("unit", 128, lk, d, dt, g)
    kvs = [_regime("unit", 1, lk, d, dt, g)[1:] for _ in range(n_sets)]
    sets = [_restate(q, k, v, d ** -0.5, 128, dt) for k, v in kvs]
    good, bad = _store(sets, dt), _store(sets, dt, "unrounded-set")
    m = attention_model(q, lambda i: kvs, 1, 1, 128, d, d ** -0.5, dt)
    _, row, _ = model_ratios(bad, m)
    assert row <= TAU
    composed = _store([o.to(dt).float() for o in sets], dt)  # what one launch per set, composed, gives
    assert torch.equal(composed, good) and not torch.equal(composed, bad)
