"""Every fused-attention entry point under the float64 error model of tests/attention_model.py: `attention` without and with
kv_index (1 to 8 sets, empty slots), `attention_multi` over three K/V sources, `attention(kv_len=...)` on the streaming
path and on the KVRES path (one set, lk <= 256, key tiles resident while a CTA walks its query tiles), `attention_causal`,
and the f16 twins of all but the causal kernel.  Head dims 32, 40, 64, 80 and 160; for bf16 each key-tile width
(MDB_ATTN_KERNEL tc2 | tc2d | tc); multi-Q on and off where it applies.  Key counts 1, BN - 1, BN, BN + 1, 98, 333, 1400,
5300 and 8400, query counts 1, 63, 64, 65, 127, 129 and 1400, causal lengths 77, 300 and 1000.

Each shape runs in the score regimes where an online softmax goes wrong: unit scores, peaked (q x 3), the row maximum in
the last key tile (every tile rescales by corr < 1), in the first (corr = 1 afterwards), scores over about ±100 in log2
units (most p underflow; f16 P goes subnormal), V offset by 20, and for f16 |V| near 1e3.  Keys past kv_len hold 1e4 in K
and V: they must take no weight.  Every output is guard-banded (test_kernel_edges_gpu.Guarded) and every case records its
worst elementwise and row ratios (tests/common.py::record, attention_model_gpu.txt).  Several sets are also checked bit for
bit against one launch per set composed in the kernel's rounding order: each set rounded to the storage type, added in fp32
to the stored partial sum, rounded again."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from magicdrive_b200 import ops  # noqa: E402
from tests.attention_model import attention_model, check_model  # noqa: E402
from tests.common import record  # noqa: E402
from tests.test_kernel_edges_gpu import ATTN_DT_KERNELS, BF16, F16, HEADS, Guarded, _gen, _randn, with_dt  # noqa: E402

DEV = "cuda"
REGIMES = ["unit", "peaked", "late-max", "early-max", "wide", "v-offset"]


def _regimes(dt):
    return REGIMES + (["v-1e3"] if dt == F16 else [])


def _bn(kernel, d):
    return {"tc2": 128 if d <= 64 else 64, "tc2d": 64, "tc": 128}[kernel]


def _shape_scores(regime, q, k, v, lk, heads, d):
    """Apply a score regime in place to fp32 q [rows, heads*d] and k / v [n*lk, heads*d] views (lk keys per batch)."""
    cols = torch.arange(heads, device=DEV) * d  # one column of each head carries the ramp
    ramp = (torch.arange(k.shape[0], device=DEV) % lk).float() / max(lk - 1, 1)
    if regime == "peaked":
        q.mul_(3)
    elif regime in ("late-max", "early-max"):
        q[:, cols] = 3.0
        k[:, cols] = (4.0 * math.sqrt(d) * (ramp if regime == "late-max" else 1 - ramp))[:, None]
    elif regime == "wide":
        q.mul_(25)
    elif regime == "v-offset":
        v.add_(20)
    elif regime == "v-1e3":
        v.mul_(250).add_(1000)


def _qkv(regime, g, b, lq, n_kv, lk, heads, d, dt):
    """q [b*lq, c] and kv [n_kv*lk, 2c] (K in the first c columns, V in the next) in `dt`."""
    c = heads * d
    q = _randn(b * lq, c, g=g)
    kv = _randn(n_kv * lk, 2 * c, g=g)
    _shape_scores(regime, q, kv[:, :c], kv[:, c:], lk, heads, d)
    return q.to(dt), kv.to(dt)


def _check(request, out, m, what):
    name = f"{request.node.name} {what}"
    out.check(name)
    elem, row = check_model(out.out, m, name)
    record(f"[attn-model] {name}: elementwise {elem:.3f} row {row:.3f}", "attention_model_gpu.txt")


def _sym(lk, bn):
    return {"BN-1": bn - 1, "BN": bn, "BN+1": bn + 1}.get(lk, lk)


# (lq, lk): every query count and every key count of one launch, the key-tile edges resolved per width
SHAPES = [(1, 1), (63, "BN-1"), (64, "BN"), (65, "BN+1"), (127, 98), (129, 333), (1400, 1400)]


@pytest.mark.parametrize("lq,lk", SHAPES, ids=[f"{a}x{b}" for a, b in SHAPES])
@pytest.mark.parametrize("d", list(HEADS))
@pytest.mark.parametrize("dt,kernel", ATTN_DT_KERNELS)
def test_attention_shapes(cuda_lib, monkeypatch, request, dt, kernel, d, lq, lk):
    """One set, kv_index=None."""
    monkeypatch.setenv("MDB_ATTN_KERNEL", kernel)
    heads, lk, b = HEADS[d], _sym(lk, _bn(kernel, d)), 2
    c = heads * d
    g = _gen(200 + d)
    for regime in _regimes(dt):
        q, kv = _qkv(regime, g, b, lq, b, lk, heads, d, dt)
        out = Guarded(b * lq, c, dt, ld=c + 16, col0=8)
        ops.attention(q, kv, kv[:, c:], b=b, heads=heads, lq=lq, lk=lk, d=d, ldq=c, ldk=2 * c, ldv=2 * c, scale=d ** -0.5,
                      out=out.out)
        m = attention_model(q, lambda i: [(kv[i * lk:(i + 1) * lk, :c], kv[i * lk:(i + 1) * lk, c:])], b, heads, lq, d,
                            d ** -0.5, dt)
        _check(request, out, m, regime)


@pytest.mark.parametrize("lk", [1, 98, "BN"])
@pytest.mark.parametrize("d", list(HEADS))
@pytest.mark.parametrize("dt,multiq", with_dt(["1", "0"]))
def test_attention_multi_q(cuda_lib, monkeypatch, request, dt, multiq, d, lk):
    """One key tile and more query tiles than SMs: with MDB_ATTN_MULTIQ=1 a CTA keeps its K/V tile and walks several query
    tiles."""
    monkeypatch.delenv("MDB_ATTN_KERNEL", raising=False)
    monkeypatch.setenv("MDB_ATTN_MULTIQ", multiq)
    heads, lk, b, lq = HEADS[d], _sym(lk, _bn("tc2", d)), 12, 1400
    c = heads * d
    assert b * heads * ((lq + 127) // 128) > torch.cuda.get_device_properties(0).multi_processor_count
    g = _gen(300 + d)
    for regime in ("unit", "late-max", "wide"):
        q, kv = _qkv(regime, g, b, lq, b, lk, heads, d, dt)
        out = Guarded(b * lq, c, dt, ld=c + 16, col0=8)
        ops.attention(q, kv, kv[:, c:], b=b, heads=heads, lq=lq, lk=lk, d=d, ldq=c, ldk=2 * c, ldv=2 * c, scale=d ** -0.5,
                      out=out.out)
        m = attention_model(q, lambda i: [(kv[i * lk:(i + 1) * lk, :c], kv[i * lk:(i + 1) * lk, c:])], b, heads, lq, d,
                            d ** -0.5, dt)
        _check(request, out, m, regime)


def _kv_views(x, c):
    """K and V of a [rows, 2C] buffer (columns 0 / C) or a [rows, 3C] one (columns C / 2C)."""
    return (x[:, :c], x[:, c:2 * c]) if x.shape[1] == 2 * c else (x[:, c:2 * c], x[:, 2 * c:])


def _compose(per_slot, present, dt):
    """The kernel's sum of several sets from one launch per slot: per batch, the first present set as stored, each next
    one added in fp32 to the stored partial sum and rounded to `dt`; zero where no set is present."""
    b, n_sets = present.shape
    acc = torch.zeros_like(per_slot[0])
    started = torch.zeros(b, dtype=torch.bool, device=DEV)
    for s in range(n_sets):
        o, here = per_slot[s], present[:, s]
        summed = (o.float() + acc.float()).to(dt)
        new = torch.where(started[:, None, None], summed, o)
        acc = torch.where(here[:, None, None], new, acc)
        started |= here
    return acc


@pytest.mark.parametrize("n_sets", range(1, 9))
@pytest.mark.parametrize("d", list(HEADS))
@pytest.mark.parametrize("dt,kernel", ATTN_DT_KERNELS)
def test_attention_sets(cuda_lib, monkeypatch, request, dt, kernel, d, n_sets):
    """kv_index with 1 to 8 sets: batch i < n_sets has slot i empty, batch n_sets none, batch n_sets + 1 all.  Odd set
    counts read K/V from three sources (attention_multi: 6 / 3 / 3 batches, row strides 2C / 2C / 3C), even ones from one
    (attention).  The sum is also bit for bit one launch per slot composed in the kernel's rounding order."""
    monkeypatch.setenv("MDB_ATTN_KERNEL", kernel)
    heads, lq, lk = HEADS[d], 150, 140
    c = heads * d
    n_src = 3 if n_sets % 2 else 1
    nb = [6, 3, 3][:n_src]
    b = n_sets + 2
    g = _gen(400 + n_sets)
    rows = [[None if (s == i or i == n_sets + 1) else ((i + s) % n_src, (5 * i + 3 * s) % nb[(i + s) % n_src])
             for s in range(n_sets)] for i in range(b)]
    idx = torch.tensor([[-1 if e is None else (e[0] << 24) | e[1] for e in r] for r in rows], dtype=torch.int32, device=DEV)
    present = idx >= 0
    for regime in ("unit", "v-offset") + (("v-1e3",) if dt == F16 else ()):
        q = _randn(b * lq, c, g=g)
        bufs = [_randn(nb[0] * lk, 2 * c, g=g), _randn(3 * lk, 2 * c, g=g), _randn(3 * lk, 3 * c, g=g)][:n_src]
        for x in bufs:  # these regimes shape V only
            _shape_scores(regime, q[:0], *_kv_views(x, c), lk, heads, d)
        q, bufs = q.to(dt), [x.to(dt) for x in bufs]
        views = [_kv_views(x, c) for x in bufs]
        srcs = [(k, v, x.shape[1], n) for (k, v), x, n in zip(views, bufs, nb)]

        def run(index, sets, out=None):
            if n_src == 1:
                return ops.attention(q, srcs[0][0], srcs[0][1], b=b, b_kv=nb[0], heads=heads, lq=lq, lk=lk, d=d, ldq=c,
                                     ldk=2 * c, ldv=2 * c, scale=d ** -0.5, kv_index=index, n_sets=sets, out=out)
            return ops.attention_multi(q, srcs, b=b, heads=heads, lq=lq, lk=lk, d=d, ldq=c, scale=d ** -0.5, kv_index=index,
                                       n_sets=sets, out=out)

        out = Guarded(b * lq, c, dt, ld=c + 16, col0=8)
        run(idx, n_sets, out.out)

        def kv_of(i):
            return [(views[e[0]][0][e[1] * lk:(e[1] + 1) * lk], views[e[0]][1][e[1] * lk:(e[1] + 1) * lk])
                    for e in rows[i] if e]

        _check(request, out, attention_model(q, kv_of, b, heads, lq, d, d ** -0.5, dt), regime)
        per_slot = [run(idx[:, s:s + 1].contiguous(), 1).reshape(b, lq, c) for s in range(n_sets)]
        assert torch.equal(out.out.reshape(b, lq, c), _compose(per_slot, present, dt)), f"{regime}: composition"


# (path, lq, lk, n_sets, MDB_ATTN_MULTIQ): kv_len on the streaming kernel (lk > 256, or several sets) and on the KVRES kernel
KV_LEN_PATHS = {"stream": (130, 333, 1, "1"), "stream-3sets": (130, 200, 3, "1"), "kvres": (1400, 200, 1, "1"),
                "kvres-one-q-tile": (1400, 200, 1, "0")}


@pytest.mark.parametrize("path", list(KV_LEN_PATHS))
@pytest.mark.parametrize("d", list(HEADS))
@pytest.mark.parametrize("dt,kernel", ATTN_DT_KERNELS)
def test_attention_kv_len(cuda_lib, monkeypatch, request, dt, kernel, d, path):
    """Per-batch key counts 0, 1, BN - 1, BN, BN + 1, lk and the clamped -5 and lk + 40; keys past the count hold 1e4 in K
    and V.  With three sets the middle slot is empty."""
    monkeypatch.setenv("MDB_ATTN_KERNEL", kernel)
    lq, lk, n_sets, multiq = KV_LEN_PATHS[path]
    monkeypatch.setenv("MDB_ATTN_MULTIQ", multiq)
    heads, bn = HEADS[d], _bn(kernel, d)
    c = heads * d
    lens = [0, 1, bn - 1, bn, bn + 1, lk, -5, lk + 40]
    eff = [min(max(x, 0), lk) for x in lens]
    b = len(lens)
    kv_len = torch.tensor(lens, dtype=torch.int32, device=DEV)
    slots = [[(i + 1) % b, -1, (i + 4) % b] for i in range(b)] if n_sets == 3 else [[i] for i in range(b)]
    idx = torch.tensor(slots, dtype=torch.int32, device=DEV) if n_sets == 3 else None
    # a set of query batch i counts eff[i] keys of the K/V batch it names: K/V batch j holds 1e4 past the most any reader counts
    counted = torch.tensor([max([eff[i] for i in range(b) if j in slots[i]], default=0) for j in range(b)], device=DEV)
    past = (torch.arange(b * lk, device=DEV) % lk >= counted.repeat_interleave(lk))[:, None]
    g = _gen(500 + d)
    for regime in ("unit", "late-max", "wide") + (("v-1e3",) if dt == F16 else ()):
        q, kv = _qkv(regime, g, b, lq, b, lk, heads, d, dt)
        kv = torch.where(past, torch.tensor(1e4, dtype=dt, device=DEV), kv)
        out = Guarded(b * lq, c, dt, ld=c + 16, col0=8)
        ops.attention(q, kv, kv[:, c:], b=b, heads=heads, lq=lq, lk=lk, d=d, ldq=c, ldk=2 * c, ldv=2 * c, scale=d ** -0.5,
                      kv_index=idx, n_sets=n_sets, kv_len=kv_len, out=out.out)

        def kv_of(i):
            n = eff[i]  # every set of query batch i counts that batch's keys
            return [(kv[j * lk:j * lk + n, :c], kv[j * lk:j * lk + n, c:]) for j in slots[i] if j >= 0]

        _check(request, out, attention_model(q, kv_of, b, heads, lq, d, d ** -0.5, dt), regime)


@pytest.mark.parametrize("l", [77, 300, 1000])
@pytest.mark.parametrize("d", list(HEADS))
@pytest.mark.parametrize("kernel", ["tc2", "tc2d", "tc"])
def test_attention_causal(cuda_lib, monkeypatch, request, kernel, d, l):
    """The CLIP text encoder's masked self-attention: several diagonal tiles at both key-tile widths."""
    monkeypatch.setenv("MDB_ATTN_KERNEL", kernel)
    heads, b = HEADS[d], 2
    c = heads * d
    g = _gen(600 + d)
    for regime in REGIMES:
        q = _randn(b * l, 3 * c, g=g)
        _shape_scores(regime, q[:, :c], q[:, c:2 * c], q[:, 2 * c:], l, heads, d)
        qkv = q.to(BF16)
        out = Guarded(b * l, c, BF16, ld=c + 16, col0=8)
        ops.attention_causal(qkv, qkv[:, c:], qkv[:, 2 * c:], b=b, heads=heads, l=l, d=d, ldq=3 * c, ldk=3 * c, ldv=3 * c,
                             scale=d ** -0.5, out=out.out)
        m = attention_model(qkv, lambda i: [(qkv[i * l:(i + 1) * l, c:2 * c], qkv[i * l:(i + 1) * l, 2 * c:])], b, heads, l,
                            d, d ** -0.5, BF16, causal=True)
        _check(request, out, m, regime)


@pytest.mark.parametrize("dt,l", with_dt([5300, 8400]))
def test_attention_long_self(cuda_lib, monkeypatch, request, dt, l):
    """The 424x800 level's 5300-token self-attention and the 'self' cross-view mode over six 1400-token views, from a
    fused-QKV buffer: at these lengths |o| is about 0.02 and one key tile handled wrongly hides under any absolute
    tolerance."""
    monkeypatch.delenv("MDB_ATTN_KERNEL", raising=False)
    heads, d = 8, 40
    c = heads * d
    g = _gen(700)
    for regime in ("unit", "late-max"):
        q = _randn(l, 3 * c, g=g)
        _shape_scores(regime, q[:, :c], q[:, c:2 * c], q[:, 2 * c:], l, heads, d)
        qkv = q.to(dt)
        out = Guarded(l, c, dt, ld=c + 16, col0=8)
        ops.attention(qkv, qkv[:, c:], qkv[:, 2 * c:], b=1, heads=heads, lq=l, lk=l, d=d, ldq=3 * c, ldk=3 * c, ldv=3 * c,
                      scale=d ** -0.5, out=out.out)
        m = attention_model(qkv, lambda i: [(qkv[:, c:2 * c], qkv[:, 2 * c:])], 1, heads, l, d, d ** -0.5, dt)
        _check(request, out, m, regime)
