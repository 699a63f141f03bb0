"""The folded LayerNorm and the row statistics it reads, `mdb_layernorm` and `mdb_softmax_rows`, against float64.

Most LayerNorms of the product never run as a LayerNorm kernel: every GEMM that writes a residual stream also writes per-row
(sum, sum of squares) partials, one slot per N tile (`stats_out`), and the GEMM that consumes LayerNorm(X) reads the raw X
and normalises in its epilogue, rstd * (acc - mean * colsum) + c.  This file holds both halves to elementwise bounds:

* every statistics slot against the float64 sum and sum of squares of the stored row segment it covers, within
  3e-5 * sum|x| and 3e-5 * sum x^2: the statistics describe the values as stored (bf16-rounded for bf16 outputs), because
  those are the values the consumer multiplies;
* every consumer output within one bf16 rounding step of ((X - mean) * rstd) @ W'^T + c in float64 (`_close_bf16`), where
  W' = bf16(W * gamma) and c = W beta + b, alone and chained behind a real producer at the engines' shapes.

Input rows have means 0, 16 and 64 standard deviations from zero, and a few rows per batch carry two outlier channels at
+-100 sigma (the massive-activation pattern of CLIP).  Isolated consumers also see exactly constant rows (variance 0: eps
and the clamp at zero decide the output) and rows whose variance is about eps.  Rows a few hundred sigma from zero are out
of scope for the fold: the fp32 (sum, sum sq) format itself loses their variance to cancellation.

Every output and statistics buffer is guard-banded as in test_kernel_edges_gpu.py."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from magicdrive_b200 import _lib, ops  # noqa: E402
from magicdrive_b200.params import pack_geglu  # noqa: E402
from tests.test_kernel_edges_gpu import BF16, F32, F64, Guarded, _bf, _close_bf16, _close_f32, _gen, _randn  # noqa: E402

OFFSETS = [0, 16, 64]  # row means, in standard deviations from zero
OUTLIER = 100.0
EPI = {"linear": 0, "geglu": 1, "qgelu": 2}  # mdb_gemm_desc.epi_mode
INVALID, UNSUPPORTED = -1, -3


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _hot_rows(m):
    """The rows of an m-row batch that carry two outlier channels."""
    return sorted({0, m // 3, (2 * m) // 3, m - 1})


def _rows(m, c, offset, g, hot=()):
    """fp32 [m, c]: N(0, 1) + per-channel means N(0, 0.25^2) + `offset`; rows in `hot` get +100 and -100 in two channels."""
    x = _randn(m, c, g=g) + _randn(c, g=g, scale=0.25) + offset
    for i, r in enumerate(hot):
        c0 = (37 * i + 5) % c
        c1 = (c0 + c // 2 + 3) % c
        x[r, c0] += OUTLIER
        x[r, c1] -= OUTLIER
    return x


def _desc(a, w, out, *, n_img=1, **kw):
    """mdb_gemm_desc of a token GEMM: a [M, K] bf16 view (M = n_img images of M / n_img rows), w [N, K], out a 2-D view;
    keyword arguments set the remaining fields (tensors by their address)."""
    m, k = a.shape
    d = _lib.GemmDesc()
    d.a0, d.c0, d.lda0 = a.data_ptr(), k, a.stride(0)
    d.n_img, d.h_in, d.w_in, d.h_out, d.w_out = n_img, 1, m // n_img, 1, m // n_img
    d.taps_h = d.taps_w = d.stride = 1
    d.w, d.n_out = w.data_ptr(), w.shape[0]
    d.out, d.ldo, d.out_scale = out.data_ptr(), out.stride(0), 1.0
    for key, v in kw.items():
        setattr(d, key, v.data_ptr() if torch.is_tensor(v) else v)
    return d


def _launch(d, what=""):
    L = _lib.lib()
    rc = L.mdb_gemm_conv(C.byref(d), _stream())
    assert rc == 0, f"{what}: mdb_gemm_conv returned {rc}: {L.mdb_last_error()}"


def _block_n(d):
    plan = (C.c_int * 5)()
    assert _lib.lib().mdb_gemm_conv_plan(C.byref(d), plan) == 0
    return plan[0]


def _check_stats(stats, stored, bn, what=""):
    """stats: the Guarded [rows, 2 * parts] fp32 statistics; stored: the [rows, n] output as written.  Slot nt must hold the
    sum and sum of squares of stored[:, nt*bn : min((nt+1)*bn, n)]."""
    stats.check(what + " statistics")
    x = stored.to(F64)
    m, n = x.shape
    parts = stats.cols // 2
    assert parts == -(-n // bn), (what, parts, n, bn)
    seg = F.pad(x, (0, parts * bn - n)).view(m, parts, bn)
    want = torch.stack([seg.sum(-1), (seg * seg).sum(-1)], -1)
    bound = 3e-5 * torch.stack([seg.abs().sum(-1), (seg * seg).sum(-1)], -1)
    got = stats.out.reshape(m, parts, 2).to(F64)
    bad = ((got - want).abs() > bound).nonzero()
    if bad.shape[0]:
        r, s, j = bad[0].tolist()
        raise AssertionError(f"{what}: {bad.shape[0]} statistics off, first at row {r} slot {s} "
                             f"({'sum' if j == 0 else 'sum sq'}): {got[r, s, j].item():.7g} vs {want[r, s, j].item():.7g} "
                             f"(bound {bound[r, s, j].item():.3g})")


def _producer(*, m, k, n, offset, n_img=1, bias=True, rowbias=None, residual=True, out_f32=False, out_scale=1.0,
              slice_=False, bn=0, variant=4, seed=0, what=""):
    """One guarded GEMM with row statistics.  The row means sit `offset` standard deviations from zero (carried by the
    residual when there is one, else by the bias); the outlier rows come through the residual, else through A.  Checks the
    output and every statistics slot; returns (output Guarded, statistics Guarded)."""
    assert bias or residual
    g = _gen(seed)
    hot = _hot_rows(m)
    a = _bf(_rows(m, k, 0.0, g, () if residual else hot))
    w = _bf(_randn(n, k, g=g, scale=k ** -0.5))
    b = _randn(n, g=g, scale=0.25) + (0.0 if residual else offset) if bias else None
    rb, rb_ld = None, 0
    if rowbias == "image":  # one row per image, a column slice of a wider table
        rb = _randn(n_img, n + 24, g=g, scale=0.5)[:, 8:8 + n]
        rb_ld = n + 24
    elif rowbias == "shared":  # one row for every image
        rb = _randn(1, n, g=g, scale=0.5)
    res = _bf(_rows(m, n, offset, g, hot)) if residual else None
    out = Guarded(m, n, F32 if out_f32 else BF16, ld=n + 24 if slice_ else None, col0=8 if slice_ else 0)
    kw = dict(n_img=n_img, out_is_f32=int(out_f32), out_scale=out_scale, force_block_n=bn, kernel_variant=variant,
              stats_out=1)
    if b is not None:
        kw["bias"] = b
    if rb is not None:
        kw.update(rowbias=rb, rowbias_ld=rb_ld)
    if res is not None:
        kw.update(residual=res, ldr=n)
    d = _desc(a, w, out.out, **kw)
    bn_used = _block_n(d)
    parts = _lib.lib().mdb_gemm_conv_stats_parts(C.byref(d))
    assert parts == -(-n // bn_used), (parts, n, bn_used)
    stats = Guarded(m, 2 * parts, F32)
    d.stats_out = stats.out.data_ptr()
    _launch(d, what)
    out.check(what)
    ref = a.to(F64) @ w.to(F64).t()
    if b is not None:
        ref = ref + b.to(F64)
    if rb is not None:
        ref = ref + (rb.to(F64).repeat_interleave(m // n_img, 0) if rb.shape[0] > 1 else rb.to(F64))
    ref = ref * out_scale
    if res is not None:
        ref = ref + res.to(F64)
    (_close_f32 if out_f32 else _close_bf16)(out.out, ref, what)
    _check_stats(stats, out.out, bn_used, what)
    return out, stats


def _fold_weights(n, c, g):
    """A LayerNorm(c) + Linear(c -> n) folded as the engines fold it: W' = bf16(W * gamma), colsum = sum_k W' in fp32,
    c = W beta + b."""
    w = _randn(n, c, g=g, scale=c ** -0.5)
    gamma = 1.0 + _randn(c, g=g, scale=0.3)
    beta = _randn(c, g=g, scale=0.2)
    b = _randn(n, g=g, scale=0.5)
    wg = _bf(w * gamma)
    return wg, wg.float().sum(1), (w.to(F64) @ beta.to(F64) + b.to(F64)).float()


def _fold_ref(x, wg, cvec, epi, eps):
    xd = x.to(F64)
    mu = xd.mean(1, keepdim=True)
    var = ((xd - mu) ** 2).mean(1, keepdim=True)
    h = ((xd - mu) * torch.rsqrt(var + eps)) @ wg.to(F64).t() + cvec.to(F64)
    if epi == "qgelu":
        return h * torch.sigmoid(1.702 * h)
    if epi == "geglu":
        val, gate = h.chunk(2, -1)
        return val * F.gelu(gate)
    return h


def _consume(x, stats, parts, wg, colsum, cvec, *, epi, eps, bn=0, variant=0, slice_=False, what=""):
    """One guarded consumer launch reading X = x, its statistics [rows, parts, 2] fp32 and the folded weights."""
    m = x.shape[0]
    n = wg.shape[0]
    if epi == "geglu":  # [128 value | 128 gate] tiles; the column sums and c are packed the same way
        wk, ck = pack_geglu(wg, cvec)
        _, csk = pack_geglu(wg.float(), colsum)
    else:
        wk, ck, csk = wg, cvec, colsum
    width = n // 2 if epi == "geglu" else n
    out = Guarded(m, width, ld=width + 16 if slice_ else None, col0=8 if slice_ else 0)
    d = _desc(x, wk, out.out, bias=ck, epi_mode=EPI[epi], force_block_n=bn, kernel_variant=variant, ln_stats=stats,
              ln_parts=parts, ln_eps=eps, ln_colsum=csk)
    _launch(d, what)
    out.check(what)
    _close_bf16(out.out, _fold_ref(x, wg, cvec, epi, eps), what)


# ------------------------------------------------------------------------------------------- a. producer statistics
PRODUCER_EPILOGUES = {
    "bias": dict(residual=False),  # proj_in
    "bias+residual": {},  # to_out, fc2
    "rowbias_image+scale+residual": dict(n_img=3, rowbias="image", out_scale=0.75),
    "rowbias_shared+residual": dict(n_img=3, rowbias="shared"),
    "f32+residual": dict(out_f32=True),
    "slice+residual": dict(slice_=True),
}


@pytest.mark.parametrize("case", list(PRODUCER_EPILOGUES))
@pytest.mark.parametrize("bn", [0, 64, 128, 160, 256], ids=["planner", "bn64", "bn128", "bn160", "bn256"])
@pytest.mark.parametrize("variant", [3, 4], ids=["pair", "single"])
@pytest.mark.parametrize("offset", OFFSETS)
def test_producer_statistics(cuda_lib, offset, variant, bn, case):
    """999 rows (an M tail, tiles spanning images) x 328 columns (an N tail for every block width), K = 320."""
    _producer(m=999, k=320, n=328, offset=offset, bn=bn, variant=variant, seed=40, what=case,
              **PRODUCER_EPILOGUES[case])


# (n_img, rows per image): single rows, 128k -+ 1, and the uneven-rig connector call (one image per view, per-view bias)
M_TAILS = {"m1": (1, 1), "m127": (1, 127), "m129": (1, 129), "rig_5x77": (5, 77), "rig_5x350": (5, 350)}


@pytest.mark.parametrize("tail", list(M_TAILS))
@pytest.mark.parametrize("variant", [3, 4], ids=["pair", "single"])
@pytest.mark.parametrize("offset", OFFSETS)
def test_producer_statistics_m_tails(cuda_lib, offset, variant, tail):
    n_img, rows = M_TAILS[tail]
    _producer(m=n_img * rows, k=320, n=320, offset=offset, n_img=n_img, rowbias="image" if n_img > 1 else None,
              variant=variant, seed=41, what=tail)


@pytest.mark.parametrize("bn", [64, 128, 160, 256])
@pytest.mark.parametrize("n_out", [8, 136])
@pytest.mark.parametrize("offset", OFFSETS)
def test_producer_statistics_n_tails(cuda_lib, offset, n_out, bn):
    _producer(m=300, k=320, n=n_out, offset=offset, bn=bn, seed=42, what=f"n_out={n_out}")


# ----------------------------------------------------------------------------------------------- b. isolated consumer
def _consumer_rows(m, c, offset, eps, g):
    """bf16 X: `offset` rows with outliers, three exactly constant rows and two rows of variance about eps."""
    x = _rows(m, c, offset, g, _hot_rows(m))
    for r, v in zip((10, 11, 12), (0.0, 0.75, -1.5)):
        x[r] = v
    for r in (20, 21):
        x[r] = math.sqrt(eps) * torch.where(_randn(c, g=g) > 0, 1.0, -1.0)
    return _bf(x)


def _split_stats(x, parts, g):
    """float64 (sum, sum sq) of the stored X over `parts` slots of unequal widths, cast to fp32 -> [rows, parts, 2]."""
    c = x.shape[1]
    cuts = (torch.randperm(c - 1, device="cuda", generator=g)[:parts - 1] + 1).sort().values.tolist()
    xd = x.to(F64)
    slots = [xd[:, a:b] for a, b in zip([0] + cuts, cuts + [c])]
    return torch.stack([torch.stack([s.sum(1), (s * s).sum(1)], -1) for s in slots], 1).float().contiguous()


# (ln_parts, consumer block_n, ln_eps, column-slice output): one launch each per test
CONSUMER_CALLS = [(1, 0, 1e-5, False), (2, 64, 1e-6, True), (3, 128, 1e-5, False), (5, 160, 1e-6, True),
                  (20, 256, 1e-5, True), (20, 0, 1e-6, False)]


@pytest.mark.parametrize("variant", [0, 3, 4], ids=["planner", "pair", "single"])
@pytest.mark.parametrize("epi", list(EPI))
@pytest.mark.parametrize("offset", OFFSETS)
def test_folded_layernorm_consumer(cuda_lib, offset, epi, variant):
    """Statistics built in float64 from the stored X and split over 1 to 20 slots; linear / GEGLU / quick-GELU epilogues,
    block widths 64 to 256 and the planner's, eps 1e-5 and 1e-6, contiguous and column-slice outputs (the kv projection
    of the view-sharded cross-view attention writes a column slice).  GEGLU always runs 256-wide tiles."""
    g = _gen(50)
    m, c = 300, 320
    n = 1024 if epi == "geglu" else 960
    wg, colsum, cvec = _fold_weights(n, c, g)
    for parts, bn, eps, slice_ in CONSUMER_CALLS:
        x = _consumer_rows(m, c, offset, eps, g)
        stats = _split_stats(x, parts, g)
        _consume(x, stats, parts, wg, colsum, cvec, epi=epi, eps=eps, bn=bn, variant=variant, slice_=slice_,
                 what=f"parts={parts} bn={bn} eps={eps} slice={slice_}")


# ------------------------------------------------------------------------------------- c. chains at the engines' shapes
UNET_CHAIN = {"28x50_C320": (16800, 320), "14x25_C640": (4200, 640), "7x13_C1280": (1092, 1280),
              "4x7_C1280": (336, 1280)}


@pytest.mark.parametrize("producer", ["proj_in", "to_out"])
@pytest.mark.parametrize("shape", list(UNET_CHAIN))
@pytest.mark.parametrize("offset", OFFSETS)
def test_chain_unet(cuda_lib, offset, shape, producer):
    """A transformer block's residual stream: proj_in (bias) or to_out (bias + residual) writes X and its statistics
    with the planner's tiling, and the QKV, q, kv (column slice) and GEGLU projections normalise it in their epilogues."""
    m, c = UNET_CHAIN[shape]
    x, stats = _producer(m=m, k=c, n=c, offset=offset, residual=producer == "to_out", variant=0, seed=43,
                         what=f"{producer} {shape}")
    parts = stats.cols // 2
    g = _gen(44)
    for name, n, epi in (("qkv", 3 * c, "linear"), ("q", c, "linear"), ("kv", 2 * c, "linear"), ("ff", 8 * c, "geglu")):
        wg, colsum, cvec = _fold_weights(n, c, g)
        _consume(x.out, stats.out, parts, wg, colsum, cvec, epi=epi, eps=1e-5, slice_=name == "kv",
                 what=f"{producer} {shape} -> {name}")


@pytest.mark.parametrize("producer", ["embed", "fc2"])
@pytest.mark.parametrize("m", [77, 154, 924])
@pytest.mark.parametrize("offset", OFFSETS)
def test_chain_clip(cuda_lib, offset, m, producer):
    """The text encoder's residual stream: the token + position embedding or an fc2-like GEMM (K = 3072, bias +
    residual) writes X and its statistics; the fused QKV projection and fc1 with quick-GELU normalise it."""
    c = 768
    if producer == "embed":
        g = _gen(45)
        vocab = 1000
        tok = _bf(_rows(vocab, c, offset, g, _hot_rows(vocab)))
        pos = _bf(_randn(77, c, g=g, scale=0.3))
        ids = torch.randint(0, vocab, (m // 77, 77), device="cuda", generator=g, dtype=torch.int32)
        ids[:, 5], ids[-1, -1] = 0, vocab - 1  # outlier tokens in every sequence
        x = Guarded(m, c, ld=c + 16, col0=8)
        stats = Guarded(m, 2, F32)
        rc = cuda_lib.mdb_clip_embed(ids.data_ptr(), 0, m // 77, 77, tok.data_ptr(), vocab, pos.data_ptr(), c,
                                     x.out.data_ptr(), x.ld, stats.out.data_ptr(), _stream())
        assert rc == 0, cuda_lib.mdb_last_error()
        x.check("embed")
        assert torch.equal(x.out, (tok[ids.long()] + pos[None]).reshape(m, c))
        _check_stats(stats, x.out, c, "embed")
    else:
        x, stats = _producer(m=m, k=3072, n=c, offset=offset, variant=0, seed=46, what="fc2")
    parts = stats.cols // 2
    g = _gen(47)
    for name, n, epi in (("qkv", 3 * c, "linear"), ("fc1", 4 * c, "qgelu")):
        wg, colsum, cvec = _fold_weights(n, c, g)
        _consume(x.out, stats.out, parts, wg, colsum, cvec, epi=epi, eps=1e-5, what=f"{producer} M={m} -> {name}")


# ------------------------------------------------------------------------------------------ d. planner and validation
def test_split_k_request_with_statistics_runs_unsplit(cuda_lib):
    """force_splits > 1 is ignored, not obeyed, when the launch writes or reads row statistics: split-K partials carry no
    statistics, and a partial sum cannot be normalised."""
    L = _lib.lib()
    g = _gen(48)
    m, k, n = 256, 1280, 320
    a = _bf(_rows(m, k, 0.0, g))
    w = _bf(_randn(n, k, g=g, scale=k ** -0.5))
    res = _bf(_rows(m, n, 16, g, _hot_rows(m)))
    ws = ops.workspace(64 << 20, a.device)
    split = dict(workspace=ws.data_ptr(), workspace_bytes=ws.numel(), force_splits=4, kernel_variant=0)
    scratch = torch.empty(m, 3 * n, dtype=BF16, device="cuda")
    assert L.mdb_gemm_conv_launches(C.byref(_desc(a, w, scratch[:, :n], residual=res, ldr=n, **split))) == 2

    x = Guarded(m, n)
    d = _desc(a, w, x.out, residual=res, ldr=n, stats_out=1, **split)
    assert L.mdb_gemm_conv_launches(C.byref(d)) == 1
    bn = _block_n(d)
    stats = Guarded(m, 2 * (-(-n // bn)), F32)
    d.stats_out = stats.out.data_ptr()
    _launch(d, "producer")
    x.check("producer")
    _close_bf16(x.out, a.to(F64) @ w.to(F64).t() + res.to(F64), "producer")
    _check_stats(stats, x.out, bn, "producer")

    wg, colsum, cvec = _fold_weights(3 * n, n, g)
    assert L.mdb_gemm_conv_launches(C.byref(_desc(x.out, wg, scratch, bias=cvec, **split))) == 2
    y = Guarded(m, 3 * n)
    d = _desc(x.out, wg, y.out, bias=cvec, ln_stats=stats.out, ln_parts=stats.cols // 2, ln_eps=1e-5, ln_colsum=colsum,
              **split)
    assert L.mdb_gemm_conv_launches(C.byref(d)) == 1
    _launch(d, "consumer")
    y.check("consumer")
    _close_bf16(y.out, _fold_ref(x.out, wg, cvec, "linear", 1e-5), "consumer")


def test_folded_layernorm_and_statistics_rejections(cuda_lib):
    L = _lib.lib()
    m, c = 128, 64
    a = torch.zeros(m, c, dtype=BF16, device="cuda")
    w3 = torch.zeros(256, 9 * c, dtype=BF16, device="cuda")
    w = torch.zeros(256, c, dtype=BF16, device="cuda")
    out = torch.empty(m, 256, dtype=BF16, device="cuda")
    stats = torch.zeros(m, 4, 2, dtype=F32, device="cuda")
    colsum = torch.zeros(256, dtype=F32, device="cuda")
    ln = dict(ln_stats=stats, ln_parts=1, ln_eps=1e-5, ln_colsum=colsum)
    st = _stream()

    conv = _desc(a, w3, out, **ln)  # a 3x3 convolution over one 8 x 16 image
    conv.h_in, conv.w_in, conv.h_out, conv.w_out = 8, 16, 8, 16
    conv.taps_h = conv.taps_w = 3
    conv.pad_h = conv.pad_w = 1
    assert L.mdb_gemm_conv(C.byref(conv), st) == INVALID
    assert L.mdb_gemm_conv(C.byref(_desc(a, w, out, **{**ln, "ln_colsum": None})), st) == INVALID
    assert L.mdb_gemm_conv(C.byref(_desc(a, w, out, **{**ln, "ln_parts": 0})), st) == INVALID
    geglu = _desc(a, w, out[:, :128], epi_mode=1, stats_out=stats)
    assert L.mdb_gemm_conv(C.byref(geglu), st) == UNSUPPORTED
    assert L.mdb_gemm_conv(C.byref(_desc(a, w, out, **ln)), st) == 0  # the same inputs, well formed
    geglu.stats_out = None
    assert L.mdb_gemm_conv(C.byref(geglu), st) == 0
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------- e. mdb_layernorm
LN_C = [8, 64, 320, 512, 520, 768, 1280, 1288, 2048]  # both sides of the 512 / 1280 kernel boundaries, and the maximum
LN_ROWS = [1, 7, 9, 77, 1003, 16800]


@pytest.mark.parametrize("offset", [0, 16, 64, 256])
@pytest.mark.parametrize("c", LN_C)
def test_layernorm_kernel(cuda_lib, c, offset):
    """Two-pass LayerNorm: rows whose means sit up to 256 sigma from zero, inputs dense (ldx = C), padded (C + 8) or a
    column slice of a fused [rows, 3C] buffer, output into a column slice of a wider buffer, eps 1e-5 and 1e-6."""
    g = _gen(51)
    gamma = 1.0 + _randn(c, g=g, scale=0.3)
    beta = _randn(c, g=g, scale=0.2)
    for i, rows in enumerate(LN_ROWS):
        layout = ("dense", "padded", "fused")[i % 3]
        eps = (1e-5, 1e-6)[i % 2]
        ldx = {"dense": c, "padded": c + 8, "fused": 3 * c}[layout]
        col0 = c if layout == "fused" else 0
        buf = _bf(_randn(rows, ldx, g=g, scale=1e3))  # whatever lies beside the row must not leak in
        x = buf[:, col0:col0 + c]
        x.copy_(_bf(_rows(rows, c, offset, g, _hot_rows(rows))))
        out = Guarded(rows, c, ld=c + 16, col0=8)
        rc = cuda_lib.mdb_layernorm(x.data_ptr(), rows, c, ldx, gamma.data_ptr(), beta.data_ptr(), eps,
                                    out.out.data_ptr(), out.ld, _stream())
        what = f"rows={rows} {layout} eps={eps}"
        assert rc == 0, (what, cuda_lib.mdb_last_error())
        out.check(what)
        _close_bf16(out.out, F.layer_norm(x.to(F64), (c,), gamma.to(F64), beta.to(F64), eps), what)


def test_layernorm_rejects_unsupported(cuda_lib):
    x = torch.zeros(4, 2 * 2056, dtype=BF16, device="cuda")
    out = torch.empty_like(x)
    gb = torch.zeros(2056, dtype=F32, device="cuda")
    for c, ldx in ((2056, 2056), (12, 16), (64, 68)):
        rc = cuda_lib.mdb_layernorm(x.data_ptr(), 4, c, ldx, gb.data_ptr(), gb.data_ptr(), 1e-5, out.data_ptr(), 2056,
                                    _stream())
        assert rc == UNSUPPORTED, (c, ldx, rc)


# ---------------------------------------------------------------------------------------------- f. mdb_softmax_rows
@pytest.mark.parametrize("kind", ["normal", "peaked", "shifted"])
@pytest.mark.parametrize("pad", [False, True], ids=["unpadded", "padded"])
@pytest.mark.parametrize("cols", [1, 31, 32, 33, 77, 1400])
def test_softmax_rows(cuda_lib, cols, pad, kind):
    """Scores N(0, 1), x30 (peaked) or shifted by +1e4, read with a row stride past `cols` (the columns there are NaN and
    must not be read); probabilities written with a row stride past `cols_out`, and the padding columns up to the next
    multiple of 64 exactly zero."""
    g = _gen(52)
    rows = 37
    cols_out = -(-cols // 64) * 64 if pad else cols
    lds = cols + 5
    s = torch.full((rows, lds), float("nan"), dtype=F32, device="cuda")
    s[:, :cols] = _randn(rows, cols, g=g, scale=30.0 if kind == "peaked" else 1.0) + (1e4 if kind == "shifted" else 0.0)
    out = Guarded(rows, cols_out, ld=cols_out + 16, col0=8)
    rc = cuda_lib.mdb_softmax_rows(s.data_ptr(), lds, rows, cols, out.out.data_ptr(), out.ld, cols_out, _stream())
    assert rc == 0, cuda_lib.mdb_last_error()
    out.check()
    _close_bf16(out.out[:, :cols], torch.softmax(s[:, :cols].to(F64), -1))
    assert (out.out[:, cols:].view(torch.int16) == 0).all(), "padding columns are not +0"
