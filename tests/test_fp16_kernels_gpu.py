"""The f16 instantiations of the denoising step's kernels (models with fp16 parameters): GEMM / implicit-GEMM convolution with
every epilogue the step uses, fused attention, GroupNorm(+SiLU) and the glue, each against float64 (attention under the error
model of tests/attention_model.py) and every output guard-banded as in test_kernel_edges_gpu.py, which runs the same kernels
at the tiling edges in both element types.  Here: fp16's own range (overflow to inf, subnormal results and operands), and
the operators' refusal of operands whose element types disagree."""
import math
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from magicdrive_b200 import f16_ops, ops  # noqa: E402
from magicdrive_b200.params import pack_geglu  # noqa: E402
from tests.attention_model import attention_model, check_model  # noqa: E402
from tests.test_kernel_edges_gpu import BF16, F16, F32, F64, Guarded, _close_f16  # noqa: E402


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _randn(*shape, g, scale=1.0):
    return (torch.randn(*shape, device="cuda", generator=g) * scale).to(F16)


def _conv_ref(a, w, n, h, wd, cin, cout, taps, pad):
    x = a.to(F64).reshape(n, h, wd, cin).permute(0, 3, 1, 2)
    k = w.to(F64).reshape(cout, taps, taps, cin).permute(0, 3, 1, 2)
    return F.conv2d(x, k, padding=pad).permute(0, 2, 3, 1).reshape(-1, cout)


# ---------------------------------------------------------------------------------------------------------------- GEMM
@pytest.mark.parametrize("bn", [64, 128, 160, 256])
@pytest.mark.parametrize("m,k,n", [(300, 320, 320), (1000, 136, 168), (129, 64, 512)])
def test_linear_bias_residual_scale(cuda_lib, bn, m, k, n):
    g = _gen(1)
    a, w = _randn(m, k, g=g), _randn(n, k, g=g, scale=k ** -0.5)
    bias, res = torch.randn(n, device="cuda", generator=g), _randn(m, n, g=g)
    o = Guarded(m, n, F16)
    wk = F.pad(w, (0, -k % 64))  # K64 layout: a partial last K block reads zeros past k
    ops.linear(a, wk, bias=bias, residual=res, out=o.out, ldo=n, out_scale=0.7, force_block_n=bn, allow_split_k=False)
    o.check(f"linear bn={bn}")
    _close_f16(o.out, 0.7 * (a.to(F64) @ w.to(F64).T + bias.to(F64)) + res.to(F64), f"linear bn={bn} {m}x{k}x{n}")


@pytest.mark.parametrize("n_img,h,w,c0,c1,cout", [(2, 14, 25, 64, 0, 128), (3, 7, 13, 64, 128, 160), (1, 9, 11, 40, 24, 64)])
def test_conv3x3_two_sources_rowbias(cuda_lib, n_img, h, w, c0, c1, cout):
    """Implicit-GEMM 3x3 convolution over the concat of two f16 sources, with the per-image time shift."""
    from magicdrive_b200.params import pack_conv_weight_k64
    g = _gen(2)
    pix = n_img * h * w
    a0, a1 = _randn(pix, c0, g=g), _randn(pix, max(c1, 8), g=g)
    wt = torch.randn(cout, c0 + c1, 3, 3, device="cuda", generator=g) * (9 * (c0 + c1)) ** -0.5
    wk = pack_conv_weight_k64(wt.to(F16).float(), splits=[c0, c1] if c1 else None, dtype=F16)
    bias, rowbias = torch.randn(cout, device="cuda", generator=g), torch.randn(n_img, cout, device="cuda", generator=g)
    o = Guarded(pix, cout, F16)
    ops.gemm_conv(a0, wk, n_img=n_img, h_in=h, w_in=w, c0=c0, lda0=c0, a1=a1 if c1 else None, c1=c1, lda1=a1.stride(0),
                  n_out=cout, taps=3, pad=1, bias=bias, rowbias=rowbias, out=o.out, ldo=cout)
    o.check("conv3x3")
    x = torch.cat([a0.to(F64), a1[:, :c1].to(F64)], 1) if c1 else a0.to(F64)
    ref = _conv_ref(x, wt.to(F16).permute(0, 2, 3, 1).reshape(cout, -1), n_img, h, w, c0 + c1, cout, 3, 1)
    ref = ref + bias.to(F64) + rowbias.to(F64).repeat_interleave(h * w, 0)
    _close_f16(o.out, ref, "conv3x3 two sources")


def test_forced_split_k_with_residual_and_f32_output(cuda_lib):
    g = _gen(3)
    m, k, n = 200, 1280, 320
    a, w = _randn(m, k, g=g), _randn(n, k, g=g, scale=k ** -0.5)
    bias, res = torch.randn(n, device="cuda", generator=g), _randn(m, n, g=g)
    ref = a.to(F64) @ w.to(F64).T + bias.to(F64)
    o = Guarded(m, n, F16)
    ops.linear(a, w, bias=bias, residual=res, out=o.out, ldo=n, force_splits=4)
    o.check("split-K")
    _close_f16(o.out, ref + res.to(F64), "split-K + residual")
    o32 = Guarded(m, n, F32)
    ops.linear(a, w, bias=bias, out=o32.out, ldo=n, out_f32=True, force_splits=3)
    o32.check("split-K fp32")
    err = (o32.out.to(F64) - ref).abs().max().item()
    assert err <= 3e-5 * ref.abs().max().item(), err


@pytest.mark.parametrize("bn", [128, 160, 256])
def test_residual_aliases_the_output(cuda_lib, bn):
    """The zero convolutions add into the UNet skip in place: residual == out, in a column slice of a wider buffer."""
    g = _gen(4)
    m, k, n, ld = 700, 320, 320, 640
    a, w = _randn(m, k, g=g), _randn(n, k, g=g, scale=k ** -0.5)
    buf = _randn(m, ld, g=g)
    before = buf.clone()
    view = buf[:, 160:160 + n]
    ops.linear(a, w, residual=view, out=view, ldo=ld, out_scale=0.5, force_block_n=bn, allow_split_k=False)
    torch.cuda.synchronize()
    _close_f16(view, 0.5 * (a.to(F64) @ w.to(F64).T) + before[:, 160:160 + n].to(F64), f"in place bn={bn}")
    assert torch.equal(buf[:, :160], before[:, :160]) and torch.equal(buf[:, 160 + n:], before[:, 160 + n:])


def test_geglu(cuda_lib):
    g = _gen(5)
    m, k, inner = 333, 320, 1280
    a = _randn(m, k, g=g)
    wf, bf = torch.randn(2 * inner, k, device="cuda", generator=g) * k ** -0.5, torch.randn(2 * inner, device="cuda", generator=g)
    wp, bp = pack_geglu(wf, bf, dtype=F16)
    o = Guarded(m, inner, F16)
    ops.linear(a, wp, bias=bp, geglu=True, out=o.out, ldo=inner)
    o.check("geglu")
    y = a.to(F64) @ wf.to(F16).to(F64).T + bf.to(F64)
    _close_f16(o.out, y[:, :inner] * F.gelu(y[:, inner:]), "geglu")


@pytest.mark.parametrize("offset", [0.0, 30.0])
def test_row_statistics_and_folded_layernorm(cuda_lib, offset):
    """The producer's row statistics are those of its f16-rounded stored values; the consumer folds LayerNorm(gamma, beta)
    into its weights (W * gamma rounded to f16) and normalises with them."""
    g = _gen(6)
    m, k, c, n = 500, 320, 320, 960
    a, w = _randn(m, k, g=g), _randn(c, k, g=g, scale=k ** -0.5)
    bias = torch.randn(c, device="cuda", generator=g) + offset
    x, st = ops.linear(a, w, bias=bias, emit_stats=True)
    torch.cuda.synchronize()
    xs = x.to(F64)
    tot = st.data.to(F64).sum(1)
    assert torch.allclose(tot[:, 0], xs.sum(1), rtol=1e-5, atol=1e-4 * c), "row sums"
    assert torch.allclose(tot[:, 1], (xs * xs).sum(1), rtol=1e-5, atol=1e-4 * c), "row sums of squares"
    gam, beta = 1 + 0.1 * torch.randn(c, device="cuda", generator=g), 0.1 * torch.randn(c, device="cuda", generator=g)
    wl, bl = torch.randn(n, c, device="cuda", generator=g) * c ** -0.5, torch.randn(n, device="cuda", generator=g)
    wg = (wl * gam[None]).to(F16)
    cvec = wl @ beta + bl
    o = Guarded(m, n, F16)
    ops.linear(x, wg, bias=cvec, ln=st, ln_colsum=wg.float().sum(1), ln_eps=1e-5, out=o.out, ldo=n)
    o.check("folded layernorm")
    ref = F.layer_norm(xs, (c,), eps=1e-5) @ wg.to(F64).T + cvec.to(F64)
    err = (o.out.to(F64) - ref).abs()
    assert (err <= ref.abs() * 2.0 ** -10 + 2e-3 * ref.abs().max()).all(), err.max().item()


def test_f16_rejections(cuda_lib):
    g = _gen(7)
    a, w = _randn(128, 64, g=g), _randn(64, 64, g=g)
    for kw in (dict(quick_gelu=True), dict(relu=True), dict(kernel_variant=3)):
        with pytest.raises(Exception):
            ops.linear(a, w, **kw)


# ---------------------------------------------------------------------------------------------------------- attention
def _attn_ref(q, k, v, b, heads, lq, lk, d, scale, n_keys=None):
    """The float64 attention of q [b*lq, C] over k / v [b*lk, C] (the first n_keys[i] keys of batch i) and its error model
    (tests/attention_model.py)."""
    n = [lk] * b if n_keys is None else n_keys.tolist()
    return attention_model(q, lambda i: [(k[i * lk:i * lk + n[i]], v[i * lk:i * lk + n[i]])], b, heads, lq, d, scale, F16)


@pytest.mark.parametrize("d", [32, 40, 64, 80, 160])
@pytest.mark.parametrize("lq,lk", [(350, 350), (700, 97)])
def test_attention(cuda_lib, d, lq, lk):
    g = _gen(8)
    b, heads = 3, 2
    q, k, v = (_randn(n, heads * d, g=g) for n in (b * lq, b * lk, b * lk))
    o = Guarded(b * lq, heads * d, F16)
    ops.attention(q, k, v, b=b, heads=heads, lq=lq, lk=lk, d=d, ldq=heads * d, ldk=heads * d, ldv=heads * d,
                  scale=d ** -0.5, out=o.out)
    o.check(f"attention d={d}")
    check_model(o.out, _attn_ref(q, k, v, b, heads, lq, lk, d, d ** -0.5), f"attention d={d}")


@pytest.mark.parametrize("d", [40, 64, 80])
def test_attention_add_sets_with_empty_slots(cuda_lib, d):
    """Cross-view "add" mode: per-set softmax, each set's output rounded to f16 before the sum in slot order; -1 slots add
    nothing, [a, -1, b] is bitwise [a, b] and a row with no present set is zero."""
    g = _gen(9)
    b, heads, L = 4, 2, 200
    qkv = _randn(b * L, 3 * heads * d, g=g)
    C = heads * d
    q, k, v = qkv, qkv[:, C:], qkv[:, 2 * C:]
    idx3 = torch.tensor([[1, -1, 3], [0, -1, 2], [-1, -1, -1], [2, -1, 0]], dtype=torch.int32, device="cuda")
    idx2 = torch.tensor([[1, 3], [0, 2], [-1, -1], [2, 0]], dtype=torch.int32, device="cuda")
    kw = dict(b=b, heads=heads, lq=L, lk=L, d=d, ldq=3 * C, ldk=3 * C, ldv=3 * C, scale=d ** -0.5)
    o3 = ops.attention(q, k, v, kv_index=idx3, n_sets=3, **kw)
    o2 = ops.attention(q, k, v, kv_index=idx2, n_sets=2, **kw)
    torch.cuda.synchronize()
    assert torch.equal(o3, o2)
    for i, row in enumerate(idx2.tolist()):
        present = [j for j in row if j >= 0]
        if not present:
            assert (o3.reshape(b, L, C)[i] == 0).all()
            continue
        t = qkv.reshape(b, L, 3 * C)
        qi = t[i, :, :C].contiguous()
        kvs = [(t[j, :, C:2 * C], t[j, :, 2 * C:]) for j in present]
        check_model(o3.reshape(b, L, C)[i], attention_model(qi, lambda _: kvs, 1, heads, L, d, d ** -0.5, F16),
                    f"add mode d={d} row {i}")


@pytest.mark.parametrize("d", [40, 80, 160])
def test_attention_kv_len_resident_and_multi_q_bitwise(cuda_lib, d):
    """kv_len (the KVRES kernel of a box capacity) is bitwise the exact-length launch; multi-Q launches are bitwise the
    one-query-tile-per-CTA launch."""
    g = _gen(10)
    b, heads, lq, cap = 12, 8, 1400, 256
    C = heads * d
    q, kv = _randn(b * lq, C, g=g), _randn(b * cap, 2 * C, g=g)
    lens = torch.tensor([78 + (7 * i) % 150 for i in range(b)], dtype=torch.int32, device="cuda")
    kw = dict(b=b, heads=heads, lq=lq, d=d, ldq=C, ldk=2 * C, ldv=2 * C, scale=d ** -0.5)
    o = ops.attention(q, kv, kv[:, C:], lk=cap, kv_len=lens, **kw)
    torch.cuda.synchronize()
    for i in (0, 5, 11):
        n = int(lens[i])
        kvi = kv.reshape(b, cap, 2 * C)[i, :n].contiguous()
        oi = ops.attention(q.reshape(b, lq, C)[i].contiguous(), kvi, kvi[:, C:], lk=n, **dict(kw, b=1))
        torch.cuda.synchronize()
        assert torch.equal(o.reshape(b, lq, C)[i], oi), (d, i)
    check_model(o, _attn_ref(q, kv[:, :C], kv[:, C:], b, heads, lq, cap, d, d ** -0.5, lens), f"kv_len d={d}")
    # multi-Q: one key tile (lk <= BN), more query tiles than SMs hold at once
    lk = 64
    kv2 = kv[: b * lk]
    prev = os.environ.get("MDB_ATTN_MULTIQ")
    try:
        os.environ["MDB_ATTN_MULTIQ"] = "0"
        one = ops.attention(q, kv2, kv2[:, C:], lk=lk, **kw)
        os.environ.pop("MDB_ATTN_MULTIQ")
        multi = ops.attention(q, kv2, kv2[:, C:], lk=lk, **kw)
        torch.cuda.synchronize()
    finally:
        if prev is not None:
            os.environ["MDB_ATTN_MULTIQ"] = prev
    assert torch.equal(one, multi), d


# ---------------------------------------------------------------------------------------------------------- GroupNorm
@pytest.mark.parametrize("rows", ["0", "1"])
@pytest.mark.parametrize("n_img,hw,c0,c1,silu", [(12, 350, 320, 0, True), (6, 1400, 640, 320, True), (4, 91, 1280, 0, False)])
def test_groupnorm(cuda_lib, monkeypatch, rows, n_img, hw, c0, c1, silu):
    """gn_fused_kernel (MDB_GN_ROWS=0) and the cluster gn_rows_kernel (=1), two sources included."""
    monkeypatch.setenv("MDB_GN_ROWS", rows)
    g = _gen(11)
    x0, x1 = _randn(n_img * hw, c0, g=g, scale=3.0), _randn(n_img * hw, max(c1, 8), g=g)
    x0 = (x0.float() + 5.0).half()
    gam, beta = 1 + 0.1 * torch.randn(c0 + c1, device="cuda", generator=g), 0.1 * torch.randn(c0 + c1, device="cuda", generator=g)
    out = ops.groupnorm(x0, c0, c0, n_img, hw, gam, beta, 1e-5, silu, x1=x1 if c1 else None, c1=c1, ld1=x1.stride(0))
    torch.cuda.synchronize()
    assert out.dtype == F16
    x = torch.cat([x0.to(F64), x1[:, :c1].to(F64)], 1) if c1 else x0.to(F64)
    y = F.group_norm(x.reshape(n_img, hw, -1).permute(0, 2, 1), 32, gam.to(F64), beta.to(F64), 1e-5)
    y = (F.silu(y) if silu else y).permute(0, 2, 1).reshape(n_img * hw, -1)
    _close_f16(out, y, f"groupnorm rows={rows}")


# ---------------------------------------------------------------------------------------------------------------- glue
def test_conversions_over_every_f16_pattern(cuda_lib):
    bits = torch.arange(-32768, 32768, dtype=torch.int32, device="cuda").to(torch.int16)
    h = bits.view(F16)
    f = f16_ops.f16_to_f32(h.contiguous())
    torch.cuda.synchronize()
    assert torch.equal(f.view(torch.int32), h.float().view(torch.int32))
    # every finite pattern, and the midpoints between neighbours (ties round to even) and just off them
    fin = f[torch.isfinite(f)].to(F64).unique()
    mids = (fin[1:] + fin[:-1]) / 2
    x = torch.cat([fin, mids, mids * (1 + 2.0 ** -20), mids * (1 - 2.0 ** -20), torch.tensor([7e4, -7e4, 65520.0], device="cuda",
                                                                                             dtype=F64)]).float()
    x = torch.cat([x, torch.tensor([float("nan"), float("inf"), -float("inf")], device="cuda")])
    y = f16_ops.f32_to_f16(x.contiguous())
    torch.cuda.synchronize()
    ref = x.half()
    same = (y.view(torch.int16) == ref.view(torch.int16)) | (torch.isnan(y) & torch.isnan(ref))
    assert same.all(), x[~same][:8]


def test_add_upsample_pack_bitwise(cuda_lib):
    g = _gen(12)
    a, b = _randn(6 * 28 * 50, 320, g=g, scale=40.0), _randn(6 * 28 * 50, 320, g=g, scale=40.0)
    s = ops.add(a, b)
    x = _randn(2 * 14 * 25, 640, g=g)
    u = ops.upsample_nearest(x, 2, 14, 25, 640, 28, 50)
    lat = torch.randn(6 * 28 * 50, 4, device="cuda", generator=g)
    p = f16_ops.pack_latents_f16(lat, 64, repeat=2)
    torch.cuda.synchronize()
    assert s.dtype == u.dtype == p.dtype == F16
    assert torch.equal(s, a + b)
    ref = F.interpolate(x.reshape(2, 14, 25, 640).permute(0, 3, 1, 2), size=(28, 50), mode="nearest")
    assert torch.equal(u, ref.permute(0, 2, 3, 1).reshape(-1, 640))
    assert torch.equal(p, F.pad(lat, (0, 60)).half().repeat(2, 1))


# ------------------------------------------------------------------------------------------------------------ fp16 range
# Every f16 store rounds the fp32 result to nearest even (__floats2half2_rn / __float2half_rn, Act<true> in csrc/ptx.cuh):
# magnitudes from 65520 up become inf, as torch's fp16 rounding of the same exact value does.  The exact results below are
# either far past that (|ref| >= 1.5 * 65520) or well inside (|ref| <= 6e4), never in between, where the fp32 accumulation
# order could fall on either side of the boundary.
F16_INF_AT = 65520.0


def _check_range(out, ref, what):
    ref = ref.to(F64)
    big = ref.abs() >= 1.5 * F16_INF_AT
    assert big.any() and (~big).any() and not (ref.abs()[~big] > 6e4).any(), f"{what}: operands outside the design"
    o = out.to(F64)
    assert torch.equal(o[big], ref[big].sign() * math.inf), f"{what}: overflowed results are not ±inf"
    _close_f16(out[~big], ref[~big], what)


@pytest.mark.parametrize("splits", [0, 4], ids=["one_cta", "split4"])
def test_gemm_overflow_to_inf(cuda_lib, splits):
    """The linear epilogue (single CTA, and the forced split-K finalise) storing results past the f16 range: bias columns of
    ±4e5 or ±2.5e4 on accumulations of up to ~1.3e3 (rows scaled by 2^8), times out_scale 1.5, plus an f16 residual."""
    g = _gen(20)
    m, k, n = 300, 640, 320
    a = torch.randn(m, k, device="cuda", generator=g).clamp(-4, 4)
    a[: m // 3] *= 256.0
    a = a.to(F16)
    w = _randn(n, k, g=g, scale=k ** -0.5)
    col = torch.arange(n, device="cuda")
    bias = torch.where(col % 5 == 0, 4e5, torch.where(col % 5 == 1, 2.5e4, 0.0)) * torch.where(col % 2 == 0, 1.0, -1.0)
    bias = bias + torch.randn(n, device="cuda", generator=g)
    res = _randn(m, n, g=g)
    o = Guarded(m, n, F16)
    kw = dict(force_splits=splits) if splits else dict(allow_split_k=False)
    ops.linear(a, w, bias=bias, residual=res, out=o.out, ldo=n, out_scale=1.5, **kw)
    o.check("overflow")
    ref = 1.5 * (a.to(F64) @ w.to(F64).T + bias.to(F64)) + res.to(F64)
    _check_range(o.out, ref, f"gemm splits={splits}")


def test_add_overflow_to_inf(cuda_lib):
    """add_f16: sums of two in-range f16 values past the range (±6e4 + ±6e4) are ±inf; the rest (|a|, |b| <= 2.5e4 and
    0 + -0, subnormal + subnormal) are the f16 rounding of the exact sum, i.e. torch's a + b, bit for bit."""
    g = _gen(21)
    n = 8 * 4001
    a = (torch.rand(n, device="cuda", generator=g) * 5e4 - 2.5e4).to(F16)
    b = (torch.rand(n, device="cuda", generator=g) * 5e4 - 2.5e4).to(F16)
    over = torch.arange(n, device="cuda") % 7 == 3
    sign = torch.where(torch.arange(n, device="cuda") % 2 == 0, 1.0, -1.0).to(F16)
    a[over], b[over] = (6e4 * sign[over]).to(F16), (6.2e4 * sign[over]).to(F16)
    a[:4] = torch.tensor([0.0, -0.0, 2.0 ** -24, -(2.0 ** -20)], dtype=F16, device="cuda")
    b[:4] = torch.tensor([-0.0, -0.0, 2.0 ** -24, 3 * 2.0 ** -24], dtype=F16, device="cuda")
    o = Guarded(n // 8, 8, F16)
    assert cuda_lib.mdb_add_f16(a.data_ptr(), b.data_ptr(), o.out.data_ptr(), n, torch.cuda.current_stream().cuda_stream) == 0
    o.check("add_f16")
    out = o.out.reshape(-1)
    _check_range(out, a.to(F64) + b.to(F64), "add_f16")
    assert torch.equal(out.view(torch.int16), (a + b).view(torch.int16))


def test_gemm_subnormal_results(cuda_lib):
    """Results around 1e-6, in the f16 subnormal range (below 2^-14), from normal operands (|a| in [2^-11, 2^-10),
    |w| in [2^-12, 2^-11)): each within 2^-24 (one subnormal step) + 2^-20 (|a| @ |w|) of float64, for the plain epilogue
    and the split-K finalise.  1e-4 * max|ref| would be no criterion at this scale."""
    g = _gen(22)
    m, k, n = 256, 256, 192

    def operand(rows, e):
        mag = 1 + torch.rand(rows, k, device="cuda", generator=g)
        sgn = torch.where(torch.rand(rows, k, device="cuda", generator=g) < 0.5, -1.0, 1.0)
        return (sgn * mag * 2.0 ** e).to(F16)

    a, w = operand(m, -11), operand(n, -12)
    ref = a.to(F64) @ w.to(F64).T
    bound = 2.0 ** -24 + 2.0 ** -20 * (a.to(F64).abs() @ w.to(F64).abs().T)
    assert ref.abs().max() < 2.0 ** -14 and ref.abs().median() > 2.0 ** -22
    for kw in (dict(allow_split_k=False), dict(force_splits=2)):
        o = Guarded(m, n, F16)
        ops.linear(a, w, out=o.out, ldo=n, **kw)
        o.check(f"subnormal results {kw}")
        err = (o.out.to(F64) - ref).abs()
        assert (err <= bound).all(), f"{kw}: max err / bound {(err / bound).max().item():.3f}"


def test_gemm_subnormal_operands(cuda_lib):
    """Subnormal f16 operands (k * 2^-24, 1 <= k < 1024) in rows of A and in rows of W against normal ones: H100's f16 wgmma
    takes them as they are (not flushed to zero), so every block of the product meets float64 within one f16 ulp of the
    result + 2^-20 (|a| @ |w|)."""
    g = _gen(23)
    m, k, n = 256, 320, 256

    def operand(rows):
        x = torch.randn(rows, k, device="cuda", generator=g)
        sub = torch.randint(1, 1024, (rows // 2, k), device="cuda", generator=g) * 2.0 ** -24
        x[rows // 2:] = sub * torch.where(torch.rand(rows // 2, k, device="cuda", generator=g) < 0.5, -1.0, 1.0)
        return x.to(F16)

    a, w = operand(m), operand(n)
    assert (a[m // 2:].abs() < 2.0 ** -14).all() and (a[m // 2:] != 0).all()
    ref = a.to(F64) @ w.to(F64).T
    ulp = torch.exp2(torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** -14))) - 10)
    bound = ulp + 2.0 ** -20 * (a.to(F64).abs() @ w.to(F64).abs().T)
    o = Guarded(m, n, F16)
    ops.linear(a, w, out=o.out, ldo=n, allow_split_k=False)
    o.check("subnormal operands")
    err = (o.out.to(F64) - ref).abs()
    bad = (err > bound).nonzero()
    assert bad.shape[0] == 0, f"{bad.shape[0]} elements off, first at {tuple(bad[0].tolist())}, " \
                              f"max err / bound {(err / bound).max().item():.3e}"


# ----------------------------------------------------------------------------------------------- mixed element types
# Each operator reads every operand in one element type, so a tensor of the other type would be read as garbage bits: the
# wrappers raise before anything is launched, and leave a given output untouched.
def _refused(fn, out=None):
    before = ops.launch_count()
    bits = None if out is None else out.view(torch.int16 if out.element_size() == 2 else torch.int32).clone()
    with pytest.raises(TypeError):
        fn()
    assert ops.launch_count() == before
    if out is not None:
        torch.cuda.synchronize()
        assert torch.equal(out.view(bits.dtype), bits), "a refused call wrote to its output"


def _t(rows, cols, dt):
    return torch.ones(rows, cols, dtype=dt, device="cuda")


@pytest.mark.parametrize("case", ["w", "a1", "residual", "out", "out_f32", "out_not_f32"])
@pytest.mark.parametrize("act", [BF16, F16], ids=["bf16", "f16"])
def test_gemm_conv_refuses_mixed_types(cuda_lib, act, case):
    other = F16 if act == BF16 else BF16
    m, k, n = 128, 64, 64
    t = {"a0": _t(m, k, act), "w": _t(n, 2 * k, act), "a1": _t(m, k, act), "residual": _t(m, n, act)}
    out_dt, out_f32 = act, False
    if case in t:
        t[case] = _t(*t[case].shape, other)
    elif case == "out":
        out_dt = other
    elif case == "out_f32":  # an fp32 output asked for, a 2-byte buffer given
        out_dt, out_f32 = act, True
    else:  # an fp32 buffer given for a 2-byte output
        out_dt = F32
    out = torch.full((m, n), float("nan"), dtype=out_dt, device="cuda")
    _refused(lambda: ops.gemm_conv(t["a0"], t["w"], n_img=1, h_in=1, w_in=m, c0=k, lda0=k, a1=t["a1"], c1=k, lda1=k,
                                   n_out=n, residual=t["residual"], ldr=n, out=out, ldo=n, out_f32=out_f32), out)


@pytest.mark.parametrize("case", ["k", "v", "out", "source1_k", "source1_v"])
@pytest.mark.parametrize("act", [BF16, F16], ids=["bf16", "f16"])
def test_attention_refuses_mixed_types(cuda_lib, act, case):
    other = F16 if act == BF16 else BF16
    b, heads, d, l = 2, 2, 64, 128
    c = heads * d
    q, k, v = _t(b * l, c, act), _t(b * l, c, act), _t(b * l, c, act)
    k1, v1 = _t(b * l, c, act), _t(b * l, c, act)
    out = torch.full((b * l, c), float("nan"), dtype=other if case == "out" else act, device="cuda")
    swap = {"k": "k", "v": "v", "source1_k": "k1", "source1_v": "v1"}.get(case)
    tensors = {"k": k, "v": v, "k1": k1, "v1": v1}
    if swap:
        tensors[swap] = _t(b * l, c, other)
    kw = dict(b=b, heads=heads, lq=l, lk=l, d=d, ldq=c, scale=d ** -0.5, out=out)
    if case.startswith("source1"):
        idx = torch.tensor([[1 << 24], [0]], dtype=torch.int32, device="cuda")
        _refused(lambda: ops.attention_multi(q, [(tensors["k"], tensors["v"], c, b), (tensors["k1"], tensors["v1"], c, b)],
                                             kv_index=idx, **kw), out)
    else:
        _refused(lambda: ops.attention(q, tensors["k"], tensors["v"], ldk=c, ldv=c, **kw), out)
        _refused(lambda: ops.attention(q, tensors["k"], tensors["v"], ldk=c, ldv=c,
                                       kv_len=torch.full((b,), l, dtype=torch.int32, device="cuda"), **kw), out)


@pytest.mark.parametrize("act", [BF16, F16], ids=["bf16", "f16"])
def test_groupnorm_refuses_mixed_types(cuda_lib, act):
    other = F16 if act == BF16 else BF16
    x0, x1 = _t(64, 32, act), _t(64, 32, other)
    gam, beta = torch.ones(64, device="cuda"), torch.zeros(64, device="cuda")
    _refused(lambda: ops.groupnorm(x0, 32, 32, 1, 64, gam, beta, 1e-5, False, x1=x1, c1=32, ld1=32))


@pytest.mark.parametrize("act", [BF16, F16], ids=["bf16", "f16"])
def test_add_refuses_mixed_types(cuda_lib, act):
    other = F16 if act == BF16 else BF16
    _refused(lambda: ops.add(_t(8, 8, act), _t(8, 8, other)))


@pytest.mark.parametrize("case", ["x_bf16", "x_f16", "w_f32"])
def test_linear_small_refuses_mixed_types(cuda_lib, case):
    x = _t(4, 64, {"x_bf16": BF16, "x_f16": F16}.get(case, F32))
    w = _t(8, 64, F32 if case == "w_f32" else F16)
    _refused(lambda: ops.linear_small(x, w))


def test_pack_latents_f16_refuses_bf16(cuda_lib):
    _refused(lambda: f16_ops.pack_latents_f16(_t(16, 4, BF16)))
