"""TEST INFRASTRUCTURE ONLY — a census of the kernel launches a forward really issues, each one checked in place.

`Census()` is a context manager that replaces every operator of magicdrive_b200.ops, f16_ops and vae_f16_ops (the engines
look them up as module attributes at call time, so every call is seen) by a wrapper that, per call:

1. redirects the output into a guard-banded buffer (tests/test_kernel_edges_gpu.Guarded) with the engine's row stride and
   column offset when the engine passed `out=`, and every float buffer the operator allocates (out=None outputs, row
   statistics, scratch) into one as well; an in-place residual (residual is out) is copied into the guarded output first,
   and the operands an operator updates in place (the scheduler updates, pin_views) are guarded copies;
2. launches the real operator, synchronises, and checks every guard bitwise untouched and no output element still holding
   the fill;
3. recomputes the result in float64 from the operands the launch read (the GEMM through tests/ops_emulator.gemm_conv in
   float64, whose argument assertions also hold every product descriptor to what the library accepts; attention through
   tests/attention_model.py) one image or row chunk at a time, and holds it to the criterion the kernel tests already state
   for that operator (CRITERIA), recording the worst err / tol;
4. hands the result back where the engine expects it (the same `out`, or a fresh tensor), so the forward goes on unchanged;
5. records the call's signature: the operator, its scalar arguments, each operand's dtype, shape and row stride, and for
   gemm_conv the planner's tiling (mdb_gemm_conv_plan).

Launch accounting: ops.launch_count() is read around every wrapped call; on exit the sum of those deltas must equal the
whole block's delta, so no launch escapes a wrapper.  EXEMPT names the operators left unchecked here, each with the test that
already checks the product's calls bit for bit.  An operator function that is in neither table is an error at entry.

Failures do not stop the forward: they are collected with the operator and signature, and `assert_clean()` raises them."""
import inspect
import math
import re
import types
from collections import defaultdict

import torch
import torch.nn.functional as F

from magicdrive_b200 import box_overlay, f16_ops, image_ops, jpeg_ops, ops, vae_f16_ops
from tests import ops_emulator
from tests.attention_model import TAU, attention_model, check_model
from tests.test_kernel_edges_gpu import _FILL, G, Guarded, _tol_bf16, _tol_f16, _tol_f32
from tests.test_layernorm_fold_gpu import _check_stats

BF16, F16, F32, F64 = torch.bfloat16, torch.float16, torch.float32, torch.float64
MODULES = (ops, f16_ops, vae_f16_ops, image_ops, jpeg_ops, box_overlay)
CHUNK = 1 << 25  # elements of one float64 reference chunk (rows x widest operand), 256 MB

# module functions that launch nothing of their own.  The wrappers guard what an operator allocates by standing a proxy in
# for the `torch` attribute of ops, f16_ops and vae_f16_ops while it runs: an operator must allocate its outputs through
# that module attribute (torch.empty / empty_like), which every operator there does; Census asserts it for every returned
# float tensor (guarded_outputs=True)
PLUMBING = {"start_profile", "stop_profile", "launch_count", "reset_launch_count", "workspace", "pdl_region", "linear",
            "check", "scratch_bytes", "view_transforms", "project_boxes"}
EXEMPT = {
    "resample_u8": "test_fid_protocol_gpu.py holds the product's resampling bit for bit to Pillow",
    "jpeg_roundtrip_u8": "test_fid_protocol_gpu.py holds the product's JPEG round trip bit for bit to libjpeg",
    "jpeg_encode_u8": "test_jpeg_encode_gpu.py holds the product's .jpg files byte for byte to the reference's",
    "encode_jpeg": "test_jpeg_encode_gpu.py holds the product's .jpg files byte for byte to the reference's",
    "_project": "test_box_overlay_gpu.py holds the product's box overlays byte for byte to the reference's",
    "show_box_on_views": "test_box_overlay_gpu.py holds the product's box overlays byte for byte to the reference's",
    "peer_barrier": "multi-GPU only (test_dist_cpu.py, tools/check_peer.py)",
}
# operators whose outputs are the updated operands: (argument names updated in place)
INPLACE = {"cfg_ddim_step": ("latents",), "cfg_unipc_step": ("latents", "last_sample", "m0", "m1"), "pin_views": ("dst",)}


def _family(name):
    return {"attention_multi": "attention", "attention_causal": "attention", "softmax_rows_f16": "softmax_rows",
            "conv_direct_f16": "conv_direct", "fid_input_f16": "fid_input", "pack_latents_f16": "pack_latents"}.get(name, name)


# ------------------------------------------------------------------------------------------------ signatures
_DT = {BF16: "bf16", F16: "f16", F32: "f32", F64: "f64", torch.int32: "i32", torch.int64: "i64", torch.uint8: "u8"}


def _desc(v):
    if torch.is_tensor(v):
        ld = v.stride(0) if v.dim() >= 2 else 1
        return f"{_DT.get(v.dtype, v.dtype)}{list(v.shape)}" + (f"/{ld}" if v.dim() >= 2 and ld != v.shape[-1] else "")
    if isinstance(v, ops.RowStats):
        return f"stats{list(v.data.shape)}"
    if isinstance(v, (list, tuple)):
        return "(" + ",".join(_desc(x) for x in v) + ")"
    return repr(v)


def signature(name, bound, defaults):
    """operator(argument=value, ...) over the arguments that differ from their defaults."""
    parts = [f"{k}={_desc(v)}" for k, v in bound.items() if v is not None and not (k in defaults and _same_default(v, defaults[k]))]
    return f"{name}(" + ", ".join(parts) + ")"


def _same_default(v, d):
    return not torch.is_tensor(v) and not isinstance(v, (list, tuple, ops.RowStats)) and d is not inspect.Parameter.empty \
        and type(v) is type(d) and v == d


# ------------------------------------------------------------------------------------------------ guarded allocation
class _GuardedTorch(types.ModuleType):
    """Stands in for `torch` inside an operator wrapper: empty / empty_like of a float type return the interior of a
    Guarded buffer (rows = the leading dimensions, except that a 3-D [rows, parts, 2] statistics tensor keeps its rows);
    everything else is torch."""

    def __init__(self):
        super().__init__("torch")
        self.allocated = []

    def __getattr__(self, k):
        return getattr(torch, k)

    def empty(self, *shape, dtype=None, device=None, **kw):
        shape = tuple(shape[0]) if len(shape) == 1 and isinstance(shape[0], (tuple, list, torch.Size)) else shape
        dtype = dtype or torch.get_default_dtype()
        if dtype not in _FILL or kw:
            return torch.empty(shape, dtype=dtype, device=device, **kw)
        n = math.prod(shape)
        cols = 1 if len(shape) < 2 else math.prod(shape[1:]) if len(shape) == 3 else shape[-1]
        g = Guarded(n // max(cols, 1), cols, dtype, device=device)
        self.allocated.append(g)
        return g.out.view(shape)

    def empty_like(self, t, **kw):
        return self.empty(tuple(t.shape), dtype=kw.get("dtype", t.dtype), device=t.device)


def _guard_like(t, fill_from=None):
    """A Guarded [rows, cols] with t's row stride and column offset (16-byte alignment as t's) for a 2-D view t."""
    rows, cols = t.shape[0], t.shape[1] if t.dim() > 1 else 1
    ld = t.stride(0) if t.dim() > 1 else cols
    col0 = t.storage_offset() % ld if ld > cols else 0
    g = Guarded(rows, cols, t.dtype, ld=ld, col0=col0, device=t.device)
    if fill_from is not None:
        g.out.copy_(fill_from.reshape(rows, cols))
    return g


def _window(name, a):
    """(rows, cols, row stride) of what operator `name` writes at its `out` argument."""
    o = a["out"]
    if name == "gemm_conv":
        th = a["taps"] if a["taps_h"] is None else a["taps_h"]
        tw = a["taps"] if a["taps_w"] is None else a["taps_w"]
        ph = a["pad"] if a["pad_h"] is None else a["pad_h"]
        pw = a["pad"] if a["pad_w"] is None else a["pad_w"]
        ho = a["h_out"] if a["h_out"] is not None else (a["h_in"] + 2 * ph + a["pad_h_end"] - th) // a["stride"] + 1
        wo = a["w_out"] if a["w_out"] is not None else (a["w_in"] + 2 * pw + a["pad_w_end"] - tw) // a["stride"] + 1
        ld = a["ldo"] if a["ldo"] is not None else o.stride(0) if o.dim() == 2 else o.shape[-1]
        return a["n_img"] * ho * wo, a["n_out"] // 2 if a["geglu"] else a["n_out"], ld
    if name in ("attention", "attention_multi"):
        return a["b"] * a["lq"], a["heads"] * a["d"], o.stride(0)
    if name == "attention_causal":
        return a["b"] * a["l"], a["heads"] * a["d"], o.stride(0)
    if name == "clip_embed":
        return a["ids"].numel(), a["tok"].shape[1], o.stride(0)
    if name == "pool2d":
        n, h, w, k, s, p = a["n"], a["h"], a["w"], a["k"], a["stride"], a["pad"]
        rows = n if a["mode"] == ops.POOL_GLOBAL_AVG else n * ((h + 2 * p - k) // s + 1) * ((w + 2 * p - k) // s + 1)
        return rows, a["c"], a["ldo"] if a["ldo"] is not None else o.stride(0)
    raise AssertionError(f"{name}: no output window for out=")


def _guards_intact(g, what):
    """The guard elements of a Guarded scratch buffer bitwise untouched (its interior may stay partly unwritten)."""
    if g.buf.is_cuda:
        torch.cuda.synchronize()
    bits = g.buf.view(g.itype)
    outside = torch.ones_like(bits, dtype=torch.bool)
    outside[G:G + g.rows, g.col0:g.col0 + g.cols] = False
    hit = int(((bits != g.fill) & outside).sum())
    assert hit == 0, f"{what}: {hit} guard elements overwritten"


def _2d(t, rows, cols, ld):
    """The [rows, cols] row-stride-ld window a kernel writes at t's address."""
    return t.as_strided((rows, cols), (ld, 1), t.storage_offset())


# ------------------------------------------------------------------------------------------------ comparisons
class Mismatch(AssertionError):
    pass


def _ratio(err, tol):
    r = torch.where(tol > 0, err / tol.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    return torch.nan_to_num(r, nan=math.inf)


def _close_pieces(pieces, what):
    """pieces: [(out, float64 ref)] of one output, held to _close_bf16 / _close_f16 / _close_f32 by the output's type with
    max |ref| taken over the whole output.  Returns the worst err / tol."""
    ref_max = max((r.abs().max().item() for _, r in pieces if r.numel()), default=0.0)
    worst = 0.0
    for o, r in pieces:
        tol = {BF16: _tol_bf16, F16: _tol_f16, F32: _tol_f32}[o.dtype](r, ref_max)
        worst = max(worst, _ratio((o.to(F64) - r).abs(), tol * torch.ones_like(r)).max().item() if r.numel() else 0.0)
    if not worst <= 1.0:
        raise Mismatch(f"{what}: err / tol reaches {worst:.3g} (max |ref| {ref_max:.3e})")
    return worst


def _bound(out, ref, bound, what):
    """|out - ref| <= bound elementwise (a stated bound of test_small_ops_gpu.py / test_fid_gpu.py); worst ratio."""
    r = _ratio((out.to(F64) - ref).abs(), bound).max().item() if ref.numel() else 0.0
    if not r <= 1.0:
        raise Mismatch(f"{what}: err / bound reaches {r:.3g}")
    return r


def _bitwise(out, ref, what):
    """Bitwise equal, NaN compared as NaN (test_small_ops_gpu._same)."""
    if out.is_floating_point():
        it = {2: torch.int16, 4: torch.int32, 8: torch.int64}[out.element_size()]
        ok = (out.view(it) == ref.view(it)) | (out.isnan() & ref.isnan())
    else:
        ok = out == ref
    bad = (~ok).sum().item()
    if bad:
        raise Mismatch(f"{what}: {bad} elements differ from torch")
    return 0.0


def _bitwise_chunks(n, per, pair, what):
    """_bitwise over n items of `per` elements, a chunk at a time: pair(i0, i1) -> (out, ref) of items [i0, i1)."""
    for i0, i1 in _chunks(n, per):
        _bitwise(*pair(i0, i1), what)
    return 0.0


def _chunks(n, per, budget=CHUNK):
    """[start, stop) ranges over n items of `per` elements each, at least one item per range."""
    step = max(1, budget // max(per, 1))
    return [(i, min(i + step, n)) for i in range(0, n, step)]


# ------------------------------------------------------------------------------------------------ criteria
def _gemm_conv(a, res, plan):
    out, stats = (res if a["emit_stats"] else (res, None))
    th = a["taps"] if a["taps_h"] is None else a["taps_h"]
    tw = a["taps"] if a["taps_w"] is None else a["taps_w"]
    ph = a["pad"] if a["pad_h"] is None else a["pad_h"]
    pw = a["pad"] if a["pad_w"] is None else a["pad_w"]
    n, h, w, s = a["n_img"], a["h_in"], a["w_in"], a["stride"]
    ho = a["h_out"] if a["h_out"] is not None else (h + 2 * ph + a["pad_h_end"] - th) // s + 1
    wo = a["w_out"] if a["w_out"] is not None else (w + 2 * pw + a["pad_w_end"] - tw) // s + 1
    width = a["n_out"] // 2 if a["geglu"] else a["n_out"]
    ldo = width if a["out"] is None else a["ldo"] if a["ldo"] is not None else out.stride(0)
    stored = _2d(out, n * ho * wo, width, ldo)
    token = n == 1 and h == 1 and th == tw == s == 1 and ph == pw == 0 and not a["pad_h_end"] and not a["pad_w_end"]
    units, per_in, per_out = (w, 1, 1) if token else (n, h * w, ho * wo)  # chunk over rows of a token GEMM, else images
    wide = max(a["c0"] + a["c1"], a["n_out"]) * th * tw
    pieces = []
    kw = {k: v for k, v in a.items() if k not in ("out", "ldo", "emit_stats", "h_out", "w_out")}
    for u0, u1 in _chunks(units, per_in * wide):
        ck = dict(kw)
        rin, rout = slice(u0 * per_in, u1 * per_in), slice(u0 * per_out, u1 * per_out)
        ck["a0"] = a["a0"][rin]
        if a["a1"] is not None:
            ck["a1"] = a["a1"][rin]
        if a["residual"] is not None:
            ck["residual"] = a["residual"].reshape(-1, a["residual"].shape[-1])[rout]
        if a["ln"] is not None:
            ck["ln"] = ops.RowStats(a["ln"].data[rout], a["ln"].parts)
        if token:
            ck["w_in"] = u1 - u0
        else:
            ck["n_img"] = u1 - u0
            if a["rowbias"] is not None and a["rowbias"].shape[0] > 1:
                ck["rowbias"] = a["rowbias"][u0:u1]
        with ops_emulator.compute(F64):
            ref = ops_emulator.gemm_conv(**ck, h_out=ho, w_out=u1 - u0 if token else wo)
        pieces.append((stored[rout], ref))
    worst = _close_pieces(pieces, "output")
    if stats is not None:
        sg = _STATS_GUARD.get(stats.data.data_ptr())
        if sg is None:  # statistics the operator did not allocate through torch.empty (a CPU restatement)
            sg = Guarded(stats.data.shape[0], 2 * stats.parts, F32, device=stats.data.device)
            sg.out.copy_(stats.data.reshape(sg.rows, -1))
        bn = plan[0] if plan is not None else -(-width // stats.parts)
        _check_stats(sg, stored, bn, "gemm_conv")
    return worst


_STATS_GUARD = {}  # data_ptr of a statistics tensor allocated in a wrapper -> its Guarded (for _check_stats)


def _attention_sets(a, multi):
    """kv_of(i) for attention_model from the arguments of attention / attention_multi."""
    b, lk = a["b"], a["lk"]
    n_sets = a["n_sets"]
    if multi:
        srcs = a["sources"]
    else:
        srcs = [(a["k"], a["v"], a["ldk"], b if a["b_kv"] is None else a["b_kv"], a["ldv"])]
    idx = a["kv_index"]
    idx = [[i] for i in range(b)] if idx is None else idx.reshape(b, n_sets).tolist()
    if not multi:
        idx = [[-1 if e < 0 else e for e in row] for row in idx]  # plain batch indices: source 0
    kl = [lk] * b if a["kv_len"] is None else [min(max(int(x), 0), lk) for x in a["kv_len"].tolist()]

    def kv_of(i):
        sets = []
        for e in idx[i]:
            if e < 0 or kl[i] == 0:
                continue
            src, j = e >> 24, e & 0xFFFFFF
            k, v = srcs[src][0], srcs[src][1]
            sets.append((k[j * lk: j * lk + kl[i]], v[j * lk: j * lk + kl[i]]))
        return sets
    return kv_of


def _attention(a, out, multi):
    m = attention_model(a["q"], _attention_sets(a, multi), a["b"], a["heads"], a["lq"], a["d"], a["scale"], out.dtype)
    elem, row = check_model(out, m, "attention")
    return max(elem, row / TAU)


def _attention_causal(a, out, _plan):
    b, l = a["b"], a["l"]
    m = attention_model(a["q"], lambda i: [(a["k"][i * l:(i + 1) * l], a["v"][i * l:(i + 1) * l])], b, a["heads"], l, a["d"],
                        a["scale"], out.dtype, causal=True)
    elem, row = check_model(out, m, "attention_causal")
    return max(elem, row / TAU)


def _groupnorm(a, out, _plan):
    n, hw, c0, c1, g = a["n_img"], a["hw"], a["c0"], a["c1"], a["groups"]
    pieces = []
    for i0, i1 in _chunks(n, hw * (c0 + c1)):
        rows = slice(i0 * hw, i1 * hw)
        x = a["x0"][rows, :c0].to(F64)
        if c1:
            x = torch.cat([x, a["x1"][rows, :c1].to(F64)], 1)
        y = F.group_norm(x.reshape(i1 - i0, hw, c0 + c1).permute(0, 2, 1), g, a["gamma"].to(F64), a["beta"].to(F64), a["eps"])
        y = F.silu(y) if a["silu"] else y
        pieces.append((out[rows], y.permute(0, 2, 1).reshape(-1, c0 + c1)))
    return _close_pieces(pieces, "groupnorm")


def _conv_direct(a, out, _plan):
    n, h, w, cin, cout, k = a["n"], a["h"], a["w"], a["cin"], a["cout"], a["k"]
    o2 = out.reshape(n, -1, cout)
    pieces = []
    for i0, i1 in _chunks(n, h * w * max(cin, cout)):
        x = a["x"].reshape(n, h, w, cin)[i0:i1].to(F64).permute(0, 3, 1, 2)
        y = F.conv2d(x, a["wgt"].to(F64).permute(3, 2, 0, 1), a["bias"].to(F64), stride=a["stride"], padding=a["pad"])
        y = F.silu(y) if a["silu"] else y
        y = y.permute(0, 2, 3, 1).reshape(i1 - i0, -1, cout)
        if a["residual"] is not None:
            y = y + a["residual"].reshape(n, -1, cout)[i0:i1].to(F64)
        pieces.append((o2[i0:i1], y))
    return _close_pieces(pieces, "conv_direct")


def _layernorm(a, out, _plan):
    x = a["x"]
    pieces = [(out[r0:r1], F.layer_norm(x[r0:r1].to(F64), (x.shape[1],), a["gamma"].to(F64), a["beta"].to(F64), a["eps"]))
              for r0, r1 in _chunks(x.shape[0], x.shape[1])]
    return _close_pieces(pieces, "layernorm")


def _softmax_rows(a, out, _plan):
    """bf16: _close_bf16 (test_softmax_rows); f16: within one f16 ulp (test_vae_fp16_gpu.test_softmax_rows_f16), i.e.
    _tol_f16 without its max |ref| term.  The padding columns are +0."""
    s, cols = a["s"], a["cols"]
    pieces = [(out[r0:r1, :cols], torch.softmax(s[r0:r1, :cols].to(F64), -1)) for r0, r1 in _chunks(s.shape[0], cols)]
    if out.dtype == F16:
        worst = 0.0
        for o, r in pieces:
            worst = max(worst, _ratio((o.to(F64) - r).abs(), _tol_f16(r, 0.0)).max().item())
        if not worst <= 1.0:
            raise Mismatch(f"softmax_rows_f16: err / ulp reaches {worst:.3g}")
    else:
        worst = _close_pieces(pieces, "softmax_rows")
    if (out[:, cols:].view(torch.int16) != 0).any():
        raise Mismatch("softmax_rows: padding columns are not +0")
    return worst


def _add(a, out, _plan):
    x, y, o = a["a"].reshape(-1), a["b"].reshape(-1), out.reshape(-1)
    return _bitwise_chunks(o.numel(), 1, lambda i0, i1: (o[i0:i1], (x[i0:i1].float() + y[i0:i1].float()).to(o.dtype)),
                           "add")


def _upsample(a, out, _plan):
    n, h, w, c, ho, wo = a["n"], a["h"], a["w"], a["c"], a["ho"], a["wo"]
    x = a["x"].reshape(n, h, w, c)

    def pair(i0, i1):
        ref = F.interpolate(x[i0:i1].permute(0, 3, 1, 2).float(), size=(ho, wo), mode="nearest")
        return out[i0 * ho * wo:i1 * ho * wo], ref.permute(0, 2, 3, 1).reshape(-1, c).to(out.dtype)
    return _bitwise_chunks(n, ho * wo * c, pair, "upsample_nearest")


def _adaptive_avgpool(a, out, _plan):
    n, h, w, c = a["n"], a["h"], a["w"], a["c"]
    x = a["x"].reshape(n, h, w, c)
    o = out.reshape(n, -1, c)
    pieces = []
    for i0, i1 in _chunks(n, h * w * c):
        y = F.adaptive_avg_pool2d(x[i0:i1].to(F64).permute(0, 3, 1, 2), (a["ho"], a["wo"]))
        y = F.silu(y) if a["silu"] else y
        pieces.append((o[i0:i1], y.permute(0, 2, 3, 1).reshape(i1 - i0, -1, c)))
    return _close_pieces(pieces, "adaptive_avgpool")


def _pool2d(a, out, _plan):
    """test_fid_gpu.test_pools: max exact, average and global average _close."""
    n, h, w, c, mode = a["n"], a["h"], a["w"], a["c"], a["mode"]
    xi = a["x"][:, :c].to(F64).reshape(n, h, w, c).permute(0, 3, 1, 2)
    if mode == ops.POOL_GLOBAL_AVG:
        return _close_pieces([(out[:, :c], xi.mean((2, 3)))], "pool2d global")
    k, s, p = a["k"], a["stride"], a["pad"]
    ref = F.max_pool2d(xi, k, s, p) if mode == ops.POOL_MAX else F.avg_pool2d(xi, k, s, p, count_include_pad=False)
    ref = ref.permute(0, 2, 3, 1).reshape(-1, c)
    if mode == ops.POOL_MAX:
        return _bitwise(out[:, :c].to(F64), ref, "max pool")
    return _close_pieces([(out[:, :c], ref)], "avg pool")


def _fid_input(a, out, _plan):
    """test_fid_gpu.test_input_kernel: without resampling within half a step of the output type plus 1e-7 of the float64
    value, with it within 2^-8 max |ref| + 1e-6; channels 3..7 zero.  One image chunk at a time."""
    src = a["x"].permute(0, 3, 1, 2) if a["nhwc"] else a["x"]
    n, _, h, w = src.shape
    size = a["size"]
    resize = size is not None and tuple(size) != (h, w)
    ho, wo = tuple(size) if size is not None else (h, w)
    o = out.reshape(n, ho, wo, 8)
    if o[..., 3:].any():
        raise Mismatch("fid_input: channels 3..7 are not zero")
    worst, err_max, ref_max = 0.0, 0.0, 0.0
    for i0, i1 in _chunks(n, 3 * max(h * w, ho * wo)):
        s = src[i0:i1]
        # 255 x in fp32, then rint and an exact division, as test_input_kernel
        x = torch.round(s.float() * 255).clamp(0, 255).to(F64) / 255 if a["quantize"] else s.to(F64)
        if resize:
            x = F.interpolate(x, size=(ho, wo), mode="bilinear", align_corners=False)
        if a["normalize"]:
            x = 2 * x - 1
        oc = o[i0:i1, ..., :3].permute(0, 3, 1, 2).to(F64)
        if resize:  # the bound needs max |ref| over the whole output: collect, compare after the loop
            err_max = max(err_max, torch.nan_to_num((oc - x).abs(), nan=math.inf).max().item())
            ref_max = max(ref_max, x.abs().max().item())
        else:
            bits = 8 if out.dtype == BF16 else 11
            bound = torch.exp2(torch.floor(torch.log2(x.abs().clamp_min(2.0 ** -100))) - bits) + 1e-7
            worst = max(worst, _bound(oc, x, bound, "fid_input"))
    if resize:
        worst = err_max / (2.0 ** -8 * ref_max + 1e-6)
        if not worst <= 1.0:
            raise Mismatch(f"fid_input: err / bound reaches {worst:.3g}")
    return worst


def _linear_small(a, out, _plan):
    from tests.test_small_ops_gpu import _linear_small_ref
    k = a["x"].shape[1]
    y, bound = _linear_small_ref(a["x"], a["w"][:, :k], a["bias"], a["pre_silu"], a["post_silu"])
    return _bound(out, y, bound, "linear_small")


def _timestep_embedding(a, out, _plan):
    """test_small_ops_gpu.test_timestep_embedding: 2^-20 max(1, |arg|)."""
    t, dim, shift = a["t"], a["dim"], a["freq_shift"]
    half = dim // 2
    j = torch.arange(half, dtype=F64, device=t.device)
    arg = t.to(F64).reshape(-1)[:, None] * torch.exp(-math.log(10000.0) * j / (half - shift))[None]
    ref = torch.cat([torch.cos(arg), torch.sin(arg)] if a["flip_sin_to_cos"] else [torch.sin(arg), torch.cos(arg)], -1)
    bound = 2.0 ** -20 * arg.abs().clamp_min(1.0).repeat(1, 2)
    if dim % 2:
        ref, bound = F.pad(ref, (0, 1)), F.pad(bound, (0, 1), value=2.0 ** -20)
    return _bound(out, ref, bound, "timestep_embedding")


def _fourier_embed(a, out, _plan):
    """test_small_ops_gpu.test_fourier_embed: the identity part bitwise, sin / cos within 2^-21 max(1, |arg|)."""
    x = a["x"]
    d = x.shape[1]
    _bitwise(out[:, :d], x, "fourier identity part")
    parts, bounds = [], []
    for k in range(a["num_freqs"]):
        arg = x.to(F64) * 2.0 ** k
        parts += [torch.sin(arg), torch.cos(arg)]
        bounds += [2.0 ** -21 * arg.abs().clamp_min(1.0)] * 2
    return _bound(out[:, d:], torch.cat(parts, -1), torch.cat(bounds, -1), "fourier_embed")


def _clip_embed(a, res, _plan):
    """test_clip_text_gpu.test_clip_embed: bf16(tok[id] + pos) bit for bit, statistics within 3e-5."""
    out, stats = res
    ids, tok, pos = a["ids"], a["tok"], a["pos"]
    ln = ids.shape[1]
    ref = (tok[ids.long()] + pos[None, :ln]).reshape(-1, tok.shape[1])
    _bitwise(out, ref, "clip_embed")
    o64 = out.to(F64)
    st = stats.data[:, 0].to(F64)
    r = max(_ratio((st[:, 0] - o64.sum(1)).abs(), 3e-5 * o64.abs().sum(1)).max().item(),
            _ratio((st[:, 1] - (o64 * o64).sum(1)).abs(), 3e-5 * (o64 * o64).sum(1)).max().item())
    if not r <= 1.0:
        raise Mismatch(f"clip_embed statistics: err / bound reaches {r:.3g}")
    return r


def _nchw_to_nhwc(a, out, _plan):
    x = a["x"] if a["x"].dtype in (F32, BF16) else a["x"].float()
    n, c, h, w = x.shape
    return _bitwise_chunks(n, c * h * w, lambda i0, i1: (out[i0 * h * w:i1 * h * w],
                                                         x[i0:i1].permute(0, 2, 3, 1).reshape(-1, c).to(BF16)),
                           "nchw_to_nhwc")


def _nhwc_to_nchw(a, out, _plan):
    n, c, h, w = a["n"], a["c"], a["h"], a["w"]
    x = a["x"].reshape(n, h, w, -1)
    return _bitwise_chunks(n, c * h * w, lambda i0, i1: (out[i0:i1], x[i0:i1, ..., :c].permute(0, 3, 1, 2).to(a["dtype"])),
                           "nhwc_to_nchw")


def _convert(dtype):
    def check(a, out, _plan):
        x, o = a["x"].reshape(-1), out.reshape(-1)
        return _bitwise_chunks(o.numel(), 1, lambda i0, i1: (o[i0:i1], x[i0:i1].to(dtype)), "conversion")
    return check


def _pack(dtype):
    def check(a, out, _plan):
        x, cpad = a["x"], a["cpad"]
        pix = x.shape[0]
        o = out.reshape(a["repeat"], pix, cpad)  # repeat r holds rows [r pix, (r + 1) pix)
        return _bitwise_chunks(pix, cpad, lambda i0, i1: (o[:, i0:i1], F.pad(x[i0:i1].to(dtype), (0, cpad - x.shape[1]))
                                                          .expand(a["repeat"], -1, -1)), "pack_latents")
    return check


def _cfg_ddim_step(a, out, _plan):
    """test_small_ops_gpu.test_cfg_ddim_step: 2^-21 sum |terms|."""
    from tests.test_small_ops_gpu import _combine
    lat = a["latents"]
    npix, c = lat.shape[0], a["c"]
    e64 = a["eps"][:, :c].to(F64)
    e, ea = _combine(e64[:npix], e64[npix:], a["cfg"], a["guidance"])
    c0, c1 = a["coef"].to(F64).tolist()[:2]
    x0 = lat.to(F64)
    return _bound(out, c0 * x0 + c1 * e, 2.0 ** -21 * (abs(c0) * x0.abs() + abs(c1) * ea), "cfg_ddim_step")


def _cfg_unipc_step(a, out, _plan):
    from tests.test_small_ops_gpu import _unipc_ref
    npix, c = a["latents"].shape[0], a["c"]
    e64 = a["eps"][:, :c].to(F64)
    ref = _unipc_ref(a["coef"].to(F64).tolist(), *(a[k].to(F64) for k in ("latents", "last_sample", "m0", "m1")),
                     e64[:npix], e64[npix:], a["cfg"], a["guidance"])
    r = max(_bound(_INPLACE_OUT[k], *ref[k2], f"cfg_unipc_step {k}") for k, k2 in
            (("latents", "latents"), ("last_sample", "last"), ("m0", "m0")))
    _bitwise(_INPLACE_OUT["m1"], a["m0"], "cfg_unipc_step m1")
    return r


def _pin_views(a, out, _plan):
    """test_small_ops_gpu.test_pin_views: pinned rows within 2^-21 sum |terms|, the other rows untouched."""
    dst, c = a["dst"], a["c"]
    sel = a["view_mask"].bool().repeat_interleave(a["rows_per_view"])
    k0, k1 = a["coef"].to(F64).tolist()[:2]
    b = a["b"][:, :c].to(F64)
    ref = k1 * b + (k0 * a["a"][:, :c].to(F64) if a["a"] is not None else 0)
    bound = 2.0 ** -21 * (abs(k1) * b.abs() + (abs(k0) * a["a"][:, :c].to(F64).abs() if a["a"] is not None else 0))
    _bitwise(out[~sel], dst[~sel], "rows of unpinned views")
    return _bound(out[sel, :c], ref[sel], bound[sel], "pin_views") if bool(sel.any()) else 0.0


_INPLACE_OUT = {}  # argument name -> the guarded result of the in-place operator being checked

CRITERIA = {
    "gemm_conv": _gemm_conv,
    "attention": lambda a, out, _p: _attention(a, out, False),
    "attention_multi": lambda a, out, _p: _attention(a, out, True),
    "attention_causal": _attention_causal,
    "groupnorm": _groupnorm,
    "conv_direct": _conv_direct,
    "conv_direct_f16": _conv_direct,
    "layernorm": _layernorm,
    "softmax_rows": _softmax_rows,
    "softmax_rows_f16": _softmax_rows,
    "add": _add,
    "upsample_nearest": _upsample,
    "adaptive_avgpool": _adaptive_avgpool,
    "pool2d": _pool2d,
    "fid_input": _fid_input,
    "fid_input_f16": _fid_input,
    "linear_small": _linear_small,
    "timestep_embedding": _timestep_embedding,
    "fourier_embed": _fourier_embed,
    "clip_embed": _clip_embed,
    "nchw_to_nhwc": _nchw_to_nhwc,
    "nhwc_to_nchw": _nhwc_to_nchw,
    "f32_to_bf16": _convert(BF16),
    "f32_to_f16": _convert(F16),
    "f16_to_f32": _convert(F32),
    "pack_latents": _pack(BF16),
    "pack_latents_f16": _pack(F16),
    "cfg_ddim_step": _cfg_ddim_step,
    "cfg_unipc_step": _cfg_unipc_step,
    "pin_views": _pin_views,
}


def _operators(mod):
    """The functions of `mod` that launch kernels: its own public functions minus PLUMBING, and whatever stands in for an
    operator of CRITERIA / EXEMPT (a CPU restatement in the host tests)."""
    names = []
    for k, v in vars(mod).items():
        if not inspect.isfunction(v) or k in PLUMBING:
            continue
        if k in CRITERIA or k in EXEMPT or (v.__module__ == mod.__name__ and not k.startswith("_")):
            names.append(k)
    return names


# ------------------------------------------------------------------------------------------------ the census
class Census:
    """with Census() as c: <forward>;  c.assert_clean().  c.rows: signature -> [count, worst ratio, plan];
    c.failures: (signature, message).  guarded_outputs: every float tensor an operator returns must be a guarded buffer
    (one it allocated through the `torch` proxy, the guarded `out=` or an in-place operand); off only for restatements that
    allocate through their own module's torch (the host tests)."""

    def __init__(self, guarded_outputs=True):
        self.guarded_outputs = guarded_outputs
        self.rows = {}
        self.failures = []
        self.counted = 0
        self.exempt = 0
        self._depth = 0
        self._saved = []

    # -- install / remove
    def __enter__(self):
        for mod in MODULES:
            for name in _operators(mod):
                if name not in CRITERIA and name not in EXEMPT:
                    raise AssertionError(f"{mod.__name__}.{name}: an operator without a census criterion or exemption")
                fn = getattr(mod, name)
                self._saved.append((mod, name, fn))
                setattr(mod, name, self._wrap(name, fn, name in EXEMPT))
        self._start = ops.launch_count()
        return self

    def __exit__(self, *exc):
        for mod, name, fn in reversed(self._saved):
            setattr(mod, name, fn)
        self._saved = []
        self.total = ops.launch_count() - self._start
        if exc[0] is None:
            self.unaccounted = self.total - self.counted - self.exempt
            assert self.unaccounted == 0, (f"{self.unaccounted} kernel launches outside the census wrappers "
                                           f"({self.total} in all, {self.counted} checked, {self.exempt} exempt)")
        return False

    # -- one call
    def _wrap(self, name, fn, exempt):
        sig_params = inspect.signature(fn).parameters
        defaults = {k: p.default for k, p in sig_params.items()}

        def wrapped(*args, **kw):
            if self._depth:  # an operator called by another one (attention -> attention_multi): the outer call checks it
                return fn(*args, **kw)
            n0 = ops.launch_count()
            if exempt:
                try:
                    self._depth += 1
                    return fn(*args, **kw)
                finally:
                    self._depth -= 1
                    self.exempt += ops.launch_count() - n0
            bound = inspect.signature(fn).bind(*args, **kw)
            bound.apply_defaults()
            a = dict(bound.arguments)
            sig = signature(name, a, defaults)
            try:
                self._depth += 1
                res, plan, guards, outs, unguarded = self._launch(name, fn, a)
            finally:
                self._depth -= 1
                self.counted += ops.launch_count() - n0
            ratio, msg = None, None
            try:
                if unguarded and self.guarded_outputs:
                    raise Mismatch(f"{unguarded} returned float tensors are not guarded buffers (allocated past the "
                                   f"module's `torch`)")
                for g in guards:
                    _guards_intact(g, sig)
                for o in outs:
                    if o is not None:
                        o.check(sig)
                ratio = CRITERIA[name](a, res if name in ("gemm_conv", "clip_embed") else _first(res), plan)
            except AssertionError as e:
                msg = str(e)
            if plan is not None:
                sig += f" | BN={plan[0]} tiles={plan[1]}x{plan[2]}x{plan[3]} waves={plan[4]}"
            row = self.rows.setdefault(sig, [0, 0.0, name])
            row[0] += 1
            if msg is not None:
                self.failures.append((sig, msg))
                row[1] = math.inf
            else:
                row[1] = max(row[1], ratio)
            return self._hand_back(name, a, res)
        return wrapped

    def _launch(self, name, fn, a):
        """Run fn on guarded outputs; returns (result as written, plan, guards to check, guarded outputs to check)."""
        proxy = _GuardedTorch()
        mods = [m for m in (ops, f16_ops, vae_f16_ops) if hasattr(m, "torch")]
        real = {m: m.torch for m in mods}
        call = dict(a)
        given = None
        if a.get("out") is not None:
            o = a["out"]
            rows, cols, ld = _window(name, a)
            col0 = o.storage_offset() % ld if ld > cols else 0
            given = Guarded(rows, cols, o.dtype, ld=ld, col0=col0 if col0 + cols <= ld else 0, device=o.device)
            call["out"] = given.out
            if name == "gemm_conv" and a["residual"] is not None and a["residual"].data_ptr() == o.data_ptr():
                given.out.copy_(_2d(o, rows, cols, ld))  # residual is out: the kernel reads and writes the guarded copy
                call["residual"] = given.out
                call["ldr"] = given.ld
        inplace = {}
        for k in INPLACE.get(name, ()):
            if a[k] is not None:
                inplace[k] = _guard_like(a[k], fill_from=a[k])
                call[k] = inplace[k].out
        plan = None
        for m in mods:
            m.torch = proxy
        if name == "gemm_conv" and a["a0"].is_cuda:
            ops._profile = []  # the wrapper asks the planner for its tiling only while profiling
        b = inspect.signature(fn).bind(**call)
        try:
            res = fn(*b.args, **b.kwargs)
        finally:
            for m in mods:
                m.torch = real[m]
            if name == "gemm_conv" and ops._profile is not None:
                prof, ops._profile = ops._profile, None
                if prof:
                    plan = [int(x) for x in re.findall(r"BN=(\d+) tiles=(\d+)x(\d+)x(\d+) waves=(\d+)", prof[-1][4])[0]]
        if any(t.is_cuda for t in _tensors(res)):
            torch.cuda.synchronize()
        # what the caller's pointers now hold: results in the guarded buffers
        outs = []
        guards = list(proxy.allocated)
        _STATS_GUARD.clear()
        for g in proxy.allocated:
            if res is not None and name == "gemm_conv" and a["emit_stats"] and g.out.data_ptr() == res[1].data.data_ptr():
                _STATS_GUARD[g.out.data_ptr()] = g
                guards.remove(g)  # _check_stats checks it
        returned = {t.data_ptr() for t in _tensors(res)}
        for g in proxy.allocated:
            if g.out.data_ptr() in returned and g in guards and name not in INPLACE:
                guards.remove(g)
                outs.append(g)
        if given is not None:
            outs.append(given)
        _INPLACE_OUT.clear()
        for k, g in inplace.items():
            guards.append(g)
            _INPLACE_OUT[k] = g.out
        if name in INPLACE:
            res = inplace[INPLACE[name][0]].out
        guarded = {g.out.data_ptr() for g in proxy.allocated + list(inplace.values()) + ([given] if given else [])}
        unguarded = sum(1 for t in _tensors(res) if t.is_floating_point() and t.data_ptr() not in guarded)
        return res, plan, guards, outs, unguarded

    def _hand_back(self, name, a, res):
        """Copy guarded results to where the engine expects them and return what the operator would have returned."""
        if name in INPLACE:
            for k, t in _INPLACE_OUT.items():
                a[k].copy_(t)
            _INPLACE_OUT.clear()
            return a[INPLACE[name][0]]
        o = a.get("out")

        def back(t):
            if isinstance(t, ops.RowStats):
                return ops.RowStats(t.data.clone(), t.parts)
            return t.clone() if torch.is_tensor(t) else t
        if o is not None:
            first = _first(res)
            _2d(o, first.shape[0], first.shape[1], first.stride(0)).copy_(first)
            if isinstance(res, tuple):
                return (o,) + tuple(back(t) for t in res[1:])
            return o
        if isinstance(res, tuple):
            return tuple(back(t) for t in res)
        return back(res)

    # -- results
    def assert_clean(self):
        if self.failures:
            lines = [f"{len(self.failures)} launches failed their criterion:"]
            lines += [f"  {sig}\n    {msg}" for sig, msg in self.failures[:20]]
            raise AssertionError("\n".join(lines))

    def table(self):
        """Lines: count, worst ratio, signature (most frequent first), then the worst ratio per operator family."""
        lines = [f"{n:5d} {r:7.3f}  {sig}" for sig, (n, r, _) in sorted(self.rows.items(), key=lambda kv: (-kv[1][0], kv[0]))]
        fam = defaultdict(float)
        for n, r, name in self.rows.values():
            fam[_family(name)] = max(fam[_family(name)], r)
        lines.append("worst err/tol per family: " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(fam.items())))
        return lines


def _first(res):
    return res[0] if isinstance(res, tuple) else res


def _tensors(res):
    items = res if isinstance(res, tuple) else (res,)
    out = []
    for t in items:
        if torch.is_tensor(t):
            out.append(t)
        elif isinstance(t, ops.RowStats):
            out.append(t.data)
    return out
