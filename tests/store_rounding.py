"""Store rounding of the bf16 / f16 outputs, and a float64 error model of the GEMM / implicit-GEMM convolution's fp32 value
(csrc/gemm_wgmma.cuh, csrc/gemm_tc.cuh).

Why a storage-type output can be held bit for bit.  The GEMM kernel has an fp32 output mode: `out_is_f32` is a runtime branch
at the store (gemm_wgmma_kernel, splitk_finalize_kernel) and the planner (capi_gemm.cu plan_for) does not read it, so a launch
with fp32 output runs the same tiles, K order and fp32 epilogue as the bf16 / f16 launch and stores the value the other one
rounds.  The storage-type output must therefore equal `out_f32.to(dt)` bitwise (torch rounds fp32 -> bf16 / f16 to nearest
even), and only the fp32 value needs a float64 bound.

The bracket.  Let v be the float64 value and x̂ the kernel's fp32 value with |x̂ − v| ≤ δ.  f = RN_dt ∘ RN_fp32 is monotone
(each rounding is), and f(x̂) = RN_dt(x̂) because x̂ is already fp32, so the stored value lies in [f(v − δ), f(v + δ)], which
torch computes as `(v ∓ δ).to(float32).to(dt)`.  Rounding through fp32 first moves each end by at most an fp32 rounding,
2⁻²⁴|v|, which is below any δ of this model.  The ends become ±0, subnormals or ±inf exactly as the store does (f16 past 65520
rounds to inf); a NaN output lies in no bracket.

Store statistics.  For elements whose float64 reference r lies in the normal range of dt, e = (out − r)·sign(r)/ulp(r) has
mean about 0 and rms 1/√12 ≈ 0.289 for a round-to-nearest store of an accurate value; truncation moves the mean to −0.5 and a
second rounding raises the rms to about 0.41.  This criterion is statistical by design: it is for the stores that have no fp32
twin, where only the distribution of the rounding errors can tell a correct store from a biased one.

The fp32 value's bound (gemm_model).  v is tests/ops_emulator.gemm_conv in float64.  The kernel accumulates in fp32 on the
tensor cores: one wgmma per k16 step, whose products are exact.  With S_j the float64 prefix sum after k16 step j
(restarting at every split-K boundary), the model allows the accumulator an error of at most U·(Σ_j |S_j| + Σ_k |a_k w_k|),
U = ACC_ULPS·2⁻²³ per k16 step.  One fp32 ulp per step (ACC_ULPS = 1) is not enough on an H100: operands that are all
nonnegative, where every rounding toward zero adds up, reach 1.76 x that bound at K = 11520 and 23040, the error always
toward zero (DESIGN §4).  ACC_ULPS = 4 is one truncation per k4 group of the step.  The model takes the prefix sums S_b at
the end of each 64-wide K block b: a k16 prefix inside block b differs from S_b by at most the block's Σ|a w|, so
Σ_j |S_j| ≤ 4 Σ_b |S_b| + 4 Σ|a w| and

    δ_acc = U·(4 Σ_b |S_b| + 5 Σ_k |a_k w_k|) + 2⁻²⁴ Σ_{s=1}^{splits−1} |P_s|,

the last term for the split-K finalise, which adds the splits in order (P_s: float64 sum of splits 0..s).  The epilogue then
takes at most four fp32 roundings (bias + rowbias, the scale, the fma with the accumulator, the residual add; the finalise
rounds bias, rowbias, scale and residual adds), each of a quantity no larger than T = |scale|·(Σ|a w| + |bias| + |rowbias|) +
|residual|, which is the same emulator call on the absolute values of every operand:

    δ = |scale|·δ_acc + 4·2⁻²⁴·T.

This is a model of Hopper's tensor cores, not a measured fact; test_store_rounding_gpu.py records the worst |out − v|/δ per
family.  Everything is computed on the operands' device, CHUNK elements of the widest operand (or one image) at a time.

Activation epilogues (gelu_erf, quick_gelu in csrc/gemm_tc.cuh) are evaluated here in float64 on the kernel's fp32 value,
and the bracket widened by their approximation error, derived once below (EPS_ERF, quick_gelu_eps)."""
import inspect
import math

import torch
import torch.nn.functional as F

from tests import ops_emulator

BF16, F16, F32, F64 = torch.bfloat16, torch.float16, torch.float32, torch.float64
MANT = {BF16: 7, F16: 10}  # explicit mantissa bits
EMIN = {BF16: -126, F16: -14}  # exponent of the smallest normal
CHUNK = 1 << 25  # elements of one float64 chunk (rows x widest operand), as tests/launch_census.py
ACC_ULPS = 4  # fp32 ulps the tensor cores may lose per k16 step (module docstring)

# gelu_erf: erf by Abramowitz-Stegun 7.1.26, erf(y) = 1 - P(t) e^(-y^2) with t = 1 / (1 + 0.3275911 y), |error| <= 1.5e-7.
# The kernel takes t from rcp.approx and e^(-y^2) from ex2.approx, each within 2^-22 relative.  Over t in (0, 1],
# |t P'(t)| e^(-y^2) <= 3.45 (at y = 0) and P(t) e^(-y^2) = erfc(y) <= 1, whose argument -log2(e) y^2 carries three fp32
# roundings (erfc(y) y^2 <= 0.17); the Horner chain and the final fma add about eight fp32 roundings of numbers <= 1.
# Together 1.5e-7 + (3.45 + 1.2 + 2) 2^-22 < 1.5e-7 + 2^-19 absolute in erf.
EPS_ERF = 1.5e-7 + 2.0 ** -19


def gelu_eps(g):
    """Bound on |gelu_erf(g) - gelu(g)| for the kernel's fp32 g: |g| / 2 * EPS_ERF for erf, plus the roundings of
    0.5 g and of the final fma (2^-23 |gelu(g)|)."""
    g = g.to(F64)
    return g.abs() * (0.5 * EPS_ERF) + 2.0 ** -23 * F.gelu(g).abs()


def quick_gelu_eps(x):
    """Bound on |quick_gelu(x) - x sigmoid(1.702 x)| for the kernel's fp32 x.  The kernel computes x * rcp(1 + ex2(c x))
    with c = fp32(-1.702 log2 e): c and c x carry three 2^-24 relative roundings (1.702f included), which ex2 turns into a
    relative error ln 2 |c x| 3 2^-24 <= 2^-22 |1.702 x| of e, next to ex2's own 2^-22; the sigmoid passes e's relative
    error on damped by e / (1 + e) <= 1; 1 + e, rcp.approx and the product add 2^-24 + 2^-22 + 2^-24.  So the relative
    error is below 2^-21 + 2^-22 (1 + |1.702 x|).  rcp.approx.ftz flushes 1 / (1 + e) below 2^-126 to zero: an absolute
    |x| 2^-126 more."""
    x = x.to(F64)
    f = x * torch.sigmoid(1.702 * x)
    return f.abs() * (2.0 ** -21 + 2.0 ** -22 * (1 + 1.702 * x.abs())) + x.abs() * 2.0 ** -126


# ------------------------------------------------------------------------------------------------- rounding, bracket
def ulp(ref, dt):
    """The spacing of dt at |ref| (float64), floored at dt's smallest step in its subnormal range (2^-133 bf16, 2^-24 f16)."""
    e = torch.floor(torch.log2(ref.to(F64).abs().clamp_min(2.0 ** EMIN[dt])))
    return torch.exp2(e - MANT[dt])


def bracket(v, delta, dt):
    """(lo, hi) in dt: RN_dt(RN_fp32(v - delta)), RN_dt(RN_fp32(v + delta)) elementwise."""
    v, delta = v.to(F64), delta.to(F64)
    return (v - delta).to(F32).to(dt), (v + delta).to(F32).to(dt)


def outside(out, v, delta):
    """Boolean mask of the elements of `out` (bf16 / f16) outside their bracket; a NaN is outside every bracket."""
    lo, hi = bracket(v, delta, out.dtype)
    o = out.to(F64)
    return ~((o >= lo.to(F64)) & (o <= hi.to(F64)))


def check_bracket(out, v, delta, what=""):
    bad = outside(out, v, delta)
    n = int(bad.sum())
    if n:
        i = tuple(bad.nonzero()[0].tolist())
        raise AssertionError(f"{what}: {n} of {bad.numel()} elements outside [RN(v - d), RN(v + d)], first at {i}: "
                             f"out {out[i].item():.8g}, v {v[i].item():.10g}, d {delta[i].item():.3g}")


def store_stats(out, ref):
    """(signed mean, rms, count) of (out - ref) sign(ref) / ulp(ref) in units of out's type, over the elements whose
    float64 reference lies in the normal range of that type."""
    dt = out.dtype
    r = ref.to(F64)
    a = r.abs()
    keep = (a >= 2.0 ** EMIN[dt]) & (a <= torch.finfo(dt).max) & torch.isfinite(out.to(F64))
    e = ((out.to(F64) - r) * torch.sign(r) / ulp(r, dt))[keep]
    if e.numel() == 0:
        return 0.0, 0.0, 0
    return e.mean().item(), e.pow(2).mean().sqrt().item(), e.numel()


MEAN_MAX, RMS_MAX, MIN_COUNT = 0.05, 0.35, 10_000


def check_stats(out, ref, what=""):
    """|signed mean| <= 0.05 ulp and rms <= 0.35 ulp over at least 10^4 normal-range elements (round to nearest: 0 +- 0.003
    and 0.289 at that count).  Returns (mean, rms, count)."""
    mean, rms, n = store_stats(out, ref)
    assert n >= MIN_COUNT, f"{what}: only {n} normal-range elements"
    assert abs(mean) <= MEAN_MAX and rms <= RMS_MAX, \
        f"{what}: store error mean {mean:+.4f} ulp, rms {rms:.4f} ulp over {n} elements (bounds {MEAN_MAX}, {RMS_MAX})"
    return mean, rms, n


def check_f32(out, v, delta, what=""):
    """|out - v| <= delta elementwise for an fp32 output; returns the worst ratio."""
    err = (out.to(F64) - v).abs()
    r = torch.where(delta > 0, err / delta.clamp_min(1e-300), torch.where(err > 0, math.inf, 0.0))
    r = torch.nan_to_num(r, nan=math.inf)
    worst = r.max().item() if r.numel() else 0.0
    if not worst <= 1.0:
        i = tuple((r == r.max()).nonzero()[0].tolist())
        raise AssertionError(f"{what}: |out - v| reaches {worst:.3g} x the model's bound, at {i}: out {out[i].item():.9g}, "
                             f"v {v[i].item():.12g}, bound {delta[i].item():.3g}")
    return worst


# ------------------------------------------------------------------------------------------------- GEMM model
_GEMM_DEFAULTS = {k: p.default for k, p in inspect.signature(ops_emulator.gemm_conv).parameters.items()
                  if p.default is not inspect.Parameter.empty}


def _chunks(n, per, budget=CHUNK):
    step = max(1, budget // max(per, 1))
    return [(i, min(i + step, n)) for i in range(0, n, step)]


def _abs_operands(ck):
    """The emulator arguments with every operand replaced by its absolute value (row strides follow the copies)."""
    a = dict(ck)
    a["a0"] = ck["a0"][:, :ck["c0"]].abs()
    a["lda0"] = a["a0"].stride(0)
    if ck["c1"]:
        a["a1"] = ck["a1"][:, :ck["c1"]].abs()
        a["lda1"] = a["a1"].stride(0)
    a["w"] = ck["w"].abs()
    for k in ("bias", "rowbias"):
        if ck[k] is not None:
            a[k] = ck[k].abs()
    if ck["residual"] is not None:
        a["residual"] = ck["residual"].reshape(-1, ck["residual"].shape[-1])[:, :ck["n_out"]].abs()
        a["ldr"] = a["residual"].stride(0)
    a["out_scale"] = abs(ck["out_scale"])
    return a


def _k_blocks(ck, kh, kw, ph, pw, ho, wo):
    """(A block [pixels, <= 64], W block [n_out, <= 64]) in float64, in the kernel's K order: filter tap, then source 0's
    64-channel blocks, then source 1's (the last block of a source partial when its channel count is not a multiple of 64)."""
    n, h, w, s = ck["n_img"], ck["h_in"], ck["w_in"], ck["stride"]
    srcs = [(ck["a0"], ck["c0"])] + ([(ck["a1"], ck["c1"])] if ck["c1"] else [])
    widths = [-(-c // 64) * 64 for _, c in srcs]
    kt = sum(widths)
    wt = ck["w"].to(F64)
    xs = []
    for a, c in srcs:
        x = a[:, :c].to(F64).reshape(n, h, w, c).permute(0, 3, 1, 2)
        xs.append(F.pad(x, (pw, pw + ck["pad_w_end"], ph, ph + ck["pad_h_end"])))
    for r in range(kh):
        for q in range(kw):
            tap = r * kw + q
            off = 0
            for x, width in zip(xs, widths):
                cols = x[:, :, r:r + s * (ho - 1) + 1:s, q:q + s * (wo - 1) + 1:s].permute(0, 2, 3, 1).reshape(n * ho * wo, -1)
                for c0 in range(0, width, 64):
                    ab = cols[:, c0:c0 + 64]
                    yield ab, wt[:, tap * kt + off + c0: tap * kt + off + c0 + ab.shape[1]]
                off += width


def _acc_bound(ck, kh, kw, ph, pw, ho, wo, splits):
    """δ_acc of the module docstring for one chunk: [pixels, n_out] float64."""
    kb_total = kh * kw * sum(-(-c // 64) for c in (ck["c0"], ck["c1"]) if c)
    kps = -(-kb_total // splits)
    assert -(-kb_total // kps) == splits, (kb_total, splits)
    pre = absk = fin = tot = s_ = None
    for kb, (ab, wb) in enumerate(_k_blocks(ck, kh, kw, ph, pw, ho, wo)):
        p = ab @ wb.t()
        pa = ab.abs() @ wb.abs().t()
        if s_ is None:
            s_, pre, absk, fin, tot = p, p.abs(), pa, torch.zeros_like(p), torch.zeros_like(p)
        else:
            s_ = s_ + p
            pre += s_.abs()
            absk += pa
        if (kb + 1) % kps == 0 or kb + 1 == kb_total:  # a split ends: the finalise adds it to the running sum
            tot += s_
            if kb + 1 > kps:
                fin += tot.abs()
            s_ = torch.zeros_like(p)
    assert kb + 1 == kb_total, (kb, kb_total)
    u = ACC_ULPS * 2.0 ** -23
    return u * (4 * pre + 5 * absk) + 2.0 ** -24 * fin


def gemm_model(call, splits=1):
    """(v, δ) [pixels, n_out] float64 of one linear-epilogue ops.gemm_conv launch: `call` holds its arguments by name
    (inspect.signature(ops.gemm_conv).bind(...).arguments; out, ldo, out_f32 and emit_stats are ignored), `splits` the
    planner's split count (mdb_gemm_conv_plan)."""
    a = {k: v for k, v in call.items() if k in _GEMM_DEFAULTS or k in ("a0", "w", "n_img", "h_in", "w_in", "c0", "lda0",
                                                                       "n_out")}
    assert a.get("ln") is None and not a.get("geglu") and not a.get("quick_gelu") and not a.get("relu"), \
        "the model describes the linear epilogue"
    for k in ("out", "ldo", "emit_stats", "h_out", "w_out"):
        a.pop(k, None)
    a = {**{k: v for k, v in _GEMM_DEFAULTS.items() if k not in ("out", "ldo", "emit_stats", "h_out", "w_out")}, **a,
         "out_f32": True}
    kh = a["taps"] if a["taps_h"] is None else a["taps_h"]
    kw = a["taps"] if a["taps_w"] is None else a["taps_w"]
    ph = a["pad"] if a["pad_h"] is None else a["pad_h"]
    pw = a["pad"] if a["pad_w"] is None else a["pad_w"]
    n, h, w, s = a["n_img"], a["h_in"], a["w_in"], a["stride"]
    ho = (h + 2 * ph + a["pad_h_end"] - kh) // s + 1
    wo = (w + 2 * pw + a["pad_w_end"] - kw) // s + 1
    token = n == 1 and h == 1 and kh == kw == s == 1 and ph == pw == 0 and not a["pad_h_end"] and not a["pad_w_end"]
    units, per_in, per_out = (w, 1, 1) if token else (n, h * w, ho * wo)  # rows of a token GEMM, else images
    wide = max(a["c0"] + a["c1"], a["n_out"]) * kh * kw
    vs, ds = [], []
    for u0, u1 in _chunks(units, per_in * wide):
        ck = dict(a)
        rin, rout = slice(u0 * per_in, u1 * per_in), slice(u0 * per_out, u1 * per_out)
        ck["a0"] = a["a0"][rin]
        if a["a1"] is not None:
            ck["a1"] = a["a1"][rin]
        if a["residual"] is not None:
            ck["residual"] = a["residual"].reshape(-1, a["residual"].shape[-1])[rout]
        if token:
            ck["w_in"] = u1 - u0
        else:
            ck["n_img"] = u1 - u0
            if a["rowbias"] is not None and a["rowbias"].shape[0] > 1:
                ck["rowbias"] = a["rowbias"][u0:u1]
        hw = dict(h_out=ho, w_out=u1 - u0 if token else wo)
        with ops_emulator.compute(F64):
            v = ops_emulator.gemm_conv(**ck, **hw)
            t = ops_emulator.gemm_conv(**_abs_operands(ck), **hw)
        d_acc = _acc_bound(ck, kh, kw, ph, pw, ho, u1 - u0 if token else wo, splits)
        vs.append(v)
        ds.append(abs(a["out_scale"]) * d_acc + 4 * 2.0 ** -24 * t)
    return torch.cat(vs), torch.cat(ds)
