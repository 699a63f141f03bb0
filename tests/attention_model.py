"""float64 attention and an error model of the fused attention kernel's roundings (csrc/attention_wgmma.cuh).

The kernel takes S = Q Kᵀ and P V in fp32 on the tensor cores, exponentiates in fp32 (ex2.approx: capi_attention.cu is built
with --use_fast_math), packs each P element to the storage type for the P V product, sums the row normaliser l from the
unrounded p, and rounds each set's normalised output to the storage type before adding it to the stored partial sum, which
is rounded again.  With u the unit roundoff of the storage type (2⁻⁸ bf16, 2⁻¹¹ f16), η = 2⁻²⁰ the slack for fp32
accumulation, ex2.approx and the approximate reciprocal, and a = 2⁻²⁵ the absolute rounding of an f16 P element in the
subnormal range (0 for bf16, whose exponent range is fp32's), the model computes per query row and per set s, from the
stored q, k, v over the counted keys (past kv_len and above the causal diagonal excluded):

    p̂ = softmax(q kᵀ · scale),  o_s = p̂ v,  A_s = p̂ |v|,  B_s = p̂² v²,  p̂max_s,  V1_s = Σ_j |v_j|,  S_s = Σ_{t≤s} o_t

and holds the kernel's output to two criteria against ref = S_last:

* elementwise, rigorous: |out − ref| ≤ Σ_s [u (A_s + |o_s|) + η A_s + a p̂max_s V1_s] + Σ_{s≥2} u |S_s|: one rounding of
  every P element, of every set's output and of every partial sum;
* per (query row, head), statistical: rms over the head's d columns of (out − ref) ≤ τ √mean(σ²) with
  σ² = Σ_s (u²/3)(B_s + o_s²) + Σ_{s≥2} (u²/3) S_s² + (η Σ_s A_s)², u²/3 being the largest variance of one
  round-to-nearest relative error.

The row criterion is the discriminating one: a key tile or a single key that takes no weight, or a normaliser that misses a
rescale, moves every column of a row by far more than σ even where it hides under an absolute tolerance.  A row whose counted
key set is empty (kv_len 0, or every slot -1) must be exactly zero."""
from dataclasses import dataclass

import torch

F64 = torch.float64
ETA = 2.0 ** -20
TAU = 2.0


def unit_roundoff(dt):
    return {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}[dt]


def subnormal_step(dt):
    return 2.0 ** -25 if dt == torch.float16 else 0.0


@dataclass
class AttnModel:
    ref: torch.Tensor    # [rows, heads*d] float64: the exact sum of the sets' outputs
    bound: torch.Tensor  # [rows, heads*d] the elementwise bound on |out - ref|
    var: torch.Tensor    # [rows, heads*d] σ²
    empty: torch.Tensor  # [rows] bool: no counted key in any set
    heads: int
    d: int


def attention_model(q, kv_of, b, heads, lq, d, scale, dt, causal=False, chunk=512):
    """The model for q [b*lq, >= heads*d] (row stride free) and kv_of(i) -> list of (k, v) [keys, >= heads*d] of query batch
    i's present sets in slot order, each cut to the keys it counts (an empty list: no present set).  causal: key j is
    visible to query row r iff j <= r.  Computed on q's device, `chunk` query rows at a time."""
    u, a = unit_roundoff(dt), subnormal_step(dt)
    c = heads * d
    dev = q.device
    ref, bound, var = (torch.zeros(b * lq, c, dtype=F64, device=dev) for _ in range(3))
    empty = torch.ones(b * lq, dtype=torch.bool, device=dev)
    for i in range(b):
        qi = q[i * lq:(i + 1) * lq, :c].to(F64).reshape(lq, heads, d).transpose(0, 1)
        sets = [(k[:, :c].to(F64).reshape(-1, heads, d).transpose(0, 1), v[:, :c].to(F64).reshape(-1, heads, d).transpose(0, 1))
                for k, v in kv_of(i) if k.shape[0] > 0]
        if not sets:
            continue
        empty[i * lq:(i + 1) * lq] = False
        for r in range(0, lq, chunk):
            rows = slice(r, min(r + chunk, lq))
            n = rows.stop - r
            S = bnd = vv = atot = 0
            for s, (kh, vh) in enumerate(sets):
                sc = qi[:, rows] @ kh.transpose(1, 2) * scale
                if causal:
                    j = torch.arange(kh.shape[1], device=dev)
                    sc = sc.masked_fill(j[None, None, :] > torch.arange(r, r + n, device=dev)[None, :, None], float("-inf"))
                p = torch.softmax(sc, -1)
                o = p @ vh
                A = p @ vh.abs()
                B = (p * p) @ (vh * vh)
                S = S + o
                bnd = bnd + u * (A + o.abs()) + ETA * A + a * p.amax(-1, keepdim=True) * vh.abs().sum(1, keepdim=True)
                vv = vv + (u * u / 3) * (B + o * o)
                atot = atot + A
                if s >= 1:
                    bnd = bnd + u * S.abs()
                    vv = vv + (u * u / 3) * S * S
            vv = vv + (ETA * atot) ** 2
            dst = slice(i * lq + r, i * lq + r + n)
            ref[dst], bound[dst], var[dst] = (t.transpose(0, 1).reshape(n, c) for t in (S, bnd, vv))
    return AttnModel(ref, bound, var, empty, heads, d)


def _ratio(num, den):
    """num / den, with 0 / 0 = 0, x / 0 = inf for x > 0 and NaN (a NaN output) = inf."""
    r = torch.where(den > 0, num / den.clamp_min(1e-300), torch.where(num > 0, float("inf"), 0.0))
    return torch.nan_to_num(r, nan=float("inf"))


def model_ratios(out, m: AttnModel):
    """(worst |out - ref| / bound over the elements, worst row rms / √mean σ² over the (query row, head) pairs) of the
    non-empty rows, and the number of nonzero elements in the empty ones."""
    o = out.to(F64)
    err = (o - m.ref).abs()
    full = ~m.empty
    elem = _ratio(err[full], m.bound[full])
    rows = err[full].reshape(-1, m.heads, m.d)
    rms = rows.pow(2).mean(-1).sqrt()
    sig = m.var[full].reshape(-1, m.heads, m.d).mean(-1).sqrt()
    row = _ratio(rms, sig)
    nonzero = (o[m.empty] != 0).sum().item()
    worst = lambda t: t.max().item() if t.numel() else 0.0  # noqa: E731
    return worst(elem), worst(row), nonzero


def check_model(out, m: AttnModel, what="", tau=TAU):
    """Assert both criteria (and exact zeros in empty rows); returns (elementwise ratio, row ratio)."""
    elem, row, nonzero = model_ratios(out, m)
    assert nonzero == 0, f"{what}: {nonzero} nonzero elements in rows without a counted key"
    assert elem <= 1.0, f"{what}: |out - ref| reaches {elem:.3g} x the elementwise bound (row ratio {row:.3g})"
    assert row <= tau, f"{what}: a row's rms error reaches {row:.3g} x the modelled sigma (tau {tau}; elementwise {elem:.3g})"
    return elem, row
