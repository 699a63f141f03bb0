"""Weight packing for the sm_90a kernels (bf16, K-major, tap-major conv filters, GEGLU tile interleave)."""
import torch


def pack_conv_weight(w: torch.Tensor) -> torch.Tensor:
    """[Cout, Cin, kh, kw] -> bf16 [Cout, kh*kw*Cin] with K ordered (tap, channel) as mdb_gemm_conv expects."""
    co, ci, kh, kw = w.shape
    return w.permute(0, 2, 3, 1).reshape(co, kh * kw * ci).contiguous().to(torch.bfloat16)


def pack_conv_weight_k64(w: torch.Tensor, splits=None, dtype=torch.bfloat16) -> torch.Tensor:
    """[Cout, Cin, kh, kw] -> bf16 [Cout, kh*kw*K64] for mdb_gemm_conv with channel counts that are multiples of 8: the
    input channels, split into the A sources' counts `splits` (default: one source), are each zero-padded to a multiple
    of 64 inside every tap.  Equals pack_conv_weight when every count is a multiple of 64."""
    co, ci, kh, kw = w.shape
    splits = [ci] if splits is None else list(splits)
    assert sum(splits) == ci
    parts, c0 = [], 0
    for c in splits:
        p = torch.zeros((co, kh, kw, (c + 63) // 64 * 64), dtype=w.dtype, device=w.device)
        p[..., :c] = w[:, c0:c0 + c].permute(0, 2, 3, 1)
        parts.append(p)
        c0 += c
    return torch.cat(parts, -1).reshape(co, -1).contiguous().to(dtype)


def pack_geglu(w: torch.Tensor, b: torch.Tensor, tile: int = 256, dtype=torch.bfloat16):
    """GEGLU.proj (attention.py:270) [2*inner, C]: rows [0, inner) are the value half, [inner, 2*inner) the gate
    half.  Re-order rows so every `tile`-row block holds tile/2 value rows followed by the matching gate rows;
    the GEMM epilogue then forms value * gelu(gate) inside one CTA tile."""
    two_inner = w.shape[0]
    inner = two_inner // 2
    half = tile // 2
    assert inner % half == 0, (inner, half)
    idx = []
    for j in range(inner // half):
        idx += list(range(j * half, (j + 1) * half))
        idx += list(range(inner + j * half, inner + (j + 1) * half))
    idx = torch.tensor(idx, device=w.device)
    return w[idx].contiguous().to(dtype), b[idx].contiguous().float()
