"""Weight packing for the sm_90a kernels (bf16, K-major, tap-major conv filters, GEGLU tile interleave)."""
import torch


def pack_conv_weight(w: torch.Tensor) -> torch.Tensor:
    """[Cout, Cin, kh, kw] -> bf16 [Cout, kh*kw*Cin] with K ordered (tap, channel) as mdb_gemm_conv expects."""
    co, ci, kh, kw = w.shape
    return w.permute(0, 2, 3, 1).reshape(co, kh * kw * ci).contiguous().to(torch.bfloat16)


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
