"""The linear GEMM epilogue loads residuals in batches ahead of the output stores of the batch.  The residual may be the
output buffer itself (the zero convolutions add into the UNet skip in place), so every tile width must still read each
residual element before its own result overwrites it, and give bitwise what a separate residual buffer gives."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from magicdrive_b200 import ops  # noqa: E402
from tests.test_kernel_edges_gpu import BF16, F64, _close  # noqa: E402


@pytest.mark.parametrize("block_n", [64, 128, 160, 256])
@pytest.mark.parametrize("shape", [(3, 7, 13, 128, 96, 3), (2, 14, 25, 320, 328, 1)], ids=["conv3x3_n96", "gemm_n328"])
def test_residual_in_place(block_n, shape):
    n, h, w, c0, co, taps = shape
    g = torch.Generator(device="cuda").manual_seed(block_n + co)
    pix = n * h * w
    k = taps * taps * c0
    x = torch.randn(pix, c0, device="cuda", generator=g).to(BF16)
    wm = (torch.randn(co, k, device="cuda", generator=g) / math.sqrt(k)).to(BF16)
    b = torch.randn(co, device="cuda", generator=g)
    rb = torch.randn(n, co, device="cuda", generator=g)
    ld = co + 24  # the output is a column slice of a wider buffer, as the skip concat buffers are
    buf = torch.randn(pix, ld, device="cuda", generator=g).to(BF16)
    res = buf[:, 8:8 + co]
    kw = dict(n_img=n, h_in=h, w_in=w, c0=c0, lda0=c0, n_out=co, taps=taps, pad=taps // 2, bias=b, rowbias=rb,
              out_scale=0.75, force_block_n=block_n, kernel_variant=4)

    separate = torch.empty(pix, co, dtype=BF16, device="cuda")
    ops.gemm_conv(x, wm, residual=res.clone(), ldr=co, out=separate, ldo=co, **kw)
    before = buf.clone()
    ops.gemm_conv(x, wm, residual=res, ldr=ld, out=res, ldo=ld, **kw)
    torch.cuda.synchronize()

    assert torch.equal(buf[:, :8], before[:, :8]) and torch.equal(buf[:, 8 + co:], before[:, 8 + co:]), \
        "columns outside the output slice changed"
    assert torch.equal(res.contiguous().view(torch.int16), separate.view(torch.int16)), \
        "in-place residual differs from a separate residual buffer"
    xi = x.to(F64).view(n, h, w, c0).permute(0, 3, 1, 2)
    wt = wm.to(F64).view(co, taps, taps, c0).permute(0, 3, 1, 2)
    ref = torch.nn.functional.conv2d(xi, wt, padding=taps // 2).permute(0, 2, 3, 1).reshape(pix, co)
    ref = (ref + b.to(F64) + rb.to(F64).repeat_interleave(h * w, 0)) * 0.75 + before[:, 8:8 + co].to(F64)
    _close(separate, ref, f"block_n={block_n}")
