"""TEST INFRASTRUCTURE ONLY — a torch restatement of the C-ABI operators the FID InceptionV3 uses (include/magicdrive_b200.h:
mdb_gemm_conv with K64-packed weights, rectangular filters and the ReLU epilogue; mdb_pool2d; mdb_fid_input), so that
engine.InceptionEngine's host side (BatchNorm folding, weight packing, branch wiring into column slices) runs in the build
container against oracle/fid_inception.py.  Activations stay fp32.  `install(monkeypatch)` swaps them in for one test."""
import torch
import torch.nn.functional as F

from magicdrive_b200 import ops


def gemm_conv(a0, w, *, n_img, h_in, w_in, c0, lda0, n_out, taps=1, stride=1, pad=0, taps_h=None, taps_w=None, pad_h=None,
              pad_w=None, bias=None, relu=False, out=None, ldo=None, **_):
    kh, kw = taps_h or taps, taps_w or taps
    ph, pw = pad if pad_h is None else pad_h, pad if pad_w is None else pad_w
    k64 = (c0 + 63) // 64 * 64
    assert a0.stride(0) == lda0 and w.shape == (n_out, kh * kw * k64), (w.shape, n_out, kh, kw, k64)
    wt = w.float().view(n_out, kh, kw, k64)
    assert torch.all(wt[..., c0:] == 0), "the K64 gap must hold zeros"
    x = a0[:, :c0].float().reshape(n_img, h_in, w_in, c0).permute(0, 3, 1, 2)
    y = F.conv2d(x, wt[..., :c0].permute(0, 3, 1, 2), bias.float() if bias is not None else None, stride=stride,
                 padding=(ph, pw))
    if relu:
        y = F.relu(y)
    y = y.permute(0, 2, 3, 1).reshape(-1, n_out)
    if out is not None:
        out[:, :n_out] = y
        return out
    return y.contiguous()


def pool2d(x, *, n, h, w, c, mode, k=3, stride=1, pad=0, ldx=None, out=None, ldo=None):
    assert x.stride(0) == (ldx or c)
    xi = x[:, :c].float().reshape(n, h, w, c).permute(0, 3, 1, 2)
    if mode == ops.POOL_GLOBAL_AVG:
        y = xi.mean((2, 3))
    else:
        y = F.max_pool2d(xi, k, stride, pad) if mode == ops.POOL_MAX else F.avg_pool2d(xi, k, stride, pad,
                                                                                          count_include_pad=False)
        y = y.permute(0, 2, 3, 1).reshape(-1, c)
    if out is not None:
        out[:, :c] = y
        return out
    return y.contiguous()


def fid_input(x, *, nhwc, quantize, normalize, size=None):
    x = (x.permute(0, 3, 1, 2) if nhwc else x).float()
    if quantize:
        x = torch.round(x * 255).clamp(0, 255) / 255
    if size is not None and tuple(size) != tuple(x.shape[2:]):
        x = F.interpolate(x, size=size, mode="bilinear", align_corners=False)
    if normalize:
        x = 2 * x - 1
    return F.pad(x.permute(0, 2, 3, 1), (0, 5)).reshape(-1, 8).contiguous()


def nhwc_to_nchw(x, n, c, h, w, dtype=torch.float32):
    return x.float().reshape(n, h, w, c).permute(0, 3, 1, 2).contiguous()


def install(monkeypatch):
    for name in ("gemm_conv", "pool2d", "fid_input", "nhwc_to_nchw"):
        monkeypatch.setattr(ops, name, globals()[name])
