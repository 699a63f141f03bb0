"""torch.Tensor-facing wrappers of the C-ABI 8-bit image operators of the FID evaluation protocol (mdb_resample_u8,
mdb_jpeg_roundtrip_u8; csrc/capi_fid_protocol.cu).

They sit beside ops.py, whose operators are the network's, and share its plumbing: raw pointers and the current stream
go to `libmagicdrive_b200.so`, launches count in `ops.launch_count()`, and there is no CPU or eager fallback.  Their CPU
restatement for host tests is tests/image_ops_emulator.py.
"""
import torch

from . import _lib, ops
from ._lib import check
from .ops import _need_cuda, _ptr, _stream


def resample_u8(x, size, coef_w, coef_h, *, nhwc: bool = True, crop=None, canvas=None, offset=(0, 0), tmp=None, out=None):
    """mdb_resample_u8: Pillow's 8-bit bicubic resample of x (uint8 [n, h, w, 3], or fp32 [0, 1] NHWC / NCHW with
    nhwc=False, rounded to uint8 first) to size = (rh, rw).  coef_w / coef_h: int32 [rw | rh, taps + 2] device tables
    (fid.bicubic_table), None where that size is unchanged.  The window crop = (top, left, h, w) of the result (all of it
    by default) lands at offset = (top, left) of a zero canvas = (out_h, out_w) (the window's size by default): uint8
    [n, out_h, out_w, 3]."""
    _need_cuda(x, coef_w, coef_h)
    if x.dtype not in (torch.uint8, torch.float32):
        raise ValueError(f"resample_u8 takes uint8 or float32 images, got {x.dtype}")
    x = x.contiguous()
    if x.dtype == torch.uint8 and not nhwc:
        raise ValueError("uint8 images must be NHWC")
    n, h, w = (x.shape[0], x.shape[1], x.shape[2]) if nhwc else (x.shape[0], x.shape[2], x.shape[3])
    if (x.shape[3] if nhwc else x.shape[1]) != 3:
        raise ValueError(f"expected 3 channels, got shape {tuple(x.shape)}")
    rh, rw = size
    crop = (0, 0, rh, rw) if crop is None else tuple(crop)
    canvas = crop[2:] if canvas is None else tuple(canvas)
    if out is None:
        out = torch.empty((n, *canvas, 3), dtype=torch.uint8, device=x.device)
    if coef_w is not None and tmp is None:
        tmp = torch.empty((n, h, crop[3], 3), dtype=torch.uint8, device=x.device)
    taps_w = 0 if coef_w is None else coef_w.shape[1] - 2
    taps_h = 0 if coef_h is None else coef_h.shape[1] - 2
    check(_lib.lib().mdb_resample_u8(_ptr(x), int(x.dtype == torch.float32), int(nhwc), n, h, w, _ptr(coef_w), taps_w, rw,
                                     _ptr(coef_h), taps_h, rh, *crop, _ptr(tmp), _ptr(out), canvas[0], canvas[1], *offset,
                                     _stream()), "mdb_resample_u8")
    ops._launches += 2 if coef_w is not None else 1
    return out


def jpeg_roundtrip_u8(x, quality: int = 75, *, planes=None, out=None):
    """mdb_jpeg_roundtrip_u8: uint8 RGB [n, h, w, 3] -> the image Pillow decodes from a baseline 4:2:0 JPEG it saved at
    `quality`.  planes: uint8 scratch of at least n * hp * wp * 3 / 2 bytes (hp, wp: h, w rounded up to 16); out may be x."""
    _need_cuda(x)
    if x.dtype != torch.uint8 or x.dim() != 4 or x.shape[3] != 3:
        raise ValueError(f"expected uint8 [n, h, w, 3], got {x.dtype} {tuple(x.shape)}")
    x = x.contiguous()
    n, h, w = x.shape[:3]
    need = n * (-(-h // 16) * 16) * (-(-w // 16) * 16) * 3 // 2
    if planes is None:
        planes = torch.empty(need, dtype=torch.uint8, device=x.device)
    elif planes.numel() < need:
        raise ValueError(f"planes holds {planes.numel()} bytes, {need} needed")
    if out is None:
        out = torch.empty_like(x)
    check(_lib.lib().mdb_jpeg_roundtrip_u8(_ptr(x), n, h, w, quality, _ptr(planes), _ptr(out), _stream()),
          "mdb_jpeg_roundtrip_u8")
    ops._launches += 2
    return out
