"""TEST INFRASTRUCTURE ONLY — a torch / numpy restatement of the operators of magicdrive_b200/image_ops.py (the FID
protocol's 8-bit image kernels), following include/magicdrive_b200.h, so that FIDProtocol's host logic runs in the build
container, which has no GPU.  Never imported by the package; `install(monkeypatch)` swaps it in for one test.  Every
function takes exactly the arguments of its image_ops.py counterpart (tests/test_image_ops_emulator_cpu.py holds them
equal).  The resample follows the coefficient tables it is given, as the kernel does; the JPEG round trip is the integer
restatement of oracle/fid_protocol.py."""
import torch

from magicdrive_b200 import image_ops


def _resample_pass(x, axis, coef):
    """One pass of the 8-bit resample along `axis` of int64 x with table rows [first, count, weights...]."""
    first, count, k = coef[:, 0].long(), coef[:, 1].long(), coef[:, 2:].long()
    x = x.movedim(axis, -1)
    acc = torch.full(x.shape[:-1] + (coef.shape[0],), 1 << 21, dtype=torch.int64)
    for t in range(k.shape[1]):
        idx = (first + t).clamp_max(x.shape[-1] - 1)
        acc += x[..., idx] * torch.where(t < count, k[:, t], 0)
    return (acc >> 22).clamp(0, 255).movedim(-1, axis)


def resample_u8(x, size, coef_w, coef_h, *, nhwc=True, crop=None, canvas=None, offset=(0, 0), tmp=None, out=None):
    if x.dtype == torch.uint8:
        assert nhwc, "uint8 images must be NHWC"
        v = x.long()
    else:
        v = (x if nhwc else x.permute(0, 2, 3, 1)).float()
        v = torch.round(v * 255).clamp(0, 255).long()
    h, w = v.shape[1:3]
    assert (coef_w is None) == (size[1] == w) and (coef_h is None) == (size[0] == h), "tables exactly for changed sizes"
    if coef_w is not None:
        v = _resample_pass(v, 2, coef_w.cpu())
    if coef_h is not None:
        v = _resample_pass(v, 1, coef_h.cpu())
    ct, cl, ch, cw = (0, 0, *size) if crop is None else crop
    assert 0 <= ct and 0 <= cl and ct + ch <= size[0] and cl + cw <= size[1], "crop outside the resize"
    canvas = (ch, cw) if canvas is None else canvas
    assert offset[0] + ch <= canvas[0] and offset[1] + cw <= canvas[1], "window outside the canvas"
    res = torch.zeros((v.shape[0], *canvas, 3), dtype=torch.uint8)
    res[:, offset[0]:offset[0] + ch, offset[1]:offset[1] + cw] = v[:, ct:ct + ch, cl:cl + cw].to(torch.uint8)
    if out is not None:
        out.copy_(res)
        return out
    return res


def jpeg_roundtrip_u8(x, quality=75, *, planes=None, out=None):
    from oracle import fid_protocol
    assert x.dtype == torch.uint8 and x.dim() == 4 and x.shape[3] == 3, (x.dtype, tuple(x.shape))
    res = torch.from_numpy(fid_protocol.jpeg_roundtrip_u8(x.cpu().numpy(), quality))
    if out is not None:
        out.copy_(res)
        return out
    return res


EMULATED = ["resample_u8", "jpeg_roundtrip_u8"]


def install(monkeypatch):
    """Swap every operator of magicdrive_b200.image_ops for its CPU restatement."""
    for name in EMULATED:
        assert hasattr(image_ops, name), name
        monkeypatch.setattr(image_ops, name, globals()[name])
