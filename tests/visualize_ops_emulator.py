"""TEST INFRASTRUCTURE ONLY — a torch restatement of the operators of magicdrive_b200/visualize_ops.py (the map-image and
mosaic kernels), following include/magicdrive_b200.h, so that visualize.py's host logic runs in the build container,
which has no GPU.  Never imported by the package; `install(monkeypatch)` swaps it in for one test.  Every function takes
exactly the arguments of its visualize_ops.py counterpart (tests/test_visualize_ops_emulator_cpu.py holds them equal).
`place_map_u8` reads the legends through the addresses in `desc`, as the kernel does, so they must be CPU tensors that
are alive."""
import ctypes

import numpy as np
import torch

from magicdrive_b200 import visualize_ops


def render_bev_map(maps, n_static, n_dynamic, priority, colors, *, out=None, info=None):
    B, C, H, W = maps.shape
    assert 0 < n_static + n_dynamic <= min(C, 64), (n_static, n_dynamic, C)
    m = maps.cpu()
    bits = m.view(torch.int32) & 0x7fffffff if m.dtype == torch.float32 else m.to(torch.int32)
    act = bits != 0
    binary = ~act | ((m == 1) if m.dtype != torch.float32 else (m.view(torch.int32) == 0x3f800000))
    status = (~binary[:, :n_static + n_dynamic]).flatten(1).any(1).long()
    cols = colors.cpu().long()
    img = torch.tensor([200, 200, 200]).expand(B, H, W, 3).clone()
    used = torch.zeros(B, dtype=torch.int64)
    none = torch.full((B,), -1, dtype=torch.int64)  # all ones
    no_rank, no_colour = none.clone(), none.clone()

    def first(hit, cls):
        """per map, (pixel << 6 | cls at that pixel) of the first pixel in raster order where hit, else all ones"""
        hit, cls = hit.flatten(1), cls.flatten(1)
        p = hit.long().argmax(1)
        word = p << 6 | cls.gather(1, p[:, None])[:, 0]
        return torch.where(hit.any(1), word, none)

    if n_static:
        sa = act[:, :n_static]
        prio = priority.cpu()[:n_static].long().view(1, -1, 1, 1)
        ranked = torch.where(sa, prio, torch.iinfo(torch.int64).min)
        chosen = ranked.argmax(1)  # the first maximum
        any_s = sa.any(1)
        unranked = sa & (prio < 0)
        no_rank = first(unranked.any(1), unranked.to(torch.int8).argmax(1))
        no_colour = first(any_s & (cols[chosen][..., 3] == 0), chosen)
        img = torch.where(any_s[..., None], cols[chosen][..., :3], img)
        for c in range(n_static):
            used |= sa[:, c].flatten(1).any(1).long() << c
    if n_dynamic:
        da = act[:, n_static:n_static + n_dynamic]
        k = da.to(torch.int8).argmax(1)  # the first layer set, 0 where none is
        any_d = da.any(1)
        img = torch.where(any_d[..., None], cols[n_static + k][..., :3], img)
        for c in range(n_dynamic):
            used |= (k == c).flatten(1).any(1).long() << (n_static + c)
    res = img.to(torch.uint8)
    inf = torch.stack([used, status, no_rank, no_colour], 1)
    if out is not None:
        out.copy_(res)
        res = out
    if info is not None:
        info.copy_(inf)
        inf = info
    return res, inf


def _read(addr, shape):
    n = int(np.prod(shape))
    if n == 0:
        return np.zeros(shape, np.uint8)
    return np.frombuffer((ctypes.c_uint8 * n).from_address(addr), np.uint8).reshape(shape).copy()


def place_map_u8(resized, desc, max_pixels, out):
    r = resized.cpu().numpy()
    s = r.shape[1]
    for m, (addr, lh, lw, right, off) in enumerate(desc.cpu().tolist()):
        rot = np.rot90(r[m])
        img = np.concatenate([rot, _read(addr, (s, lw, 3))], 1) if right else \
            np.concatenate([rot, _read(addr, (lh, s, 3))], 0)
        assert img.shape[0] * img.shape[1] <= max_pixels
        out[off:off + img.size] = torch.from_numpy(img.reshape(-1).copy())
    return out


def concat_views_u8(views, oneline=False, *, out=None):
    v = views.cpu()
    S, V, H, W, C = v.shape
    assert V >= (2 if oneline else 5), V
    if oneline:
        res = v.permute(0, 2, 1, 3, 4).reshape(S, H, V * W, C)
    else:
        ow = max(3, V - 3) * W
        res = torch.zeros((S, 2 * H, ow, C), dtype=torch.uint8)
        if C == 4:
            res[..., 3] = 255
        res[:, :H, :3 * W] = v[:, :3].permute(0, 2, 1, 3, 4).reshape(S, H, 3 * W, C)
        res[:, H:, :(V - 3) * W] = v[:, 3:].permute(0, 2, 1, 3, 4).reshape(S, H, (V - 3) * W, C)
    if out is not None:
        out.copy_(res)
        return out
    return res


def m11_to_u8(x, *, out=None):
    assert x.dtype == torch.float32 and x.dim() == 4 and x.shape[1] == 3
    res = ((x.cpu() * 0.5 + 0.5) * 255).to(torch.int32).to(torch.uint8).permute(0, 2, 3, 1).contiguous()
    if out is not None:
        out.copy_(res)
        return out
    return res


EMULATED = ["render_bev_map", "place_map_u8", "concat_views_u8", "m11_to_u8"]


def install(monkeypatch):
    """Swap every operator of magicdrive_b200.visualize_ops for its CPU restatement, and let visualize.py's device checks
    pass CPU tensors."""
    for name in EMULATED:
        assert hasattr(visualize_ops, name), name
        monkeypatch.setattr(visualize_ops, name, globals()[name])
    from magicdrive_b200 import visualize
    monkeypatch.setattr(visualize, "_need_cuda", lambda *ts: None)
