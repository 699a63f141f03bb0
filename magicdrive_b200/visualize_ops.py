"""torch.Tensor-facing wrappers of the C-ABI map-image and mosaic kernels (mdb_render_bev_map, mdb_place_map_u8,
mdb_concat_views_u8, mdb_m11_to_u8; csrc/capi_visualize.cu).  visualize.py builds the reference's test-run images from
them.

They sit beside ops.py and share its plumbing: raw pointers and the current stream go to `libmagicdrive_b200.so`, launches
count in `ops.launch_count()`, and there is no CPU or eager fallback.  Their CPU restatement for host tests is
tests/visualize_ops_emulator.py.
"""
import torch

from . import _lib, ops
from ._lib import check
from .ops import _need_cuda, _ptr, _stream


def render_bev_map(maps, n_static: int, n_dynamic: int, priority, colors, *, out=None, info=None):
    """mdb_render_bev_map: maps (B, C, H, W) fp32, uint8 or bool -> (out uint8 (B, H, W, 3), info int64 (B, 4)).
    Channels [0, n_static) are coloured by the highest int32 `priority` (-1: no rank), [n_static, n_static + n_dynamic)
    by the first set; colors: uint8 (n_static + n_dynamic, 4), RGB and a has-colour flag.  info per map: semantic_used as
    a class mask, a status word (bit 0: a value other than 0 or 1), and the first (pixel << 6 | class) where an active
    static class has no rank and where the chosen static class has no colour (all ones: never)."""
    _need_cuda(maps, priority, colors, out, info)
    if maps.dtype not in (torch.float32, torch.uint8, torch.bool) or maps.dim() != 4:
        raise ValueError(f"expected fp32, uint8 or bool maps (B, C, H, W), got {maps.dtype} {tuple(maps.shape)}")
    if priority.dtype != torch.int32 or colors.dtype != torch.uint8 or colors.shape != (n_static + n_dynamic, 4):
        raise ValueError("priority must be int32 and colors uint8 (n_static + n_dynamic, 4)")
    maps = maps.contiguous()
    B, C, H, W = maps.shape
    if out is None:
        out = torch.empty((B, H, W, 3), dtype=torch.uint8, device=maps.device)
    if info is None:
        info = torch.empty((B, 4), dtype=torch.int64, device=maps.device)
    check(_lib.lib().mdb_render_bev_map(_ptr(maps), int(maps.dtype == torch.float32), B, C, H, W, n_static, n_dynamic,
                                        _ptr(priority.contiguous()), _ptr(colors.contiguous()), _ptr(out), _ptr(info),
                                        _stream()), "mdb_render_bev_map")
    ops._launches += 1
    return out, info


def place_map_u8(resized, desc, max_pixels: int, out):
    """mdb_place_map_u8: resized uint8 (B, s, s, 3) -> each map rotated by 90 degrees counter-clockwise with its legend
    beside or below it, written into the flat uint8 `out`.  desc: int64 (B, 5) device rows (legend address, lh, lw, right,
    byte offset in out); max_pixels: the largest image's pixel count."""
    _need_cuda(resized, desc, out)
    if resized.dtype != torch.uint8 or resized.dim() != 4 or resized.shape[1] != resized.shape[2] or resized.shape[3] != 3:
        raise ValueError(f"expected uint8 (B, s, s, 3), got {resized.dtype} {tuple(resized.shape)}")
    if desc.dtype != torch.int64 or desc.shape != (resized.shape[0], 5) or out.dtype != torch.uint8:
        raise ValueError("desc must be int64 (B, 5) and out uint8")
    resized = resized.contiguous()
    check(_lib.lib().mdb_place_map_u8(_ptr(resized), resized.shape[0], resized.shape[1], _ptr(desc.contiguous()),
                                      int(max_pixels), _ptr(out), _stream()), "mdb_place_map_u8")
    ops._launches += 1
    return out


def concat_views_u8(views, oneline: bool = False, *, out=None):
    """mdb_concat_views_u8: uint8 views (S, V, H, W, C), C = 3 or 4 -> concat_6_views mosaics (S, 2H, max(3, V - 3) W, C),
    or with oneline (S, H, V W, C)."""
    _need_cuda(views, out)
    if views.dtype != torch.uint8 or views.dim() != 5 or views.shape[-1] not in (3, 4):
        raise ValueError(f"expected uint8 views (S, V, H, W, 3 | 4), got {views.dtype} {tuple(views.shape)}")
    views = views.contiguous()
    S, V, H, W, C = views.shape
    shape = (S, H, V * W, C) if oneline else (S, 2 * H, max(3, V - 3) * W, C)
    if out is None:
        out = torch.empty(shape, dtype=torch.uint8, device=views.device)
    check(_lib.lib().mdb_concat_views_u8(_ptr(views), S, V, H, W, C, int(oneline), _ptr(out), _stream()),
          "mdb_concat_views_u8")
    ops._launches += 1
    return out


def m11_to_u8(x, *, out=None):
    """mdb_m11_to_u8: fp32 (N, 3, H, W) in [-1, 1] -> uint8 (N, H, W, 3), to_pil_image(img_m11_to_01(x)) per image."""
    _need_cuda(x, out)
    if x.dtype != torch.float32 or x.dim() != 4 or x.shape[1] != 3:
        raise ValueError(f"expected fp32 (N, 3, H, W), got {x.dtype} {tuple(x.shape)}")
    x = x.contiguous()
    N, _, H, W = x.shape
    if out is None:
        out = torch.empty((N, H, W, 3), dtype=torch.uint8, device=x.device)
    check(_lib.lib().mdb_m11_to_u8(_ptr(x), N, H, W, _ptr(out), _stream()), "mdb_m11_to_u8")
    ops._launches += 1
    return out
