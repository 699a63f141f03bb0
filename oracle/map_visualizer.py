"""TEST INFRASTRUCTURE ONLY — a numpy restatement of the reference's test-run images (magicdrive/runner/map_visualizer.py
`visualize_map`, runner/img_utils.py `concat_6_views` and `img_m11_to_01` with torchvision's `to_pil_image`), written
for whole arrays instead of the reference's per-pixel loop, and without matplotlib: the legend is a callable.
tests/test_visualize_cpu.py holds it to the reference's own output (tests/golden/map_visualizer.pt); the GPU tests hold
magicdrive_b200.visualize to it.  The resize is oracle/fid_protocol.py's restatement of Pillow's bicubic resample.

Departure, as in magicdrive_b200.visualize: a map value other than 0 or 1 raises ValueError.
"""
import numpy as np

from magicdrive_b200.visualize import COLORS, STATIC_PRIORITY, resized_side
from oracle import fid_protocol


def render(bev_map, map_classes, object_classes):
    """bev_map (C, H, W), values 0 / 1 -> (uint8 (H, W, 3) image, set of the class names the legend shows)."""
    m = np.asarray(bev_map)
    if not np.isin(m, (0, 1)).all():
        raise ValueError("map values must be 0 or 1")
    C, H, W = m.shape
    S = min(len(map_classes), C)
    D = max(0, min(len(object_classes), C - len(map_classes)))
    if S + D == 0:
        raise ValueError("no static and no dynamic layers")
    img = np.broadcast_to(np.array(COLORS["nothing"], np.uint8), (H, W, 3)).copy()
    used = set()
    if S:
        act = m[:S] != 0
        used |= {map_classes[i] for i in range(S) if act[i].any()}
        prio = np.array([STATIC_PRIORITY.index(c) if c in STATIC_PRIORITY else -1 for c in map_classes[:S]])
        chosen = np.where(act, prio[:, None, None], -(1 << 30)).argmax(0)  # the first maximum
        any_s = act.any(0)
        # get_color_by_priority at each pixel in raster order: the rank lookup, then the colour of the class it chose
        unranked = (act & (prio < 0)[:, None, None]).any(0).ravel()
        colourless = (any_s & ~np.isin(chosen, [i for i, c in enumerate(map_classes[:S]) if c in COLORS])).ravel()
        p_rank = unranked.argmax() if unranked.any() else unranked.size
        p_colour = colourless.argmax() if colourless.any() else colourless.size
        if p_rank < unranked.size and p_rank <= p_colour:
            bad = [map_classes[i] for i in range(S) if act.reshape(S, -1)[i, p_rank] and prio[i] < 0][0]
            raise ValueError(f"{bad!r} is not in list")
        if p_colour < colourless.size:
            raise KeyError(map_classes[chosen.ravel()[p_colour]])
        for i in np.unique(chosen[any_s]):
            img[any_s & (chosen == i)] = COLORS[map_classes[i]]
    if D:
        dyn = m[S:S + D]
        colors = np.array([COLORS[c] for c in object_classes], np.uint8)  # KeyError, as render_dynamic
        k = dyn.argmax(0)
        used |= {object_classes[i] for i in np.unique(k)}  # every pixel's argmax, set or not
        any_d = (dyn != 0).any(0)
        img[any_d] = colors[k[any_d]]
    return img, used


def attach_legend(rendered, legend):
    """visualize_map's legend placement: beside the image when the legend is taller than wide, else below."""
    h, w, _ = rendered.shape
    lh, lw, _ = legend.shape
    if lh > lw:
        out = np.pad(rendered, ((0, 0), (0, lw), (0, 0)))
        out[:, w:] = legend
    else:
        out = np.pad(rendered, ((0, lh), (0, 0), (0, 0)))
        out[h:, :] = legend
    return out


def visualize_map(bev_map, map_classes, object_classes, target_size, legend):
    """uint8 image of visualize_map(cfg, bev_map, target_size) with show_legend replaced by legend(names, size).
    Square maps only.  Returns (image, frozenset of the names passed to the legend)."""
    img, used = render(bev_map, map_classes, object_classes)
    H, W, _ = img.shape
    if H != W:
        raise ValueError("only square maps")
    s = resized_side(W, target_size)
    if s != W:
        img = fid_protocol.resample_u8(img, s, s)
    names = frozenset(used)
    return attach_legend(np.rot90(img), np.asarray(legend(names, target_size))), names


def concat_6_views(views, oneline=False):
    """views uint8 (V, H, W, C) -> the concat_6_views mosaic; black fill, alpha 255 for RGBA."""
    V, H, W, C = views.shape
    row = lambda vs: np.concatenate(list(vs), 1)
    if oneline:
        return row(views)
    top, bottom = row(views[:3]), row(views[3:])
    out = np.zeros((2 * H, max(top.shape[1], bottom.shape[1]), C), np.uint8)
    if C == 4:
        out[..., 3] = 255
    out[:H, :top.shape[1]] = top
    out[H:, :bottom.shape[1]] = bottom
    return out


def m11_to_u8(img):
    """to_pil_image(img_m11_to_01(img)) pixels: fp32 (..., 3, H, W) -> uint8 (..., H, W, 3), each step rounded to fp32,
    then truncated toward zero."""
    x = np.asarray(img, np.float32)
    v = (x * np.float32(0.5) + np.float32(0.5)) * np.float32(255)
    return np.moveaxis(v.astype(np.int32).astype(np.uint8), -3, -1)
