"""The images the reference saves for each generated sample (magicdrive/misc/test_utils.py:258-321 `run_one_batch`,
tools/test.py:74-99), made on the device and equal to the reference's pixel arrays byte for byte:

* `visualize_maps`: the BEV map image `{n}_map.png` (runner/map_visualizer.py:143-211 `visualize_map`): each pixel
  coloured from its static and dynamic layers, resized (Pillow bicubic) so its edge is `target_size`, rotated by 90
  degrees, with the class legend pasted beside or below it;
* `camera_views_u8`: the given views as the `{n}_ori.png` route converts them (`to_pil_image(img_m11_to_01(x))`);
* `concat_views`: the `concat_6_views` mosaic (runner/img_utils.py:5-40) of every saved view image;
* `save_run_images`: the PNG files of one batch, with tools/test.py's names.

The kernels are in csrc/capi_visualize.cu (wrappers: visualize_ops.py); the resize is image_ops.resample_u8.  The legend
is a matplotlib figure and is drawn on the host, once per distinct set of classes and size.  Only map arrays whose values
are all 0 or 1 are taken (the data pipeline's masks are booleans); the reference's uint8 wrap-around on other values is
not reproduced.  oracle/map_visualizer.py restates all of it in numpy.
"""
import io
import os
from typing import Callable, Dict, FrozenSet, List, Optional, Sequence

import numpy as np
import torch

from . import fid, image_ops, visualize_ops
from .box_overlay import NUSCENES_OBJECT_CLASSES
from .ops import _need_cuda

NUSCENES_MAP_CLASSES = ("drivable_area", "ped_crossing", "walkway", "stop_line", "carpark_area", "road_divider",
                        "lane_divider", "road_block")  # configs/dataset/Nuscenes.yaml map_classes

# runner/map_visualizer.py:13-44; the legend lists its patches in this order
COLORS = {
    "drivable_area": (166, 206, 227), "drivable_area*": (144, 196, 255), "lane": (110, 110, 110),
    "road_segment": (90, 90, 90), "ped_crossing": (251, 154, 153), "walkway": (227, 26, 28),
    "stop_line": (253, 191, 111), "carpark_area": (255, 127, 0), "road_block": (178, 223, 138),
    "road_divider": (255, 200, 0), "lane_divider": (130, 130, 130),
    "car": (255, 158, 0), "truck": (255, 99, 71), "construction_vehicle": (233, 150, 70), "bus": (255, 127, 80),
    "trailer": (255, 140, 0), "barrier": (112, 128, 144), "motorcycle": (255, 61, 99), "bicycle": (220, 20, 60),
    "pedestrian": (0, 0, 230), "traffic_cone": (47, 79, 79),
    "nothing": (200, 200, 200),
}
# runner/map_visualizer.py:49-60: where static classes overlap, the one listed last is drawn
STATIC_PRIORITY = ("drivable_area", "drivable_area*", "road_block", "walkway", "stop_line", "carpark_area", "ped_crossing",
                   "divider", "road_divider", "lane_divider")

Legend = Callable[[FrozenSet[str], int], np.ndarray]
# show_legend's legends for the process: (names, size) -> uint8 (h, w, 3) numpy copy, and (names, size, slot shape,
# device) -> contiguous uint8 device tensor.  A caller's callable gets caches of its own, kept only while it is the last
# callable passed: a stable callable draws each legend once, and a fresh callable per call replaces them.
_LEGENDS: Dict = {}
_DEVICE_LEGENDS: Dict = {}
_CALLER: list = [None, {}, {}]  # [callable, host cache, device cache]
_TABLES: Dict = {}
_NONE = (1 << 64) - 1  # an error word of mdb_render_bev_map where the error never arises
_BICUBIC: Dict = {}


def show_legend(names: FrozenSet[str], long_edge_size: int) -> np.ndarray:
    """The reference's legend (runner/map_visualizer.py:80-103): a matplotlib "Legend plot" figure with one patch per
    class of `names` that has a colour, in COLORS order, 4 columns, saved as a tight PNG, resized (nearest) so its long
    edge is `long_edge_size`, alpha dropped -> uint8 (h, w, 3)."""
    try:
        import matplotlib.patches as mpatches
        import matplotlib.pyplot as plt
    except ImportError as e:
        raise ImportError("the default map legend is drawn with matplotlib, which is not installed; install it or pass "
                          "legend=") from e
    from PIL import Image
    fig = plt.figure("Legend plot")
    try:
        handles = [mpatches.Patch(color=[c / 255.0 for c in rgb], label=k) for k, rgb in COLORS.items() if k in names]
        fig.legend(handles=handles, loc="center", ncol=4)
        with io.BytesIO() as buf:
            fig.savefig(buf, format="png", bbox_inches="tight")
            im = Image.open(buf)
            w, h = im.size
            ratio = long_edge_size / max(w, h)
            if w > h:
                size = (long_edge_size, int(h * ratio))
            elif h > w:
                size = (int(w * ratio), long_edge_size)
            else:
                size = (long_edge_size, long_edge_size)
            return np.array(im.resize(size, resample=Image.NEAREST))[..., :3]
    finally:
        plt.close(fig)


def _legend(fn: Legend, names: FrozenSet[str], size: int, cache: Dict) -> np.ndarray:
    key = (names, size)
    if key not in cache:
        a = fn(names, size)
        a = a.cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a)
        if a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3:
            raise ValueError(f"a legend must be uint8 (h, w, 3), got {a.dtype} {a.shape}")
        cache[key] = np.array(a, order="C", copy=True)  # the caller may reuse the array it returned
    return cache[key]


def _device_legend(fn, names, size, s, device, host_cache, device_cache):
    """The legend as it lands in the image: (right, device tensor (s, lw, 3) or (lh, s, 3)), broadcast as numpy's slice
    assignment broadcasts it; ValueError where numpy refuses."""
    a = _legend(fn, names, size, host_cache)
    lh, lw = a.shape[:2]
    right = lh > lw
    slot = (s, lw, 3) if right else (lh, s, 3)
    key = (names, size, slot, str(device))
    if key not in device_cache:
        if any(n not in (1, m) for n, m in zip(a.shape, slot)):
            raise ValueError(f"the legend ({lh}, {lw}) does not fit {'beside' if right else 'below'} the {s} x {s} map "
                             f"(could not broadcast to {slot})")
        device_cache[key] = torch.from_numpy(a).expand(slot).contiguous().to(device, non_blocking=True)
    return right, device_cache[key]


def _tables(map_classes, object_classes, n_static, n_dynamic, device):
    key = (map_classes, object_classes, n_static, n_dynamic, str(device))
    if key not in _TABLES:
        prio = [STATIC_PRIORITY.index(c) if c in STATIC_PRIORITY else -1 for c in map_classes[:n_static]]
        cols = [(*COLORS[c], 1) if c in COLORS else (0, 0, 0, 0) for c in map_classes[:n_static]]
        cols += [(*COLORS[c], 1) if c in COLORS else (0, 0, 0, 0) for c in object_classes[:n_dynamic]]
        _TABLES[key] = (torch.tensor(prio + [0], dtype=torch.int32).to(device),
                        torch.tensor(cols, dtype=torch.uint8).to(device))
    return _TABLES[key]


def _bicubic(n_in, n_out, device):
    key = (n_in, n_out, str(device))
    if key not in _BICUBIC:
        _BICUBIC[key] = torch.from_numpy(fid.bicubic_table(n_in, n_out)).to(device)
    return _BICUBIC[key]


def resized_side(side: int, target_size) -> int:
    """The edge of a side x side map after visualize_map's resize: int(side * ratio), ratio = max(target_size / w,
    target_size / h), in Python floats as the reference computes it."""
    ratio = max(target_size / side, target_size / side)
    return int(side * ratio)


def visualize_maps(bev_maps: torch.Tensor, map_classes: Sequence[str] = NUSCENES_MAP_CLASSES,
                   object_classes: Sequence[str] = NUSCENES_OBJECT_CLASSES, target_size: int = 400,
                   legend: Optional[Legend] = None) -> List[torch.Tensor]:
    """The reference's `visualize_map(cfg, bev_maps[b], target_size)` for each map of a batch: bev_maps (B, C, H, W) on
    the device, fp32, uint8 or bool, every value 0 or 1, H == W; the first len(map_classes) channels are the static
    layers, the next len(object_classes) (those present) the dynamic ones, the rest are ignored.  -> B uint8 (h_b, w_b, 3)
    device tensors.

    legend(names, long_edge_size) -> uint8 (h, w, 3) draws the legend of a set of class names; by default `show_legend`
    (matplotlib), whose legends are drawn once per process and kept on the host and on the device.  The legends of a
    callable passed here are kept while it is the last one passed.

    Errors, all raised before anything is returned: ValueError for a value other than 0 or 1, a non-square map, no
    static and no dynamic layers, or a legend that does not fit the map.  As the reference, for the first map that fails
    and at the first pixel where it fails: ValueError when an active static class is missing from STATIC_PRIORITY,
    KeyError when the static class drawn there has no colour in COLORS; then KeyError for an object class without a
    colour, when the maps have dynamic layers.

    The call synchronises once: it reads the B class masks and error words back to the host to choose the legends."""
    if not isinstance(bev_maps, torch.Tensor):
        raise TypeError(f"bev_maps must be a torch.Tensor, got {type(bev_maps).__name__}")
    if bev_maps.dtype not in (torch.float32, torch.uint8, torch.bool) or bev_maps.dim() != 4 or min(bev_maps.shape) == 0:
        raise ValueError(f"expected fp32, uint8 or bool maps (B, C, H, W), got {bev_maps.dtype} {tuple(bev_maps.shape)}")
    _need_cuda(bev_maps)
    B, C, H, W = bev_maps.shape
    map_classes, object_classes = tuple(map_classes or ()), tuple(object_classes or ())
    n_static = min(len(map_classes), C)
    n_dynamic = max(0, min(len(object_classes), C - len(map_classes)))
    if n_static + n_dynamic == 0:
        raise ValueError("the maps have neither static nor dynamic layers for these classes")
    if n_static + n_dynamic > 64:
        raise ValueError(f"at most 64 static and dynamic classes, got {n_static + n_dynamic}")
    if H != W:
        raise ValueError(f"only square maps are supported, got {H} x {W}")
    s = resized_side(W, target_size)
    if s <= 0:
        raise ValueError(f"target_size {target_size} resizes the {H} x {W} maps to nothing")
    dev = bev_maps.device
    prio, cols = _tables(map_classes, object_classes, n_static, n_dynamic, dev)
    rendered, info = visualize_ops.render_bev_map(bev_maps, n_static, n_dynamic, prio, cols)
    if s != W:
        table = _bicubic(W, s, dev)
        rendered = image_ops.resample_u8(rendered, (s, s), table, table)
    info = info.cpu().numpy().view(np.uint64)  # the call's one synchronisation

    names = []
    for b, (used, status, no_rank, no_colour) in enumerate(info.tolist()):
        if status:
            raise ValueError(f"map {b} holds values other than 0 and 1")
        # render_static fails at the first pixel where get_color_by_priority does: the rank lookup before the colour's
        if no_rank != _NONE and no_rank >> 6 <= no_colour >> 6:
            raise ValueError(f"{map_classes[no_rank & 63]!r} is not in list")  # STATIC_PRIORITY.index
        if no_colour != _NONE:
            raise KeyError(map_classes[no_colour & 63])
        if n_dynamic:
            for c in object_classes:
                COLORS[c]  # KeyError, as render_dynamic raises for an object class without a colour
        names.append(frozenset([map_classes[i] for i in range(n_static) if used >> i & 1] +
                               [object_classes[j] for j in range(n_dynamic) if used >> (n_static + j) & 1]))
    if legend is None:
        caches = (_LEGENDS, _DEVICE_LEGENDS)
    else:
        if _CALLER[0] is not legend:
            _CALLER[:] = [legend, {}, {}]
        caches = tuple(_CALLER[1:])
    placed = [_device_legend(legend or show_legend, n, target_size, s, dev, *caches) for n in names]

    desc, shapes, offset = [], [], 0
    for right, leg in placed:
        shape = (s, s + leg.shape[1], 3) if right else (s + leg.shape[0], s, 3)
        desc.append([leg.data_ptr(), leg.shape[0], leg.shape[1], int(right), offset])
        shapes.append(shape)
        offset += shape[0] * shape[1] * 3
    out = torch.empty(offset, dtype=torch.uint8, device=dev)
    visualize_ops.place_map_u8(rendered, torch.tensor(desc, dtype=torch.int64).to(dev, non_blocking=True),
                               max(h * w for h, w, _ in shapes), out)
    images, offset = [], 0
    for shape in shapes:
        n = shape[0] * shape[1] * 3
        images.append(out[offset:offset + n].view(shape))
        offset += n
    return images


def camera_views_u8(pixel_values: torch.Tensor) -> torch.Tensor:
    """The given views as the reference saves them, to_pil_image(img_m11_to_01(x)): fp32 (S, V, 3, H, W) in [-1, 1] on
    the device -> uint8 (S, V, H, W, 3)."""
    if not isinstance(pixel_values, torch.Tensor):
        raise TypeError(f"pixel_values must be a torch.Tensor, got {type(pixel_values).__name__}")
    if pixel_values.dtype != torch.float32 or pixel_values.dim() != 5 or pixel_values.shape[2] != 3 or \
            min(pixel_values.shape) == 0:
        raise ValueError(f"expected fp32 (S, V, 3, H, W), got {pixel_values.dtype} {tuple(pixel_values.shape)}")
    S, V, _, H, W = pixel_values.shape
    return visualize_ops.m11_to_u8(pixel_values.reshape(S * V, 3, H, W)).view(S, V, H, W, 3)


def concat_views(views: torch.Tensor, oneline: bool = False) -> torch.Tensor:
    """The reference's `concat_6_views` for each scene: views (S, V, H, W, C) on the device, uint8 with C = 3 (RGB) or 4
    (RGBA, as show_box_on_views(..., transparent_bg=True) returns), or fp32 [0, 1] RGB as decode_latents returns them
    (rounded as numpy_to_pil does).  -> uint8 (S, 2H, max(3, V - 3) W, C): views 0-2 on the first row, the rest on the
    second, black (alpha 255) where a row is shorter; with oneline (S, H, V W, C).  ValueError for fewer than 5 views
    (2 with oneline), where the reference fails."""
    if not isinstance(views, torch.Tensor):
        raise TypeError(f"views must be a torch.Tensor, got {type(views).__name__}")
    ok = views.dim() == 5 and (views.dtype == torch.uint8 and views.shape[-1] in (3, 4) or
                               views.dtype == torch.float32 and views.shape[-1] == 3)
    if not ok or min(views.shape) == 0:
        raise ValueError(f"expected uint8 (S, V, H, W, 3 | 4) or fp32 (S, V, H, W, 3) views, got {views.dtype} "
                         f"{tuple(views.shape)}")
    S, V, H, W, C = views.shape
    if V < (2 if oneline else 5):
        raise ValueError(f"concat_6_views needs at least {2 if oneline else 5} views{' with oneline' if oneline else ''}, "
                         f"got {V}")
    _need_cuda(views)
    if views.dtype == torch.float32:  # numpy_to_pil's rounding: the resample with no size change is a copy
        views = image_ops.resample_u8(views.reshape(S * V, H, W, 3), (H, W), None, None).view(S, V, H, W, 3)
    return visualize_ops.concat_views_u8(views, oneline)


def _batch(name, x, n):
    if x is None:
        return None
    if len(x) != n:
        raise ValueError(f"{name} holds {len(x)} images for {n} maps")
    return x


def save_run_images(log_root, first_index: int, maps: Sequence[torch.Tensor], ori=None, ori_box=None, gen=(),
                    gen_box=()) -> List[str]:
    """Write one batch's images as tools/test.py does, sample n = first_index + b: `{n}_map.png` from maps[b],
    `{n}_ori.png` from ori[b], `{n}_gen{t}.png` from gen[t][b], `{n}_ori_box.png` from ori_box[b] and
    `{n}_gen{t}_box.png` from gen_box[t][b].  maps: the B images of visualize_maps; ori, ori_box: (B, h, w, 3 | 4) mosaics
    or None; gen, gen_box: one (B, h, w, 3 | 4) mosaic batch per generation.  Each image is copied to the host once and
    written by Pillow (Image.fromarray(a).save(path)).  Returns the paths written, in that order."""
    from PIL import Image
    B = len(maps)
    ori, ori_box = _batch("ori", ori, B), _batch("ori_box", ori_box, B)
    gen = [_batch(f"gen[{t}]", g, B) for t, g in enumerate(gen or ())]
    gen_box = [_batch(f"gen_box[{t}]", g, B) for t, g in enumerate(gen_box or ())]
    for x in [*maps, *(ori if ori is not None else []), *(ori_box if ori_box is not None else []), *gen, *gen_box]:
        if x.dtype != torch.uint8 or x.dim() not in (3, 4) or x.shape[-1] not in (3, 4):
            raise ValueError(f"images must be uint8 (h, w, 3 | 4), got {x.dtype} {tuple(x.shape)}")
    paths = []

    def save(img, name):
        paths.append(os.path.join(log_root, name))
        Image.fromarray(img.cpu().numpy()).save(paths[-1])

    for b in range(B):
        n = first_index + b
        save(maps[b], f"{n}_map.png")
        if ori is not None:
            save(ori[b], f"{n}_ori.png")
        for t, g in enumerate(gen):
            save(g[b], f"{n}_gen{t}.png")
        if ori_box is not None:
            save(ori_box[b], f"{n}_ori_box.png")
        for t, g in enumerate(gen_box):
            save(g[b], f"{n}_gen{t}_box.png")
    return paths
