"""TEST INFRASTRUCTURE ONLY — golden images for the test-run images: the reference's own `visualize_map`
(magicdrive/runner/map_visualizer.py:143-211) and `concat_6_views` / `img_m11_to_01` (runner/img_utils.py) with
torchvision's `to_pil_image`, as `run_one_batch` (magicdrive/misc/test_utils.py:258-321) calls them.

The definitions are taken from the two files' source text with `ast` and executed unmodified, with numpy, torch and Pillow
as the reference imports them.  matplotlib is not installed here, so `plt` and `mpatches` are stubs that fail when used,
and `show_legend`, the one function that draws with them, is replaced by `fake_legend`, a deterministic function of the
sorted class names and the size.  Sets whose size is a multiple of 3 give a legend taller than wide, so both of
visualize_map's placements are covered.  The fixture records the name sets the reference passed to it.

Inputs: the six demo samples' `gt_masks_bev` (8 x 200 x 200) at target_size 400 and 800, and the first at 150 (a
downsizing); seeded 18- and 26-channel maps (8 static, 10 dynamic, 8 aux) with overlapping static classes, the 26-channel
one with empty dynamic layers; an all-zero 18-channel map; a 400 x 400 map at 400 (no resize).  Maps are stored as
xz-compressed np.packbits, outputs as sha256 and, for a few, xz-compressed bytes.  Mosaics: concat_6_views of seeded RGB
and RGBA views with 6 and 5 views, in both layouts.  Camera views: to_pil_image(img_m11_to_01(x)) of every value the demo samples' `img`
holds, seeded values in [-1, 1] and edge values.

    python -m oracle.make_golden_map_visualizer      # build container only (needs /root/reference)
"""
import ast
import glob
import hashlib
import io
import lzma
import os
import sys
from types import SimpleNamespace
from typing import Tuple, Union

import numpy as np
import torch

REF = os.environ.get("MAGICDRIVE_REFERENCE_SRC", "/root/reference")
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "map_visualizer.pt")
MAP_NEEDED = ["COLORS", "STATIC_PRIORITY", "get_colors", "get_color_by_priority", "rgb_to_01range", "render_static",
              "render_dynamic", "classes_to_np", "visualize_map"]
IMG_NEEDED = ["concat_6_views", "img_m11_to_01", "img_concat_h", "img_concat_v"]
MAP_CLASSES = ["drivable_area", "ped_crossing", "walkway", "stop_line", "carpark_area", "road_divider", "lane_divider",
               "road_block"]  # configs/dataset/Nuscenes.yaml
OBJECT_CLASSES = ["car", "truck", "construction_vehicle", "bus", "trailer", "barrier", "motorcycle", "bicycle",
                  "pedestrian", "traffic_cone"]
SEED = 20261018
FULL = {"demo0@400", "seeded18@400", "zeros18@400"}  # cases stored in full


def fake_legend(names, size: int) -> np.ndarray:
    """A deterministic stand-in for show_legend: uint8 (size, k, 3) when len(names) is a multiple of 3, else (k, size, 3),
    k = size // 8 + len(names), filled from a generator seeded by the sorted names and the size (with few levels, so
    that the fixture compresses)."""
    digest = hashlib.sha256(("|".join(sorted(names)) + f"#{size}").encode()).digest()
    rng = np.random.default_rng(int.from_bytes(digest[:8], "little"))
    k = size // 8 + len(names)
    shape = (size, k, 3) if len(names) % 3 == 0 else (k, size, 3)
    return (rng.integers(0, 8, shape) * 32 + rng.integers(0, 2, shape)).astype(np.uint8)


def _stub(name):
    def fail(*a, **k):
        raise RuntimeError(f"{name} is a stub: matplotlib is not installed")
    return SimpleNamespace(__getattr__=fail, figure=fail, close=fail, Patch=fail)


def reference_namespace(legend_calls):
    from PIL import Image

    def show_legend(semantic_in_use, long_edge_size=200, ncol=4):
        legend_calls.append((sorted(str(n) for n in semantic_in_use), long_edge_size))
        return fake_legend(semantic_in_use, long_edge_size)

    ns = {"np": np, "torch": torch, "io": io, "Image": Image, "Tuple": Tuple, "Union": Union, "plt": _stub("plt"),
          "mpatches": _stub("mpatches")}
    for rel, needed in (("magicdrive/runner/map_visualizer.py", MAP_NEEDED), ("magicdrive/runner/img_utils.py", IMG_NEEDED)):
        src = open(os.path.join(REF, rel)).read()
        for node in ast.parse(src).body:
            name = node.targets[0].id if isinstance(node, ast.Assign) and isinstance(node.targets[0], ast.Name) else \
                getattr(node, "name", None)
            if name in needed:
                exec(compile(ast.Module([node], []), rel, "exec"), ns)
        assert all(n in ns for n in needed), rel
    ns["show_legend"] = show_legend
    return ns


def seeded_maps(seed=SEED):
    """The seeded maps: name -> (int64 (C, H, W), target_size)."""
    rng = np.random.default_rng(seed)

    def blobs(c, h, w, density):
        # overlapping rectangles, so that static classes overlap as road layers do
        m = np.zeros((c, h, w), np.int64)
        for i in range(c):
            while m[i].mean() < density[i]:
                y, x = rng.integers(0, h), rng.integers(0, w)
                dy, dx = rng.integers(2, h // 4), rng.integers(2, w // 4)
                m[i, y:y + dy, x:x + dx] = 1
        return m

    static = [0.35, 0.05, 0.15, 0.05, 0.05, 0.04, 0.04, 0.25]
    m18 = np.concatenate([blobs(8, 200, 200, static), blobs(10, 200, 200, [0.01] * 10)])
    m26 = np.concatenate([blobs(8, 200, 200, static), np.zeros((10, 200, 200), np.int64), blobs(8, 200, 200, [0.1] * 8)])
    m400 = np.concatenate([blobs(8, 400, 400, static), blobs(10, 400, 400, [0.005] * 10)])
    return {"seeded18@400": (m18, 400), "seeded26@400": (m26, 400), "zeros18@400": (np.zeros((18, 200, 200), np.int64), 400),
            "identity400@400": (m400, 400)}


def mosaic_views(V, C, seed=SEED, H=24, W=40):
    return np.random.default_rng([seed, V, C]).integers(0, 256, (V, H, W, C), dtype=np.uint8)


def m11_values(seed=SEED):
    """fp32 (3, 40, 40): every value of the demo samples' img first (passed in by main), then edges and seeded values."""
    rng = np.random.default_rng(seed)
    edges = np.array([-1, -0.0, 0.0, 1, np.nextafter(np.float32(-1), 1), np.nextafter(np.float32(1), 0), 0.5, -0.5,
                      1 / 255, -1 / 255, 2 / 255 - 1, 1 - 2 / 255], np.float32)
    return edges, rng.uniform(-1, 1, 3 * 40 * 40).astype(np.float32)


def _xz(a):
    b = lzma.compress(np.ascontiguousarray(a).tobytes(), preset=9 | lzma.PRESET_EXTREME)
    return torch.from_numpy(np.frombuffer(b, np.uint8).copy())


def _unxz(t, dtype, shape):
    return np.frombuffer(lzma.decompress(t.numpy().tobytes()), dtype).reshape(shape)


def sha(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def main():
    from PIL import Image
    from torchvision.transforms.functional import to_pil_image
    calls = []
    ns = reference_namespace(calls)
    cfg = SimpleNamespace(dataset=SimpleNamespace(map_classes=MAP_CLASSES, object_classes=OBJECT_CLASSES))
    files = sorted(glob.glob(os.path.join(REF, "demo", "data", "*.pth")))
    samples = [torch.load(f, weights_only=False) for f in files]
    inputs = {}
    for i, s in enumerate(samples):
        for t in (400, 800):
            inputs[f"demo{i}@{t}"] = (s["gt_masks_bev"], t)
    inputs["demo0@150"] = (samples[0]["gt_masks_bev"], 150)
    inputs.update(seeded_maps())

    bits, maps = {}, []
    for name, (m, t) in inputs.items():
        key = name.split("@")[0]
        if key not in bits:
            bits[key] = dict(shape=m.shape, bits_xz=_xz(np.packbits(m.astype(bool))))
        del calls[:]
        img = ns["visualize_map"](cfg, torch.from_numpy(m), target_size=t)
        assert img.dtype == np.uint8 and len(calls) == 1
        names, size = calls[0]
        lh, lw, _ = fake_legend(names, size).shape
        maps.append(dict(name=name, map_key=key, target_size=t,
                         legend_names=names, legend_size=size, right=lh > lw, out_shape=img.shape, sha256=sha(img),
                         **({"out_xz": _xz(img)} if name in FULL else {})))
        print(name, m.shape, t, "->", img.shape, "legend", names, "right" if lh > lw else "below")

    mosaics = []
    for V in (6, 5):
        for C in (3, 4):
            views = mosaic_views(V, C)
            for oneline in (False, True):
                pil = [Image.fromarray(v) for v in views]
                out = np.asarray(ns["concat_6_views"](pil, oneline=oneline))
                mosaics.append(dict(V=V, C=C, oneline=oneline, out_shape=out.shape, out_xz=_xz(out)))

    demo_values = np.unique(np.concatenate([s["img"].numpy().ravel() for s in samples]))
    edges, rand = m11_values()
    vals = np.concatenate([demo_values, edges, rand])[:3 * 40 * 40].reshape(3, 40, 40)
    ori = np.asarray(to_pil_image(ns["img_m11_to_01"](torch.from_numpy(vals))))
    assert ori.shape == (40, 40, 3)
    torch.save(dict(seed=SEED, map_classes=MAP_CLASSES, object_classes=OBJECT_CLASSES, map_bits=bits, maps=maps,
                    mosaics=mosaics,
                    m11=dict(x=torch.from_numpy(vals.copy()), n_demo_values=len(demo_values), out=torch.from_numpy(ori.copy()))),
               OUT)
    print(OUT, os.path.getsize(OUT) // 1024, "KiB")


def load(path):
    """The fixture with each map case's `map` (uint8 (C, H, W)) and, where stored, `out` decoded, and each mosaic's
    `views` and `out`."""
    fx = torch.load(path, weights_only=False)
    arrays = {k: np.unpackbits(_unxz(v["bits_xz"], np.uint8, (-1,)), count=int(np.prod(v["shape"]))).reshape(v["shape"])
              for k, v in fx.pop("map_bits").items()}
    for c in fx["maps"]:
        c["map"] = arrays[c["map_key"]]
        if "out_xz" in c:
            c["out"] = _unxz(c.pop("out_xz"), np.uint8, c["out_shape"])
    for c in fx["mosaics"]:
        c["views"] = mosaic_views(c["V"], c["C"], fx["seed"])
        c["out"] = _unxz(c.pop("out_xz"), np.uint8, c["out_shape"])
    return fx


if __name__ == "__main__":
    sys.exit(main())
