"""TEST INFRASTRUCTURE ONLY — golden images for the 3D-box overlays: the reference's own `draw_box_on_imgs` /
`show_box_on_views` / `visualize_camera` (demo/helper.py:197-307, the mmdet3d-free copy of runner/box_visualizer.py) run
on the six nuScenes samples it ships (demo/data/*.pth), over seeded random uint8 views at 224 x 400, with and without
`transparent_bg`.

The needed definitions are taken from demo/helper.py's source text with `ast` and executed unmodified, with cv2 and Pillow
as the reference imports them.  Two things in the namespace are not the reference's:
* `OmegaConf.to_container` is a stand-in that returns the class list unchanged (omegaconf is not installed here, and
  `cfg.dataset.object_classes` is given as a plain list);
* `np.int = int`: the reference's `astype(np.int)` predates numpy 2, which removed the alias.  It was the builtin int,
  so this restores the reference's behaviour (truncation to int64).

The fixture stores the seed and, per sample, only the pixels the overlay touched: `at` (view, y, x) where the drawn view
differs from its background or the transparent layer is opaque, and there `drawn` (RGB) and `layer` (RGBA).  Every
other pixel equals the background in the drawn views and is 0 in the layer.  To keep the file small, the three arrays
are stored xz-compressed: `at` as the gaps between successive flat indices (view * 224 * 400 + y * 400 + x, uint32),
`drawn` and `layer` as their uint8 bytes.  `load()` decodes it.

    python -m oracle.make_golden_box_overlay      # build container only (needs /root/reference and cv2)
"""
import ast
import copy
import glob
import lzma
import os
import sys
from types import SimpleNamespace
from typing import List, Optional, Tuple

import numpy as np
import torch

REF = os.environ.get("MAGICDRIVE_REFERENCE_SRC", "/root/reference")
OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "box_overlay.pt")
NEEDED = ["OBJECT_PALETTE", "rotation_3d_in_axis", "LiDARInstance3DBoxes", "visualize_camera", "show_box_on_views",
          "draw_box_on_imgs", "box_center_shift", "precompute_cam_ext"]
CLASSES = ["car", "truck", "construction_vehicle", "bus", "trailer", "barrier", "motorcycle", "bicycle", "pedestrian",
           "traffic_cone"]  # configs/dataset/Nuscenes.yaml object_classes
SEED = 20261017
H, W = 224, 400


def reference_namespace():
    import cv2
    from PIL import Image
    np.int = int  # numpy 2 removed this alias of the builtin int; the reference's astype(np.int) needs it
    src = open(os.path.join(REF, "demo", "helper.py")).read()
    ns = {"np": np, "torch": torch, "copy": copy, "cv2": cv2, "Image": Image, "List": List, "Optional": Optional,
          "Tuple": Tuple, "OmegaConf": SimpleNamespace(to_container=lambda x, resolve=True: list(x))}
    for node in ast.parse(src).body:
        name = node.targets[0].id if isinstance(node, ast.Assign) and isinstance(node.targets[0], ast.Name) else \
            getattr(node, "name", None)
        if name in NEEDED:
            exec(compile(ast.Module([node], []), "demo/helper.py", "exec"), ns)
    assert all(n in ns for n in NEEDED)
    return ns


def main():
    from PIL import Image
    ns = reference_namespace()
    cfg = SimpleNamespace(dataset=SimpleNamespace(object_classes=CLASSES))
    files = sorted(glob.glob(os.path.join(REF, "demo", "data", "*.pth")))
    cases = []
    for f, bg in zip(files, backgrounds(len(files))):
        ex = ns["precompute_cam_ext"](torch.load(f, weights_only=False))  # lidar2image = K @ lidar2camera
        drawn = np.stack([np.asarray(im) for im in ns["draw_box_on_imgs"](cfg, ex, [Image.fromarray(v) for v in bg])])
        layer = np.stack([np.asarray(im) for im in ns["draw_box_on_imgs"](cfg, ex, [Image.fromarray(v) for v in bg],
                                                                          transparent_bg=True)])
        assert drawn.shape == bg.shape and layer.shape == bg.shape[:3] + (4,)
        at = np.nonzero(np.any(drawn != bg, axis=-1) | (layer[..., 3] > 0))
        cases.append(dict(
            name=os.path.basename(f), gt_bboxes_3d=ex["gt_bboxes_3d"].clone(), gt_labels_3d=ex["gt_labels_3d"].clone(),
            camera_intrinsics=ex["camera_intrinsics"].clone(), lidar2camera=ex["lidar2camera"].clone(),
            img_aug_matrix=ex["img_aug_matrix"].clone(),
            **_encode(at, drawn[at], layer[at])))
        print(cases[-1]["name"], "boxes", tuple(ex["gt_bboxes_3d"].shape), "pixels", len(at[0]))
    torch.save(dict(seed=SEED, size=(H, W), classes=CLASSES, cases=cases), OUT)
    print(OUT, os.path.getsize(OUT) // 1024, "KiB")


def _xz(a):  # a uint8 tensor: torch.save pickles raw bytes objects at up to twice their size
    b = lzma.compress(np.ascontiguousarray(a).tobytes(), preset=9 | lzma.PRESET_EXTREME)
    return torch.from_numpy(np.frombuffer(b, np.uint8).copy())


def _unxz(t):
    return lzma.decompress(t.numpy().tobytes())


def _encode(at, drawn, layer):
    flat = (at[0].astype(np.int64) * H + at[1]) * W + at[2]  # ascending: np.nonzero's order
    return dict(n=len(flat), at_gaps_xz=_xz(np.diff(flat, prepend=0).astype(np.uint32)), drawn_xz=_xz(drawn),
                layer_xz=_xz(layer))


def load(path):
    """The fixture with each case's `at` (int64 (n, 3): view, y, x), `drawn` (uint8 (n, 3)) and `layer` (uint8 (n, 4))
    decoded."""
    fx = torch.load(path, weights_only=False)
    for c in fx["cases"]:
        n = c["n"]
        flat = np.cumsum(np.frombuffer(_unxz(c.pop("at_gaps_xz")), np.uint32).astype(np.int64))
        c["at"] = np.stack([flat // (H * W), flat // W % H, flat % W], 1)
        c["drawn"] = np.frombuffer(_unxz(c.pop("drawn_xz")), np.uint8).reshape(n, 3)
        c["layer"] = np.frombuffer(_unxz(c.pop("layer_xz")), np.uint8).reshape(n, 4)
    return fx


def backgrounds(n_samples, seed=SEED):
    """The seeded views the fixture's images were drawn on: uint8 (n_samples, 6, 224, 400, 3)."""
    return np.random.default_rng(seed).integers(0, 256, (n_samples, 6, H, W, 3), dtype=np.uint8)


if __name__ == "__main__":
    sys.exit(main())
