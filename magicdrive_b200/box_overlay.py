"""3D-box overlays on the generated or given camera views, as the reference writes them with `show_box` on
(demo/helper.py:197-307 `draw_box_on_imgs`; magicdrive/misc/test_utils.py `run_one_batch`): every 3D box of a sample drawn
on each view with OpenCV's anti-aliased 1-pixel lines, equal byte for byte to the reference's images, and the box-only
RGBA layer of `transparent_bg=True`.

Two C-ABI kernels do the work (csrc/capi_box_overlay.cu): mdb_project_boxes projects and orders the boxes of a batch,
mdb_draw_box_edges_aa draws their edges.  The few host steps are the reference's own operations on the sample's small
arrays, so that their roundings are the reference's: the per-view 4 x 4 transforms (numpy float32) and the sine and
cosine of each yaw (torch on the CPU).  There is no CPU fallback; oracle/box_overlay.py restates the kernels for tests.
"""
from typing import Dict, List, Sequence

import numpy as np
import torch

from . import _lib, ops
from ._lib import check
from .ops import _need_cuda, _ptr, _stream

NUSCENES_OBJECT_CLASSES = ("car", "truck", "construction_vehicle", "bus", "trailer", "barrier", "motorcycle", "bicycle",
                           "pedestrian", "traffic_cone")
# demo/helper.py:25-36, equal to mmdet3d's; the reference's two BGR swaps cancel, so these are drawn as RGB
OBJECT_PALETTE = {
    "car": (255, 158, 0), "truck": (255, 99, 71), "construction_vehicle": (233, 150, 70), "bus": (255, 69, 0),
    "trailer": (255, 140, 0), "barrier": (112, 128, 144), "motorcycle": (255, 61, 99), "bicycle": (220, 20, 60),
    "pedestrian": (0, 0, 230), "traffic_cone": (47, 79, 79),
}


def _host(x, dtype):
    return (torch.from_numpy(x) if isinstance(x, np.ndarray) else torch.as_tensor(x)).to(dtype)


def view_transforms(example: Dict, n_views: int) -> np.ndarray:
    """float32 (n_views, 4, 4): img_aug_matrix[v] @ lidar2image[v] (numpy float32, show_box_on_views), lidar2image being
    torch.bmm(camera_intrinsics, lidar2camera) when the example has none (precompute_cam_ext, demo/helper.py:495-505)."""
    if example.get("lidar2image") is not None:
        l2i = _host(example["lidar2image"], torch.float32)
    else:
        l2i = torch.bmm(_host(example["camera_intrinsics"], torch.float32), _host(example["lidar2camera"], torch.float32))
    l2i = l2i.numpy()
    if l2i.shape != (n_views, 4, 4):
        raise ValueError(f"lidar2image is {tuple(l2i.shape)}, expected ({n_views}, 4, 4)")
    if example.get("img_aug_matrix") is None:
        return l2i
    aug = _host(example["img_aug_matrix"], torch.float32).numpy()
    if aug.shape != (n_views, 4, 4):
        raise ValueError(f"img_aug_matrix is {tuple(aug.shape)}, expected ({n_views}, 4, 4)")
    return np.stack([aug[v] @ l2i[v] for v in range(n_views)])


def _stage(examples: List[Dict], n_views: int, classes: Sequence[str]) -> Dict:
    """Check a batch's samples and gather them on the host for mdb_project_boxes."""
    if not classes:
        raise ValueError("classes is empty")
    boxes, labels, sincos, trans = [], [], [], []
    for s, e in enumerate(examples):
        b = _host(e["gt_bboxes_3d"], torch.float32)
        lab = _host(e["gt_labels_3d"], torch.int64).reshape(-1)
        if b.numel() == 0:
            b = b.reshape(0, 9)
        if b.dim() != 2 or b.shape[1] not in (7, 9) or b.shape[0] != lab.shape[0]:
            raise ValueError(f"sample {s}: gt_bboxes_3d {tuple(b.shape)} with {lab.shape[0]} labels; expected (n, 7 | 9)")
        if lab.numel() and (int(lab.min()) < 0 or int(lab.max()) >= len(classes)):
            raise ValueError(f"sample {s}: labels must lie in [0, {len(classes)}), got {lab.tolist()}")
        for name in {classes[i] for i in lab.tolist()}:
            OBJECT_PALETTE[name]  # KeyError for a class without a colour, as the reference raises
        boxes.append(b[:, :7])
        labels.append(lab)
        # LiDARInstance3DBoxes.corners: torch.sin / torch.cos of the yaw column, on the CPU like the reference
        sincos.append(torch.stack([torch.sin(b[:, 6]), torch.cos(b[:, 6])], 1))
        trans.append(view_transforms(e, n_views))
    n = [len(lab) for lab in labels]
    cap = max([1] + n)
    if cap > 4096:
        raise ValueError(f"at most 4096 boxes per sample, got {cap}")
    return {"boxes": torch.cat(boxes) if sum(n) else torch.zeros(1, 7),
            "sincos": torch.cat(sincos) if sum(n) else torch.zeros(1, 2),
            "labels": torch.cat(labels) if sum(n) else torch.zeros(1, dtype=torch.int64),
            "offsets": torch.tensor([0] + np.cumsum(n).tolist(), dtype=torch.int32),
            "transforms": torch.from_numpy(np.stack(trans)), "capacity": cap,
            "palette": torch.tensor([OBJECT_PALETTE.get(c, (0, 0, 0)) for c in classes], dtype=torch.uint8)}


def _project(st: Dict, n_views: int, device) -> Dict:
    dev = torch.device(device)
    if dev.type != "cuda":
        raise _lib.MdbError("project_boxes runs on a CUDA device; there is no CPU fallback")
    S, cap = st["offsets"].numel() - 1, st["capacity"]
    d = lambda t: t.contiguous().to(dev, non_blocking=True)
    bx, sc, lb, off, tr = d(st["boxes"]), d(st["sincos"]), d(st["labels"]), d(st["offsets"]), d(st["transforms"])
    res = {"endpoints": torch.empty((S, n_views, cap, 8, 2), dtype=torch.int32, device=dev),
           "colors": torch.empty((S, n_views, cap), dtype=torch.int32, device=dev),
           "counts": torch.empty((S, n_views), dtype=torch.int32, device=dev),
           "status": torch.empty((S, n_views), dtype=torch.int32, device=dev)}
    check(_lib.lib().mdb_project_boxes(bx.data_ptr(), 7, sc.data_ptr(), lb.data_ptr(), off.data_ptr(), S, tr.data_ptr(),
                                       n_views, cap, _ptr(res["endpoints"]), _ptr(res["colors"]), _ptr(res["counts"]),
                                       _ptr(res["status"]), _stream()), "mdb_project_boxes")
    ops._launches += 1
    return res


def project_boxes(examples: List[Dict], n_views: int, device, classes: Sequence[str] = NUSCENES_OBJECT_CLASSES) -> Dict:
    """mdb_project_boxes over a batch of samples -> dict of device tensors: endpoints int32 (S, V, capacity, 8, 2) and
    colors int32 (S, V, capacity) (the label) of the boxes drawn in each view, far to near; counts int32 (S, V), how many
    are drawn; status int32 (S, V), 1 where an endpoint falls outside int32."""
    return _project(_stage(examples, n_views, classes), n_views, device)


def show_box_on_views(images: torch.Tensor, examples: List[Dict], classes: Sequence[str] = NUSCENES_OBJECT_CLASSES, *,
                      transparent_bg: bool = False, out: torch.Tensor = None) -> torch.Tensor:
    """The reference's `draw_box_on_imgs` for a batch: images (S, V, H, W, 3) on the device, uint8 or fp32 in [0, 1] as
    `decode_latents` returns them (rounded as numpy_to_pil does); examples: S sample dicts with gt_bboxes_3d (n, 7 | 9),
    gt_labels_3d (n,), lidar2image (V, 4, 4) or camera_intrinsics and lidar2camera, and optionally img_aug_matrix.
    Labels index `classes`.  -> uint8 (S, V, H, W, 3) with the boxes drawn, or with transparent_bg the boxes alone on
    black as RGBA (S, V, H, W, 4).  out may be a uint8 `images` (drawn in place).  Raises ValueError, as cv2 does, when a
    corner projects outside the int32 range; out is then left untouched."""
    if not isinstance(images, torch.Tensor):
        raise TypeError(f"images must be a torch.Tensor, got {type(images).__name__}")
    if images.dtype not in (torch.uint8, torch.float32):
        raise TypeError(f"show_box_on_views takes uint8 or float32 images, got {images.dtype}")
    if images.dim() != 5 or images.shape[-1] != 3 or min(images.shape) == 0:
        raise ValueError(f"expected images (S, V, H, W, 3), got {tuple(images.shape)}")
    S, V, H, W = images.shape[:4]
    if len(examples) != S:
        raise ValueError(f"{len(examples)} examples for {S} scenes")
    shape = (S, V, H, W, 4 if transparent_bg else 3)
    if out is not None:
        if out.dtype != torch.uint8:
            raise TypeError(f"out must be uint8, got {out.dtype}")
        if tuple(out.shape) != shape or not out.is_contiguous() or out.device != images.device:
            raise ValueError(f"out must be a contiguous {shape} tensor on {images.device}")
    st = _stage(examples, V, classes)
    _need_cuda(images, out)
    images = images.contiguous()
    proj = _project(st, V, images.device)
    if out is None:
        out = torch.empty(shape, dtype=torch.uint8, device=images.device)
    pal = st["palette"].to(images.device)
    check(_lib.lib().mdb_draw_box_edges_aa(_ptr(images), int(images.dtype == torch.float32), S * V, H, W,
                                           _ptr(proj["endpoints"]), _ptr(proj["colors"]), _ptr(proj["counts"]),
                                           _ptr(proj["status"]), proj["colors"].shape[-1], _ptr(pal), len(classes),
                                           int(transparent_bg), _ptr(out), _stream()), "mdb_draw_box_edges_aa")
    ops._launches += 1
    bad = torch.nonzero(proj["status"]).tolist()
    if bad:
        raise ValueError(f"a box corner projects outside the int32 range in (scene, view) {bad}; cv2.line refuses it")
    return out
