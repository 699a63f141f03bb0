"""Input preparation on the device (the step before the denoising path): the parts of the reference's `collate_fn`
(magicdrive/dataset/utils.py:243-352; one-sample form demo/helper.py:506-590) that feed the pipeline — `camera_param`,
`bev_map_with_aux`, `kwargs["bboxes_3d_data"]` — computed by two small CUDA kernels (mdb_prepare_boxes, mdb_camera_param)
instead of per-sample numpy / Python loops.  Tokenising and CLIP-encoding the captions stays outside (SURVEY.md section 2.1).

`examples` are the dicts the reference's dataset / demo fixtures hold: gt_bboxes_3d (n, 9), gt_labels_3d (n,), camera_intrinsics,
lidar2camera, img_aug_matrix (6, 4, 4) each, gt_masks_bev (8, 200, 200).
"""
from typing import Dict, List, Optional

import numpy as np
import torch

from . import _lib
from ._lib import check

F32 = torch.float32


def _t(x, dtype):
    return (torch.from_numpy(x) if isinstance(x, np.ndarray) else x).to(dtype)


def collate_on_device(examples: List[Dict], device, max_len: Optional[int] = None, stream=None,
                      capacity: Optional[int] = None) -> Dict:
    """-> dict(camera_param (B, V, 3, 7) fp32, bev_map_with_aux (B, C, H, W) fp32, kwargs={"bboxes_3d_data": dict | None}) on
    `device`, the same values `collate_fn(..., bbox_mode="all-xyz", bbox_view_shared=False)` produces.
    max_len=None pads the boxes to the longest visible list of the batch like the reference (needs one device -> host read
    of the per-view counts); an int fixes the capacity (`bbox_max_length` semantics) and stays asynchronous.
    capacity=N (instead of max_len) is the reference's padding without that read: the tensors have N slots per view, the
    first `count` of them are what max_len=None returns, and `count`, an int32 device scalar holding the batch's longest
    visible list, comes back as bboxes_3d_data["count"] for a BEVControlNetDenoiser(box_capacity=N) to attend by.  Lists
    longer than N are cut at N (`counts` holds the uncut per-view numbers)."""
    if capacity is not None and max_len is not None:
        raise ValueError("pass max_len or capacity, not both")
    dev = torch.device(device)
    if dev.type != "cuda":
        raise _lib.MdbError("collate_on_device runs on a CUDA device; there is no CPU fallback")
    L = _lib.lib()
    B = len(examples)
    V = int(examples[0]["lidar2camera"].shape[0])
    st = torch.cuda.current_stream(dev).cuda_stream if stream is None else stream
    # ---- host -> device staging of the raw per-sample arrays (small)
    counts = [int(e["gt_bboxes_3d"].shape[0]) for e in examples]
    off = torch.tensor([0] + list(np.cumsum(counts)), dtype=torch.int32)
    box_dim = int(examples[0]["gt_bboxes_3d"].shape[-1]) if counts and max(counts) > 0 else 9
    boxes = torch.cat([_t(e["gt_bboxes_3d"], F32).reshape(-1, box_dim) for e in examples]) if sum(counts) else torch.zeros(1, box_dim)
    labels = torch.cat([_t(e["gt_labels_3d"], torch.int64).reshape(-1) for e in examples]) if sum(counts) else torch.zeros(1, dtype=torch.int64)
    l2c = torch.stack([_t(e["lidar2camera"], F32) for e in examples]).contiguous()
    aug = torch.stack([_t(e["img_aug_matrix"], F32) for e in examples]).contiguous()
    K = torch.stack([_t(e["camera_intrinsics"], F32) for e in examples]).contiguous()
    bev = torch.stack([_t(e["gt_masks_bev"], F32) for e in examples])
    d = lambda t: t.to(dev, non_blocking=True)
    boxes_d, labels_d, off_d, l2c_d, aug_d, K_d = d(boxes.contiguous()), d(labels), d(off), d(l2c), d(aug), d(K)
    cam = torch.empty((B, V, 3, 7), dtype=F32, device=dev)
    check(L.mdb_camera_param(K_d.data_ptr(), l2c_d.data_ptr(), B * V, cam.data_ptr(), st), "mdb_camera_param")
    ret = {"camera_param": cam, "bev_map_with_aux": d(bev), "kwargs": {"bboxes_3d_data": None}}
    if sum(counts) == 0:
        return ret
    cap = int(capacity) if capacity is not None else max(counts) if max_len is None else int(max_len)
    ob = torch.empty((B, V, cap, 8, 3), dtype=F32, device=dev)
    oc = torch.empty((B, V, cap), dtype=torch.int64, device=dev)
    om = torch.empty((B, V, cap), dtype=torch.uint8, device=dev)
    cnt = torch.empty((B, V), dtype=torch.int32, device=dev)
    check(L.mdb_prepare_boxes(boxes_d.data_ptr(), box_dim, labels_d.data_ptr(), off_d.data_ptr(), B, l2c_d.data_ptr(),
                              aug_d.data_ptr(), V, cap, ob.data_ptr(), oc.data_ptr(), om.data_ptr(), cnt.data_ptr(), st),
          "mdb_prepare_boxes")
    if capacity is not None:
        ret["kwargs"]["bboxes_3d_data"] = {"bboxes": ob, "classes": oc, "masks": om.bool(), "counts": cnt,
                                           "count": cnt.max().clamp(max=cap).to(torch.int32)}
        return ret
    if max_len is None:
        longest = int(cnt.max().item())  # the reference sizes the padding by the batch's longest visible list (utils.py:222-239)
        if longest == 0:
            return ret
        ob, oc, om = ob[:, :, :longest].contiguous(), oc[:, :, :longest].contiguous(), om[:, :, :longest].contiguous()
    ret["kwargs"]["bboxes_3d_data"] = {"bboxes": ob, "classes": oc, "masks": om.bool(), "counts": cnt}
    return ret
