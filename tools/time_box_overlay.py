"""Views/s of the 3D-box overlay (box_overlay.show_box_on_views: one projection and one drawing launch per batch) on the
device against the reference's host route: the uint8 views copied to the host, then per view a PIL image, the corner
projection in numpy and cv2.line for each edge (what visualize_camera does), one view per process of a pool of all
cores.  Workload: 24 scenes x 6 views at 224x400, the boxes of the six nuScenes demo samples (tests/golden/box_overlay.pt)
tiled over the scenes.  A report, not a gate; prints the card, its power limit and one JSON line.

    python tools/time_box_overlay.py [--scenes 24] [--iters 50]
"""
import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from magicdrive_b200 import box_overlay  # noqa: E402
from oracle import box_overlay as O  # noqa: E402
from oracle.make_golden_box_overlay import load  # noqa: E402
from tests.common import GOLDEN  # noqa: E402


def _host_view(args):
    """The reference's host route for one view: PIL image in, PIL image with the boxes out."""
    import cv2
    from PIL import Image
    a, boxes, labels, trans = args
    canvas = np.asarray(Image.fromarray(a)).copy()
    ends, lab, _ = O.project(boxes, labels, trans)
    for b in range(len(lab)):
        color = O.OBJECT_PALETTE[O.NUSCENES_OBJECT_CLASSES[int(lab[b])]]
        for s, e in O.EDGES:
            cv2.line(canvas, ends[b, s], ends[b, e], color, 1, cv2.LINE_AA)
    return Image.fromarray(canvas)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", type=int, default=24)
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_box_overlay needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    cases = load(os.path.join(GOLDEN, "box_overlay.pt"))["cases"]
    examples = [cases[i % len(cases)] for i in range(args.scenes)]
    rng = np.random.default_rng(0)
    u8 = torch.from_numpy(rng.integers(0, 256, (args.scenes, 6, 224, 400, 3), dtype=np.uint8)).cuda()
    f32 = u8.float() / 255
    n_views = args.scenes * 6
    res = {"card": card, "scenes": args.scenes, "views": n_views, "size": [224, 400],
           "boxes_drawn": int(box_overlay.project_boxes(examples, 6, "cuda")["counts"].sum())}

    def device_time(fn):
        fn()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.iters):
            fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / 1e3 / args.iters

    out = torch.empty_like(u8)
    # the whole call (host staging of the boxes and transforms, both launches, the status read) and the two kernels alone
    res["call_u8_ms"] = device_time(lambda: box_overlay.show_box_on_views(u8, examples, out=out)) * 1e3
    res["call_f32_ms"] = device_time(lambda: box_overlay.show_box_on_views(f32, examples)) * 1e3
    res["call_transparent_ms"] = device_time(lambda: box_overlay.show_box_on_views(u8, examples, transparent_bg=True)) * 1e3
    proj = box_overlay.project_boxes(examples, 6, "cuda")
    st = box_overlay._stage(examples, 6, box_overlay.NUSCENES_OBJECT_CLASSES)
    res["project_kernel_ms"] = device_time(lambda: box_overlay._project(st, 6, "cuda")) * 1e3
    pal = st["palette"].cuda()
    from magicdrive_b200 import _lib
    L = _lib.lib()
    draw = lambda: L.mdb_draw_box_edges_aa(u8.data_ptr(), 0, n_views, 224, 400, proj["endpoints"].data_ptr(),
                                           proj["colors"].data_ptr(), proj["counts"].data_ptr(), proj["status"].data_ptr(),
                                           proj["colors"].shape[-1], pal.data_ptr(), 10, 0, out.data_ptr(),
                                           torch.cuda.current_stream().cuda_stream)
    res["draw_kernel_ms"] = device_time(draw) * 1e3
    res["device_views_per_s"] = n_views / (res["call_u8_ms"] / 1e3)

    try:
        import cv2  # noqa: F401
        jobs = []
        for s, ex in enumerate(examples):
            tr = O.view_transforms(ex)
            jobs += [(None, np.asarray(ex["gt_bboxes_3d"], np.float32), np.asarray(ex["gt_labels_3d"]), tr[v])
                     for v in range(6)]
        with ProcessPoolExecutor(os.cpu_count()) as pool:
            list(pool.map(_host_view, [(u8[0, 0].cpu().numpy(),) + j[1:] for j in jobs[:os.cpu_count()]]))  # warm
            times = []
            for _ in range(3):
                t0 = time.perf_counter()
                host = u8.cpu().numpy().reshape(n_views, 224, 400, 3)
                list(pool.map(_host_view, [(host[i],) + jobs[i][1:] for i in range(n_views)], chunksize=4))
                times.append(time.perf_counter() - t0)
        res["host_cores"] = os.cpu_count()
        res["host_ms"] = min(times) * 1e3
        res["host_views_per_s"] = n_views / min(times)
    except ImportError:
        res["host_ms"] = "cv2 not installed"
    print(card)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
