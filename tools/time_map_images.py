"""Maps/s and mosaics/s of the test-run images on the device (visualize.visualize_maps: render, bicubic resize, rotate
and legend, one synchronisation per call; visualize.concat_views: one copy launch per batch), next to the host time of
the numpy restatement (oracle/map_visualizer.py; not the reference's own route, whose per-pixel Python loop is slower).
Workload: 24 scenes, the six demo samples' maps (tests/golden/map_visualizer.pt) tiled over them, at 200 x 200 and, tiled
2 x 2, 400 x 400, drawn at target_size 400 with a fixed legend so that matplotlib is not what is timed; mosaics of 24
scenes x 6 views at 224 x 400, uint8 RGB, RGBA and fp32 [0, 1].  A report, not a gate; prints the card, its power limit
and one JSON line.

    python tools/time_map_images.py [--scenes 24] [--iters 50]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from magicdrive_b200 import visualize  # noqa: E402
from oracle import map_visualizer as O  # noqa: E402
from oracle.make_golden_map_visualizer import load  # noqa: E402
from tests.common import GOLDEN  # noqa: E402

LEGEND = np.full((50, 400, 3), 255, np.uint8)


def legend(names, size):
    return LEGEND


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", type=int, default=24)
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_map_images needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    fx = load(os.path.join(GOLDEN, "map_visualizer.pt"))
    demo = [c["map"] for c in fx["maps"] if c["name"].startswith("demo") and c["name"].endswith("@400")]
    m200 = np.stack([demo[i % len(demo)] for i in range(args.scenes)])
    m400 = np.tile(m200, (1, 1, 2, 2))
    res = {"card": card, "scenes": args.scenes, "target_size": 400}

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

    for side, m in ((200, m200), (400, m400)):
        x = torch.from_numpy(m).to("cuda", torch.float32)
        t = device_time(lambda: visualize.visualize_maps(x, target_size=400, legend=legend))
        res[f"maps{side}_call_ms"] = t * 1e3
        res[f"maps{side}_per_s"] = args.scenes / t
        n_host = 3
        t0 = time.perf_counter()
        for i in range(n_host):
            O.visualize_map(m[i], visualize.NUSCENES_MAP_CLASSES, visualize.NUSCENES_OBJECT_CLASSES, 400, legend)
        res[f"maps{side}_host_numpy_restatement_ms_per_map"] = (time.perf_counter() - t0) / n_host * 1e3

    rng = np.random.default_rng(0)
    u8 = torch.from_numpy(rng.integers(0, 256, (args.scenes, 6, 224, 400, 3), dtype=np.uint8)).cuda()
    rgba = torch.from_numpy(rng.integers(0, 256, (args.scenes, 6, 224, 400, 4), dtype=np.uint8)).cuda()
    f32 = u8.float() / 255
    for name, v in (("rgb", u8), ("rgba", rgba), ("f32", f32)):
        t = device_time(lambda: visualize.concat_views(v))
        res[f"mosaic_{name}_call_ms"] = t * 1e3
        res[f"mosaics_{name}_per_s"] = args.scenes / t
    px = f32 * 2 - 1
    px = px.permute(0, 1, 4, 2, 3).contiguous()
    t = device_time(lambda: visualize.concat_views(visualize.camera_views_u8(px)))
    res["ori_mosaics_per_s"] = args.scenes / t
    t0 = time.perf_counter()
    for s in range(3):
        O.concat_6_views(u8[s].cpu().numpy())
    res["mosaic_host_numpy_restatement_ms"] = (time.perf_counter() - t0) / 3 * 1e3
    print(f"card, power limit: {card}")
    for k, v in res.items():
        print(f"  {k}: {v:.3f}" if isinstance(v, float) else f"  {k}: {v}")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
