"""Views/s of the FID evaluation protocol (FIDProtocol.generated: bicubic resize and pad to 900x1600, JPEG round trip,
scoring resize and crop) on the device against the reference's Pillow route on the host cores (resize, pad, .jpg save
and load in memory, resize, crop: one view per process of a pool of all cores), each with and without the Inception
features (2048-d, synthetic weights).  Views: 224x400 fp32 device images, batch 48 (8 scenes x 6 cameras).  A report,
not a gate; prints the card, its power limit and one JSON line.

    python tools/time_fid_protocol.py [--config 224x400] [--batch 48] [--iters 20]
"""
import argparse
import io
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from magicdrive_b200 import arch, fid  # noqa: E402
from magicdrive_b200.models import InceptionV3  # noqa: E402
from oracle import fid_protocol as O  # noqa: E402


def _device_time(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 1e3 / iters


def _pillow_view(args):
    """The reference's route for one uint8 view, all in memory: returns the scored uint8 image."""
    from PIL import Image
    a, cfg = args
    image_size, back_resize, pad, ratio = cfg
    canvas = Image.new("RGB", (back_resize[1] + pad[0] + pad[2], back_resize[0] + pad[1] + pad[3]))
    canvas.paste(Image.fromarray(a).resize(back_resize[::-1], Image.BICUBIC), (pad[0], pad[1]))
    buf = io.BytesIO()
    canvas.save(buf, format="JPEG")
    (rh, rw), (top, left, fh, fw) = O.scoring_window(image_size, ratio)
    with Image.open(io.BytesIO(buf.getvalue())) as im:
        im = im.convert("RGB").resize((rw, rh), Image.BICUBIC).crop((left, top, left + fw, top + fh))
        return np.asarray(im)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="224x400", choices=sorted(fid.PROTOCOL_CONFIGS))
    ap.add_argument("--batch", type=int, default=48)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: this tool measures the device protocol and reports nothing without one")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print(f"card: {card}; host cores: {os.cpu_count()}")
    cfg = fid.PROTOCOL_CONFIGS[args.config]
    if args.batch % 6:
        sys.exit("--batch must be a multiple of 6 (scenes x 6 cameras)")
    v = torch.from_numpy(O.views(0, args.batch, *cfg[0])).cuda().reshape(args.batch // 6, 6, *cfg[0], 3)
    p = fid.FIDProtocol.for_config(args.config)
    model = InceptionV3([3]).cuda()
    model.load_state_dict(arch.inception_synthetic_state_dict(3, seed=3))
    stats = fid.FIDStatistics(model, 2048, protocol=p)

    t_proto = _device_time(lambda: p.generated(v), args.iters)
    t_full = _device_time(lambda: stats.update(v), max(3, args.iters // 4))
    # device vs host bytes: the host route must give the same images
    u8 = O.to_u8(v.reshape(-1, *cfg[0], 3).cpu().numpy())
    with ProcessPoolExecutor(os.cpu_count()) as pool:
        list(pool.map(_pillow_view, [(a, cfg) for a in u8[:os.cpu_count()]]))  # warm the workers
        t0 = time.perf_counter()
        host = np.stack(list(pool.map(_pillow_view, [(a, cfg) for a in u8])))
        t_pil = (time.perf_counter() - t0)
    same = bool(np.array_equal(host, p.generated(v).cpu().numpy()))
    scored = torch.from_numpy(host).cuda()
    t_incep = _device_time(lambda: stats._update_u8(scored), max(3, args.iters // 4))
    res = {"config": args.config, "batch": args.batch, "bytes_equal": same,
           "device_protocol_views_per_s": args.batch / t_proto,
           "device_protocol_plus_inception_views_per_s": args.batch / t_full,
           "pillow_host_views_per_s": args.batch / t_pil,
           "pillow_host_then_device_inception_views_per_s": args.batch / (t_pil + t_incep)}
    print(json.dumps({k: (round(x, 1) if isinstance(x, float) else x) for k, x in res.items()}))


if __name__ == "__main__":
    main()
