"""Time from fp32 device views to `.jpg` bytes in host memory: FIDProtocol.encode_generated (device resize, pad and
encoder; the files' bytes copied to the host) against the reference's route (the views copied to the host, numpy_to_pil,
post_trans = Resize(back_resize, BICUBIC) + Pad(back_pad), PIL save to BytesIO) on one host core and on all of them.
Also the encoder's kernels alone (mdb_jpeg_encode_u8 on the 900 x 1600 canvases) with CUDA events.  A report, not a
gate; prints the card, its power limit and one JSON line.

    python tools/time_jpeg_encode.py [--iters 20]
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
from magicdrive_b200 import fid, jpeg_ops  # noqa: E402
from oracle import fid_protocol as O  # noqa: E402

CONFIG = "224x400"


def _host_view(a):
    """The reference's route for one uint8 view: post_trans, then the PIL save."""
    import torchvision
    from PIL import Image
    from torchvision.transforms import InterpolationMode
    _, back_resize, back_pad, _ = fid.PROTOCOL_CONFIGS[CONFIG]
    post = torchvision.transforms.Compose([
        torchvision.transforms.Resize(list(back_resize), interpolation=InterpolationMode.BICUBIC),
        torchvision.transforms.Pad(list(back_pad))])
    buf = io.BytesIO()
    post(Image.fromarray(a)).save(buf, "JPEG")
    return buf.getvalue()


def host_route(views_dev, pool):
    u8 = O.to_u8(views_dev.cpu().numpy())  # numpy_to_pil's rounding
    return list(pool.map(_host_view, list(u8), chunksize=1)) if pool else [_host_view(a) for a in u8]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("time_jpeg_encode needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    protocol = fid.FIDProtocol.for_config(CONFIG)
    cores = os.cpu_count()
    res = {"card": card, "config": CONFIG, "host_cores": cores, "cases": []}
    with ProcessPoolExecutor(cores) as pool:
        for n in (6, 48):
            views = torch.from_numpy(O.views(5, n, 224, 400)).cuda()
            files = protocol.encode_generated(views[None])
            assert files == host_route(views, None), "device and reference files differ"

            def timed(fn, iters):
                fn()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(iters):
                    fn()
                torch.cuda.synchronize()
                return (time.perf_counter() - t0) / iters * 1e3

            dev = timed(lambda: protocol.encode_generated(views[None]), args.iters)
            one = timed(lambda: host_route(views, None), max(2, args.iters // 10))
            pool.map(_host_view, [np.zeros((224, 400, 3), np.uint8)] * cores)  # start the workers
            allc = timed(lambda: host_route(views, pool), max(2, args.iters // 5))
            # the encoder's kernels alone on the canvases
            left, top, _, _ = protocol.back_pad
            canvas = protocol._resize(views, True, protocol.back_resize, canvas=protocol.canvas, offset=(top, left))
            big = jpeg_ops.scratch_bytes(n, *protocol.canvas, 256 * n)  # 1 MiB of entropy-coded data per view
            meta = jpeg_ops.jpeg_encode_u8(canvas, 75, scratch=torch.empty(big, dtype=torch.uint8, device="cuda"),
                                           out=torch.empty(big, dtype=torch.uint8, device="cuda"))
            assert bool((meta[:, 2] >= 0).all())
            chunks = int(((meta[:, 0] + 4095) // 4096).sum())
            scratch = torch.empty(jpeg_ops.scratch_bytes(n, *protocol.canvas, chunks), dtype=torch.uint8, device="cuda")
            out = torch.empty(int(meta[:, 1].sum()), dtype=torch.uint8, device="cuda")
            lib = jpeg_ops._lib.lib()
            st = torch.cuda.current_stream().cuda_stream
            m = torch.empty((n, 3), dtype=torch.int64, device="cuda")
            launch = lambda: lib.mdb_jpeg_encode_u8(canvas.data_ptr(), n, *protocol.canvas, 75, scratch.data_ptr(),
                                                    scratch.numel(), out.data_ptr(), out.numel(), m.data_ptr(), st)
            launch()
            torch.cuda.synchronize()
            assert bool((m[:, 2] >= 0).all())
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                launch()
            e1.record()
            torch.cuda.synchronize()
            kern = e0.elapsed_time(e1) / args.iters
            res["cases"].append({"views": n, "device_ms": round(dev, 3), "host_1core_ms": round(one, 2),
                                 f"host_{cores}core_ms": round(allc, 2), "encoder_kernels_ms": round(kern, 3),
                                 "bytes": sum(len(f) for f in files)})
            print(f"[time_jpeg_encode] {card}: {n} views {CONFIG} -> canvas {protocol.canvas}: device {dev:.2f} ms, "
                  f"encoder kernels {kern:.3f} ms, reference route {one:.1f} ms (1 core) / {allc:.1f} ms ({cores} cores)")
    print(json.dumps(res))


if __name__ == "__main__":
    main()
