"""Images/s of the FID InceptionV3 (all four blocks, 224x400 inputs resized to 299x299) at batch 50 and 512: ours (CUDA-graph
replay on the sm_90a kernels) next to the reference's own InceptionV3 (magicdrive/misc/inception.py from the reference tree
or its oracle/_ref snapshot, built through oracle/make_golden_fid.py's seeded loader, so the same weights) on cuDNN in fp32
and in bf16.  A report, not a gate; prints the card and its power limit.

    python tools/time_fid.py
"""
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from magicdrive_b200 import arch  # noqa: E402
from magicdrive_b200.models import InceptionV3  # noqa: E402
from oracle import make_golden_fid  # noqa: E402
from oracle.ref_shim import REF  # noqa: E402


def _time(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 1e3 / iters


def main():
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print(f"card: {card}")
    model = InceptionV3([3]).cuda()
    model.load_state_dict(arch.inception_synthetic_state_dict(3, make_golden_fid.SEED_W))
    if not os.path.isfile(os.path.join(REF, "magicdrive/misc/inception.py")):
        sys.exit(f"the reference's inception.py is not under {REF}: run `python -m oracle.make_ref_snapshot` where the "
                 "reference tree exists")
    ref = make_golden_fid.reference_inception().InceptionV3([3]).eval().cuda()
    refs = {"reference_fp32": (ref, torch.float32), "reference_bf16": (ref, torch.bfloat16)}
    for batch in (50, 512):
        x = torch.rand(batch, 3, 224, 400, device="cuda")
        iters = 10 if batch == 50 else 3
        res = {"batch": batch, "ours": batch / _time(lambda: model(x), iters)}
        with torch.no_grad(), torch.backends.cudnn.flags(enabled=True, benchmark=True, allow_tf32=False):
            for name, (m, dt) in refs.items():
                m.to(dt)
                xd = x.to(dt)
                res[name] = batch / _time(lambda: m(xd), iters)
        print(json.dumps({k: (round(v, 1) if isinstance(v, float) else v) for k, v in res.items()}))


if __name__ == "__main__":
    main()
