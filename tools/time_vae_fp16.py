#!/usr/bin/env python
"""Decode and encode time of an fp16 and a bf16 SD-1.5 AutoencoderKL for six views at 224 x 400 and 424 x 800, alternated
in one process.

Each (arm, size) is captured once: decode_latents / encode_latents replay one CUDA graph per shape.  A run times `--reps`
calls between CUDA events.  Arms alternate bf16, fp16, bf16, fp16, ... `--runs` times each, so the spread is visible.
The card's name, power limit and SM clock are printed with the numbers; a run without a CUDA device fails."""
import argparse
import os
import subprocess
import sys
from dataclasses import asdict

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from magicdrive_b200 import arch  # noqa: E402
from magicdrive_b200.models import AutoencoderKL  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=10, help="calls per timed run")
ap.add_argument("--runs", type=int, default=3, help="timed runs per arm (at least 2)")
args = ap.parse_args()
assert torch.cuda.is_available(), "needs a CUDA device"


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                          text=True).stdout.strip()


dev = torch.device("cuda", 0)
print(f"[card] name, power limit, SM clock, max SM clock: {card()}")
cfg = arch.VaeConfig()
sd = arch.synthetic_state_dict({**arch.vae_encoder_param_shapes(cfg), **arch.vae_decoder_param_shapes(cfg)}, 13)
vaes = {}
for name, dt in (("bf16", torch.bfloat16), ("fp16", torch.float16)):
    vae = AutoencoderKL(**asdict(cfg))
    vae.load_state_dict(sd)
    vaes[name] = vae.to(dev, dt)
g = torch.Generator().manual_seed(0)
work = {}
for h, w in ((224, 400), (424, 800)):
    lat = torch.randn(1, 6, 4, h // 8, w // 8, generator=g).to(dev)
    pix = (torch.rand(1, 6, 3, h, w, generator=g) * 2 - 1).to(dev)
    work[f"decode {h}x{w}"] = lambda v, lat=lat: v.decode_latents(lat)
    work[f"encode {h}x{w}"] = lambda v, pix=pix: v.encode_latents(pix)
for fn in work.values():
    for v in vaes.values():
        fn(v)  # eager call to size scratch, then the capture
        fn(v)
torch.cuda.synchronize()

times = {(w_, a): [] for w_ in work for a in vaes}
for r in range(max(2, args.runs)):
    for wname, fn in work.items():
        for aname, v in vaes.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.reps):
                fn(v)
            e1.record()
            torch.cuda.synchronize()
            times[(wname, aname)].append(e0.elapsed_time(e1) / args.reps)
            print(f"[run {r}] {wname} {aname}: {times[(wname, aname)][-1]:.2f} ms/call")
for (wname, aname), ts in times.items():
    s = sorted(ts)
    print(f"[summary] {wname} {aname}: median {s[len(s) // 2]:.2f} ms/call, min {s[0]:.2f}, max {s[-1]:.2f} "
          f"over {len(s)} runs")
print(f"[card] after the runs: {card()}")
