#!/usr/bin/env python
"""Denoising-step time of an fp16 and a bf16 BEVControlNetDenoiser at configs[2] (SD-1.5 size, 224 x 400, six views,
20 boxes, BEV map, guidance 2.0: a batch of 12 view-samples), alternated in one process.

Each arm is prepared once (one eager step, then the captured step graph); a run times `--steps` graph replays of
run_steps between CUDA events.  Arms alternate bf16, fp16, bf16, fp16, ... `--runs` times each, so the spread is visible.
The card's name, power limit and SM clock are printed with the numbers; a run without a CUDA device fails."""
import argparse
import os
import subprocess
import sys
from dataclasses import asdict

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from magicdrive_b200 import arch  # noqa: E402
from magicdrive_b200.models import BEVControlNetModel, UNet2DConditionModelMultiview  # noqa: E402
from magicdrive_b200.pipeline import BEVControlNetDenoiser  # noqa: E402
from magicdrive_b200.synthetic import synthetic_inputs  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--steps", type=int, default=30, help="graph replays per timed run")
ap.add_argument("--runs", type=int, default=3, help="timed runs per arm (at least 2)")
args = ap.parse_args()
assert torch.cuda.is_available(), "needs a CUDA device"


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", "0"], capture_output=True,
                          text=True).stdout.strip()


dev = torch.device("cuda", 0)
print(f"[card] name, power limit, SM clock, max SM clock: {card()}")
inp = synthetic_inputs(1, 6, 28, 50, n_box=20, map_hw=200, seed=0)
arms = {}
for name, dt in (("bf16", torch.bfloat16), ("fp16", torch.float16)):
    un = UNet2DConditionModelMultiview(**asdict(arch.UNetConfig())).reset_parameters_synthetic(11).to(dev, dt)
    cn = BEVControlNetModel(**asdict(arch.ControlNetConfig())).reset_parameters_synthetic(12).to(dev, dt)
    pipe = BEVControlNetDenoiser(un, cn, use_cuda_graph=True, overlap_controlnet=True)
    st = pipe.prepare(inp["latents"], inp["prompt_embeds"], inp["negative_prompt_embeds"], inp["camera_param"],
                      inp["bboxes_3d_data"], inp["bev_map"], guidance_scale=2.0)
    pipe.set_schedule(st, args.steps)
    pipe.run_steps(st, 0, 2)  # eager step + capture + one replay
    torch.cuda.synchronize()
    arms[name] = (pipe, st)

times = {n: [] for n in arms}
for r in range(max(2, args.runs)):
    for name, (pipe, st) in arms.items():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        pipe.run_steps(st, 0, args.steps)
        e1.record()
        torch.cuda.synchronize()
        times[name].append(e0.elapsed_time(e1) / args.steps)
        print(f"[run {r}] {name}: {times[name][-1]:.2f} ms/step")
for name, ts in times.items():
    s = sorted(ts)
    print(f"[summary] {name}: median {s[len(s) // 2]:.2f} ms/step, min {s[0]:.2f}, max {s[-1]:.2f} over {len(s)} runs")
print(f"[card] after the runs: {card()}")
