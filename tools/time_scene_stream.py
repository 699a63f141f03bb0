#!/usr/bin/env python
"""A stream of scenes with different box counts through BEVControlNetDenoiser, timed three ways, and the conditioning
cross-attention launch alone.

Stream: 24 seeded scenes at SD-1.5 size (224 x 400, six views, guidance on, 20 UniPC steps) with box counts spread over
4..49; host clock around the whole stream, ending in a synchronise, after one warm-up stream per arm:
  (a) default mode, a call per scene (a new resident state and two graph captures whenever the box count changes);
  (b) default mode with bbox_max_length=159 (one state, but 159 attended box tokens: different images);
  (c) box_capacity=159 (one state, the scene's own count attended).
(a) and (c) are alternated twice so that their spread is visible.
Attention: q [12, lq, heads*d] against 98 keys, CUDA events over many launches: the exact launch (lk = 98) and the launch
with a device key count of 98 at lk = 256 (resident key tiles), each as a CUDA graph of many launches so that the device, not
the host's launch rate, is timed.
The card's name and power limit are printed with the numbers; a run without a CUDA device fails."""
import argparse
import os
import subprocess
import sys
import time
from dataclasses import asdict

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from magicdrive_b200 import arch, ops  # noqa: E402
from magicdrive_b200.models import BEVControlNetModel, UNet2DConditionModelMultiview  # noqa: E402
from magicdrive_b200.pipeline import BEVControlNetDenoiser  # noqa: E402
from magicdrive_b200.synthetic import synthetic_inputs  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--scenes", type=int, default=24)
ap.add_argument("--steps", type=int, default=20)
ap.add_argument("--capacity", type=int, default=159)
ap.add_argument("--attention-launches", type=int, default=100, help="launches per captured graph (replayed 20 times)")
args = ap.parse_args()

dev = torch.device("cuda", 0)
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True).stdout.strip()
print(f"[card] {card}")

un = UNet2DConditionModelMultiview(**asdict(arch.UNetConfig())).reset_parameters_synthetic(11).to(dev, torch.bfloat16)
cn = BEVControlNetModel(**asdict(arch.ControlNetConfig())).reset_parameters_synthetic(12).to(dev, torch.bfloat16)
counts = [4 + (i * 19) % 46 for i in range(args.scenes)]  # 4..49, neighbours far apart
scenes = [synthetic_inputs(1, 6, 28, 50, n_box=n, map_hw=200, seed=100 + i) for i, n in enumerate(counts)]
print(f"[stream] {args.scenes} scenes, box counts {counts}, {args.steps} UniPC steps, guidance 2.0")


def run(pipe, **extra):
    t0 = time.perf_counter()
    for s in scenes:
        out = pipe(image=s["bev_map"], camera_param=s["camera_param"], prompt_embeds=s["prompt_embeds"],
                   negative_prompt_embeds=s["negative_prompt_embeds"], latents=s["latents"], num_inference_steps=args.steps,
                   guidance_scale=2.0, bev_controlnet_kwargs={"bboxes_3d_data": s["bboxes_3d_data"]}, **extra)
    torch.cuda.synchronize()
    assert torch.isfinite(out).all()
    return time.perf_counter() - t0


arms = {"a default": (BEVControlNetDenoiser(un, cn, scheduler="unipc"), {}),
        "b default + bbox_max_length=159": (BEVControlNetDenoiser(un, cn, scheduler="unipc"), {"bbox_max_length": 159}),
        f"c box_capacity={args.capacity}": (BEVControlNetDenoiser(un, cn, scheduler="unipc", box_capacity=args.capacity), {})}
for name, (pipe, extra) in arms.items():
    if args.scenes:
        run(pipe, **extra)  # warm-up stream
a, b, c = arms
for name in (a, c, b, a, c) if args.scenes else ():
    pipe, extra = arms[name]
    t = run(pipe, **extra)
    print(f"[stream] {name}: {t:.3f} s, {1e3 * t / args.scenes:.1f} ms per scene")

B, LEN = 12, 98
kv_len = torch.full((B,), LEN, dtype=torch.int32, device=dev)
for d, heads, lq in ((40, 8, 1400), (80, 8, 350), (160, 8, 91)):
    c_ = heads * d
    q = torch.randn(B * lq, c_, device=dev).bfloat16()
    exact = torch.randn(B * LEN, 2 * c_, device=dev).bfloat16()
    wide = torch.zeros(B * 256, 2 * c_, device=dev).bfloat16()
    wide.view(B, 256, -1)[:, :LEN] = exact.view(B, LEN, -1)
    out = torch.empty(B * lq, c_, dtype=torch.bfloat16, device=dev)
    kw = dict(b=B, heads=heads, lq=lq, d=d, ldq=c_, ldk=2 * c_, ldv=2 * c_, scale=d ** -0.5, out=out)
    launches = {"exact lk=98": lambda: ops.attention(q, exact, exact[:, c_:], lk=LEN, **kw),
                "kv_len=98, lk=256": lambda: ops.attention(q, wide, wide[:, c_:], lk=256, kv_len=kv_len, **kw)}
    ref = launches["exact lk=98"]().clone()
    assert torch.equal(launches["kv_len=98, lk=256"](), ref)
    graphs = {}
    for name, fn in launches.items():
        fn()
        torch.cuda.synchronize()
        graphs[name] = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graphs[name]):
            for _ in range(args.attention_launches):
                fn()
    for rep in range(3):
        for name, g in graphs.items():
            g.replay()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(20):
                g.replay()
            e1.record()
            torch.cuda.synchronize()
            print(f"[attention] d={d} heads={heads} lq={lq} {name}: "
                  f"{1e3 * e0.elapsed_time(e1) / (20 * args.attention_launches):.2f} us per launch (run {rep})")
