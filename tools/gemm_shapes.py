#!/usr/bin/env python
"""Per-shape timing of the GEMM / implicit-GEMM conv launches of one bench.py step.

  python tools/gemm_shapes.py [--res 224x400|424x800] [--out FILE]

Runs one eager, single-stream denoising step of bench.py's default workload (configs[2], one six-view scene, CFG on) with
every tensor-core launch bracketed by CUDA events, queued behind a spin kernel so the events bracket back-to-back device
execution.  Launches are grouped by shape; each row gives the launch count, the total kernel time, the achieved TFLOP/s
and the planner's tiling (block_n, M x N x K-split tiles, waves of the persistent grid).
"""
import argparse
import os
import sys
from collections import defaultdict
from dataclasses import asdict

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--res", default="224x400", choices=["224x400", "424x800"])
    ap.add_argument("--out", help="also write the table to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gemm_shapes.py needs a CUDA device")

    from magicdrive_b200 import arch, ops
    from magicdrive_b200.models import BEVControlNetModel, UNet2DConditionModelMultiview
    from magicdrive_b200.pipeline import BEVControlNetDenoiser
    from magicdrive_b200.synthetic import synthetic_inputs

    dev = torch.device("cuda", 0)
    h, w, mhw = (28, 50, 200) if args.res == "224x400" else (53, 100, 400)
    ucfg, ccfg = arch.UNetConfig(), arch.ControlNetConfig(map_size=(8, mhw, mhw))
    un = UNet2DConditionModelMultiview(**asdict(ucfg)).reset_parameters_synthetic(11).to(dev, torch.bfloat16)
    cn = BEVControlNetModel(**asdict(ccfg)).reset_parameters_synthetic(12).to(dev, torch.bfloat16)
    pipe = BEVControlNetDenoiser(un, cn, use_cuda_graph=False, overlap_controlnet=False)
    inp = synthetic_inputs(1, 6, h, w, n_box=20, map_hw=mhw, seed=0)
    st = pipe.prepare(inp["latents"], inp["prompt_embeds"], inp["negative_prompt_embeds"], inp["camera_param"],
                      inp["bboxes_3d_data"], inp["bev_map"], guidance_scale=2.0)
    pipe.set_schedule(st, 50)
    for i in range(2):  # sizes workspaces, loads every kernel
        pipe.run_steps(st, i, i + 1)
    torch.cuda.synchronize()
    torch.cuda._sleep(int(50e6))
    ops.start_profile()
    pipe.run_steps(st, 2, 3)
    prof = ops.stop_profile(with_info=True)

    rows = defaultdict(lambda: [0, 0.0, 0.0])
    for kind, flops, sec, info in prof:
        if kind != "gemm_conv":
            continue
        r = rows[info]
        r[0] += 1
        r[1] += sec
        r[2] += flops
    tot_s = sum(r[1] for r in rows.values())
    tot_f = sum(r[2] for r in rows.values())
    name = torch.cuda.get_device_name(dev)
    lines = [f"# {name}, {args.res}, one eager single-stream step: {sum(r[0] for r in rows.values())} GEMM/conv launches, "
             f"{tot_s * 1e3:.3f} ms, {tot_f / 1e12:.3f} TFLOP, {tot_f / tot_s / 1e12:.1f} TFLOP/s",
             f"{'count':>5} {'ms':>8} {'%time':>6} {'TFLOP/s':>8}  shape | plan"]
    for info, (n, sec, flops) in sorted(rows.items(), key=lambda kv: -kv[1][1]):
        lines.append(f"{n:5d} {sec * 1e3:8.3f} {100 * sec / tot_s:6.1f} {flops / sec / 1e12:8.1f}  {info}")
    text = "\n".join(lines)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
