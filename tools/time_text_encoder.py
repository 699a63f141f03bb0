"""Time the CLIP text encoder (SD-1.5 size, seeded weights) on the GPU with CUDA events: CLIPTextModel with CUDA-graph replay
and eager, next to the same arithmetic in bf16 torch (oracle/clip_text.py at dtype=bfloat16) on the same card.  Batches of 2 x
77 tokens (one scene's [uncond ; cond] captions) and 8 x 77.  Prints the card's name and power limit with the numbers.

    python tools/time_text_encoder.py [--iters 50] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from magicdrive_b200 import arch, models  # noqa: E402
from oracle.clip_text import clip_text_forward, draw_weights  # noqa: E402


def card():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        power = q[torch.cuda.current_device()] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def time_ms(fn, iters, warmup=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU only")
    cfg = arch.ClipTextConfig()
    sd = draw_weights(cfg, 12)
    m = models.CLIPTextModel()
    m.load_state_dict(sd)
    m = m.cuda()
    sd16 = {k: v.to("cuda", torch.bfloat16) for k, v in sd.items()}
    name, power = card()
    res = dict(card=name, power_limit_and_max_sm_clock=power, iters=args.iters, ms={})
    with torch.no_grad():
        for n in (2, 8):
            ids = torch.randint(0, cfg.vocab_size - 2, (n, 77), generator=torch.Generator().manual_seed(n))
            ids[:, 0], ids[:, 20:] = cfg.vocab_size - 2, cfg.vocab_size - 1
            ids = ids.cuda()
            m.use_cuda_graph = True
            graph = time_ms(lambda: m(ids), args.iters)
            m.use_cuda_graph = False
            eager = time_ms(lambda: m(ids), args.iters)
            torch_bf16 = time_ms(lambda: clip_text_forward(sd16, cfg, ids, dtype=torch.bfloat16), args.iters)
            res["ms"][f"{n}x77"] = dict(graph=round(graph, 4), eager=round(eager, 4), torch_bf16=round(torch_bf16, 4))
            print(f"{n}x77 tokens: CLIPTextModel graph {graph:.3f} ms | eager {eager:.3f} ms | "
                  f"same arithmetic in bf16 torch {torch_bf16:.3f} ms", flush=True)
    print(f"card: {name}; power limit, max SM clock: {power}")
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
