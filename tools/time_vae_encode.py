"""Time of AutoencoderKL.encode for 6 camera views at 224x400 and 424x800 with SD-1.5-size seeded weights: ours as the
CUDA-graph replay of encode_latents and as the eager encode call, next to the reference's own AutoencoderKL.encode (the
vendored diffusers from the reference tree or its oracle/_ref snapshot, same weights) in fp32 and in bf16.  CUDA events;
prints the card and its power limit.  A report, not a gate.

    python tools/time_vae_encode.py
"""
import json
import os
import subprocess
import sys
from dataclasses import asdict

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from magicdrive_b200 import arch  # noqa: E402
from magicdrive_b200.models import AutoencoderKL  # noqa: E402
from oracle import ref_shim  # noqa: E402
from oracle.make_golden_vae_encode import full_state_dict, reference_vae  # noqa: E402


def _time(fn, iters):
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
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    print(f"card: {card}")
    if not ref_shim.available():
        sys.exit(f"the reference's diffusers is not under {ref_shim.REF}: run `python -m oracle.make_ref_snapshot` where the "
                 "reference tree exists")
    cfg = arch.VaeConfig()
    sd = full_state_dict(cfg, 3)
    vae = AutoencoderKL(**asdict(cfg))
    vae.load_state_dict(sd)
    vae = vae.cuda()
    ref = reference_vae(ref_shim.load(), cfg)
    ref.load_state_dict(sd)
    ref = ref.cuda()
    for h, w in ((224, 400), (424, 800)):
        pix = torch.rand(1, 6, 3, h, w, device="cuda") * 2 - 1
        x = pix[0]
        iters = 10 if h == 224 else 4
        res = {"views": 6, "size": f"{h}x{w}", "tflop": round(_flops(cfg, h, w) * 6 / 1e12, 2)}
        with torch.no_grad():
            res["ours_graph_ms"] = _time(lambda: vae.encode_latents(pix), iters)
            res["ours_eager_ms"] = _time(lambda: vae.encode(x), iters)
            with torch.backends.cudnn.flags(enabled=True, benchmark=True, allow_tf32=False):
                for name, dt in (("reference_fp32_ms", torch.float32), ("reference_bf16_ms", torch.bfloat16)):
                    ref.to(dt)
                    xd = x.to(dt)
                    res[name] = _time(lambda: ref.encode(xd).latent_dist.mean, iters)
        res["ours_graph_tflops"] = round(res["tflop"] / res["ours_graph_ms"] * 1e3, 1)
        print(json.dumps({k: (round(v, 2) if isinstance(v, float) else v) for k, v in res.items()}))
        ref.to(torch.float32)


def _flops(cfg, h, w):
    """Multiply-adds x 2 of one image's convolutions and attention GEMMs (GroupNorm / softmax / elementwise not counted)."""
    f = 2 * h * w * 9 * cfg.in_channels * cfg.block_out_channels[0]
    for _, resnets, down in arch.vae_encoder_blocks(cfg):
        for _, ci, co in resnets:
            f += 2 * h * w * 9 * (ci * co + co * co) + (2 * h * w * ci * co if ci != co else 0)
        if down:
            h, w = (h - 2) // 2 + 1, (w - 2) // 2 + 1
            f += 2 * h * w * 9 * co * co
    c, L = cfg.block_out_channels[-1], h * w
    f += 2 * 2 * h * w * 9 * c * c + 2 * L * c * c * 4 + 2 * 2 * L * L * c
    return f + 2 * h * w * 9 * c * 2 * cfg.latent_channels


if __name__ == "__main__":
    main()
