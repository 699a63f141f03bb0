"""TEST INFRASTRUCTURE ONLY — tests/golden/vae_encode.pt: AutoencoderKL.encode of the reference's diffusers (autoencoder_kl.py:
160-171) run on seeded images with name-keyed synthetic weights (block_out_channels 32/64/64/64), via oracle/ref_shim.py.
Two batches: 50x70, odd at every level (25x35 -> 12x17 -> 6x8, where the encoder's end padding floors), and 64x96.  Stored
per batch: the input, the moments, latent_dist.mean / .std and one latent_dist.sample(generator) from a seeded CPU
generator.  Run in the build container (needs /root/reference):  python -m oracle.make_golden_vae_encode"""
import os
import sys

import torch

from magicdrive_b200 import arch
from oracle import ref_shim
from oracle.make_golden import OUT

SEED_W = 13
CASES = {"odd": (2, 50, 70, 21), "even": (1, 64, 96, 22)}  # name: (n, H, W, input / sample seed)


def vae_config():
    return arch.VaeConfig(block_out_channels=(32, 64, 64, 64))


def full_state_dict(cfg, seed=SEED_W):
    return arch.synthetic_state_dict({**arch.vae_encoder_param_shapes(cfg), **arch.vae_decoder_param_shapes(cfg)}, seed)


def reference_vae(R, cfg):
    return R.AutoencoderKL(block_out_channels=list(cfg.block_out_channels), down_block_types=["DownEncoderBlock2D"] * 4,
                           up_block_types=["UpDecoderBlock2D"] * 4, latent_channels=cfg.latent_channels,
                           layers_per_block=cfg.layers_per_block).eval()


def images(n, h, w, seed):
    return torch.rand(n, 3, h, w, generator=torch.Generator().manual_seed(seed)) * 2 - 1


@torch.no_grad()
def main():
    R = ref_shim.load()
    cfg = vae_config()
    vae = reference_vae(R, cfg)
    vae.load_state_dict(full_state_dict(cfg), strict=True)
    out = dict(block_out_channels=cfg.block_out_channels, seed=SEED_W, cases={})
    for name, (n, h, w, seed) in CASES.items():
        x = images(n, h, w, seed)
        dist = vae.encode(x).latent_dist
        smp = dist.sample(torch.Generator().manual_seed(seed + 100))
        out["cases"][name] = dict(x=x, sample_seed=seed + 100, moments=dist.parameters, mean=dist.mean, std=dist.std,
                                  sample=smp)
        print(name, tuple(x.shape), "->", tuple(dist.parameters.shape))
    torch.save(out, os.path.join(OUT, "vae_encode.pt"))
    print("vae_encode.pt", os.path.getsize(os.path.join(OUT, "vae_encode.pt")) // 1024, "KiB")


if __name__ == "__main__":
    sys.exit(main())
