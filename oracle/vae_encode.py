"""TEST INFRASTRUCTURE ONLY — plain-torch restatement of diffusers' AutoencoderKL.encode (the reference's given-view demo,
demo/run_cond_on_view.py:80-85), from state-dict tensors by their checkpoint names.  Line numbers cite the reference's
vendored diffusers 0.17.1 (third_party/diffusers/src/diffusers/models/): Encoder.forward vae.py:39-149, AutoencoderKL.encode
autoencoder_kl.py:160-171, DiagonalGaussianDistribution vae.py:397-441.

fp32 by default; `dtype=torch.bfloat16` runs the same arithmetic in bf16 torch (the yardstick of how far a bf16
implementation may sit from fp32)."""
import torch
import torch.nn.functional as F

from magicdrive_b200 import arch
from oracle.torch_oracle import resnet_block


def vae_encode_moments(sd, cfg: arch.VaeConfig, x: torch.Tensor, dtype=torch.float32) -> torch.Tensor:
    """x: (n, in_channels, H, W) -> moments (n, 2 * latent_channels, h, w) = quant_conv(encoder(x))."""
    sd = {k: v.to(device=x.device, dtype=dtype) for k, v in sd.items() if k.startswith(("encoder.", "quant_conv."))}
    g, eps = cfg.norm_num_groups, 1e-6
    conv = lambda p, t, **kw: F.conv2d(t, sd[p + ".weight"], sd[p + ".bias"], **kw)
    h = conv("encoder.conv_in", x.to(dtype), padding=1)
    for _, resnets, down in arch.vae_encoder_blocks(cfg):
        # DownEncoderBlock2D (unet_2d_blocks.py:1032-1086): resnets with temb None, then Downsample2D(padding=0), which pads
        # the bottom and right edge by one before its 3x3 stride-2 conv (resnet.py:199,213-217)
        for p, _, _ in resnets:
            h = resnet_block(sd, p, h, None, g, eps)
        if down:
            h = conv(down, F.pad(h, (0, 1, 0, 1)), stride=2)
    # UNetMidBlock2D (unet_2d_blocks.py:395-473): resnet, single-head attention with GroupNorm and residual, resnet
    h = resnet_block(sd, "encoder.mid_block.resnets.0", h, None, g, eps)
    a = "encoder.mid_block.attentions.0"
    b, c, hh, ww = h.shape
    t = F.group_norm(h.reshape(b, c, hh * ww), g, sd[a + ".group_norm.weight"], sd[a + ".group_norm.bias"], eps).transpose(1, 2)
    q, k, v = (F.linear(t, sd[f"{a}.{n}.weight"], sd[f"{a}.{n}.bias"]) for n in ("to_q", "to_k", "to_v"))
    o = torch.softmax((q @ k.transpose(1, 2)).float() * c ** -0.5, dim=-1).to(dtype) @ v
    h = h + F.linear(o, sd[a + ".to_out.0.weight"], sd[a + ".to_out.0.bias"]).transpose(1, 2).reshape(b, c, hh, ww)
    h = resnet_block(sd, "encoder.mid_block.resnets.1", h, None, g, eps)
    # conv_norm_out, SiLU, conv_out (vae.py:144-147), then quant_conv (autoencoder_kl.py:165-166)
    h = F.silu(F.group_norm(h, g, sd["encoder.conv_norm_out.weight"], sd["encoder.conv_norm_out.bias"], eps))
    h = conv("encoder.conv_out", h, padding=1)
    return conv("quant_conv", h)


def posterior(moments: torch.Tensor):
    """DiagonalGaussianDistribution.__init__ (vae.py:398-408): (mean, logvar clamped to [-30, 20], std, var)."""
    mean, logvar = torch.chunk(moments, 2, dim=1)
    logvar = logvar.clamp(-30.0, 20.0)
    return mean, logvar, torch.exp(0.5 * logvar), torch.exp(logvar)


def sample(moments: torch.Tensor, generator: torch.Generator) -> torch.Tensor:
    """DiagonalGaussianDistribution.sample (vae.py:410-416) with randn_tensor's rule (utils/torch_utils.py:36-77): a CPU
    generator draws on the CPU in the moments' dtype, then the noise moves to their device."""
    mean, _, std, _ = posterior(moments)
    noise = torch.randn(mean.shape, generator=generator, device=generator.device, dtype=moments.dtype).to(moments.device)
    return mean + std * noise


def encode_latents(sd, cfg: arch.VaeConfig, pixel_values: torch.Tensor, dtype=torch.float32) -> torch.Tensor:
    """The given-view demo's three lines (run_cond_on_view.py:80-85): (b, n_cam, 3, H, W) -> latent_dist.mean *
    scaling_factor, (b, n_cam, latent_channels, H/8, W/8)."""
    b, n = pixel_values.shape[:2]
    m = vae_encode_moments(sd, cfg, pixel_values.reshape(b * n, *pixel_values.shape[2:]), dtype)
    mean = m[:, : cfg.latent_channels] * cfg.scaling_factor
    return mean.reshape(b, n, *mean.shape[1:])
