"""Drop-in boundary check: our modules are placed inside the REFERENCE's own StableDiffusionBEVControlNetPipeline
(imported through oracle/ref_shim.py) and its unmodified `__call__` drives them: CFG batching, add_uncond_to_kwargs,
uncond_cam_param, the 5-D / 4-D reshapes, `.sample`, `return_dict=False` tuples, `.config.in_channels`, `.dtype`.

There is no GPU in the build container and the product has no CPU path, so for THIS test the CUDA engines are replaced by
oracle-backed stand-ins (NHWC in / NHWC out, like the real engines) and the layout / dtype operators the module wrappers
call run on their torch restatements (tests/ops_emulator.py).  What is exercised is the host logic of magicdrive_b200.models against the reference pipeline; the
arithmetic of the real engines is covered by tests/test_model_gpu.py.  Skipped when /root/reference is absent."""
from dataclasses import asdict

import pytest
import torch

from magicdrive_b200 import models
from oracle import ref_shim
from oracle import torch_oracle as O
from tests import ops_emulator
from tests.common import golden, tiny_configs, tiny_state_dicts

pytestmark = pytest.mark.skipif(not ref_shim.available(), reason="reference tree not mounted")


class _FakeUNetEngine:
    CIN_PAD, COUT_PAD = 64, 8

    def __init__(self, cfg, sd, device):
        self.cfg, self.sd = cfg, {k: v.float() for k, v in sd.items()}

    def context_kv(self, ctx_bf16):
        return {"ctx": ctx_bf16.float()}

    def forward(self, latents_pad, n, h, w, t_f32, ctx_kv, lc, down_res=None, mid_res=None, temb_all=None):
        x = latents_pad[:, :4].float().reshape(n, h, w, 4).permute(0, 3, 1, 2)
        ctx = ctx_kv["ctx"].reshape(n, lc, -1)

        def nchw(t, c):
            hw = t.shape[0] // n
            hh = {h * w: (h, w)}.get(hw)
            if hh is None:  # lower resolutions: recover (h', w') from the conv arithmetic
                hh, ww = h, w
                while hh * ww != hw:
                    hh, ww = (hh + 2 - 3) // 2 + 1, (ww + 2 - 3) // 2 + 1
                hh = (hh, ww)
            return t.float().reshape(n, hh[0], hh[1], c).permute(0, 3, 1, 2)
        down = None if down_res is None else [nchw(d, d.shape[1]) for d in down_res]
        mid = None if mid_res is None else nchw(mid_res, mid_res.shape[1])
        eps = O.unet_forward(self.sd, self.cfg, x, t_f32, ctx, down, mid)
        out = torch.zeros(n * h * w, 8)
        out[:, :4] = eps.permute(0, 2, 3, 1).reshape(-1, 4)
        return out


class _FakeControlNetEngine:
    CIN_PAD = 64

    def __init__(self, cfg, sd, device):
        self.cfg, self.sd = cfg, {k: v.float() if v.is_floating_point() else v for k, v in sd.items()}

    def context(self, camera_param, boxes, text):
        ctx = O.controlnet_context(self.sd, self.cfg, camera_param.float(), boxes, text.float())
        return ctx.reshape(-1, ctx.shape[2], ctx.shape[3])

    def context_kv(self, ctx_bf16):
        return {"ctx": ctx_bf16.float()}

    def map_embedding(self, cond):
        return O.map_encode(self.sd, self.cfg, cond.float()).permute(0, 2, 3, 1).contiguous()

    def forward(self, latents_pad, n, h, w, t_f32, ctx_kv, lc, map_emb_per_view, conditioning_scale=1.0, temb_all=None):
        x = latents_pad[:, :4].float().reshape(n, h, w, 4).permute(0, 3, 1, 2)
        ctx = ctx_kv["ctx"].reshape(n, lc, -1)
        emb = O.time_embedding(self.sd, O.timestep_embedding(t_f32, self.cfg.block_out_channels[0]))
        x = O._conv(self.sd, "conv_in", x) + map_emb_per_view.float().permute(0, 3, 1, 2)
        xm, skips = O._encoder(self.sd, self.cfg, x, emb, ctx, False, None)
        F = torch.nn.functional
        down = [F.conv2d(s, self.sd[f"controlnet_down_blocks.{i}.weight"], self.sd[f"controlnet_down_blocks.{i}.bias"])
                * conditioning_scale for i, s in enumerate(skips)]
        mid = F.conv2d(xm, self.sd["controlnet_mid_block.weight"], self.sd["controlnet_mid_block.bias"]) * conditioning_scale

        class FM:
            def __init__(s, t):
                s.n, s.c, s.h, s.w = t.shape
        flat = lambda t: t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])
        return [flat(d) for d in down], flat(mid), [FM(s) for s in skips], FM(xm)


@pytest.fixture
def cpu_standins(monkeypatch):
    ops_emulator.install(monkeypatch)
    monkeypatch.setattr(models, "UNetEngine", _FakeUNetEngine)
    monkeypatch.setattr(models, "ControlNetEngine", _FakeControlNetEngine)


@torch.no_grad()
def test_modules_run_inside_the_reference_pipeline(cpu_standins):
    R = ref_shim.load()
    g = golden("tiny_pipeline.pt")
    ucfg, ccfg = tiny_configs()
    usd, csd = tiny_state_dicts(g["seed"])
    un = models.UNet2DConditionModelMultiview(**asdict(ucfg))
    cn = models.BEVControlNetModel(**asdict(ccfg))
    un.load_state_dict(usd)
    cn.load_state_dict(csd)

    class Pipe(R.StableDiffusionBEVControlNetPipeline):
        def prepare_extra_step_kwargs(self, generator, eta):  # DDIM eta = 0 (SURVEY.md §0.3)
            return {"eta": eta}

    class TextStub(torch.nn.Module):
        dtype = torch.float32

        def __init__(self):
            super().__init__()
            self.p = torch.nn.Parameter(torch.zeros(1))

        @property
        def device(self):
            return self.p.device

    vae = R.AutoencoderKL(block_out_channels=[32, 64, 64, 64], down_block_types=["DownEncoderBlock2D"] * 4,
                          up_block_types=["UpDecoderBlock2D"] * 4, latent_channels=4)
    sched = R.DDIMScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False,
                            set_alpha_to_one=False, steps_offset=1)
    pipe = Pipe(vae=vae, text_encoder=TextStub(), unet=un, controlnet=cn, scheduler=sched, tokenizer=None)
    pipe.set_progress_bar_config(disable=True)
    inp = g["inputs"]
    h, w = inp["latents"].shape[-2:]
    out = pipe(prompt=None, image=inp["bev_map"], camera_param=inp["camera_param"], height=h * 8, width=w * 8,
               num_inference_steps=g["steps"], guidance_scale=g["guidance"], latents=inp["latents"].clone(),
               prompt_embeds=inp["prompt_embeds"], negative_prompt_embeds=inp["negative_prompt_embeds"],
               output_type="latent", bev_controlnet_kwargs={"bboxes_3d_data": inp["bboxes_3d_data"]})
    assert out.images.shape == g["latents_out"].shape
    torch.testing.assert_close(out.images, g["latents_out"], rtol=1e-3, atol=3e-4 * g["latents_out"].abs().max().item())
