"""Host logic of pipeline.BEVControlNetDenoiser on CPU: scheduler tables (DDIM / UniPC), multistep history handling, the two
given-view modes, call ordering -- checked against fixtures produced by the REFERENCE pipelines themselves.

There is no GPU in the build container and the product has no CPU path, so the operators the denoiser launches run on
their torch restatements (tests/ops_emulator.py) and the CUDA engines are replaced by stand-ins whose arithmetic is the
oracle's (the same stand-ins as tests/test_dropin_reference_pipeline_cpu.py).  The real kernels are compared with the same fixtures in
tests/test_model_gpu.py and tests/test_zz_sampling_gpu.py."""
from dataclasses import asdict

import pytest
import torch

from magicdrive_b200 import models
from magicdrive_b200.pipeline import BEVControlNetDenoiser
from tests import ops_emulator
from tests.common import golden, tiny_configs, tiny_state_dicts
from tests.test_dropin_reference_pipeline_cpu import _FakeControlNetEngine, _FakeUNetEngine


class _UNetEngine(_FakeUNetEngine):
    def time_embed(self, tt):
        return torch.zeros(len(tt), 8)

    def set_view_shard(self, shard):
        assert shard is None


class _ControlNetEngine(_FakeControlNetEngine):
    def time_embed(self, tt):
        return torch.zeros(len(tt), 8)


@pytest.fixture
def cpu_standins(monkeypatch):
    ops_emulator.install(monkeypatch)
    monkeypatch.setattr(models, "UNetEngine", _UNetEngine)
    monkeypatch.setattr(models, "ControlNetEngine", _ControlNetEngine)


def _denoiser(seed, scheduler):
    ucfg, ccfg = tiny_configs()
    usd, csd = tiny_state_dicts(seed)
    un = models.UNet2DConditionModelMultiview(**asdict(ucfg))
    cn = models.BEVControlNetModel(**asdict(ccfg))
    un.load_state_dict(usd)
    cn.load_state_dict(csd)
    pipe = BEVControlNetDenoiser(un, cn, use_cuda_graph=False, overlap_controlnet=False, scheduler=scheduler)
    pipe.fuse_residual_adds = False  # the stand-in engines only restate whole forwards (the fused path: test_engine_host_cpu.py)
    return pipe


def _call(pipe, inp, steps, guidance, **kw):
    return pipe(image=inp["bev_map"], camera_param=inp["camera_param"], prompt_embeds=inp["prompt_embeds"],
                negative_prompt_embeds=inp["negative_prompt_embeds"], latents=inp["latents"], num_inference_steps=steps,
                guidance_scale=guidance, bev_controlnet_kwargs={"bboxes_3d_data": inp["bboxes_3d_data"]}, **kw)


@torch.no_grad()
@pytest.mark.parametrize("fixture,scheduler", [("tiny_pipeline.pt", "ddim"), ("tiny_pipeline_unipc.pt", "unipc")])
def test_denoiser_host_logic_reproduces_reference_pipeline(cpu_standins, fixture, scheduler):
    p = golden(fixture)
    inp = golden(p.get("inputs_from", fixture))["inputs"]
    pipe = _denoiser(p["seed"], scheduler)
    ref = p["latents_out"]
    for _ in range(2):  # the second call reuses the resident state: multistep history must restart
        out = _call(pipe, inp, p["steps"], p["guidance"])
        torch.testing.assert_close(out, ref, rtol=1e-3, atol=3e-4 * ref.abs().max().item())


@torch.no_grad()
@pytest.mark.parametrize("case,scheduler,change", [("ddim_change", "ddim", True), ("ddim_once", "ddim", False),
                                                   ("unipc_change", "unipc", True)])
def test_denoiser_host_logic_reproduces_reference_given_view_pipeline(cpu_standins, case, scheduler, change):
    from oracle.make_golden_given_view import pinned_latents
    p = golden("tiny_given_view.pt")
    inp = golden(p["inputs_from"])["inputs"]
    pipe = _denoiser(p["seed"], scheduler)
    out = _call(pipe, inp, p["steps"], p["guidance"], conditional_latents=pinned_latents(p["pinned_seed"]),
                conditional_latents_change_every_input=change)
    ref = p["outputs"][case]
    torch.testing.assert_close(out, ref, rtol=1e-3, atol=3e-4 * ref.abs().max().item())
    # switching back to plain generation on the same denoiser drops the pinning
    plain = golden("tiny_pipeline.pt" if scheduler == "ddim" else "tiny_pipeline_unipc.pt")
    if plain["steps"] == p["steps"]:
        out = _call(pipe, inp, plain["steps"], plain["guidance"])
        torch.testing.assert_close(out, plain["latents_out"], rtol=1e-3, atol=3e-4 * plain["latents_out"].abs().max().item())


@torch.no_grad()
@pytest.mark.parametrize("case", ["zero_map", "negative1", "max_len9"])
def test_unconditional_map_options_reproduce_the_reference(cpu_standins, case):
    """use_zero_map_as_unconditional (pipeline_bev_controlnet.py:296-300) and a ControlNet configured with
    use_uncond_map='negative1' (unet_addon_rawbox.py:188-202, 676-679), fixtures from the reference pipeline."""
    from oracle import torch_oracle as O
    p = golden("tiny_uncond_map.pt")
    inp = golden(p["inputs_from"])["inputs"]
    ucfg, ccfg = tiny_configs()
    usd, csd = tiny_state_dicts(p["seed"])
    un = models.UNet2DConditionModelMultiview(**asdict(ucfg))
    extra = dict(use_uncond_map="negative1", drop_cond_ratio=0.25) if case == "negative1" else {}
    cn = models.BEVControlNetModel(**asdict(ccfg), **extra)
    un.load_state_dict(usd)
    if case == "negative1":
        assert "uncond_map" in cn.state_dict() and torch.all(cn.uncond_map == -1)
        csd = dict(csd, uncond_map=cn.uncond_map.clone())
    cn.load_state_dict(csd)
    pipe = BEVControlNetDenoiser(un, cn, use_cuda_graph=False, overlap_controlnet=False)
    pipe.fuse_residual_adds = False  # stand-in engines restate whole forwards only
    opts = dict(use_zero_map_as_unconditional=(case == "zero_map"), bbox_max_length=9 if case == "max_len9" else None)
    out = _call(pipe, inp, p["steps"], p["guidance"], **opts)
    ref = p["outputs"][case]
    torch.testing.assert_close(out, ref, rtol=1e-3, atol=3e-4 * ref.abs().max().item())
    orc = O.denoise_loop(usd, csd, ucfg, ccfg, inp["latents"], inp["prompt_embeds"], inp["negative_prompt_embeds"],
                         inp["camera_param"], inp["bboxes_3d_data"], inp["bev_map"], p["steps"], p["guidance"],
                         **opts)
    torch.testing.assert_close(orc, ref, rtol=1e-3, atol=3e-4 * ref.abs().max().item())
