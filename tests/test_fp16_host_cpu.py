"""Host side of fp16 models on the CPU (operators on their torch restatements, tests/f16_ops_emulator.py): which engines compute
in fp16, the rejected combinations, engine rebuilds on a dtype change, and the tiny denoiser in fp16 against the oracle."""
from dataclasses import asdict

import pytest
import torch

from magicdrive_b200 import engine, models
from magicdrive_b200.pipeline import BEVControlNetDenoiser
from oracle import torch_oracle as O
from tests import f16_ops_emulator
from tests.common import golden, rel_l2, tiny_configs, tiny_state_dicts

F16, BF16 = torch.float16, torch.bfloat16


@pytest.fixture
def emulated(monkeypatch):
    f16_ops_emulator.install(monkeypatch)


def _models(seed=7, dtype=None):
    ucfg, ccfg = tiny_configs()
    usd, csd = tiny_state_dicts(seed)
    un = models.UNet2DConditionModelMultiview(**asdict(ucfg))
    cn = models.BEVControlNetModel(**asdict(ccfg))
    un.load_state_dict(usd)
    cn.load_state_dict(csd)
    if dtype is not None:
        un, cn = un.to(dtype), cn.to(dtype)
    return un, cn


def test_storage_dtype_rule():
    un, _ = _models()
    sd = un.state_dict()
    assert engine.storage_dtype(sd) == BF16  # fp32 parameters: today's bf16 path
    assert engine.storage_dtype({k: v.half() for k, v in sd.items()}) == F16
    assert engine.storage_dtype({k: v.bfloat16() for k, v in sd.items()}) == BF16
    mixed = {k: v.half() for k, v in sd.items()}
    mixed[next(iter(mixed))] = mixed[next(iter(mixed))].float()
    assert engine.storage_dtype(mixed) == BF16  # fp16 only when every floating tensor is
    assert un.storage_dtype() == BF16 and un.half().storage_dtype() == F16


def test_engines_take_the_module_dtype(emulated):
    un, cn = _models(dtype=F16)
    eu, ec = un.engine(), cn.engine()
    assert eu.dtype == ec.dtype == F16 and eu.W.fold_dtype == F16
    w, _ = eu.W.lin("down_blocks.0.attentions.0.transformer_blocks.0.attn1.to_out.0")
    assert w.dtype == F16
    assert eu.W.conv_k_padded("conv_in", 64)[0].dtype == F16
    un2, _ = _models()
    assert un2.engine().dtype == BF16 and un2.engine().W.lin("time_embedding.linear_1")[0].dtype == BF16


def test_dtype_change_rebuilds_the_engine():
    un, _ = _models(dtype=F16)
    assert un.storage_dtype() == F16
    un._engine = object()  # a built engine
    un.to(BF16)
    assert un._engine is None and un.storage_dtype() == BF16
    un.to(F16)
    assert un.storage_dtype() == F16


def test_mixed_dtypes_and_view_shard_raise():
    un, cn = _models(dtype=F16)
    with pytest.raises(ValueError, match="fp16"):
        BEVControlNetDenoiser(un, _models()[1])
    with pytest.raises(ValueError, match="view-sharded"):
        BEVControlNetDenoiser(un, cn, view_shard=object())
    pipe = BEVControlNetDenoiser(un, cn, use_cuda_graph=False)
    cn.to(BF16)  # the modules change dtype after the denoiser was built: the next call refuses
    inp = golden("tiny_pipeline.pt")["inputs"]
    with pytest.raises(ValueError, match="fp16"):
        pipe.prepare(inp["latents"], inp["prompt_embeds"], inp["negative_prompt_embeds"], inp["camera_param"],
                     inp["bboxes_3d_data"], inp["bev_map"])


@torch.no_grad()
@pytest.mark.parametrize("scheduler", ["ddim", "unipc"])
def test_tiny_denoiser_fp16_against_the_oracle(emulated, scheduler):
    """The real engines in fp16 (activations rounded to fp16 by the restated operators) over 3 CFG steps, against the fp32
    oracle loop: within fp16 noise, and well inside the same run in bf16 storage."""
    p = golden("tiny_pipeline.pt")
    inp = p["inputs"]
    ucfg, ccfg = tiny_configs()
    usd, csd = tiny_state_dicts(p["seed"])
    truth = O.denoise_loop(usd, csd, ucfg, ccfg, inp["latents"], inp["prompt_embeds"], inp["negative_prompt_embeds"],
                           inp["camera_param"], inp["bboxes_3d_data"], inp["bev_map"], 3, p["guidance"], scheduler=scheduler)
    un, cn = _models(p["seed"], F16)
    pipe = BEVControlNetDenoiser(un, cn, use_cuda_graph=False, overlap_controlnet=False, scheduler=scheduler)
    out = pipe(image=inp["bev_map"], camera_param=inp["camera_param"], prompt_embeds=inp["prompt_embeds"],
               negative_prompt_embeds=inp["negative_prompt_embeds"], latents=inp["latents"], num_inference_steps=3,
               guidance_scale=p["guidance"], bev_controlnet_kwargs={"bboxes_3d_data": inp["bboxes_3d_data"]})
    assert un.engine().dtype == F16
    e = rel_l2(out, truth)
    assert e < 3e-3, e
