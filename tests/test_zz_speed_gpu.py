"""GPU-reference timing (SURVEY.md §8d-i): the reference's arithmetic for one CFG scene-step -- the oracle restatement
in bf16 on torch's own CUDA kernels (cuDNN convolutions, cuBLAS GEMMs, F.scaled_dot_product_attention like the reference's
AttnProcessor2_0) -- timed on the same GPU next to this repo's path.  The reference itself cannot travel to the GPU box
and its vendored xformers only dispatches below compute capability 9.0 (SURVEY.md §0.4), so this is the stand-in for
"the reference's CUDA path on 1xH100".  Named test_zz_* so that it runs after the parity tests; the oracle is only the thing compared with."""
import sys
import os
from dataclasses import asdict

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from magicdrive_b200 import arch  # noqa: E402
from magicdrive_b200.models import BEVControlNetModel, UNet2DConditionModelMultiview  # noqa: E402
from magicdrive_b200.pipeline import BEVControlNetDenoiser  # noqa: E402
from magicdrive_b200.synthetic import synthetic_inputs  # noqa: E402
from oracle import torch_oracle as O  # noqa: E402  (baseline being timed, never the product path)

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module")
def cuda_lib():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from magicdrive_b200 import _lib
    return _lib.lib()


def _ms(fn, iters):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


@torch.no_grad()
def test_scene_step_time_vs_torch_eager_reference_arithmetic(cuda_lib, monkeypatch):
    ucfg, ccfg = arch.UNetConfig(), arch.ControlNetConfig()
    un = UNet2DConditionModelMultiview(**asdict(ucfg)).reset_parameters_synthetic(11).to(DEV, torch.bfloat16)
    cn = BEVControlNetModel(**asdict(ccfg)).reset_parameters_synthetic(12).to(DEV, torch.bfloat16)
    inp = synthetic_inputs(1, 6, 28, 50, n_box=20, map_hw=200, seed=2)
    # ---- ours: the denoiser, CUDA graph + two-stream overlap (bench.py's device-timed loop)
    den = BEVControlNetDenoiser(un, cn)
    st = den.prepare(inp["latents"], inp["prompt_embeds"], inp["negative_prompt_embeds"], inp["camera_param"],
                     inp["bboxes_3d_data"], inp["bev_map"], guidance_scale=2.0)
    den.set_schedule(st, 50)
    den.run_steps(st, 0, 3)
    step = [3]

    def ours():
        den.run_steps(st, step[0] % 50, step[0] % 50 + 1)
        step[0] += 1
    ms_ours = _ms(ours, 20)
    # ---- the reference's arithmetic on torch kernels, bf16, CFG batch of 12 view-samples, SDPA attention
    monkeypatch.setattr(O, "USE_SDPA", True)
    usd = {k: v.detach() for k, v in un.state_dict().items()}
    csd = {k: v.detach() for k, v in cn.state_dict().items()}
    bf = torch.bfloat16
    cam, boxes = O.add_uncond_to_kwargs(csd, ccfg, inp["camera_param"].to(DEV, bf),
                                        {k: (v.to(DEV, bf) if v.is_floating_point() else v.to(DEV)) for k, v in inp["bboxes_3d_data"].items()})
    text = torch.cat([inp["negative_prompt_embeds"], inp["prompt_embeds"]]).to(DEV, bf)
    image = torch.cat([inp["bev_map"]] * 2).to(DEV, bf)
    lat = torch.stack([inp["latents"]] * 6, 1).to(DEV, bf)
    lat2 = torch.cat([lat] * 2)
    t = torch.full((2,), 601, device=DEV, dtype=torch.int64)

    def reference():
        down, mid, ctx = O.controlnet_forward(csd, ccfg, lat2, t, cam, boxes, text, image)
        eps = O.unet_forward(usd, ucfg, lat2.reshape(-1, 4, 28, 50), t[0], ctx, down, mid)
        eu, ec = eps.chunk(2)
        return eu + 2.0 * (ec - eu)
    ms_ref = _ms(reference, 5)
    from tests.common import record
    record(f"[speed] 6-view 224x400 CFG scene-step on this GPU: ours {ms_ours:.2f} ms ({1e3 / ms_ours:.1f} scene-steps/s), "
          f"reference arithmetic on torch bf16 kernels (eager, SDPA) {ms_ref:.2f} ms ({1e3 / ms_ref:.1f} scene-steps/s), "
          f"ratio {ms_ref / ms_ours:.2f}x")
    assert ms_ours < ms_ref
