"""Models with fp16 parameters compute in fp16 (test_model_gpu.py's criterion with an fp16 yardstick).  At every tap:
  rel-L2(ours fp16 vs fp32 truth) <= 1.0 x rel-L2(reference arithmetic in fp16 vs fp32 truth) + 1e-4, and
  rel-L2(ours fp16) <= 0.5 x rel-L2(ours bf16) + 1e-5  (the arithmetic really is fp16, not bf16).
"Reference arithmetic in fp16" is the oracle restatement run with fp16 weights / activations through torch's CUDA kernels,
built like test_model_gpu._bf16_yardstick."""
from dataclasses import asdict

import pytest
import torch

pytestmark = pytest.mark.gpu

from magicdrive_b200 import arch  # noqa: E402
from magicdrive_b200.models import BEVControlNetModel, UNet2DConditionModelMultiview  # noqa: E402
from magicdrive_b200.pipeline import BEVControlNetDenoiser  # noqa: E402
from oracle import torch_oracle as O  # noqa: E402  (checker only)
from tests.common import golden, record, rel_l2, tiny_configs, tiny_state_dicts, to_dev  # noqa: E402

DEV = "cuda"
F16, BF16 = torch.float16, torch.bfloat16


def _models(ucfg, ccfg, usd, csd, dtype):
    un = UNet2DConditionModelMultiview(**asdict(ucfg))
    cn = BEVControlNetModel(**asdict(ccfg))
    un.load_state_dict(usd)
    cn.load_state_dict(csd)
    return un.to(DEV, dtype), cn.to(DEV, dtype)


def _fp16_yardstick(fn, usd, csd):
    ub = {k: v.to(DEV, F16) for k, v in usd.items()}
    cb = {k: v.to(DEV, F16) for k, v in csd.items()}
    return fn(ub, cb, F16)


def _check(name, ours16, ours_bf, truth, yard):
    e16, ebf, eref = rel_l2(ours16, truth), rel_l2(ours_bf, truth), rel_l2(yard, truth)
    record(f"[parity fp16] {name}: rel-L2 ours fp16 {e16:.3e}  reference-fp16 {eref:.3e}  ours bf16 {ebf:.3e}")
    assert e16 <= eref + 1e-4, (name, e16, eref)
    assert e16 <= 0.5 * ebf + 1e-5, (name, e16, ebf)


def _forward(un, cn, lat5, t, inp, h, w, dt):
    down, mid, ctx = cn(lat5.to(dt), t, inp["camera_param"], inp["bboxes_3d_data"], inp["prompt_embeds"], inp["bev_map"],
                        return_dict=False)
    eps = un(lat5.reshape(-1, 4, h, w).to(dt), t[0], encoder_hidden_states=ctx, down_block_additional_residuals=down,
             mid_block_additional_residual=mid).sample
    return down, mid, ctx, eps


def _yard_fn(ucfg, ccfg, lat5, t, inp, h, w):
    def yard(ub, cb, dt):
        l5 = lat5.to(dt)
        d, m, c = O.controlnet_forward(cb, ccfg, l5, t, inp["camera_param"].to(dt), to_dev(inp["bboxes_3d_data"], DEV, dt),
                                       inp["prompt_embeds"].to(dt), inp["bev_map"].to(dt))
        return d, m, c, O.unet_forward(ub, ucfg, l5.reshape(-1, 4, h, w), t[0], c, d, m)
    return yard


@torch.no_grad()
def test_engines_follow_the_parameter_dtype(cuda_lib):
    ucfg, ccfg = tiny_configs()
    usd, csd = tiny_state_dicts(3)
    un, cn = _models(ucfg, ccfg, usd, csd, F16)
    assert un.engine().dtype == cn.engine().dtype == F16
    assert un.engine().W.lin("down_blocks.0.attentions.0.transformer_blocks.0.attn1.to_out.0")[0].dtype == F16
    un.to(BF16)
    assert un.engine().dtype == BF16


@torch.no_grad()
def test_tiny_forward_every_tap(cuda_lib):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    g = golden("tiny_forward.pt")
    ucfg, ccfg = tiny_configs()
    usd, csd = tiny_state_dicts(g["seed"])
    inp = to_dev(g["inputs"], DEV)
    s, n, h, w = g["shape"]
    lat5 = torch.stack([inp["latents"]] * n, 1)
    t = torch.tensor([g["t"]], device=DEV)
    d16, m16, c16, e16 = _forward(*_models(ucfg, ccfg, usd, csd, F16), lat5, t, inp, h, w, F16)
    dbf, mbf, cbf, ebf = _forward(*_models(ucfg, ccfg, usd, csd, BF16), lat5, t, inp, h, w, BF16)
    assert e16.dtype == F16 and all(x.dtype == F16 for x in d16)
    yd, ym, yc, ye = _fp16_yardstick(_yard_fn(ucfg, ccfg, lat5, t, inp, h, w), usd, csd)
    _check("tiny ctx", c16, cbf, g["ctx"], yc)
    for i, (a, b, c, y) in enumerate(zip(d16, dbf, g["down"], yd)):
        _check(f"tiny down[{i}]", a, b, c, y)
    _check("tiny mid", m16, mbf, g["mid"], ym)
    _check("tiny eps", e16, ebf, g["eps"], ye)


@torch.no_grad()
@pytest.mark.parametrize("h,w,map_hw", [(28, 50, 200), (53, 100, 400)])
def test_sd15_forward_every_tap(cuda_lib, h, w, map_hw):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    from oracle.make_golden import synthetic_inputs
    ucfg, ccfg = arch.UNetConfig(), arch.ControlNetConfig(map_size=(8, map_hw, map_hw))
    usd = arch.synthetic_state_dict(arch.unet_param_shapes(ucfg), 11)
    csd = arch.synthetic_state_dict(arch.controlnet_param_shapes(ccfg), 12)
    inp = to_dev(synthetic_inputs(1, 6, h, w, n_box=20, map_hw=map_hw, seed=5), DEV)
    lat5 = torch.stack([inp["latents"]] * 6, 1)
    t = torch.tensor([601], device=DEV)
    outs = {}
    for dt in (F16, BF16):
        un, cn = _models(ucfg, ccfg, usd, csd, dt)
        outs[dt] = _forward(un, cn, lat5, t, inp, h, w, dt)
        del un, cn
    d32, m32, c32 = O.controlnet_forward({k: v.to(DEV) for k, v in csd.items()}, ccfg, lat5, t, inp["camera_param"],
                                         inp["bboxes_3d_data"], inp["prompt_embeds"], inp["bev_map"])
    e32 = O.unet_forward({k: v.to(DEV) for k, v in usd.items()}, ucfg, lat5.reshape(-1, 4, h, w), t[0], c32, d32, m32)
    if (h, w) == (28, 50):  # the reference's own output of this step
        gs = golden("sd15_forward.pt")
        cs = gs["ch_step"]
        assert rel_l2(outs[F16][3], gs["eps"]) <= 0.5 * rel_l2(outs[BF16][3], gs["eps"]) + 1e-5
        assert rel_l2(outs[F16][0][0][:, ::cs], gs["down0"]) <= 0.5 * rel_l2(outs[BF16][0][0][:, ::cs], gs["down0"]) + 1e-5
    yd, ym, yc, ye = _fp16_yardstick(_yard_fn(ucfg, ccfg, lat5, t, inp, h, w), usd, csd)
    (d16, m16, c16, e16), (dbf, mbf, cbf, ebf) = outs[F16], outs[BF16]
    _check(f"sd15 {h}x{w} ctx", c16, cbf, c32, yc)
    for i in range(len(d16)):
        _check(f"sd15 {h}x{w} down[{i}]", d16[i], dbf[i], d32[i], yd[i])
    _check(f"sd15 {h}x{w} mid", m16, mbf, m32, ym)
    _check(f"sd15 {h}x{w} eps", e16, ebf, e32, ye)


@torch.no_grad()
@pytest.mark.parametrize("scheduler,capacity", [("ddim", None), ("unipc", None), ("ddim", 32)])
def test_sd15_three_step_cfg_loop(cuda_lib, scheduler, capacity):
    """The benchmarked configuration (CUDA graph + two-stream overlap, fused residual adds) in fp16 for 3 steps, against the
    fp32 oracle loop; once with a box capacity (resident K/V buffers, device key counts)."""
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    from magicdrive_b200.synthetic import synthetic_inputs
    ucfg, ccfg = arch.UNetConfig(), arch.ControlNetConfig()
    usd = arch.synthetic_state_dict(arch.unet_param_shapes(ucfg), 11)
    csd = arch.synthetic_state_dict(arch.controlnet_param_shapes(ccfg), 12)
    inp = synthetic_inputs(1, 6, 28, 50, n_box=20, map_hw=200, seed=0)
    outs = {}
    for dt in (F16, BF16):
        un, cn = _models(ucfg, ccfg, usd, csd, dt)
        pipe = BEVControlNetDenoiser(un, cn, use_cuda_graph=True, overlap_controlnet=True, scheduler=scheduler,
                                     box_capacity=capacity)
        outs[dt] = pipe(image=inp["bev_map"], camera_param=inp["camera_param"], prompt_embeds=inp["prompt_embeds"],
                        negative_prompt_embeds=inp["negative_prompt_embeds"], latents=inp["latents"], num_inference_steps=3,
                        guidance_scale=2.0, bev_controlnet_kwargs={"bboxes_3d_data": inp["bboxes_3d_data"]})
        del pipe, un, cn
    di = to_dev(inp, DEV)

    def loop(usd_, csd_, dt):
        d = to_dev(di, DEV, dt)
        return O.denoise_loop(usd_, csd_, ucfg, ccfg, d["latents"], d["prompt_embeds"], d["negative_prompt_embeds"],
                              d["camera_param"], d["bboxes_3d_data"], d["bev_map"], 3, 2.0, scheduler=scheduler)
    truth = loop({k: v.to(DEV) for k, v in usd.items()}, {k: v.to(DEV) for k, v in csd.items()}, torch.float32)
    yard = _fp16_yardstick(loop, usd, csd)
    _check(f"sd15 3-step CFG loop {scheduler} capacity={capacity}", outs[F16], outs[BF16], truth, yard)
