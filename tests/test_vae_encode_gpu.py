"""GPU parity of AutoencoderKL.encode: the end-padded implicit-GEMM convolution (mdb_gemm_conv pad_h_end / pad_w_end) under
guard bands against float64, the whole encoder against the fp32 oracle (oracle/vae_encode.py) and the reference fixture
(tests/golden/vae_encode.pt), encode_latents' CUDA graph, and given-view generation started from camera images.

The encoder's criterion is the project's bf16 one: rel-L2(ours, fp32) <= 1.0 x rel-L2(the oracle run in bf16, fp32) + 5e-4,
on the mean and on the full moments."""
import math
import os
import sys
from dataclasses import asdict

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from magicdrive_b200 import _lib, arch, ops  # noqa: E402
from magicdrive_b200.models import AutoencoderKL, BEVControlNetModel, UNet2DConditionModelMultiview  # noqa: E402
from magicdrive_b200.pipeline import BEVControlNetDenoiser  # noqa: E402
from oracle import torch_oracle as O  # noqa: E402  (checker only)
from oracle import vae_encode as OV  # noqa: E402  (checker only)
from oracle.make_golden_vae_encode import full_state_dict, images, vae_config  # noqa: E402
from tests.common import GOLDEN, golden, record, rel_l2, tiny_configs, tiny_state_dicts  # noqa: E402
from tests.test_kernel_edges_gpu import Guarded, _bf, _close, _gen, _randn  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
F64 = torch.float64


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


# ------------------------------------------------------------------------------------------------ end-padded conv
# name: (n, h, w, c0, c_out, pad_h, pad_w, pad_h_end, pad_w_end, stride)
END_PAD = {
    # the SD-1.5 encoder's three Downsample2D launches at 224x400 and at 424x800
    "down_224x400": (6, 224, 400, 128, 128, 0, 0, 1, 1, 2),
    "down_112x200": (6, 112, 200, 256, 256, 0, 0, 1, 1, 2),
    "down_56x100": (6, 56, 100, 512, 512, 0, 0, 1, 1, 2),
    "down_424x800": (6, 424, 800, 128, 128, 0, 0, 1, 1, 2),
    "down_212x400": (6, 212, 400, 256, 256, 0, 0, 1, 1, 2),
    "down_106x200": (6, 106, 200, 512, 512, 0, 0, 1, 1, 2),
    # odd inputs, K tails (c0 = 8 as conv_in reads the RGB operand, 32 as the small config), one dimension only, end padding
    # on top of symmetric padding, stride 1
    "odd_13x27": (3, 13, 27, 64, 64, 0, 0, 1, 1, 2),
    "odd_25x35_c32": (2, 25, 35, 32, 64, 0, 0, 1, 1, 2),
    "c8_tail": (2, 25, 35, 8, 64, 0, 0, 1, 1, 2),
    "bottom_only": (2, 25, 35, 64, 64, 0, 0, 1, 0, 2),
    "right_only": (2, 25, 35, 64, 128, 0, 0, 0, 1, 2),
    "sym_plus_end_s1": (2, 13, 27, 64, 64, 1, 1, 0, 2, 1),
}
VARIANTS = {"planner": {}, "splitk": dict(force_splits=3), "nosplit": dict(kernel_variant=4)}


def _end_padded_conv(n, h, w, c0, co, ph, pw, eh, ew, stride, seed=0, **kw):
    """One guarded end-padded gemm_conv on random bf16 operands and its float64 reference: F.pad, then the convolution."""
    g = _gen(seed)
    ho, wo = (h + 2 * ph + eh - 3) // stride + 1, (w + 2 * pw + ew - 3) // stride + 1
    a = _bf(_randn(n * h * w, c0, g=g))
    wt = _bf(_randn(co, 3, 3, c0, g=g, scale=1 / math.sqrt(9 * c0)))
    k64 = (c0 + 63) // 64 * 64
    wm = torch.zeros((co, 3, 3, k64), dtype=torch.bfloat16, device=DEV)
    wm[..., :c0] = wt
    b = _randn(co, g=g)
    out = Guarded(n * ho * wo, co)
    ops.gemm_conv(a, wm.reshape(co, -1), n_img=n, h_in=h, w_in=w, c0=c0, lda0=c0, n_out=co, taps=3, stride=stride, pad_h=ph,
                  pad_w=pw, pad_h_end=eh, pad_w_end=ew, bias=b, out=out.out, ldo=co, **kw)
    x = F.pad(a.to(F64).view(n, h, w, c0).permute(0, 3, 1, 2), (pw, pw + ew, ph, ph + eh))
    ref = F.conv2d(x, wt.to(F64).permute(0, 3, 1, 2), stride=stride).permute(0, 2, 3, 1).reshape(-1, co) + b.to(F64)
    return out, ref


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("case", list(END_PAD))
def test_end_padded_conv(cuda_lib, case, variant):
    n, h, w, c0, co, ph, pw, eh, ew, stride = END_PAD[case]
    ho, wo = (h + 2 * ph + eh - 3) // stride + 1, (w + 2 * pw + ew - 3) // stride + 1
    forced = variant == "splitk" and 3 * n * ho * wo * co * 4 <= 64 << 20  # the forced split fits the split-K scratch
    if variant == "splitk" and not forced:
        pytest.skip("the split-K scratch is too small for a forced split at this size (the planner runs it unsplit)")
    before = ops.launch_count()
    out, ref = _end_padded_conv(n, h, w, c0, co, ph, pw, eh, ew, stride, seed=len(case), **VARIANTS[variant])
    assert ops.launch_count() - before == (2 if forced else 1)
    out.check(case)
    _close(out.out, ref, case)


@pytest.mark.parametrize("kw", [dict(pad_h_end=-1), dict(pad_w_end=-3), dict(pad_h_end=130), dict(pad_w_end=128, pad_w=2)],
                         ids=["neg_h", "neg_w", "corner_h", "corner_w"])
def test_end_padding_rejections_launch_nothing(cuda_lib, kw):
    n, h, w, c = 1, 4, 4, 64
    a = torch.ones((n * h * w, c), dtype=torch.bfloat16, device=DEV)
    wm = torch.ones((64, 9 * c), dtype=torch.bfloat16, device=DEV)
    ph, pw = kw.get("pad_h", 0), kw.get("pad_w", 0)
    ho = max((h + 2 * ph + kw.get("pad_h_end", 0) - 3) + 1, 1)
    wo = max((w + 2 * pw + kw.get("pad_w_end", 0) - 3) + 1, 1)
    out = Guarded(n * ho * wo, 64)
    before = ops.launch_count()
    with pytest.raises(_lib.MdbError, match="end padding must not be negative|TMA im2col limits"):
        ops.gemm_conv(a, wm, n_img=n, h_in=h, w_in=w, c0=c, lda0=c, n_out=64, taps=3, stride=1, h_out=ho, w_out=wo, out=out.out,
                      ldo=64, **kw)
    torch.cuda.synchronize()
    assert ops.launch_count() == before
    assert bool((out.buf.view(out.itype) == out.fill).all()), "a rejected descriptor wrote to the output"


# ------------------------------------------------------------------------------------------------ whole encoder
def _vae(cfg, seed):
    sd = full_state_dict(cfg, seed)
    vae = AutoencoderKL(**asdict(cfg))
    vae.load_state_dict(sd)
    return vae.to(DEV), {k: v.to(DEV) for k, v in sd.items()}


def _latent_size(x):
    for _ in range(3):  # three Downsample2D(padding=0): (x + 1 - 3) // 2 + 1
        x = (x - 2) // 2 + 1
    return x


def _criterion(what, ours, truth, yard):
    e, ey = rel_l2(ours, truth), rel_l2(yard, truth)
    record(f"[parity] vae encode {what}: rel-L2 ours {e:.3e} oracle-bf16 {ey:.3e}")
    assert e <= 1.0 * ey + 5e-4, (what, e, ey)


ENCODER_CASES = {  # name: (config, n, H, W, input dtype)
    "small_50x70": (vae_config(), 2, 50, 70, torch.float32),
    "small_27x45_bf16_in": (vae_config(), 3, 27, 45, torch.bfloat16),
    "sd15_224x400": (arch.VaeConfig(), 6, 224, 400, torch.float32),
    "sd15_272x736": (arch.VaeConfig(), 2, 272, 736, torch.float32),
    "sd15_424x800": (arch.VaeConfig(), 6, 424, 800, torch.float32),
}


@torch.no_grad()
@pytest.mark.parametrize("case", list(ENCODER_CASES))
def test_encoder_vs_fp32_oracle(cuda_lib, case):
    cfg, n, h, w, dt = ENCODER_CASES[case]
    vae, sd = _vae(cfg, 17)
    x = images(n, h, w, 5).to(DEV, dt)
    dist = vae.encode(x).latent_dist
    assert dist.parameters.dtype == dt and dist.parameters.shape == (n, 8, _latent_size(h), _latent_size(w))
    truth = OV.vae_encode_moments(sd, cfg, x.float())
    yard = OV.vae_encode_moments(sd, cfg, x.float(), dtype=torch.bfloat16).float()
    _criterion(f"{case} moments", dist.parameters, truth, yard)
    _criterion(f"{case} mean", dist.mean, truth[:, :4], yard[:, :4])
    del truth, yard
    torch.cuda.empty_cache()


@torch.no_grad()
@pytest.mark.parametrize("case", ["odd", "even"])
def test_encoder_vs_reference_fixture(cuda_lib, case):
    fx = torch.load(os.path.join(GOLDEN, "vae_encode.pt"), map_location="cpu", weights_only=False)
    cfg = arch.VaeConfig(block_out_channels=tuple(fx["block_out_channels"]))
    vae, sd = _vae(cfg, fx["seed"])
    c = fx["cases"][case]
    x = c["x"].to(DEV)
    dist = vae.encode(x).latent_dist
    yard = OV.vae_encode_moments(sd, cfg, x, dtype=torch.bfloat16).float()
    _criterion(f"fixture {case} moments", dist.parameters, c["moments"], yard)
    _criterion(f"fixture {case} mean", dist.mean, c["mean"], yard[:, :4])
    g = torch.Generator().manual_seed(c["sample_seed"])
    assert rel_l2(dist.sample(g), c["sample"]) <= rel_l2(OV.sample(yard, torch.Generator().manual_seed(c["sample_seed"])),
                                                         c["sample"]) + 5e-4


@torch.no_grad()
def test_encode_latents_graph_replay_is_bitwise_the_eager_call(cuda_lib):
    # 64 / 128 channels: GroupNorm(32) has an even channel count per group and runs its deterministic single-kernel path
    # (the small config's 32 channels take the two-kernel path, whose float atomics differ in the last bits from run to run)
    cfg = arch.VaeConfig(block_out_channels=(64, 128, 128, 128))
    vae, sd = _vae(cfg, 23)
    pix = images(6, 80, 104, 8).reshape(1, 6, 3, 80, 104).to(DEV)
    first = vae.encode_latents(pix)   # captures the graph
    replay = vae.encode_latents(pix)
    vae.use_cuda_graph = False
    eager = vae.encode_latents(pix)
    assert first.shape == (1, 6, 4, 10, 13) and torch.equal(first, replay) and torch.equal(replay, eager)
    truth = OV.encode_latents(sd, cfg, pix)
    yard = OV.encode_latents(sd, cfg, pix, dtype=torch.bfloat16).float()
    _criterion("encode_latents", eager, truth, yard)
    other = images(6, 80, 104, 9).reshape(1, 6, 3, 80, 104).to(DEV)  # new input, same shape: the same graph, new result
    vae.use_cuda_graph = True
    replay_other = vae.encode_latents(other)
    vae.use_cuda_graph = False
    assert torch.equal(replay_other, vae.encode_latents(other)) and not torch.equal(replay_other, first)


# ------------------------------------------------------------------------------------------------ given view from images
PINNED = (0, 3)


@torch.no_grad()
def test_given_view_from_camera_images(cuda_lib):
    """Images -> encode_latents -> BEVControlNetDenoiser(conditional_latents=...) at the tiny config, 3 CFG steps, against
    the oracle's encode + given-view chain in fp32.  Yardstick: the denoiser's own error (our denoiser fed the fp32 oracle's
    latents) plus how far the oracle's chain moves when it is fed the bf16 oracle's latents."""
    inp = golden("tiny_pipeline.pt")["inputs"]
    ucfg, ccfg = tiny_configs()
    usd, csd = tiny_state_dicts(7)
    un, cn = UNet2DConditionModelMultiview(**asdict(ucfg)), BEVControlNetModel(**asdict(ccfg))
    un.load_state_dict(usd)
    cn.load_state_dict(csd)
    pipe = BEVControlNetDenoiser(un.to(DEV), cn.to(DEV), use_cuda_graph=True, scheduler="ddim")
    cfg = vae_config()
    vae, vsd = _vae(cfg, 29)
    pix = images(6, 80, 104, 12).reshape(1, 6, 3, 80, 104)
    pin = lambda lat: [[lat[0, j] if j in PINNED else None for j in range(6)]]
    kw = dict(image=inp["bev_map"], camera_param=inp["camera_param"], prompt_embeds=inp["prompt_embeds"],
              negative_prompt_embeds=inp["negative_prompt_embeds"], latents=inp["latents"], num_inference_steps=3,
              guidance_scale=2.0, bev_controlnet_kwargs={"bboxes_3d_data": inp["bboxes_3d_data"]})
    ours = pipe(conditional_latents=pin(vae.encode_latents(pix.to(DEV))), **kw)
    cpu_vsd = {k: v.cpu() for k, v in vsd.items()}
    lat32 = OV.encode_latents(cpu_vsd, cfg, pix)
    lat16 = OV.encode_latents(cpu_vsd, cfg, pix, dtype=torch.bfloat16).float()
    chain = lambda lat: O.denoise_loop(usd, csd, ucfg, ccfg, inp["latents"], inp["prompt_embeds"], inp["negative_prompt_embeds"],
                                       inp["camera_param"], inp["bboxes_3d_data"], inp["bev_map"], 3, 2.0,
                                       conditional_latents=pin(lat))
    truth = chain(lat32)
    e = rel_l2(ours, truth)
    e_den = rel_l2(pipe(conditional_latents=pin(lat32.to(DEV)), **kw), truth)
    e_enc = rel_l2(chain(lat16), truth)
    record(f"[parity] given view from images: rel-L2 {e:.3e}; denoiser alone {e_den:.3e}, bf16 encode in the oracle {e_enc:.3e}")
    assert ours.shape == truth.shape and e <= e_den + e_enc + 5e-4
