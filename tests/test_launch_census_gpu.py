"""The launch census (tests/launch_census.py) of the product's forwards at SD-1.5 size, in every storage type each supports:
every operator call of the denoising step (prepare + one CFG step), of the VAE's decode_latents and encode_latents, of the
CLIP text encoder and of the FID Inception network, checked in place under guard bands against float64 by the criterion the
kernel tests state for that operator, with every launch accounted for.

The forwards run eagerly on one stream so that each call can be checked on its own.  That this is the arithmetic the product
runs is held separately: the eager single-stream step is bitwise equal to the product's step (CUDA graph replay with the
ControlNet on a second stream) on the same inputs.

Each workload records its census (tests/common.record, launch_census_gpu_latest.txt): launches, distinct signatures with the
launch count and worst err/tol of each, the planner's tiling of every GEMM, and the worst ratio per operator family."""
import time
from dataclasses import asdict

import pytest
import torch

pytestmark = pytest.mark.gpu

from magicdrive_b200 import arch, models  # noqa: E402
from magicdrive_b200.models import AutoencoderKL, BEVControlNetModel, UNet2DConditionModelMultiview  # noqa: E402
from magicdrive_b200.pipeline import BEVControlNetDenoiser  # noqa: E402
from magicdrive_b200.synthetic import synthetic_inputs  # noqa: E402
from tests.common import golden, record  # noqa: E402
from tests.launch_census import Census  # noqa: E402

DEV = "cuda"
BF16, F16 = torch.bfloat16, torch.float16
DTS = [pytest.param(BF16, id="bf16"), pytest.param(F16, id="f16")]
LOG = "launch_census_gpu_latest.txt"


@pytest.fixture(autouse=True)
def _no_tf32():
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
    torch.cuda.empty_cache()


def _census(name, run):
    """run() under a census; records the census and returns run()'s result."""
    t0 = time.perf_counter()
    with Census() as c:
        res = run()
    secs = time.perf_counter() - t0
    record(f"[census] {name}: {c.total} launches ({c.counted} checked, {c.exempt} exempt, {c.unaccounted} unaccounted), "
           f"{len(c.rows)} distinct signatures, {secs:.1f} s with the float64 checks", LOG)
    for line in c.table():
        record(f"[census] {name}  {line}", LOG)
    c.assert_clean()
    return res


# ------------------------------------------------------------------------------------------------ denoising step
# name: (latent h, latent w, BEV map size, map_embedding_size (the Plus map encoder) or None)
STEPS = {"224x400": (28, 50, 200, None), "272x736": (34, 92, 200, (34, 92)), "424x800": (53, 100, 400, None)}


def _step(un, cn, inp, *, graph, overlap, capacity):
    """prepare + one CFG step (DDIM, 20-step schedule) -> the updated latents."""
    pipe = BEVControlNetDenoiser(un, cn, use_cuda_graph=graph, overlap_controlnet=overlap, box_capacity=capacity)
    st = pipe.prepare(inp["latents"], inp["prompt_embeds"], inp["negative_prompt_embeds"], inp["camera_param"],
                      inp["bboxes_3d_data"], inp["bev_map"], guidance_scale=2.0)
    pipe.set_schedule(st, 20)
    pipe.run_steps(st, 0, 1)
    torch.cuda.synchronize()
    return st["latents"].clone()


# every size in both storage types, and once more at 224x400 with a box capacity (the attention reads its key count from
# the device)
STEP_CASES = ([pytest.param(r, dt, None, id=f"{r}-{i}") for r in STEPS for dt, i in ((BF16, "bf16"), (F16, "f16"))] +
              [pytest.param("224x400", dt, 32, id=f"224x400-{i}-capacity32") for dt, i in ((BF16, "bf16"), (F16, "f16"))])


@torch.no_grad()
@pytest.mark.parametrize("res,dt,capacity", STEP_CASES)
def test_census_step(cuda_lib, res, dt, capacity):
    """The step's launches (camera / box / map encoders, time embedding, ControlNet, UNet, guidance + DDIM update).  Then
    the same step as the product runs it, bit for bit."""
    h, w, mhw, emb = STEPS[res]
    ucfg = arch.UNetConfig()
    ccfg = arch.ControlNetConfig(map_size=(8, mhw, mhw), **({"map_embedding_size": emb} if emb else {}))
    un = UNet2DConditionModelMultiview(**asdict(ucfg)).reset_parameters_synthetic(11).to(DEV, dt)
    cn = BEVControlNetModel(**asdict(ccfg)).reset_parameters_synthetic(12).to(DEV, dt)
    inp = synthetic_inputs(1, 6, h, w, n_box=20, map_hw=mhw, seed=0)
    name = f"step {res} {str(dt)[6:]}" + ("" if capacity is None else f" box_capacity={capacity}")
    eager = _census(name, lambda: _step(un, cn, inp, graph=False, overlap=False, capacity=capacity))
    product = _step(un, cn, inp, graph=True, overlap=True, capacity=capacity)
    assert torch.equal(eager, product), "the eager single-stream step differs from the product's graph + overlap step"


# ------------------------------------------------------------------------------------------------ VAE
VAE_CASES = {"224x400x6": (6, 28, 50), "272x736x1": (1, 34, 92), "424x800x6": (6, 53, 100)}  # (views, latent h, latent w)


@torch.no_grad()
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("case", list(VAE_CASES))
def test_census_vae(cuda_lib, case, dt):
    from oracle.make_golden_vae_encode import full_state_dict, images  # checker only: synthetic weights and images
    n, h, w = VAE_CASES[case]
    cfg = arch.VaeConfig()
    vae = AutoencoderKL(**asdict(cfg))
    vae.load_state_dict(full_state_dict(cfg, 17))
    vae = vae.to(DEV, dt)
    vae.use_cuda_graph = False
    lat = torch.randn(1, n, 4, h, w, generator=torch.Generator().manual_seed(h * w)).to(DEV)
    img = _census(f"vae decode_latents {case} {str(dt)[6:]}", lambda: vae.decode_latents(lat))
    assert img.shape == (1, n, 8 * h, 8 * w, 3)
    del img
    torch.cuda.empty_cache()
    pix = images(n, 8 * h, 8 * w, 5).to(DEV).reshape(1, n, 3, 8 * h, 8 * w)
    z = _census(f"vae encode_latents {case} {str(dt)[6:]}", lambda: vae.encode_latents(pix))
    assert z.shape == (1, n, 4, h, w)


# ------------------------------------------------------------------------------------------------ CLIP, FID
@torch.no_grad()
def test_census_clip_text(cuda_lib):
    from oracle.clip_text import draw_weights  # checker only: the synthetic weights
    g = golden("clip_text_sd15.pt")
    cfg = arch.ClipTextConfig(**g["config"])
    m = models.CLIPTextModel(**g["config"])
    m.load_state_dict(draw_weights(cfg, g["seed_weights"]))
    m = m.to(DEV)
    m.use_cuda_graph = False
    ids = torch.randint(0, cfg.vocab_size - 2, (2, 77), generator=torch.Generator().manual_seed(35))
    ids[:, 0], ids[:, 30:] = cfg.vocab_size - 2, cfg.vocab_size - 1  # two 77-token captions: BOS, words, EOS padding
    out = _census("clip text 2x77", lambda: m(ids.to(DEV)))
    assert out.last_hidden_state.shape == (2, 77, cfg.hidden_size)


@torch.no_grad()
def test_census_fid_inception(cuda_lib):
    from oracle import fid_inception  # checker only: the test images
    m = models.InceptionV3([0, 1, 2, 3]).to(DEV)
    m.load_state_dict(arch.inception_synthetic_state_dict(3, seed=3))
    m.use_cuda_graph = False
    x = fid_inception.images(2, 224, 400, seed=2).to(DEV)
    feats = _census("fid inception 2x224x400", lambda: m(x))
    assert len(feats) == 4
