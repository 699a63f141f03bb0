"""AutoencoderKL.encode without a GPU: the encoder's parameter names against the reference, the fp32 oracle
(oracle/vae_encode.py) against the reference's own encode (fixture tests/golden/vae_encode.pt, oracle/make_golden_vae_encode.py,
and directly when the reference tree is present), the real VaeEncoderEngine / AutoencoderKL.encode / encode_latents host code
through tests/ops_emulator.py, and the loading rules of the encoder weights."""
import json
import os
from dataclasses import asdict

import pytest
import torch

from magicdrive_b200 import arch, engine, models
from oracle import ref_shim
from oracle import vae_encode as OV
from oracle.make_golden_vae_encode import CASES, full_state_dict, images, reference_vae, vae_config
from tests import ops_emulator
from tests.common import GOLDEN, rel_l2

needs_ref = pytest.mark.skipif(not ref_shim.available(), reason="needs the reference tree (or its oracle/_ref snapshot)")


def _fixture():
    return torch.load(os.path.join(GOLDEN, "vae_encode.pt"), map_location="cpu", weights_only=False)


def _bf16_exact(sd):
    return {k: v.to(torch.bfloat16).float() for k, v in sd.items()}


@pytest.fixture
def emulated(monkeypatch):
    ops_emulator.install(monkeypatch)
    monkeypatch.setattr(engine._Weights, "fold_dtype", torch.float32)  # the quant_conv fold's algebra to fp32


# ------------------------------------------------------------------------------------------------------------ shapes
@needs_ref
@pytest.mark.parametrize("cfg", [vae_config(), arch.VaeConfig()], ids=["small", "sd15"])
def test_encoder_param_shapes_match_reference(cfg):
    vae = reference_vae(ref_shim.load(), cfg)
    ref = {k: tuple(v.shape) for k, v in vae.state_dict().items() if k.startswith(("encoder.", "quant_conv."))}
    assert dict(arch.vae_encoder_param_shapes(cfg)) == ref


def test_sd15_encoder_tensor_count():
    sh = arch.vae_encoder_param_shapes(arch.VaeConfig())
    assert len(sh) == 108
    assert sum(torch.Size(s).numel() for s in sh.values()) == 34_163_664
    assert sh["encoder.down_blocks.1.resnets.0.conv_shortcut.weight"] == (256, 128, 1, 1)
    assert sh["encoder.conv_out.weight"] == (8, 512, 3, 3) and sh["quant_conv.weight"] == (8, 8, 1, 1)


# ------------------------------------------------------------------------------------------------------------ oracle
@pytest.mark.parametrize("case", list(CASES))
def test_oracle_reproduces_reference_fixture(case):
    fx = _fixture()
    cfg = arch.VaeConfig(block_out_channels=tuple(fx["block_out_channels"]))
    sd = full_state_dict(cfg, fx["seed"])
    c = fx["cases"][case]
    m = OV.vae_encode_moments(sd, cfg, c["x"])
    torch.testing.assert_close(m, c["moments"], rtol=1e-4, atol=1e-5)
    mean, _, std, _ = OV.posterior(m)
    torch.testing.assert_close(mean, c["mean"], rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(std, c["std"], rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(OV.sample(m, torch.Generator().manual_seed(c["sample_seed"])), c["sample"], rtol=1e-4,
                               atol=1e-5)
    # the odd batch floors at every level: 50x70 -> 25x35 -> 12x17 -> 6x8
    assert c["moments"].shape == {"odd": (2, 8, 6, 8), "even": (1, 8, 8, 12)}[case]


@needs_ref
@torch.no_grad()
def test_oracle_and_posterior_match_reference_encode():
    """Reference AutoencoderKL.encode vs the oracle, with quant_conv biases that push two logvar channels past both clamp
    bounds; and our DiagonalGaussianDistribution on the reference's moments vs the reference's own posterior."""
    cfg = vae_config()
    sd = full_state_dict(cfg)
    sd["quant_conv.bias"] = sd["quant_conv.bias"].clone()
    sd["quant_conv.bias"][4] += 60.0
    sd["quant_conv.bias"][5] -= 60.0
    vae = reference_vae(ref_shim.load(), cfg)
    vae.load_state_dict(sd)
    x = images(3, 42, 58, 5)
    ref = vae.encode(x).latent_dist
    m = OV.vae_encode_moments(sd, cfg, x)
    torch.testing.assert_close(m, ref.parameters, rtol=1e-4, atol=1e-5)
    mean, logvar, std, var = OV.posterior(m)
    assert logvar[:, 0].max() == 20.0 and logvar[:, 1].min() == -30.0  # both clamps engaged
    for a, b in ((mean, ref.mean), (logvar, ref.logvar), (std, ref.std), (var, ref.var)):
        torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(OV.sample(m, torch.Generator().manual_seed(9)), ref.sample(torch.Generator().manual_seed(9)),
                               rtol=1e-4, atol=1e-5)
    ours = models.DiagonalGaussianDistribution(ref.parameters)
    for name in ("mean", "logvar", "std", "var"):
        assert torch.equal(getattr(ours, name), getattr(ref, name)), name
    assert torch.equal(ours.mode(), ref.mode())
    assert torch.equal(ours.sample(torch.Generator().manual_seed(3)), ref.sample(torch.Generator().manual_seed(3)))
    assert torch.equal(ours.kl(), ref.kl())
    gens = [torch.Generator().manual_seed(s) for s in (1, 2, 3)]
    gens_ref = [torch.Generator().manual_seed(s) for s in (1, 2, 3)]
    assert torch.equal(ours.sample(gens), ref.sample(gens_ref))


# ------------------------------------------------------------------------------------------------ engine via emulator
@torch.no_grad()
@pytest.mark.parametrize("n,h,w", [(2, 50, 70), (1, 27, 45)])
def test_encoder_engine_through_emulated_operators_matches_the_oracle(emulated, n, h, w):
    cfg = vae_config()
    sd = _bf16_exact(full_state_dict(cfg, 31))
    vae = models.AutoencoderKL(**asdict(cfg))
    vae.load_state_dict(sd)
    x = images(n, h, w, 2)
    dist = vae.encode(x).latent_dist
    ref = OV.vae_encode_moments(sd, cfg, x)
    assert dist.parameters.shape == ref.shape and rel_l2(dist.parameters, ref) < 1e-5
    assert rel_l2(dist.mean, ref[:, :4]) < 1e-5 and rel_l2(dist.std, OV.posterior(ref)[2]) < 1e-5
    assert vae.encode(x, return_dict=False)[0].mean.shape == dist.mean.shape
    pix = images(n * 3, h, w, 3).reshape(n, 3, 3, h, w)
    lat = vae.encode_latents(pix)
    ref_lat = OV.encode_latents(sd, cfg, pix)
    assert lat.shape == ref_lat.shape == (n, 3, 4, *ref.shape[2:]) and rel_l2(lat, ref_lat) < 1e-5


@torch.no_grad()
def test_sd15_encoder_layout_through_emulated_operators(emulated):
    """The SD-1.5 encoder (128/256/512/512, the two channel-changing shortcuts), one small image."""
    cfg = arch.VaeConfig()
    sd = _bf16_exact(arch.synthetic_state_dict(arch.vae_encoder_param_shapes(cfg), 8))
    sd.update(_bf16_exact(arch.synthetic_state_dict(arch.vae_decoder_param_shapes(cfg), 8)))
    vae = models.AutoencoderKL(**asdict(cfg))
    vae.load_state_dict(sd)
    x = images(1, 26, 34, 4)
    out = vae.encode(x).latent_dist.parameters
    ref = OV.vae_encode_moments(sd, cfg, x)
    assert out.shape == ref.shape == (1, 8, 3, 4) and rel_l2(out, ref) < 1e-5


# ------------------------------------------------------------------------------------------------------------ loading
def _sets(cfg):
    return set(arch.vae_encoder_param_shapes(cfg)), set(arch.vae_decoder_param_shapes(cfg))


def test_loading_full_decoder_only_and_partial_state_dicts():
    cfg = vae_config()
    enc, dec = _sets(cfg)
    full = full_state_dict(cfg)
    vae = models.AutoencoderKL(**asdict(cfg))
    # decoder only: exactly today's keys
    vae.load_state_dict({k: full[k] for k in dec})
    assert set(vae.state_dict()) == dec
    # full: the encoder is kept, returned by state_dict() and moved by .to()
    vae.load_state_dict(full)
    got = vae.state_dict()
    assert set(got) == enc | dec and all(torch.equal(got[k], full[k]) for k in full)
    vae = vae.to(torch.bfloat16)
    assert all(v.dtype == torch.bfloat16 for v in vae.state_dict().values())
    vae.load_state_dict(full)  # loads into bf16 parameters like any other load
    # a decoder-only load after a full one drops the encoder again
    vae.load_state_dict({k: full[k] for k in dec})
    assert set(vae.state_dict()) == dec
    with pytest.raises(NotImplementedError, match="encoder"):
        vae.encode(torch.zeros(1, 3, 16, 16))
    # a partial encoder set is ignored and encode names what is missing
    partial = {k: v for k, v in full.items() if k != "encoder.mid_block.attentions.0.to_k.weight"}
    vae.load_state_dict(partial)
    assert set(vae.state_dict()) == dec
    with pytest.raises(NotImplementedError, match=r"1 of them \(encoder\.mid_block\.attentions\.0\.to_k\.weight\)"):
        vae.encode(torch.zeros(1, 3, 16, 16))


def test_loading_pre_017_attention_names_in_the_encoder():
    cfg = vae_config()
    full = full_state_dict(cfg)
    old = dict(full)
    for half in ("encoder", "decoder"):
        for new, name in (("to_q", "query"), ("to_k", "key"), ("to_v", "value"), ("to_out.0", "proj_attn")):
            for leaf in ("weight", "bias"):
                old[f"{half}.mid_block.attentions.0.{name}.{leaf}"] = old.pop(f"{half}.mid_block.attentions.0.{new}.{leaf}")
    vae = models.AutoencoderKL(**asdict(cfg))
    vae.load_state_dict(old)
    got = vae.state_dict()
    assert set(got) == set(full) and all(torch.equal(got[k], full[k]) for k in full)


@pytest.mark.parametrize("which", ["full", "decoder_only"])
def test_from_pretrained_round_trip(tmp_path, which):
    from safetensors.torch import save_file
    cfg = vae_config()
    full = full_state_dict(cfg)
    sd = full if which == "full" else {k: full[k] for k in arch.vae_decoder_param_shapes(cfg)}
    (tmp_path / "config.json").write_text(json.dumps({"_class_name": "AutoencoderKL", "_diffusers_version": "0.17.1",
                                                      **{k: (list(v) if isinstance(v, tuple) else v)
                                                         for k, v in asdict(cfg).items()}}))
    save_file({k: v.contiguous() for k, v in sd.items()}, str(tmp_path / "diffusion_pytorch_model.safetensors"))
    m = models.AutoencoderKL.from_pretrained(str(tmp_path), torch_dtype=torch.bfloat16)
    got = m.state_dict()
    assert set(got) == set(sd) and m.dtype == torch.bfloat16
    assert all(torch.equal(got[k], sd[k].to(torch.bfloat16)) for k in sd)
    assert bool(m._encoder_missing) == (which == "decoder_only")
