"""Host side of an fp16 AutoencoderKL on the CPU (operators on their torch restatements, tests/f16_ops_emulator.py and
tests/vae_f16_ops_emulator.py, which round to f16 wherever the device writes f16): which VAE engines compute in f16, the f16
packing of their weights and folds, engine and graph-cache rebuilds on a dtype change, the restatement of vae_f16_ops.py, and
the tiny VAE's fp16 decode and encode against the fp32 oracle."""
import inspect
from dataclasses import asdict

import pytest
import torch

from magicdrive_b200 import engine, models, ops, vae_f16_ops
from oracle import torch_oracle as O
from oracle import vae_encode as OV
from oracle.make_golden_vae_encode import full_state_dict, images, vae_config
from tests import vae_f16_ops_emulator
from tests.common import rel_l2

F16, BF16, F32 = torch.float16, torch.bfloat16, torch.float32


def _vae(seed=31, dtype=None):
    cfg = vae_config()
    sd = full_state_dict(cfg, seed)
    vae = models.AutoencoderKL(**asdict(cfg))
    vae.load_state_dict(sd)
    return (vae if dtype is None else vae.to(dtype)), cfg, sd


def _cpu_engines(monkeypatch):
    """The module's own engine caching (rebuilt when `_engine` is dropped), with the engine built on the CPU."""
    def get_engine(self, cls_):
        if self._engine is None:
            self._engine = cls_(self.arch_cfg, dict(self.state_dict()), self.device)
        return self._engine
    monkeypatch.setattr(models._B200Module, "_get_engine", get_engine)


@pytest.fixture
def emulated(monkeypatch):
    vae_f16_ops_emulator.install(monkeypatch)
    _cpu_engines(monkeypatch)


# ------------------------------------------------------------------------------------------------ dtype routing
@pytest.mark.parametrize("dtype,expect", [(None, BF16), (BF16, BF16), (F16, F16)], ids=["fp32", "bf16", "fp16"])
def test_vae_engines_take_the_storage_dtype_rule(dtype, expect):
    vae, cfg, _ = _vae(dtype=dtype)
    sd = dict(vae.state_dict())
    dec, enc = engine.VaeDecoderEngine(cfg, sd, "cpu"), engine.VaeEncoderEngine(cfg, sd, "cpu")
    assert dec.dtype == enc.dtype == dec.W.dtype == enc.W.dtype == expect
    assert dec._conv("decoder.mid_block.resnets.0.conv1")[0].dtype == expect
    assert dec._conv("decoder.mid_block.resnets.0.conv1")[1].dtype == F32  # biases stay fp32
    assert dec.W.lin("decoder.mid_block.attentions.0.to_q")[0].dtype == expect
    assert dec.W.conv_n_padded("decoder.conv_out", dec.COUT_PAD)[0].dtype == expect
    assert enc._conv_in()[0].dtype == expect and enc._conv_in()[1].dtype == F32
    wm, bm = enc._conv_out(0.18215)
    assert bm.dtype == F32 and wm.dtype == (F16 if expect == F16 else engine._Weights.fold_dtype)
    wd, bd = dec.W.conv_direct("decoder.conv_in")  # the fp32-weight direct convolution keeps fp32 weights
    assert wd.dtype == bd.dtype == F32


def test_mixed_parameter_dtypes_stay_bf16():
    vae, cfg, _ = _vae(dtype=F16)
    vae.decoder.conv_in.bias.data = vae.decoder.conv_in.bias.data.float()
    sd = dict(vae.state_dict())
    assert engine.storage_dtype(sd) == BF16
    assert engine.VaeDecoderEngine(cfg, sd, "cpu").dtype == BF16 and engine.VaeEncoderEngine(cfg, sd, "cpu").dtype == BF16


def test_folds_are_composed_in_fp32_and_rounded_once_to_f16():
    vae, cfg, sd = _vae(dtype=F16)
    enc = engine.VaeEncoderEngine(cfg, dict(vae.state_dict()), "cpu")
    half = {k: v.half().float() for k, v in sd.items()}
    w, b = half["encoder.conv_out.weight"], half["encoder.conv_out.bias"]
    q, bq = half["quant_conv.weight"][:, :, 0, 0], half["quant_conv.bias"]
    wf, bf = torch.einsum("om,mchw->ochw", q, w), q @ b + bq
    wf[:4] *= 0.5
    bf[:4] *= 0.5
    wm, bm = enc._conv_out(0.5)
    ref = torch.zeros((8, *w.shape[1:]))
    ref[:8] = wf
    assert torch.equal(wm.float().reshape(8, 3, 3, -1)[..., : w.shape[1]], ref.permute(0, 2, 3, 1).half().float())
    assert torch.equal(bm, bf)


def test_dtype_change_rebuilds_both_engines_and_drops_the_graphs(monkeypatch):
    """The module's own engine() / encoder_engine() and graph caches; the engines pack nothing until they run, so they are
    built here with a CUDA device reported and CPU parameters."""
    monkeypatch.setattr(models._B200Module, "device", property(lambda self: torch.device("cuda")))
    vae, _, _ = _vae(dtype=F16)
    d16, e16 = vae.engine(), vae.encoder_engine()
    assert d16.dtype == e16.dtype == F16
    vae._decode_graphs[("stale",)] = object()
    vae._encode_graphs[("stale",)] = object()
    vae.to(BF16)
    d, e = vae.engine(), vae.encoder_engine()
    assert d is not d16 and e is not e16 and d.dtype == e.dtype == BF16
    assert not vae._decode_graphs and not vae._encode_graphs
    vae._decode_graphs[("stale",)] = object()
    vae.to(F16)
    assert vae.engine().dtype == vae.encoder_engine().dtype == F16 and not vae._decode_graphs


# ------------------------------------------------------------------------------------------------ restatement
def _params(fn):
    return [(p.name, p.kind, p.default) for p in inspect.signature(fn).parameters.values()]


def test_emulated_names_are_the_launching_operators():
    launching = {n for n, f in inspect.getmembers(vae_f16_ops, inspect.isfunction)
                 if f.__module__ == vae_f16_ops.__name__ and "_lib.lib()" in inspect.getsource(f)}
    E = vae_f16_ops_emulator.EMULATED
    assert set(E) == launching and len(E) == len(set(E))


@pytest.mark.parametrize("name", vae_f16_ops_emulator.EMULATED)
def test_emulated_signature_equals_vae_f16_ops(name):
    assert _params(getattr(vae_f16_ops_emulator, name)) == _params(getattr(vae_f16_ops, name))


@pytest.mark.parametrize("name", vae_f16_ops_emulator.EMULATED)
def test_bf16_twin_takes_the_same_arguments(name):
    """Each f16 wrapper takes exactly the arguments of its bf16 twin in ops.py."""
    assert _params(getattr(vae_f16_ops, name)) == _params(getattr(ops, name[: -len("_f16")]))


def test_restatements_round_once_to_f16():
    E = vae_f16_ops_emulator
    x = images(2, 7, 9, 1)
    a = E.fid_input_f16(x, nhwc=False, quantize=False, normalize=False)
    assert a.dtype == F16 and a.shape == (2 * 7 * 9, 8) and not a[:, 3:].any()
    assert torch.equal(a[:, :3], x.permute(0, 2, 3, 1).reshape(-1, 3).half())
    s = torch.randn(5, 70) * 4
    p = E.softmax_rows_f16(s, 70, 128)
    assert p.dtype == F16 and torch.equal(p[:, :70], torch.softmax(s, -1).half()) and not p[:, 70:].any()
    xc, wd, b = torch.randn(1, 5, 6, 4), torch.randn(3, 3, 4, 16), torch.randn(16)
    kw = dict(n=1, h=5, w=6, cin=4, cout=16, k=3)
    y32 = E.conv_direct_f16(xc, wd, b, out_f32=True, **kw)
    assert y32.dtype == F32 and torch.equal(E.conv_direct_f16(xc, wd, b, **kw), y32.half())


# ------------------------------------------------------------------------------------------------ tiny VAE in fp16
# rel-L2 bounds against the fp32 oracle run on the fp16-rounded weights: f16 activations (unit roundoff 2^-11 = 4.9e-4)
# through ~30 layers.  Measured on this restatement: decode 4.9e-4 (decode_latents) and 1.1e-3 (decode); encode 1.4e-3 to
# 2.0e-3 (moments and encode_latents, the three input dtypes)
DECODE_BOUND, ENCODE_BOUND = 3e-3, 4e-3


@torch.no_grad()
def test_tiny_vae_fp16_decode_against_the_oracle(emulated):
    vae, cfg, sd = _vae(dtype=F16)
    half = {k: v.half().float() for k, v in sd.items()}
    lat = torch.randn(1, 3, 4, 6, 7, generator=torch.Generator().manual_seed(3))
    imgs = vae.decode_latents(lat)
    assert vae.engine().dtype == F16 and imgs.dtype == F32 and imgs.shape == (1, 3, 48, 56, 3)
    assert imgs.min() >= 0 and imgs.max() <= 1
    e = rel_l2(imgs, O.decode_latents(half, cfg, lat))
    z = lat[0] / cfg.scaling_factor
    out = vae.decode(z.half()).sample
    assert out.dtype == F16
    e2 = rel_l2(out, O.vae_decode(half, cfg, z))
    print(f"[fp16 host] tiny decode rel-L2: decode_latents {e:.3e}, decode {e2:.3e}")
    assert e < DECODE_BOUND and e2 < DECODE_BOUND


@torch.no_grad()
@pytest.mark.parametrize("in_dtype", [F32, F16, BF16])
def test_tiny_vae_fp16_encode_against_the_oracle(emulated, in_dtype):
    vae, cfg, sd = _vae(dtype=F16)
    half = {k: v.half().float() for k, v in sd.items()}
    x = images(2, 50, 70, 2).to(in_dtype)
    dist = vae.encode(x).latent_dist
    assert vae.encoder_engine().dtype == F16 and dist.parameters.dtype == in_dtype
    ref = OV.vae_encode_moments(half, cfg, x.half().float())
    e = rel_l2(dist.parameters, ref)
    pix = images(6, 50, 70, 3).reshape(1, 6, 3, 50, 70).to(in_dtype)
    lat = vae.encode_latents(pix)
    el = rel_l2(lat, OV.encode_latents(half, cfg, pix.half().float()))
    print(f"[fp16 host] tiny encode ({in_dtype}) rel-L2: moments {e:.3e}, encode_latents {el:.3e}")
    assert lat.dtype == F32 and e < ENCODE_BOUND and el < ENCODE_BOUND
