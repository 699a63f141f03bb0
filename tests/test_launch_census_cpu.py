"""The launch census (tests/launch_census.py) on the CPU: the tiny fp16 denoiser runs one CFG step with every operator on its
torch restatement (tests/vae_f16_ops_emulator.py and the emulators under it), each restated call counting one launch as the
device wrappers do, and so does the tiny fp16 VAE's decode.  A clean step and decode pass with every launch accounted for;
a one-element error planted in one launch, a write one row past one output, and a launch outside the wrappers are each
reported.  The restatements allocate their results through their own module's torch, so the census runs with
guarded_outputs=False here; on the device every result is a guarded buffer."""
import functools
from dataclasses import asdict

import pytest
import torch

from magicdrive_b200 import f16_ops, models, ops, vae_f16_ops
from magicdrive_b200.pipeline import BEVControlNetDenoiser
from oracle.make_golden_vae_encode import full_state_dict, vae_config
from tests import vae_f16_ops_emulator
from tests.common import golden, tiny_configs, tiny_state_dicts
from tests.launch_census import CRITERIA, Census

F16 = torch.float16


def _counting(fn):
    @functools.wraps(fn)
    def counted(*a, **kw):
        ops._launches += 1
        return fn(*a, **kw)
    return counted


def _stats_of_stored(fn):
    """gemm_conv's restatement with its row statistics taken from the stored (f16-rounded) values, as the device takes them
    (f16_ops_emulator sums the unrounded ones)."""
    @functools.wraps(fn)
    def restated(*a, **kw):
        res = fn(*a, **kw)
        if not kw.get("emit_stats"):
            return res
        out, st = res
        x = out.double()
        half = x.shape[1] // 2
        parts = [x[:, :half], x[:, half:]]
        st.data.copy_(torch.stack([torch.stack([p.sum(1), (p * p).sum(1)], -1) for p in parts], 1))
        return res
    return restated


@pytest.fixture
def emulated(monkeypatch):
    vae_f16_ops_emulator.install(monkeypatch)
    monkeypatch.setattr(ops, "gemm_conv", _stats_of_stored(ops.gemm_conv))
    for mod in (ops, f16_ops, vae_f16_ops):
        for name in CRITERIA:
            if hasattr(mod, name):
                monkeypatch.setattr(mod, name, _counting(getattr(mod, name)))


def _step():
    """prepare + the schedule + one eager single-stream CFG step of the tiny fp16 denoiser."""
    p = golden("tiny_pipeline.pt")
    inp = p["inputs"]
    ucfg, ccfg = tiny_configs()
    usd, csd = tiny_state_dicts(p["seed"])
    un, cn = models.UNet2DConditionModelMultiview(**asdict(ucfg)), models.BEVControlNetModel(**asdict(ccfg))
    un.load_state_dict(usd)
    cn.load_state_dict(csd)
    pipe = BEVControlNetDenoiser(un.to(F16), cn.to(F16), use_cuda_graph=False, overlap_controlnet=False)

    def run():
        st = pipe.prepare(inp["latents"], inp["prompt_embeds"], inp["negative_prompt_embeds"], inp["camera_param"],
                          inp["bboxes_3d_data"], inp["bev_map"], guidance_scale=p["guidance"])
        pipe.set_schedule(st, 3)
        pipe.run_steps(st, 0, 1)
        return st["latents"].clone()
    return run


def _decode():
    """decode_latents of the tiny fp16 VAE (its mid-block attention writes into given outputs)."""
    cfg = vae_config()
    vae = models.AutoencoderKL(**asdict(cfg))
    vae.load_state_dict(full_state_dict(cfg, 31))
    vae = vae.to(F16)
    lat = torch.randn(1, 3, 4, 6, 7, generator=torch.Generator().manual_seed(3))
    return lambda: vae.decode_latents(lat)


@torch.no_grad()
def test_clean_step_passes_and_accounts_every_launch(emulated):
    run = _step()
    with Census(guarded_outputs=False) as c:
        lat = run()
    c.assert_clean()
    assert c.unaccounted == 0 and c.counted == c.total > 0
    names = {row[2] for row in c.rows.values()}
    assert {"gemm_conv", "attention", "groupnorm", "linear_small", "cfg_ddim_step", "pack_latents_f16"} <= names, names
    assert torch.isfinite(lat).all()
    # the census hands every result back unchanged: the same step without it
    assert torch.equal(lat, _step()())
    dec = _decode()
    with Census(guarded_outputs=False) as c:
        img = dec()
    c.assert_clean()
    names = {row[2] for row in c.rows.values()}
    assert {"gemm_conv", "softmax_rows_f16", "conv_direct_f16", "groupnorm", "upsample_nearest"} <= names, names
    assert any("out=" in sig for sig in c.rows)
    assert torch.equal(img, _decode()())


@torch.no_grad()
def test_planted_error_is_reported_with_operator_and_signature(emulated, monkeypatch):
    real = ops.gemm_conv
    seen = []

    @functools.wraps(real)
    def off_by_one_element(*a, **kw):
        res = real(*a, **kw)
        out = res[0] if isinstance(res, tuple) else res
        if kw.get("n_out") == 128 and not seen:
            seen.append(kw)
            out.view(-1)[7] += 1.0 + out.abs().max()
        return res
    monkeypatch.setattr(ops, "gemm_conv", off_by_one_element)
    with Census(guarded_outputs=False) as c:
        _step()()
    assert seen and len(c.failures) == 1, c.failures
    sig, msg = c.failures[0]
    assert sig.startswith("gemm_conv(") and "n_out=128" in sig and "err / tol" in msg, (sig, msg)
    with pytest.raises(AssertionError, match="gemm_conv"):
        c.assert_clean()


@torch.no_grad()
def test_guard_write_past_the_output_is_reported(emulated, monkeypatch):
    real = ops.gemm_conv
    seen = []

    @functools.wraps(real)
    def one_row_too_many(*a, **kw):
        res = real(*a, **kw)
        out = kw.get("out")
        if out is not None and out.dim() == 2 and not seen:
            seen.append(kw)
            rows, ld = out.shape[0], out.stride(0)
            out.as_strided((1,), (1,), out.storage_offset() + rows * ld).fill_(1.0)  # first element of the next row
        return res
    monkeypatch.setattr(ops, "gemm_conv", one_row_too_many)
    with Census(guarded_outputs=False) as c:
        _decode()()
    assert seen, "no gemm_conv launch of the decode writes into a given output"
    assert len(c.failures) == 1 and "guard elements overwritten" in c.failures[0][1], c.failures


@torch.no_grad()
def test_unguarded_output_is_reported(emulated):
    """With guarded_outputs on, a result allocated past the `torch` proxy (here: every restated result) is a failure."""
    with Census() as c:
        _step()()
    assert c.failures and all("not guarded buffers" in msg for _, msg in c.failures)


@torch.no_grad()
def test_launch_outside_the_wrappers_fails_the_accounting(emulated):
    def unwrapped_operator():  # an operator the census does not know, launching one kernel
        ops._launches += 1
    run = _step()
    with pytest.raises(AssertionError, match="1 kernel launches outside the census wrappers"):
        with Census(guarded_outputs=False):
            run()
            unwrapped_operator()
