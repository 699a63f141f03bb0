"""Host side of the denoiser's box-capacity mode (BEVControlNetDenoiser(box_capacity=N)) and of generate_stream on CPU: the
real engines over tests/ops_emulator.py.  A stream of scenes with different box counts through ONE capacity-mode denoiser
must give, scene by scene, what a fresh default-mode denoiser gives on the same inputs, on one resident state.

The emulator's attention masks keys past kv_len with -inf, whose softmax weight is exactly 0, and every other operator
works row by row; the capacity-mode result can still differ from the exact-shape one in the last bits, because the CPU GEMM
behind the context's K/V projection may block a matrix with more rows differently.  Hence 1e-5 relative, not equality."""
from dataclasses import asdict

import pytest
import torch

from magicdrive_b200 import arch, engine, models
from magicdrive_b200.pipeline import BEVControlNetDenoiser
from magicdrive_b200.synthetic import synthetic_inputs
from tests import ops_emulator
from tests.common import rel_l2, tiny_configs

CAP = 7
H, W, MAP = 10, 13, 52


@pytest.fixture
def emulated(monkeypatch):
    ops_emulator.install(monkeypatch)
    monkeypatch.setattr(engine._Weights, "fold_dtype", torch.float32)


def _modules(seed=41):
    ucfg, ccfg = tiny_configs()
    un = models.UNet2DConditionModelMultiview(**asdict(ucfg))
    cn = models.BEVControlNetModel(**asdict(ccfg))
    un.load_state_dict(arch.synthetic_state_dict(arch.unet_param_shapes(ucfg), seed))
    cn.load_state_dict(arch.synthetic_state_dict(arch.controlnet_param_shapes(ccfg), seed + 1))
    return un, cn


def _denoiser(un, cn, scheduler, **kw):
    return BEVControlNetDenoiser(un, cn, use_cuda_graph=False, overlap_controlnet=False, scheduler=scheduler, **kw)


def _scene(n_box, seed):
    """One scene's call arguments; n_box None = no box data at all."""
    inp = synthetic_inputs(1, 6, H, W, n_box=n_box or 0, map_hw=MAP, seed=seed)
    return dict(image=inp["bev_map"], camera_param=inp["camera_param"], prompt_embeds=inp["prompt_embeds"],
                negative_prompt_embeds=inp["negative_prompt_embeds"], latents=inp["latents"],
                bev_controlnet_kwargs={"bboxes_3d_data": inp["bboxes_3d_data"]})


def _resident_ptrs(st):
    ts = [st["latents"], st["t_dev"], st["coef_dev"], st["ctx_len"], st["map"], *st["hist"], *st["inputs"].values(),
          *st["c_kv"].values(), *st["u_kv"].values()]
    return [t.data_ptr() for t in ts]


@torch.no_grad()
@pytest.mark.parametrize("scheduler,guidance", [("ddim", 2.0), ("unipc", 2.0), ("unipc", 1.0)])
def test_stream_of_box_counts_on_one_state_equals_exact_shape_calls(emulated, scheduler, guidance):
    un, cn = _modules()
    cap = _denoiser(un, cn, scheduler, box_capacity=CAP)
    state = ptrs = key = None
    for i, n in enumerate([5, 0, CAP, 1, None, 5]):
        kw = dict(_scene(n, 100 + i), num_inference_steps=3, guidance_scale=guidance)
        out = cap(**kw)
        ref = _denoiser(un, cn, scheduler)(**kw)
        assert out.shape == ref.shape and rel_l2(out, ref) < 1e-5, (n, rel_l2(out, ref))
        st = cap._static
        assert st["ctx_len"].tolist() == [1 + 77 + (n or 0)] * st["V"] and int(st["lc"]) == 1 + 77 + CAP
        assert st["inputs"]["bboxes"].shape[2] == CAP and st["c_kv"]
        if i == 0:
            state, ptrs = st, _resident_ptrs(st)
        else:  # no new state, no new buffer: what a captured graph needs to stay valid
            assert st is state and _resident_ptrs(st) == ptrs
        k = (st["sig"], id(st["latents"]), st["guidance"], st["cond_scale"])  # run_steps' graph key
        key = key or k
        assert k == key


@torch.no_grad()
def test_given_views_in_capacity_mode(emulated):
    un, cn = _modules()
    g = torch.Generator().manual_seed(3)
    pinned = [[torch.randn(4, H, W, generator=g) if v in (1, 4) else None for v in range(6)]]
    cap = _denoiser(un, cn, "ddim", box_capacity=CAP)
    for i, n in enumerate([2, 6]):
        kw = dict(_scene(n, 200 + i), num_inference_steps=3, guidance_scale=2.0, conditional_latents=pinned)
        out, ref = cap(**kw), _denoiser(un, cn, "ddim")(**kw)
        assert rel_l2(out, ref) < 1e-5


@torch.no_grad()
def test_capacity_limits_and_bbox_max_length(emulated):
    un, cn = _modules()
    cap = _denoiser(un, cn, "ddim", box_capacity=CAP)
    with pytest.raises(ValueError, match=rf"{CAP + 1} boxes per view exceed box_capacity={CAP}"):
        cap(**_scene(CAP + 1, 1), num_inference_steps=2)
    with pytest.raises(ValueError, match="box_capacity"):
        _denoiser(un, cn, "ddim", box_capacity=0)
    with pytest.raises(ValueError, match="view-sharded"):
        BEVControlNetDenoiser(un, cn, view_shard=object(), box_capacity=CAP)
    # bbox_max_length keeps the reference's meaning: null tokens up to that length are attended
    kw = dict(_scene(3, 5), num_inference_steps=2, guidance_scale=2.0, bbox_max_length=6)
    out, ref = cap(**kw), _denoiser(un, cn, "ddim")(**kw)
    assert cap._static["ctx_len"].tolist() == [1 + 77 + 6] * 12 and rel_l2(out, ref) < 1e-5
    plain = _denoiser(un, cn, "ddim")(**dict(kw, bbox_max_length=None))
    assert rel_l2(ref, plain) > 1e-4  # and that is a different computation from attending the 3 boxes only


@torch.no_grad()
def test_device_count_sets_the_attended_length(emulated):
    """Boxes already padded to the capacity with their number in bboxes_3d_data["count"] (collate_on_device(capacity=))."""
    un, cn = _modules()
    cap = _denoiser(un, cn, "ddim", box_capacity=CAP)
    kw = dict(_scene(4, 9), num_inference_steps=2, guidance_scale=2.0)
    ref = _denoiser(un, cn, "ddim")(**kw)
    boxes = kw["bev_controlnet_kwargs"]["bboxes_3d_data"]
    padded = {k: torch.cat([v, torch.zeros_like(v[:, :, :1]).expand(-1, -1, CAP - 4, *v.shape[3:])], 2) for k, v in boxes.items()}
    padded["classes"][:, :, 4:] = -1  # the collate kernel's padding
    padded["count"] = torch.tensor(4, dtype=torch.int32)
    out = cap(**dict(kw, bev_controlnet_kwargs={"bboxes_3d_data": padded}))
    assert cap._static["ctx_len"].tolist() == [1 + 77 + 4] * 12 and rel_l2(out, ref) < 1e-5
    out = cap(**dict(kw, bev_controlnet_kwargs={"bboxes_3d_data": padded}, bbox_max_length=6))
    assert cap._static["ctx_len"].tolist() == [1 + 77 + 6] * 12
    assert rel_l2(out, _denoiser(un, cn, "ddim")(**dict(kw, bbox_max_length=6))) < 1e-5


@torch.no_grad()
@pytest.mark.parametrize("capacity", [None, CAP])
def test_generate_stream_equals_calls_threaded_with_one_generator(emulated, capacity):
    un, cn = _modules()
    extra = {} if capacity is None else {"box_capacity": capacity}
    batches = []
    for i, n in enumerate([3, 5]):
        s = _scene(n, 300 + i)
        batches.append(dict(bev_map_with_aux=s["image"], camera_param=s["camera_param"], prompt_embeds=s["prompt_embeds"],
                            negative_prompt_embeds=s["negative_prompt_embeds"], kwargs=s["bev_controlnet_kwargs"]))
    call = dict(num_inference_steps=3, guidance_scale=2.0, height=8 * H, width=8 * W)
    stream = _denoiser(un, cn, "unipc", **extra)
    got = list(stream.generate_stream(batches, samples_per_scene=3, generator=torch.Generator().manual_seed(11), **call))
    single = _denoiser(un, cn, "unipc", **extra)
    gen = torch.Generator().manual_seed(11)
    for b, results in zip(batches, got):
        assert len(results) == 3
        for r in results:
            ref = single(b["bev_map_with_aux"], b["camera_param"], prompt_embeds=b["prompt_embeds"],
                         negative_prompt_embeds=b["negative_prompt_embeds"], bev_controlnet_kwargs=b["kwargs"], generator=gen,
                         **call)
            assert torch.equal(r, ref)
        assert not torch.equal(results[0], results[1])
    with pytest.raises(ValueError, match="generator"):
        next(stream.generate_stream(batches, latents=torch.zeros(1, 4, H, W)))


@torch.no_grad()
def test_a_second_denoiser_keeps_the_engines_index_tensors(emulated):
    """A denoiser's captured step graph holds the address of the UNet engine's kv_index tensor: building another denoiser on
    the same modules (same view_shard) must not drop it."""
    un, cn = _modules()
    first = _denoiser(un, cn, "ddim")
    first(**_scene(2, 1), num_inference_steps=1)
    idx = un.engine().kv_index(12)
    _denoiser(un, cn, "ddim", box_capacity=CAP)
    assert un.engine().kv_index(12) is idx
