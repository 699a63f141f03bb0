"""Host side of the engines on CPU: weight packing (tap-major conv filters, K/N padding, fused QKV, GEGLU tile interleave,
folded cross-view connector), layer sequencing, skip concats as two-source operands, non-integer nearest resizes, the
hoisted conditioning, kv_index — executed through tests/ops_emulator.py (torch restatements of the C-ABI operators) and
compared with the fp32 oracle.  Weights are made exactly bf16-representable so the only expected difference is the bf16
rounding of the folded connector weight W_c W_o (engine._Weights.folded_connector)."""
from dataclasses import asdict

import pytest
import torch

from magicdrive_b200 import arch, models
from magicdrive_b200.pipeline import BEVControlNetDenoiser
from magicdrive_b200.synthetic import synthetic_inputs
from oracle import torch_oracle as O
from tests import ops_emulator
from tests.common import rel_l2, tiny_configs


def _bf16_exact(sd):
    return {k: (v.to(torch.bfloat16).float() if v.is_floating_point() else v) for k, v in sd.items()}


def _four_level_configs():
    """Every block type of the SD-1.5 layout (3 cross-attention levels + plain level, 2 layers per block) at small width."""
    kw = dict(block_out_channels=(64, 128, 256, 256), attention_head_dim=8)
    return arch.UNetConfig(**kw), arch.ControlNetConfig(map_size=(8, 200, 200), **kw)


@pytest.fixture
def emulated(monkeypatch):
    ops_emulator.install(monkeypatch)
    # LayerNorm gains folded into the consuming GEMM's weights (W * gamma) are kept in fp32 here, so that the fold's algebra
    # (column sums, beta term, per-row statistics, GEGLU tile order) is checked to 1e-5; the bf16 rounding of W * gamma
    # that the device path adds is bounded separately in test_layernorm_fold_rounding_is_bf16_weight_noise
    from magicdrive_b200 import engine
    monkeypatch.setattr(engine._Weights, "fold_dtype", torch.float32)


def _modules(ucfg, ccfg, seed):
    usd = _bf16_exact(arch.synthetic_state_dict(arch.unet_param_shapes(ucfg), seed))
    csd = _bf16_exact(arch.synthetic_state_dict(arch.controlnet_param_shapes(ccfg), seed + 1))
    un = models.UNet2DConditionModelMultiview(**asdict(ucfg))
    cn = models.BEVControlNetModel(**asdict(ccfg))
    un.load_state_dict(usd)
    cn.load_state_dict(csd)
    return un, cn, usd, csd


@torch.no_grad()
@pytest.mark.parametrize("layout,h,w,map_hw", [("tiny", 10, 13, 52), ("four_level", 28, 50, 200), ("four_level_272x736", 34, 92, 200)])
def test_module_forwards_through_emulated_operators_match_the_oracle(emulated, layout, h, w, map_hw):
    ucfg, ccfg = tiny_configs() if layout == "tiny" else _four_level_configs()
    if layout == "four_level_272x736":
        # configs/exp/272x736.yaml: 34 x 92 latents (odd sizes down the pyramid: 17 x 46, 9 x 23, 5 x 12) and the ...Plus map
        # encoder pooling the 200 x 200 BEV map to the latent grid
        from dataclasses import replace
        ccfg = replace(ccfg, map_embedding_size=(h, w))
    un, cn, usd, csd = _modules(ucfg, ccfg, 31)
    inp = synthetic_inputs(1, 6, h, w, n_box=4, map_hw=map_hw, seed=8)
    lat5 = torch.stack([inp["latents"]] * 6, 1)
    t = torch.tensor([481])
    down, mid, ctx = cn(lat5, t, inp["camera_param"], inp["bboxes_3d_data"], inp["prompt_embeds"], inp["bev_map"],
                        return_dict=False)
    eps = un(lat5.reshape(-1, 4, h, w), t[0], encoder_hidden_states=ctx, down_block_additional_residuals=down,
             mid_block_additional_residual=mid).sample
    d32, m32, c32 = O.controlnet_forward(csd, ccfg, lat5, t, inp["camera_param"], inp["bboxes_3d_data"],
                                         inp["prompt_embeds"], inp["bev_map"])
    e32 = O.unet_forward(usd, ucfg, lat5.reshape(-1, 4, h, w), t[0], c32, d32, m32)
    assert rel_l2(ctx, c32) < 1e-5
    assert len(down) == len(d32)
    for a, b in zip(down, d32):
        assert a.shape == b.shape and rel_l2(a, b) < 2e-5
    assert rel_l2(mid, m32) < 2e-5
    assert eps.shape == e32.shape and rel_l2(eps, e32) < 3e-3  # folded connector weight is rounded to bf16
    # without the ControlNet residuals (plain UNet2DConditionModel.forward call shape)
    e_plain = un(lat5.reshape(-1, 4, h, w), t[0], encoder_hidden_states=ctx).sample
    assert rel_l2(e_plain, O.unet_forward(usd, ucfg, lat5.reshape(-1, 4, h, w), t[0], c32)) < 3e-3


@torch.no_grad()
def test_configs0_one_view_text_only_stock_unet(emulated):
    """BASELINE.json configs[0]: the stock SD-1.5 UNet2DConditionModel call (one view, text-only conditioning, single
    denoise step, fp32 CPU plumbing).  (i) tiny config against the REFERENCE's own UNet2DConditionModel output
    (tests/golden/plain_unet.pt <- oracle/make_golden_plain_unet.py) and the oracle; (ii) the real SD-1.5 config at
    224x400 (28x50 latents), one view, against the oracle."""
    from oracle.make_golden_plain_unet import tiny_plain_config
    from tests.common import golden
    g = golden("plain_unet.pt")
    cfg = tiny_plain_config()
    sd = arch.synthetic_state_dict(arch.unet_param_shapes(cfg), g["seed"])
    assert not any(".attn4." in k or ".connector." in k for k in sd)  # stock BasicTransformerBlock
    e32 = O.unet_forward(sd, cfg, g["sample"], torch.tensor(g["t"]), g["text"])
    assert torch.allclose(e32, g["eps"], rtol=1e-3, atol=1e-4)  # oracle == reference, literal north-star tolerance
    sdb = _bf16_exact(sd)
    un = models.UNet2DConditionModelMultiview.stock_unet(**{k: v for k, v in asdict(cfg).items() if k != "neighboring_view_pair"})
    un.load_state_dict(sdb)
    out = un(g["sample"], g["t"], encoder_hidden_states=g["text"]).sample
    assert out.shape == g["eps"].shape
    assert rel_l2(out, O.unet_forward(sdb, cfg, g["sample"], torch.tensor(g["t"]), g["text"])) < 2e-5
    # (ii) SD-1.5 size, 1 view, 77 text tokens
    big = arch.UNetConfig(neighboring_view_pair={})
    sdb = _bf16_exact(arch.synthetic_state_dict(arch.unet_param_shapes(big), 19))
    un = models.UNet2DConditionModelMultiview.stock_unet()
    un.load_state_dict(sdb)
    gen = torch.Generator().manual_seed(6)
    x, text = torch.randn(1, 4, 28, 50, generator=gen), torch.randn(1, 77, 768, generator=gen)
    out = un(x, torch.tensor(981), encoder_hidden_states=text).sample
    assert rel_l2(out, O.unet_forward(sdb, big, x, torch.tensor(981), text)) < 2e-5


@torch.no_grad()
def test_layernorm_fold_rounding_is_bf16_weight_noise(monkeypatch):
    """With the device's storage (W * gamma rounded to bf16) the folded path stays within bf16 weight-rounding noise of the
    fp32 oracle: the same size as the folded connector's rounding, far below the bf16 activation noise (8e-3, below)."""
    ops_emulator.install(monkeypatch)
    ucfg, ccfg = tiny_configs()
    un, cn, usd, csd = _modules(ucfg, ccfg, 31)
    inp = synthetic_inputs(1, 6, 10, 13, n_box=4, map_hw=52, seed=8)
    lat5 = torch.stack([inp["latents"]] * 6, 1)
    t = torch.tensor([481])
    down, mid, ctx = cn(lat5, t, inp["camera_param"], inp["bboxes_3d_data"], inp["prompt_embeds"], inp["bev_map"],
                        return_dict=False)
    eps = un(lat5.reshape(-1, 4, 10, 13), t[0], encoder_hidden_states=ctx, down_block_additional_residuals=down,
             mid_block_additional_residual=mid).sample
    d32, m32, c32 = O.controlnet_forward(csd, ccfg, lat5, t, inp["camera_param"], inp["bboxes_3d_data"],
                                         inp["prompt_embeds"], inp["bev_map"])
    e32 = O.unet_forward(usd, ucfg, lat5.reshape(-1, 4, 10, 13), t[0], c32, d32, m32)
    assert rel_l2(mid, m32) < 4e-3 and rel_l2(eps, e32) < 4e-3, (rel_l2(mid, m32), rel_l2(eps, e32))


@torch.no_grad()
@pytest.mark.parametrize("attn_type", ["concat", "self"])
def test_cross_view_attention_types_through_emulated_operators(emulated, attn_type):
    """neighboring_attn_type 'concat' (one softmax over both neighbours' keys) and 'self' (one attention over all views' tokens),
    blocks.py:122-138: the engine's gather / batch re-interpretation against the reference's own outputs."""
    from dataclasses import replace
    from tests.common import golden
    g = golden("tiny_attn_types.pt")
    ucfg = replace(tiny_configs()[0], neighboring_attn_type=attn_type)
    usd = _bf16_exact(arch.synthetic_state_dict(arch.unet_param_shapes(ucfg), g["seed"]))
    un = models.UNet2DConditionModelMultiview(**asdict(ucfg))
    un.load_state_dict(usd)
    eps = un(g["sample"], torch.tensor(g["t"]), encoder_hidden_states=g["ctx"]).sample
    ref = O.unet_forward(usd, ucfg, g["sample"], torch.tensor(g["t"]), g["ctx"])
    assert eps.shape == ref.shape and rel_l2(eps, ref) < 3e-3, rel_l2(eps, ref)
    assert rel_l2(eps, g["eps"][attn_type]) < 2e-2  # weights rounded to bf16-exact values here: loose against the fp32 fixture


@torch.no_grad()
def test_map_embedder_plus_through_emulated_operators(emulated):
    """map_embedder_cls = ...BEVControlNetConditioningEmbeddingPlus with map_embedder_param, as configs/exp/272x736.yaml passes
    them: layer strides / pads, the adaptive pooling block and its SiLU (map_embedder.py:79-126)."""
    from tests.test_oracle_cpu import _map_plus_case
    g, gf, ccfg, csd = _map_plus_case()
    kw = {k: v for k, v in asdict(ccfg).items() if k not in ("map_embedding_size", "map_size", "conditioning_embedding_out_channels")}
    cn = models.BEVControlNetModel(map_embedder_cls="magicdrive.networks.map_embedder.BEVControlNetConditioningEmbeddingPlus",
                                   map_embedder_param=dict(conditioning_embedding_size=[10, 13], conditioning_size=[8, 52, 60],
                                                           block_out_channels=[16, 32, 96, 256]), **kw)
    assert cn.arch_cfg == ccfg
    csd = _bf16_exact(csd)
    cn.load_state_dict(csd)
    inp = gf["inputs"]
    lat5 = torch.stack([inp["latents"]] * 6, 1)[:1]
    down, mid, _ = cn(lat5, torch.tensor([gf["t"]]), inp["camera_param"][:1], None, inp["prompt_embeds"][:1], g["bev_map"],
                      return_dict=False)
    d32, m32, _ = O.controlnet_forward(csd, ccfg, lat5, torch.tensor([gf["t"]]), inp["camera_param"][:1], None,
                                       inp["prompt_embeds"][:1], g["bev_map"])
    assert rel_l2(mid, m32) < 2e-5 and rel_l2(down[0], d32[0]) < 2e-5
    with pytest.raises(ValueError):
        models.BEVControlNetModel(map_embedder_cls="some.other.Embedder", **kw)


@torch.no_grad()
def test_guess_mode_residual_scales_through_emulated_operators(emulated):
    """BEVControlNetModel.forward(guess_mode=True): per-residual out_scale of the zero convolutions (unet_addon_rawbox.py:897-905)."""
    ucfg, ccfg = tiny_configs()
    _, cn, _, csd = _modules(ucfg, ccfg, 31)
    inp = synthetic_inputs(1, 6, 10, 13, n_box=4, map_hw=52, seed=8)
    lat5 = torch.stack([inp["latents"]] * 6, 1)
    t = torch.tensor([481])
    down, mid, _ = cn(lat5, t, inp["camera_param"], inp["bboxes_3d_data"], inp["prompt_embeds"], inp["bev_map"],
                      conditioning_scale=0.7, guess_mode=True, return_dict=False)
    d32, m32, _ = O.controlnet_forward(csd, ccfg, lat5, t, inp["camera_param"], inp["bboxes_3d_data"], inp["prompt_embeds"],
                                       inp["bev_map"], conditioning_scale=0.7, guess_mode=True)
    for a, b in zip(down + [mid], d32 + [m32]):
        assert a.shape == b.shape and rel_l2(a, b) < 2e-5


@torch.no_grad()
@pytest.mark.parametrize("scheduler,guidance,fused", [("ddim", 2.0, True), ("unipc", 2.0, True), ("ddim", 1.0, True),
                                                      ("ddim", 2.0, False)])
def test_denoiser_through_emulated_operators_matches_the_oracle_loop(emulated, scheduler, guidance, fused):
    """fused: the ControlNet residual additions (unet_2d_condition_multiview.py:479-497) ride the zero convolutions' epilogues
    (ControlNetEngine.residuals(add_to=...)); not fused: the separate additions of UNetEngine.forward_decoder."""
    ucfg, ccfg = tiny_configs()
    un, cn, usd, csd = _modules(ucfg, ccfg, 41)
    inp = synthetic_inputs(2, 6, 10, 13, n_box=3, map_hw=52, seed=9)
    pipe = BEVControlNetDenoiser(un, cn, use_cuda_graph=False, overlap_controlnet=False, scheduler=scheduler)
    pipe.fuse_residual_adds = fused
    out = pipe(image=inp["bev_map"], camera_param=inp["camera_param"], prompt_embeds=inp["prompt_embeds"],
               negative_prompt_embeds=inp["negative_prompt_embeds"], latents=inp["latents"], num_inference_steps=3,
               guidance_scale=guidance, bev_controlnet_kwargs={"bboxes_3d_data": inp["bboxes_3d_data"]})
    ref = O.denoise_loop(usd, csd, ucfg, ccfg, inp["latents"], inp["prompt_embeds"], inp["negative_prompt_embeds"],
                         inp["camera_param"], inp["bboxes_3d_data"], inp["bev_map"], 3, guidance, scheduler=scheduler)
    assert out.shape == ref.shape and rel_l2(out, ref) < 3e-3


@torch.no_grad()
def test_sd15_vae_layout_through_emulated_operators(emulated):
    """The real SD-1.5 decoder layout (512/512/256/128 with the two channel-changing shortcuts), one small image."""
    cfg = arch.VaeConfig()
    sd = _bf16_exact(arch.synthetic_state_dict(arch.vae_decoder_param_shapes(cfg), 9))
    vae = models.AutoencoderKL(**asdict(cfg))
    vae.load_state_dict(sd)
    z = torch.randn(1, 4, 6, 7, generator=torch.Generator().manual_seed(2))
    assert rel_l2(vae.decode(z).sample, O.vae_decode(sd, cfg, z)) < 1e-5


@torch.no_grad()
@pytest.mark.parametrize("h,w", [(10, 13), (7, 9)])
def test_vae_decoder_through_emulated_operators_matches_the_oracle(emulated, h, w):
    """VaeDecoderEngine host logic (post_quant folding, single-head attention as GEMM + row softmax + GEMM with padded
    keys, x2 upsampling chain, unit-range epilogue) vs the oracle restatement of AutoencoderKL.decode."""
    cfg = arch.VaeConfig(block_out_channels=(64, 128, 128, 128))
    sd = _bf16_exact(arch.synthetic_state_dict(arch.vae_decoder_param_shapes(cfg), 51))
    vae = models.AutoencoderKL(**asdict(cfg))
    # a full AutoencoderKL checkpoint with pre-0.17 attention names loads too
    full = dict(sd)
    for new, old in (("to_q", "query"), ("to_k", "key"), ("to_v", "value"), ("to_out.0", "proj_attn")):
        for leaf in ("weight", "bias"):
            full[f"decoder.mid_block.attentions.0.{old}.{leaf}"] = full.pop(f"decoder.mid_block.attentions.0.{new}.{leaf}")
    full["encoder.conv_in.weight"] = torch.zeros(64, 3, 3, 3)
    full["quant_conv.weight"] = torch.zeros(8, 8, 1, 1)
    vae.load_state_dict(full)
    g = torch.Generator().manual_seed(4)
    z = torch.randn(3, 4, h, w, generator=g)
    out = vae.decode(z).sample
    ref = O.vae_decode(sd, cfg, z)
    assert out.shape == ref.shape == (3, 3, 8 * h, 8 * w) and rel_l2(out, ref) < 1e-5
    lat = torch.randn(1, 3, 4, h, w, generator=g) * 0.2
    imgs = vae.decode_latents(lat)
    ref_imgs = O.decode_latents(sd, cfg, lat)
    assert imgs.shape == ref_imgs.shape == (1, 3, 8 * h, 8 * w, 3)
    assert (imgs - ref_imgs).abs().max() < 1e-5 and 0.0 <= imgs.min() and imgs.max() <= 1.0
    with pytest.raises(NotImplementedError):
        vae.encode(z)


@torch.no_grad()
def test_denoiser_decodes_images_when_given_a_vae(emulated):
    ucfg, ccfg = tiny_configs()
    un, cn, usd, csd = _modules(ucfg, ccfg, 41)
    vcfg = arch.VaeConfig(block_out_channels=(64, 64, 64, 64))
    vsd = _bf16_exact(arch.synthetic_state_dict(arch.vae_decoder_param_shapes(vcfg), 52))
    vae = models.AutoencoderKL(**asdict(vcfg))
    vae.load_state_dict(vsd)
    inp = synthetic_inputs(1, 6, 10, 13, n_box=3, map_hw=52, seed=9)
    kw = dict(image=inp["bev_map"], camera_param=inp["camera_param"], prompt_embeds=inp["prompt_embeds"],
              negative_prompt_embeds=inp["negative_prompt_embeds"], latents=inp["latents"], num_inference_steps=2,
              guidance_scale=2.0, bev_controlnet_kwargs={"bboxes_3d_data": inp["bboxes_3d_data"]})
    pipe = BEVControlNetDenoiser(un, cn, use_cuda_graph=False, overlap_controlnet=False, vae=vae)
    lat = pipe(**kw)
    img = pipe(output_type="np", **kw)
    ref = O.decode_latents(vsd, vcfg, lat)
    assert img.shape == (1, 6, 80, 104, 3) and abs(img - ref.numpy()).max() < 1e-4
    with pytest.raises(ValueError):
        BEVControlNetDenoiser(un, cn, use_cuda_graph=False)(output_type="pt", **kw)


@torch.no_grad()
@pytest.mark.parametrize("scheduler", ["ddim", "unipc"])
def test_cfg_streams_mode_computes_the_same_step(emulated, scheduler):
    """The opt-in guidance-half branches (BEVControlNetDenoiser(cfg_streams=True)) slice the hoisted conditioning per half
    and must reproduce the batched step; here on CPU, where the two branches run one after the other."""
    ucfg, ccfg = tiny_configs()
    un, cn, usd, csd = _modules(ucfg, ccfg, 41)
    inp = synthetic_inputs(2, 6, 10, 13, n_box=3, map_hw=52, seed=9)
    kw = dict(image=inp["bev_map"], camera_param=inp["camera_param"], prompt_embeds=inp["prompt_embeds"],
              negative_prompt_embeds=inp["negative_prompt_embeds"], latents=inp["latents"], num_inference_steps=3,
              guidance_scale=2.0, bev_controlnet_kwargs={"bboxes_3d_data": inp["bboxes_3d_data"]})
    base = BEVControlNetDenoiser(un, cn, use_cuda_graph=False, overlap_controlnet=False, scheduler=scheduler)(**kw)
    split = BEVControlNetDenoiser(un, cn, use_cuda_graph=False, overlap_controlnet=False, scheduler=scheduler,
                                  cfg_streams=True)(**kw)
    assert rel_l2(split, base) < 1e-5


@torch.no_grad()
def test_full_sd15_width_engines_through_emulated_operators(emulated):
    """The real SD-1.5 / MagicDrive layout (320-640-1280-1280, 8 heads, GEGLU inner 1280..5120, 13 ControlNet residuals) at a
    small latent size: packing and sequencing of the full-width networks against the oracle (~1.3 G parameters, ~80 s)."""
    ucfg, ccfg = arch.UNetConfig(), arch.ControlNetConfig(map_size=(8, 52, 52))
    un, cn, usd, csd = _modules(ucfg, ccfg, 31)
    h, w = 10, 13
    inp = synthetic_inputs(1, 6, h, w, n_box=4, map_hw=52, seed=8)
    lat5 = torch.stack([inp["latents"]] * 6, 1)
    t = torch.tensor([481])
    down, mid, ctx = cn(lat5, t, inp["camera_param"], inp["bboxes_3d_data"], inp["prompt_embeds"], inp["bev_map"],
                        return_dict=False)
    eps = un(lat5.reshape(-1, 4, h, w), t[0], encoder_hidden_states=ctx, down_block_additional_residuals=down,
             mid_block_additional_residual=mid).sample
    d32, m32, c32 = O.controlnet_forward(csd, ccfg, lat5, t, inp["camera_param"], inp["bboxes_3d_data"],
                                         inp["prompt_embeds"], inp["bev_map"])
    e32 = O.unet_forward(usd, ucfg, lat5.reshape(-1, 4, h, w), t[0], c32, d32, m32)
    assert rel_l2(ctx, c32) < 1e-5 and len(down) == 12
    assert max(rel_l2(a, b) for a, b in zip(down, d32)) < 2e-5 and rel_l2(mid, m32) < 2e-5
    assert rel_l2(eps, e32) < 6e-3  # 16 folded connector weights rounded to bf16


@torch.no_grad()
def test_bf16_storage_alone_accounts_for_the_gpu_parity_gap(emulated, monkeypatch):
    """With the operator restatements rounding every activation to bf16 exactly where the device stores one (fp32
    arithmetic otherwise), the 3-step CFG pipeline lands 8.4e-3 (rel-L2) from the reference fixture — the same distance the
    CUDA path measures on an H100 (tests/test_model_gpu.py, pipeline parity: 8.3e-3).  The GPU tolerance (2e-2) is therefore
    a statement about bf16 storage, not slack for kernel error."""
    from tests.common import golden, tiny_state_dicts
    monkeypatch.setattr(ops_emulator, "ROUND_ACTIVATIONS", True)
    p = golden("tiny_pipeline.pt")
    inp = p["inputs"]
    ucfg, ccfg = tiny_configs()
    usd, csd = tiny_state_dicts(p["seed"])
    un = models.UNet2DConditionModelMultiview(**asdict(ucfg))
    cn = models.BEVControlNetModel(**asdict(ccfg))
    un.load_state_dict(usd)
    cn.load_state_dict(csd)
    pipe = BEVControlNetDenoiser(un, cn, use_cuda_graph=False, overlap_controlnet=False)
    out = pipe(image=inp["bev_map"], camera_param=inp["camera_param"], prompt_embeds=inp["prompt_embeds"],
               negative_prompt_embeds=inp["negative_prompt_embeds"], latents=inp["latents"], num_inference_steps=p["steps"],
               guidance_scale=p["guidance"], bev_controlnet_kwargs={"bboxes_3d_data": inp["bboxes_3d_data"]})
    e = rel_l2(out, p["latents_out"])
    assert 4e-3 < e < 1.3e-2, e
