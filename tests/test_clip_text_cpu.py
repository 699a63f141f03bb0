"""CLIP text encoder without a GPU: the fp32 oracle against the transformers fixtures, and the real host code (weight
packing, layer sequencing, pooling, CLIPTextModel, the denoiser's `prompt=`) run through the torch restatements of the
operators in tests/ops_emulator.py."""
import json
from dataclasses import asdict
from types import SimpleNamespace

import pytest
import torch

from magicdrive_b200 import arch, engine, models
from oracle.clip_text import TINY, clip_text_forward, draw_weights
from tests import ops_emulator
from tests.common import golden, tiny_configs, tiny_state_dicts

# a CLIP whose hidden size is the UNet's cross-attention width (768) but small everywhere else, for the pipeline checks
MID = dict(vocab_size=512, hidden_size=768, intermediate_size=256, num_hidden_layers=1, num_attention_heads=12,
           max_position_embeddings=77, eos_token_id=2)


def _rel(a, b):
    return ((a.float() - b.float()).abs().max() / b.float().abs().max()).item()


@pytest.fixture
def emulated(monkeypatch):
    ops_emulator.install(monkeypatch)
    monkeypatch.setattr(engine._Weights, "fold_dtype", torch.float32)


def _model(cfg_kwargs, sd):
    m = models.CLIPTextModel(**cfg_kwargs)
    m.load_state_dict(sd)
    return m


class StubTokenizer:
    """CLIPTokenizer's calling convention: BOS, one id per word, EOS, padded with EOS (<|endoftext|>)."""
    model_max_length = 77
    added_tokens_encoder = {}  # read by the reference pipeline's textual-inversion hook

    def __init__(self, vocab):
        self.bos, self.eos, self.n = vocab - 2, vocab - 1, vocab - 2

    def _ids(self, text):
        return [self.bos] + [sum(map(ord, w)) * 7 % self.n for w in text.split()] + [self.eos]

    def __call__(self, texts, padding="do_not_pad", max_length=None, truncation=False, return_tensors="pt"):
        rows = [self._ids(t) for t in ([texts] if isinstance(texts, str) else texts)]
        if truncation:
            rows = [r[:max_length - 1] + [self.eos] if len(r) > max_length else r for r in rows]
        width = max_length if padding == "max_length" else max(map(len, rows))
        if padding != "do_not_pad":
            rows = [r + [self.eos] * (width - len(r)) for r in rows]
        return SimpleNamespace(input_ids=torch.tensor(rows), attention_mask=torch.ones(len(rows), len(rows[0]), dtype=torch.long))

    def tokenize(self, text):
        return text.split()

    def batch_decode(self, ids):
        return [" ".join(map(str, r.tolist())) for r in ids]


# --------------------------------------------------------------------------------------------------------- oracle
@pytest.mark.parametrize("name", ["tiny", "sd15"])
def test_oracle_reproduces_the_transformers_fixture(name):
    g = golden(f"clip_text_{name}.pt")
    cfg = arch.ClipTextConfig(**g["config"])
    sd = g["state_dict"] if name == "tiny" else draw_weights(cfg, g["seed_weights"])
    for case in g["cases"]:
        h, p = clip_text_forward(sd, cfg, case["ids"])
        assert _rel(h, case["last_hidden_state"]) <= 1e-5
        assert _rel(p, case["pooler_output"]) <= 1e-5


# --------------------------------------------------------------------------------------------------------- host code
def test_state_dict_names_and_shapes():
    m = models.CLIPTextModel()  # SD-1.5 defaults
    sd = m.state_dict()
    assert len(sd) == 196
    assert sd["text_model.embeddings.token_embedding.weight"].shape == (49408, 768)
    assert sd["text_model.encoder.layers.11.mlp.fc1.weight"].shape == (3072, 768)
    assert m.config.hidden_act == "quick_gelu" and m.config.eos_token_id == 2
    transformers = pytest.importorskip("transformers")
    ref = transformers.CLIPTextModel(transformers.CLIPTextConfig(**TINY))
    ours = models.CLIPTextModel(**TINY)
    assert {k: tuple(v.shape) for k, v in ref.state_dict().items()} == {k: tuple(v.shape) for k, v in ours.state_dict().items()}
    with pytest.raises(ValueError):
        models.CLIPTextModel(hidden_act="gelu")


def test_host_code_matches_the_fixture(emulated):
    g = golden("clip_text_tiny.pt")
    m = _model(g["config"], g["state_dict"])
    for case in g["cases"]:
        out = m(case["ids"])
        assert out[0] is out.last_hidden_state
        # tolerance of the bf16-rounded weight matrices; a wrong position, mask or pooled row is O(1)
        assert _rel(out.last_hidden_state, case["last_hidden_state"]) < 2e-2
        assert _rel(out.pooler_output, case["pooler_output"]) < 2e-2
    # config object instead of kwargs
    m2 = models.CLIPTextModel(SimpleNamespace(to_dict=lambda: dict(g["config"])))
    assert m2.config.hidden_size == g["config"]["hidden_size"]


def test_pooling_takes_the_row_at_argmax_of_the_ids(emulated):
    g = golden("clip_text_tiny.pt")
    m = _model(g["config"], g["state_dict"])
    ids = torch.tensor([[510, 3, 511, 511, 9], [510, 511, 4, 5, 6], [510, 7, 8, 9, 511]])
    out = m(ids)
    for i, j in enumerate([2, 1, 4]):
        assert torch.equal(out.pooler_output[i], out.last_hidden_state[i, j])
    with pytest.raises(ValueError):
        m(ids, attention_mask=torch.tensor([[1, 1, 1, 0, 0]] * 3))
    m(ids, attention_mask=torch.ones(3, 5, dtype=torch.long))
    with pytest.raises(ValueError):
        m(ids, output_hidden_states=True)
    with pytest.raises(ValueError):
        m(torch.full((1, 78), 511))


@pytest.mark.parametrize("fmt", ["safetensors", "bin"])
def test_from_pretrained(emulated, tmp_path, fmt):
    g = golden("clip_text_tiny.pt")
    d = tmp_path / "text_encoder"
    d.mkdir()
    cfg = dict(g["config"], architectures=["CLIPTextModel"], model_type="clip_text_model", torch_dtype="float32")
    (d / "config.json").write_text(json.dumps(cfg))
    sd = dict(g["state_dict"])
    if fmt == "safetensors":
        from safetensors.torch import save_file
        save_file({k: v.contiguous() for k, v in sd.items()}, str(d / "model.safetensors"))
    else:  # older checkpoints carry the position_ids buffer
        sd["text_model.embeddings.position_ids"] = torch.arange(77)[None]
        torch.save(sd, str(d / "pytorch_model.bin"))
    m = models.CLIPTextModel.from_pretrained(str(tmp_path), subfolder="text_encoder")
    ids = g["cases"][0]["ids"]
    assert torch.equal(m(ids).last_hidden_state, _model(g["config"], g["state_dict"])(ids).last_hidden_state)


def test_prepare_class_tokens_are_the_pooled_outputs(emulated):
    cfg_t = arch.ClipTextConfig(**MID)
    sd = draw_weights(cfg_t, 5)
    enc = _model(MID, sd)
    tok = StubTokenizer(MID["vocab_size"])
    names = ["car", "truck", "construction_vehicle", "bus", "traffic_cone"]
    _, ccfg = tiny_configs()
    cn = models.BEVControlNetModel(**asdict(ccfg), bbox_embedder_param=dict(n_classes=10, class_token_dim=768,
                                                                            use_text_encoder_init=True))
    cn.reset_parameters_synthetic(1)
    cn.prepare(SimpleNamespace(dataset=SimpleNamespace(object_classes=names)), tokenizer=tok, text_encoder=enc)
    for i, n in enumerate(names):
        ids = tok([n], padding="do_not_pad").input_ids
        assert 3 <= ids.shape[1] <= 7
        _, pooled = clip_text_forward(sd, cfg_t, ids)
        assert _rel(cn.bbox_embedder._class_tokens[i], pooled[0]) < 2e-2


def _denoiser(text_encoder=None, tokenizer=None):
    from magicdrive_b200.pipeline import BEVControlNetDenoiser
    ucfg, ccfg = tiny_configs()
    usd, csd = tiny_state_dicts(3)
    un, cn = models.UNet2DConditionModelMultiview(**asdict(ucfg)), models.BEVControlNetModel(**asdict(ccfg))
    un.load_state_dict(usd)
    cn.load_state_dict(csd)
    return BEVControlNetDenoiser(un, cn, use_cuda_graph=False, text_encoder=text_encoder, tokenizer=tokenizer)


class _Captured(Exception):
    pass


def _captured_embeds(den, **kw):
    """The (prompt_embeds, negative_prompt_embeds) a denoiser call hands to prepare()."""
    seen = {}

    def prepare(latents, prompt_embeds, negative_prompt_embeds, *a, **k):
        seen.update(p=prompt_embeds, n=negative_prompt_embeds)
        raise _Captured

    den.prepare = prepare
    with pytest.raises(_Captured):
        den(image=torch.zeros(2, 8, 52, 52), camera_param=torch.zeros(2, 6, 3, 7), **kw)
    return seen["p"], seen["n"]


def test_denoiser_prompt_gives_the_prompt_embeds_inputs(emulated):
    enc = _model(MID, draw_weights(arch.ClipTextConfig(**MID), 6))
    tok = StubTokenizer(MID["vocab_size"])
    den = _denoiser(enc, tok)
    caps = ["a rainy night street", "sunny day, parked cars"]
    enc_ids = lambda t: enc(tok(t, padding="max_length", max_length=77, truncation=True).input_ids)[0]
    p, n = _captured_embeds(den, prompt=caps)
    assert torch.equal(p, enc_ids(caps)) and torch.equal(n, enc_ids(["", ""]))
    p, n = _captured_embeds(den, prompt=caps, negative_prompt=["blurry", "dark"])
    assert torch.equal(n, enc_ids(["blurry", "dark"]))
    p2, n2 = _captured_embeds(den, prompt_embeds=p, negative_prompt_embeds=n)
    assert p2 is p and n2 is n
    _, n1 = _captured_embeds(den, prompt="one scene", guidance_scale=1.0)
    assert n1 is None
    with pytest.raises(TypeError):
        _captured_embeds(den, prompt=caps, negative_prompt="blurry")
    with pytest.raises(ValueError):
        _captured_embeds(den, prompt=caps, negative_prompt=["blurry"])
    with pytest.raises(ValueError):
        _captured_embeds(den, prompt=3)
    with pytest.raises(ValueError):
        _captured_embeds(_denoiser(), prompt=caps)
    # without a text encoder, prompt_embeds behave as before
    e = torch.randn(2, 77, 768)
    p3, n3 = _captured_embeds(_denoiser(), prompt_embeds=e, negative_prompt_embeds=e)
    assert p3 is e and n3 is e


def test_reference_pipeline_encodes_captions_with_our_text_encoder(emulated, monkeypatch):
    """The reference's unmodified StableDiffusionBEVControlNetPipeline.__call__(prompt=...) with a stub tokenizer and our
    CLIPTextModel gives the latents of the same call with our encoder's embeddings passed in."""
    from oracle import ref_shim
    if not ref_shim.available():
        pytest.skip("reference tree not mounted")
    from tests import test_dropin_reference_pipeline_cpu as D
    monkeypatch.setattr(models, "UNetEngine", D._FakeUNetEngine)
    monkeypatch.setattr(models, "ControlNetEngine", D._FakeControlNetEngine)
    R = ref_shim.load()
    g = golden("tiny_pipeline.pt")
    ucfg, ccfg = tiny_configs()
    usd, csd = tiny_state_dicts(g["seed"])
    un, cn = models.UNet2DConditionModelMultiview(**asdict(ucfg)), models.BEVControlNetModel(**asdict(ccfg))
    un.load_state_dict(usd)
    cn.load_state_dict(csd)
    enc = _model(MID, draw_weights(arch.ClipTextConfig(**MID), 7))
    tok = StubTokenizer(MID["vocab_size"])

    class Pipe(R.StableDiffusionBEVControlNetPipeline):
        def prepare_extra_step_kwargs(self, generator, eta):
            return {"eta": eta}

    vae = R.AutoencoderKL(block_out_channels=[32, 64, 64, 64], down_block_types=["DownEncoderBlock2D"] * 4,
                          up_block_types=["UpDecoderBlock2D"] * 4, latent_channels=4)
    sched = R.DDIMScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False,
                            set_alpha_to_one=False, steps_offset=1)
    pipe = Pipe(vae=vae, text_encoder=enc, unet=un, controlnet=cn, scheduler=sched, tokenizer=tok)
    pipe.set_progress_bar_config(disable=True)
    inp = g["inputs"]
    h, w = inp["latents"].shape[-2:]
    common = dict(image=inp["bev_map"], camera_param=inp["camera_param"], height=h * 8, width=w * 8,
                  num_inference_steps=g["steps"], guidance_scale=g["guidance"], output_type="latent",
                  bev_controlnet_kwargs={"bboxes_3d_data": inp["bboxes_3d_data"]})
    cap = ["a busy intersection at dusk"]
    out = pipe(prompt=cap, latents=inp["latents"].clone(), **common)
    ids = lambda t: tok(t, padding="max_length", max_length=77, truncation=True).input_ids
    ref = pipe(prompt=None, prompt_embeds=enc(ids(cap))[0], negative_prompt_embeds=enc(ids([""]))[0],
               latents=inp["latents"].clone(), **common)
    assert torch.equal(out.images, ref.images)
