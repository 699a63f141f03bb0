"""CLIP text encoder on the GPU: the causal attention kernel, the quick-GELU GEMM epilogue and the token + position embedding
(every output guard-banded as in test_kernel_edges_gpu.py, references in float64 from the same bf16 inputs), the whole
encoder at SD-1.5 size against the fp32 oracle and the transformers fixtures (DESIGN §4 criterion), CUDA-graph reuse, and
the denoiser's `prompt=` path."""
import ctypes as C
from dataclasses import asdict

import pytest
import torch

pytestmark = pytest.mark.gpu

from magicdrive_b200 import _lib, arch, models, ops  # noqa: E402
from oracle.clip_text import clip_text_forward, draw_weights  # noqa: E402  (checker only)
from tests.common import golden, record, rel_l2, tiny_configs, tiny_state_dicts  # noqa: E402
from tests.test_kernel_edges_gpu import BF16, F32, F64, Guarded, _bf, _close_bf16, _gen, _randn  # noqa: E402

DEV = "cuda"
ATTN_KERNELS = ["tc2", "tc2d", "tc"]
HEADS = 12


# ------------------------------------------------------------------------------------------------ causal attention
def _causal_ref(qkv, b, l, d):
    c = HEADS * d
    x = qkv.to(F64).reshape(b, l, 3, HEADS, d).permute(2, 0, 3, 1, 4)  # [3, b, heads, l, d]
    s = x[0] @ x[1].transpose(-1, -2) * d ** -0.5
    s = s + torch.full((l, l), float("-inf"), dtype=F64, device=DEV).triu(1)
    return (torch.softmax(s, -1) @ x[2]).transpose(1, 2).reshape(b * l, c)


def _causal(qkv, b, l, d, out):
    c = HEADS * d
    return ops.attention_causal(qkv, qkv[:, c:], qkv[:, 2 * c:], b=b, heads=HEADS, l=l, d=d, ldq=3 * c, ldk=3 * c, ldv=3 * c,
                                scale=d ** -0.5, out=out)


@pytest.mark.parametrize("multiq", ["1", "0"])
@pytest.mark.parametrize("d", [64, 40, 80, 160])
@pytest.mark.parametrize("kernel", ATTN_KERNELS)
def test_attention_causal(cuda_lib, monkeypatch, kernel, d, multiq):
    """b in {1, 2, 8} x L in {1 .. 300} (one key, a partial tile, the text length, tile edges 128 / 129, several query tiles)
    from a fused-QKV buffer into a column slice.  With lq == lk a single K/V tile also means a single query tile, so multi-Q
    mode never engages: both settings must give the same bits."""
    monkeypatch.setenv("MDB_ATTN_KERNEL", kernel)
    monkeypatch.setenv("MDB_ATTN_MULTIQ", multiq)
    g = _gen(31)
    c = HEADS * d
    for b in (1, 2, 8):
        for l in (1, 4, 7, 77, 128, 129, 300):
            qkv = _bf(_randn(b * l, 3 * c, g=g, scale=1.5))
            out = Guarded(b * l, c, ld=c + 16, col0=8)
            _causal(qkv, b, l, d, out.out)
            out.check(f"b={b} L={l}")
            torch.testing.assert_close(out.out.to(F64), _causal_ref(qkv, b, l, d), atol=2e-2, rtol=5e-3,
                                       msg=lambda m: f"b={b} L={l}: {m}")
            if multiq == "0":
                monkeypatch.setenv("MDB_ATTN_MULTIQ", "1")
                again = _causal(qkv, b, l, d, None)
                monkeypatch.setenv("MDB_ATTN_MULTIQ", "0")
                assert torch.equal(again, out.out)


@pytest.mark.parametrize("kernel,d,l,ms", [("tc2", 64, 300, [1, 128, 129, 200, 300]), ("tc2d", 80, 77, [1, 64, 65, 77])])
def test_attention_causal_rows_equal_truncated_keys(cuda_lib, monkeypatch, kernel, d, l, ms):
    """Row m-1 sees keys 0 .. m-1: bit for bit the unmasked kernel with lk = m (extra fully-masked tiles add exact zeros)."""
    monkeypatch.setenv("MDB_ATTN_KERNEL", kernel)
    g = _gen(32)
    b, c = 2, HEADS * d
    qkv = _bf(_randn(b * l, 3 * c, g=g, scale=1.5))
    full = _causal(qkv, b, l, d, None).reshape(b, l, c)
    for m in ms:
        kv = qkv.reshape(b, l, 3 * c)[:, :m].contiguous().reshape(b * m, 3 * c)  # row stride 3C, batch stride m rows
        trunc = ops.attention(qkv, kv[:, c:], kv[:, 2 * c:], b=b, heads=HEADS, lq=l, lk=m, d=d, ldq=3 * c, ldk=3 * c,
                              ldv=3 * c, scale=d ** -0.5).reshape(b, l, c)
        assert torch.equal(full[:, m - 1], trunc[:, m - 1]), f"row {m - 1}"


def test_attention_causal_rejects_bad_calls(cuda_lib):
    q = torch.zeros(2 * 77, 3 * 768, dtype=BF16, device=DEV)
    o = torch.empty(2 * 77, 768, dtype=BF16, device=DEV)
    L = _lib.lib()
    p = lambda t: t.data_ptr()
    st = torch.cuda.current_stream().cuda_stream
    assert L.mdb_attention_causal(p(q), 2304, p(q), 2304, p(q), 2304, p(o), 768, 2, 12, 77, 76, 64, 0.125, st) == -1
    assert L.mdb_attention_causal(p(q), 2304, p(q), 2304, p(q), 2304, p(o), 768, 2, 12, 77, 77, 48, 0.125, st) == -3


# ------------------------------------------------------------------------------------------------ quick-GELU epilogue
def _desc(x, w, out, **kw):
    d = _lib.GemmDesc()
    m, k = x.shape
    d.a0, d.c0, d.lda0, d.n_img, d.h_in, d.w_in = x.data_ptr(), k, k, 1, 1, m
    d.w, d.n_out = w.data_ptr(), w.shape[0]
    d.taps_h = d.taps_w = d.stride = 1
    d.h_out, d.w_out = 1, m
    d.out, d.ldo, d.out_scale, d.epi_mode = out.data_ptr(), w.shape[0], 1.0, 2
    for key, v in kw.items():
        setattr(d, key, v)
    return d


@pytest.mark.parametrize("ln", [False, True])
@pytest.mark.parametrize("m", [1, 5, 77, 129, 154, 924])
def test_gemm_quick_gelu(cuda_lib, m, ln):
    """fc1 of the text encoder: N = 3072, K = 768, with and without layer_norm2 folded in."""
    g = _gen(33)
    n, k = 3072, 768
    x = _bf(_randn(m, k, g=g, scale=2.0) + 0.5)
    w = _bf(_randn(n, k, g=g, scale=k ** -0.5 * 2.0))
    bias = _randn(n, g=g, scale=0.5)
    out = Guarded(m, n, ld=n + 64, col0=32)
    kw = {}
    y = x.to(F64) @ w.to(F64).t()
    if ln:
        xf = x.float()
        kw["ln"] = ops.RowStats(torch.stack([xf.sum(1), (xf * xf).sum(1)], -1)[:, None].contiguous(), 1)
        kw["ln_colsum"] = w.float().sum(1)
        mean = x.to(F64).mean(1, keepdim=True)
        rstd = torch.rsqrt(x.to(F64).var(1, unbiased=False, keepdim=True) + 1e-5)
        y = rstd * (y - mean * kw["ln_colsum"].to(F64)[None])
    y = y + bias.to(F64)
    ops.linear(x, w, bias=bias, out=out.out, ldo=n + 64, quick_gelu=True, ln_eps=1e-5, **kw)
    out.check(f"M={m}")
    _close_bf16(out.out, y * torch.sigmoid(1.702 * y), f"M={m} ln={ln}")


def test_gemm_quick_gelu_rejects_other_epilogue_inputs(cuda_lib):
    x = torch.zeros(77, 768, dtype=BF16, device=DEV)
    w = torch.zeros(3072, 768, dtype=BF16, device=DEV)
    out = torch.empty(77, 3072, dtype=BF16, device=DEV)
    res = torch.zeros(77, 3072, dtype=BF16, device=DEV)
    rb = torch.zeros(1, 3072, dtype=F32, device=DEV)
    stats = torch.empty(77 * 64, dtype=F32, device=DEV)
    st = torch.cuda.current_stream().cuda_stream
    L = _lib.lib()
    for kw in (dict(residual=res.data_ptr(), ldr=3072), dict(rowbias=rb.data_ptr()), dict(stats_out=stats.data_ptr()),
               dict(out_is_f32=1)):
        assert L.mdb_gemm_conv(C.byref(_desc(x, w, out, **kw)), st) == -3, kw
    assert L.mdb_gemm_conv(C.byref(_desc(x, w, out)), st) == 0
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ embedding
@pytest.mark.parametrize("i64", [True, False])
def test_clip_embed(cuda_lib, i64):
    g = _gen(34)
    vocab, dim, n_seq, ln = 49408, 768, 8, 77
    tok = _bf(_randn(vocab, dim, g=g))
    pos = _bf(_randn(ln, dim, g=g, scale=0.3))
    ids = torch.randint(0, vocab, (n_seq, ln), device=DEV, generator=g)
    ids[:, 0], ids[:, -1] = 0, vocab - 1
    bad = [(1, 3, -1), (2, 5, vocab), (4, 76, 1 << 40 if i64 else 1 << 30)]
    for s, p, v in bad:
        ids[s, p] = v
    ids = ids if i64 else ids.to(torch.int32)
    out = Guarded(n_seq * ln, dim, ld=dim + 16, col0=8)
    _, stats = ops.clip_embed(ids, tok, pos, out=out.out)
    out.check()
    badrow = torch.zeros(n_seq, ln, dtype=torch.bool, device=DEV)
    for s, p, _ in bad:
        badrow[s, p] = True
    badrow = badrow.reshape(-1)
    ref = tok[ids.clamp(0, vocab - 1).long()] + pos[None]  # bf16 + bf16: the fp32 sum rounded once
    ref = ref.reshape(-1, dim)
    assert torch.equal(out.out[~badrow], ref[~badrow])
    assert torch.isnan(out.out[badrow].float()).all() and torch.isnan(stats.data[badrow]).all()
    o64 = out.out[~badrow].to(F64)
    st = stats.data[~badrow, 0].to(F64)
    assert ((st[:, 0] - o64.sum(1)).abs() <= 3e-5 * o64.abs().sum(1)).all()
    assert ((st[:, 1] - (o64 * o64).sum(1)).abs() <= 3e-5 * (o64 * o64).sum(1)).all()


# ------------------------------------------------------------------------------------------------ whole encoder
@pytest.fixture(scope="module")
def sd15_encoder():
    g = golden("clip_text_sd15.pt")
    cfg = arch.ClipTextConfig(**g["config"])
    sd = draw_weights(cfg, g["seed_weights"])
    m = models.CLIPTextModel(**g["config"])
    m.load_state_dict(sd)
    return g, cfg, {k: v.to(DEV) for k, v in sd.items()}, m.to(DEV)


def _criterion(ours, oracle32, oracle16, what):
    e, y = rel_l2(ours, oracle32), rel_l2(oracle16, oracle32)
    record(f"[parity] clip text {what}: ours {e:.3e}  bf16 oracle {y:.3e}")
    assert e <= 1.0 * y + 5e-4, (what, e, y)


def test_text_encoder_sd15(cuda_lib, sd15_encoder):
    g, cfg, sd, m = sd15_encoder
    gen = torch.Generator().manual_seed(35)
    big = torch.randint(0, cfg.vocab_size - 2, (8, 77), generator=gen)
    big[:, 0], big[:, 30:] = cfg.vocab_size - 2, cfg.vocab_size - 1
    for i, ids in enumerate([c["ids"] for c in g["cases"]] + [big]):
        idd = ids.to(DEV)
        out = m(idd)
        o32 = clip_text_forward(sd, cfg, idd)
        o16 = clip_text_forward(sd, cfg, idd, dtype=BF16)
        what = f"{tuple(ids.shape)}"
        _criterion(out.last_hidden_state, o32[0], o16[0], what + " hidden")
        _criterion(out.pooler_output, o32[1], o16[1], what + " pooled")
        if i < len(g["cases"]):  # the transformers fixture
            c = g["cases"][i]
            _criterion(out.last_hidden_state, c["last_hidden_state"].to(DEV), o16[0], what + " hidden vs fixture")
            _criterion(out.pooler_output, c["pooler_output"].to(DEV), o16[1], what + " pooled vs fixture")


def test_text_encoder_graph_reuse(cuda_lib, sd15_encoder):
    _, cfg, _, m = sd15_encoder
    gen = torch.Generator().manual_seed(36)
    for shape in ((2, 77), (1, 5)):
        for _ in range(2):  # the second call replays the graph captured by the first on new ids
            ids = torch.randint(0, cfg.vocab_size, shape, generator=gen).to(DEV)
            out = m(ids)
            m.use_cuda_graph = False
            eager = m(ids)
            m.use_cuda_graph = True
            assert torch.equal(out.last_hidden_state, eager.last_hidden_state)
            assert torch.equal(out.pooler_output, eager.pooler_output)


# ------------------------------------------------------------------------------------------------ denoiser prompt=
class _Tok:
    model_max_length = 77

    def __call__(self, texts, padding="do_not_pad", max_length=None, truncation=False, return_tensors="pt"):
        rows = [[510] + [sum(map(ord, w)) * 7 % 510 for w in t.split()][:75] + [511] for t in texts]
        return type("T", (), {"input_ids": torch.tensor([r + [511] * (max_length - len(r)) for r in rows])})


@pytest.mark.parametrize("scheduler", ["ddim", "unipc"])
def test_denoiser_prompt_equals_prompt_embeds(cuda_lib, scheduler):
    from magicdrive_b200.pipeline import BEVControlNetDenoiser
    mid = dict(vocab_size=512, hidden_size=768, intermediate_size=3072, num_hidden_layers=2, num_attention_heads=12)
    enc = models.CLIPTextModel(**mid)
    enc.load_state_dict(draw_weights(arch.ClipTextConfig(**mid), 37))
    enc = enc.to(DEV)
    inp = golden("tiny_pipeline.pt")["inputs"]
    ucfg, ccfg = tiny_configs()
    usd, csd = tiny_state_dicts(5)
    un, cn = models.UNet2DConditionModelMultiview(**asdict(ucfg)), models.BEVControlNetModel(**asdict(ccfg))
    un.load_state_dict(usd)
    cn.load_state_dict(csd)
    den = BEVControlNetDenoiser(un.to(DEV), cn.to(DEV), scheduler=scheduler, text_encoder=enc, tokenizer=_Tok())
    kw = dict(image=inp["bev_map"], camera_param=inp["camera_param"], latents=inp["latents"], num_inference_steps=3,
              guidance_scale=2.0, bev_controlnet_kwargs={"bboxes_3d_data": inp["bboxes_3d_data"]})
    caps = ["a wet road at night with parked trucks"]
    a = den(prompt=caps, **kw)
    ids = lambda t: _Tok()(t, padding="max_length", max_length=77, truncation=True).input_ids.to(DEV)
    b = den(prompt_embeds=enc(ids(caps))[0], negative_prompt_embeds=enc(ids([""]))[0], **kw)
    assert torch.equal(a, b)
