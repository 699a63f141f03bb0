"""Camera rigs other than nuScenes' six-camera ring on the GPU: the fused attention kernel with empty K/V slots (kv_index -1)
and per-batch key counts (kv_len) under the guard-band scheme of test_kernel_edges_gpu.py, the whole UNet on the reference's
rig fixtures (tests/golden/tiny_rigs.pt) and at SD-1.5 size against the fp32 oracle, and the denoiser at n_cam = 5."""
from dataclasses import asdict, replace

import pytest
import torch

pytestmark = pytest.mark.gpu

from magicdrive_b200 import arch, ops  # noqa: E402
from magicdrive_b200.models import BEVControlNetModel, UNet2DConditionModelMultiview  # noqa: E402
from magicdrive_b200.pipeline import BEVControlNetDenoiser  # noqa: E402
from oracle import torch_oracle as O  # noqa: E402  (checker only)
from tests.attention_model import attention_model, check_model  # noqa: E402
from tests.common import golden, rel_l2, tiny_configs, to_dev  # noqa: E402
from tests.test_kernel_edges_gpu import ATTN_DT_KERNELS, ATTN_KERNELS, Guarded, _bf, _gen  # noqa: E402
from tests.test_kernel_edges_gpu import _randn  # noqa: E402
from tests.test_model_gpu import _bf16_yardstick, _check  # noqa: E402

BF16, F16, F64 = torch.bfloat16, torch.float16, torch.float64
DEV = "cuda"
HEADS = {40: 4, 80: 2, 160: 2}
CHAIN5 = {0: [1, 2], 1: [0, 3], 2: [0, 4], 3: [1], 4: [2]}


def _block_n(kernel, d):
    return {"tc2": 128 if d <= 64 else 64, "tc2d": 64, "tc": 128}[kernel]


def _ref(q, kv_of, rows, heads, lq, d, scale, dt=BF16):
    """The float64 sum over each query batch's present sets (kv_of(i) -> list of (k, v)) and its error model
    (tests/attention_model.py); a batch without sets is zero."""
    return attention_model(q, kv_of, len(rows), heads, lq, d, scale, dt)


def _close(out, model, n_sets):
    check_model(out, model, f"{n_sets} sets")


def _sources(g, c, lk, n_src):
    """K/V batches in n_src buffers (6 / 3 / 3 batches, row strides 2C / 2C / 3C) like the view-sharded layout."""
    b0 = _bf(_randn(6 * lk, 2 * c, g=g))
    if n_src == 1:
        return [(b0[:, :c], b0[:, c:], 2 * c, 6)]
    b1 = _bf(_randn(3 * lk, 2 * c, g=g))
    b2 = _bf(_randn(3 * lk, 3 * c, g=g))
    return [(b0[:, :c], b0[:, c:], 2 * c, 6), (b1[:, :c], b1[:, c:], 2 * c, 3), (b2[:, c:2 * c], b2[:, 2 * c:], 3 * c, 3)]


def _entries(n_sets, n_src):
    """Rows 0..n_sets-1 have their empty slot at position i, row n_sets has none, row n_sets + 1 is all empty."""
    rows = []
    for i in range(n_sets + 2):
        row = []
        for s in range(n_sets):
            src = (i + s) % n_src
            empty = s == i or i == n_sets + 1
            row.append(None if empty else (src, (5 * i + 3 * s) % (6 if src == 0 else 3)))
        rows.append(row)
    return rows


def _kv_index(rows):
    return torch.tensor([[-1 if e is None else (e[0] << 24) | e[1] for e in row] for row in rows], dtype=torch.int32,
                        device=DEV)


@pytest.mark.parametrize("n_src", [1, 3])
@pytest.mark.parametrize("n_sets", range(1, 9))
@pytest.mark.parametrize("d", list(HEADS))
@pytest.mark.parametrize("kernel", ATTN_KERNELS)
def test_attention_sets_with_empty_slots(cuda_lib, monkeypatch, kernel, d, n_sets, n_src):
    monkeypatch.setenv("MDB_ATTN_KERNEL", kernel)
    g = _gen(100 + n_sets)
    heads = HEADS[d]
    c = heads * d
    lq, lk = 150, 140
    scale = d ** -0.5
    rows = _entries(n_sets, n_src)
    b = len(rows)
    q = _bf(_randn(b * lq, c, g=g))
    srcs = _sources(g, c, lk, n_src)
    out = Guarded(b * lq, c, ld=c + 16, col0=8)
    ops.attention_multi(q, srcs, b=b, heads=heads, lq=lq, lk=lk, d=d, ldq=c, scale=scale, kv_index=_kv_index(rows),
                        n_sets=n_sets, out=out.out)
    out.check(f"n_sets={n_sets}")

    def kv_of(i):
        return [(srcs[e[0]][0][e[1] * lk:(e[1] + 1) * lk], srcs[e[0]][1][e[1] * lk:(e[1] + 1) * lk]) for e in rows[i] if e]

    _close(out.out, _ref(q, kv_of, rows, heads, lq, d, scale), n_sets)
    assert torch.equal(out.out[(b - 1) * lq:], torch.zeros_like(out.out[(b - 1) * lq:]))  # all-empty row


@pytest.mark.parametrize("d", list(HEADS))
@pytest.mark.parametrize("kernel", ATTN_KERNELS)
def test_attention_empty_slots_are_bitwise_absent(cuda_lib, monkeypatch, kernel, d):
    """[a, -1, b] gives bit for bit [a, b], and [-1, a] bit for bit [a]."""
    monkeypatch.setenv("MDB_ATTN_KERNEL", kernel)
    g = _gen(9)
    heads = HEADS[d]
    c = heads * d
    b, lq, lk = 4, 200, 190
    q = _bf(_randn(b * lq, c, g=g))
    kv = _bf(_randn(6 * lk, 2 * c, g=g))

    def run(idx):
        t = torch.tensor(idx, dtype=torch.int32, device=DEV)
        return ops.attention(q, kv, kv[:, c:], b=b, b_kv=6, heads=heads, lq=lq, lk=lk, d=d, ldq=c, ldk=2 * c, ldv=2 * c,
                             scale=d ** -0.5, kv_index=t, n_sets=t.shape[1])
    pairs = [[5, 1], [0, 2], [3, 3], [4, 0]]
    assert torch.equal(run([[a, -1, bb] for a, bb in pairs]), run(pairs))
    assert torch.equal(run([[-1, a, -1, -1] for a, _ in pairs]), run([[a] for a, _ in pairs]))


@pytest.mark.parametrize("d", list(HEADS))
@pytest.mark.parametrize("dt,kernel", ATTN_DT_KERNELS)
def test_attention_kv_len(cuda_lib, monkeypatch, dt, kernel, d):
    """Per-batch key counts 0, 1, below one key tile, BN - 1 / BN / BN + 1, lk, and out-of-range values the kernel clamps;
    one set and three sets with an empty slot.  lk = 2 BN + 37 puts the 128-key tiles (d <= 64) past the KVRES kernel's
    256 keys: the varlen kernel without resident key tiles, in bf16 and f16."""
    monkeypatch.setenv("MDB_ATTN_KERNEL", kernel)
    g = _gen(10)
    heads = HEADS[d]
    c = heads * d
    bn = _block_n(kernel, d)
    lq, lk = 130, 2 * bn + 37
    lens = [0, 1, 17, bn - 1, bn, bn + 1, lk, -5, lk + 40]
    b = len(lens)
    scale = d ** -0.5
    q = _randn(b * lq, c, g=g).to(dt)
    kv = _randn(b * lk, 2 * c, g=g).to(dt)
    kv_len = torch.tensor(lens, dtype=torch.int32, device=DEV)
    eff = [min(max(x, 0), lk) for x in lens]
    out = Guarded(b * lq, c, dt, ld=c + 16, col0=8)
    ops.attention(q, kv, kv[:, c:], b=b, heads=heads, lq=lq, lk=lk, d=d, ldq=c, ldk=2 * c, ldv=2 * c, scale=scale,
                  kv_len=kv_len, out=out.out)
    out.check("kv_len")

    def kv_of(i):
        return [(kv[i * lk:i * lk + eff[i], :c], kv[i * lk:i * lk + eff[i], c:])] if eff[i] else []

    _close(out.out, _ref(q, kv_of, lens, heads, lq, d, scale, dt), 1)
    # three sets of which one empty, each set cut to its query batch's key count
    rows = [[(0, (i + 1) % b), None, (0, (i + 4) % b)] for i in range(b)]
    out3 = Guarded(b * lq, c, dt)
    ops.attention(q, kv, kv[:, c:], b=b, heads=heads, lq=lq, lk=lk, d=d, ldq=c, ldk=2 * c, ldv=2 * c, scale=scale,
                  kv_index=_kv_index(rows), n_sets=3, kv_len=kv_len, out=out3.out)
    out3.check("kv_len, three sets")

    def kv3(i):
        return [(kv[e[1] * lk:e[1] * lk + eff[i], :c], kv[e[1] * lk:e[1] * lk + eff[i], c:]) for e in rows[i] if e and eff[i]]

    _close(out3.out, _ref(q, kv3, rows, heads, lq, d, scale, dt), 3)
    # kv_len = lk everywhere is bit for bit the call without kv_len
    full = ops.attention(q, kv, kv[:, c:], b=b, heads=heads, lq=lq, lk=lk, d=d, ldq=c, ldk=2 * c, ldv=2 * c, scale=scale,
                         kv_len=torch.full((b,), lk, dtype=torch.int32, device=DEV))
    plain = ops.attention(q, kv, kv[:, c:], b=b, heads=heads, lq=lq, lk=lk, d=d, ldq=c, ldk=2 * c, ldv=2 * c, scale=scale)
    assert torch.equal(full, plain)


def test_attention_rejects_too_many_sets(cuda_lib):
    q = torch.zeros(128, 64, dtype=BF16, device=DEV)
    idx = torch.zeros(1, 9, dtype=torch.int32, device=DEV)
    with pytest.raises(Exception, match="n_sets"):
        ops.attention(q, q, q, b=1, heads=1, lq=128, lk=128, d=64, ldq=64, ldk=64, ldv=64, scale=0.125, kv_index=idx, n_sets=9)


# ------------------------------------------------------------------------------------------------------ whole networks
@torch.no_grad()
@pytest.mark.parametrize("rig", ["chain5_add", "ring5_concat", "ring8_3_add", "six_empty_add"])
def test_unet_rigs_vs_reference_fixture(cuda_lib, rig):
    g = golden("tiny_rigs.pt")
    nb, at = g["rigs"][rig]
    ucfg = replace(tiny_configs()[0], neighboring_view_pair=nb, neighboring_attn_type=at)
    v = g["scenes"] * len(nb)
    usd = arch.synthetic_state_dict(arch.unet_param_shapes(ucfg), g["seed"])
    un = UNet2DConditionModelMultiview(**asdict(ucfg))
    un.load_state_dict(usd)
    un = un.to(DEV)
    sample, ctx, t = g["sample"][:v].to(DEV), g["ctx"][:v].to(DEV), torch.tensor(g["t"], device=DEV)
    eps = un(sample, t, encoder_hidden_states=ctx).sample
    ub = {k: x.to(DEV, BF16) for k, x in usd.items()}
    yard = O.unet_forward(ub, ucfg, sample.bfloat16(), t, ctx.bfloat16())
    _check(f"rig {rig} eps", eps, g["eps"][rig], yard)


@torch.no_grad()
def test_unet_uneven_concat_matches_per_view_runs(cuda_lib):
    """'concat' on the 5-camera chain, where the reference cannot batch the uneven key counts: the engine's padded gather
    with kv_len gives, view by view, the attention over exactly that view's concatenated neighbours."""
    g = _gen(12)
    heads, d, L = 2, 32, 130
    c = heads * d
    counts = [2, 2, 2, 1, 1]
    V = 10
    kvv = _bf(_randn(V * L, 2 * c, g=g))
    q = _bf(_randn(V * L, c, g=g))
    idx = torch.tensor([[s * 5 + x for x in CHAIN5[i]] + [-1] * (2 - len(CHAIN5[i])) for s in range(2) for i in range(5)],
                       dtype=torch.int32, device=DEV)
    kvc = kvv.view(V, L, 2 * c)[idx.long()].reshape(V * 2 * L, 2 * c)
    lens = torch.tensor([counts[i % 5] * L for i in range(V)], dtype=torch.int32, device=DEV)
    out = ops.attention(q, kvc, kvc[:, c:], b=V, heads=heads, lq=L, lk=2 * L, d=d, ldq=c, ldk=2 * c, ldv=2 * c,
                        scale=d ** -0.5, kv_len=lens)
    for vi in range(V):
        nbk = torch.cat([kvv[(vi // 5 * 5 + x) * L:(vi // 5 * 5 + x + 1) * L] for x in CHAIN5[vi % 5]]).contiguous()
        one = ops.attention(q[vi * L:(vi + 1) * L], nbk, nbk[:, c:], b=1, heads=heads, lq=L, lk=nbk.shape[0], d=d, ldq=c,
                            ldk=2 * c, ldv=2 * c, scale=d ** -0.5)
        torch.testing.assert_close(out[vi * L:(vi + 1) * L].float(), one.float(), atol=1e-2, rtol=1e-2)


@torch.no_grad()
def test_sd15_chain5_add_vs_fp32_oracle(cuda_lib):
    """SD-1.5-size UNet on the 5-camera open chain ('add': two views with one neighbour, so the per-view connector bias)."""
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    ucfg = replace(arch.UNetConfig(), neighboring_view_pair=CHAIN5)
    usd = arch.synthetic_state_dict(arch.unet_param_shapes(ucfg), 21)
    un = UNet2DConditionModelMultiview(**asdict(ucfg))
    un.load_state_dict(usd)
    un = un.to(DEV, BF16)
    gg = torch.Generator().manual_seed(4)
    h, w = 28, 50
    sample = torch.randn(5, 4, h, w, generator=gg).to(DEV)
    ctx = torch.randn(5, 20, 768, generator=gg).to(DEV)
    t = torch.tensor(601, device=DEV)
    eps = un(sample.bfloat16(), t, encoder_hidden_states=ctx.bfloat16()).sample
    e32 = O.unet_forward({k: x.to(DEV) for k, x in usd.items()}, ucfg, sample, t, ctx)
    yard = O.unet_forward({k: x.to(DEV, BF16) for k, x in usd.items()}, ucfg, sample.bfloat16(), t, ctx.bfloat16())
    _check("sd15 chain5 add eps", eps, e32, yard)


@torch.no_grad()
@pytest.mark.parametrize("scheduler", ["ddim", "unipc"])
def test_denoiser_five_cameras_graph_vs_eager_and_oracle(cuda_lib, scheduler):
    """n_cam = 5 (chain rig), boxes, captions passed as embeddings, CFG: CUDA-graph replay bit for bit the eager loop, and
    both against the oracle pipeline."""
    from magicdrive_b200.synthetic import synthetic_inputs
    ucfg, ccfg = tiny_configs()
    ucfg = replace(ucfg, neighboring_view_pair=CHAIN5)
    usd = arch.synthetic_state_dict(arch.unet_param_shapes(ucfg), 41)
    csd = arch.synthetic_state_dict(arch.controlnet_param_shapes(ccfg), 42)
    un, cn = UNet2DConditionModelMultiview(**asdict(ucfg)), BEVControlNetModel(**asdict(ccfg))
    un.load_state_dict(usd)
    cn.load_state_dict(csd)
    un, cn = un.to(DEV), cn.to(DEV)
    inp = synthetic_inputs(1, 5, 10, 13, n_box=4, map_hw=52, seed=17, text_len=12)
    outs = []
    for graph in (False, True):
        pipe = BEVControlNetDenoiser(un, cn, use_cuda_graph=graph, scheduler=scheduler)
        outs.append(pipe(image=inp["bev_map"], camera_param=inp["camera_param"], prompt_embeds=inp["prompt_embeds"],
                         negative_prompt_embeds=inp["negative_prompt_embeds"], latents=inp["latents"], num_inference_steps=3,
                         guidance_scale=2.0, bev_controlnet_kwargs={"bboxes_3d_data": inp["bboxes_3d_data"]}))
    assert torch.equal(outs[0], outs[1])
    truth = O.denoise_loop(usd, csd, ucfg, ccfg, inp["latents"], inp["prompt_embeds"], inp["negative_prompt_embeds"],
                           inp["camera_param"], inp["bboxes_3d_data"], inp["bev_map"], 3, 2.0, scheduler=scheduler)
    assert outs[1].shape == truth.shape == (1, 5, 4, 10, 13)
    assert rel_l2(outs[1].cpu(), truth) < 2e-2, rel_l2(outs[1].cpu(), truth)
    assert (outs[1][:, 3] - outs[1][:, 4]).abs().max() > 1e-3
