"""Scene streams on the GPU: the attention kernel's resident-K/V multi-Q mode (a device key count with lk <= 256) against the
exact-lk launch bit for bit and against float64, the device collate at a capacity, and a stream of scenes with different box
counts through ONE capacity-mode denoiser (graphs on) against a default-mode call per scene, with launch and memory
accounting."""
from dataclasses import asdict

import pytest
import torch

pytestmark = pytest.mark.gpu

from magicdrive_b200 import arch, ops  # noqa: E402
from magicdrive_b200.input_prep import collate_on_device  # noqa: E402
from magicdrive_b200.pipeline import BEVControlNetDenoiser  # noqa: E402
from magicdrive_b200.synthetic import synthetic_inputs  # noqa: E402
from oracle import torch_oracle as O  # noqa: E402  (checker only)
from tests.common import golden, rel_l2, tiny_configs, tiny_state_dicts, to_dev  # noqa: E402
from tests.test_kernel_edges_gpu import ATTN_KERNELS, Guarded, _bf, _gen, _randn  # noqa: E402
from tests.test_model_gpu import _bf16_yardstick, _check, _models  # noqa: E402
from tests.test_rigs_gpu import _block_n, _close, _ref  # noqa: E402

DEV = "cuda"
LK = 256  # the largest lk that takes the resident mode
LENS = [0, 1, 63, 64, 65, 78, 98, 127, 128, 129, 237, LK]


@pytest.mark.parametrize("lq", [28, 91, 350, 1400])
@pytest.mark.parametrize("d", [40, 80, 160])
@pytest.mark.parametrize("kernel,multiq", [(k, "1") for k in ATTN_KERNELS] + [("tc2", "0")])
def test_resident_multi_q_is_bitwise_the_exact_lk_launch(cuda_lib, monkeypatch, kernel, multiq, d, lq):
    """Twelve batches with different key counts in one launch at lk = 256.  With 4 heads and lq >= 350 the grid exceeds the
    SMs, so CTAs walk several query tiles against their resident key tiles (or stream them where the count needs more
    tiles than the ring holds: head dim 160 from 193 keys).  K rows past a batch's count are NaN, and so are the V rows
    past its last walked key tile: tiles beyond the count are never loaded.  The V rows that share the last tile with
    counted keys are loaded and take weight 0, so they hold large finite values, as the denoiser's buffers hold null-token
    projections there."""
    monkeypatch.setenv("MDB_ATTN_KERNEL", kernel)
    monkeypatch.setenv("MDB_ATTN_MULTIQ", multiq)
    g = _gen(7 + d + lq)
    heads, b = 4, len(LENS)
    c = heads * d
    bn = _block_n(kernel, d)
    scale = d ** -0.5
    q = _bf(_randn(b * lq, c, g=g))
    kv = _bf(_randn(b * LK, 2 * c, g=g))
    dirty = kv.clone()
    for i, n in enumerate(LENS):
        rows = dirty[i * LK:(i + 1) * LK]
        rows[n:, :c] = float("nan")
        rows[n:, c:] = 3e4
        rows[-(-n // bn) * bn:, c:] = float("nan")
    out = Guarded(b * lq, c, ld=c + 16, col0=8)
    ops.attention(q, dirty, dirty[:, c:], b=b, heads=heads, lq=lq, lk=LK, d=d, ldq=c, ldk=2 * c, ldv=2 * c, scale=scale,
                  kv_len=torch.tensor(LENS, dtype=torch.int32, device=DEV), out=out.out)
    out.check(f"resident multi-Q d={d} lq={lq}")
    for i, n in enumerate(LENS):
        got = out.out[i * lq:(i + 1) * lq]
        if n == 0:
            assert not got.any(), "a batch without keys is written as zeros"
            continue
        ki = kv[i * LK:i * LK + n]
        exact = ops.attention(q[i * lq:(i + 1) * lq], ki, ki[:, c:], b=1, heads=heads, lq=lq, lk=n, d=d, ldq=c, ldk=2 * c,
                              ldv=2 * c, scale=scale)
        assert torch.equal(got, exact), (n, (got.float() - exact.float()).abs().max().item())

    def kv_of(i):
        return [(kv[i * LK:i * LK + LENS[i], :c], kv[i * LK:i * LK + LENS[i], c:])] if LENS[i] else []

    _close(out.out, _ref(q, kv_of, LENS, heads, lq, d, scale), 1)


def test_device_collate_at_capacity(cuda_lib):
    """collate_on_device(capacity=N) on the reference's six demo samples: the first `count` slots are the max_len=None result,
    the rest is padding, and `count` is the batch's longest visible list."""
    cases = golden("input_prep.pt")
    examples = [dict(gt_bboxes_3d=c["gt_bboxes_3d"], gt_labels_3d=c["gt_labels_3d"], lidar2camera=c["lidar2camera"],
                     img_aug_matrix=c["img_aug_matrix"], camera_intrinsics=c["camera_intrinsics"],
                     gt_masks_bev=torch.zeros(8, 20, 20)) for c in cases]
    for batch in ([0], [1, 4], list(range(len(cases)))):
        ex = [examples[i] for i in batch]
        ref = collate_on_device(ex, DEV)["kwargs"]["bboxes_3d_data"]
        assert ref["bboxes"].shape[2] == max(cases[i]["bboxes"].shape[1] for i in batch)  # the reference's batch max
        cap = collate_on_device(ex, DEV, capacity=64)
        bx = cap["kwargs"]["bboxes_3d_data"]
        n = ref["bboxes"].shape[2]
        assert bx["count"].dtype == torch.int32 and bx["count"].dim() == 0 and bx["count"].item() == n
        assert bx["bboxes"].shape[2] == bx["classes"].shape[2] == bx["masks"].shape[2] == 64
        for k in ("bboxes", "classes", "masks"):
            assert torch.equal(bx[k][:, :, :n], ref[k]), k
        assert not bx["masks"][:, :, n:].any() and not bx["bboxes"][:, :, n:].any()
        assert torch.equal(bx["counts"], ref["counts"])
    with pytest.raises(ValueError, match="max_len or capacity"):
        collate_on_device(ex, DEV, max_len=64, capacity=64)


def _kw(inp, steps, **extra):
    return dict(image=inp["bev_map"], camera_param=inp["camera_param"], prompt_embeds=inp["prompt_embeds"],
                negative_prompt_embeds=inp["negative_prompt_embeds"], latents=inp["latents"], num_inference_steps=steps,
                guidance_scale=2.0, bev_controlnet_kwargs={"bboxes_3d_data": inp["bboxes_3d_data"]}, **extra)


def _stream_vs_calls(un, cn, usd, csd, ucfg, ccfg, scenes, steps, capacity, scheduler, oracle_for):
    default = BEVControlNetDenoiser(un, cn, use_cuda_graph=True, scheduler=scheduler)
    ones = [default(**_kw(inp, steps)) for inp in scenes]  # a new state and new graphs per box count
    default.release_graph()
    cap = BEVControlNetDenoiser(un, cn, use_cuda_graph=True, scheduler=scheduler, box_capacity=capacity)
    state = None
    for i, (inp, one) in enumerate(zip(scenes, ones)):
        out = cap(**_kw(inp, steps))
        state = state or cap._static
        assert cap._static is state
        assert rel_l2(out, one) < 2e-2
        if i not in oracle_for:
            continue
        di = to_dev(inp, DEV)

        def loop(usd_, csd_, dt):
            d = to_dev(di, DEV, dt)
            return O.denoise_loop(usd_, csd_, ucfg, ccfg, d["latents"], d["prompt_embeds"], d["negative_prompt_embeds"],
                                  d["camera_param"], d["bboxes_3d_data"], d["bev_map"], steps, 2.0, scheduler=scheduler)
        truth = loop({k: v.to(DEV) for k, v in usd.items()}, {k: v.to(DEV) for k, v in csd.items()}, torch.float32)
        yard = _bf16_yardstick(loop, usd, csd)
        n = 0 if inp["bboxes_3d_data"] is None else inp["bboxes_3d_data"]["bboxes"].shape[2]
        _check(f"scene stream, capacity {capacity}, {n} boxes ({scheduler})", out, truth, yard)
        _check(f"scene stream, default mode, {n} boxes ({scheduler})", one, truth, yard)


@torch.no_grad()
@pytest.mark.parametrize("scheduler", ["ddim", "unipc"])
def test_tiny_stream_vs_default_mode_and_oracle(cuda_lib, scheduler):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    ucfg, ccfg = tiny_configs()
    usd, csd = tiny_state_dicts(21)
    un, cn = _models(ucfg, ccfg, usd, csd)
    scenes = [synthetic_inputs(1, 6, 10, 13, n_box=n, map_hw=52, seed=60 + n) for n in (5, 0, 9, 1, 3)]
    _stream_vs_calls(un, cn, usd, csd, ucfg, ccfg, scenes, 3, 9, scheduler, oracle_for=range(len(scenes)))


@torch.no_grad()
def test_sd15_stream_vs_default_mode_and_oracle(cuda_lib):
    """SD-1.5 size (224 x 400, V = 12 with guidance), box counts 4 / 49 / 23 at capacity 159 (1 + 77 + 159 = 237 keys)."""
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    ucfg, ccfg = arch.UNetConfig(), arch.ControlNetConfig()
    usd = arch.synthetic_state_dict(arch.unet_param_shapes(ucfg), 11)
    csd = arch.synthetic_state_dict(arch.controlnet_param_shapes(ccfg), 12)
    un, cn = _models(ucfg, ccfg, usd, csd, torch.bfloat16)
    scenes = [synthetic_inputs(1, 6, 28, 50, n_box=n, map_hw=200, seed=70 + n) for n in (4, 49, 23)]
    _stream_vs_calls(un, cn, usd, csd, ucfg, ccfg, scenes, 2, 159, "unipc", oracle_for=[1])


@torch.no_grad()
def test_sd15_stream_is_bitwise_default_mode_without_split_k(cuda_lib, monkeypatch):
    """The context's K/V GEMM has more rows at capacity, and split-K is the one place where its plan, and so a summation
    order, can follow the row count.  With single CTAs without split-K (kernel_variant 4) on both sides every row is the
    same sum, and the attention is bitwise the exact-lk launch: the final latents are equal bit for bit."""
    monkeypatch.setattr(ops, "GEMM_VARIANT", 4)
    ucfg, ccfg = arch.UNetConfig(), arch.ControlNetConfig()
    usd = arch.synthetic_state_dict(arch.unet_param_shapes(ucfg), 11)
    csd = arch.synthetic_state_dict(arch.controlnet_param_shapes(ccfg), 12)
    un, cn = _models(ucfg, ccfg, usd, csd, torch.bfloat16)
    scenes = [synthetic_inputs(1, 6, 28, 50, n_box=n, map_hw=200, seed=80 + n) for n in (30, 7)]
    default = BEVControlNetDenoiser(un, cn, use_cuda_graph=True, scheduler="unipc")
    ones = [default(**_kw(inp, 2)) for inp in scenes]
    default.release_graph()
    cap = BEVControlNetDenoiser(un, cn, use_cuda_graph=True, scheduler="unipc", box_capacity=159)
    for inp, one in zip(scenes, ones):
        out = cap(**_kw(inp, 2))
        assert torch.equal(out, one), (inp["bboxes_3d_data"]["bboxes"].shape[2], (out - one).abs().max().item())


@torch.no_grad()
def test_stream_replays_two_graphs_without_allocating(cuda_lib):
    """From the second scene on a call is the condition graph plus `steps` replays of the step graph: nothing is launched
    outside them but the in-place refresh of the inputs, and device memory does not grow over ten scenes."""
    ucfg, ccfg = tiny_configs()
    usd, csd = tiny_state_dicts(21)
    un, cn = _models(ucfg, ccfg, usd, csd)
    cap = BEVControlNetDenoiser(un, cn, use_cuda_graph=True, scheduler="unipc", box_capacity=12)
    steps = 4
    scenes = [synthetic_inputs(1, 6, 10, 13, n_box=n, map_hw=52, seed=90 + n) for n in (3, 7, 12, 0, 5, 1, 9, 2, 11, 4, 8, 6)]
    graphs = state = mem = None
    for i, inp in enumerate(scenes):
        ops.reset_launch_count()
        out = cap(**_kw(inp, steps))
        launched = ops.launch_count()  # kernels issued through ops outside a graph replay
        torch.cuda.synchronize()
        assert torch.isfinite(out).all()
        if i == 1:  # the condition graph was captured on this first refresh of the state
            graphs, state = (cap._graph, cap._cond_graph), cap._static
            mem = torch.cuda.memory_allocated()
        elif i > 1:
            assert (cap._graph, cap._cond_graph) == graphs and cap._static is state
            # the schedule's two time-embedding tables (4 small kernels per network), as in default mode
            assert launched == 8, (i, launched)
            assert torch.cuda.memory_allocated() <= mem, (i, torch.cuda.memory_allocated(), mem)
