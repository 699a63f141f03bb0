"""Camera rigs other than nuScenes' six-camera ring (neighboring_view_pair of any size, any neighbour count per view) on CPU:
the oracle against the reference's own outputs (tests/golden/tiny_rigs.pt, oracle/make_golden_rigs.py), the engine's host
side through tests/ops_emulator.py against the oracle, and the constructor / view-sharding validation."""
from dataclasses import asdict, replace

import pytest
import torch

from magicdrive_b200 import arch, models
from magicdrive_b200.dist import ShardPlan
from oracle import torch_oracle as O
from tests import ops_emulator
from tests.common import golden, rel_l2, tiny_configs

RIGS = ["chain5_add", "ring5_concat", "ring8_3_add", "six_empty_add"]
CHAIN5 = {0: [1, 2], 1: [0, 3], 2: [0, 4], 3: [1], 4: [2]}


def _bf16_exact(sd):
    return {k: (v.to(torch.bfloat16).float() if v.is_floating_point() else v) for k, v in sd.items()}


@pytest.fixture
def emulated(monkeypatch):
    ops_emulator.install(monkeypatch)
    from magicdrive_b200 import engine
    monkeypatch.setattr(engine._Weights, "fold_dtype", torch.float32)


def _rig(g, name):
    nb, at = g["rigs"][name]
    ucfg = replace(tiny_configs()[0], neighboring_view_pair=nb, neighboring_attn_type=at)
    v = g["scenes"] * len(nb)
    return ucfg, g["sample"][:v], g["ctx"][:v]


@torch.no_grad()
@pytest.mark.parametrize("rig", RIGS)
def test_oracle_reproduces_reference_rigs(rig):
    g = golden("tiny_rigs.pt")
    ucfg, sample, ctx = _rig(g, rig)
    usd = arch.synthetic_state_dict(arch.unet_param_shapes(ucfg), g["seed"])
    eps = O.unet_forward(usd, ucfg, sample, torch.tensor(g["t"]), ctx)
    torch.testing.assert_close(eps, g["eps"][rig], rtol=1e-3, atol=1e-4)


@torch.no_grad()
def test_oracle_reproduces_reference_controlnet_unet_five_cameras():
    g = golden("tiny_rigs.pt")
    c = g["controlnet_chain5"]
    ucfg, ccfg = tiny_configs()
    ucfg = replace(ucfg, neighboring_view_pair=CHAIN5)
    usd = arch.synthetic_state_dict(arch.unet_param_shapes(ucfg), c["seed"])
    csd = arch.synthetic_state_dict(arch.controlnet_param_shapes(ccfg), c["seed"] + 1)
    inp = c["inputs"]
    lat5 = torch.stack([inp["latents"]] * 5, 1)
    t = torch.tensor([c["t"]])
    d, m, ctx = O.controlnet_forward(csd, ccfg, lat5, t, inp["camera_param"], inp["bboxes_3d_data"], inp["prompt_embeds"],
                                     inp["bev_map"])
    eps = O.unet_forward(usd, ucfg, lat5.reshape(-1, 4, *lat5.shape[-2:]), t[0], ctx, d, m)
    torch.testing.assert_close(m, c["mid"], rtol=1e-3, atol=1e-4 * max(1.0, c["mid"].abs().max().item()))
    torch.testing.assert_close(eps, c["eps"], rtol=1e-3, atol=1e-4)


@torch.no_grad()
@pytest.mark.parametrize("rig", RIGS)
def test_engine_through_emulated_operators_matches_the_oracle_on_rigs(emulated, rig):
    g = golden("tiny_rigs.pt")
    ucfg, sample, ctx = _rig(g, rig)
    usd = _bf16_exact(arch.synthetic_state_dict(arch.unet_param_shapes(ucfg), g["seed"]))
    un = models.UNet2DConditionModelMultiview(**asdict(ucfg))
    un.load_state_dict(usd)
    eps = un(sample, torch.tensor(g["t"]), encoder_hidden_states=ctx).sample
    ref = O.unet_forward(usd, ucfg, sample, torch.tensor(g["t"]), ctx)
    assert eps.shape == ref.shape and rel_l2(eps, ref) < 3e-3, rel_l2(eps, ref)
    assert rel_l2(eps, g["eps"][rig]) < 2e-2


@torch.no_grad()
def test_engine_through_emulated_operators_controlnet_unet_five_cameras(emulated):
    g = golden("tiny_rigs.pt")
    c = g["controlnet_chain5"]
    ucfg, ccfg = tiny_configs()
    ucfg = replace(ucfg, neighboring_view_pair=CHAIN5)
    usd = _bf16_exact(arch.synthetic_state_dict(arch.unet_param_shapes(ucfg), c["seed"]))
    csd = _bf16_exact(arch.synthetic_state_dict(arch.controlnet_param_shapes(ccfg), c["seed"] + 1))
    un, cn = models.UNet2DConditionModelMultiview(**asdict(ucfg)), models.BEVControlNetModel(**asdict(ccfg))
    un.load_state_dict(usd)
    cn.load_state_dict(csd)
    inp = c["inputs"]
    lat5 = torch.stack([inp["latents"]] * 5, 1)
    t = torch.tensor([c["t"]])
    down, mid, ctx = cn(lat5, t, inp["camera_param"], inp["bboxes_3d_data"], inp["prompt_embeds"], inp["bev_map"],
                        return_dict=False)
    eps = un(lat5.reshape(-1, 4, *lat5.shape[-2:]), t[0], encoder_hidden_states=ctx, down_block_additional_residuals=down,
             mid_block_additional_residual=mid).sample
    assert rel_l2(eps, c["eps"]) < 2e-2 and rel_l2(mid, c["mid"]) < 2e-2


@torch.no_grad()
def test_uneven_concat_gathers_each_views_own_neighbours():
    """'concat' with uneven neighbour counts: view v's gathered keys are its own neighbours' tokens followed by padding that
    the per-view key count k_v * L cuts off (mdb_attention_varlen)."""
    from magicdrive_b200 import engine as E
    ucfg = replace(tiny_configs()[0], neighboring_view_pair=CHAIN5, neighboring_attn_type="concat")
    net = E.UNetEngine(ucfg, arch.synthetic_state_dict(arch.unet_param_shapes(ucfg), 3), "cpu")
    assert net.kv_index(10).tolist()[3] == [1, -1] and net.kv_index(10).tolist()[5] == [6, 7]
    assert net.kv_len(10, 7).tolist() == [14, 14, 14, 7, 7] * 2


def test_kv_index_and_connector_bias_per_rig():
    from magicdrive_b200 import engine as E
    ucfg = replace(tiny_configs()[0], neighboring_view_pair={0: [1, 2, 3], 1: [0], 2: [], 3: [0, 1]})
    sd = arch.synthetic_state_dict(arch.unet_param_shapes(ucfg), 3)
    net = E.UNetEngine(ucfg, sd, "cpu")
    assert net.kv_index(8).tolist() == [[1, 2, 3], [0, -1, -1], [-1, -1, -1], [0, 1, -1],
                                        [5, 6, 7], [4, -1, -1], [-1, -1, -1], [4, 5, -1]]
    blk = net.transformers[0].prefix + ".transformer_blocks.0"
    rb = net.W.connector_rowbias(blk, [3, 1, 0, 2])
    wc, bc = sd[blk + ".connector.weight"], sd[blk + ".connector.bias"]
    cb = wc @ sd[blk + ".attn4.to_out.0.bias"]
    for v, k in enumerate([3, 1, 0, 2]):
        torch.testing.assert_close(rb[v], k * cb + bc, rtol=1e-6, atol=1e-6)
    ring = E.UNetEngine(tiny_configs()[0], arch.synthetic_state_dict(arch.unet_param_shapes(tiny_configs()[0]), 3), "cpu")
    assert ring.kv_index(12).shape == (12, 2) and ring._uniform_neighbors()  # nuScenes: today's [V, 2], shared bias


@pytest.mark.parametrize("nb,at,view", [
    ({0: [1], 2: [0]}, "add", "keys"),                    # keys not 0..n_cam-1
    ({0: [1], 1: [2]}, "add", "[1]"),                     # neighbour out of range
    ({0: [1], 1: [-1]}, "add", "[1]"),
    ({i: [(i + 1) % 10] * (9 if i == 4 else 1) for i in range(10)}, "add", "[4]"),  # more than MDB_ATT_MAX_SETS
    ({0: [1], 1: []}, "concat", "[1]"),                   # empty list under concat
])
def test_constructor_rejects_rigs_the_engine_cannot_run(nb, at, view):
    ucfg = replace(tiny_configs()[0], neighboring_view_pair=nb, neighboring_attn_type=at)
    with pytest.raises(ValueError, match=view.replace("[", r"\[").replace("]", r"\]")):
        models.UNet2DConditionModelMultiview(**asdict(ucfg))


def test_constructor_accepts_general_rigs():
    for nb, at in ((CHAIN5, "add"), (CHAIN5, "concat"), ({0: [1], 1: []}, "add"),
                   ({i: [(i + 1) % 9] * 8 for i in range(9)}, "add"), (CHAIN5, "self")):
        models.UNet2DConditionModelMultiview(**asdict(replace(tiny_configs()[0], neighboring_view_pair=nb,
                                                              neighboring_attn_type=at)))


def test_view_sharding_rejects_rigs_without_two_neighbours_per_view():
    with pytest.raises(ValueError, match="exactly two neighbours"):
        ShardPlan(0, 2, 5, False, [CHAIN5[i] for i in range(5)])
    ring8_3 = [[(i - 1) % 8, (i + 1) % 8, (i + 4) % 8] for i in range(8)]
    with pytest.raises(ValueError, match="exactly two neighbours"):
        ShardPlan(0, 2, 8, False, ring8_3)
    ShardPlan(0, 2, 5, False, [[(i - 1) % 5, (i + 1) % 5] for i in range(5)])  # a 5-camera ring is fine
