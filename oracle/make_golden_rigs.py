"""TEST INFRASTRUCTURE ONLY -- tests/golden/tiny_rigs.pt: the REFERENCE UNet2DConditionModelMultiview (via oracle/ref_shim.py)
on camera rigs other than nuScenes' six-camera ring (neighboring_view_pair, magicdrive/networks/blocks.py:106-142, 209-218),
tiny config, two scenes; plus one ControlNet + UNet forward with camera and box conditioning at n_cam = 5.

Run in the build container (needs /root/reference):  python -m oracle.make_golden_rigs
Weights are rebuilt on both sides from arch.synthetic_state_dict(seed); stored: seeded inputs and the reference outputs (fp32).
"""
import os
from dataclasses import replace

import torch

from magicdrive_b200 import arch
from magicdrive_b200.synthetic import synthetic_inputs
from oracle import ref_shim
from oracle.make_golden import OUT, load_ref, tiny_configs

CHAIN5 = {0: [1, 2], 1: [0, 3], 2: [0, 4], 3: [1], 4: [2]}  # open chain: the outer cameras see one neighbour
RING5 = {i: [(i + 1) % 5, (i - 1) % 5] for i in range(5)}
RING8_3 = {i: [(i - 1) % 8, (i + 1) % 8, (i + 4) % 8] for i in range(8)}  # ring plus the opposite view
SIX_EMPTY = {0: [5, 1], 1: [0, 2], 2: [1, 3], 3: [], 4: [3, 5], 5: [4, 0]}  # view 3 attends to no neighbour
# "concat" with uneven neighbour counts (CHAIN5) is absent: the reference stacks every view's concatenated keys into one
# batch (blocks.py:122-133) and raises there, so it has no output to pin
RIGS = {"chain5_add": (CHAIN5, "add"), "ring5_concat": (RING5, "concat"), "ring8_3_add": (RING8_3, "add"),
        "six_empty_add": (SIX_EMPTY, "add")}


@torch.no_grad()
def main():
    ucfg0, ccfg = tiny_configs()
    seed, scenes, h, w, lc = 29, 2, 10, 13, 4
    g = torch.Generator().manual_seed(11)
    sample = torch.randn(scenes * 8, 4, h, w, generator=g)  # rig r uses the first scenes * n_cam views
    ctx = torch.randn(scenes * 8, lc, ucfg0.cross_attention_dim, generator=g)
    out = dict(seed=seed, scenes=scenes, t=413, sample=sample, ctx=ctx, rigs={}, eps={})
    for name, (nb, at) in RIGS.items():
        ucfg = replace(ucfg0, neighboring_view_pair=nb, neighboring_attn_type=at)
        mv, _ = ref_shim.build_reference_models(ucfg, ccfg)
        mv.load_state_dict(arch.synthetic_state_dict(arch.unet_param_shapes(ucfg), seed), strict=True)
        v = scenes * len(nb)
        out["rigs"][name] = (nb, at)
        out["eps"][name] = mv(sample[:v], torch.tensor(413), encoder_hidden_states=ctx[:v]).sample.clone()
        print(name, tuple(out["eps"][name].shape), float(out["eps"][name].abs().mean()))
    # ControlNet (camera + box tokens, BEV map) + UNet on the 5-camera chain, one scene
    ucfg = replace(ucfg0, neighboring_view_pair=CHAIN5)
    mv, cn, _, _ = load_ref(ucfg, ccfg, seed=seed)
    inp = synthetic_inputs(1, 5, h, w, n_box=4, map_hw=52, seed=13, text_len=6)
    lat5 = torch.stack([inp["latents"]] * 5, 1)
    t = torch.tensor([557])
    down, mid, ctx5 = cn(lat5, t, inp["camera_param"], inp["bboxes_3d_data"], inp["prompt_embeds"], inp["bev_map"],
                         return_dict=False)
    eps = mv(lat5.reshape(-1, 4, h, w), t[0], encoder_hidden_states=ctx5, down_block_additional_residuals=down,
             mid_block_additional_residual=mid).sample
    out["controlnet_chain5"] = dict(seed=seed, t=557, inputs={k: v for k, v in inp.items() if k != "negative_prompt_embeds"},
                                    mid=mid.clone(), eps=eps.clone())
    print("controlnet_chain5", tuple(eps.shape), float(eps.abs().mean()))
    torch.save(out, os.path.join(OUT, "tiny_rigs.pt"))
    print("tiny_rigs.pt", os.path.getsize(os.path.join(OUT, "tiny_rigs.pt")) // 1024, "KiB")


if __name__ == "__main__":
    main()
