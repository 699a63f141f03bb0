"""TEST INFRASTRUCTURE ONLY -- tests/golden/tiny_attn_types.pt: the REFERENCE UNet2DConditionModelMultiview (via oracle/ref_shim.py)
with neighboring_attn_type = "concat" and "self" (magicdrive/networks/blocks.py:122-138, 209-211), tiny config, two scenes.

Run in the build container (needs /root/reference):  python -m oracle.make_golden_attn_types
Weights are rebuilt on both sides from arch.synthetic_state_dict(seed); stored: seeded inputs and the reference outputs (fp32).
"""
import os
from dataclasses import replace

import torch

from magicdrive_b200 import arch
from oracle import ref_shim
from oracle.make_golden import OUT, tiny_configs


@torch.no_grad()
def main():
    ucfg0, ccfg = tiny_configs()
    seed, scenes, n_cam, h, w, lc = 23, 2, 6, 10, 13, 9
    g = torch.Generator().manual_seed(5)
    sample = torch.randn(scenes * n_cam, 4, h, w, generator=g)
    ctx = torch.randn(scenes * n_cam, lc, ucfg0.cross_attention_dim, generator=g)
    out = dict(seed=seed, shape=(scenes, n_cam, h, w), t=337, sample=sample, ctx=ctx, eps={})
    for at in ("concat", "self"):
        ucfg = replace(ucfg0, neighboring_attn_type=at)
        mv, _ = ref_shim.build_reference_models(ucfg, ccfg)
        usd = arch.synthetic_state_dict(arch.unet_param_shapes(ucfg), seed)
        mv.load_state_dict(usd, strict=True)
        out["eps"][at] = mv(sample, torch.tensor(337), encoder_hidden_states=ctx).sample.clone()
        print(at, out["eps"][at].shape, float(out["eps"][at].abs().mean()))
    # ControlNet with guess_mode=True, conditioning_scale 0.7 (unet_addon_rawbox.py:897-905): inputs of tiny_forward.pt
    from oracle.make_golden import load_ref
    from tests.common import golden, save_golden
    gf = golden("tiny_forward.pt")
    _, cn, _, _ = load_ref(ucfg0, ccfg, seed=gf["seed"])
    inp = gf["inputs"]
    lat5 = torch.stack([inp["latents"]] * n_cam, 1)
    down, mid, _ = cn(lat5, torch.tensor([gf["t"]]), inp["camera_param"], inp["bboxes_3d_data"], inp["prompt_embeds"], inp["bev_map"],
                      conditioning_scale=0.7, guess_mode=True, return_dict=False)
    out["guess_mode"] = dict(inputs_from="tiny_forward.pt", conditioning_scale=0.7, down=[d.clone() for d in down], mid=mid.clone())
    # BEVControlNetConditioningEmbeddingPlus (map_embedder.py:79-126; configs/exp/272x736.yaml:16-22): a 52 x 60 map pooled to the
    # 10 x 13 latent grid; the embedder's own output and the ControlNet's mid residual with it
    mpar = dict(conditioning_embedding_size=[h, w], conditioning_size=[8, 52, 60], block_out_channels=[16, 32, 96, 256])
    ccfg_p = replace(ccfg, map_size=(8, 52, 60), map_embedding_size=(h, w))
    _, cnp = ref_shim.build_reference_models(ucfg0, ccfg_p, map_embedder_cls="magicdrive.networks.map_embedder."
                                             "BEVControlNetConditioningEmbeddingPlus", map_embedder_param=mpar)
    csd_p = arch.synthetic_state_dict(arch.controlnet_param_shapes(ccfg_p), seed + 1)
    cnp.load_state_dict(csd_p, strict=True)
    bev = torch.randn(1, 8, 52, 60, generator=g)
    emb = cnp.controlnet_cond_embedding(bev)
    down, mid, _ = cnp(lat5[:1], torch.tensor([gf["t"]]), inp["camera_param"][:1], None, inp["prompt_embeds"][:1], bev,
                       return_dict=False)
    out["map_plus"] = dict(seed=seed + 1, bev_map=bev, embedding=emb.clone(), mid=mid.clone(), down0=down[0].clone(),
                           inputs_from="tiny_forward.pt")
    save_golden(out, "tiny_attn_types.pt")


if __name__ == "__main__":
    main()
