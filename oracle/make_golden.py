"""TEST INFRASTRUCTURE ONLY — generate tests/golden/*.pt by running the REFERENCE ITSELF (via oracle/ref_shim.py).

Run in the build container (needs /root/reference):  python -m oracle.make_golden
Weights are not stored: both sides rebuild them from parameter names with arch.synthetic_state_dict(seed).
Stored: seeded inputs (small) and the reference outputs in fp32.
"""
import os
import sys

import torch

from magicdrive_b200 import arch
from oracle import ref_shim
from tests.common import save_golden

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def tiny_configs():
    u = arch.UNetConfig(block_out_channels=(64, 128), down_block_types=("CrossAttnDownBlock2D", "DownBlock2D"),
                        up_block_types=("UpBlock2D", "CrossAttnUpBlock2D"), layers_per_block=1, attention_head_dim=2)
    c = arch.ControlNetConfig(block_out_channels=(64, 128), down_block_types=("CrossAttnDownBlock2D", "DownBlock2D"),
                              layers_per_block=1, attention_head_dim=2, map_size=(8, 52, 52))
    return u, c  # BEV map 52x52 -> 10x13 latent grid (odd width: exercises the non-integer nearest resize)


from magicdrive_b200.synthetic import synthetic_inputs  # noqa: E402,F401  (shared seeded input generator)


def load_ref(ucfg, ccfg, seed):
    mv, cn = ref_shim.build_reference_models(ucfg, ccfg)
    usd = arch.synthetic_state_dict(arch.unet_param_shapes(ucfg), seed)
    csd = arch.synthetic_state_dict(arch.controlnet_param_shapes(ccfg), seed + 1)
    mv.load_state_dict(usd, strict=True)
    cn.load_state_dict(csd, strict=True)
    return mv, cn, usd, csd


@torch.no_grad()
def main():
    os.makedirs(OUT, exist_ok=True)
    torch.manual_seed(0)
    ucfg, ccfg = tiny_configs()
    mv, cn, usd, csd = load_ref(ucfg, ccfg, seed=7)
    scenes, n_cam, h, w = 1, 6, 10, 13
    inp = synthetic_inputs(scenes, n_cam, h, w, n_box=5, map_hw=52, seed=3)

    # ---- golden 1: one ControlNet + UNet forward (no CFG), t = 481
    lat5 = torch.stack([inp["latents"]] * n_cam, 1)
    t = torch.tensor([481])
    down, mid, ctx = cn(lat5, t, inp["camera_param"], inp["bboxes_3d_data"], inp["prompt_embeds"], inp["bev_map"],
                        return_dict=False)
    eps = mv(lat5.reshape(-1, 4, h, w), t[0], encoder_hidden_states=ctx, down_block_additional_residuals=down,
             mid_block_additional_residual=mid).sample
    eps_noctrl = mv(lat5.reshape(-1, 4, h, w), t[0], encoder_hidden_states=ctx).sample
    save_golden(dict(inputs=inp, t=481, down=[d.clone() for d in down], mid=mid, ctx=ctx, eps=eps,
                     eps_noctrl=eps_noctrl, seed=7, shape=(scenes, n_cam, h, w)), "tiny_forward.pt")

    # ---- golden 2: the reference pipeline loop (CFG 2.0, 3 DDIM steps, boxes + map)
    R = ref_shim.load()

    class Pipe(R.StableDiffusionBEVControlNetPipeline):
        def prepare_extra_step_kwargs(self, generator, eta):  # DDIM eta=0 is deterministic (SURVEY.md §0.3)
            return {"eta": eta}

    class TextStub(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.p = torch.nn.Parameter(torch.zeros(1))
        dtype = torch.float32

        @property
        def device(self):
            return self.p.device

    vae = R.AutoencoderKL(block_out_channels=[32, 64, 64, 64], down_block_types=["DownEncoderBlock2D"] * 4,
                          up_block_types=["UpDecoderBlock2D"] * 4, latent_channels=4)
    sched = R.DDIMScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False,
                            set_alpha_to_one=False, steps_offset=1)
    pipe = Pipe(vae=vae, text_encoder=TextStub(), unet=mv, controlnet=cn, scheduler=sched, tokenizer=None)
    pipe.set_progress_bar_config(disable=True)
    out = pipe(prompt=None, image=inp["bev_map"], camera_param=inp["camera_param"], height=h * 8, width=w * 8,
               num_inference_steps=3, guidance_scale=2.0, latents=inp["latents"].clone(),
               prompt_embeds=inp["prompt_embeds"], negative_prompt_embeds=inp["negative_prompt_embeds"],
               output_type="latent", bev_controlnet_kwargs={"bboxes_3d_data": inp["bboxes_3d_data"]})
    torch.save(dict(inputs=inp, steps=3, guidance=2.0, latents_out=out.images, seed=7), os.path.join(OUT, "tiny_pipeline.pt"))

    # ---- golden 3: encoders alone on realistic value ranges (camera intrinsics ~1.2e3, boxes +-50 m)
    cam_emb = cn._embed_camera(inp["camera_param"])
    box = {k: v.reshape(scenes * n_cam, *v.shape[2:]) for k, v in inp["bboxes_3d_data"].items()}
    box_emb = cn.bbox_embedder(**box)
    map_emb = cn.controlnet_cond_embedding(inp["bev_map"])
    uncond = cn.uncond_cam_param([2, n_cam])
    torch.save(dict(camera_param=inp["camera_param"], cam_emb=cam_emb, boxes=box, box_emb=box_emb,
                    bev_map=inp["bev_map"].to(torch.uint8), map_emb=map_emb, uncond_cam=uncond, seed=7),
               os.path.join(OUT, "tiny_encoders.pt"))
    for f in sorted(os.listdir(OUT)):
        print(f, os.path.getsize(os.path.join(OUT, f)) // 1024, "KiB")


if __name__ == "__main__":
    sys.exit(main())
