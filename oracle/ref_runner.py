"""TEST / MEASUREMENT INFRASTRUCTURE ONLY — drive the UNMODIFIED reference (StableDiffusionBEVControlNetPipeline with its
own UNet2DConditionModelMultiview + BEVControlNetModel, loaded through oracle/ref_shim.py from /root/reference or from the
oracle/_ref snapshot) on this repo's synthetic workload, and time its denoising steps.

Used by `bench.py --impl reference` (CPU, fp32: the reference arm), by bench.py's `gpu_reference` field (same GPU, bf16,
diffusers' AttnProcessor2_0 = torch SDPA, since the vendored xformers only dispatches below compute capability 9.0: SURVEY.md section 0.4) and by
tests.  The product never imports this module.
"""
import time

import torch

from magicdrive_b200 import arch
from oracle import ref_shim


def available() -> bool:
    return ref_shim.available()


def build_pipeline(res="224x400", device="cpu", dtype=torch.float32, seeds=(11, 12)):
    """Reference pipeline at the SD-1.5 config with the bench's seeded random weights (arch.synthetic_state_dict)."""
    R = ref_shim.load()
    ucfg = arch.UNetConfig()
    ccfg = arch.ControlNetConfig(map_size=(8, 200, 200) if res == "224x400" else (8, 400, 400))
    img = (224, 400) if res == "224x400" else (424, 800)
    mv, cn = ref_shim.build_reference_models(ucfg, ccfg, img_size=img)
    mv.load_state_dict(arch.synthetic_state_dict(arch.unet_param_shapes(ucfg), seeds[0]), strict=True)
    cn.load_state_dict(arch.synthetic_state_dict(arch.controlnet_param_shapes(ccfg), seeds[1]), strict=True)
    mv, cn = mv.to(device, dtype), cn.to(device, dtype)

    class Pipe(R.StableDiffusionBEVControlNetPipeline):
        def prepare_extra_step_kwargs(self, generator, eta):  # DDIM eta = 0 is deterministic (SURVEY.md section 0.3)
            return {"eta": eta}

    class TextStub(torch.nn.Module):  # prompt embeddings are passed in; the pipeline only reads dtype / device
        def __init__(self):
            super().__init__()
            self.p = torch.nn.Parameter(torch.zeros(1))

        @property
        def dtype(self):
            return self.p.dtype

        @property
        def device(self):
            return self.p.device

    vae = R.AutoencoderKL(block_out_channels=[32, 64, 64, 64], down_block_types=["DownEncoderBlock2D"] * 4,
                          up_block_types=["UpDecoderBlock2D"] * 4, latent_channels=4)
    sched = R.DDIMScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear", clip_sample=False,
                            set_alpha_to_one=False, steps_offset=1)
    pipe = Pipe(vae=vae.to(device, dtype), text_encoder=TextStub().to(device, dtype), unet=mv, controlnet=cn, scheduler=sched,
                tokenizer=None)
    pipe.set_progress_bar_config(disable=True)
    return pipe


def _to(x, device, dtype):
    if isinstance(x, dict):
        return {k: _to(v, device, dtype) for k, v in x.items()}
    if torch.is_tensor(x):
        return x.to(device, dtype) if x.is_floating_point() else x.to(device)
    return x


@torch.no_grad()
def time_steps(pipe, inp, h, w, steps, warmup, device="cpu", dtype=torch.float32, guidance_scale=2.0):
    """Run the reference pipeline's own __call__ (pipeline_bev_controlnet.py:114-470) for warmup + steps denoising steps
    and return (seconds per step over the last `steps`, latents).  Step boundaries come from the pipeline's `callback`."""
    inp = _to(inp, device, dtype)
    marks = []
    cuda = torch.device(device).type == "cuda"

    def cb(i, t, latents):
        if cuda:
            torch.cuda.synchronize()
        marks.append(time.perf_counter())

    if cuda:
        torch.cuda.synchronize()
    out = pipe(prompt=None, image=inp["bev_map"], camera_param=inp["camera_param"], height=h * 8, width=w * 8,
               num_inference_steps=warmup + steps, guidance_scale=guidance_scale, latents=inp["latents"].clone(),
               prompt_embeds=inp["prompt_embeds"], negative_prompt_embeds=inp["negative_prompt_embeds"],
               output_type="latent", bev_controlnet_kwargs={"bboxes_3d_data": inp["bboxes_3d_data"]}, callback=cb,
               callback_steps=1)
    assert len(marks) == warmup + steps, (len(marks), warmup, steps)
    # marks[i] = end of step i; steps warmup .. warmup+steps-1 are timed from the end of the last warm-up step
    t0 = marks[warmup - 1] if warmup > 0 else None
    if t0 is None:
        raise ValueError("need at least one warm-up step to mark the start of the timed region")
    return (marks[-1] - t0) / steps, out.images
