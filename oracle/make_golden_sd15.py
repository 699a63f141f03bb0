"""TEST INFRASTRUCTURE ONLY — SD-1.5-size fixture produced by running the REFERENCE ITSELF (via oracle/ref_shim.py):
one BEVControlNetModel.forward + UNet2DConditionModelMultiview.forward of the unmodified reference classes at the
configuration the benchmark times (4 levels, head dims 40 / 80 / 160, 6 views, 20 boxes per view, 200x200 BEV map,
28x50 latents), fp32 on the CPU, weights from arch.synthetic_state_dict(seeds 11 / 12) exactly like bench.py.

    python -m oracle.make_golden_sd15       # build container (needs /root/reference or the oracle/_ref snapshot), ~3 min

Stored (tests/golden/sd15_forward.pt + sd15_forward.down0.pt): the predicted noise in full; the mid residual, ControlNet residuals 0 and 11
and the conditioning tokens on a fixed channel subset (every 16th / 8th channel), enough to pin a structural error anywhere
on the path without committing 40 MB of activations.  The oracle (tests/test_oracle_cpu.py) and the CUDA path
(tests/test_model_gpu.py) are both checked against it.
"""
import os
import sys

import torch

from magicdrive_b200 import arch
from magicdrive_b200.synthetic import synthetic_inputs
from oracle import ref_shim
from tests.common import save_golden

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "sd15_forward.pt")
SEEDS = (11, 12)
INPUT_SEED, T, H, W, N_BOX, MAP_HW = 5, 601, 28, 50, 20, 200
CH_STEP, CTX_STEP = 16, 8


@torch.no_grad()
def main():
    ucfg, ccfg = arch.UNetConfig(), arch.ControlNetConfig(map_size=(8, MAP_HW, MAP_HW))
    mv, cn = ref_shim.build_reference_models(ucfg, ccfg)
    mv.load_state_dict(arch.synthetic_state_dict(arch.unet_param_shapes(ucfg), SEEDS[0]), strict=True)
    cn.load_state_dict(arch.synthetic_state_dict(arch.controlnet_param_shapes(ccfg), SEEDS[1]), strict=True)
    inp = synthetic_inputs(1, 6, H, W, n_box=N_BOX, map_hw=MAP_HW, seed=INPUT_SEED)
    lat5 = torch.stack([inp["latents"]] * 6, 1)
    t = torch.tensor([T])
    down, mid, ctx = cn(lat5, t, inp["camera_param"], inp["bboxes_3d_data"], inp["prompt_embeds"], inp["bev_map"],
                        return_dict=False)
    eps = mv(lat5.reshape(-1, 4, H, W), t[0], encoder_hidden_states=ctx, down_block_additional_residuals=down,
             mid_block_additional_residual=mid).sample
    save_golden(dict(seeds=SEEDS, input_seed=INPUT_SEED, t=T, shape=(1, 6, H, W), n_box=N_BOX, map_hw=MAP_HW,
                    ch_step=CH_STEP, ctx_step=CTX_STEP, eps=eps.clone(), mid=mid[:, ::CH_STEP].clone(),
                    down0=down[0][:, ::CH_STEP].clone(), down11=down[11][:, ::CH_STEP].clone(),
                    ctx=ctx[:, :, ::CTX_STEP].clone(), n_down=len(down),
                    down_norms=[float(d.norm()) for d in down]), os.path.basename(OUT))
    print(OUT, os.path.getsize(OUT) // 1024, "KiB; eps", tuple(eps.shape), "|eps|", float(eps.norm()))


if __name__ == "__main__":
    sys.exit(main())
