"""Fixtures of the CLIP text encoder (tests/golden/clip_text_{tiny,sd15}.pt), produced with transformers' own CLIPTextModel
(eager attention, fp32, eos_token_id = 2 as in SD-1.5's text_encoder/config.json) on the weights and ids of
oracle/clip_text.py.  The tiny fixture stores its weights; the SD-1.5-size one stores only the seed (the tests draw the
weights again).  Each stores the input ids, last_hidden_state and pooler_output.  Run on the CPU:

    python -m oracle.make_golden_clip
"""
import torch

from magicdrive_b200 import arch
from oracle.clip_text import TINY, draw_weights, fixture_ids
from tests.common import save_golden

SEED_W, SEED_IDS = {"tiny": 11, "sd15": 12}, {"tiny": 21, "sd15": 22}


def make(name, cfg_kwargs):
    from transformers import CLIPTextConfig, CLIPTextModel
    cfg = arch.ClipTextConfig(**cfg_kwargs)
    sd = draw_weights(cfg, SEED_W[name])
    tcfg = CLIPTextConfig(**{k: v for k, v in vars(cfg).items()}, attn_implementation="eager")
    model = CLIPTextModel(tcfg).eval()
    model.load_state_dict(sd, strict=True)
    pair, short = fixture_ids(cfg, SEED_IDS[name])
    cases = []
    with torch.no_grad():
        for ids in [pair] + short:
            out = model(ids)
            cases.append(dict(ids=ids, last_hidden_state=out.last_hidden_state.clone(), pooler_output=out.pooler_output.clone()))
    fx = dict(config=vars(cfg), seed_weights=SEED_W[name], cases=cases)
    if name == "tiny":
        fx["state_dict"] = sd
    save_golden(fx, f"clip_text_{name}.pt")


if __name__ == "__main__":
    torch.set_num_threads(1)  # fixed reduction order: a re-run reproduces the files bit for bit
    make("tiny", TINY)
    make("sd15", {})
