"""TEST INFRASTRUCTURE ONLY — plain-torch restatement of transformers' CLIPTextModel forward (the CLIP text encoder the
reference pipeline calls in _encode_prompt, third_party/diffusers/src/diffusers/pipelines/controlnet/pipeline_controlnet.py:
365-369 and 417-421, and in bbox_embedder.py:123-135), from state-dict tensors by their checkpoint names.  Line numbers cite
transformers/models/clip/modeling_clip.py (transformers 5.5.0); the arithmetic is the same in the reference's pinned 4.27.4.

fp32 by default; `dtype=torch.bfloat16` runs the same arithmetic in bf16 torch (the yardstick of how far a bf16
implementation may sit from fp32)."""
from typing import Dict

import torch
import torch.nn.functional as F

from magicdrive_b200 import arch


def _lin(sd, p, x):
    return F.linear(x, sd[p + ".weight"], sd[p + ".bias"])


def _ln(sd, p, x, eps):
    return F.layer_norm(x, (x.shape[-1],), sd[p + ".weight"], sd[p + ".bias"], eps)


def clip_text_forward(sd: Dict[str, torch.Tensor], cfg: arch.ClipTextConfig, ids: torch.Tensor, dtype=torch.float32):
    """ids: int [n, L] -> (last_hidden_state [n, L, C], pooler_output [n, C]) in `dtype`."""
    sd = {k: v.to(device=ids.device, dtype=dtype) for k, v in sd.items() if k != "text_model.embeddings.position_ids"}
    t = "text_model"
    n, L = ids.shape
    C, H = cfg.hidden_size, cfg.num_attention_heads
    d, eps = C // H, cfg.layer_norm_eps
    # CLIPTextEmbeddings.forward (:234-258): token + position embedding of positions 0..L-1
    x = sd[t + ".embeddings.token_embedding.weight"][ids.long()] + sd[t + ".embeddings.position_embedding.weight"][:L][None]
    # CLIPTextTransformer.forward (:544-560): causal mask, key j visible to query i iff j <= i
    mask = torch.full((L, L), float("-inf"), device=ids.device, dtype=dtype).triu(1)
    for i in range(cfg.num_hidden_layers):
        p = f"{t}.encoder.layers.{i}"
        a = p + ".self_attn"
        # CLIPEncoderLayer.forward (:363-395): pre-LN attention and MLP, each with a residual
        h = _ln(sd, p + ".layer_norm1", x, eps)
        # CLIPAttention.forward (:300-336): softmax(q k^T * head_dim^-0.5 + mask) v, then out_proj
        q, k, v = (_lin(sd, f"{a}.{n_}_proj", h).reshape(n, L, H, d).transpose(1, 2) for n_ in ("q", "k", "v"))
        s = (q @ k.transpose(-1, -2)) * d ** -0.5 + mask
        o = (torch.softmax(s.float(), -1).to(dtype) @ v).transpose(1, 2).reshape(n, L, C)
        x = x + _lin(sd, a + ".out_proj", o)
        h = _ln(sd, p + ".layer_norm2", x, eps)
        # CLIPMLP.forward (:347-351) with quick_gelu (activations.py QuickGELUActivation: x * sigmoid(1.702 x))
        h = _lin(sd, p + ".mlp.fc1", h)
        h = h * torch.sigmoid(1.702 * h)
        x = x + _lin(sd, p + ".mlp.fc2", h)
    x = _ln(sd, t + ".final_layer_norm", x, eps)
    # pooling (:564-575): with eos_token_id == 2 (SD-1.5's config) the row at argmax(input_ids)
    pooled = x[torch.arange(n, device=ids.device), ids.to(torch.int).argmax(-1)]
    return x, pooled


TINY = dict(vocab_size=512, hidden_size=64, intermediate_size=128, num_hidden_layers=2, num_attention_heads=2,
            max_position_embeddings=77, eos_token_id=2)


def draw_weights(cfg: arch.ClipTextConfig, seed: int) -> Dict[str, torch.Tensor]:
    """Seeded CPU weights, drawn in sorted key order: every LayerNorm gain / bias and linear bias random (none left at 1 / 0),
    linear weights scaled by fan_in^-0.5 so that attention is neither uniform nor one-hot."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, shape in sorted(arch.clip_text_param_shapes(cfg).items()):
        r = torch.randn(shape, generator=g, dtype=torch.float32)
        if "embedding" in k:
            sd[k] = r
        elif "layer_norm" in k and k.endswith(".weight"):
            sd[k] = 1.0 + 0.2 * r
        elif k.endswith(".weight"):
            sd[k] = r * shape[1] ** -0.5
        else:
            sd[k] = 0.1 * r
    return sd


def fixture_ids(cfg: arch.ClipTextConfig, seed: int):
    """The fixtures' inputs, shaped like the tokenizer's output (BOS = vocab-2, EOS = pad = vocab-1, as CLIPTokenizer pads
    with <|endoftext|>): a padded [uncond ; cond] 2 x max_length pair of one scene, and unpadded class-name lookups of
    lengths 3-7 (padding="do_not_pad")."""
    g = torch.Generator().manual_seed(seed)
    bos, eos, L = cfg.vocab_size - 2, cfg.vocab_size - 1, cfg.max_position_embeddings
    pair = torch.full((2, L), eos, dtype=torch.long)
    pair[:, 0] = bos
    pair[1, 1:22] = torch.randint(0, bos, (21,), generator=g)
    short = []
    for n in range(3, 8):
        ids = torch.full((1, n), eos, dtype=torch.long)
        ids[0, 0] = bos
        ids[0, 1:n - 1] = torch.randint(0, bos, (n - 2,), generator=g)
        short.append(ids)
    return pair, short
