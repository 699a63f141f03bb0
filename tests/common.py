"""Shared test helpers (configs, golden loading, error metrics)."""
import os

import torch

from magicdrive_b200 import arch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def tiny_configs():
    u = arch.UNetConfig(block_out_channels=(64, 128), down_block_types=("CrossAttnDownBlock2D", "DownBlock2D"),
                        up_block_types=("UpBlock2D", "CrossAttnUpBlock2D"), layers_per_block=1, attention_head_dim=2)
    c = arch.ControlNetConfig(block_out_channels=(64, 128), down_block_types=("CrossAttnDownBlock2D", "DownBlock2D"),
                              layers_per_block=1, attention_head_dim=2, map_size=(8, 52, 52))
    return u, c


# Fixtures are kept below 1 MB per file, losslessly: a large top-level entry `key` of `<stem>.pt` is stored on its own as
# `<stem>.<key>.pt`, and a `ctx` tensor whose rows [a, b) are a copy of inputs["prompt_embeds"] (the text tokens every view
# carries) is stored without them, with `ctx_text_rows` = (a, b).
SPLIT_KEYS = {"tiny_forward.pt": ("down",), "tiny_attn_types.pt": ("guess_mode", "map_plus"), "sd15_forward.pt": ("down0",)}


def golden(name):
    g = torch.load(os.path.join(GOLDEN, name), map_location="cpu", weights_only=False)
    stem = name[:-len(".pt")]
    for key in SPLIT_KEYS.get(name, ()):
        g[key] = torch.load(os.path.join(GOLDEN, f"{stem}.{key}.pt"), map_location="cpu", weights_only=False)
    if "ctx_text_rows" in g:
        a, b = g.pop("ctx_text_rows")
        ctx = g["ctx"]
        text = g["inputs"]["prompt_embeds"].expand(ctx.shape[0], -1, -1)
        assert text.shape[1] == b - a
        g["ctx"] = torch.cat([ctx[:, :a], text, ctx[:, a:]], 1)
    return g


def save_golden(obj, name):
    """Inverse of golden(): writes `name` (and its split parts) under tests/golden."""
    obj = dict(obj)
    stem = name[:-len(".pt")]
    for key in SPLIT_KEYS.get(name, ()):
        torch.save(obj.pop(key), os.path.join(GOLDEN, f"{stem}.{key}.pt"))
    if "inputs" in obj and "ctx" in obj:
        text = obj["inputs"]["prompt_embeds"]
        ctx = obj["ctx"]
        a, b = 1, 1 + text.shape[1]
        if ctx.dim() == 3 and ctx.shape[1] >= b and ctx.shape[2] == text.shape[2] and \
                torch.equal(ctx[:, a:b], text.expand(ctx.shape[0], -1, -1)):
            obj["ctx"] = torch.cat([ctx[:, :a], ctx[:, b:]], 1).contiguous()
            obj["ctx_text_rows"] = (a, b)
    torch.save(obj, os.path.join(GOLDEN, name))


def tiny_state_dicts(seed=7):
    u, c = tiny_configs()
    return (arch.synthetic_state_dict(arch.unet_param_shapes(u), seed),
            arch.synthetic_state_dict(arch.controlnet_param_shapes(c), seed + 1))


def rel_l2(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


def max_rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).abs().max() / (b.abs().max() + 1e-12)).item()


def to_dev(x, dev, dtype=None):
    if isinstance(x, dict):
        return {k: to_dev(v, dev, dtype) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return [to_dev(v, dev, dtype) for v in x]
    if torch.is_tensor(x):
        if dtype is not None and x.is_floating_point():
            return x.to(dev, dtype)
        return x.to(dev)
    return x


def record(line: str, name: str = "parity_gpu_latest.txt"):
    """Print a `[parity]` / `[speed]` evidence line (visible with `pytest -s`); with MDB_RECORD_DIR set, also append it to
    $MDB_RECORD_DIR/<name> so that a GPU run of the test-suite can leave its measured numbers behind."""
    print(line)
    d = os.environ.get("MDB_RECORD_DIR")
    if d and os.path.isdir(d):
        with open(os.path.join(d, name), "a") as fh:
            fh.write(line.rstrip("\n") + "\n")
