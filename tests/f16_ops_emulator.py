"""TEST INFRASTRUCTURE ONLY — the CPU side of fp16 models: a torch restatement of every operator of magicdrive_b200/f16_ops.py
(include/magicdrive_b200.h semantics, the signatures held equal by tests/test_f16_ops_emulator_cpu.py), and `install`, which
puts them in place on top of tests/ops_emulator.py.

The operators of ops.py that also take f16 tensors (gemm_conv, groupnorm, attention, add, upsample_nearest) return f16 results
on the device where they are handed f16 ones.  `install` wraps ops_emulator's restatements of them so that they do the same:
their fp32 result is rounded to f16 once, where the device rounds its output (per set in add-mode attention, and row
statistics taken from the rounded values, are finer than this restatement goes).  So the host code of an fp16 model runs here
in its own storage type; the bf16 restatements are untouched."""
import functools

import torch
import torch.nn.functional as F

from magicdrive_b200 import f16_ops, ops
from tests import ops_emulator

F16, F32 = torch.float16, torch.float32


def f32_to_f16(x):
    assert x.dtype == F32
    return x.to(F16)


def f16_to_f32(x):
    assert x.dtype == F16
    return x.float()


def pack_latents_f16(x, cpad=64, repeat=1):
    return F.pad(x.float(), (0, cpad - x.shape[1])).to(F16).repeat(repeat, 1)


EMULATED = ["f32_to_f16", "f16_to_f32", "pack_latents_f16"]

# ops.py operators whose f16 launches write f16 outputs (the first tensor argument decides)
ROUNDED = ["gemm_conv", "groupnorm", "attention", "attention_multi", "add", "upsample_nearest"]


def _rounding(fn):
    @functools.wraps(fn)
    def wrapped(*args, **kw):
        res = fn(*args, **kw)
        if args[0].dtype != F16 or kw.get("out_f32", False):
            return res
        if isinstance(res, tuple):  # gemm_conv(emit_stats=True): (out, RowStats)
            return (res[0].to(F16),) + res[1:]
        return res.to(F16)
    return wrapped


def install(monkeypatch):
    """ops_emulator.install, then the f16_ops restatements and the f16 rounding of the shared operators."""
    ops_emulator.install(monkeypatch)
    for name in EMULATED:
        assert hasattr(f16_ops, name), name
        monkeypatch.setattr(f16_ops, name, globals()[name])
    for name in ROUNDED:
        monkeypatch.setattr(ops, name, _rounding(getattr(ops_emulator, name)))
