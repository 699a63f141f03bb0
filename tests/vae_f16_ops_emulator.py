"""TEST INFRASTRUCTURE ONLY — the CPU side of an fp16 VAE: a torch restatement of every operator of
magicdrive_b200/vae_f16_ops.py (include/magicdrive_b200.h semantics, the signatures held equal by
tests/test_vae_fp16_host_cpu.py), and `install`, which puts them in place on top of tests/f16_ops_emulator.py.

Each restates its bf16 twin in tests/ops_emulator.py in fp32 and rounds the result to f16 once, where the device writes
f16 (an fp32 output with out_f32 stays unrounded)."""
import torch

from magicdrive_b200 import vae_f16_ops
from tests import f16_ops_emulator, ops_emulator

F16 = torch.float16


def softmax_rows_f16(s, cols, cols_out):
    return ops_emulator.softmax_rows(s, cols, cols_out).to(F16)


def conv_direct_f16(x, wgt, bias, *, n, h, w, cin, cout, k, stride=(1, 1), pad=(1, 1), silu=False, residual=None,
                    out_f32=False):
    y = ops_emulator.conv_direct(x, wgt, bias, n=n, h=h, w=w, cin=cin, cout=cout, k=k, stride=stride, pad=pad, silu=silu,
                                 residual=residual, out_f32=True)
    return y if out_f32 else y.to(F16)


def fid_input_f16(x, *, nhwc, quantize, normalize, size=None):
    return ops_emulator.fid_input(x, nhwc=nhwc, quantize=quantize, normalize=normalize, size=size).to(F16)


EMULATED = ["softmax_rows_f16", "conv_direct_f16", "fid_input_f16"]


def install(monkeypatch):
    """f16_ops_emulator.install, then the restatements of vae_f16_ops."""
    f16_ops_emulator.install(monkeypatch)
    for name in EMULATED:
        assert hasattr(vae_f16_ops, name), name
        monkeypatch.setattr(vae_f16_ops, name, globals()[name])
