"""torch.Tensor-facing wrappers of the C-ABI operators that only models with fp16 parameters need: fp32 <-> f16 conversion
(mdb_f32_to_f16, mdb_f16_to_f32) and the f16 conv_in operand (mdb_pack_latents_f16).  The operators both precisions share
take f16 tensors in ops.py itself.

They sit beside ops.py and share its plumbing: raw pointers and the current stream go to `libmagicdrive_b200.so`, launches
count in `ops.launch_count()`, and there is no CPU or eager fallback.  Their CPU restatement for host tests is
tests/f16_ops_emulator.py.
"""
import torch

from . import _lib, ops
from ._lib import check
from .ops import _need_cuda, _ptr, _stream

F16, F32 = torch.float16, torch.float32


def f32_to_f16(x):
    """fp32 -> f16, round to nearest even (mdb_f32_to_f16): the conditioning context of an fp16 model."""
    _need_cuda(x)
    assert x.dtype == F32 and x.is_contiguous()
    out = torch.empty(x.shape, dtype=F16, device=x.device)
    check(_lib.lib().mdb_f32_to_f16(_ptr(x), _ptr(out), x.numel(), _stream()), "mdb_f32_to_f16")
    ops._launches += 1
    return out


def f16_to_f32(x):
    """f16 -> fp32, exact (mdb_f16_to_f32)."""
    _need_cuda(x)
    assert x.dtype == F16 and x.is_contiguous()
    out = torch.empty(x.shape, dtype=F32, device=x.device)
    check(_lib.lib().mdb_f16_to_f32(_ptr(x), _ptr(out), x.numel(), _stream()), "mdb_f16_to_f32")
    ops._launches += 1
    return out


def pack_latents_f16(x, cpad: int = 64, repeat: int = 1):
    """[pix, cin] fp32/f16 -> f16 [repeat*pix, cpad] zero-padded channels (the conv_in operand of an fp16 model)."""
    _need_cuda(x)
    if x.dtype not in (F32, F16):  # the kernel reads any other source as f16 bits
        raise TypeError(f"pack_latents_f16: x is {x.dtype}, expected float32 or float16")
    pix, cin = x.shape
    out = torch.empty((repeat * pix, cpad), dtype=F16, device=x.device)
    check(_lib.lib().mdb_pack_latents_f16(_ptr(x), int(x.dtype == F32), pix, cin, cpad, repeat, _ptr(out), _stream()),
          "mdb_pack_latents_f16")
    ops._launches += 1
    return out
