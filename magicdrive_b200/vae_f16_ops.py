"""torch.Tensor-facing wrappers of the C-ABI operators that only a VAE with fp16 parameters needs: the f16 twins of the row
softmax of the mid-block attention (mdb_softmax_rows_f16), of the direct convolution that writes the decoder's first feature
map (mdb_conv_direct_f16) and of the encoder's 8-channel image operand (mdb_fid_input_f16).  Their bf16 versions are
ops.softmax_rows, ops.conv_direct and ops.fid_input; these take the same arguments and write f16 where those write bf16.

They sit beside ops.py and share its plumbing: raw pointers and the current stream go to `libmagicdrive_b200.so`, launches
count in `ops.launch_count()`, there is no CPU or eager fallback, and an operand of another element type is a TypeError
before anything is launched.  Their CPU restatement for host tests is tests/vae_f16_ops_emulator.py.
"""
import torch

from . import _lib, ops
from ._lib import check
from .ops import _need_cuda, _need_dtype, _ptr, _stream

F16, F32 = torch.float16, torch.float32


def softmax_rows_f16(s, cols: int, cols_out: int):
    """fp32 scores [rows, >=cols] -> f16 probabilities [rows, cols_out], columns >= cols zero (mdb_softmax_rows_f16)."""
    _need_cuda(s)
    _need_dtype("softmax_rows_f16", F32, s=s)
    out = torch.empty((s.shape[0], cols_out), dtype=F16, device=s.device)
    check(_lib.lib().mdb_softmax_rows_f16(_ptr(s), s.stride(0), s.shape[0], cols, _ptr(out), cols_out, cols_out, _stream()),
          "mdb_softmax_rows_f16")
    ops._launches += 1
    return out


def conv_direct_f16(x, wgt, bias, *, n, h, w, cin, cout, k, stride=(1, 1), pad=(1, 1), silu=False, residual=None,
                    out_f32=False):
    """Direct convolution of an NHWC fp32 or f16 map with fp32 weights [k, k, cin, cout] and fp32 bias
    (mdb_conv_direct_f16): the output, and a residual added to it, are fp32 with out_f32, else f16."""
    _need_cuda(x, wgt)
    if x.dtype not in (F32, F16):  # the kernel reads any other source as f16 bits
        raise TypeError(f"conv_direct_f16: x is {x.dtype}, expected float32 or float16")
    _need_dtype("conv_direct_f16", F32, wgt=wgt, bias=bias)
    _need_dtype("conv_direct_f16", F32 if out_f32 else F16, residual=residual)
    ho = (h + 2 * pad[0] - k) // stride[0] + 1
    wo = (w + 2 * pad[1] - k) // stride[1] + 1
    out = torch.empty((n, ho, wo, cout), dtype=F32 if out_f32 else F16, device=x.device)
    check(_lib.lib().mdb_conv_direct_f16(_ptr(x), int(x.dtype == F32), n, h, w, cin, _ptr(wgt), _ptr(bias), cout, k, k,
                                         stride[0], stride[1], pad[0], pad[1], ho, wo, int(silu), _ptr(residual), _ptr(out),
                                         int(out_f32), _stream()), "mdb_conv_direct_f16")
    ops._launches += 1
    return out


def fid_input_f16(x, *, nhwc: bool, quantize: bool, normalize: bool, size=None):
    """ops.fid_input with an f16 output (mdb_fid_input_f16): a [0, 1] image batch, NCHW [n, 3, h, w] (or NHWC with nhwc=True),
    fp32 or f16 -> f16 [n*ho*wo, 8], channels 3..7 zero: conv_in's operand in an fp16 VAE's encoder.  Without quantize, size
    or normalize each value is x rounded to f16 once (x.to(torch.float16))."""
    _need_cuda(x)
    if x.dtype not in (F32, F16):  # the kernel reads any other source as f16 bits
        raise TypeError(f"fid_input_f16: x is {x.dtype}, expected float32 or float16")
    x = x.contiguous()
    n, h, w = (x.shape[0], x.shape[1], x.shape[2]) if nhwc else (x.shape[0], x.shape[2], x.shape[3])
    assert (x.shape[3] if nhwc else x.shape[1]) == 3
    ho, wo = (h, w) if size is None else size
    out = torch.empty((n * ho * wo, 8), dtype=F16, device=x.device)
    check(_lib.lib().mdb_fid_input_f16(_ptr(x), int(x.dtype == F32), int(nhwc), n, h, w, int(quantize), int(normalize),
                                       _ptr(out), ho, wo, _stream()), "mdb_fid_input_f16")
    ops._launches += 1
    return out
