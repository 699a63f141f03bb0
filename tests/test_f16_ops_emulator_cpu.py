"""tests/f16_ops_emulator.py on the CPU: it restates exactly the operators of f16_ops.py that launch a kernel, with their
signatures, and its install rounds the shared operators' results to f16 where they are handed f16."""
import inspect

import pytest
import torch

from magicdrive_b200 import f16_ops, ops
from tests import f16_ops_emulator as E


def _launching_operators():
    return {n for n, f in inspect.getmembers(f16_ops, inspect.isfunction)
            if f.__module__ == f16_ops.__name__ and "_lib.lib()" in inspect.getsource(f)}


def _params(fn):
    return [(p.name, p.kind, p.default) for p in inspect.signature(fn).parameters.values()]


def test_emulated_names_are_the_launching_operators():
    assert set(E.EMULATED) == _launching_operators() and len(E.EMULATED) == len(set(E.EMULATED))


@pytest.mark.parametrize("name", E.EMULATED)
def test_emulated_signature_equals_f16_ops(name):
    assert _params(getattr(E, name)) == _params(getattr(f16_ops, name))


def test_unknown_keyword_raises_type_error():
    for name in E.EMULATED:
        with pytest.raises(TypeError, match="unexpected keyword argument 'not_an_argument'"):
            getattr(E, name)(not_an_argument=1)


def test_conversions_and_packing_follow_torch():
    x = torch.randn(37, 4) * 1e3
    assert torch.equal(E.f32_to_f16(x), x.half()) and torch.equal(E.f16_to_f32(x.half()), x.half().float())
    p = E.pack_latents_f16(x, 64, repeat=2)
    assert p.dtype == torch.float16 and p.shape == (74, 64) and torch.equal(p[37:, :4], x.half()) and not p[:, 4:].any()


def test_install_rounds_f16_inputs_only(monkeypatch):
    E.install(monkeypatch)
    a, b = torch.randn(8, 16), torch.randn(8, 16)
    assert ops.add(a, b).dtype == torch.float32  # the bf16 restatement as before (unrounded fp32)
    s = ops.add(a.half(), b.half())
    assert s.dtype == torch.float16 and torch.equal(s, (a.half().float() + b.half().float()).half())
    w = torch.randn(64, 64).half()
    y = ops.linear(torch.randn(8, 64).half(), w)
    assert y.dtype == torch.float16
    assert ops.linear(torch.randn(8, 64).half(), w, out_f32=True).dtype == torch.float32
    assert f16_ops.f32_to_f16 is E.f32_to_f16
