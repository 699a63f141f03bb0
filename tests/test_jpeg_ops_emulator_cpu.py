"""tests/jpeg_ops_emulator.py on the CPU: it restates exactly the operators of jpeg_ops.py that call the library, with
their signatures."""
import inspect

import pytest

from magicdrive_b200 import jpeg_ops
from tests import jpeg_ops_emulator as E


def _launching_operators():
    return {n for n, f in inspect.getmembers(jpeg_ops, inspect.isfunction)
            if f.__module__ == jpeg_ops.__name__ and "_lib.lib()" in inspect.getsource(f)}


def _params(fn):
    return [(p.name, p.kind, p.default) for p in inspect.signature(fn).parameters.values()]


def test_emulated_names_are_the_launching_operators():
    assert set(E.EMULATED) == _launching_operators() and len(E.EMULATED) == len(set(E.EMULATED))


@pytest.mark.parametrize("name", E.EMULATED)
def test_emulated_signature_equals_jpeg_ops(name):
    assert _params(getattr(E, name)) == _params(getattr(jpeg_ops, name))


def test_unknown_keyword_raises_type_error():
    for name in E.EMULATED:
        with pytest.raises(TypeError, match="unexpected keyword argument 'not_an_argument'"):
            getattr(E, name)(not_an_argument=1)


def test_scratch_layout_matches_the_library_formula():
    # coefficients, MCU bits and first bits, image layout and flags, then 8 + 4096 bytes per chunk (256-byte aligned)
    assert E.scratch_bytes(1, 16, 16, 1) == 768 + 256 + 256 + 256 + 256 + 256 + 4096
    assert E.scratch_bytes(2, 17, 33, 5) - E.scratch_bytes(2, 17, 33, 4) in (4096, 4096 + 256)
