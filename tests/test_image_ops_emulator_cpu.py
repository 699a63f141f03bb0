"""tests/image_ops_emulator.py on the CPU: it restates exactly the operators of image_ops.py that launch a kernel, with their
signatures, and rejects unknown keywords."""
import inspect

import pytest

from magicdrive_b200 import image_ops
from tests import image_ops_emulator as E


def _launching_operators():
    fns = {n for n, f in inspect.getmembers(image_ops, inspect.isfunction)
           if f.__module__ == image_ops.__name__ and "_lib.lib()" in inspect.getsource(f)}
    return fns


def _params(fn):
    return [(p.name, p.kind, p.default) for p in inspect.signature(fn).parameters.values()]


def test_emulated_names_are_the_launching_operators():
    assert set(E.EMULATED) == _launching_operators() and len(E.EMULATED) == len(set(E.EMULATED))


@pytest.mark.parametrize("name", E.EMULATED)
def test_emulated_signature_equals_image_ops(name):
    assert _params(getattr(E, name)) == _params(getattr(image_ops, name))


def test_unknown_keyword_raises_type_error():
    for name in E.EMULATED:
        with pytest.raises(TypeError, match="unexpected keyword argument 'not_an_argument'"):
            getattr(E, name)(not_an_argument=1)
