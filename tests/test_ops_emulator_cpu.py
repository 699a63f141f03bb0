"""tests/ops_emulator.py on the CPU: it restates exactly the operators of ops.py that launch a kernel, with their signatures,
and against torch where its restatement has a rule of its own to get right."""
import inspect

import pytest
import torch
import torch.nn.functional as F

from magicdrive_b200 import ops
from tests import ops_emulator as E


def _launching_operators():
    """The functions of ops.py that call into the library, apart from the peer barrier and the launch-mode switch."""
    fns = {n for n, f in inspect.getmembers(ops, inspect.isfunction)
           if f.__module__ == ops.__name__ and "_lib.lib()" in inspect.getsource(f)}
    return fns - {"peer_barrier", "pdl_region"}


def _params(fn):
    return [(p.name, p.kind, p.default) for p in inspect.signature(fn).parameters.values()]


def test_emulated_names_are_the_launching_operators():
    assert set(E.EMULATED) == _launching_operators() and len(E.EMULATED) == len(set(E.EMULATED))


@pytest.mark.parametrize("name", E.EMULATED)
def test_emulated_signature_equals_ops(name):
    assert _params(getattr(E, name)) == _params(getattr(ops, name))


def test_unknown_keyword_raises_type_error():
    for name in E.EMULATED:
        with pytest.raises(TypeError, match="unexpected keyword argument 'not_an_argument'"):
            getattr(E, name)(not_an_argument=1)


def _exact_floor_differs(n_in, n_out):
    """True where floor(j * n_in / n_out) and ATen's float-scale index disagree for some output j."""
    exact = torch.div(torch.arange(n_out) * n_in, n_out, rounding_mode="floor")
    return not torch.equal(exact.clamp_max(n_in - 1), E.nearest_index(n_in, n_out))


# every (in, out) pair up to 64 -> 160 where the two rules disagree
DIFFER = [(i, o) for i in range(1, 65) for o in range(1, 161) if _exact_floor_differs(i, o)]


def test_size_pairs_where_the_rules_differ_exist():
    assert (26, 44) in DIFFER and len(DIFFER) > 20
    assert E.nearest_index(26, 44)[22].item() == 12  # the exact rule would read row 13


def test_upsample_nearest_follows_f_interpolate_where_the_rules_differ():
    g = torch.Generator().manual_seed(0)
    for h, ho in DIFFER:
        w, wo = DIFFER[(h * 7 + ho) % len(DIFFER)]  # a second differing pair along the width
        x = torch.randn(2, h, w, 8, generator=g)
        ref = F.interpolate(x.permute(0, 3, 1, 2), size=(ho, wo), mode="nearest").permute(0, 2, 3, 1).reshape(-1, 8)
        assert torch.equal(E.upsample_nearest(x.reshape(-1, 8), 2, h, w, 8, ho, wo), ref), (h, w, ho, wo)


def test_upsample_nearest_on_the_product_pyramids():
    """The UNet's up-path pairs at 224x400, 272x736 and 424x800 and the VAE's 2x steps: both rules agree there."""
    pairs = [((4, 7), (7, 13)), ((7, 13), (14, 25)), ((14, 25), (28, 50)), ((5, 12), (9, 23)), ((9, 23), (17, 46)),
             ((17, 46), (34, 92)), ((14, 25), (27, 50)), ((27, 50), (53, 100)), ((28, 50), (56, 100)), ((53, 100), (106, 200))]
    g = torch.Generator().manual_seed(1)
    for (h, w), (ho, wo) in pairs:
        x = torch.randn(1, h, w, 8, generator=g)
        ref = F.interpolate(x.permute(0, 3, 1, 2), size=(ho, wo), mode="nearest").permute(0, 2, 3, 1).reshape(-1, 8)
        assert torch.equal(E.upsample_nearest(x.reshape(-1, 8), 1, h, w, 8, ho, wo), ref), (h, w, ho, wo)
        assert not _exact_floor_differs(h, ho) and not _exact_floor_differs(w, wo)
