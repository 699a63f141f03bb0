"""TEST INFRASTRUCTURE ONLY — tests/ops_emulator.py plus the attention semantics that camera rigs other than nuScenes' ring
need (include/magicdrive_b200.h: mdb_attention's empty kv_index slots, mdb_attention_varlen's per-batch key counts), so the
engine's host side can run on such rigs in the build container.  `install(monkeypatch)` swaps in every operator of
ops_emulator and then this module's `attention`."""
import math

import torch

from magicdrive_b200 import ops
from tests import ops_emulator


def attention(q, k, v, *, b, heads, lq, lk, d, ldq, ldk, ldv, scale, kv_index=None, n_sets=1, out=None, b_kv=None,
              kv_len=None):
    """ops_emulator.attention, where a kv_index entry < 0 is an empty slot that adds nothing (a row without a present set is
    zero) and kv_len[b] (clamped to [0, lk]) cuts query batch b's keys; a batch with 0 keys adds nothing either."""
    b_kv = b if b_kv is None else b_kv
    c = heads * d
    assert q.stride(0) == ldq and k.stride(0) == ldk and v.stride(0) == ldv
    qh = q[:, :c].float().reshape(b, lq, heads, d).transpose(1, 2)
    kh = k[:, :c].float().reshape(b_kv, lk, heads, d).transpose(1, 2)
    vh = v[:, :c].float().reshape(b_kv, lk, heads, d).transpose(1, 2)
    if kv_index is None:
        assert n_sets == 1 and b_kv == b
        sels = [torch.arange(b)]
    else:
        idx = kv_index.reshape(b, n_sets).long().cpu()
        sels = [idx[:, s] for s in range(n_sets)]
    n_keys = torch.full((b,), lk) if kv_len is None else kv_len.long().cpu().clamp(0, lk)
    key_mask = torch.where(torch.arange(lk)[None] < n_keys[:, None], 0.0, -math.inf)[:, None, None, :]
    res = torch.zeros(b, heads, lq, d)
    for sel in sels:
        present = ((sel >= 0) & (n_keys > 0))[:, None, None, None]
        sel = sel.clamp_min(0)
        o = torch.softmax(qh @ kh[sel].transpose(-1, -2) * scale + key_mask, -1) @ vh[sel]
        res = res + torch.where(present, ops_emulator._act(o), 0.0)  # each branch is rounded to bf16 before the sum
    res = ops_emulator._act(res.transpose(1, 2).reshape(b * lq, c))
    if out is not None:
        out[:, :c] = res
        return out
    return res


def install(monkeypatch):
    ops_emulator.install(monkeypatch)
    monkeypatch.setattr(ops, "attention", attention)
