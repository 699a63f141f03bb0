"""The JPEG encoder on the sm_90a path: mdb_jpeg_encode_u8's files byte for byte against Pillow over the CPU suite's case
matrix and on batches of 900 x 1600 canvases, FIDProtocol.encode_generated and fid.save_generated_views against the
reference's own copy_save_image (tests/golden/val_set_jpeg.pt), the files decoded against mdb_jpeg_roundtrip_u8, guard
bands around scratch and output, capacities found too small on the device, rejected arguments and repeatability."""
import ctypes
import hashlib
import io

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from magicdrive_b200 import _lib, fid, image_ops, jpeg_ops  # noqa: E402
from oracle import fid_protocol as O  # noqa: E402
from oracle import jpeg_encode as J  # noqa: E402
from tests.test_jpeg_encode_cpu import (QUALITIES, SIZES, _expected_paths, _views, content, golden,  # noqa: E402
                                        pil_jpeg)

Image = pytest.importorskip("PIL.Image")
GUARD = 4096  # bytes of guard band on each side (keeps the scratch 256-byte aligned)


def encode(x, quality=None):
    return jpeg_ops.encode_jpeg(torch.from_numpy(np.ascontiguousarray(x)).cuda(), 75 if quality is None else quality)


@pytest.mark.parametrize("h,w", SIZES)
def test_case_matrix_equals_pillow(cuda_lib, h, w):
    kinds = ["views", "noise", "black", "white", "grey"]
    batch = np.stack([content(k, h, w, h * 131 + w) for k in kinds])
    for q in QUALITIES:
        got = encode(batch, q)
        for k, x, g in zip(kinds, batch, got):
            assert g == pil_jpeg(x, q), (k, h, w, q)


def test_edge_cases_equal_pillow(cuda_lib):
    yy, xx = np.mgrid[0:32, 0:48]
    checker = np.where(((yy + xx) & 1)[..., None], 255, 0).astype(np.uint8).repeat(3, -1)
    checker[:16, :16] = 0
    checker[16:, 16:32] = 255
    sparse = np.full((48, 64, 3), 90, np.uint8)
    sparse[5, 7] = 255
    sparse[21, 40:44] = 0
    sparse[40:48, 56:64] = np.eye(8, dtype=np.uint8)[..., None] * 200
    dense = np.random.default_rng(3).integers(0, 256, (64, 64, 3), dtype=np.uint8)
    pad_ff = np.random.default_rng(5).integers(0, 256, (8, 8, 3), dtype=np.uint8)
    for x, qs in [(checker, [100]), (sparse, [50, 90, 100]), (dense, [100]), (pad_ff, [100])]:
        for q in qs:
            assert encode(x[None], q)[0] == pil_jpeg(x, q), (x.shape, q)


def test_batches_of_900x1600_mixed(cuda_lib):
    """48 canvases of mixed content and lengths in one call (noise needs a second, larger attempt)."""
    v = O.to_u8(O.views(21, 40, 900, 1600))
    rng = np.random.default_rng(4)
    extra = [rng.integers(0, 256, (900, 1600, 3), dtype=np.uint8) for _ in range(3)]
    extra += [np.full((900, 1600, 3), c, np.uint8) for c in (0, 255, 128)]
    extra += [O.to_u8(O.views(22, 1, 900, 1600, noise=0.2)[0]), np.zeros((900, 1600, 3), np.uint8)]
    batch = np.concatenate([v[:20], np.stack(extra), v[20:]])
    assert batch.shape[0] == 48
    for q in (75, 95):
        got = encode(batch, q)
        lengths = {len(g) for g in got}
        assert len(lengths) > 10
        for i, (x, g) in enumerate(zip(batch, got)):
            assert g == pil_jpeg(x, q), (i, q)
    assert encode(batch[:6], 95) == got[:6]


@pytest.mark.parametrize("name", ["224x400", "272x736", "424x800"])
def test_encode_generated_reproduces_the_reference_files(cuda_lib, name):
    entry = golden()[name]
    views = torch.from_numpy(_views(name, entry)).cuda()
    protocol = fid.FIDProtocol(*entry["config"])
    files = protocol.encode_generated(views.reshape(-1, *views.shape[2:]))
    paths = _expected_paths(entry)
    assert len(files) == len(paths)
    for p, data in zip(paths, files):
        assert (len(data), hashlib.sha256(data).hexdigest()) == entry["files"][p], p
    # bf16 views are widened as generated() widens them
    assert protocol.encode_generated(views[0, 0].to(torch.bfloat16)[None]) == \
        protocol.encode_generated(views[0, 0].to(torch.bfloat16).float()[None])


@pytest.mark.parametrize("name", ["224x400", "272x736", "424x800", "raw_224x400"])
def test_writer_reproduces_the_reference_files(cuda_lib, name, tmp_path):
    entry = golden()[name]
    views = torch.from_numpy(_views(name, entry)).cuda()
    for v in entry["view_order"]:
        (tmp_path / v).mkdir()
    protocol = None if entry["config"] is None else fid.FIDProtocol(*entry["config"])
    labels = fid.save_generated_views(views, entry["templates"], str(tmp_path), entry["view_order"], protocol)
    assert labels == entry["labels"]
    assert sorted(str(p.relative_to(tmp_path)) for p in tmp_path.rglob("*.jpg")) == sorted(entry["files"])
    for rel, (n, sha) in entry["files"].items():
        data = (tmp_path / rel).read_bytes()
        assert (len(data), hashlib.sha256(data).hexdigest()) == (n, sha), rel


def test_decoded_files_equal_the_round_trip(cuda_lib):
    """Pillow decoding the device's files gives what mdb_jpeg_roundtrip_u8 computes for the same canvas."""
    protocol = fid.FIDProtocol.for_config("224x400")
    views = torch.from_numpy(O.views(31, 4, 224, 400)).cuda()
    files = protocol.encode_generated(views[None])
    left, top, _, _ = protocol.back_pad
    canvas = protocol._resize(views, True, protocol.back_resize, canvas=protocol.canvas, offset=(top, left))
    rt = image_ops.jpeg_roundtrip_u8(canvas, protocol.quality).cpu().numpy()
    for f, want in zip(files, rt):
        with Image.open(io.BytesIO(f)) as im:
            assert np.array_equal(np.asarray(im.convert("RGB")), want)
    for q in (1, 50, 100):
        x = content("views", 37, 53, 9)
        with Image.open(io.BytesIO(encode(x[None], q)[0])) as im:
            got = np.asarray(im.convert("RGB"))
        assert np.array_equal(got, image_ops.jpeg_roundtrip_u8(torch.from_numpy(x[None]).cuda(), q).cpu().numpy()[0])


def _guarded(nbytes, fill):
    buf = torch.full((nbytes + 2 * GUARD,), fill, dtype=torch.uint8, device="cuda")
    return buf, buf[GUARD:GUARD + nbytes]


def _guards_intact(buf, fill):
    return bool((buf[:GUARD] == fill).all()) and bool((buf[-GUARD:] == fill).all())


def test_guard_bands_and_exact_buffers(cuda_lib):
    x = np.stack([content("views", 70, 90, 1), content("noise", 70, 90, 2), content("grey", 70, 90, 3)])
    want = [pil_jpeg(v, 90) for v in x]
    xs = torch.from_numpy(x).cuda()
    scan = [len(f) - 625 - f[623:-2].count(b"\xff") for f in want]
    chunks = sum(-(-s // 4096) for s in scan)
    sbuf, scratch = _guarded(jpeg_ops.scratch_bytes(3, 70, 90, chunks), 0xA5)
    obuf, out = _guarded(sum(len(f) for f in want), 0x5A)
    meta = jpeg_ops.jpeg_encode_u8(xs, 90, scratch=scratch, out=out)
    assert meta[:, 0].tolist() == scan and meta[:, 1].tolist() == [len(f) for f in want]
    data = out.cpu().numpy().tobytes()
    assert [data[o:o + n] for o, n in meta[:, 1:].flip(1).tolist()] == want
    assert _guards_intact(sbuf, 0xA5) and _guards_intact(obuf, 0x5A)


def test_capacities_found_too_small_on_the_device(cuda_lib):
    x = torch.from_numpy(np.stack([content("noise", 64, 64, 7)] * 2)).cuda()
    want = pil_jpeg(x[0].cpu().numpy(), 100)
    # out one byte short: lengths measured, nothing written
    sbuf, scratch = _guarded(jpeg_ops.scratch_bytes(2, 64, 64, 64), 0xA5)
    obuf, out = _guarded(2 * len(want) - 1, 0x5A)
    meta = jpeg_ops.jpeg_encode_u8(x, 100, scratch=scratch, out=out)
    assert meta[:, 1].tolist() == [len(want)] * 2 and (meta[:, 2] == -1).all()
    assert bool((obuf == 0x5A).all()) and _guards_intact(sbuf, 0xA5)
    # scratch with one chunk per image: entropy-coded sizes measured, lengths unknown, nothing written
    sbuf, scratch = _guarded(jpeg_ops.scratch_bytes(2, 64, 64, 2), 0xA5)
    obuf, out = _guarded(4 * len(want), 0x5A)
    meta = jpeg_ops.jpeg_encode_u8(x, 100, scratch=scratch, out=out)
    assert (meta[:, 0] > 4096).all() and (meta[:, 1] == -1).all() and (meta[:, 2] == -1).all()
    assert bool((obuf == 0x5A).all()) and _guards_intact(sbuf, 0xA5)


def test_bad_arguments_raise_before_any_launch(cuda_lib):
    lib = _lib.lib()
    x = torch.zeros((2, 16, 16, 3), dtype=torch.uint8, device="cuda")
    need = jpeg_ops.scratch_bytes(2, 16, 16, 2)
    scratch = torch.zeros(need, dtype=torch.uint8, device="cuda")
    out = torch.full((4096,), 0x5A, dtype=torch.uint8, device="cuda")
    meta = torch.full((2, 3), 7, dtype=torch.int64, device="cuda")
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    base = dict(x=p(x), n=2, h=16, w=16, q=75, s=p(scratch), sb=need, o=p(out), ob=4096, m=p(meta))
    bad = [dict(x=None), dict(s=None), dict(o=None), dict(m=None), dict(n=0), dict(n=-1), dict(h=0), dict(w=0),
           dict(h=65536), dict(w=70000), dict(q=0), dict(q=101), dict(sb=need - 1), dict(ob=2 * 626 - 1),
           dict(s=ctypes.c_void_p(scratch.data_ptr() + 8)), dict(m=ctypes.c_void_p(meta.data_ptr() + 4))]
    torch.cuda.synchronize()
    for b in bad:
        a = {**base, **b}
        st = lib.mdb_jpeg_encode_u8(a["x"], a["n"], a["h"], a["w"], a["q"], a["s"], a["sb"], a["o"], a["ob"], a["m"], None)
        assert st == -1, b
    torch.cuda.synchronize()
    assert bool((out == 0x5A).all()) and bool((meta == 7).all())
    with pytest.raises(_lib.MdbError, match="scratch"):
        jpeg_ops.jpeg_encode_u8(x, 75, scratch=scratch[:need - 1], out=out)
    with pytest.raises(_lib.MdbError, match="quality"):
        jpeg_ops.jpeg_encode_u8(x, 0, scratch=scratch, out=out)
    assert bool((out == 0x5A).all())
    with pytest.raises(ValueError):
        jpeg_ops.scratch_bytes(0, 16, 16, 1)
    assert lib.mdb_jpeg_scratch_bytes(1, 65536, 1, 1) == -1


def test_repeated_calls_are_bitwise_equal(cuda_lib):
    batch = torch.from_numpy(np.stack([content(k, 150, 260, 5) for k in ("views", "noise", "white")])).cuda()
    first = jpeg_ops.encode_jpeg(batch, 80)
    for _ in range(5):
        assert jpeg_ops.encode_jpeg(batch, 80) == first
