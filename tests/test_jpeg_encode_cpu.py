"""oracle/jpeg_encode.py against Pillow byte for byte, the reference's generated data set (tests/golden/val_set_jpeg.pt),
and the writer's host logic through tests/jpeg_ops_emulator.py."""
import copy
import hashlib
import io
import os

import numpy as np
import pytest
import torch
from PIL import Image

from magicdrive_b200 import fid
from oracle import fid_protocol as O
from oracle import jpeg_encode as J
from tests import image_ops_emulator, jpeg_ops_emulator
from tests.common import GOLDEN

QUALITIES = [1, 10, 24, 25, 50, 75, 90, 95, 100, None]
SIZES = [(1, 1), (1, 17), (8, 8), (9, 9), (15, 33), (16, 16), (17, 31), (224, 400)]
SIZES += [(16 * 2 + r, 16 * 3 + c) for r, c in [(1, 9), (2, 10), (3, 11), (4, 12), (5, 13), (6, 14), (7, 15), (8, 1),
                                                (9, 2), (10, 3), (11, 4), (12, 5), (13, 6), (14, 7), (15, 8)]]


def pil_jpeg(x, quality=None):
    buf = io.BytesIO()
    Image.fromarray(x).save(buf, "JPEG", **({} if quality is None else {"quality": quality}))
    return buf.getvalue()


def ours(x, quality=None):
    return J.encode(x, 75 if quality is None else quality)


def content(kind, h, w, seed):
    rng = np.random.default_rng(seed)
    if kind == "views":
        return O.to_u8(O.views(seed, 1, max(h, 4), max(w, 4))[0])[:h, :w].copy()
    if kind == "noise":
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    return np.full((h, w, 3), {"black": 0, "white": 255, "grey": 128}[kind], np.uint8)


def test_header_is_pillows():
    for h, w, q in [(1, 1, 75), (900, 1600, 75), (65535, 65535, 1), (37, 4099, 100)]:
        x = np.zeros((min(h, 8), min(w, 8), 3), np.uint8)
        ref = pil_jpeg(x, q)
        assert J.header(x.shape[0], x.shape[1], q) == ref[:J.HEADER_BYTES]
    # the frame size is the only part that depends on the image
    hd = J.header(900, 1600, 75)
    assert hd[:2] == b"\xff\xd8" and hd[-14:-12] == b"\xff\xda" and len(hd) == 623
    assert b"\xff\xc0\x00\x11\x08\x03\x84\x06\x40" in hd


@pytest.mark.parametrize("h,w", SIZES)
@pytest.mark.parametrize("quality", QUALITIES)
def test_sizes_and_qualities(h, w, quality):
    kinds = ["views", "noise"] if h * w > 4096 else ["views", "noise", "black", "white", "grey"]
    for kind in kinds:
        x = content(kind, h, w, h * 131 + w)
        assert ours(x, quality) == pil_jpeg(x, quality), (kind, h, w, quality)


@pytest.mark.parametrize("quality", [75, 100])
def test_900x1600(quality):
    x = O.to_u8(O.views(11, 1, 900, 1600)[0])
    assert ours(x, quality) == pil_jpeg(x, quality)


def test_checkerboard_reaches_the_largest_categories():
    yy, xx = np.mgrid[0:32, 0:48]
    x = np.where(((yy + xx) & 1)[..., None], 255, 0).astype(np.uint8).repeat(3, -1)
    x[:16, :16] = 0  # a black block then a white one: the DC difference spans category 11
    x[16:, 16:32] = 255
    b = J.quantised_blocks(x, 100)
    pred, dc_cats = [0, 0, 0], []
    for mcu in b:
        for k, blk in enumerate(mcu):
            c = 0 if k < 4 else k - 3
            dc_cats.append(J._category(int(blk[0]) - pred[c]))
            pred[c] = int(blk[0])
    assert max(dc_cats) == 11
    assert max(J._category(int(v)) for v in b[..., 1:].ravel()) == 10
    assert ours(x, 100) == pil_jpeg(x, 100)


def test_zero_runs_zrl_and_eob():
    """Coefficients placed directly: ZRL only before a nonzero coefficient, EOB only when coefficient 63 is zero."""
    for last in (17, 33, 48, 62, 63):
        blk = np.zeros((1, 6, 64), np.int64)
        blk[0, 0, last] = 5
        blk[0, 4, 63] = -3
        words = J.block_codes(blk[0, 0], 0, 0)
        zrl = J.AC_CODES[0][0xF0]
        assert words.count(zrl) == (last - 1) // 16
        assert (words[-1] == J.AC_CODES[0][0x00]) == (last < 63)
    # image content with long zero runs: flat blocks with one sharp feature
    x = np.full((48, 64, 3), 90, np.uint8)
    x[5, 7] = 255
    x[21, 40:44] = 0
    x[40:48, 56:64] = np.eye(8, dtype=np.uint8)[..., None] * 200
    for q in (50, 90, 100):
        assert ours(x, q) == pil_jpeg(x, q)


def test_scan_dense_in_ff_bytes():
    x = np.random.default_rng(3).integers(0, 256, (64, 64, 3), dtype=np.uint8)
    ref = pil_jpeg(x, 100)
    assert ref[J.HEADER_BYTES:-2].count(b"\xff\x00") > 50
    assert ours(x, 100) == ref


def test_padding_forms_an_ff_byte():
    """Seed found with the restatement: the 1-bits padding the last byte make it 0xFF, which is stuffed too."""
    x = np.random.default_rng(5).integers(0, 256, (8, 8, 3), dtype=np.uint8)
    blocks = J.quantised_blocks(x, 100)
    assert J.scan_bits(blocks) % 8 != 0
    seg = J.entropy_code(blocks)
    assert seg.endswith(b"\xff\x00")
    assert ours(x, 100) == pil_jpeg(x, 100)


# ------------------------------------------------------------------------------------------------ the generated data set
def golden():
    return torch.load(os.path.join(GOLDEN, "val_set_jpeg.pt"), weights_only=False)


def _views(name, entry):
    from oracle.make_golden_val_set import case_views
    return case_views(name, entry["seed"])


def _expected_paths(entry):
    paths = []
    for template in entry["templates"]:
        for t in range(entry["T"]):
            for idx, view in enumerate(entry["view_order"]):
                stem, ext = os.path.splitext(os.path.basename(template["filename"][idx]))
                paths.append(f"{view}/{stem}_gen_{t}{ext}")
    return paths


@pytest.mark.parametrize("name", ["224x400", "272x736", "424x800", "raw_224x400"])
def test_oracle_reproduces_the_reference_files(name):
    entry = golden()[name]
    views = _views(name, entry)
    paths = _expected_paths(entry)
    u8 = O.to_u8(views).reshape(-1, *views.shape[3:])
    picks = range(len(paths)) if entry["config"] is None else (0, len(paths) - 1)  # 900 x 1600 canvases: two of them
    for i in picks:
        x = u8[i]
        if entry["config"] is not None:
            _, back_resize, pad, _ = entry["config"]
            canvas = (back_resize[0] + pad[1] + pad[3], back_resize[1] + pad[0] + pad[2])
            x = O.place(O.resample_u8(x, *back_resize), canvas, pad[1], pad[0])
        data = J.encode(x, 75)
        assert (len(data), hashlib.sha256(data).hexdigest()) == entry["files"][paths[i]], paths[i]


@pytest.mark.parametrize("name", ["224x400", "raw_224x400"])
def test_writer_host_logic(name, tmp_path, monkeypatch):
    """save_generated_views through the CPU restatements: the reference's paths, names, files and returned labels."""
    jpeg_ops_emulator.install(monkeypatch)
    image_ops_emulator.install(monkeypatch)
    entry = golden()[name]
    views = torch.from_numpy(_views(name, entry))
    for v in entry["view_order"]:
        (tmp_path / v).mkdir()
    protocol = None
    if entry["config"] is not None:
        protocol = fid.FIDProtocol(*entry["config"])
        protocol.use_cuda_graph = False
    templates = copy.deepcopy(entry["templates"])
    labels = fid.save_generated_views(views, templates, str(tmp_path), entry["view_order"], protocol)
    assert labels == entry["labels"] and labels is not templates and labels[0] is not templates[0]
    written = sorted(str(p.relative_to(tmp_path)) for p in tmp_path.rglob("*.jpg"))
    assert written == sorted(entry["files"]) == sorted(_expected_paths(entry))
    for rel, (n, sha) in entry["files"].items():
        data = (tmp_path / rel).read_bytes()
        assert (len(data), hashlib.sha256(data).hexdigest()) == (n, sha), rel


def test_writer_rejects_bad_arguments(tmp_path):
    entry = golden()["raw_224x400"]
    views = torch.zeros(2, 1, 6, 8, 8, 3)
    with pytest.raises(ValueError, match="B, T, n_cam"):
        fid.save_generated_views(views[0], entry["templates"], str(tmp_path), entry["view_order"])
    with pytest.raises(ValueError, match="templates"):
        fid.save_generated_views(views, entry["templates"][:1], str(tmp_path), entry["view_order"])
    bad = copy.deepcopy(entry["templates"])
    bad[1]["filename"][2] = bad[1]["filename"][2][:-4] + ".png"
    with pytest.raises(ValueError, match="JPEG"):
        fid.save_generated_views(views, bad, str(tmp_path), entry["view_order"])
    assert not any(tmp_path.iterdir())


def test_encoder_buffers_grow_to_what_was_measured(monkeypatch):
    """encode_jpeg's retry: noise needs more than its first guess of entropy-coded bytes."""
    from magicdrive_b200 import jpeg_ops
    jpeg_ops_emulator.install(monkeypatch)
    calls = []
    inner = jpeg_ops.jpeg_encode_u8

    def counting(*a, **k):
        calls.append(inner(*a, **k))
        return calls[-1]
    monkeypatch.setattr(jpeg_ops, "jpeg_encode_u8", counting)
    x = np.random.default_rng(1).integers(0, 256, (3, 40, 72, 3), dtype=np.uint8)
    x[1] = 128
    files = jpeg_ops.encode_jpeg(torch.from_numpy(x), 100)
    assert files == [pil_jpeg(v, 100) for v in x]
    assert len(calls) == 2 and (calls[0][:, 2] == -1).all() and (calls[1][:, 2] >= 0).all()
