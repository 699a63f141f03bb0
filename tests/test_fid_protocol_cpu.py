"""The FID protocol on the CPU: the integer restatement (oracle/fid_protocol.py) against Pillow byte for byte, the library's
coefficient tables against it, FIDProtocol's configuration and argument checks, and its host logic over the operator
emulator."""
import io

import numpy as np
import pytest
import torch

from magicdrive_b200 import fid
from oracle import fid_protocol as O
from tests import image_ops_emulator

Image = pytest.importorskip("PIL.Image")


def images(h, w, kind, seed=0):
    rng = np.random.default_rng(seed)
    if kind == "random":
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind == "flat":
        return np.full((h, w, 3), rng.integers(0, 256, 3), np.uint8)
    if kind == "edges":  # a black / white step, the green channel flipped in the lower half
        a = np.zeros((h, w, 3), np.uint8)
        a[:, w // 3:] = 255
        a[h // 2:, :, 1] = 255 - a[h // 2:, :, 1]
        return a
    yy, xx = np.mgrid[0:h, 0:w]
    a = np.stack([(xx * 7 + yy * 3) % 256, np.sin(xx / 9.0) * 120 + 128, yy * 255 // max(h - 1, 1)], -1)
    return (a + rng.integers(-20, 20, a.shape)).clip(0, 255).astype(np.uint8)


KINDS = ("random", "flat", "edges", "smooth")


def pil_resize(a, h, w):
    return np.asarray(Image.fromarray(a).resize((w, h), Image.BICUBIC))


def pil_jpeg(a, quality=None):
    """Save under Pillow's defaults (or at `quality`, 4:2:0) and load back as RGB."""
    buf = io.BytesIO()
    kw = {} if quality is None else dict(quality=quality, subsampling=2)
    Image.fromarray(a).save(buf, format="JPEG", **kw)
    with Image.open(io.BytesIO(buf.getvalue())) as im:
        return np.asarray(im.convert("RGB"))


# every resize of the three configs, then odd sizes: 1-pixel images, non-integer factors up and down, one axis unchanged
RESIZES = [((224, 400), (896, 1600)), ((900, 1600), (225, 400)), ((272, 736), (544, 1472)), ((900, 1600), (450, 800)),
           ((424, 800), (848, 1600)), ((1, 1), (5, 7)), ((7, 5), (1, 1)), ((13, 17), (29, 11)), ((33, 45), (20, 100)),
           ((50, 3), (50, 9)), ((101, 67), (37, 67)), ((97, 7), (41, 3)), ((3, 100), (10, 33))]


@pytest.mark.parametrize("src,dst", RESIZES, ids=lambda v: "x".join(map(str, v)))
def test_resample_oracle_equals_pillow(src, dst):
    for i, kind in enumerate(KINDS):
        a = images(*src, kind, seed=i)
        assert np.array_equal(O.resample_u8(a, *dst), pil_resize(a, *dst)), kind


JPEG_SIZES = [(900, 1600), (224, 400), (225, 400), (1, 1), (2, 2), (3, 5), (4, 4), (5, 6), (8, 8), (9, 17), (16, 16),
              (17, 33), (31, 7), (101, 67), (6, 1), (1, 9)]


@pytest.mark.parametrize("hw", JPEG_SIZES, ids=lambda v: "x".join(map(str, v)))
def test_jpeg_oracle_equals_pillow_defaults(hw):
    for i, kind in enumerate(KINDS):
        a = images(*hw, kind, seed=10 + i)
        assert np.array_equal(O.jpeg_roundtrip_u8(a), pil_jpeg(a)), kind


@pytest.mark.parametrize("quality", [1, 30, 50, 90, 100])
def test_jpeg_oracle_equals_pillow_at_other_qualities(quality):
    for hw in [(37, 53), (16, 16)]:
        for i, kind in enumerate(KINDS):
            a = images(*hw, kind, seed=20 + i)
            assert np.array_equal(O.jpeg_roundtrip_u8(a, quality), pil_jpeg(a, quality)), (hw, kind)


@pytest.mark.parametrize("name", sorted(O.CONFIGS))
def test_whole_chain_oracle_equals_pillow(name):
    """Pillow's route: resize and pad the view, save as .jpg, load, resize to the scoring size, crop the top centre."""
    image_size, back_resize, pad, ratio = O.CONFIGS[name]
    a = images(*image_size, "smooth", seed=3)
    canvas = Image.new("RGB", (back_resize[1] + pad[0] + pad[2], back_resize[0] + pad[1] + pad[3]))
    canvas.paste(Image.fromarray(a).resize(back_resize[::-1], Image.BICUBIC), (pad[0], pad[1]))
    b = pil_jpeg(np.asarray(canvas))
    (rh, rw), (top, left, fh, fw) = O.scoring_window(image_size, ratio)
    want = np.asarray(Image.fromarray(b).resize((rw, rh), Image.BICUBIC).crop((left, top, left + fw, top + fh)))
    assert np.array_equal(O.generated(a, O.CONFIGS[name]), want)


@pytest.mark.parametrize("n_in,n_out", [(224, 896), (400, 1600), (900, 225), (1600, 400), (900, 450), (272, 544),
                                        (736, 1472), (1, 5), (7, 1), (13, 29), (97, 41), (3, 10), (100, 33)])
def test_bicubic_table_equals_oracle(n_in, n_out):
    first, count, kk = O.bicubic_coeffs(n_in, n_out)
    t = fid.bicubic_table(n_in, n_out)
    assert t.dtype == np.int32 and t.shape == (n_out, kk.shape[1] + 2)
    assert np.array_equal(t[:, 0], first) and np.array_equal(t[:, 1], count) and np.array_equal(t[:, 2:], kk)


def test_protocol_configs():
    assert fid.PROTOCOL_CONFIGS == O.CONFIGS
    p = fid.FIDProtocol.for_config("224x400")
    assert (p.canvas, p.score_resize, p.crop, p.jpeg, p.quality) == ((900, 1600), (225, 400), (1, 0, 224, 400), True, 75)
    p = fid.FIDProtocol.for_config("272x736", jpeg=False)
    assert (p.canvas, p.score_resize, p.crop, p.jpeg) == ((900, 1600), (450, 800), (178, 32, 272, 736), False)
    p = fid.FIDProtocol.for_config("424x800")
    assert (p.canvas, p.score_resize, p.crop) == ((900, 1600), (450, 800), (26, 0, 424, 800))
    q = fid.FIDProtocol((424, 800), (848, 1600), (0, 52, 0, 0), 0.5)
    assert repr(q) == repr(p)


def test_protocol_argument_errors():
    with pytest.raises(ValueError, match="unknown config"):
        fid.FIDProtocol.for_config("256x704")
    with pytest.raises(ValueError, match="smaller than image_size"):
        fid.FIDProtocol((224, 400), (896, 1600), (0, 4, 0, 0), 0.2)
    with pytest.raises(ValueError, match="non-negative"):
        fid.FIDProtocol((224, 400), (896, 1600), (0, -4, 0, 0), 0.25)
    with pytest.raises(ValueError, match="left, top, right, bottom"):
        fid.FIDProtocol((224, 400), (896, 1600), (0, 4), 0.25)
    with pytest.raises(ValueError, match="quality"):
        fid.FIDProtocol.for_config("224x400", quality=0)
    p = fid.FIDProtocol.for_config("224x400")
    with pytest.raises(ValueError, match="expected"):
        p.generated(torch.zeros(2, 224, 400))
    with pytest.raises(ValueError, match="expected uint8"):
        p.real(torch.zeros(1, 900, 1600, 3))
    with pytest.raises(ValueError, match="update_real needs"):
        fid.FIDStatistics(_FakeInception(), 2048).update_real(torch.zeros(1, 900, 1600, 3, dtype=torch.uint8))
    with pytest.raises(TypeError, match="FIDProtocol"):
        fid.FIDStatistics(_FakeInception(), 2048, protocol="224x400")


class _FakeInception:
    output_blocks = [3]


@pytest.fixture
def emulated(monkeypatch):
    image_ops_emulator.install(monkeypatch)
    monkeypatch.setattr(fid.FIDProtocol, "use_cuda_graph", False)


def _views(s, n_cam, h, w, seed):
    """Seeded float32 views in [0, 1] with smooth structure and noise."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    base = np.stack([0.5 + 0.4 * np.sin(xx / 13.0 + yy / 29.0), (xx / w) * 0.8 + 0.1, 0.5 + 0.45 * np.cos(yy / 7.0)], -1)
    v = base[None, None] + rng.standard_normal((s, n_cam, h, w, 3)).astype(np.float32) * 0.05
    return np.clip(v, 0, 1).astype(np.float32)


@pytest.mark.parametrize("name", ["224x400", "272x736"])
def test_protocol_host_logic_on_the_emulator(emulated, name):
    v = _views(1, 2, *O.CONFIGS[name][0], seed=1)
    p = fid.FIDProtocol.for_config(name)
    got = p.generated(torch.from_numpy(v))
    assert got.dtype == torch.uint8 and tuple(got.shape) == (2, *O.CONFIGS[name][0], 3)
    assert np.array_equal(got.numpy(), O.generated(O.to_u8(v.reshape(2, *v.shape[2:])), O.CONFIGS[name]))
    nchw = torch.from_numpy(v.reshape(2, *v.shape[2:])).permute(0, 3, 1, 2).contiguous()
    assert torch.equal(fid.FIDProtocol.for_config(name).generated(nchw), got)
    real = images(900, 1600, "smooth", seed=5)[None]
    assert np.array_equal(p.real(torch.from_numpy(real), device="cpu").numpy(), O.real(real, O.CONFIGS[name]))
    no_jpeg = fid.FIDProtocol.for_config(name, jpeg=False).generated(torch.from_numpy(v))
    assert np.array_equal(no_jpeg.numpy(), O.generated(O.to_u8(v.reshape(2, *v.shape[2:])), O.CONFIGS[name], jpeg=False))
