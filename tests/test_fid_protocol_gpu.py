"""The FID protocol on the sm_90a path: mdb_resample_u8 and mdb_jpeg_roundtrip_u8 byte for byte against the integer
restatement (oracle/fid_protocol.py) and Pillow, FIDProtocol.generated against the reference's own chain
(tests/golden/fid_protocol.pt), FIDStatistics(protocol=...) against the reference's Pillow-and-files route, graph replay
against eager runs, and FIDStatistics without a protocol unchanged."""
import io

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from magicdrive_b200 import _lib, arch, fid, image_ops  # noqa: E402
from magicdrive_b200.models import InceptionV3  # noqa: E402
from oracle import fid_protocol as O  # noqa: E402
from tests.common import GOLDEN, record  # noqa: E402
from tests.test_fid_protocol_cpu import JPEG_SIZES, KINDS, RESIZES, images  # noqa: E402

Image = pytest.importorskip("PIL.Image")


def _pil_resize(a, h, w):
    return np.asarray(Image.fromarray(a).resize((w, h), Image.BICUBIC))


def _pil_jpeg(a, quality=None):
    buf = io.BytesIO()
    Image.fromarray(a).save(buf, format="JPEG", **({} if quality is None else dict(quality=quality, subsampling=2)))
    with Image.open(io.BytesIO(buf.getvalue())) as im:
        return np.asarray(im.convert("RGB"))


def _tables(h, w, rh, rw):
    t = lambda i, o: None if i == o else torch.from_numpy(fid.bicubic_table(i, o)).cuda()
    return t(w, rw), t(h, rh)


def _first_diff(a, b):
    idx = np.argwhere(a != b)
    return f"{len(idx)} bytes differ, first at {tuple(idx[0])}: {a[tuple(idx[0])]} vs {b[tuple(idx[0])]}" if len(idx) else ""


@pytest.mark.parametrize("src,dst", RESIZES, ids=lambda v: "x".join(map(str, v)))
def test_resample_u8_bit_exact(cuda_lib, src, dst):
    batch = np.stack([images(*src, kind, seed=i) for i, kind in enumerate(KINDS)])
    got = image_ops.resample_u8(torch.from_numpy(batch).cuda(), dst, *_tables(*src, *dst)).cpu().numpy()
    want = np.stack([_pil_resize(a, *dst) for a in batch])
    assert np.array_equal(O.resample_u8(batch, *dst), want)
    assert np.array_equal(got, want), _first_diff(got, want)


@pytest.mark.parametrize("nhwc", [True, False])
def test_resample_u8_fused_rounding_pad_and_crop(cuda_lib, nhwc):
    """fp32 [0, 1] input with numpy_to_pil's rounding (ties included), written at an offset of a zero canvas, and an
    output crop window; a guard byte pattern in `out` must be overwritten everywhere."""
    v = O.views(7, 2, 37, 53)
    x = torch.from_numpy(v).cuda()
    x = x if nhwc else x.permute(0, 3, 1, 2).contiguous()
    u8 = O.to_u8(v)
    for size, crop, canvas, offset in [((74, 106), None, (80, 120), (4, 9)), ((20, 30), (3, 5, 15, 21), (15, 21), (0, 0)),
                                       ((37, 106), (0, 2, 37, 100), (40, 104), (1, 3)), ((37, 53), None, (40, 60), (2, 2)),
                                       ((90, 53), (10, 0, 70, 53), (70, 53), (0, 0))]:
        out = torch.full((2, *canvas, 3), 0xA5, dtype=torch.uint8, device="cuda")
        image_ops.resample_u8(x, size, *_tables(37, 53, *size), nhwc=nhwc, crop=crop, canvas=canvas, offset=offset, out=out)
        want = O.place(O.resample_u8(u8, *size), canvas, *offset, crop)
        got = out.cpu().numpy()
        assert np.array_equal(got, want), (size, crop, _first_diff(got, want))


@pytest.mark.parametrize("hw", JPEG_SIZES, ids=lambda v: "x".join(map(str, v)))
def test_jpeg_roundtrip_u8_bit_exact(cuda_lib, hw):
    batch = np.stack([images(*hw, kind, seed=10 + i) for i, kind in enumerate(KINDS)])
    got = image_ops.jpeg_roundtrip_u8(torch.from_numpy(batch).cuda()).cpu().numpy()
    want = np.stack([_pil_jpeg(a) for a in batch])
    assert np.array_equal(got, want), _first_diff(got, want)
    assert np.array_equal(O.jpeg_roundtrip_u8(batch), want)


@pytest.mark.parametrize("quality", [1, 30, 50, 90, 100])
def test_jpeg_roundtrip_u8_other_qualities(cuda_lib, quality):
    batch = np.stack([images(37, 53, kind, seed=20 + i) for i, kind in enumerate(KINDS)])
    x = torch.from_numpy(batch).cuda()
    got = image_ops.jpeg_roundtrip_u8(x, quality, out=x).cpu().numpy()  # in place
    want = np.stack([_pil_jpeg(a, quality) for a in batch])
    assert np.array_equal(got, want), _first_diff(got, want)


def test_kernel_argument_errors(cuda_lib):
    x = torch.zeros(1, 16, 16, 3, dtype=torch.uint8, device="cuda")
    tw, th = _tables(16, 16, 8, 8)
    with pytest.raises(_lib.MdbError, match="outside the 8x8 resize"):
        image_ops.resample_u8(x, (8, 8), tw, th, crop=(2, 0, 8, 8))
    with pytest.raises(_lib.MdbError, match="outside the"):
        image_ops.resample_u8(x, (8, 8), tw, th, canvas=(8, 8), offset=(1, 0))
    with pytest.raises(_lib.MdbError, match="coefficients are required"):
        image_ops.resample_u8(x, (8, 8), None, th)
    with pytest.raises(_lib.MdbError, match="quality"):
        image_ops.jpeg_roundtrip_u8(x, 0)
    with pytest.raises(ValueError, match="planes holds"):
        image_ops.jpeg_roundtrip_u8(x, planes=torch.empty(10, dtype=torch.uint8, device="cuda"))


@pytest.mark.parametrize("name", sorted(O.CONFIGS))
def test_generated_equals_reference_chain_fixture(cuda_lib, name):
    """protocol.generated on the fixture's seeded views == the reference's numpy_to_pil, post_trans, .jpg save and load,
    scoring resize and top_center_crop, stored in tests/golden/fid_protocol.pt."""
    e = torch.load(f"{GOLDEN}/fid_protocol.pt", weights_only=False)[name]
    assert tuple(e["config"]) == O.CONFIGS[name]
    v = O.views(e["seed"], e["n_views"], *e["config"][0], **e["view_args"])
    p = fid.FIDProtocol.for_config(name)
    got = p.generated(torch.from_numpy(v).cuda()[None]).cpu().numpy()
    want = O.golden_images(e)
    assert np.array_equal(got, want), _first_diff(got, want)
    nchw = torch.from_numpy(v).cuda().permute(0, 3, 1, 2).contiguous()
    assert np.array_equal(p.generated(nchw).cpu().numpy(), want)


@pytest.mark.parametrize("name", sorted(O.CONFIGS))
def test_generated_and_real_equal_oracle_on_batches(cuda_lib, name):
    cfg = O.CONFIGS[name]
    v = O.views(40, 3, *cfg[0])
    p = fid.FIDProtocol.for_config(name)
    got = p.generated(torch.from_numpy(v).cuda().reshape(1, 3, *v.shape[1:])).cpu().numpy()
    assert np.array_equal(got, O.generated(O.to_u8(v), cfg))
    real = np.stack([images(900, 1600, k, seed=50 + i) for i, k in enumerate(("smooth", "random"))])
    got = p.real(torch.from_numpy(real)).cpu().numpy()
    assert np.array_equal(got, O.real(real, cfg)), _first_diff(got, O.real(real, cfg))


def test_graph_replay_equals_eager(cuda_lib):
    cfg = O.CONFIGS["224x400"]
    p, eager = fid.FIDProtocol.for_config("224x400"), fid.FIDProtocol.for_config("224x400")
    eager.use_cuda_graph = False
    for seed in (1, 2, 3):  # the first call captures, the later ones replay with new inputs
        x = torch.from_numpy(O.views(seed, 2, *cfg[0])).cuda()[None]
        assert torch.equal(p.generated(x), eager.generated(x))
        r = torch.from_numpy(np.stack([images(900, 1600, "smooth", seed=seed)]))
        assert torch.equal(p.real(r), eager.real(r))
    assert len(p._graphs) == 2


_MODEL = {}


def _model():
    if not _MODEL:
        m = InceptionV3([3]).cuda()
        m.load_state_dict(arch.inception_synthetic_state_dict(3, seed=3))
        _MODEL["m"] = m
    return _MODEL["m"]


def test_statistics_match_the_reference_file_route(cuda_lib, tmp_path):
    """FIDStatistics(protocol=...) on device views == the reference's route on files: Pillow resize and pad, save as .jpg,
    load, scoring resize and top_center_crop, ToTensor, then the same Inception.  Real images: the path helper over
    the saved JPEGs == the same files through PIL's scoring resize and crop."""
    import torchvision.transforms as TF
    model = _model()
    name = "272x736"
    cfg = O.CONFIGS[name]
    image_size, back_resize, pad, ratio = cfg
    p = fid.FIDProtocol.for_config(name)
    v = O.views(60, 4, *image_size)
    st = fid.FIDStatistics(model, dims=2048, protocol=p)
    st.update(torch.from_numpy(v).cuda().reshape(2, 2, *v.shape[1:]))
    files = []
    for i, a in enumerate(O.to_u8(v)):
        canvas = Image.new("RGB", (back_resize[1] + pad[0] + pad[2], back_resize[0] + pad[1] + pad[3]))
        canvas.paste(Image.fromarray(a).resize(back_resize[::-1], Image.BICUBIC), (pad[0], pad[1]))
        f = tmp_path / f"CAM_{i}_gen_0.jpg"
        canvas.save(f)
        files.append(f)
    (rh, rw), (top, left, fh, fw) = O.scoring_window(image_size, ratio)
    score = TF.Compose([TF.Resize((rh, rw), interpolation=TF.InterpolationMode.BICUBIC),
                        lambda im: im.crop((left, top, left + fw, top + fh)), TF.ToTensor()])
    act = fid.get_activations(files, model, batch_size=4, dims=2048, device="cuda", num_workers=0, transforms=score)
    err = np.abs(st.activations() - act).max()
    record(f"[parity] FIDStatistics(protocol) vs the reference's file route: max abs diff {err:.3e}")
    assert err <= 1e-6 * np.abs(act).max()
    mu, sigma = st.statistics()
    assert np.allclose(mu, act.mean(0), rtol=1e-12, atol=1e-12)
    assert np.allclose(sigma, np.cov(act, rowvar=False), rtol=1e-10, atol=1e-12)
    mu_r, sigma_r = fid.protocol_statistics_of_path(tmp_path, model, p, batch_size=4)
    assert np.allclose(mu_r, mu, rtol=1e-12, atol=1e-12) and np.allclose(sigma_r, sigma, rtol=1e-10, atol=1e-12)


def test_statistics_without_protocol_unchanged(cuda_lib):
    model = _model()
    g = torch.Generator(device="cuda").manual_seed(4)
    views = torch.rand(1, 3, 224, 400, 3, device="cuda", generator=g)
    st = fid.FIDStatistics(model, dims=2048)
    st.update(views)
    direct = model.features(views.reshape(-1, 224, 400, 3), nhwc=True, quantize=True)[0]
    assert np.array_equal(st.activations(), fid._to_features(direct))
