"""FID host side without a GPU: the Fréchet distance and statistics, the InceptionV3 wrapper's names, loading and
rejections, and the real InceptionEngine host code (BatchNorm folding, K64 packing, column-slice wiring) through
tests/ops_emulator.py against the fp32 oracle (oracle/fid_inception.py)."""
import numpy as np
import pytest
import torch
from scipy import linalg

from magicdrive_b200 import arch, engine, fid
from magicdrive_b200.engine import InceptionEngine
from magicdrive_b200.models import InceptionV3
from oracle import fid_inception as fid_oracle
from tests import ops_emulator


def _direct_fid(mu1, s1, mu2, s2):
    """The same distance through the eigenvalues of s1 s2 (real and >= 0 for covariances)."""
    ev = np.linalg.eigvals(s1 @ s2)
    return float(((mu1 - mu2) ** 2).sum() + np.trace(s1) + np.trace(s2) - 2 * np.sqrt(np.clip(ev.real, 0, None)).sum())


def _stats(n, d, seed):
    a = np.random.default_rng(seed).standard_normal((n, d)) @ np.random.default_rng(seed + 1).standard_normal((d, d))
    return a.mean(0), np.cov(a, rowvar=False)


def test_frechet_distance_matches_formula():
    m1, s1 = _stats(400, 32, 0)
    m2, s2 = _stats(400, 32, 5)
    d = fid.calculate_frechet_distance(m1, s1, m2, s2)
    assert abs(d - _direct_fid(m1, s1, m2, s2)) <= 1e-8 * abs(d)
    assert abs(fid.calculate_frechet_distance(m1, s1, m1, s1)) < 1e-6


def test_frechet_distance_singular_takes_eps_branch(monkeypatch):
    m1, s1 = _stats(400, 16, 0)
    calls = []
    real = linalg.sqrtm

    def sqrtm(a):
        calls.append(a)
        return real(a) if len(calls) > 1 else np.full_like(a, np.inf)  # a product whose root is not finite
    monkeypatch.setattr(fid.linalg, "sqrtm", sqrtm)
    d = fid.calculate_frechet_distance(m1, s1, m1, s1, eps=1e-3)
    assert len(calls) == 2 and np.allclose(calls[1], (s1 + 1e-3 * np.eye(16)) @ (s1 + 1e-3 * np.eye(16)))
    assert np.isfinite(d)


def test_frechet_distance_raises():
    with pytest.raises(AssertionError):
        fid.calculate_frechet_distance(np.zeros(3), np.eye(3), np.zeros(4), np.eye(4))
    neg = np.diag([-1.0, 1.0])  # sqrtm(neg) = diag(i, 1): a large imaginary diagonal
    with pytest.raises(ValueError):
        fid.calculate_frechet_distance(np.zeros(2), neg, np.zeros(2), np.eye(2))


def test_statistics_are_numpy_mean_and_cov(tmp_path):
    class Fake(torch.nn.Module):
        output_blocks = [3]

        def forward(self, x):
            return [x.mean((2, 3), keepdim=True).repeat(1, 4, 1, 1)[:, :8]]
    from PIL import Image
    rng = np.random.default_rng(0)
    for i in range(7):
        Image.fromarray(rng.integers(0, 256, (9 + i, 11, 3), dtype=np.uint8)).save(tmp_path / f"{i}.png")
    files = sorted(tmp_path.glob("*.png"))
    act = fid.get_activations(files, Fake(), batch_size=1, dims=8, num_workers=0)
    mu, sigma = fid.calculate_activation_statistics(files, Fake(), batch_size=1, dims=8, num_workers=0)
    assert np.array_equal(mu, np.mean(act, 0)) and np.array_equal(sigma, np.cov(act, rowvar=False))
    m2, s2 = fid.compute_statistics_of_path(str(tmp_path), Fake(), 1, 8, "cpu", 0)
    assert np.array_equal(m2, mu) and np.array_equal(s2, sigma)
    fid.save_fid_stats([str(tmp_path), str(tmp_path / "s.npz")], 1, "cpu", 8, 0, model=Fake())
    m3, s3 = fid.compute_statistics_of_path(str(tmp_path / "s.npz"), None, 1, 8, "cpu")
    assert np.array_equal(m3, mu) and np.array_equal(s3, sigma)
    with pytest.raises(ValueError):
        fid.calculate_fid_given_paths([str(tmp_path), str(tmp_path)], 1, "cpu", 2048)  # no model, no weights path


def _torchvision_state_dict():
    from torchvision.models import inception as tvi
    return tvi.Inception3(num_classes=1008, aux_logits=False, init_weights=False).state_dict()


def test_parameter_names_and_shapes_match_the_reference_wrapper():
    """The reference wrapper takes torchvision's Inception3 layers into blocks 0-3 in this order (inception.py:84-124)."""
    tv = _torchvision_state_dict()
    want = []
    for i, mods in enumerate(arch.INCEPTION_BLOCKS):
        for j, m in enumerate(mods):
            want += [(f"blocks.{i}.{j}" + k[len(m):], tuple(v.shape)) for k, v in tv.items() if k.split(".")[0] == m]
    got = [(k, tuple(v.shape)) for k, v in InceptionV3([3]).state_dict().items()]
    assert got == want
    assert [k for k, _ in InceptionV3([1]).state_dict().items()] == [k for k, _ in want if k.startswith(("blocks.0", "blocks.1"))]


def test_both_naming_schemes_load_and_missing_keys_raise(tmp_path):
    sd = arch.inception_synthetic_state_dict(3, seed=1)
    m = InceptionV3([3])
    m.load_state_dict(sd)
    tvnames = {p: n for n, (p, _) in arch.inception_convs(3).items()}
    fid_file = {}
    for k, v in sd.items():
        if k.endswith("num_batches_tracked"):
            continue
        layer = k.rsplit(".", 2)[0]
        fid_file[tvnames[layer] + k[len(layer):]] = v
    fid_file["fc.weight"], fid_file["fc.bias"] = torch.zeros(1008, 2048), torch.zeros(1008)
    torch.save(fid_file, tmp_path / "pt_inception.pth")
    m2 = InceptionV3.from_pretrained(tmp_path / "pt_inception.pth", [0, 3])
    for k, v in m2.state_dict().items():
        assert torch.equal(v, sd[k]), k
    del fid_file["Mixed_6b.branch7x7_2.bn.running_var"]
    with pytest.raises(RuntimeError, match="Missing"):
        InceptionV3([3]).load_state_dict(fid_file)


def test_constructor_rejections():
    with pytest.raises(ValueError):
        InceptionV3(use_fid_inception=False)
    with pytest.raises(ValueError):
        InceptionV3(requires_grad=True)
    m = InceptionV3([2, 0])
    assert m.output_blocks == [0, 2] and m.DEFAULT_BLOCK_INDEX == 3 and m.BLOCK_INDEX_BY_DIM == {64: 0, 192: 1, 768: 2, 2048: 3}


@pytest.mark.parametrize("size,resize", [((299, 299), True), ((97, 131), True), ((150, 171), False)])
def test_engine_host_logic_through_emulated_ops(monkeypatch, size, resize):
    ops_emulator.install(monkeypatch)
    monkeypatch.setattr(engine._Weights, "fold_dtype", torch.float32)  # the fold's algebra to fp32, apart from bf16 storage
    sd = arch.inception_synthetic_state_dict(3, seed=2)
    eng = InceptionEngine(sd, torch.device("cpu"))
    x = fid_oracle.images(2, *size, seed=3)
    ours = eng.forward(x, nhwc=False, quantize=False, resize=resize, normalize=True, output_blocks=(0, 1, 2, 3))
    ref = fid_oracle.forward(sd, x, (0, 1, 2, 3), resize=resize)
    for o, r in zip(ours, ref):
        assert o.shape == r.shape
        torch.testing.assert_close(o, r, rtol=1e-4, atol=1e-4 * r.abs().max().item())
    # NHWC input with 8-bit rounding: the FIDStatistics route
    ours = eng.forward(x.permute(0, 2, 3, 1), nhwc=True, quantize=True, resize=resize, normalize=True, output_blocks=(3,))
    torch.testing.assert_close(ours[0], ref[3], rtol=1e-4, atol=1e-4 * ref[3].abs().max().item())


# ------------------------------------------------------------------ against the reference's own code (oracle/make_golden_fid.py)
def _fixture():
    from tests.common import golden
    return golden("fid_inception.pt")


def test_frechet_distance_matches_the_reference():
    """tools/fid_score.py:calculate_frechet_distance on the stored pairs, including the eps branch (zero covariances) and
    the ValueError on an imaginary diagonal."""
    for c in _fixture()["frechet"]:
        if isinstance(c["value"], str):
            with pytest.raises(ValueError):
                fid.calculate_frechet_distance(c["mu1"], c["sigma1"], c["mu2"], c["sigma2"], eps=c["eps"])
            continue
        d = fid.calculate_frechet_distance(c["mu1"], c["sigma1"], c["mu2"], c["sigma2"], eps=c["eps"])
        assert abs(d - c["value"]) <= 1e-8 * abs(c["value"]), (d, c["value"])


def test_parameter_names_and_shapes_equal_the_reference_run():
    assert [(k, tuple(v.shape)) for k, v in InceptionV3([0, 1, 2, 3]).state_dict().items()] == \
        [(k, tuple(s)) for k, s in _fixture()["param_shapes"]]


@pytest.mark.parametrize("key", ["224x400", "299x299", "75x97"])
def test_oracle_reproduces_the_reference_at_every_block(key):
    fx = _fixture()
    sd = arch.inception_synthetic_state_dict(3, fx["seed_weights"])
    entry = fx["taps"][key]
    with torch.no_grad():
        outs = fid_oracle.forward(sd, fx["inputs"][key].float() / 255, (0, 1, 2, 3))
    torch.testing.assert_close(outs[3][:, :, 0, 0], entry["features"], rtol=1e-4, atol=1e-5)
    for i in range(3):
        assert tuple(outs[i].shape) == tuple(entry[f"block{i}_shape"])
        torch.testing.assert_close(outs[i].mean((2, 3)), entry[f"block{i}_mean"], rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(outs[i].reshape(-1)[entry[f"block{i}_idx"]], entry[f"block{i}_val"], rtol=1e-4, atol=1e-5)
