"""Fixture of the FID InceptionV3 and Fréchet distance (tests/golden/fid_inception.pt), produced by the reference's own code:
magicdrive/misc/inception.py:InceptionV3([0, 1, 2, 3]) and tools/fid_score.py:calculate_frechet_distance, loaded unmodified
from the reference tree (or its oracle/_ref snapshot).  Run on the CPU:

    python -m oracle.make_golden_fid

* Weights.  fid_inception_v3() (inception.py:197-221) fetches the pytorch-fid weights with `load_state_dict_from_url`.  That
  name is replaced in the loaded module's namespace, before InceptionV3 is built, by a function that returns seeded
  weights under torchvision's names (arch.inception_synthetic_state_dict, seed SEED_W; fc.* drawn the same way).  The
  reference's construction code runs unchanged and nothing reaches the network.
* Inputs.  Procedural uint8 images at 224x400, 299x299 and 75x97 (oracle/fid_inception.images), fed as x / 255.
* Stored per input: the 2048-d features (block 3); for blocks 0-2 the per-channel means and SAMPLE_N seeded elements.
* Fréchet distance.  tools/fid_score.py imports hydra, omegaconf and perception.common.nuscenes_utils at module level and
  `from magicdrive.misc.inception import InceptionV3`: those are stubbed.  It calls scipy.linalg.sqrtm(..., disp=False),
  whose `disp` argument current scipy no longer has; its `linalg` is given a sqrtm that accepts it and returns
  (sqrtm(a), 0.0) for disp=False (the reference discards the second value).  Stored: (mu1, sigma1, mu2, sigma2, eps,
  value or the exception's type) for seeded pairs, a pair of zero covariances (its root is not finite: the eps branch),
  a rank-deficient pair (complex root with a negligible imaginary part) and one that raises ValueError.
"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch

from magicdrive_b200 import arch
from oracle import fid_inception
from oracle.ref_shim import REF
from tests.common import GOLDEN

SEED_W = 5
SIZES = {"224x400": (1, 224, 400), "299x299": (1, 299, 299), "75x97": (2, 75, 97)}
SAMPLE_N = 500  # keeps the file below 1 MB with the uint8 inputs


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    sys.modules[name] = mod
    spec.loader.exec_module(mod)
    return mod


def _seeded_torchvision_state_dict(*a, **k):
    """Stands in for load_state_dict_from_url(FID_WEIGHTS_URL): seeded weights under torchvision Inception3's names."""
    from torchvision.models import inception as tvi
    keys = tvi.Inception3(num_classes=1008, aux_logits=False, init_weights=False).state_dict()
    sd = arch.inception_synthetic_state_dict(3, SEED_W)
    tv_of = {prefix: name for name, (prefix, _) in arch.inception_convs(3).items()}
    out = {}
    for k_, v in sd.items():
        layer = k_.rsplit(".", 2)[0]
        out[tv_of[layer] + k_[len(layer):]] = v
    g = torch.Generator().manual_seed(SEED_W)
    out["fc.weight"] = torch.randn(keys["fc.weight"].shape, generator=g) * 0.02
    out["fc.bias"] = torch.zeros(keys["fc.bias"].shape)
    assert set(out) == set(keys), set(keys) ^ set(out)
    return out


def reference_inception():
    """magicdrive/misc/inception.py as a module, with load_state_dict_from_url replaced by the seeded loader."""
    inception = _load("magicdrive.misc.inception", os.path.join(REF, "magicdrive/misc/inception.py"))
    inception.load_state_dict_from_url = _seeded_torchvision_state_dict
    return inception


def reference_modules():
    inception = reference_inception()
    for name in ("magicdrive", "magicdrive.misc", "perception", "perception.common"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["magicdrive.misc"].inception = inception
    nus = types.ModuleType("perception.common.nuscenes_utils")
    nus.sample_token_from_scene = lambda *a, **k: None
    sys.modules["perception.common.nuscenes_utils"] = nus
    omega = types.ModuleType("omegaconf")
    omega.OmegaConf = object
    hydra = types.ModuleType("hydra")
    hydra.main = lambda *a, **k: (lambda f: f)
    hu, hc, hcc = types.ModuleType("hydra.utils"), types.ModuleType("hydra.core"), types.ModuleType("hydra.core.hydra_config")
    hu.to_absolute_path = lambda p: p
    hcc.HydraConfig = object
    sys.modules.update({"omegaconf": omega, "hydra": hydra, "hydra.utils": hu, "hydra.core": hc,
                        "hydra.core.hydra_config": hcc})
    fid_score = _load("fid_score", os.path.join(REF, "tools/fid_score.py"))
    from scipy import linalg

    def sqrtm(a, disp=True):
        r = linalg.sqrtm(a)
        return r if disp else (r, 0.0)
    fid_score.linalg = types.SimpleNamespace(sqrtm=sqrtm)
    return inception, fid_score


def frechet_cases(fid_score):
    rng = np.random.default_rng(SEED_W)
    cases = []

    def add(mu1, s1, mu2, s2, eps=1e-6):
        try:
            val = float(fid_score.calculate_frechet_distance(mu1, s1, mu2, s2, eps=eps))
        except ValueError as e:
            val = type(e).__name__
        cases.append(dict(mu1=mu1, sigma1=s1, mu2=mu2, sigma2=s2, eps=eps, value=val))

    for d in (16, 64):
        a, b = rng.standard_normal((300, d)), rng.standard_normal((300, d)) * 1.3 + 0.2
        b = b @ (np.eye(d) + 0.1 * rng.standard_normal((d, d)))
        add(a.mean(0), np.cov(a, rowvar=False), b.mean(0), np.cov(b, rowvar=False))
    add(np.zeros(8), np.zeros((8, 8)), np.full(8, 0.5), np.zeros((8, 8)), eps=1e-3)  # one repeated image per set
    u, v = np.array([1.0, 2.0, 3.0]), np.array([3.0, -1.0, 0.0])
    add(np.zeros(3), np.outer(u, u), np.ones(3), np.outer(v, v))
    add(np.zeros(2), np.diag([-1.0, 1.0]), np.zeros(2), np.eye(2))  # raises: imaginary diagonal
    assert any(isinstance(c["value"], str) for c in cases)
    return cases


def main():
    torch.set_num_threads(1)  # fixed reduction order: a re-run reproduces the file bit for bit
    inception, fid_score = reference_modules()
    model = inception.InceptionV3([0, 1, 2, 3]).eval()
    sd = model.state_dict()
    g = torch.Generator().manual_seed(SEED_W)
    inputs, taps = {}, {}
    with torch.no_grad():
        for key, (n, h, w) in SIZES.items():
            img = (fid_inception.images(n, h, w, seed=len(inputs) + 1) * 255).round().to(torch.uint8)
            outs = model(img.float() / 255)
            feats = outs[3][:, :, 0, 0].clone()
            assert (feats > 0).float().mean() > 0.2, "features mostly dead"
            assert n == 1 or feats.std(0).mean() > 1e-3, "features do not vary across images"
            entry = dict(features=feats)
            for i in range(3):
                o = outs[i]
                idx = torch.randint(0, o.numel(), (SAMPLE_N,), generator=g)
                entry[f"block{i}_mean"] = o.mean((2, 3)).clone()
                entry[f"block{i}_idx"] = idx
                entry[f"block{i}_val"] = o.reshape(-1)[idx].clone()
                entry[f"block{i}_shape"] = tuple(o.shape)
            inputs[key], taps[key] = img, entry
    fx = dict(seed_weights=SEED_W, param_shapes=[(k, tuple(v.shape)) for k, v in sd.items()], inputs=inputs, taps=taps,
              frechet=frechet_cases(fid_score))
    torch.save(fx, os.path.join(GOLDEN, "fid_inception.pt"))
    print(f"[make_golden_fid] wrote {os.path.join(GOLDEN, 'fid_inception.pt')}")


if __name__ == "__main__":
    main()
