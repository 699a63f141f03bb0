"""Fixture of the FID evaluation protocol (tests/golden/fid_protocol.pt), produced by the reference's own steps on the CPU:

    python -m oracle.make_golden_fid_protocol

For each shipped config (image_size, back_resize, back_pad and augment2d.resize read from the reference's dataset yaml
files), seeded float32 views (oracle/fid_protocol.views) go through:
* diffusers' numpy_to_pil (utils/pil_utils.py, loaded from the reference tree);
* the generation post-processing of perception/data_prepare/val_set_gen.py:107-116, torchvision
  Resize(back_resize, BICUBIC) and Pad(back_pad), saved under a nuScenes-style `.jpg` name as copy_save_image does;
* the scoring side of tools/fid_score.py:474-482 on the saved file: its ImagePathDataset (Image.open().convert("RGB")),
  Resize((int(900 r), int(1600 r)), BICUBIC) and its own top_center_crop.  ToTensor is left out: the stored result is
  the uint8 image it would divide by 255.
Stored: the config values, the seeds and the final uint8 images (lzma-compressed differences along the width) with
their sha256.  The 900 x 1600 intermediates are not stored.
"""
import hashlib
import importlib.util
import os
import sys
import tempfile

import numpy as np
import torch
import yaml

from oracle import fid_protocol as O
from oracle.make_golden_fid import reference_modules
from oracle.ref_shim import REF
from tests.common import GOLDEN

N_VIEWS = 1
VIEW_ARGS = dict(noise=0.0, ties=0.002)  # smooth views: the file stays below 1 MB
SEEDS = {"224x400": 101, "272x736": 102, "424x800": 103}
YAML = {"224x400": "Nuscenes.yaml", "272x736": "Nuscenes_map_cache_box_272x736.yaml",
        "424x800": "Nuscenes_400_map_cache_box_424x800.yaml"}


def _find(d, key):
    if isinstance(d, dict):
        if key in d:
            return d[key]
        for v in d.values():
            r = _find(v, key)
            if r is not None:
                return r
    return None


def reference_config(name):
    with open(os.path.join(REF, "configs/dataset", YAML[name])) as f:
        d = yaml.safe_load(f)
    image_size = tuple(_find(d, "image_size"))
    ratio = float(np.mean(_find(d, "augment2d")["resize"][0]))
    return image_size, tuple(_find(d, "back_resize")), tuple(_find(d, "back_pad")), ratio


def _pil_utils():
    spec = importlib.util.spec_from_file_location("ref_pil_utils", os.path.join(
        REF, "third_party/diffusers/src/diffusers/utils/pil_utils.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def reference_chain(views, cfg, fid_score, numpy_to_pil, tmp):
    import torchvision
    from torchvision.transforms import InterpolationMode
    image_size, back_resize, back_pad, ratio = cfg
    post_trans = torchvision.transforms.Compose([
        torchvision.transforms.Resize(list(back_resize), interpolation=InterpolationMode.BICUBIC),
        torchvision.transforms.Pad(list(back_pad))])
    files = []
    for i, img in enumerate(numpy_to_pil(views)):
        path = os.path.join(tmp, f"n008-2018-08-01-15-16-36-0400__CAM_FRONT__15331032{i:05d}_gen_0.jpg")
        post_trans(img).save(path)
        files.append(path)
    size = (int(900 * ratio), int(1600 * ratio))
    score = torchvision.transforms.Compose([
        torchvision.transforms.Resize(size, interpolation=torchvision.transforms.InterpolationMode.BICUBIC),
        lambda x: fid_score.top_center_crop(x, target_size=list(image_size))])
    ds = fid_score.ImagePathDataset(files, transforms=score)
    return np.stack([np.asarray(ds[i]) for i in range(len(ds))])


def main():
    _, fid_score = reference_modules()
    numpy_to_pil = _pil_utils().numpy_to_pil
    entries = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, seed in SEEDS.items():
            cfg = reference_config(name)
            assert cfg == O.CONFIGS[name], (name, cfg)
            v = O.views(seed, N_VIEWS, *cfg[0], **VIEW_ARGS)
            out = reference_chain(v, cfg, fid_score, numpy_to_pil, tmp)
            assert out.shape == (N_VIEWS, *cfg[0], 3) and out.dtype == np.uint8
            assert np.array_equal(out, O.generated(O.to_u8(v), cfg)), f"{name}: oracle and reference chain differ"
            entries[name] = dict(config=cfg, seed=seed, n_views=N_VIEWS, view_args=VIEW_ARGS, shape=out.shape,
                                 delta_lzma=O.golden_delta(out), sha256=hashlib.sha256(out.tobytes()).hexdigest())
            assert np.array_equal(O.golden_images(entries[name]), out)
    path = os.path.join(GOLDEN, "fid_protocol.pt")
    torch.save(entries, path)
    print(f"[make_golden_fid_protocol] wrote {path}: {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    sys.exit(main())
