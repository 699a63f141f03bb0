"""Fixture of the generated data set's JPEG files (tests/golden/val_set_jpeg.pt), written by the reference's own code on the
CPU:

    python -m oracle.make_golden_val_set

`copy_save_image` is taken from perception/data_prepare/val_set_gen.py by `ast` (the module itself imports hydra,
accelerate and mmdet3d) and run as the reference runs it: its `post_trans` is built as lines 103-116 build it (torchvision
Resize(back_resize, BICUBIC) and Pad(back_pad) of each config, or nothing with `fid.raw_output: true`), on views that
diffusers' numpy_to_pil (loaded from the reference tree) turned into PIL images.  The views are seeded
(oracle/fid_protocol.views), B = 2 items x T = 2 generations x the 6 nuScenes cameras, with nuScenes-style file names.
Stored per case: the config, the seed, the templates, view_order, copy_save_image's returned list and, for every file it
wrote, the path relative to img_gen_dir, the length and the sha256.  No image and no reference source is stored.
"""
import ast
import hashlib
import os
import sys
import tempfile
import types

import torch

from oracle import fid_protocol as O
from oracle.make_golden_fid_protocol import _pil_utils, reference_config
from oracle.ref_shim import REF
from tests.common import GOLDEN

VIEW_ORDER = ["CAM_FRONT_LEFT", "CAM_FRONT", "CAM_FRONT_RIGHT", "CAM_BACK_RIGHT", "CAM_BACK", "CAM_BACK_LEFT"]
B, T = 2, 2
VIEW_ARGS = dict(noise=0.01, ties=0.01)
CASES = {"224x400": 201, "272x736": 202, "424x800": 203, "raw_224x400": 204}


def templates(seed):
    """B label entries as val_set_gen.py builds them: the 6 camera file names and the sample token."""
    out = []
    for b in range(B):
        stamp = 1533151603512404 + 1000 * seed + 37 * b
        out.append({"filename": [f"./data/nuscenes/samples/{v}/n008-2018-08-01-15-16-36-0400__{v}__{stamp + i}.jpg"
                                 for i, v in enumerate(VIEW_ORDER)],
                    "token": hashlib.sha256(f"{seed}-{b}".encode()).hexdigest()[:32]})
    return out


def case_views(name, seed):
    """float32 (B, T, 6, h, w, 3) views in [0, 1] of one case."""
    h, w = O.CONFIGS[name.replace("raw_", "")][0]
    return O.views(seed, B * T * len(VIEW_ORDER), h, w, **VIEW_ARGS).reshape(B, T, len(VIEW_ORDER), h, w, 3)


def copy_save_image():
    """The reference's copy_save_image, compiled from its source with the module's imports."""
    path = os.path.join(REF, "perception/data_prepare/val_set_gen.py")
    with open(path) as f:
        tree = ast.parse(f.read(), path)
    fn = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "copy_save_image")
    import copy
    from pathlib import Path
    scope = {"os": os, "copy": copy, "Path": Path}
    exec(compile(ast.Module(body=[fn], type_ignores=[]), path, "exec"), scope)
    return scope["copy_save_image"]


def post_trans(name):
    import torchvision
    from torchvision.transforms import InterpolationMode
    if name.startswith("raw_"):  # cfg.fid.raw_output
        return torchvision.transforms.Compose([])
    _, back_resize, back_pad, _ = reference_config(name)
    return torchvision.transforms.Compose([
        torchvision.transforms.Resize(list(back_resize), interpolation=InterpolationMode.BICUBIC),
        torchvision.transforms.Pad(list(back_pad))])


def main():
    save = copy_save_image()
    numpy_to_pil = _pil_utils().numpy_to_pil
    entries = {}
    for name, seed in CASES.items():
        views = case_views(name, seed)
        gen_imgs_list = [[numpy_to_pil(views[b, t]) for t in range(T)] for b in range(B)]
        tmp = templates(seed)
        with tempfile.TemporaryDirectory() as d:
            for v in VIEW_ORDER:
                os.makedirs(os.path.join(d, v))
            cfg = types.SimpleNamespace(dataset=types.SimpleNamespace(view_order=VIEW_ORDER),
                                        fid=types.SimpleNamespace(img_gen_dir=d))
            labels = save(tmp, cfg, gen_imgs_list, post_trans(name))
            files = {}
            for v in VIEW_ORDER:
                for f in sorted(os.listdir(os.path.join(d, v))):
                    data = open(os.path.join(d, v, f), "rb").read()
                    files[f"{v}/{f}"] = (len(data), hashlib.sha256(data).hexdigest())
        assert len(files) == B * T * len(VIEW_ORDER)
        entries[name] = dict(config=None if name.startswith("raw_") else reference_config(name), seed=seed, B=B, T=T,
                             view_args=VIEW_ARGS, view_order=VIEW_ORDER, templates=tmp, labels=labels, files=files)
    path = os.path.join(GOLDEN, "val_set_jpeg.pt")
    torch.save(entries, path)
    print(f"[make_golden_val_set] wrote {path}: {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    sys.exit(main())
