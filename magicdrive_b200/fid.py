"""Fréchet Inception Distance, host side (the reference's tools/fid_score.py:93-276, 341-358).

The Inception features come from `models.InceptionV3` on the device; statistics (np.mean, np.cov in float64) and the
Fréchet distance (scipy's sqrtm) are computed on the host, as the reference does.  `FIDStatistics` accumulates the
features of device image batches -- the denoiser's decoded views -- rounded to the 8-bit levels a saved PNG would hold,
so a generated set's FID needs no PNGs on disk.  Nothing here downloads weights: pass a model, or the path of the
pytorch-fid weights file.
"""
import os
import pathlib

import numpy as np
import torch
from scipy import linalg

from .models import InceptionV3

IMAGE_EXTENSIONS = {"bmp", "jpg", "jpeg", "pgm", "png", "ppm", "tif", "tiff", "webp"}


def calculate_frechet_distance(mu1, sigma1, mu2, sigma2, eps=1e-6):
    """d^2 = |mu1 - mu2|^2 + Tr(sigma1 + sigma2 - 2 (sigma1 sigma2)^(1/2)), in float64.

    When the matrix square root is not finite (a singular product), both covariances get eps added to their diagonal
    and the root is taken again.  A square root with a significant imaginary part on its diagonal (|imag| > 1e-3)
    raises ValueError; otherwise its real part is used."""
    mu1, mu2 = np.atleast_1d(np.asarray(mu1, np.float64)), np.atleast_1d(np.asarray(mu2, np.float64))
    sigma1, sigma2 = np.atleast_2d(np.asarray(sigma1, np.float64)), np.atleast_2d(np.asarray(sigma2, np.float64))
    if mu1.shape != mu2.shape:
        raise AssertionError("Training and test mean vectors have different lengths")
    if sigma1.shape != sigma2.shape:
        raise AssertionError("Training and test covariances have different dimensions")
    diff = mu1 - mu2
    root = linalg.sqrtm(sigma1 @ sigma2)
    if not np.isfinite(root).all():
        shift = np.eye(sigma1.shape[0]) * eps
        root = linalg.sqrtm((sigma1 + shift) @ (sigma2 + shift))
    if np.iscomplexobj(root):
        if not np.allclose(np.diagonal(root).imag, 0, atol=1e-3):
            raise ValueError(f"Imaginary component {np.max(np.abs(root.imag))}")
        root = root.real
    return float(diff @ diff + np.trace(sigma1) + np.trace(sigma2) - 2 * np.trace(root))


class _ImagePaths(torch.utils.data.Dataset):
    def __init__(self, files, transforms):
        self.files, self.transforms = files, transforms

    def __len__(self):
        return len(self.files)

    def __getitem__(self, i):
        from PIL import Image
        return self.transforms(Image.open(self.files[i]).convert("RGB"))


def _to_features(pred: torch.Tensor) -> np.ndarray:
    """[n, c, h, w] block output -> float64 [n, c]; blocks that are not 1x1 are averaged over space."""
    a = pred.detach().cpu().numpy().astype(np.float64)
    return a.mean(axis=(2, 3)) if a.shape[2:] != (1, 1) else a[:, :, 0, 0]


def get_activations(files, model, batch_size=50, dims=2048, device="cpu", num_workers=1, transforms=None):
    """Features [len(files), dims] of image files loaded with PIL as RGB, through `transforms` (default ToTensor)."""
    import torchvision.transforms as TF
    if batch_size > len(files):
        batch_size = len(files)
    loader = torch.utils.data.DataLoader(_ImagePaths(files, transforms or TF.ToTensor()), batch_size=batch_size,
                                         shuffle=False, drop_last=False, num_workers=num_workers)
    out = np.empty((len(files), dims))
    i = 0
    for batch in loader:
        f = _to_features(model(batch.to(device))[0])
        out[i:i + len(f)] = f
        i += len(f)
    return out


def calculate_activation_statistics(files, model, batch_size=50, dims=2048, device="cpu", num_workers=1,
                                    transforms=None):
    act = get_activations(files, model, batch_size, dims, device, num_workers, transforms=transforms)
    return np.mean(act, axis=0), np.cov(act, rowvar=False)


def compute_statistics_of_path(path, model, batch_size, dims, device, num_workers=1, transforms=None):
    """(mu, sigma) of an .npz holding `mu` / `sigma`, or of every image under a directory (sorted, any depth)."""
    path = str(path)
    if path.endswith(".npz"):
        with np.load(path) as f:
            return f["mu"][:], f["sigma"][:]
    root = pathlib.Path(path)
    files = sorted(f for ext in IMAGE_EXTENSIONS for f in root.glob(f"**/*.{ext}"))
    return calculate_activation_statistics(files, model, batch_size, dims, device, num_workers, transforms)


def _model(dims, device, model, weights):
    if model is not None:
        return model
    if weights is None:
        raise ValueError("pass `model` or `weights` (the local path of the pytorch-fid Inception weights file)")
    return InceptionV3.from_pretrained(weights, [InceptionV3.BLOCK_INDEX_BY_DIM[dims]]).to(device)


def calculate_fid_given_paths(paths, batch_size, device, dims, num_workers=1, model=None, weights=None,
                              transforms=None):
    """FID between two directories / .npz statistics files."""
    for p in paths:
        if not os.path.exists(p):
            raise RuntimeError(f"Invalid path: {p}")
    model = _model(dims, device, model, weights)
    m1, s1 = compute_statistics_of_path(paths[0], model, batch_size, dims, device, num_workers, transforms)
    m2, s2 = compute_statistics_of_path(paths[1], model, batch_size, dims, device, num_workers, transforms)
    return calculate_frechet_distance(m1, s1, m2, s2)


def save_fid_stats(paths, batch_size, device, dims, num_workers=1, model=None, weights=None, transforms=None):
    """Statistics of paths[0] written to the .npz paths[1] (mu, sigma)."""
    if not os.path.exists(paths[0]):
        raise RuntimeError(f"Invalid path: {paths[0]}")
    if os.path.exists(paths[1]):
        raise RuntimeError(f"Existing output file: {paths[1]}")
    model = _model(dims, device, model, weights)
    m, s = compute_statistics_of_path(paths[0], model, batch_size, dims, device, num_workers, transforms)
    np.savez_compressed(paths[1], mu=m, sigma=s)


class FIDStatistics:
    """Accumulates Inception features of device image batches in [0, 1]: the denoiser's decoded views
    (S, n_cam, H, W, 3) (pipeline output_type="pt", AutoencoderKL.decode_latents) or (N, 3, H, W).  Each batch is rounded
    to the 8-bit levels a saved PNG holds, then features are computed on the device and appended on the host."""

    def __init__(self, model: InceptionV3, dims: int = 2048):
        self.model, self.dims = model, dims
        self.block = InceptionV3.BLOCK_INDEX_BY_DIM[dims]
        if self.block not in model.output_blocks:
            raise ValueError(f"the model does not output block {self.block} ({dims} features)")
        self._feats = []

    def update(self, images: torch.Tensor) -> None:
        if images.dim() == 5:
            nhwc = images.reshape(-1, *images.shape[2:])
            outs = self.model.features(nhwc, nhwc=True, quantize=True)
        elif images.dim() == 4:
            outs = self.model.features(images, nhwc=False, quantize=True)
        else:
            raise ValueError(f"expected (S, n_cam, H, W, 3) or (N, 3, H, W) images, got {tuple(images.shape)}")
        self._feats.append(_to_features(outs[self.model.output_blocks.index(self.block)]))

    @property
    def count(self) -> int:
        return sum(len(f) for f in self._feats)

    def activations(self) -> np.ndarray:
        return np.concatenate(self._feats, 0) if self._feats else np.empty((0, self.dims))

    def statistics(self):
        act = self.activations()
        return np.mean(act, axis=0), np.cov(act, rowvar=False)

    def save(self, path) -> None:
        mu, sigma = self.statistics()
        np.savez_compressed(path, mu=mu, sigma=sigma)
