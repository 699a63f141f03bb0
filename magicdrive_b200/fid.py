"""Fréchet Inception Distance, host side (the reference's tools/fid_score.py:93-276, 341-358).

The Inception features come from `models.InceptionV3` on the device; statistics (np.mean, np.cov in float64) and the
Fréchet distance (scipy's sqrtm) are computed on the host, as the reference does.  `FIDStatistics` accumulates the
features of device image batches -- the denoiser's decoded views -- rounded to the 8-bit levels a saved PNG would hold,
so a generated set's FID needs no PNGs on disk.  `FIDProtocol` instead reproduces the reference's evaluation chain
(bicubic resize, zero pad, JPEG save and load, scoring resize and crop) on the device, byte for byte; only statistics taken
through it compare with the published FIDs.  Nothing here downloads weights: pass a model, or the path of the
pytorch-fid weights file.
"""
import copy
import os
import pathlib

import numpy as np
import torch
from scipy import linalg

from . import image_ops, jpeg_ops
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


def bicubic_table(in_size: int, out_size: int) -> np.ndarray:
    """int32 [out_size, taps + 2] coefficient rows of Pillow's 8-bit bicubic resample (Resample.c): [first input index,
    tap count, weights in 22-bit fixed point...].  The Keys cubic (a = -0.5) is evaluated in float64 at
    (x - centre + 0.5) / max(scale, 1), so downsampling widens the support (antialiasing); each row is normalised by its
    sum taken left to right and rounded half away from zero."""
    if in_size <= 0 or out_size <= 0:
        raise ValueError(f"bad resample sizes {in_size} -> {out_size}")
    scale = in_size / out_size
    fscale = max(scale, 1.0)
    support = 2.0 * fscale
    taps = int(np.ceil(support)) * 2 + 1
    center = (np.arange(out_size) + 0.5) * scale
    first = np.maximum(np.trunc(center - support + 0.5), 0).astype(np.int64)
    count = np.minimum(np.trunc(center + support + 0.5), in_size).astype(np.int64) - first
    x = np.abs((np.arange(taps)[None, :] + first[:, None] - center[:, None] + 0.5) * (1.0 / fscale))
    a = -0.5
    w = np.where(x < 1.0, ((a + 2.0) * x - (a + 3.0)) * x * x + 1, np.where(x < 2.0, (((x - 5) * x + 8) * x - 4) * a, 0.0))
    w = np.where(np.arange(taps)[None, :] < count[:, None], w, 0.0)
    total = np.zeros(out_size)
    for t in range(taps):  # left to right, as the C loop adds them
        total += w[:, t]
    w = np.where(total[:, None] != 0.0, w / np.where(total == 0.0, 1.0, total)[:, None], w)
    fixed = np.trunc(w * (1 << 22) + np.where(w < 0, -0.5, 0.5)).astype(np.int64)
    return np.concatenate([first[:, None], count[:, None], fixed], 1).astype(np.int32)


# (image_size (h, w), back_resize (h, w), back_pad (left, top, right, bottom), resize_ratio) of the reference's dataset
# configs: configs/dataset/Nuscenes.yaml, Nuscenes_map_cache_box_272x736.yaml and Nuscenes_400_map_cache_box_424x800.yaml
PROTOCOL_CONFIGS = {
    "224x400": ((224, 400), (896, 1600), (0, 4, 0, 0), 0.25),
    "272x736": ((272, 736), (544, 1472), (64, 356, 64, 0), 0.5),
    "424x800": ((424, 800), (848, 1600), (0, 52, 0, 0), 0.5),
}
CAMERA_SIZE = (900, 1600)  # nuScenes camera images (h, w); tools/fid_score.py:475


class FIDProtocol:
    """The reference's FID image chain on the device, equal byte for byte to its Pillow route.

    Generation side (perception/data_prepare/val_set_gen.py): the views rounded to uint8 as numpy_to_pil does, a bicubic
    resize to `back_resize`, a zero pad by `back_pad` (left, top, right, bottom) and, with `jpeg`, the JPEG save and load
    at Pillow's defaults (quality 75, 4:2:0) that the `.jpg` file name implies.  Scoring side (tools/fid_score.py, for
    generated and real images alike): a bicubic resize of the image to int(900 r) x int(1600 r), r = `resize_ratio`, and
    the top-centre crop to `image_size`.  `generated` and `real` return the uint8 (N, h, w, 3) images Inception scores;
    each keeps one CUDA graph per input shape (set `use_cuda_graph = False` to run eagerly)."""

    use_cuda_graph = True

    def __init__(self, image_size, back_resize, back_pad, resize_ratio, jpeg: bool = True, quality: int = 75):
        self.image_size = tuple(int(v) for v in image_size)
        self.back_resize = tuple(int(v) for v in back_resize)
        self.back_pad = tuple(int(v) for v in back_pad)
        self.resize_ratio, self.jpeg, self.quality = float(resize_ratio), bool(jpeg), int(quality)
        if len(self.image_size) != 2 or len(self.back_resize) != 2 or len(self.back_pad) != 4:
            raise ValueError("image_size and back_resize are (h, w); back_pad is (left, top, right, bottom)")
        if min(self.image_size + self.back_resize) <= 0 or min(self.back_pad) < 0:
            raise ValueError(f"sizes must be positive and pads non-negative: {self.image_size}, {self.back_resize}, "
                             f"{self.back_pad}")
        if not 1 <= self.quality <= 100:
            raise ValueError(f"quality must be in 1..100, got {quality}")
        left, top, right, bottom = self.back_pad
        self.canvas = (self.back_resize[0] + top + bottom, self.back_resize[1] + left + right)
        self.score_resize = (int(CAMERA_SIZE[0] * self.resize_ratio), int(CAMERA_SIZE[1] * self.resize_ratio))
        fh, fw = self.image_size
        rh, rw = self.score_resize
        if rh < fh or rw < fw or min(rh, rw) <= 0:
            raise ValueError(f"resize_ratio {resize_ratio} gives {rh}x{rw}, smaller than image_size {fh}x{fw}")
        self.crop = (rh - fh, int(max(0, rw - fw) / 2), fh, fw)  # top_center_crop
        self._tables, self._graphs = {}, {}

    @classmethod
    def for_config(cls, name: str, **kw) -> "FIDProtocol":
        """One of PROTOCOL_CONFIGS: "224x400", "272x736" or "424x800"."""
        if name not in PROTOCOL_CONFIGS:
            raise ValueError(f"unknown config {name!r}; known: {sorted(PROTOCOL_CONFIGS)}")
        return cls(*PROTOCOL_CONFIGS[name], **kw)

    def __repr__(self):
        return (f"FIDProtocol(image_size={self.image_size}, back_resize={self.back_resize}, back_pad={self.back_pad}, "
                f"resize_ratio={self.resize_ratio}, jpeg={self.jpeg}, quality={self.quality})")

    def _table(self, n_in, n_out, device):
        if n_in == n_out:
            return None
        key = (n_in, n_out, str(device))
        t = self._tables.get(key)
        if t is None:
            t = self._tables[key] = torch.from_numpy(bicubic_table(n_in, n_out)).to(device)
        return t

    def _resize(self, x, nhwc, size, **kw):
        h, w = (x.shape[1], x.shape[2]) if nhwc else (x.shape[2], x.shape[3])
        return image_ops.resample_u8(x, size, self._table(w, size[1], x.device), self._table(h, size[0], x.device), nhwc=nhwc,
                               **kw)

    def _generated(self, x, nhwc):
        left, top, _, _ = self.back_pad
        canvas = self._resize(x, nhwc, self.back_resize, canvas=self.canvas, offset=(top, left))
        if self.jpeg:
            image_ops.jpeg_roundtrip_u8(canvas, self.quality, out=canvas)
        return self._real(canvas)

    def _real(self, u8):
        return self._resize(u8, True, self.score_resize, crop=self.crop)

    def _run(self, kind, fn, x, nhwc):
        if not self.use_cuda_graph:
            return fn(x, nhwc) if kind == "generated" else fn(x)
        key = (kind, tuple(x.shape), x.dtype, nhwc, x.device)
        g = self._graphs.get(key)
        if g is None:
            xin = x.clone()
            fn(xin, nhwc) if kind == "generated" else fn(xin)  # eager once: uploads the coefficient tables
            torch.cuda.synchronize(x.device)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                out = fn(xin, nhwc) if kind == "generated" else fn(xin)
            g = self._graphs[key] = (graph, xin, out)
        graph, xin, out = g
        xin.copy_(x)
        graph.replay()
        return out.clone()

    @staticmethod
    def _views(images):
        """(views [N, ...] contiguous, uint8 or fp32, nhwc) of generated()'s accepted inputs."""
        if images.dim() == 5 and images.shape[-1] == 3:
            x, nhwc = images.reshape(-1, *images.shape[2:]), True
        elif images.dim() == 4 and images.dtype == torch.uint8 and images.shape[-1] == 3:
            x, nhwc = images, True
        elif images.dim() == 4 and images.shape[1] == 3:
            x, nhwc = images, False
        else:
            raise ValueError(f"expected (S, n_cam, H, W, 3) or (N, 3, H, W) images, got {tuple(images.shape)}")
        if x.dtype != torch.uint8:
            x = x.float()
        return x.contiguous(), nhwc

    @torch.no_grad()
    def generated(self, images: torch.Tensor) -> torch.Tensor:
        """Device views in [0, 1], (S, n_cam, H, W, 3) or (N, 3, H, W), fp32 or bf16 (or uint8 (N, H, W, 3) already
        rounded) -> uint8 (N, h, w, 3): what the reference scores for them."""
        x, nhwc = self._views(images)
        return self._run("generated", self._generated, x, nhwc)

    @torch.no_grad()
    def encode_generated(self, images: torch.Tensor) -> list:
        """The inputs of generated() -> the bytes of the `.jpg` files copy_save_image writes for them (val_set_gen.py:
        numpy_to_pil, Resize(back_resize, BICUBIC), Pad(back_pad), PIL save at `quality`), one per view in order.  The
        resize, pad and encoder run on the device; only the files' bytes come back."""
        x, nhwc = self._views(images)
        left, top, _, _ = self.back_pad
        canvas = self._resize(x, nhwc, self.back_resize, canvas=self.canvas, offset=(top, left))
        return jpeg_ops.encode_jpeg(canvas, self.quality)

    @torch.no_grad()
    def real(self, u8_images: torch.Tensor, device=None) -> torch.Tensor:
        """Decoded camera images, uint8 (N, 900, 1600, 3) -> uint8 (N, h, w, 3) on `device` (default: the images' own
        CUDA device, or the current one for host images): the scoring resize and crop.  Decode the JPEG files with PIL
        (Image.open(f).convert("RGB")), as the reference does."""
        if u8_images.dtype != torch.uint8 or u8_images.dim() != 4 or u8_images.shape[-1] != 3:
            raise ValueError(f"expected uint8 (N, H, W, 3), got {u8_images.dtype} {tuple(u8_images.shape)}")
        if device is None:
            device = u8_images.device if u8_images.is_cuda else torch.device("cuda")
        x = u8_images.to(device).contiguous()
        return self._run("real", lambda v: self._real(v), x, True)


@torch.no_grad()
def save_generated_views(images: torch.Tensor, templates, img_gen_dir, view_order, protocol: FIDProtocol = None) -> list:
    """The reference's copy_save_image (perception/data_prepare/val_set_gen.py:29-43) for views on the device.

    images: (B, T, n_cam, H, W, 3) in [0, 1] (fp32 or bf16) or uint8, generation t of batch item b; templates: B label
    entries as the reference builds them ({"filename": n_cam camera file names, "token": ...}); view_order: the n_cam
    camera names.  Writes <img_gen_dir>/<view>/<stem>_gen_<t>.jpg for every view, in the reference's order, and returns
    its list: one deep copy of the template per (b, t).  protocol: the FIDProtocol whose back_resize, back_pad and
    quality make post_trans; None is `fid.raw_output: true`, the views saved at their own size at Pillow's default
    quality.  The directories <img_gen_dir>/<view> must exist, as the reference creates them before its loop."""
    if images.dim() != 6 or images.shape[-1] != 3:
        raise ValueError(f"expected (B, T, n_cam, H, W, 3) images, got {tuple(images.shape)}")
    B, T, n_cam = images.shape[:3]
    if len(templates) != B or len(view_order) != n_cam:
        raise ValueError(f"{len(templates)} templates and {len(view_order)} views for images {tuple(images.shape)}")
    for template in templates:
        for name in template["filename"]:
            if os.path.splitext(name)[1].lower() not in (".jpg", ".jpeg"):
                raise ValueError(f"{name}: the views are saved as JPEG files, which need a .jpg or .jpeg name")
    views = images.reshape(B * T, n_cam, *images.shape[3:])
    if protocol is not None:
        files = protocol.encode_generated(views)
    else:
        x = views.reshape(-1, *images.shape[3:])
        if x.dtype != torch.uint8:  # numpy_to_pil's rounding; the resample with no size change is a copy
            x = image_ops.resample_u8(x.float().contiguous(), x.shape[1:3], None, None)
        files = jpeg_ops.encode_jpeg(x.contiguous())
    tmp_all, k = [], 0
    for template in templates:
        for gen_id in range(T):
            for idx, view in enumerate(view_order):
                stem, ext = os.path.splitext(os.path.basename(template["filename"][idx]))
                with open(os.path.join(img_gen_dir, view, f"{stem}_gen_{gen_id}{ext}"), "wb") as f:
                    f.write(files[k])
                k += 1
            tmp_all.append(copy.deepcopy(template))
    return tmp_all


def _decode_rgb(path) -> np.ndarray:
    from PIL import Image
    with Image.open(path) as im:
        return np.asarray(im.convert("RGB"))


def protocol_statistics_of_files(files, model: InceptionV3, protocol: FIDProtocol, batch_size: int = 50,
                                 dims: int = 2048):
    """(mu, sigma) of real camera images (any files PIL reads, typically the nuScenes JPEGs in the caller's order):
    decoded on the host by PIL, then `protocol.real` and Inception on the device.  Consecutive files of one size are
    batched together."""
    stats = FIDStatistics(model, dims, protocol=protocol)
    batch = []

    def flush():
        if batch:
            stats.update_real(torch.from_numpy(np.stack(batch)))
            batch.clear()
    for f in files:
        img = _decode_rgb(f)
        if batch and (img.shape != batch[0].shape or len(batch) == batch_size):
            flush()
        batch.append(img)
    flush()
    return stats.statistics()


def protocol_statistics_of_path(path, model: InceptionV3, protocol: FIDProtocol, batch_size: int = 50, dims: int = 2048):
    """protocol_statistics_of_files over every image under a directory (sorted, any depth), or the mu / sigma of a .npz."""
    path = str(path)
    if path.endswith(".npz"):
        with np.load(path) as f:
            return f["mu"][:], f["sigma"][:]
    root = pathlib.Path(path)
    files = sorted(f for ext in IMAGE_EXTENSIONS for f in root.glob(f"**/*.{ext}"))
    return protocol_statistics_of_files(files, model, protocol, batch_size, dims)


class FIDStatistics:
    """Accumulates Inception features of device image batches in [0, 1]: the denoiser's decoded views
    (S, n_cam, H, W, 3) (pipeline output_type="pt", AutoencoderKL.decode_latents) or (N, 3, H, W).

    Without a protocol, each batch is rounded to the 8-bit levels a saved PNG holds and scored as it is.  With
    `protocol` (a FIDProtocol), each batch first goes through the reference's generation and scoring chain
    (`protocol.generated`), so the statistics are those its Pillow route would give and FIDs compare with the published
    ones; `update_real` then scores decoded real camera images through `protocol.real`.  Features are computed on the
    device and appended on the host."""

    def __init__(self, model: InceptionV3, dims: int = 2048, protocol: "FIDProtocol" = None):
        self.model, self.dims, self.protocol = model, dims, protocol
        self.block = InceptionV3.BLOCK_INDEX_BY_DIM[dims]
        if self.block not in model.output_blocks:
            raise ValueError(f"the model does not output block {self.block} ({dims} features)")
        if protocol is not None and not isinstance(protocol, FIDProtocol):
            raise TypeError(f"protocol must be a FIDProtocol, got {type(protocol).__name__}")
        self._feats = []

    def _update_u8(self, u8: torch.Tensor) -> None:
        # k / 255 in fp32 rounds back to k in mdb_fid_input's 8-bit rounding: the levels reach Inception unchanged
        outs = self.model.features(u8.float().div_(255.0), nhwc=True, quantize=True)
        self._feats.append(_to_features(outs[self.model.output_blocks.index(self.block)]))

    def update_real(self, u8_images: torch.Tensor) -> None:
        """Decoded real camera images, uint8 (N, 900, 1600, 3), through `protocol.real` on the model's device."""
        if self.protocol is None:
            raise ValueError("update_real needs FIDStatistics(..., protocol=FIDProtocol(...))")
        self._update_u8(self.protocol.real(u8_images, device=self.model.device))

    def update(self, images: torch.Tensor) -> None:
        if self.protocol is not None:
            self._update_u8(self.protocol.generated(images))
            return
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
