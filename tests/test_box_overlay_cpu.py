"""3D-box overlays on the CPU: the restatement of OpenCV's anti-aliased line (oracle/box_overlay.py) against cv2.line
byte for byte, the whole restated overlay against the reference's own images (tests/golden/box_overlay.pt), and the
argument checks of box_overlay.show_box_on_views, which all come before any launch."""
import os

import numpy as np
import pytest
import torch

from magicdrive_b200 import _lib, box_overlay
from oracle import box_overlay as O
from oracle.make_golden_box_overlay import backgrounds, load
from tests.common import GOLDEN

PALETTE = list(O.OBJECT_PALETTE.values())


def _endpoints(rng, kind, h, w):
    """Two endpoints of one of the line families the test covers."""
    if kind == "inside":
        return rng.integers(0, [w, h], 2), rng.integers(0, [w, h], 2)
    if kind == "near":  # a few pixels around the image, so edges are clipped on every side
        return rng.integers(-4, [w + 4, h + 4], 2), rng.integers(-4, [w + 4, h + 4], 2)
    if kind == "far":
        return rng.integers(-10 ** 6, 10 ** 6, 2), rng.integers(-10 ** 6, 10 ** 6, 2)
    if kind == "one_far":
        return rng.integers(0, [w, h], 2), rng.integers(-10 ** 6, 10 ** 6, 2)
    p = rng.integers(-3, [w + 3, h + 3], 2)
    d = int(rng.integers(-3 * max(h, w), 3 * max(h, w) + 1))
    q = {"horizontal": p + [d, 0], "vertical": p + [0, d], "diagonal": p + [d, d], "antidiagonal": p + [d, -d],
         "point": p.copy()}[kind]
    return p, q


KINDS = ("inside", "near", "far", "one_far", "horizontal", "vertical", "diagonal", "antidiagonal", "point")
SIZES = ((1, 1), (1, 9), (9, 1), (1, 37), (37, 1), (7, 13), (16, 16), (31, 57), (224, 400))


@pytest.mark.parametrize("h,w", SIZES, ids=lambda v: str(v))
def test_line_aa_equals_cv2(h, w):
    """2,700 seeded lines per size (24,300 in all): every family on constant and random backgrounds, palette and random
    colours, 30 overlapping lines drawn in sequence on one image."""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(h * 1000 + w)
    for trial in range(90):
        if trial % 2:
            img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        else:
            img = np.full((h, w, 3), rng.integers(0, 256, 3), np.uint8)
        want = img.copy()
        for n in range(30):
            p0, p1 = _endpoints(rng, KINDS[(trial + n) % len(KINDS)], h, w)
            col = PALETTE[n % len(PALETTE)] if n % 3 else tuple(int(c) for c in rng.integers(0, 256, 3))
            cv2.line(want, p0, p1, col, 1, cv2.LINE_AA)
            O.line_aa(img, p0, p1, col)
        assert np.array_equal(img, want), (h, w, trial)


def test_line_aa_int32_extremes():
    """Endpoints at the ends of the int32 range, which cv2 still takes."""
    cv2 = pytest.importorskip("cv2")
    lim = 2 ** 31 - 1
    img = np.zeros((224, 400, 3), np.uint8)
    want = img.copy()
    for p0, p1 in [((-lim - 1, 5), (lim, 100)), ((3, -lim - 1), (399, lim)), ((-lim - 1, -lim - 1), (lim, lim)),
                   ((100, 100), (lim, 101)), ((-7000000, 40), (7000000, 41))]:
        cv2.line(want, p0, p1, (255, 158, 0), 1, cv2.LINE_AA)
        O.line_aa(img, p0, p1, (255, 158, 0))
    assert np.array_equal(img, want)


def _fixture():
    return load(os.path.join(GOLDEN, "box_overlay.pt"))


def expected(case, bg, transparent_bg):
    """A fixture case's full reference images from its touched pixels."""
    at = tuple(case["at"].T)
    if transparent_bg:
        out = np.zeros(bg.shape[:3] + (4,), np.uint8)
        out[at] = case["layer"]
    else:
        out = bg.copy()
        out[at] = case["drawn"]
    return out


@pytest.mark.parametrize("transparent_bg", [False, True])
def test_oracle_equals_reference_fixture(transparent_bg):
    fx = _fixture()
    bgs = backgrounds(len(fx["cases"]), fx["seed"])
    for case, bg in zip(fx["cases"], bgs):
        got = O.show_box_on_views(bg, case, fx["classes"], transparent_bg=transparent_bg)
        assert np.array_equal(got, expected(case, bg, transparent_bg)), case["name"]


def test_oracle_projection_order_and_visibility():
    """Boxes behind the camera or straddling it are not drawn; the rest come far to near, ties in box order."""
    T = np.eye(4, dtype=np.float32)  # camera frame = lidar frame: depth is z
    boxes = np.array([[0, 0, 10, 1, 1, 1, 0], [0, 0, 30, 1, 1, 1, 0], [0, 0, -10, 1, 1, 1, 0], [0, 0, 0.2, 1, 1, 1, 0],
                      [5, 0, 30, 1, 1, 1, 0]], np.float32)
    ends, labels, _ = O.project(boxes, np.arange(5), T)
    assert labels.tolist() == [1, 4, 0]
    assert ends.shape == (3, 8, 2)


# ------------------------------------------------------------------------------------------------ argument checks
def _example(n=3, box_dim=9, seed=0):
    rng = np.random.default_rng(seed)
    b = np.concatenate([rng.uniform(-20, 20, (n, 3)), rng.uniform(1, 4, (n, 3)), rng.uniform(-3, 3, (n, 1)),
                        np.zeros((n, box_dim - 7))], 1).astype(np.float32)
    K = np.tile(np.eye(4, dtype=np.float32), (6, 1, 1))
    return {"gt_bboxes_3d": torch.from_numpy(b), "gt_labels_3d": torch.arange(n) % 10, "camera_intrinsics": K,
            "lidar2camera": K.copy(), "img_aug_matrix": K.copy()}


def test_argument_checks():
    img = torch.zeros((1, 6, 8, 8, 3), dtype=torch.uint8)
    out = torch.full((1, 6, 8, 8, 3), 7, dtype=torch.uint8)
    ex = [_example()]
    show = box_overlay.show_box_on_views
    with pytest.raises(TypeError):
        show(img.numpy(), ex)
    with pytest.raises(TypeError):
        show(img.to(torch.float16), ex)
    with pytest.raises(ValueError):
        show(img[0], ex)
    with pytest.raises(ValueError):
        show(torch.zeros((1, 6, 8, 8, 4), dtype=torch.uint8), ex)
    with pytest.raises(ValueError):
        show(img, ex + ex)
    with pytest.raises(TypeError):
        show(img, ex, out=out.float())
    with pytest.raises(ValueError):
        show(img, ex, out=out, transparent_bg=True)  # an RGBA layer needs a 4-channel out
    bad = _example()
    bad["gt_labels_3d"] = torch.tensor([0, 1, 10])
    with pytest.raises(ValueError):
        show(img, [bad], out=out)
    bad["gt_labels_3d"] = torch.tensor([0, -1, 2])
    with pytest.raises(ValueError):
        show(img, [bad], out=out)
    with pytest.raises(KeyError):
        show(img, ex, ("car", "lorry", "bus"), out=out)
    bad = _example()
    bad["gt_bboxes_3d"] = bad["gt_bboxes_3d"][:, :6]
    with pytest.raises(ValueError):
        show(img, [bad], out=out)
    bad = _example()
    bad["img_aug_matrix"] = bad["img_aug_matrix"][:5]
    with pytest.raises(ValueError):
        show(img, [bad], out=out)
    with pytest.raises(_lib.MdbError, match="CUDA"):  # valid arguments on the CPU: no fallback
        show(img, ex, out=out)
    assert bool((out == 7).all())


def test_view_transforms_follow_the_reference():
    """img_aug @ lidar2image in numpy float32; lidar2image = bmm(K, lidar2camera) when absent; no aug when absent."""
    ex = _example()
    rng = np.random.default_rng(3)
    for k in ("camera_intrinsics", "lidar2camera", "img_aug_matrix"):
        ex[k] = rng.normal(size=(6, 4, 4)).astype(np.float32)
    l2i = torch.bmm(torch.from_numpy(ex["camera_intrinsics"]), torch.from_numpy(ex["lidar2camera"])).numpy()
    want = np.stack([ex["img_aug_matrix"][v] @ l2i[v] for v in range(6)])
    assert np.array_equal(box_overlay.view_transforms(ex, 6), want)
    assert np.array_equal(O.view_transforms(ex), want)
    ex["lidar2image"], ex["img_aug_matrix"] = l2i * 2, None
    assert np.array_equal(box_overlay.view_transforms(ex, 6), l2i * 2)
