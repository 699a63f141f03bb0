"""3D-box overlays on the sm_90a path: show_box_on_views against the reference's own images
(tests/golden/box_overlay.pt) and against the restatement (oracle/box_overlay.py) on seeded scenes, byte for byte.

An endpoint may differ from the reference's only where the reference's float64 coordinate lies within 1e-3 px of an
integer (a last-bit difference in a corner can then change the truncation).  Every such endpoint is named; the pixels are
then checked against the restatement drawn from the kernel's endpoints."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from magicdrive_b200 import box_overlay  # noqa: E402
from oracle import box_overlay as O  # noqa: E402
from oracle.make_golden_box_overlay import backgrounds, load  # noqa: E402
from tests.common import GOLDEN  # noqa: E402
from tests.test_box_overlay_cpu import expected  # noqa: E402

NEAR_INTEGER = 1e-3


def _endpoint_differences(proj, examples, classes):
    """Compare the kernel's projection with the oracle's per (scene, view): counts, order (labels) and endpoints.
    -> the endpoints that differ, each (scene, view, box, corner, axis, reference coordinate), all near an integer."""
    ends, cols, counts = (proj[k].cpu().numpy() for k in ("endpoints", "colors", "counts"))
    assert not proj["status"].any()
    diffs = []
    for s, ex in enumerate(examples):
        trans = O.view_transforms(ex)
        for v in range(trans.shape[0]):
            want, labels, xy = O.project(np.asarray(ex["gt_bboxes_3d"], np.float32), np.asarray(ex["gt_labels_3d"]), trans[v])
            n = len(labels)
            assert counts[s, v] == n, (s, v)
            assert np.array_equal(cols[s, v, :n], labels), (s, v)
            for idx in np.argwhere(ends[s, v, :n] != want):
                c = xy[tuple(idx)]
                assert abs(c - np.round(c)) < NEAR_INTEGER, f"endpoint {(s, v, *idx)}: {ends[s, v][tuple(idx)]} vs {c!r}"
                diffs.append((s, v, *idx.tolist(), float(c)))
    return diffs


def _oracle_images(images_u8, examples, proj, classes, transparent_bg):
    """The restatement's drawing from the kernel's own endpoints and order."""
    ends, cols, counts = (proj[k].cpu().numpy() for k in ("endpoints", "colors", "counts"))
    out = []
    for s in range(len(examples)):
        views = []
        for v in range(images_u8.shape[1]):
            img = np.zeros_like(images_u8[s, v]) if transparent_bg else images_u8[s, v].copy()
            O.draw_boxes(img, ends[s, v, :counts[s, v]], cols[s, v, :counts[s, v]], classes)
            if transparent_bg:
                img = np.concatenate([img, (np.any(img > 0, axis=2) * 255).astype(np.uint8)[..., None]], axis=2)
            views.append(img)
        out.append(np.stack(views))
    return np.stack(out)


def _first_diff(a, b):
    idx = np.argwhere(a != b)
    return f"{len(idx)} bytes differ, first at {tuple(idx[0])}: {a[tuple(idx[0])]} vs {b[tuple(idx[0])]}" if len(idx) else ""


@pytest.mark.parametrize("transparent_bg", [False, True])
def test_reference_fixture_byte_for_byte(cuda_lib, transparent_bg):
    fx = load(os.path.join(GOLDEN, "box_overlay.pt"))
    cases, classes = fx["cases"], fx["classes"]
    bg = backgrounds(len(cases), fx["seed"])
    got = box_overlay.show_box_on_views(torch.from_numpy(bg).cuda(), cases, classes,
                                        transparent_bg=transparent_bg).cpu().numpy()
    diffs = _endpoint_differences(box_overlay.project_boxes(cases, 6, "cuda", classes), cases, classes)
    print("endpoints within 1e-3 px of an integer that differ:", diffs)
    assert len(diffs) == 0, diffs  # expected: none
    want = np.stack([expected(c, b, transparent_bg) for c, b in zip(cases, bg)])
    assert np.array_equal(got, want), _first_diff(got, want)


def _scene(rng, n, box_dim=9, aug=True, far=False):
    """n seeded boxes around a 6-camera rig: some behind the cameras, some straddling them, some far off-axis."""
    b = np.zeros((n, box_dim), np.float32)
    b[:, :2] = rng.uniform(-60, 60, (n, 2))
    b[:, 2] = rng.uniform(-3, 2, n)
    b[:, 3:6] = rng.uniform(0.3, 12, (n, 3))
    b[:, 6] = rng.uniform(-np.pi, np.pi, n)
    if box_dim == 9:
        b[:, 7:] = rng.normal(size=(n, 2))
    if far:  # small boxes around camera 0's image plane (depth = lidar x): corners at depths near 0 project far out
        b[: n // 4, 0] = rng.uniform(-1, 3, n // 4)
        b[: n // 4, 1] = rng.uniform(-3, 3, n // 4)
        b[: n // 4, 3:6] = rng.uniform(0.2, 1, (n // 4, 3))
    ex = {"gt_bboxes_3d": torch.from_numpy(b), "gt_labels_3d": torch.from_numpy(rng.integers(0, 10, n))}
    K, l2c = np.tile(np.eye(4, dtype=np.float32), (6, 1, 1)), np.zeros((6, 4, 4), np.float32)
    for v in range(6):
        yaw = v * np.pi / 3
        R = np.array([[-np.sin(yaw), np.cos(yaw), 0], [0, 0, -1], [np.cos(yaw), np.sin(yaw), 0]])  # lidar -> camera
        l2c[v, :3, :3], l2c[v, :3, 3], l2c[v, 3, 3] = R, rng.normal(0, 0.5, 3), 1
        K[v, :3, :3] = [[rng.uniform(200, 1300), 0, rng.uniform(100, 800)], [0, rng.uniform(200, 1300), rng.uniform(100, 450)],
                        [0, 0, 1]]
    ex["camera_intrinsics"], ex["lidar2camera"] = torch.from_numpy(K), torch.from_numpy(l2c)
    if aug:
        A = np.tile(np.eye(4, dtype=np.float32), (6, 1, 1))
        A[:, :2, :2] *= np.float32(rng.uniform(0.2, 0.6))
        A[:, :2, 3] = rng.uniform(-50, 0, (6, 2))
        ex["img_aug_matrix"] = torch.from_numpy(A)
    return ex


CASES = [  # (name, box counts per scene, box_dim, img_aug present, size, fp32 input)
    ("224x400", [0, 1, 7, 40], 9, True, (224, 400), False),
    ("272x736", [120, 3], 7, True, (272, 736), False),
    ("424x800_noaug", [300], 9, False, (424, 800), False),
    ("odd_sizes", [25, 60], 9, True, (37, 53), False),
    ("one_row", [30], 7, False, (1, 97), False),
    ("one_col", [30], 9, True, (61, 1), False),
    ("fp32_decode", [50, 10], 9, True, (224, 400), True),
]


@pytest.mark.parametrize("name,counts,box_dim,aug,size,fp32", CASES, ids=[c[0] for c in CASES])
@pytest.mark.parametrize("transparent_bg", [False, True])
def test_seeded_scenes_equal_oracle(cuda_lib, name, counts, box_dim, aug, size, fp32, transparent_bg):
    rng = np.random.default_rng(sum(map(ord, name)))
    examples = [_scene(rng, n, box_dim, aug, far=i % 2 == 1) for i, n in enumerate(counts)]
    S, (H, W) = len(examples), size
    if fp32:  # views as decode_latents returns them: fp32 in [0, 1], rounded as numpy_to_pil does
        x = torch.rand((S, 6, H, W, 3), generator=torch.Generator().manual_seed(5))
        u8 = (x.numpy() * 255).round().astype(np.uint8)
    else:
        u8 = rng.integers(0, 256, (S, 6, H, W, 3), dtype=np.uint8)
        x = torch.from_numpy(u8)
    got = box_overlay.show_box_on_views(x.cuda(), examples, transparent_bg=transparent_bg).cpu().numpy()
    proj = box_overlay.project_boxes(examples, 6, "cuda")
    diffs = _endpoint_differences(proj, examples, O.NUSCENES_OBJECT_CLASSES)
    print(name, "boxes drawn per view", proj["counts"].tolist(), "near-integer endpoint differences", diffs)
    if not diffs:
        want = np.stack([O.show_box_on_views(u8[s], examples[s], transparent_bg=transparent_bg) for s in range(S)])
        assert np.array_equal(got, want), _first_diff(got, want)
    want = _oracle_images(u8, examples, proj, O.NUSCENES_OBJECT_CLASSES, transparent_bg)
    assert np.array_equal(got, want), _first_diff(got, want)


def test_in_place_and_repeatable(cuda_lib):
    rng = np.random.default_rng(11)
    examples = [_scene(rng, 80), _scene(rng, 20)]
    x = torch.from_numpy(rng.integers(0, 256, (2, 6, 224, 400, 3), dtype=np.uint8)).cuda()
    a = box_overlay.show_box_on_views(x, examples)
    b = box_overlay.show_box_on_views(x, examples)
    assert torch.equal(a, b)
    y = x.clone()
    assert box_overlay.show_box_on_views(y, examples, out=y) is y
    assert torch.equal(y, a)


def test_endpoint_outside_int32_raises_and_leaves_out(cuda_lib):
    ex = _scene(np.random.default_rng(2), 5, aug=False)
    ex["lidar2image"] = torch.bmm(ex["camera_intrinsics"], ex["lidar2camera"])
    ex["lidar2image"][0, 0, 3] = 3e14  # x / z beyond int32 for every box in front of camera 0
    b = ex["gt_bboxes_3d"]
    b[:, :3] = torch.tensor([10.0, 0.0, 0.0])  # in front of camera 0 (+x in this rig's lidar frame)
    ends, labels, xy = O.project(b.numpy(), ex["gt_labels_3d"].numpy(), O.view_transforms(ex)[0])
    assert len(labels) and np.abs(xy).max() > 2 ** 31
    x = torch.zeros((1, 6, 32, 48, 3), dtype=torch.uint8, device="cuda")
    out = torch.full_like(x, 9)
    with pytest.raises(ValueError, match="int32"):
        box_overlay.show_box_on_views(x, [ex], out=out)
    assert bool((out == 9).all())
    with pytest.raises(ValueError):
        O.show_box_on_views(x[0].cpu().numpy(), ex)


def test_rejected_arguments_leave_out_untouched(cuda_lib):
    ex = _scene(np.random.default_rng(4), 6)
    x = torch.zeros((1, 6, 32, 48, 3), dtype=torch.uint8, device="cuda")
    out = torch.full_like(x, 9)
    bad = dict(ex, gt_labels_3d=torch.full((6,), 12))
    with pytest.raises(ValueError):
        box_overlay.show_box_on_views(x, [bad], out=out)
    with pytest.raises(KeyError):
        box_overlay.show_box_on_views(x, [ex], ["van"] * 10, out=out)
    with pytest.raises(TypeError):
        box_overlay.show_box_on_views(x.half(), [ex], out=out)
    with pytest.raises(ValueError):
        box_overlay.show_box_on_views(x, [ex], out=out, transparent_bg=True)
    torch.cuda.synchronize()
    assert bool((out == 9).all())
