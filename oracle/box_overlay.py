"""Restatement of the 3D-box overlay kernels (magicdrive_b200/csrc/capi_box_overlay.cu) without OpenCV.

The reference draws each sample's 3D boxes on its camera views (demo/helper.py:197-307, `visualize_camera`,
`show_box_on_views`, `draw_box_on_imgs`): box corners in float32 torch, a float64 projection, and `cv2.line(..., 1,
cv2.LINE_AA)` for each of a box's 12 edges.  This module states each step in plain arithmetic so that
`tests/test_box_overlay_cpu.py` can hold it to cv2 and to the reference's own images byte for byte, and the GPU tests can
hold the kernels to it.

* `corners`: the gravity-centre shift (z - dz / 2) and mmdet3d's 8 corners, computed with the same torch operations as
  the reference, so that the float32 roundings are the reference's.
* `project`: homogeneous corners in float64 times transform.T; a box is kept when all 8 corners have z > 0; kept boxes
  are ordered far to near by their smallest z (a stable sort: ties keep box order); z is clipped to [1e-5, 1e5], x and y
  divided by it and truncated toward zero.
* `line_aa`: OpenCV's anti-aliased 1-pixel line on an 8-bit 3-channel image: 16.16 fixed-point endpoints, clipping to
  the image in int64 / double, a DDA along the major axis touching 3 pixels per step, end-point corrections from the
  endpoints' sub-pixel fractions, a 64-entry filter table, and each channel blended into the existing value twice with
  the same weight.
"""
import numpy as np
import torch

NUSCENES_OBJECT_CLASSES = ("car", "truck", "construction_vehicle", "bus", "trailer", "barrier", "motorcycle", "bicycle",
                           "pedestrian", "traffic_cone")
# demo/helper.py:25-36 (mmdet3d's); drawn as RGB on the RGB image (the two BGR swaps of the reference cancel out)
OBJECT_PALETTE = {
    "car": (255, 158, 0), "truck": (255, 99, 71), "construction_vehicle": (233, 150, 70), "bus": (255, 69, 0),
    "trailer": (255, 140, 0), "barrier": (112, 128, 144), "motorcycle": (255, 61, 99), "bicycle": (220, 20, 60),
    "pedestrian": (0, 0, 230), "traffic_cone": (47, 79, 79),
}
EDGES = ((0, 1), (0, 3), (0, 4), (1, 2), (1, 5), (3, 2), (3, 7), (4, 5), (4, 7), (2, 6), (5, 6), (6, 7))

XY_SHIFT = 16
XY_ONE = 1 << XY_SHIFT
SLOPE_CORR = (181, 181, 181, 182, 182, 183, 184, 185, 187, 188, 190, 192, 194, 196, 198, 201,
              203, 206, 209, 211, 214, 218, 221, 224, 227, 231, 235, 238, 242, 246, 250, 254)
FILTER = np.array([
    168, 177, 185, 194, 202, 210, 218, 224, 231, 236, 241, 246, 249, 252, 254, 254,
    254, 254, 252, 249, 246, 241, 236, 231, 224, 218, 210, 202, 194, 185, 177, 168,
    158, 149, 140, 131, 122, 114, 105, 97, 89, 82, 75, 68, 62, 56, 50, 45,
    40, 36, 32, 28, 25, 22, 19, 16, 14, 12, 11, 9, 8, 7, 5, 5], np.int64)


def _tdiv(a, b):
    """C integer division (truncation toward zero)."""
    q = abs(a) // abs(b)
    return q if (a < 0) == (b < 0) else -q


def clip_line(w, h, x1, y1, x2, y2):
    """cv::clipLine on a w x h rectangle (int64 coordinates, double intersections) -> (inside, x1, y1, x2, y2)."""
    right, bottom = w - 1, h - 1
    c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8
    c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8
    if (c1 & c2) == 0 and (c1 | c2) != 0:
        if c1 & 12:
            a = 0 if c1 < 8 else bottom
            x1 += int(float(a - y1) * float(x2 - x1) / float(y2 - y1))
            y1 = a
            c1 = (x1 < 0) + (x1 > right) * 2
        if c2 & 12:
            a = 0 if c2 < 8 else bottom
            x2 += int(float(a - y2) * float(x2 - x1) / float(y2 - y1))
            y2 = a
            c2 = (x2 < 0) + (x2 > right) * 2
        if (c1 & c2) == 0 and (c1 | c2) != 0:
            if c1:
                a = 0 if c1 == 1 else right
                y1 += int(float(a - x1) * float(y2 - y1) / float(x2 - x1))
                x1 = a
                c1 = 0
            if c2:
                a = 0 if c2 == 1 else right
                y2 += int(float(a - x2) * float(y2 - y1) / float(x2 - x1))
                x2 = a
                c2 = 0
    return (c1 | c2) == 0, x1, y1, x2, y2


def line_aa(img, p0, p1, color):
    """cv2.line(img, p0, p1, color, 1, cv2.LINE_AA) in place on uint8 [h, w, 3]; p0, p1 integer (x, y)."""
    h, w = img.shape[:2]
    ok, x1, y1, x2, y2 = clip_line(w << XY_SHIFT, h << XY_SHIFT, int(p0[0]) << XY_SHIFT, int(p0[1]) << XY_SHIFT,
                                   int(p1[0]) << XY_SHIFT, int(p1[1]) << XY_SHIFT)
    if not ok:
        return
    dx, dy = x2 - x1, y2 - y1
    ax, ay = abs(dx), abs(dy)
    x_major = ax > ay
    if x_major:  # walk along x from the left end
        if dx < 0:
            dy = -dy
            x1, x2, y1, y2 = x2, x1, y2, y1
        step = _tdiv(dy << XY_SHIFT, ax | 1)
        x2 += XY_ONE
        ecount = (x2 >> XY_SHIFT) - (x1 >> XY_SHIFT)
        frac = -(x1 & (XY_ONE - 1))
        minor = y1 + ((step * frac) >> XY_SHIFT) + (XY_ONE >> 1)
        i, j = (x1 >> (XY_SHIFT - 7)) & 0x78, (x2 >> (XY_SHIFT - 7)) & 0x78
        major0 = x1 >> XY_SHIFT
    else:  # walk along y from the top end
        if dy < 0:
            dx = -dx
            x1, x2, y1, y2 = x2, x1, y2, y1
        step = _tdiv(dx << XY_SHIFT, ay | 1)
        y2 += XY_ONE
        ecount = (y2 >> XY_SHIFT) - (y1 >> XY_SHIFT)
        frac = -(y1 & (XY_ONE - 1))
        minor = x1 + ((step * frac) >> XY_SHIFT) + (XY_ONE >> 1)
        i, j = (y1 >> (XY_SHIFT - 7)) & 0x78, (y2 >> (XY_SHIFT - 7)) & 0x78
        major0 = y1 >> XY_SHIFT
    slope = ((step >> (XY_SHIFT - 5)) & 0x3F) ^ (0x3F if step < 0 else 0)
    slope = 0x100 if slope & 0x20 else SLOPE_CORR[slope]
    t0, t1, t2 = slope << 7, ((0x78 - i) | 4) * slope, (j | 4) * slope
    ep = np.array([0, ((((j - i) & 0x78) | 4) * slope >> 8) & 0x1FF, (t1 >> 8) & 0x1FF,
                   ((((j - i) & 0x78) | 4) * slope >> 8) & 0x1FF, ((((j - i) + 0x80) | 4) * slope >> 8) & 0x1FF,
                   ((t1 + t0) >> 8) & 0x1FF, (t2 >> 8) & 0x1FF, ((t2 + t0) >> 8) & 0x1FF, slope], np.int64)
    k = np.arange(ecount + 1, dtype=np.int64)  # step k: scount = k, ecount = ecount - k
    major = major0 + k
    mpos = minor + k * step
    keep = (major >= 0) & (major < (w if x_major else h))
    k, major, mpos = k[keep], major[keep], mpos[keep]
    corr = ep[np.minimum(k, 2) * 3 + np.minimum(ecount - k, 2)]
    dist = (mpos >> (XY_SHIFT - 5)) & 31
    base = (mpos >> XY_SHIFT) - 1
    col = np.asarray(color, np.int64)
    for off, f in ((0, FILTER[dist + 32]), (1, FILTER[dist]), (2, FILTER[63 - dist])):
        a = (corr * f >> 8) & 0xFF
        m = base + off
        inside = (m >= 0) & (m < (h if x_major else w))
        yy, xx = (m[inside], major[inside]) if x_major else (major[inside], m[inside])
        a = a[inside, None]
        v = img[yy, xx].astype(np.int64)
        v += ((col - v) * a + 127) >> 8
        v += ((col - v) * a + 127) >> 8  # OpenCV blends twice
        img[yy, xx] = v.astype(np.uint8)  # one line never touches a pixel twice


# --------------------------------------------------------------------------------------------------------------- boxes
def corners(boxes):
    """(n, box_dim) bottom-centred boxes -> float32 (n, 8, 3) corners of the boxes shifted to a gravity-centre origin, by
    the reference's own torch operations (LiDARInstance3DBoxes(origin=(0.5, 0.5, 0.5)).corners)."""
    t = torch.as_tensor(np.asarray(boxes, np.float32)).clone()
    t[:, :3] += t[:, 3:6] * (t.new_tensor((0.5, 0.5, 0)) - t.new_tensor((0.5, 0.5, 0.5)))
    dims = t[:, 3:6]
    norm = torch.from_numpy(np.stack(np.unravel_index(np.arange(8), [2] * 3), axis=1)).to(dims.dtype)
    norm = norm[[0, 1, 3, 2, 4, 5, 7, 6]] - dims.new_tensor([0.5, 0.5, 0])
    c = dims.view([-1, 1, 3]) * norm.reshape([1, 8, 3])
    s, co = torch.sin(t[:, 6]), torch.cos(t[:, 6])
    one, zero = torch.ones_like(co), torch.zeros_like(co)
    rot_t = torch.stack([torch.stack([co, -s, zero]), torch.stack([s, co, zero]), torch.stack([zero, zero, one])])
    c = torch.einsum("aij,jka->aik", (c, rot_t))
    c += t[:, :3].view(-1, 1, 3)
    return c.numpy()


def project(boxes, labels, transform):
    """One view's drawn boxes, far to near -> (int64 endpoints (m, 8, 2), labels (m,), float64 coordinates (m, 8, 2))."""
    labels = np.asarray(labels).reshape(-1)
    if len(labels) == 0:
        return np.zeros((0, 8, 2), np.int64), labels, np.zeros((0, 8, 2))
    c = corners(boxes)
    n = c.shape[0]
    coords = np.concatenate([c.reshape(-1, 3), np.ones((n * 8, 1))], axis=-1) @ np.asarray(transform, np.float32).reshape(4, 4).T
    coords = coords.reshape(-1, 8, 4)
    keep = np.all(coords[..., 2] > 0, axis=1)
    coords, labels = coords[keep], labels[keep]
    order = np.argsort(-np.min(coords[..., 2], axis=1), kind="stable")
    coords, labels = coords[order].reshape(-1, 4), labels[order]
    coords[:, 2] = np.clip(coords[:, 2], 1e-5, 1e5)
    xy = (coords[:, :2] / coords[:, 2:3]).reshape(-1, 8, 2)
    with np.errstate(invalid="ignore"):
        return xy.astype(np.int64), labels, xy


def view_transforms(example):
    """float32 (V, 4, 4): img_aug_matrix @ lidar2image per view (numpy float32), lidar2image being
    bmm(camera_intrinsics, lidar2camera) when the example has none (demo/helper.py:495-505)."""
    l2i = example.get("lidar2image")
    if l2i is None:
        l2i = torch.bmm(torch.as_tensor(example["camera_intrinsics"]), torch.as_tensor(example["lidar2camera"]))
    l2i = np.asarray(l2i, np.float32)
    aug = example.get("img_aug_matrix")
    if aug is None:
        return l2i
    aug = np.asarray(aug, np.float32)
    return np.stack([aug[v] @ l2i[v] for v in range(len(l2i))])


def draw_boxes(img, endpoints, labels, classes=NUSCENES_OBJECT_CLASSES):
    """Draw the 12 edges of each box, in the given order, on uint8 [h, w, 3] in place."""
    for b in range(len(labels)):
        color = OBJECT_PALETTE[classes[int(labels[b])]]
        for s, e in EDGES:
            line_aa(img, endpoints[b, s], endpoints[b, e], color)
    return img


def show_box_on_views(images, example, classes=NUSCENES_OBJECT_CLASSES, transparent_bg=False):
    """uint8 (V, h, w, 3) views of one sample -> uint8 (V, h, w, 3 | 4) with its boxes drawn (RGBA on black with
    transparent_bg, alpha 255 where any channel is non-zero)."""
    images = np.asarray(images)
    trans = view_transforms(example)
    boxes = np.asarray(example["gt_bboxes_3d"], np.float32)
    labels = np.asarray(example["gt_labels_3d"]).reshape(-1)
    out = []
    for v in range(images.shape[0]):
        img = np.zeros_like(images[v]) if transparent_bg else images[v].copy()
        ends, lab, _ = project(boxes, labels, trans[v])
        if np.any((ends < -2 ** 31) | (ends >= 2 ** 31)):
            raise ValueError("a box corner projects outside the int32 range")
        draw_boxes(img, ends, lab, classes)
        if transparent_bg:
            img = np.concatenate([img, (np.any(img > 0, axis=2) * 255).astype(np.uint8)[..., None]], axis=2)
        out.append(img)
    return np.stack(out)
