"""Integer restatement of the FID protocol kernels (magicdrive_b200/csrc/capi_fid_protocol.cu) in numpy.

The reference scores images that went through Pillow: an antialiased bicubic resize, a zero pad, a JPEG save at Pillow's
defaults (quality 75, 4:2:0) and a load.  This module states each of those steps as plain integer arithmetic so that
`tests/test_fid_protocol_cpu.py` can hold it to Pillow byte for byte and the GPU tests can hold the kernels to it.

* `bicubic_coeffs` / `resample_u8`: the separable resample of an 8-bit image.  Filter weights are the Keys cubic
  (a = -0.5) evaluated in float64 at the output pixel's centre, with the support widened by the scale when downsampling
  (antialiasing), normalised to sum 1 and rounded to 22-bit fixed point.  A horizontal pass is rounded and clipped to uint8
  before the vertical pass; a pass whose size is unchanged is skipped.
* `jpeg_roundtrip_u8`: baseline JPEG encode then decode without the entropy coder, which is lossless.  Encode:
  fixed-point RGB -> YCbCr (ITU-R BT.601, 16 fraction bits), 2x2 chroma averaging with a 1, 2, 1, 2 ... rounding bias,
  edge replication to whole 16 x 16 MCUs, the integer Loeffler-Ligtenberg-Moschytz forward DCT (13 fraction bits, 2 extra
  bits between the passes), division by 8 x the quantiser with rounding away from zero.  Decode: multiplication by the
  quantiser, the matching integer inverse DCT with a wrap-around range limit, triangle ("fancy") 2x upsampling of the
  chroma in both directions, fixed-point YCbCr -> RGB.
"""
import numpy as np

PRECISION_BITS = 22  # fraction bits of the 8-bit resample coefficients

# ITU-T T.81 Annex K.1, natural (row-major) order
STD_LUMA_QT = np.array([
    16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
    14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
    49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99], np.int64)
STD_CHROMA_QT = np.array([
    17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99,
    47, 66, 99, 99, 99, 99, 99, 99] + [99] * 32, np.int64)


# ---------------------------------------------------------------------------------------------------------------- resample
def _cubic(x):
    a = -0.5
    x = abs(x)
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def bicubic_coeffs(in_size: int, out_size: int):
    """(first [out], count [out], weights int32 [out, taps]) of the 8-bit bicubic resample from in_size to out_size.
    Output pixel i reads inputs first[i] .. first[i] + count[i] - 1 with weights[i, :count[i]] (the rest are 0)."""
    if in_size <= 0 or out_size <= 0:
        raise ValueError(f"bad resample sizes {in_size} -> {out_size}")
    scale = in_size / out_size
    fscale = max(scale, 1.0)
    support = 2.0 * fscale
    taps = int(np.ceil(support)) * 2 + 1
    first = np.zeros(out_size, np.int32)
    count = np.zeros(out_size, np.int32)
    kk = np.zeros((out_size, taps), np.int32)
    for i in range(out_size):
        center = (i + 0.5) * scale
        lo = max(int(center - support + 0.5), 0)  # int(): truncation toward zero, as a C cast
        hi = min(int(center + support + 0.5), in_size)
        w = [_cubic((x + lo - center + 0.5) * (1.0 / fscale)) for x in range(hi - lo)]
        total = sum(w)  # left-to-right float64 sum
        for x, v in enumerate(w):
            v = v / total if total != 0.0 else v
            kk[i, x] = int(-0.5 + v * (1 << PRECISION_BITS)) if v < 0 else int(0.5 + v * (1 << PRECISION_BITS))
        first[i], count[i] = lo, hi - lo
    return first, count, kk


def _pass(x, axis, first, count, kk):
    """One resample pass of uint8 x along `axis` -> uint8."""
    x = np.moveaxis(x.astype(np.int64), axis, -1)
    n_in = x.shape[-1]
    acc = np.full(x.shape[:-1] + (len(first),), 1 << (PRECISION_BITS - 1), np.int64)
    for t in range(kk.shape[1]):
        idx = np.minimum(first + t, n_in - 1)
        wt = np.where(t < count, kk[:, t], 0).astype(np.int64)
        acc += x[..., idx] * wt
    out = np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)
    return np.moveaxis(out, -1, axis)


def resample_u8(img: np.ndarray, out_h: int, out_w: int) -> np.ndarray:
    """uint8 [..., H, W, 3] -> [..., out_h, out_w, 3]: horizontal pass, then vertical pass (each only if its size changes)."""
    h, w = img.shape[-3], img.shape[-2]
    x = img
    if out_w != w:
        x = _pass(x, -2, *bicubic_coeffs(w, out_w))
    if out_h != h:
        x = _pass(x, -3, *bicubic_coeffs(h, out_h))
    return np.ascontiguousarray(x)


def to_u8(x: np.ndarray) -> np.ndarray:
    """float32 [0, 1] -> uint8 as diffusers' numpy_to_pil: (x * 255).round() in float32, half to even."""
    return np.clip(np.round(np.asarray(x, np.float32) * np.float32(255)), 0, 255).astype(np.uint8)


def place(img: np.ndarray, canvas_hw, top: int, left: int, crop=None) -> np.ndarray:
    """Window crop = (top, left, h, w) of img [..., H, W, 3] (all of it if None), written at (top, left) of a zero
    canvas [..., canvas_h, canvas_w, 3]."""
    if crop is not None:
        ct, cl, ch, cw = crop
        img = img[..., ct:ct + ch, cl:cl + cw, :]
    out = np.zeros(img.shape[:-3] + tuple(canvas_hw) + (3,), np.uint8)
    out[..., top:top + img.shape[-3], left:left + img.shape[-2], :] = img
    return out


# -------------------------------------------------------------------------------------------------------------------- JPEG
def quant_tables(quality: int = 75):
    """The standard tables scaled for `quality` (1..100) and clamped to the baseline range 1..255: (luma, chroma)."""
    if not 1 <= quality <= 100:
        raise ValueError(f"quality must be in 1..100, got {quality}")
    scale = 5000 // quality if quality < 50 else 200 - 2 * quality
    f = lambda t: np.clip((t * scale + 50) // 100, 1, 255)
    return f(STD_LUMA_QT), f(STD_CHROMA_QT)


def _fix(x):
    return int(x * (1 << 16) + 0.5)


def rgb_to_ycc(rgb):
    r, g, b = (rgb[..., i].astype(np.int64) for i in range(3))
    half, off = 1 << 15, 128 << 16
    y = (_fix(0.29900) * r + _fix(0.58700) * g + _fix(0.11400) * b + half) >> 16
    cb = (-_fix(0.16874) * r - _fix(0.33126) * g + _fix(0.5) * b + off + half - 1) >> 16
    cr = (_fix(0.5) * r - _fix(0.41869) * g - _fix(0.08131) * b + off + half - 1) >> 16
    return y, cb, cr


def ycc_to_rgb(y, cb, cr):
    cb, cr = cb.astype(np.int64) - 128, cr.astype(np.int64) - 128
    half = 1 << 15
    r = y + ((_fix(1.40200) * cr + half) >> 16)
    g = y + ((-_fix(0.34414) * cb - _fix(0.71414) * cr + half) >> 16)
    b = y + ((_fix(1.77200) * cb + half) >> 16)
    return np.stack([np.clip(v, 0, 255) for v in (r, g, b)], -1).astype(np.uint8)


# Loeffler-Ligtenberg-Moschytz constants, 13 fraction bits
C_BITS, P1_BITS = 13, 2
F0298, F0390, F0541, F0765, F0899, F1175 = 2446, 3196, 4433, 6270, 7373, 9633
F1501, F1847, F1961, F2053, F2562, F3072 = 12299, 15137, 16069, 16819, 20995, 25172


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _fdct_1d(d, even_shift, odd_shift):
    """Forward 8-point transform along the last axis.  even_shift < 0 means a left shift by -even_shift."""
    s = [d[..., i] for i in range(8)]
    t0, t7 = s[0] + s[7], s[0] - s[7]
    t1, t6 = s[1] + s[6], s[1] - s[6]
    t2, t5 = s[2] + s[5], s[2] - s[5]
    t3, t4 = s[3] + s[4], s[3] - s[4]
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    out = [None] * 8
    if even_shift < 0:
        out[0], out[4] = (t10 + t11) << -even_shift, (t10 - t11) << -even_shift
    else:
        out[0], out[4] = _descale(t10 + t11, even_shift), _descale(t10 - t11, even_shift)
    z1 = (t12 + t13) * F0541
    out[2] = _descale(z1 + t13 * F0765, odd_shift)
    out[6] = _descale(z1 - t12 * F1847, odd_shift)
    z1, z2, z3, z4 = t4 + t7, t5 + t6, t4 + t6, t5 + t7
    z5 = (z3 + z4) * F1175
    t4, t5, t6, t7 = t4 * F0298, t5 * F2053, t6 * F3072, t7 * F1501
    z1, z2, z3, z4 = -z1 * F0899, -z2 * F2562, -z3 * F1961 + z5, -z4 * F0390 + z5
    out[7] = _descale(t4 + z1 + z3, odd_shift)
    out[5] = _descale(t5 + z2 + z4, odd_shift)
    out[3] = _descale(t6 + z2 + z3, odd_shift)
    out[1] = _descale(t7 + z1 + z4, odd_shift)
    return np.stack(out, -1)


def _idct_1d(d, shift):
    s = [d[..., i] for i in range(8)]
    z1 = (s[2] + s[6]) * F0541
    t2, t3 = z1 - s[6] * F1847, z1 + s[2] * F0765
    t0, t1 = (s[0] + s[4]) << C_BITS, (s[0] - s[4]) << C_BITS
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    o0, o1, o2, o3 = s[7], s[5], s[3], s[1]
    z1, z2, z3, z4 = o0 + o3, o1 + o2, o0 + o2, o1 + o3
    z5 = (z3 + z4) * F1175
    o0, o1, o2, o3 = o0 * F0298, o1 * F2053, o2 * F3072, o3 * F1501
    z1, z2, z3, z4 = -z1 * F0899, -z2 * F2562, -z3 * F1961 + z5, -z4 * F0390 + z5
    o0, o1, o2, o3 = o0 + z1 + z3, o1 + z2 + z4, o2 + z2 + z3, o3 + z1 + z4
    out = [t10 + o3, t11 + o2, t12 + o1, t13 + o0, t13 - o0, t12 - o1, t11 - o2, t10 - o3]
    return np.stack([_descale(v, shift) for v in out], -1)


def _range_limit(x):
    """Centred IDCT output -> sample: the value wraps modulo 1024 into [-512, 511], then x + 128 is clipped to 0..255."""
    x = ((x + 512) & 1023) - 512
    return np.clip(x + 128, 0, 255)


def _blocks(p):
    h, w = p.shape[-2:]
    return p.reshape(p.shape[:-2] + (h // 8, 8, w // 8, 8)).swapaxes(-3, -2)


def _unblocks(b):
    b = b.swapaxes(-3, -2)
    s = b.shape
    return b.reshape(s[:-4] + (s[-4] * 8, s[-2] * 8))


def code_plane(p, qt):
    """Samples [..., H, W] (H, W multiples of 8, int) -> the decoder's reconstructed samples of the same shape."""
    b = _blocks(p.astype(np.int64) - 128)
    c = _fdct_1d(b, -P1_BITS, C_BITS - P1_BITS)  # rows
    c = _fdct_1d(c.swapaxes(-1, -2), P1_BITS, C_BITS + P1_BITS).swapaxes(-1, -2)  # columns
    q = qt.reshape(8, 8) * 8
    a = np.abs(c)
    coef = np.sign(c) * ((a + (q >> 1)) // q)
    d = coef * qt.reshape(8, 8)
    r = _idct_1d(d.swapaxes(-1, -2), C_BITS - P1_BITS).swapaxes(-1, -2)  # columns
    r = _idct_1d(r, C_BITS + P1_BITS + 3)  # rows
    return _unblocks(_range_limit(r))


def _fancy_h2v2(c, out_h, out_w):
    """Chroma [..., hc, wc] -> [..., out_h, out_w] by the triangle filter: 3/4 nearest + 1/4 next nearest in each direction,
    edges replicated, biases 8 (even output) and 7 (odd output) before >> 4.  Chroma 2 samples wide or less is replicated."""
    hc, wc = c.shape[-2:]
    c = c.astype(np.int64)
    if wc <= 2:
        up = np.repeat(np.repeat(c, 2, -2), 2, -1)
        return up[..., :out_h, :out_w]
    rows = np.arange(out_h)
    near = rows >> 1
    far = np.clip(np.where(rows & 1, near + 1, near - 1), 0, hc - 1)
    cs = 3 * c[..., near, :] + c[..., far, :]  # column sums [.., out_h, wc]
    cols = np.arange(out_w)
    cx = cols >> 1
    nb = np.clip(np.where(cols & 1, cx + 1, cx - 1), 0, wc - 1)
    bias = np.where(cols & 1, 7, 8)
    return (3 * cs[..., cx] + cs[..., nb] + bias) >> 4


def jpeg_roundtrip_u8(img: np.ndarray, quality: int = 75) -> np.ndarray:
    """uint8 RGB [..., H, W, 3] -> the RGB image a baseline 4:2:0 JPEG at `quality` decodes to (islow DCTs, fancy
    upsampling)."""
    img = np.asarray(img, np.uint8)
    h, w = img.shape[-3], img.shape[-2]
    qy, qc = quant_tables(quality)
    hp, wp = -(-h // 16) * 16, -(-w // 16) * 16
    hc, wc = -(-h // 2), -(-w // 2)
    y, cb, cr = rgb_to_ycc(img)
    # luma: replicate the last row / column to whole MCUs
    ri, ci = np.minimum(np.arange(hp), h - 1), np.minimum(np.arange(wp), w - 1)
    y_pad = y[..., ri, :][..., ci]
    # chroma: full-resolution columns replicated to the MCU width and rows to an even count, 2x2 sums with the
    # alternating bias, then the last chroma row replicated to the MCU height
    r2 = np.minimum(np.arange(2 * hc), h - 1)
    chroma = []
    for p in (cb, cr):
        f = p[..., r2, :][..., ci]
        s = f[..., 0::2, 0::2] + f[..., 0::2, 1::2] + f[..., 1::2, 0::2] + f[..., 1::2, 1::2]
        bias = np.where(np.arange(wp // 2) & 1, 2, 1)
        d = (s + bias) >> 2
        d = d[..., np.minimum(np.arange(hp // 2), hc - 1), :]
        chroma.append(code_plane(d, qc)[..., :hc, :wc])
    y_rec = code_plane(y_pad, qy)[..., :h, :w]
    cb_up, cr_up = (_fancy_h2v2(c, h, w) for c in chroma)
    return ycc_to_rgb(y_rec, cb_up, cr_up)


# ----------------------------------------------------------------------------------------------------------------- configs
# (image_size (h, w), back_resize (h, w), back_pad (left, top, right, bottom), resize_ratio) of the shipped configs
CONFIGS = {
    "224x400": ((224, 400), (896, 1600), (0, 4, 0, 0), 0.25),
    "272x736": ((272, 736), (544, 1472), (64, 356, 64, 0), 0.5),
    "424x800": ((424, 800), (848, 1600), (0, 52, 0, 0), 0.5),
}
CAMERA_HW = (900, 1600)


def scoring_window(image_size, resize_ratio, camera_hw=CAMERA_HW):
    """(resize (h, w), crop (top, left, h, w)) of the scoring side: the resize to int(900 r) x int(1600 r) and the
    top-centre crop to image_size."""
    rh, rw = int(camera_hw[0] * resize_ratio), int(camera_hw[1] * resize_ratio)
    fh, fw = image_size
    return (rh, rw), (rh - fh, int(max(0, rw - fw) / 2), fh, fw)


def views(seed: int, n: int, h: int, w: int, noise: float = 0.01, ties: float = 0.05) -> np.ndarray:
    """Seeded float32 views in [0, 1], (n, h, w, 3): smooth colour fields, a sharp-edged block and `noise` (std) of
    Gaussian noise, with a fraction `ties` of the pixels on rounding ties of x * 255."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    out = np.empty((n, h, w, 3), np.float32)
    for i in range(n):
        f = rng.uniform(5, 40, 3).astype(np.float32)
        base = np.stack([0.5 + 0.4 * np.sin(xx / f[0] + yy / f[1]), xx / w * 0.8 + 0.1, 0.5 + 0.45 * np.cos(yy / f[2])], -1)
        y0, x0 = rng.integers(0, h // 2), rng.integers(0, w // 2)
        base[y0:y0 + h // 3, x0:x0 + w // 4] = rng.uniform(0, 1, 3)
        base += rng.standard_normal(base.shape).astype(np.float32) * np.float32(noise)
        tie = rng.random(base.shape[:2]) < ties  # (k + 0.5) / 255: half-way between two levels
        base[tie] = (rng.integers(0, 255, (int(tie.sum()), 3)) + 0.5) / 255
        out[i] = np.clip(base, 0, 1)
    return out


def golden_images(entry) -> np.ndarray:
    """The uint8 images of one config entry of tests/golden/fid_protocol.pt (oracle/make_golden_fid_protocol.py), stored
    as lzma-compressed differences along the width (modulo 256)."""
    import lzma
    d = np.frombuffer(lzma.decompress(entry["delta_lzma"]), np.uint8).reshape(entry["shape"])
    return np.cumsum(d, axis=2, dtype=np.uint8)


def golden_delta(img: np.ndarray) -> bytes:
    import lzma
    d = np.diff(img.astype(np.int16), axis=2, prepend=0).astype(np.uint8)
    return lzma.compress(d.tobytes(), preset=9 | lzma.PRESET_EXTREME)


def generated(img_u8, cfg, jpeg=True, quality=75):
    """The whole generation-then-scoring chain on uint8 views [..., h, w, 3] for a config tuple of CONFIGS."""
    image_size, back_resize, pad, ratio = cfg
    canvas = (back_resize[0] + pad[1] + pad[3], back_resize[1] + pad[0] + pad[2])
    x = place(resample_u8(img_u8, *back_resize), canvas, pad[1], pad[0])
    if jpeg:
        x = jpeg_roundtrip_u8(x, quality)
    return real(x, cfg)


def real(img_u8, cfg):
    image_size, _, _, ratio = cfg
    (rh, rw), crop = scoring_window(image_size, ratio)
    return place(resample_u8(img_u8, rh, rw), crop[2:], 0, 0, crop)
