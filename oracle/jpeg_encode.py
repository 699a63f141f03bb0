"""Numpy restatement of the baseline JPEG encoder (magicdrive_b200/csrc/capi_jpeg.cu): the bytes Pillow writes for
`Image.fromarray(x).save(f, "JPEG", quality=q)` at its defaults (4:2:0, standard Huffman tables, no `optimize`, no
`progressive`, no restart interval).

* `quantised_blocks`: the coefficients.  Colour conversion, chroma sums, the islow forward DCT and the rounding are
  oracle/fid_protocol.py's (the same ones `jpeg_roundtrip_u8` decodes); the result is int [mcus, 6, 64] in zigzag order
  (Y00, Y01, Y10, Y11, Cb, Cr per MCU).  Blocks of an edge MCU that lie wholly past the luma plane's blocks are not coded
  from pixels: libjpeg gives them zero AC and the DC of the block before them in the MCU (jccoefct.c, compress_data).
* `entropy_code`: DC differences per component (predictors start at 0), AC run lengths with ZRL before a nonzero
  coefficient that follows 16 or more zeros, EOB unless coefficient 63 is nonzero, the ITU-T T.81 K.3 tables, 1-bits to the
  byte boundary and a 0x00 after every 0xFF byte.
* `header`: SOI, APP0 JFIF 1.01 (density 1 x 1, no units), DQT luma and chroma (8-bit, zigzag), SOF0, the four DHT
  segments and SOS: 623 bytes.  `encode` = header + entropy-coded data + EOI.
"""
import numpy as np

from oracle import fid_protocol as F

HEADER_BYTES = 623

# natural index of zigzag position k
ZIGZAG = np.array([
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55,
    62, 63], np.int64)

# ITU-T T.81 K.3 (bits: code counts of lengths 1..16; values in code order): DC luma, AC luma, DC chroma, AC chroma
DC_BITS = ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], [0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0])
DC_VALS = (list(range(12)), list(range(12)))
AC_BITS = ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d], [0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77])
AC_VALS = (bytes.fromhex(
    "01020300041105122131410613516107227114328191a1082342b1c11552d1f02433627282090a161718191a25262728292a3435363738393a"
    "434445464748494a535455565758595a636465666768696a737475767778797a838485868788898a92939495969798999aa2a3a4a5a6a7a8a9"
    "aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae1e2e3e4e5e6e7e8e9eaf1f2f3f4f5f6f7f8f9fa"), bytes.fromhex(
    "000102031104052131061241510761711322328108144291a1b1c109233352f0156272d10a162434e125f11718191a262728292a3536373839"
    "3a434445464748494a535455565758595a636465666768696a737475767778797a82838485868788898a92939495969798999aa2a3a4a5a6a7"
    "a8a9aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7c8c9cad2d3d4d5d6d7d8d9dae2e3e4e5e6e7e8e9eaf2f3f4f5f6f7f8f9fa"))


def huffman_codes(bits, vals):
    """{symbol: (code, length)} of a table given by its code-length counts (T.81 Annex C)."""
    codes, code, k = {}, 0, 0
    for length in range(1, 17):
        for _ in range(bits[length - 1]):
            codes[vals[k]] = (code, length)
            code += 1
            k += 1
        code <<= 1
    return codes


DC_CODES = tuple(huffman_codes(b, v) for b, v in zip(DC_BITS, DC_VALS))
AC_CODES = tuple(huffman_codes(b, v) for b, v in zip(AC_BITS, AC_VALS))


def _quantise(p, qt):
    """Samples [..., H, W] (multiples of 8) -> quantised coefficients [..., H / 8, W / 8, 64] in natural order, with
    code_plane's forward DCT and rounding."""
    b = F._blocks(p.astype(np.int64) - 128)
    c = F._fdct_1d(b, -F.P1_BITS, F.C_BITS - F.P1_BITS)
    c = F._fdct_1d(c.swapaxes(-1, -2), F.P1_BITS, F.C_BITS + F.P1_BITS).swapaxes(-1, -2)
    q = qt.reshape(8, 8) * 8
    coef = np.sign(c) * ((np.abs(c) + (q >> 1)) // q)
    return coef.reshape(coef.shape[:-2] + (64,))


def quantised_blocks(img: np.ndarray, quality: int = 75) -> np.ndarray:
    """uint8 RGB [H, W, 3] -> int64 [mcus, 6, 64]: the quantised coefficients libjpeg codes, zigzag order, MCUs row-major."""
    img = np.asarray(img, np.uint8)
    h, w = img.shape[:2]
    qy, qc = F.quant_tables(quality)
    hp, wp = -(-h // 16) * 16, -(-w // 16) * 16
    hc = -(-h // 2)
    y, cb, cr = F.rgb_to_ycc(img)
    ri, ci = np.minimum(np.arange(hp), h - 1), np.minimum(np.arange(wp), w - 1)
    yb = _quantise(y[ri][:, ci], qy)  # [hp / 8, wp / 8, 64]
    r2 = np.minimum(np.arange(2 * hc), h - 1)
    chroma = []
    for p in (cb, cr):  # as jpeg_roundtrip_u8: 2 x 2 sums with the 1, 2 bias, the last chroma row replicated
        f = p[r2][:, ci]
        s = f[0::2, 0::2] + f[0::2, 1::2] + f[1::2, 0::2] + f[1::2, 1::2]
        d = (s + np.where(np.arange(wp // 2) & 1, 2, 1)) >> 2
        chroma.append(_quantise(d[np.minimum(np.arange(hp // 2), hc - 1)], qc))
    my, mx = hp // 16, wp // 16
    out = np.empty((my, mx, 6, 64), np.int64)
    out[:, :, 0] = yb[0::2, 0::2]
    out[:, :, 1] = yb[0::2, 1::2]
    out[:, :, 2] = yb[1::2, 0::2]
    out[:, :, 3] = yb[1::2, 1::2]
    out[:, :, 4], out[:, :, 5] = chroma
    # dummy luma blocks: past ceil(w / 8) columns or ceil(h / 8) rows of blocks
    bw, bh = -(-w // 8), -(-h // 8)
    for b in (1, 2, 3):
        col = 2 * np.arange(mx) + (b & 1)
        row = 2 * np.arange(my) + (b >> 1)
        dummy = (row[:, None] >= bh) | (col[None, :] >= bw)
        out[:, :, b][dummy] = 0
        out[:, :, b, 0] = np.where(dummy, out[:, :, b - 1, 0], out[:, :, b, 0])
    return out[..., ZIGZAG].reshape(my * mx, 6, 64)


def _category(v):
    return int(abs(v)).bit_length()


def block_codes(blk, pred, table):
    """(code, length) words of one zigzag block given the previous DC of its component; table 0 luma, 1 chroma."""
    words = []
    diff = int(blk[0]) - pred
    n = _category(diff)
    words.append(DC_CODES[table][n])
    if n:
        words.append(((diff if diff >= 0 else diff - 1) & ((1 << n) - 1), n))
    ac = AC_CODES[table]
    last = 0
    for k in np.flatnonzero(blk[1:]) + 1:
        r = k - last - 1
        while r > 15:
            words.append(ac[0xF0])
            r -= 16
        v = int(blk[k])
        n = _category(v)
        words.append(ac[(r << 4) | n])
        words.append(((v if v >= 0 else v - 1) & ((1 << n) - 1), n))
        last = k
    if last < 63:
        words.append(ac[0x00])
    return words


def entropy_code(blocks: np.ndarray) -> bytes:
    """[mcus, 6, 64] zigzag coefficients -> the entropy-coded segment: padded with 1-bits, 0xFF bytes stuffed."""
    pred = [0, 0, 0]
    acc, nbits, out = 0, 0, bytearray()
    for mcu in blocks:
        for b, blk in enumerate(mcu):
            comp = 0 if b < 4 else b - 3
            for code, length in block_codes(blk, pred[comp], min(comp, 1)):
                acc = (acc << length) | code
                nbits += length
            pred[comp] = int(blk[0])
            while nbits >= 8:  # keep at most 7 pending bits
                nbits -= 8
                out.append((acc >> nbits) & 0xFF)
                acc &= (1 << nbits) - 1
    if nbits:
        out.append(((acc << (8 - nbits)) | ((1 << (8 - nbits)) - 1)) & 0xFF)
    return bytes(out).replace(b"\xff", b"\xff\x00")


def scan_bits(blocks: np.ndarray) -> int:
    """Length in bits of the entropy-coded data before padding and stuffing."""
    pred, total = [0, 0, 0], 0
    for mcu in blocks:
        for b, blk in enumerate(mcu):
            comp = 0 if b < 4 else b - 3
            total += sum(length for _, length in block_codes(blk, pred[comp], min(comp, 1)))
            pred[comp] = int(blk[0])
    return total


def _segment(marker, payload):
    return bytes([0xFF, marker]) + (len(payload) + 2).to_bytes(2, "big") + payload


def header(h: int, w: int, quality: int = 75) -> bytes:
    """The 623 bytes Pillow writes before the entropy-coded data of an h x w RGB image."""
    if not (1 <= h <= 65535 and 1 <= w <= 65535):
        raise ValueError(f"JPEG sizes are 1..65535, got {h}x{w}")
    qy, qc = F.quant_tables(quality)
    out = b"\xff\xd8" + _segment(0xE0, b"JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00")
    for i, q in enumerate((qy, qc)):
        out += _segment(0xDB, bytes([i]) + bytes(int(v) for v in q[ZIGZAG]))
    out += _segment(0xC0, bytes([8]) + h.to_bytes(2, "big") + w.to_bytes(2, "big") +
                    bytes([3, 1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1]))
    for cls, i, bits, vals in ((0, 0, DC_BITS[0], DC_VALS[0]), (1, 0, AC_BITS[0], AC_VALS[0]),
                               (0, 1, DC_BITS[1], DC_VALS[1]), (1, 1, AC_BITS[1], AC_VALS[1])):
        out += _segment(0xC4, bytes([(cls << 4) | i]) + bytes(bits) + bytes(vals))
    out += _segment(0xDA, bytes([3, 1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0]))
    assert len(out) == HEADER_BYTES
    return out


def encode(img: np.ndarray, quality: int = 75) -> bytes:
    """uint8 RGB [H, W, 3] -> the JPEG file Pillow writes at `quality`."""
    img = np.asarray(img, np.uint8)
    return header(img.shape[0], img.shape[1], quality) + entropy_code(quantised_blocks(img, quality)) + b"\xff\xd9"
