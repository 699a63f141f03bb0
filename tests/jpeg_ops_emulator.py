"""TEST INFRASTRUCTURE ONLY — a numpy restatement of the operators of magicdrive_b200/jpeg_ops.py (the JPEG encoder's
kernels), following include/magicdrive_b200.h, so that the writer's host logic runs in the build container, which has no
GPU.  Never imported by the package; `install(monkeypatch)` swaps it in for one test.  Every function takes exactly the
arguments of its jpeg_ops.py counterpart (tests/test_jpeg_ops_emulator_cpu.py holds them equal).  The files are
oracle/jpeg_encode.py's; the scratch layout and the capacity rules are the C entry points'."""
import torch

from magicdrive_b200 import jpeg_ops

CHUNK, HEADER = 4096, 623


def _align(v):
    return (v + 255) & ~255


def scratch_bytes(n, h, w, chunks):
    if n <= 0 or not (1 <= h <= 65535 and 1 <= w <= 65535) or chunks < 0:
        raise ValueError(f"bad JPEG batch {n} x {h}x{w} with {chunks} chunks")
    mcus = ((h + 15) // 16) * ((w + 15) // 16)
    off = _align(n * mcus * 384 * 2)  # coefficients
    off = _align(off + n * mcus * 4)  # MCU bits
    off = _align(off + n * mcus * 8)  # MCU first bits
    off = _align(off + n * 32)  # image layout
    off = _align(off + 64)  # flags
    off = _align(off + chunks * 8)  # chunk 0xFF counts and positions
    return off + chunks * CHUNK


def jpeg_encode_u8(x, quality=75, *, scratch, out):
    from oracle import jpeg_encode
    assert x.dtype == torch.uint8 and x.dim() == 4 and x.shape[3] == 3, (x.dtype, tuple(x.shape))
    assert 1 <= quality <= 100, quality
    n, h, w = x.shape[:3]
    assert scratch.numel() >= scratch_bytes(n, h, w, n) and out.numel() >= n * (HEADER + 3), "too small to launch"
    chunks = (scratch.numel() - scratch_bytes(n, h, w, 0)) // (CHUNK + 8)
    while chunks > 0 and scratch_bytes(n, h, w, chunks) > scratch.numel():
        chunks -= 1
    files = [jpeg_encode.encode(v, quality) for v in x.cpu().numpy()]
    scan = [len(f) - HEADER - 2 - f[HEADER:-2].count(b"\xff") for f in files]
    meta = torch.full((n, 3), -1, dtype=torch.int64)
    meta[:, 0] = torch.tensor(scan)
    if sum(-(-s // CHUNK) for s in scan) > chunks:
        return meta
    meta[:, 1] = torch.tensor([len(f) for f in files])
    if sum(len(f) for f in files) > out.numel():
        return meta
    pos = 0
    for i, f in enumerate(files):
        out[pos:pos + len(f)] = torch.frombuffer(bytearray(f), dtype=torch.uint8)
        meta[i, 2] = pos
        pos += len(f)
    return meta


EMULATED = ["scratch_bytes", "jpeg_encode_u8"]


def install(monkeypatch):
    """Swap every operator of magicdrive_b200.jpeg_ops that calls the library for its CPU restatement."""
    for name in EMULATED:
        assert hasattr(jpeg_ops, name), name
        monkeypatch.setattr(jpeg_ops, name, globals()[name])
