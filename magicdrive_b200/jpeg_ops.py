"""torch.Tensor-facing wrappers of the C-ABI JPEG encoder (mdb_jpeg_scratch_bytes, mdb_jpeg_encode_u8;
csrc/capi_jpeg.cu): uint8 RGB views on the device -> the `.jpg` files Pillow writes for them, byte for byte.

They sit beside ops.py and share its plumbing: raw pointers and the current stream go to `libmagicdrive_b200.so`, launches
count in `ops.launch_count()`, and there is no CPU or eager fallback.  Their CPU restatement for host tests is
tests/jpeg_ops_emulator.py.
"""
import torch

from . import _lib, ops
from ._lib import check
from .ops import _need_cuda, _ptr, _stream

HEADER_BYTES = 623  # MDB_JPEG_HEADER_BYTES
CHUNK = 4096  # bytes of entropy-coded data per scratch chunk


def scratch_bytes(n: int, h: int, w: int, chunks: int) -> int:
    """mdb_jpeg_scratch_bytes: scratch for n images h x w with `chunks` 4 KiB chunks of entropy-coded data."""
    v = _lib.lib().mdb_jpeg_scratch_bytes(n, h, w, chunks)
    if v < 0:
        raise ValueError(f"bad JPEG batch {n} x {h}x{w} with {chunks} chunks")
    return v


def jpeg_encode_u8(x, quality: int = 75, *, scratch, out):
    """mdb_jpeg_encode_u8, one attempt: uint8 RGB [n, h, w, 3] -> the files Pillow saves at `quality`, back to back in
    `out` (uint8, device).  scratch: uint8 device tensor of at least scratch_bytes(n, h, w, n) bytes.  Returns the host int64
    meta [n, 3]: per image (entropy-coded bytes before stuffing, file length, offset in out); a length of -1 means the
    scratch was too small to count it and an offset of -1 that the files were not written."""
    _need_cuda(x, scratch, out)
    if x.dtype != torch.uint8 or x.dim() != 4 or x.shape[3] != 3:
        raise ValueError(f"expected uint8 [n, h, w, 3], got {x.dtype} {tuple(x.shape)}")
    if scratch.dtype != torch.uint8 or out.dtype != torch.uint8 or not scratch.is_contiguous() or not out.is_contiguous():
        raise ValueError("scratch and out must be contiguous uint8 tensors")
    x = x.contiguous()
    n, h, w = x.shape[:3]
    meta = torch.empty((n, 3), dtype=torch.int64, device=x.device)
    check(_lib.lib().mdb_jpeg_encode_u8(_ptr(x), n, h, w, quality, _ptr(scratch), scratch.numel(), _ptr(out),
                                        out.numel(), _ptr(meta), _stream()), "mdb_jpeg_encode_u8")
    ops._launches += 9
    return meta.cpu()


def encode_jpeg(x, quality: int = 75) -> list:
    """uint8 RGB [n, h, w, 3] on the device -> n `bytes` objects, the JPEG files PIL.Image.fromarray(x[i]).save(f, "JPEG",
    quality=quality) writes.  The buffers start at 4 bits per pixel of entropy-coded data; a batch that needs more is
    encoded again with the sizes the first attempt measured.  Only the files' bytes are copied to the host."""
    if x.dtype != torch.uint8 or x.dim() != 4 or x.shape[3] != 3:
        raise ValueError(f"expected uint8 [n, h, w, 3], got {x.dtype} {tuple(x.shape)}")
    n, h, w = x.shape[:3]
    chunks = n * (h * w // (2 * CHUNK) + 1)
    out_bytes = n * (HEADER_BYTES + 2) + chunks * CHUNK
    for _ in range(3):
        scratch = torch.empty(scratch_bytes(n, h, w, chunks), dtype=torch.uint8, device=x.device)
        out = torch.empty(out_bytes, dtype=torch.uint8, device=x.device)
        meta = jpeg_encode_u8(x, quality, scratch=scratch, out=out)
        scan, length, offset = meta.unbind(1)
        if bool((offset >= 0).all()):
            total = int(length.sum())
            data = out[:total].cpu().numpy().tobytes()
            return [data[o:o + l] for o, l in zip(offset.tolist(), length.tolist())]
        chunks = max(chunks, int(((scan + CHUNK - 1) // CHUNK).sum()))
        # unknown lengths: every entropy-coded byte may be an 0xFF followed by a stuffed 0x00
        need = length.sum() if bool((length >= 0).all()) else (2 * scan + HEADER_BYTES + 2).sum()
        out_bytes = max(out_bytes, int(need))
    raise RuntimeError("mdb_jpeg_encode_u8 did not fit the sizes it measured")
