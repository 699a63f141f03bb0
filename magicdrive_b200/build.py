"""Build the sm_90a (H100) C-ABI shared library in-tree with nvcc (no torch extension machinery).

`python -m magicdrive_b200.build` -> magicdrive_b200/lib/libmagicdrive_b200.so
"""
import hashlib
import os
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent
CSRC = ROOT / "csrc"
LIBDIR = ROOT / "lib"
LIB = LIBDIR / "libmagicdrive_b200.so"
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "--use_fast_math",
]
# --use_fast_math is NOT applied to the files listed here (exact erf/sin/cos/exp paths that parity tests pin)
PRECISE = {"capi_pointwise.cu", "capi_gemm.cu", "capi_inputprep.cu", "capi_fid.cu"}


def _sources():
    return sorted(CSRC.glob("*.cu"))


def _digest():
    h = hashlib.sha256()
    for f in sorted(list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h")) +
                    [ROOT.parent / "include" / "magicdrive_b200.h", Path(__file__)]):
        h.update(f.name.encode())
        h.update(f.read_bytes())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> Path:
    LIBDIR.mkdir(exist_ok=True)
    stamp = LIBDIR / "build.sha256"
    dig = _digest()
    if not force and LIB.exists() and stamp.exists() and stamp.read_text().strip() == dig:
        return LIB
    nvcc = os.environ.get("NVCC", "nvcc")
    objs = []
    procs = []
    for src in _sources():
        obj = LIBDIR / (src.stem + ".o")
        flags = [f for f in NVCC_FLAGS if not (f == "--use_fast_math" and src.name in PRECISE)]
        cmd = [nvcc, *flags, "-c", str(src), "-o", str(obj)]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(str(obj))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            failed = True
            sys.stderr.write(f"[magicdrive_b200.build] {src.name} failed:\n{out}\n")
        elif verbose and out:
            sys.stderr.write(out)
    if failed:
        raise RuntimeError("nvcc failed; see stderr")
    subprocess.check_call([nvcc, "-shared", "-o", str(LIB), *objs, "-lcudart_static", "-lpthread", "-ldl", "-lrt"])
    stamp.write_text(dig)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
