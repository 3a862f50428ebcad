"""In-tree build of libb200audio.so with nvcc for sm_90a (H100; no torch headers, no JIT cache).

``python -m audio_b200._build`` (or ``__graft_entry__.build()``) compiles every ``csrc/*.cu``
into ``audio_b200/lib/libb200audio.so``.  The shared object is git-ignored but travels with
the working tree, so a GPU machine only ever loads the prebuilt file.
"""
from __future__ import annotations

import concurrent.futures
import glob
import hashlib
import os
import shutil
import subprocess
import sys

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
LIB_DIR = os.path.join(PKG_DIR, "lib")
OBJ_DIR = os.path.join(PKG_DIR, "build")
LIB_PATH = os.path.join(LIB_DIR, "libb200audio.so")
STAMP = os.path.join(LIB_DIR, "libb200audio.stamp")

GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [
    *GENCODE,
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "-Xcompiler", "-fvisibility=hidden",
    "-Xptxas", "-v",
    "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found; cannot build libb200audio.so")


def _sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def _digest() -> str:
    h = hashlib.sha256()
    files = _sources() + sorted(glob.glob(os.path.join(CSRC, "*.cuh")))
    files.append(os.path.join(PKG_DIR, "..", "include", "b200audio.h"))
    for f in files:
        with open(f, "rb") as fh:
            h.update(os.path.basename(f).encode())
            h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def is_fresh() -> bool:
    if not (os.path.exists(LIB_PATH) and os.path.exists(STAMP)):
        return False
    if not os.path.isdir(CSRC):  # sources not shipped: trust the binary
        return True
    with open(STAMP) as fh:
        return fh.read().strip() == _digest()


def _compile_one(nvcc: str, src: str, log_dir: str) -> str:
    obj = os.path.join(OBJ_DIR, os.path.basename(src)[:-3] + ".o")
    cmd = [nvcc, *NVCC_FLAGS, "-c", src, "-o", obj]
    proc = subprocess.run(cmd, capture_output=True, text=True)
    with open(os.path.join(log_dir, os.path.basename(src) + ".log"), "w") as fh:
        fh.write(" ".join(cmd) + "\n" + proc.stdout + proc.stderr)
    if proc.returncode != 0:
        raise RuntimeError(f"nvcc failed on {src}:\n{proc.stdout}\n{proc.stderr}")
    return obj


def build(force: bool = False, verbose: bool = True) -> str:
    """Compile if sources changed; returns the path of the shared object."""
    if not force and is_fresh():
        return LIB_PATH
    nvcc = _nvcc()
    os.makedirs(LIB_DIR, exist_ok=True)
    os.makedirs(OBJ_DIR, exist_ok=True)
    srcs = _sources()
    if verbose:
        print(f"[audio_b200] nvcc sm_90a build of {len(srcs)} files -> {LIB_PATH}", file=sys.stderr)
    with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as pool:
        objs = list(pool.map(lambda s: _compile_one(nvcc, s, OBJ_DIR), srcs))
    link = [nvcc, *GENCODE, "-shared", "-o", LIB_PATH, *objs]
    proc = subprocess.run(link, capture_output=True, text=True)
    if proc.returncode != 0:
        raise RuntimeError(f"link failed:\n{proc.stdout}\n{proc.stderr}")
    with open(STAMP, "w") as fh:
        fh.write(_digest())
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
