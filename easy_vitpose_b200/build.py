"""Builds csrc/libvitpose_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU)."""
from __future__ import annotations

import fcntl
import os
import shutil
import subprocess
import tempfile

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc")
LIB = os.path.join(CSRC, "libvitpose_b200.so")
SOURCES = ["engine.cu"]
HEADERS = ["ptx.cuh", "wgmma.cuh", "gemm.cuh", "expert_gemm.cuh", "chain.cuh", "attention.cuh", "qkv_attention.cuh", "simple_head.cuh", "pointwise.cuh", "decode.cuh", "draw.cuh", "track.cuh", "smooth.cuh", "oks_nms.cuh", "pairwise.cuh", "coco_eval.cuh", "preprocess.cuh",
           os.path.join("..", "..", "include", "vitpose_b200.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "--shared", "-Xcompiler", "-fPIC"]


def _nvcc() -> str:
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found; libvitpose_b200.so cannot be built")
    return exe


def is_stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(os.path.join(CSRC, f)) > t for f in SOURCES + HEADERS)


def build(force: bool = False, verbose: bool = False) -> str:
    """Compiles the library if it is missing or older than its sources.  Safe under torch.distributed.run, where every
    rank imports the package at once: an exclusive file lock serialises the ranks (the first one builds, the others find
    a fresh library when they get the lock), and nvcc writes to a temporary file that is renamed into place, so no
    process can ever dlopen a half-written .so."""
    if not force and not is_stale():
        return LIB
    with open(os.path.join(CSRC, ".build.lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if not force and not is_stale():          # another process built it while we waited
                return LIB
            fd, tmp = tempfile.mkstemp(prefix=".libvitpose_b200.", suffix=".so.tmp", dir=CSRC)
            os.close(fd)
            try:
                cmd = [_nvcc(), *NVCC_FLAGS, "-o", tmp, *SOURCES]
                if verbose:
                    cmd.insert(1, "-Xptxas=-v")
                res = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
                if res.returncode != 0:
                    raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
                os.chmod(tmp, 0o755)
                os.replace(tmp, LIB)                   # atomic on one filesystem
            finally:
                if os.path.exists(tmp):
                    os.unlink(tmp)
            if verbose:
                print(res.stderr)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)
    return LIB


if __name__ == "__main__":
    print(build(force=True, verbose=True))
