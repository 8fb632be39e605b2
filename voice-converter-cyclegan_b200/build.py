"""Build libcgvc.so (sm_90a only) in-tree with nvcc.  Used by __graft_entry__.build() and on first import."""
from __future__ import annotations

import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libcgvc.so")
SOURCES = ["engine.cu", "simt_kernels.cu", "tc_gemm.cu"]
HEADERS = ["kernels.cuh", "tc_gemm.cuh", "wgmma.cuh", "geom.h", os.path.join("..", "..", "include", "cgvc.h")]


def _nvcc():
    for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found: libcgvc.so cannot be built")


def is_stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES] + [os.path.normpath(os.path.join(CSRC, h)) for h in HEADERS]
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force=False, verbose=False):
    """Compile into a per-process temporary file under an exclusive file lock, then rename: N ranks importing at once (torchrun)
    neither run nvcc concurrently nor ever see a partially written library."""
    if not force and not is_stale():
        return LIB
    import fcntl
    with open(LIB + ".lock", "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if not force and not is_stale():          # another rank built it while we waited
                return LIB
            tmp = "%s.tmp.%d" % (LIB, os.getpid())
            cmd = [_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "--threads", "3",
                   "-Xcompiler", "-fPIC", "-shared", "-o", tmp] + [os.path.join(CSRC, s) for s in SOURCES] + ["-lcudart", "-ldl"]
            if verbose:
                cmd.insert(1, "-Xptxas"); cmd.insert(2, "-v")
            r = subprocess.run(cmd, capture_output=True, text=True)
            if r.returncode != 0:
                if os.path.exists(tmp):
                    os.remove(tmp)
                raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
            os.replace(tmp, LIB)
            if verbose:
                print(r.stderr)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)
    return LIB


if __name__ == "__main__":
    print(build(force=True, verbose=True))
