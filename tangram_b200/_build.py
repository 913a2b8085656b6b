"""Builds the sm_90a (H100) C-ABI library in-tree (tangram_b200/libtangram_b200.so) with nvcc.

nvcc cross-compiles without a GPU; the built library is git-ignored."""
import hashlib
import os
import shutil
import subprocess

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
LIB = os.path.join(PKG, "libtangram_b200.so")
STAMP = LIB + ".stamp"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC,-fvisibility=hidden", "-shared",
]


def _sources():
    out = [os.path.join(PKG, "..", "include", "tangram_b200.h")]
    for f in sorted(os.listdir(CSRC)):
        if f.endswith((".cu", ".cuh", ".h")):
            out.append(os.path.join(CSRC, f))
    return out


def _digest():
    h = hashlib.sha256()
    for p in _sources():
        with open(p, "rb") as f:
            h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def find_nvcc():
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    return None


def is_current():
    try:
        with open(STAMP) as f:
            return os.path.exists(LIB) and f.read().strip() == _digest()
    except OSError:
        return False


def build(force=False, verbose=False):
    """Compile csrc/tangram_b200.cu -> libtangram_b200.so (no-op when up to date).  Safe when several processes (the ranks of a
    torchrun launch) find a stale library at the same time: one builds under a file lock into a temporary file that is
    renamed into place, the others wait and then see the fresh stamp."""
    if not force and is_current():
        return LIB
    nvcc = find_nvcc()
    if nvcc is None:
        raise RuntimeError("nvcc not found: cannot build tangram_b200's CUDA library")
    import fcntl
    with open(LIB + ".lock", "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if not force and is_current():        # another process built it while we waited
                return LIB
            tmp = f"{LIB}.{os.getpid()}.tmp"
            cmd = [nvcc] + NVCC_FLAGS + ["-o", tmp, os.path.join(CSRC, "tangram_b200.cu"), "-ldl"]
            if verbose:
                cmd += ["-Xptxas", "-v"]
            res = subprocess.run(cmd, capture_output=True, text=True)
            if res.returncode != 0:
                if os.path.exists(tmp):
                    os.remove(tmp)
                raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
            if verbose:
                print(res.stderr)
            os.replace(tmp, LIB)
            with open(STAMP, "w") as f:
                f.write(_digest())
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)
    return LIB
