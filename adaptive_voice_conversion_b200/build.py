"""Build libavc_b200.so (sm_90a, H100) in-tree with nvcc.

    python -m adaptive_voice_conversion_b200.build [--force] [--verbose]

Every .cu under csrc/ is compiled to an object file (in parallel) with
``-gencode arch=compute_90a,code=sm_90a -lineinfo -O3`` and linked into
``adaptive_voice_conversion_b200/libavc_b200.so``.  nvcc cross-compiles, so this works in
a machine without a GPU.

Safe under ``torchrun``: the build takes an exclusive file lock (the other ranks wait, then find the
stamp up to date) and every output is written to a temporary name and renamed into place, so no
process can ever dlopen a half-written library.
"""
from __future__ import annotations

import argparse
import contextlib
import fcntl
import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
OBJ = os.path.join(PKG, "csrc", "_obj")
LIB = os.path.join(PKG, "libavc_b200.so")
VARIANTS = {  # name -> (library, object dir, extra nvcc flags)
    "default": (LIB, OBJ, []),
}
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC"]


def nvcc() -> str:
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found: libavc_b200.so cannot be built")
    return exe


def _digest(paths, extra=()) -> str:
    h = hashlib.sha256()
    for p in sorted(paths):
        with open(p, "rb") as f:
            h.update(os.path.basename(p).encode())  # location independent: the tree moves to the GPU box
            h.update(f.read())
    h.update(" ".join(ARCH + FLAGS + list(extra)).encode())
    return h.hexdigest()


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def headers():
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hs.append(os.path.join(os.path.dirname(PKG), "include", "avc_b200.h"))
    return hs


@contextlib.contextmanager
def _locked(path):
    """Exclusive inter-process lock (all ranks of a torchrun launch share the tree)."""
    with open(path, "a+") as f:
        fcntl.flock(f, fcntl.LOCK_EX)
        try:
            yield
        finally:
            fcntl.flock(f, fcntl.LOCK_UN)


def _write_atomic(path, text):
    tmp = f"{path}.{os.getpid()}.tmp"
    with open(tmp, "w") as f:
        f.write(text)
    os.replace(tmp, path)


def _up_to_date(lib, stamp, dig):
    try:
        return os.path.exists(lib) and open(stamp).read() == dig
    except OSError:
        return False


def build_variant(variant: str, force: bool = False, verbose: bool = False, allow_build: bool = True) -> str:
    lib, objdir, extra = VARIANTS[variant]
    stamp = os.path.join(objdir, "stamp.txt")
    dig = _digest(sources() + headers(), extra)
    if not force and _up_to_date(lib, stamp, dig):
        return lib
    if not allow_build:
        raise RuntimeError(f"{lib} is missing or older than its sources and building was not allowed")
    os.makedirs(objdir, exist_ok=True)
    with _locked(os.path.join(objdir, "build.lock")):
        if not force and _up_to_date(lib, stamp, dig):   # another rank built it while we waited
            return lib
        return _build_locked(lib, objdir, extra, stamp, dig, force, verbose)


def _build_locked(lib, objdir, extra, stamp, dig, force, verbose):
    cc = nvcc()
    hdr_dig = _digest(headers(), extra)

    def compile_one(src):
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + ".o")
        ostamp = obj + ".stamp"
        d = _digest([src], extra) + hdr_dig
        if not force and os.path.exists(obj) and os.path.exists(ostamp) and open(ostamp).read() == d:
            return obj
        tmp = f"{obj}.{os.getpid()}.tmp.o"
        cmd = [cc, *ARCH, *FLAGS, *extra, "-c", src, "-o", tmp]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            sys.stderr.write(r.stderr)
        os.replace(tmp, obj)
        _write_atomic(ostamp, d)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        objs = list(ex.map(compile_one, sources()))
    tmp_lib = f"{lib}.{os.getpid()}.tmp"
    cmd = [cc, *ARCH, "-shared", "-Xcompiler", "-fPIC", "-o", tmp_lib, *objs, "-lcudart"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    os.replace(tmp_lib, lib)     # atomic: a concurrent dlopen sees the old or the new file, never a partial one
    _write_atomic(stamp, dig)
    return lib


def build(force: bool = False, verbose: bool = False, allow_build: bool = True) -> str:
    """Build (or stamp-check) the library; returns its path."""
    for v in VARIANTS:
        build_variant(v, force, verbose, allow_build)
    return LIB


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    ap.add_argument("--verbose", action="store_true")
    a = ap.parse_args()
    print(build(a.force, a.verbose))
