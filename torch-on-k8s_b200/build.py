"""In-tree build of libtok8s.so (sm_90a only) — used by __graft_entry__.build() and the tests.

Objects go to torch-on-k8s_b200/build/, the library to torch-on-k8s_b200/lib/libtok8s.so.  Both are
build products and stay out of git.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(HERE, "build")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libtok8s.so")
INCLUDE = os.path.join(os.path.dirname(HERE), "include")

NVCC = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC,-Wall,-Wno-unused-function",
          "-I", INCLUDE, "-I", CSRC]


def _sources():
    out = []
    for name in sorted(os.listdir(CSRC)):
        if name.endswith((".cu", ".cpp")):
            out.append(os.path.join(CSRC, name))
    return out


def _digest(paths):
    h = hashlib.sha256()
    for p in sorted(paths):
        with open(p, "rb") as f:
            h.update(p.encode())
            h.update(f.read())
    h.update(" ".join(ARCH + COMMON).encode())
    return h.hexdigest()


def _headers():
    hs = [os.path.join(CSRC, n) for n in os.listdir(CSRC) if n.endswith(".h")]
    hs += [os.path.join(INCLUDE, n) for n in os.listdir(INCLUDE) if n.endswith(".h")]
    return hs


def _compile(src, verbose):
    obj = os.path.join(BUILD, os.path.basename(src) + ".o")
    stamp = obj + ".sha"
    want = _digest([src] + _headers())
    if os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == want:
        return obj
    cmd = [NVCC] + ARCH + COMMON
    if src.endswith(".cu"):
        cmd += ["-Xptxas", "-v"] if verbose else []
    else:
        cmd += ["-x", "cu"] if False else []
    cmd += ["-c", src, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("nvcc failed for %s" % src)
    if verbose:
        sys.stderr.write(r.stderr)
    with open(stamp, "w") as f:
        f.write(want)
    return obj


def build_lib(force: bool = False, verbose: bool = False) -> str:
    """Compile every source under csrc/ for sm_90a and link libtok8s.so. Returns its path."""
    os.makedirs(BUILD, exist_ok=True)
    os.makedirs(LIBDIR, exist_ok=True)
    if force:
        for n in os.listdir(BUILD):
            os.remove(os.path.join(BUILD, n))
    srcs = _sources()
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(lambda s: _compile(s, verbose), srcs))
    link_stamp = os.path.join(BUILD, "link.sha")
    want = _digest(objs)
    if (not force and os.path.exists(LIB) and os.path.exists(link_stamp)
            and open(link_stamp).read() == want):
        return LIB
    cmd = [NVCC] + ARCH + ["-shared", "-cudart", "static", "-Xcompiler", "-fPIC", "-o", LIB] + objs
    cmd += ["-lpthread", "-ldl", "-lrt"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("link failed")
    with open(link_stamp, "w") as f:
        f.write(want)
    return LIB


if __name__ == "__main__":
    print(build_lib(force="--force" in sys.argv, verbose="-v" in sys.argv))
