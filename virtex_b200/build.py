"""In-tree build of libvirtex_b200.so (sm_90a only).

`python -m virtex_b200.build` compiles every `csrc/*.cu` with nvcc (cross-compiles without a GPU) and links
them into `virtex_b200/libvirtex_b200.so`, next to this file, so that the built library travels with the
repository snapshot.  Objects are cached under `build/` and rebuilt when the source or any header changes.
"""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OBJ_DIR = os.path.join(ROOT, "build", "obj")
LIB_PATH = os.path.join(HERE, "libvirtex_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-DVTX_NO_FAST_MATH",  # no --use_fast_math: erff / division accuracy matters for parity
    "-I", os.path.join(ROOT, "include"),
]


def _headers_digest():
    h = hashlib.sha1()
    for d in (CSRC, os.path.join(ROOT, "include")):
        for name in sorted(os.listdir(d)):
            if name.endswith((".cuh", ".h")):
                with open(os.path.join(d, name), "rb") as f:
                    h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def _compile_one(src, hdr_digest, verbose, extra=(), tag=""):
    with open(src, "rb") as f:
        digest = hashlib.sha1(f.read() + hdr_digest.encode() + " ".join(extra).encode()).hexdigest()[:16]
    base = os.path.splitext(os.path.basename(src))[0] + tag
    obj = os.path.join(OBJ_DIR, f"{base}.{digest}.o")
    if not os.path.exists(obj):
        for old in os.listdir(OBJ_DIR):
            if old.startswith(base + ".") and old.endswith(".o"):
                os.remove(os.path.join(OBJ_DIR, old))
        cmd = [NVCC] + NVCC_FLAGS + list(extra) + ["-c", src, "-o", obj]
        if verbose:
            print(" ".join(cmd), flush=True)
        subprocess.run(cmd, check=True)
    return obj


def _link(objs, lib_path, stamp_name, verbose):
    stamp = os.path.join(OBJ_DIR, stamp_name)
    want = "\n".join(objs)
    have = open(stamp).read() if os.path.exists(stamp) else ""
    if want != have or not os.path.exists(lib_path):
        cmd = [NVCC, "-shared", "-o", lib_path] + objs
        if verbose:
            print(" ".join(cmd), flush=True)
        subprocess.run(cmd, check=True)
        with open(stamp, "w") as f:
            f.write(want)


def build(verbose=False, force=False):
    os.makedirs(OBJ_DIR, exist_ok=True)
    srcs = sorted(os.path.join(CSRC, n) for n in os.listdir(CSRC) if n.endswith(".cu"))
    hdr = _headers_digest()
    if force:
        for old in os.listdir(OBJ_DIR):
            os.remove(os.path.join(OBJ_DIR, old))
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(lambda src: _compile_one(src, hdr, verbose), srcs))
    _link(objs, LIB_PATH, "link.stamp", verbose)
    return LIB_PATH


if __name__ == "__main__":
    print(build(verbose=True, force="--force" in sys.argv))
