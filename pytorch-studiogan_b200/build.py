"""Build libsgb200.so in-tree with nvcc for sm_90a (H100).

Usage: python pytorch-studiogan_b200/build.py [--force]
The shared library lands in pytorch-studiogan_b200/sgb200/lib/libsgb200.so (git-ignored build product).
"""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIBDIR = os.path.join(HERE, "sgb200", "lib")
LIB = os.path.join(LIBDIR, "libsgb200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
         "-Xcompiler", "-fPIC", "-cudart", "static"]


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest(paths):
    h = hashlib.sha256()
    for p in sorted(paths):
        with open(p, "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def _compile(src):
    obj = os.path.join(OBJ, src[:-3] + ".o")
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    deps += [os.path.join(CSRC, src), os.path.join(HERE, "..", "include", "sgb200.h")]
    stamp = obj + ".sha"
    dig = _digest(deps)
    if os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == dig:
        return obj
    cmd = [NVCC] + FLAGS + ["-c", os.path.join(CSRC, src), "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
    with open(stamp, "w") as fh:
        fh.write(dig)
    return obj


def build(force=False):
    os.makedirs(OBJ, exist_ok=True)
    os.makedirs(LIBDIR, exist_ok=True)
    if force:
        for f in os.listdir(OBJ):
            if f.endswith(".sha"):
                os.remove(os.path.join(OBJ, f))
    srcs = _sources()
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(_compile, srcs))
    newest = max(os.path.getmtime(o) for o in objs)
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < newest:
        tmp = os.path.join(OBJ, "libsgb200.so.link")          # link aside, then rename: the in-tree library is replaced atomically
        cmd = [NVCC, "-shared", "-cudart", "static", "-o", tmp] + objs
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
        os.replace(tmp, LIB)
    return LIB


if __name__ == "__main__":
    lib = build(force="--force" in sys.argv)
    print(lib)
