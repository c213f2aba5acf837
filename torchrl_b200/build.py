"""Build libtorchrl_b200.so in-tree with nvcc for sm_90a (H100; no torch headers, plain C ABI).

    python -m torchrl_b200.build          # incremental
    python -m torchrl_b200.build --force

The shared object lands in torchrl_b200/lib/ (git-ignored).
nvcc cross-compiles without a GPU; nothing here needs one.
"""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
HEADER = os.path.join(os.path.dirname(HERE), "include", "torchrl_b200.h")     # included by csrc/common.cuh
LIBDIR = os.path.join(HERE, "lib")
OBJDIR = os.path.join(LIBDIR, "obj")
LIBNAME = "libtorchrl_b200.so"
LIBPATH = os.path.join(LIBDIR, LIBNAME)

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + [
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest(path, extra):
    h = hashlib.sha1()
    h.update(" ".join(NVCC_FLAGS).encode())
    with open(path, "rb") as f:
        h.update(f.read())
    for e in extra:
        with open(e, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def build(force=False, verbose=False):
    os.makedirs(OBJDIR, exist_ok=True)
    headers = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))) + [HEADER]
    nvcc = _nvcc()
    jobs = []
    objs = []
    for src in sources():
        base = os.path.splitext(os.path.basename(src))[0]
        obj = os.path.join(OBJDIR, base + ".o")
        stamp = obj + ".sha1"
        dig = _digest(src, headers)
        objs.append(obj)
        if not force and os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == dig:
            continue
        jobs.append((src, obj, stamp, dig))

    def compile_one(job):
        src, obj, stamp, dig = job
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
        if verbose:
            sys.stderr.write(r.stderr)
        with open(stamp, "w") as f:
            f.write(dig)
        return src

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(compile_one, jobs))
    if jobs or force or not os.path.exists(LIBPATH):
        cmd = [nvcc, "-shared", "-o", LIBPATH] + objs + ARCH + ["-Xcompiler", "-fPIC"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    return LIBPATH


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(p)
