"""Build libpnx.so (the C-ABI CUDA library, include/pnx.h) in-tree with nvcc for sm_90a (H100).

`python -m pillarnext_b200.build` or `__graft_entry__.build()`.  Cross-compiles without a GPU.
"""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libpnx.so")
OBJ = os.path.join(HERE, "build")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ARCH + ["-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC"]
# det_eval.cu's and track.cu's kernels must equal their host twins to the bit, so no multiply-add is contracted there
FILE_FLAGS = {"det_eval.cu": ["-fmad=false"], "track.cu": ["-fmad=false"]}


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest():
    h = hashlib.sha256()
    for f in sorted(os.listdir(CSRC)):
        with open(os.path.join(CSRC, f), "rb") as fh:
            h.update(f.encode())
            h.update(fh.read())
    h.update(" ".join(FLAGS).encode())
    h.update(repr(sorted(FILE_FLAGS.items())).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    stamp = os.path.join(OBJ, "stamp")
    dig = _digest()
    if not force and os.path.exists(OUT) and os.path.exists(stamp) and open(stamp).read() == dig:
        return OUT
    if not os.path.exists(NVCC):
        raise RuntimeError("nvcc not found at %s and libpnx.so is stale/missing" % NVCC)

    def one(src):
        obj = os.path.join(OBJ, src[:-3] + ".o")
        cmd = [NVCC] + FLAGS + FILE_FLAGS.get(src, []) + ["-c", os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
        if verbose and r.stderr:
            print(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        objs = list(ex.map(one, _sources()))
    cmd = [NVCC, "-shared", "-o", OUT] + objs + ARCH + ["-cudart", "static"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    with open(stamp, "w") as fh:
        fh.write(dig)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
