"""In-tree build of the C-ABI shared library (nvcc cross-compiles sm_90a without a GPU).

    python -m litepose_b200.build [--force] [--verbose]

Produces litepose_b200/_C/liblitepose_b200.so (git-ignored, travels to the GPU box).
"""
import concurrent.futures
import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT_DIR = os.path.join(HERE, "_C")
LIB = os.path.join(OUT_DIR, "liblitepose_b200.so")
INCLUDE = os.path.join(os.path.dirname(HERE), "include")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "-Xptxas", "-v",
]


def _nvcc():
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def _sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest():
    h = hashlib.sha256()
    files = _sources() + [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith(".cuh")]
    files += [os.path.join(INCLUDE, f) for f in sorted(os.listdir(INCLUDE)) if f.endswith(".h")]
    for f in files:
        h.update(f.encode())
        with open(f, "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    os.makedirs(OUT_DIR, exist_ok=True)
    stamp = os.path.join(OUT_DIR, "build.stamp")
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == dig:
        return LIB
    nvcc = _nvcc()
    objs = []

    def compile_one(src):
        obj = os.path.join(OUT_DIR, os.path.basename(src)[:-3] + ".o")
        cmd = [nvcc] + NVCC_FLAGS + ["-I", INCLUDE, "-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        return src, obj, r

    with concurrent.futures.ThreadPoolExecutor(max_workers=8) as ex:
        for src, obj, r in ex.map(compile_one, _sources()):
            if verbose or r.returncode != 0:
                sys.stderr.write("== %s\n%s%s\n" % (os.path.basename(src), r.stdout, r.stderr))
            if r.returncode != 0:
                raise RuntimeError("nvcc failed for %s" % src)
            with open(obj + ".log", "w") as fh:
                fh.write(r.stdout + r.stderr)
            objs.append(obj)
    cmd = [nvcc, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("link failed")
    with open(stamp, "w") as fh:
        fh.write(dig)
    return LIB


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(path)
