"""Build libmultimae_b200.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

    python -m multimae_b200.build [--force] [--verbose]

nvcc cross-compiles without a GPU.  The .so and the object files are build products (git-ignored).
"""
import argparse
import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "_build")
LIB = os.path.join(HERE, "libmultimae_b200.so")

ARCH = "arch=compute_90a,code=sm_90a"
NVCC_FLAGS = [
    "-gencode", ARCH,
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]


def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _fingerprint(path, extra=""):
    h = hashlib.sha1()
    h.update(extra.encode())
    for dep in [path] + sorted(
        os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))
    ) + [os.path.join(HERE, "..", "include", "multimae_b200.h")]:
        with open(dep, "rb") as fh:
            h.update(fh.read())
    return h.hexdigest()


def _compile_one(args):
    nvcc, src, verbose, force = args
    base = os.path.splitext(os.path.basename(src))[0]
    obj = os.path.join(OBJ, base + ".o")
    stamp = obj + ".sha1"
    fp = _fingerprint(src, " ".join(NVCC_FLAGS))
    if not force and os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == fp:
        return obj, False, ""
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, res.stdout, res.stderr))
    with open(stamp, "w") as fh:
        fh.write(fp)
    return obj, True, res.stderr


def build(force=False, verbose=False):
    """Compile every csrc/*.cu for sm_90a and link libmultimae_b200.so. Returns the library path."""
    os.makedirs(OBJ, exist_ok=True)
    nvcc = _nvcc()
    srcs = _sources()
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as pool:
        results = list(pool.map(_compile_one, [(nvcc, s, verbose, force) for s in srcs]))
    objs = [r[0] for r in results]
    changed = any(r[1] for r in results)
    if verbose:
        for r in results:
            if r[2]:
                sys.stderr.write(r[2])
    if changed or not os.path.exists(LIB):
        cmd = [nvcc, "-shared", "-o", LIB] + objs + ["-gencode", ARCH, "-lcudart_static",
                                                      "-Xlinker", "--no-undefined", "-lpthread", "-ldl", "-lrt"]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (res.stdout, res.stderr))
    return LIB


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    ap.add_argument("--verbose", action="store_true")
    a = ap.parse_args()
    print(build(force=a.force, verbose=a.verbose))
