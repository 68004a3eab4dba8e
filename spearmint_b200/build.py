"""In-tree build of libspearmint_b200.so with nvcc for sm_90a (no GPU needed: cross-compiles).

    python -m spearmint_b200.build [--force] [--verbose]

The library has no torch / Python dependency; the Python host binds it with ctypes
(spearmint_b200/_lib.py).  Objects and the .so are build products (git-ignored).
"""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libspearmint_b200.so")
SOURCES = ["cov.cu", "potrf.cu", "potrf_ll.cu", "solve.cu", "predict.cu", "predict_tc.cu", "kxt_tc.cu", "guard.cu", "sobol.cu", "ei.cu", "grad.cu", "constraint.cu",
           "forest.cu", "api.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
         "-Xcompiler", "-fPIC", "-Xptxas", "-v"]


def _sources():
    return [s for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]


def _digest():
    h = hashlib.sha256()
    names = sorted(os.listdir(CSRC)) + ["../../include/spearmint_b200.h"]
    for n in names:
        p = os.path.join(CSRC, n)
        if os.path.isfile(p) and (n.endswith((".cu", ".cuh", ".h"))):
            h.update(n.encode())
            with open(p, "rb") as fh:
                h.update(fh.read())
    h.update(" ".join(FLAGS).encode())
    return h.hexdigest()


def _compile(src, verbose):
    obj = os.path.join(LIBDIR, src.replace(".cu", ".o"))
    cmd = [NVCC] + FLAGS + ["-c", os.path.join(CSRC, src), "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
    if verbose:
        sys.stderr.write(r.stderr)
    return obj, r.stderr


def build(force=False, verbose=False):
    """Compile (if stale) and return the path of the shared library."""
    os.makedirs(LIBDIR, exist_ok=True)
    stamp = os.path.join(LIBDIR, "build.stamp")
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read().strip() == dig:
        return LIB
    # one builder at a time: torchrun ranks that find a stale library would otherwise run nvcc concurrently into the same
    # objects and could load a half-written .so; the others wait here and then find the fresh stamp
    import fcntl
    with open(os.path.join(LIBDIR, ".build.lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            return _build_locked(force, verbose, stamp, dig)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)


def _build_locked(force, verbose, stamp, dig):
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read().strip() == dig:
        return LIB
    if not os.path.exists(NVCC):
        if os.path.exists(LIB):
            return LIB  # GPU box without toolkit mismatch: use the shipped build
        raise RuntimeError("nvcc not found at %s and no prebuilt %s" % (NVCC, LIB))
    srcs = _sources()
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        res = list(ex.map(lambda s: _compile(s, verbose), srcs))
    objs = [o for o, _ in res]
    log = "".join(l for _, l in res)
    with open(os.path.join(LIBDIR, "ptxas.log"), "w") as fh:
        fh.write(log)
    tmp = LIB + ".tmp.%d" % os.getpid()
    cmd = [NVCC, "-shared", "-o", tmp] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    os.replace(tmp, LIB)                      # atomic: a concurrent loader sees the old or the new library, never half of one
    with open(stamp, "w") as fh:
        fh.write(dig)
    return LIB


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(p)
