"""Build libunicorn_b200.so (hand-written sm_90a CUDA + the C ABI) in-tree with nvcc.

No torch extension machinery: the library has a plain C ABI (include/unicorn_b200.h) and is loaded with ctypes.
nvcc cross-compiles without a GPU, so this runs in the CPU-only build container.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libunicorn_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
         "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr"]


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build_lib(force=False, verbose=False):
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    headers.append(os.path.join(HERE, "..", "include", "unicorn_b200.h"))
    objs, jobs = [], []
    for src in _sources():
        obj = os.path.join(HERE, "build", src[:-3] + ".o")
        objs.append(obj)
        if force or _stale(obj, [os.path.join(CSRC, src)] + headers):
            jobs.append([NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", os.path.join(CSRC, src), "-o", obj])

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed: %s\n%s\n%s" % (" ".join(cmd), r.stdout, r.stderr))
        return r.stderr

    with ThreadPoolExecutor(max_workers=8) as ex:
        logs = list(ex.map(run, jobs))
    if verbose:
        for l in logs:
            print(l)
    if jobs or force or _stale(LIB, objs):
        run([NVCC, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a"])
    return LIB


if __name__ == "__main__":
    print(build_lib(force="--force" in sys.argv, verbose="-v" in sys.argv))
