"""Builds occformer_b200/csrc/libocc_b200.so (sm_90a, H100) in-tree with nvcc.

    python -m occformer_b200.build [--force]

The .so and the object files are build products (git-ignored); nvcc cross-compiles without a GPU.  No torch headers are involved: the library is a plain C-ABI shared object
(include/occ_b200.h) loaded through ctypes.
"""
import concurrent.futures
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(CSRC, "libocc_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ARCH + ["-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
         "--expt-relaxed-constexpr"]


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def headers():
    """paths of the headers every source may include: csrc's own and the C ABI header"""
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cuh") or f.endswith(".h")) + [
        os.path.join(os.path.dirname(HERE), "include", "occ_b200.h")]


def _mtime(p):
    return os.path.getmtime(p) if os.path.exists(p) else 0.0


def needs_build():
    newest = max(_mtime(p) for p in [os.path.join(CSRC, f) for f in sources()] + headers())
    return _mtime(LIB) < newest


def _compile(src):
    obj = os.path.join(CSRC, "build", src[:-3] + ".o")
    hdr_m = max([_mtime(h) for h in headers()] + [0.0])
    if _mtime(obj) >= max(_mtime(os.path.join(CSRC, src)), hdr_m):
        return obj, ""
    cmd = [NVCC] + FLAGS + ["-c", os.path.join(CSRC, src), "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
    return obj, r.stderr


def build_library(force=False, verbose=True):
    if not force and not needs_build():
        return LIB
    if not os.path.exists(NVCC):
        raise RuntimeError(f"nvcc not found at {NVCC}; cannot build {LIB}")
    os.makedirs(os.path.join(CSRC, "build"), exist_ok=True)
    with concurrent.futures.ThreadPoolExecutor(max_workers=8) as ex:
        results = list(ex.map(_compile, sources()))
    objs = [o for o, _ in results]
    tmp = LIB + ".tmp"  # link next to the target, then rename: a concurrent reader never sees a half-written library
    cmd = [NVCC, "-shared", "-o", tmp] + objs + ARCH
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    os.replace(tmp, LIB)
    if verbose:
        print(f"built {LIB} from {len(objs)} objects", file=sys.stderr)
    return LIB


if __name__ == "__main__":
    build_library(force="--force" in sys.argv)
