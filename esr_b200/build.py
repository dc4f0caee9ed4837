"""In-tree build of libesr_b200.so (hand-written sm_90a CUDA + the C ABI of include/esr_b200.h).

    python -m esr_b200.build [--force]

nvcc cross-compiles without a GPU.  Objects go to esr_b200/csrc/_obj/, the library to
esr_b200/libesr_b200.so (both git-ignored build products).
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
OBJ = os.path.join(CSRC, "_obj")
LIB = os.path.join(PKG, "libesr_b200.so")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
CFLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
          "-Xptxas", "-v", "-Wno-deprecated-gpu-targets"]


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _headers_mtime():
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hs.append(os.path.join(os.path.dirname(PKG), "include", "esr_b200.h"))
    return max(os.path.getmtime(h) for h in hs)


def _compile(src, force, hdr_mtime):
    obj = os.path.join(OBJ, src[:-3] + ".o")
    spath = os.path.join(CSRC, src)
    if not force and os.path.exists(obj) and os.path.getmtime(obj) >= max(os.path.getmtime(spath), hdr_mtime):
        return obj, ""
    cmd = [NVCC, *ARCH, *CFLAGS, "-c", spath, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed on {src}:\n{r.stdout}\n{r.stderr}")
    return obj, r.stderr


def _flags_stamp():
    return " ".join([NVCC, *ARCH, *CFLAGS]) + "\n"


def build(force=False, verbose=False):
    os.makedirs(OBJ, exist_ok=True)
    # objects (and the library) made with another compiler, architecture or flags are stale whatever their mtimes say
    stamp = os.path.join(OBJ, "flags.txt")
    if not os.path.exists(stamp) or open(stamp).read() != _flags_stamp():
        force = True
    hdr = _headers_mtime()
    with ThreadPoolExecutor(max_workers=8) as ex:
        res = list(ex.map(lambda s: _compile(s, force, hdr), _sources()))
    objs = [o for o, _ in res]
    if verbose:
        for _, log in res:
            if log:
                print(log)
    newest = max(os.path.getmtime(o) for o in objs)
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < newest:
        cmd = [NVCC, *ARCH, "-shared", "-Xcompiler", "-fPIC", "-o", LIB, *objs, "-cudart", "static"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    with open(stamp, "w") as f:
        f.write(_flags_stamp())
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
