"""In-tree build of libvidtok_b200.so (nvcc, sm_90a only: the kernels use wgmma, TMA and setmaxnreg).  No JIT cache: the
.so sits next to this file, so the package imports from the repository tree."""
from __future__ import annotations

import os
import re
import shutil
import subprocess
from concurrent.futures import ThreadPoolExecutor

try:
    from . import sass
except ImportError:   # run as a script: python vidtok_b200/build.py
    import sass

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libvidtok_b200.so")
SOURCES = ["conv_simt.cu", "conv_tc.cu", "conv_stem.cu", "tblock_tc.cu", "attn_tc.cu", "elementwise.cu", "fsq_aux.cu", "video_io.cu", "metrics.cu", "lpips.cu", "model.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-Xptxas", "-v",
]
# ptxas's "Potential Performance Loss" notes of the C751x family: it had to wait for every wgmma.mma_async before issuing
# the next one, so a kernel's main loop runs with a single MMA in flight.  That costs tensor-pipe throughput without
# changing any result, so nothing else would notice it: the build refuses it instead.
_WGMMA_SERIALIZED = re.compile(r"\((C75\d\d)\) Potential Performance Loss: wgmma\.mma_async instructions are serialized (.*?)"
                               r"(?: in| for) the function '([^']+)'")


def _serialized_wgmma(ptxas_log: str) -> list:
    hits = _WGMMA_SERIALIZED.findall(ptxas_log)
    names = sass.demangle(h[2] for h in hits)
    return [f"{name}: {code} serialized {why.strip()}" for (code, why, _), name in zip(hits, names)]


def _nvcc() -> str:
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def _newest(paths) -> float:
    return max(os.path.getmtime(p) for p in paths)


def build(force: bool = False, verbose: bool = False) -> str:
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    headers.append(os.path.join(os.path.dirname(HERE), "include", "vidtok_b200.h"))
    srcs = [os.path.join(CSRC, s) for s in SOURCES]
    if not force and os.path.exists(LIB) and os.path.getmtime(LIB) >= _newest(srcs + headers):
        return LIB
    os.makedirs(OBJ, exist_ok=True)
    nvcc = _nvcc()

    def compile_one(src):
        obj = os.path.join(OBJ, os.path.basename(src).replace(".cu", ".o"))
        if not force and os.path.exists(obj) and os.path.getmtime(obj) >= _newest([src] + headers):
            return obj
        cmd = [nvcc] + NVCC_FLAGS + ["-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose and r.stderr:
            print(r.stderr)
        bad = _serialized_wgmma(r.stderr)
        if bad:
            os.remove(obj)   # an object that was refused must not pass the next build's freshness check
            serialized.extend(f"{os.path.basename(src)}: {b}" for b in bad)
        return obj

    serialized = []
    with ThreadPoolExecutor(max_workers=len(srcs)) as ex:
        objs = list(ex.map(compile_one, srcs))
    if serialized:
        raise RuntimeError("ptxas serialized the wgmma pipeline of:\n  " + "\n  ".join(serialized))
    cmd = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB] + objs
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in os.sys.argv, verbose=True))
