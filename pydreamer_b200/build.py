"""In-tree nvcc build of libpd_b200.so (sm_90a only).

The shared object is written next to this file, inside the package, so that an in-tree checkout is
importable after one build.  nvcc cross-compiles without a GPU, so this also runs on a CPU-only machine.
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libpd_b200.so")
STAMP = os.path.join(HERE, ".libpd_b200.stamp")
SOURCES = ["pd_api.cu", "pd_gemm_sm90.cu", "pd_gemm_skinny.cu", "pd_gemm_simt.cu", "pd_rowwise.cu", "pd_conv.cu", "pd_misc.cu",
           "pd_rssm_fwd3.cu", "pd_rssm_bptt.cu", "pd_grid.cu"]
HEADERS = [os.path.join(CSRC, "pd_common.cuh"), os.path.join(CSRC, "pd_k1_pipe.cuh"), os.path.join(HERE, "..", "include", "pd_b200.h")]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared",
]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _digest():
    h = hashlib.sha256()
    for p in [os.path.join(CSRC, s) for s in SOURCES] + HEADERS:
        with open(p, "rb") as f:
            h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    """Compile libpd_b200.so if sources changed. Returns the library path."""
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(STAMP):
        with open(STAMP) as f:
            if f.read().strip() == dig:
                return LIB
    cmd = [_nvcc()] + NVCC_FLAGS + [os.path.join(CSRC, s) for s in SOURCES] + ["-o", LIB]
    if verbose:
        print(" ".join(cmd), file=sys.stderr)
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    with open(STAMP, "w") as f:
        f.write(dig)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
