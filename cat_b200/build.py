"""In-tree build of the native library (nvcc, sm_90a only).

The product has exactly one native artefact, ``cat_b200/libctc_crf_b200.so`` (CUDA kernels + C ABI,
no torch dependency).  It is built in-tree so the file travels to the GPU box with the repository
snapshot; nothing is JIT-compiled at import time.
"""
from __future__ import annotations

import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libctc_crf_b200.so")
SOURCES = ["api.cu", "den_kernels.cu", "den_sample.cu", "beam_search.cu", "ctc_kernels.cu", "den_graph.cc", "ngram.cc", "wfst_decode.cu", "wfst.cc", "rnnt_kernels.cu", "rnnt_decode.cu", "ctct_decode.cu", "ngram_score.cu"]
HEADERS = ["common.cuh", "beam_common.cuh", "transducer_beam.cuh", "den_graph.h", "den_launch.h", "ngram.h", "wfst.h", os.path.join("..", "..", "include", "ctc_crf_b200.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-Xcompiler", "-fPIC", "-shared"]


def _stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS]
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile ``libctc_crf_b200.so`` if missing or out of date; returns its path."""
    if not force and not _stale():
        return LIB
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found: cannot build cat_b200/libctc_crf_b200.so")
    cmd = [nvcc, *NVCC_FLAGS, "-o", LIB + ".tmp", *[os.path.join(CSRC, s) for s in SOURCES]]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    subprocess.check_call(cmd, cwd=CSRC)
    os.replace(LIB + ".tmp", LIB)
    return LIB


if __name__ == "__main__":
    print(build(force=True, verbose=True))
