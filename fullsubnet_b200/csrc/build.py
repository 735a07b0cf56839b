"""Builds libfsn_b200.so in-tree with nvcc for sm_90a (H100) (no torch headers: the library is a
plain C-ABI CUDA library; the Python host binds it with ctypes)."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SOURCES = ["fsn_dsp.cu", "fsn_lstm_simt.cu", "fsn_subband_tc.cu", "fsn_fullband.cu", "fsn_lstm_rec_tc.cu", "fsn_fast_model.cu", "fsn_improved.cu", "fsn_fullband_baseline.cu", "fsn_train.cu", "fsn_fast_train.cu", "fsn_fullband_train.cu", "fsn_improved_train.cu", "fsn_mix.cu", "fsn_stoi.cu", "fsn_resample.cu", "fsn_stream.cu", "fsn_tgemm.cu", "fsn_model.cu"]
LIB = os.path.join(HERE, "libfsn_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = [*ARCH, "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC", "-DFSN_BUILT_ARCH=90", "--use_fast_math=false"]


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(HERE, f) for f in os.listdir(HERE) if f.endswith((".cu", ".cuh"))]
    deps.append(os.path.join(HERE, "..", "..", "include", "fsn_b200.h"))
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    flags = [f for f in FLAGS if not f.startswith("--use_fast_math")] + os.environ.get("FSN_EXTRA_NVCC_FLAGS", "").split()
    objs = []
    procs = []
    for s in SOURCES:
        o = os.path.join(HERE, s.replace(".cu", ".o"))
        cmd = [NVCC, *flags, "-c", os.path.join(HERE, s), "-o", o]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((s, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(o)
    for s, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode:
            print(out)
        if p.returncode:
            raise RuntimeError(f"nvcc failed on {s}")
    subprocess.check_call([NVCC, "-shared", "-o", LIB, *objs, *ARCH])
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
