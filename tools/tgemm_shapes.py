"""Times the tf32 wgmma GEMM on the shapes of the training step (config 3), with the tile width and split-K count
tgemm_launch picks for each shape: python tools/tgemm_shapes.py"""
import sys

import torch

sys.path.insert(0, ".")
from fullsubnet_b200 import _lib

lib = _lib.load()
dev = torch.device("cuda:0")
st = torch.cuda.current_stream().cuda_stream
scratch = torch.empty(16 << 20, device=dev)


def run(name, M, N, K, split, reps=20):
    A, B, C = torch.randn(M, K, device=dev), torch.randn(N, K, device=dev), torch.empty(M, N, device=dev)

    def call():
        _lib.check(lib.fsn_debug_tgemm(A.data_ptr(), K, B.data_ptr(), K, C.data_ptr(), N, M, N, K, 0,
                                       scratch.data_ptr() if split else None, scratch.numel() if split else 0, st))
    call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
    e0.record()
    for _ in range(reps):
        call()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) / reps * 1e3
    byt = 4.0 * (M * K + N * K + M * N)
    print(f"{name:34s} M={M:7d} N={N:5d} K={K:5d} split={int(split)}: {us:9.1f} us  {2.0 * M * N * K / us / 1e6:7.1f} TFLOP/s  "
          f"{byt / us / 1e3:7.1f} GB/s", flush=True)


run("hoisted sb L1 (1/8 of the rows)", 195200, 1536, 384, False, 5)
run("hoisted sb L0 (1/8 of the rows)", 195200, 1536, 32, False, 5)
run("sb fwd step", 8192, 1536, 384, False)
run("sb bwd dh / dx step", 8192, 384, 1536, False)
run("sb bwd dx L0 step", 8192, 32, 1536, False)
run("fb fwd step", 64, 2048, 512, False)
run("fb fwd step", 64, 2048, 512, True)
run("fb bwd step", 64, 512, 2048, False)
run("fb bwd step", 64, 512, 2048, True)
