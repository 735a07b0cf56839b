"""Checks the tf32 wgmma GEMM (fsn_debug_tgemm) against an exact tf32-truncated reference and times it."""
import ctypes as C
import sys

import torch

sys.path.insert(0, ".")
from fullsubnet_b200 import _lib

lib = _lib.load()
dev = torch.device("cuda:0")


def trunc_tf32(x):
    return (x.view(torch.int32) & ~0x1FFF).view(torch.float32)


def run(M, N, K, lda=None, ldb=None, ldc=None, acc=False, split=False, check=True, reps=0):
    lda, ldb, ldc = lda or K, ldb or K, ldc or N
    g = torch.Generator(device="cpu").manual_seed(M * 7 + N * 3 + K)
    A = torch.randn(M, lda, generator=g).to(dev)
    B = torch.randn(N, ldb, generator=g).to(dev)
    C0 = torch.randn(M, ldc, generator=g).to(dev)
    Cc = C0.clone()
    scratch = torch.empty(16 << 20, device=dev) if split else None
    st = torch.cuda.current_stream().cuda_stream

    def call():
        _lib.check(lib.fsn_debug_tgemm(A.data_ptr(), lda, B.data_ptr(), ldb, Cc.data_ptr(), ldc, M, N, K, int(acc),
                                       scratch.data_ptr() if split else None, scratch.numel() if split else 0, st))
    call()
    torch.cuda.synchronize()
    msg = f"M={M} N={N} K={K} lda={lda} ldb={ldb} ldc={ldc} acc={acc} split={split}: "
    if check:
        ref = trunc_tf32(A[:, :K]).double() @ trunc_tf32(B[:, :K]).double().T
        if acc:
            ref = ref + C0[:, :N].double()
        got = Cc[:, :N].double()
        err = (got - ref).abs().max().item() / ref.abs().max().item()
        full = (A[:, :K].double() @ B[:, :K].double().T + (C0[:, :N].double() if acc else 0))
        err32 = (got - full).abs().max().item() / full.abs().max().item()
        pad_ok = torch.equal(Cc[:, N:], C0[:, N:])
        msg += f"err vs tf32-trunc {err:.2e}, vs fp64 {err32:.2e}, untouched padding {pad_ok}"
    if reps:
        e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
        e0.record()
        for _ in range(reps):
            call()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        msg += f"  {ms * 1e3:.1f} us  {2.0 * M * N * K / ms / 1e9:.1f} TFLOP/s"
    print(msg, flush=True)


run(128, 128, 32)
run(128, 128, 64)
run(128, 256, 256)
run(200, 130, 100, lda=104, ldb=104, ldc=136)
run(256, 384, 1536, acc=True)
run(300, 512, 70, lda=72, ldb=72)
run(1536, 384, 100000, split=True)
run(1536, 384, 100000, split=True, acc=True)
run(8192, 1536, 384, reps=10)
run(8192, 1536, 768, reps=10)
run(8192, 384, 1536, reps=10)
run(8192, 32, 1536, lda=1536, reps=10)
run(1536, 384, 1556480, split=True, check=False, reps=2)
run(262144, 1536, 384, check=False, reps=2)
