"""The two-pass sub-band stack of the whole-clip fullsubnet enhance (`sb_l0_tc_kernel` then `sb_l1_tc_kernel`,
fsn_subband_tc.cu, 48 rows per CTA pair, h0 through global memory) through its unit-test hook `fsn_debug_sb_lstm_tc2`,
against the fused kernel `sb_lstm_tc_kernel` through `fsn_debug_sb_lstm_tc` on the same inputs.

The two paths issue the same MMAs in the same k and part order per (gate, unit, row), with m64n48k16 instead of
m64n32k16, and apply the same cell and Linear arithmetic, so they must agree bit for bit: the chunked stream stays on
the fused kernel's carry variant and is compared bit for bit with the whole-clip call.  The cases cover H = 128 / 256 /
384, both arithmetics, partial, exact and multi-wave grids, one and several row chunks, drop_band, per-(step, row)
scales and every output activation.  test_gpu_subband_tc.py checks the fused kernel against float64."""
import ctypes as C

import numpy as np
import pytest
import torch

import test_gpu_subband_tc as T

GUARD = 256


def _case(name, **kw):
    c = dict(name=name, H=384, B=1, F=33, G=1, steps=10, la=2, Ns=15, Nf=0, act=0, unit=False, weights="std",
             chunk=0, stages=0)
    c.update(kw)
    c["src_T"], c["shrink"], c["fc_out"] = c["steps"], 1, 2
    return pytest.param(c, id=name)


CASES = [
    # 48 rows (3 clips x 16 bins with G = 2): exactly one pair; 17 steps, Linear gain 200 with ReLU6
    _case("h384_exact_g2", H=384, B=3, F=33, G=2, steps=17, la=2, act=3, weights="gain"),
    # 13 rows: one partial pair; H = 128 (one warpgroup), saturated gates, ReLU, ring depth 2
    _case("h128_partial", H=128, B=1, F=13, steps=9, la=0, Ns=3, act=1, weights="saturated", stages=2),
    # 50 rows (G = 3 with B = 5) in chunks of one pair; full-band neighbours, per-(step, row) scales, Tanh
    _case("h256_chunks_unit", H=256, B=5, F=31, G=3, steps=8, la=0, Ns=7, Nf=2, act=2, unit=True, chunk=1),
    # 6168 rows = 129 pairs, one chunk: more pairs than the GPU holds at once
    _case("h384_waves", H=384, B=24, F=257, steps=3, la=2, Ns=13, Nf=1, act=0, weights="gain"),
    # the same rows in three chunks of 50 pairs (the last one partial), ring depth 3
    _case("h384_waves_chunks", H=384, B=24, F=257, steps=3, la=2, Ns=13, Nf=1, act=2, chunk=50, stages=3),
    # H = 384, per-(step, row) scales, G = 3 with B = 4 (20 rows), saturated gates, ReLU
    _case("h384_unit_g3", H=384, B=4, F=17, G=3, steps=10, la=2, Ns=15, act=1, unit=True, weights="saturated"),
    # 16 rows, Ksb = 2, a single step
    _case("h128_ksb2", H=128, B=4, F=9, G=2, steps=1, la=0, Ns=0, act=0),
]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _two_pass(dev, c, wd, d_in, x3):
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    magT, fbT, inv2, unit = d_in
    s = _lib.SeqWeights()
    for l in range(2):
        s.w_ih[l], s.w_hh[l] = wd[f"weight_ih_l{l}"].data_ptr(), wd[f"weight_hh_l{l}"].data_ptr()
        s.b_ih[l], s.b_hh[l] = wd[f"bias_ih_l{l}"].data_ptr(), wd[f"bias_hh_l{l}"].data_ptr()
    s.fc_w, s.fc_b = wd["fc_w"].data_ptr(), wd["fc_b"].data_ptr()
    packed = torch.empty(lib.fsn_debug_sb_lstm_tc_packed_bytes(c["H"], x3), dtype=torch.uint8, device=dev)
    _, Fsub, _, _ = T._row_map(c["B"], c["F"], c["G"])
    R = c["B"] * Fsub
    ws = torch.empty(lib.fsn_debug_sb_lstm_tc2_ws_bytes(R, c["steps"], c["H"], x3, c["chunk"]), dtype=torch.uint8,
                     device=dev)
    assert ws.numel() > 0
    shape = (c["B"], 2, Fsub, c["steps"] - c["la"])
    n = int(np.prod(shape))
    buf = torch.full((n + 2 * GUARD,), float("nan"), device=dev)
    _lib.check(lib.fsn_debug_sb_lstm_tc2(
        C.byref(s), c["H"], c["Ns"], c["Nf"], c["act"], x3, magT.data_ptr(), fbT.data_ptr(), c["B"], c["F"],
        c["src_T"], c["G"], inv2.data_ptr(), None if unit is None else unit.data_ptr(), c["la"], c["steps"],
        c["stages"], c["chunk"], packed.data_ptr(), ws.data_ptr(), buf[GUARD:].data_ptr(),
        torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    buf = buf.cpu()
    assert torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[GUARD + n:]).all(), (x3, "write outside crm")
    return buf[GUARD:GUARD + n].view(shape)


@pytest.mark.gpu
@pytest.mark.parametrize("x3", [1, 0], ids=["x3", "single"])
@pytest.mark.parametrize("c", CASES)
def test_two_pass_matches_fused_kernel_bits(dev, c, x3):
    Ksb = (2 * c["Ns"] + 1) + (2 * c["Nf"] + 1)
    seed = sum(map(ord, c["name"]))
    w = T._weights(c["H"], Ksb, 2, c["weights"], seed)
    wd = {k: v.to(dev).contiguous() for k, v in w.items()}
    magT, fbT, inv2, unit, _ = T._inputs(c, seed + 1)
    d_in = tuple(None if v is None else v.to(dev).contiguous() for v in (magT, fbT, inv2, unit))
    fused = T._launch(dev, c, wd, d_in, x3, 0, 0)
    two = _two_pass(dev, c, wd, d_in, x3)
    assert not torch.isnan(two).any(), f"{int(torch.isnan(two).sum())} crm elements never written"
    diff = (two - fused).abs().max().item()
    nbits = int((two.view(torch.int32) != fused.view(torch.int32)).sum())
    assert nbits == 0, f"{nbits} elements differ from the fused kernel (max |diff| {diff:.3e})"
