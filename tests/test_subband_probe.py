"""The cycle-stamp (PROBE) instantiation of the sub-band kernel, fsn_debug_sb_lstm_tc_probe: it checks its arguments
before any CUDA call (CPU), computes the same bits as the production kernel, and its stamps are ordered and cover every
block of the sampled CTAs and iterations (GPU)."""
from __future__ import annotations

import ctypes as C

import pytest
import torch

FIELDS = ["t_begin", "t_mma0", "t_mma1", "t_end", "operand", "turn", "w_full", "wait_group", "group_lat", "stages",
          "cell", "l1_done", "h1_empty", "h0_empty", "fc_done", "gt_begin"]
F_ = {n: i for i, n in enumerate(FIELDS)}


def _weights(s, H, Ksb, dev, seed=0):
    g = torch.Generator().manual_seed(seed)
    k = 1.0 / H ** 0.5
    keep = []

    def u(*shape):
        t = ((torch.rand(*shape, generator=g) * 2 - 1) * k).to(dev)
        keep.append(t)
        return t.data_ptr()

    for layer in range(2):
        s.w_ih[layer], s.w_hh[layer] = u(4 * H, Ksb if layer == 0 else H), u(4 * H, H)
        s.b_ih[layer], s.b_hh[layer] = u(4 * H), u(4 * H)
    s.fc_w, s.fc_b = u(2, H), u(2)
    return keep


def test_probe_hook_checks_arguments_without_gpu():
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    host = torch.zeros(64, dtype=torch.int64)
    p = host.data_ptr()
    s = _lib.SeqWeights()
    # B = 3 clips x 33 bins = 99 rows: 4 pairs, 8 CTAs own rows; 10 steps: iterations 0 .. 10
    ok = dict(H=384, x3=1, B=3, steps=10, stages=0, cluster=0, stamps=p, ctas=8, its=11)

    def call(**kw):
        a = dict(ok, **kw)
        return lib.fsn_debug_sb_lstm_tc_probe(C.byref(s), a["H"], 15, 0, 2, 0, a["x3"], p, p, a["B"], 33, 10, 1, p, None,
                                              2, a["steps"], 1, a["stages"], a["cluster"], p, p, a["stamps"], a["ctas"],
                                              a["its"], None)

    for kw in (dict(stamps=None), dict(ctas=0), dict(ctas=9), dict(its=0), dict(its=12), dict(B=0), dict(steps=11)):
        assert call(**kw) == _lib.FSN_ERR_SHAPE, kw
        assert lib.fsn_last_error_code() == _lib.FSN_ERR_SHAPE
    for kw in (dict(H=192), dict(stages=5), dict(cluster=3)):
        assert call(**kw) == _lib.FSN_ERR_UNSUPPORTED, kw
    assert _lib.SB_PROBE_FIELDS == len(FIELDS)
    # the binding's record layout is the header's (which the kernel static_asserts against)
    import os
    import re
    from conftest import ROOT
    header = open(os.path.join(ROOT, "include", "fsn_b200.h")).read()
    macros = dict(re.findall(r"#define (FSN_SB_PROBE_\w+) (\d+)", header))
    assert int(macros["FSN_SB_PROBE_FIELDS"]) == _lib.SB_PROBE_FIELDS
    assert int(macros["FSN_SB_PROBE_SLOTS"]) == _lib.SB_PROBE_SLOTS


def _run(dev, H, x3, B, F, steps, probe, ctas, its):
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    Ns, la = 15, 2
    s = _lib.SeqWeights()
    keep = _weights(s, H, 2 * Ns + 2, dev)
    g = torch.Generator().manual_seed(1)
    magT = torch.randn(B, steps, F, generator=g).abs().to(dev)
    fbT = torch.relu(torch.randn(B, steps, F, generator=g)).to(dev)
    inv2 = (torch.rand(B, generator=g) + 0.3).to(dev)
    packed = torch.empty(lib.fsn_debug_sb_lstm_tc_packed_bytes(H, x3), dtype=torch.uint8, device=dev)
    crm = torch.full((B, 2, F, steps - la), float("nan"), device=dev)
    stamps = torch.full((ctas, its, 2, _lib.SB_PROBE_SLOTS, _lib.SB_PROBE_FIELDS), -1, dtype=torch.int64, device=dev)
    args = (C.byref(s), H, Ns, 0, 2, 0, x3, magT.data_ptr(), fbT.data_ptr(), B, F, steps, 1, inv2.data_ptr(), None, la,
            steps, 1, 0, 0, packed.data_ptr(), crm.data_ptr())
    st = torch.cuda.current_stream().cuda_stream
    if probe:
        _lib.check(lib.fsn_debug_sb_lstm_tc_probe(*args, stamps.data_ptr(), ctas, its, st))
    else:
        _lib.check(lib.fsn_debug_sb_lstm_tc(*args, st))
    torch.cuda.synchronize()
    del keep
    return crm.cpu(), stamps.cpu()


@pytest.mark.gpu
@pytest.mark.parametrize("x3", [1, 0], ids=["x3", "single"])
@pytest.mark.parametrize("H", [384, 128])
def test_probe_same_bits_and_ordered_stamps(H, x3):
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    dev = torch.device("cuda:0")
    B, F, steps = 3, 33, 12           # 99 rows: 4 pairs, 8 CTAs
    ctas, its = 6, steps              # a sample: 6 of the 8 CTAs, iterations 0 .. steps - 1 of 0 .. steps
    ref, _ = _run(dev, H, x3, B, F, steps, False, ctas, its)
    out, st = _run(dev, H, x3, B, F, steps, True, ctas, its)
    assert not torch.isnan(ref).any()
    assert torch.equal(ref, out), "the probe instantiation changed the output bits"
    mt, parts = H // 128, 2 if x3 else 1
    nkb = (1 + H // 32, 2 * H // 32)
    for cta in range(ctas):
        prev_end = [None] * mt
        for it in range(its):
            for layer in range(2):
                exists = (layer == 0 and it < steps) or (layer == 1 and it >= 1)
                for m in range(4):
                    r = st[cta, it, layer, m]
                    if m >= mt or not exists:
                        if m < 3 or layer == 1:
                            assert (r == -1).all(), (cta, it, layer, m, "record of a block that does not exist")
                        continue
                    t = [int(r[F_[f]]) for f in ("t_begin", "t_mma0", "t_mma1", "t_end")]
                    assert t == sorted(t) and t[0] > 0, (cta, it, layer, m, t)
                    assert int(r[F_["stages"]]) == nkb[layer] * parts
                    waits = sum(int(r[F_[f]]) for f in ("operand", "turn", "w_full", "wait_group", "cell", "l1_done",
                                                        "h1_empty", "h0_empty", "fc_done"))
                    assert (r[4:15] >= 0).all() and waits <= t[3] - t[0], (cta, it, layer, m)
                    if prev_end[m] is not None:
                        assert t[0] >= prev_end[m], (cta, it, layer, m, "blocks of a warpgroup overlap")
                    prev_end[m] = t[3]
            p = st[cta, it, 0, 3]
            assert 0 < int(p[F_["t_begin"]]) <= int(p[F_["t_end"]])
            assert int(p[F_["stages"]]) == parts * mt * ((nkb[0] if it < steps else 0) + (nkb[1] if it >= 1 else 0))
            if it:
                assert int(p[F_["t_begin"]]) >= int(st[cta, it - 1, 0, 3, F_["t_end"]])
                assert int(p[F_["gt_begin"]]) >= int(st[cta, it - 1, 0, 3, F_["gt_begin"]])
