"""The dense GEMM layer alone against float64, through the hooks of include/fsn_b200.h: the fp32 Linear
(fsn_debug_fc_gemm), the fp32 SIMT GEMM and its split-K reduction (fsn_debug_sgemm), the column sums
(fsn_debug_colsum), the two-output weight gradient (fsn_debug_small_out_wgrad), the transposes (fsn_debug_transpose,
fsn_debug_transpose_blocked with its bias-gradient column sums), every tile / split-K branch of the tf32 wgmma GEMM
(fsn_debug_tgemm), the operand preparation + GEMM + epilogue of the full-band stacks (fsn_debug_gemm_tc) and the fused
training-forward step with fp16 h next to tf32 x (fsn_debug_lstm_fwd_step).

Every GEMM check is the element-wise bound of tests/test_cpu_gemm_kernels.py,
|C - C64| <= c sqrt(K) 2^-24 (|A| |B|^T) (+ 2^-21 (|A| |B|^T) for x3), with C64 the float64 product of the operands the
hardware reads.  c is per family (C_BOUND there), about 4x the worst ratio measured on an H100 80GB HBM3 (700 W):
    fc 1.23, sgemm 0.36, colsum 0.387, small_out 0.0844, tgemm 0.927, gemm_tc 0.626, gemm_tc_x3 2.29 (past its 2^-21 term)
The tf32 checks hold against the truncated operands (bits & ~0x1FFF) at these c: the tensor core truncates, it does
not round.  The training-forward step is held to absolute bounds (STEP_TOL) against float64 of its rounded operands:
worst 1.3e-6 on the gates and c, 6.7e-7 on h, with fp16 h next to tf32 x in one k loop among the cases.

The column sums (colsum, the bias sums of transpose_blocked) and small_out_wgrad also run on non-zero integer data whose
fp32 sums are exact: they must equal the float64 sums bit for bit, so one row dropped or one slab summed twice cannot
hide under sqrt(K) of rounding room, however long the sum.

Every case runs twice and must give the same bits (all reductions are fixed-order), outputs start from a sentinel, rows
past M and the columns of a padded ldc must keep it, and accumulate = 1 must add to the C given.  Scratch that is meant
to make split-K take fewer slices is followed by a sentinel guard that must stay untouched.  The largest case, the
short-K tgemm over 131 077 rows, holds two 134 MB outputs.  The worst ratio of each family is printed with -s as
`[gemm] family worst`."""
import ctypes
import math

import numpy as np
import pytest
import torch

from test_cpu_gemm_kernels import (ACT_NONE, ACT_RELU, ACT_RELU6, ACT_TANH, C_BOUND, D, TANH_ULP, blocked_floats,
                                   excess, f16, gemm_tc_ws_bytes, ref_blocked, ref_colsum, ref_linear, ref_sgemm, ref_small_out, row_scale_index,
                                   tf32)

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
SENT = -7777.0
WORST = {}
# absolute bounds of the fused step against float64 of its rounded operands (gates, c, h), about 4x the worst measured
STEP_TOL = {"gates": 5e-6, "c": 5e-6, "h": 3e-6}   # measured 1.33e-6, 1.31e-6, 6.65e-7


def _note(family, r, tol):
    WORST[family] = max(WORST.get(family, 0.0), r)
    assert r <= tol, (family, r, tol)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k, v in sorted(WORST.items()):
        print(f"[gemm] {k} worst {v:.3g}")


@pytest.fixture(scope="module")
def lib():
    from fullsubnet_b200 import _lib
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return _lib.load()


def _st():
    return torch.cuda.current_stream().cuda_stream


def _check(rc):
    from fullsubnet_b200 import _lib
    _lib.check(rc)


def _twice(run, init):
    """run(out) on a copy of init and then on init itself; both must give the same bits. Returns the first."""
    o1, o2 = init.clone(), init
    run(o1)
    run(o2)
    torch.cuda.synchronize()
    assert torch.equal(o1.view(torch.int32), o2.view(torch.int32)), "two runs differ"
    return o1


def _sent(*shape):
    return torch.full(shape, SENT, device=DEV)


def _untouched(t):
    return bool((t == SENT).all()) if t.numel() else True


GUARD = 1024


def _scratch(n):
    """n floats of scratch followed by GUARD sentinel floats; _guard_ok checks that the kernel stayed inside the n."""
    return _sent(n + GUARD)


def _guard_ok(scratch):
    return _untouched(scratch[-GUARD:])


def _ints(*shape, seed):
    """Non-zero integers in [-8, 8]: every fp32 sum of them below 2^24 in magnitude is exact, so a column sum or a
    weight gradient of such data must equal the float64 one bit for bit, whatever the slab order, and a dropped or doubled
    row or slab changes it."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    v = torch.randint(1, 9, shape, device=DEV, generator=g).float()
    return torch.where(torch.rand(shape, device=DEV, generator=g) < 0.5, -v, v)


# ------------------------------------------------------------------ fc_gemm
def _fc(lib, M, K, O, act, bias, kmajor, A=None, W=None, b=None, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    A = torch.randn(M, K, device=DEV, generator=g) if A is None else A
    W = (torch.randn(K, O, device=DEV, generator=g) if kmajor else torch.randn(O, K, device=DEV, generator=g)) if W is None else W
    b = (torch.randn(O, device=DEV, generator=g) if bias else None) if b is None else b
    out = _twice(lambda o: _check(lib.fsn_debug_fc_gemm(A.data_ptr(), W.data_ptr(), None if b is None else b.data_ptr(),
                                                         o.data_ptr(), M, K, O, act, int(kmajor), _st())), _sent(M + 2, O))
    assert _untouched(out[M:]), "rows past M written"
    ref, cond = ref_linear(A, W, b, act, w_kmajor=kmajor)
    return out[:M], ref, cond


FC_DIMS = [(M, K, O) for M in (1, 63, 64, 65, 257) for K in (1, 15, 16, 17, 257) for O in (1, 63, 64, 65, 257)]


def test_fc_gemm_every_edge_shape_act_bias_and_layout(lib):
    acts = (ACT_NONE, ACT_RELU, ACT_TANH, ACT_RELU6)
    for i, (M, K, O) in enumerate(FC_DIMS):
        act, bias, kmajor = acts[i % 4], (i // 4) % 2 == 0, (i // 8) % 2 == 1
        got, ref, cond = _fc(lib, M, K, O, act, bias, kmajor, seed=i)
        r = excess(got, ref, cond, K + 1, rel_extra=TANH_ULP if act == ACT_TANH else None)
        _note("fc", r, C_BOUND["fc"])


@pytest.mark.parametrize("M,K,O,kmajor,act", [
    (3 * 63 + 1, 512, 257, False, ACT_RELU),    # full-band Linear Hf -> F + ReLU (fullsubnet)
    (2 * 190, 257, 64, True, ACT_NONE),         # fast_fullsubnet mel filterbank, [F, M] K-major weights
    (3 * 63, 257, 2048, False, ACT_NONE),       # training hoisted projection K0 = 257 -> 4H = 2048 (K0 % 4 != 0)
])
def test_fc_gemm_production_shapes(lib, M, K, O, kmajor, act):
    got, ref, cond = _fc(lib, M, K, O, act, not kmajor, kmajor, seed=M + K + O)
    _note("fc", excess(got, ref, cond, K + 1), C_BOUND["fc"])


def test_fc_gemm_relu_clamps_are_exact(lib):
    M, K, O = 65, 17, 65
    torch.manual_seed(0)
    A = torch.randn(M, K, device=DEV)
    W = torch.randn(O, K, device=DEV)
    for act, shift, want in ((ACT_RELU, -1e4, 0.0), (ACT_RELU6, -1e4, 0.0), (ACT_RELU6, 1e4, 6.0)):
        b = torch.full((O,), shift, device=DEV)
        got, _, _ = _fc(lib, M, K, O, act, True, False, A=A, W=W, b=b)
        assert bool((got == want).all()), (act, shift)


# ------------------------------------------------------------------ sgemm
def _sgemm(lib, ta, M, N, K, acc=0, ldc_pad=0, scratch_floats=0, seed=0, lda_pad=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    lda = (M if ta else K) + lda_pad
    A = torch.randn(K if ta else M, lda, device=DEV, generator=g)
    B = torch.randn(K, N, device=DEV, generator=g)
    ldc = N + ldc_pad
    init = _sent(M + 2, ldc)
    C0 = None
    if acc:
        C0 = torch.randn(M, N, device=DEV, generator=g)
        init[:M, :N] = C0
    scratch = _scratch(scratch_floats) if scratch_floats else None
    out = _twice(lambda o: _check(lib.fsn_debug_sgemm(ta, A.data_ptr(), lda, B.data_ptr(), N, o.data_ptr(), ldc, M, N, K, acc,
                                                      None if scratch is None else scratch.data_ptr(), scratch_floats, _st())),
                 init)
    assert _untouched(out[M:]) and _untouched(out[:M, N:]), "rows past M or ldc padding written"
    assert scratch is None or _guard_ok(scratch), "split-K partials written past scratch_floats"
    ref, cond = ref_sgemm(ta, A, B, M, N, K, C0)
    _note("sgemm", excess(out[:M, :N], ref, cond, K + (1 if acc else 0)), C_BOUND["sgemm"])


SPLIT = 16 << 20


@pytest.mark.parametrize("ta", [0, 1])
@pytest.mark.parametrize("M,N,K,acc,ldc_pad,sf", [
    (64, 64, 4095, 0, 0, SPLIT),          # just below the split threshold: one slice
    (64, 64, 4096, 1, 3, SPLIT),          # at it: S = 4, accumulate through the reduction, padded ldc
    (65, 63, 5000, 0, 5, SPLIT),          # S = 5 slices of 1008, the last one 968 long; partial tiles
    (64, 64, 8192, 1, 0, 3 * 64 * 64),    # scratch for only 3 of the 8 slices it wants
    (100, 70, 300, 1, 2, 0),              # short K, accumulate without split
])
def test_sgemm_split_k_branches(lib, ta, M, N, K, acc, ldc_pad, sf):
    _sgemm(lib, ta, M, N, K, acc, ldc_pad, sf, seed=M + K + ta)


@pytest.mark.parametrize("M,N", [(17 * 64, 31 * 64), (16 * 64, 33 * 64)])
def test_sgemm_tile_count_threshold(lib, M, N):
    """527 tiles still split K = 4096, 528 do not."""
    _sgemm(lib, 1, M, N, 4096, 0, 0, SPLIT, seed=M)


@pytest.mark.parametrize("ta,M,N,K,sf", [
    (1, 257, 512, 190 * 64, SPLIT),       # linear_bwd dW = dY^T X of the full-band Linear, config 3 (64 clips x 190 frames)
    (0, 190 * 64, 512, 257, 0),           # its dX = dY W
])
def test_sgemm_linear_bwd_config3_shapes(lib, ta, M, N, K, sf):
    _sgemm(lib, ta, M, N, K, 0, 0, sf, seed=K)


# ------------------------------------------------------------------ colsum / small_out_wgrad
COLSUM_CASES = [(r, c) for r in (1, 2047, 2048, 2049) for c in (1, 2, 31, 33, 1536)] + [(512 * 2048 + 1, 1),
                                                                                        (512 * 2048 + 1, 33)]


def _colsum(lib, X, rows, cols, ldx):
    S = min((rows + 2047) // 2048, 512)
    scratch = _scratch(S * cols)
    both = _twice(lambda o: _check(lib.fsn_debug_colsum(X.data_ptr(), rows, cols, ldx, o[0].data_ptr(), o[1].data_ptr(),
                                                        scratch.data_ptr(), S * cols, _st())), _sent(2, cols + 1))
    assert torch.equal(both[0], both[1]) and _untouched(both[:, cols:])
    assert _guard_ok(scratch), "slab partials written past S * cols"
    return both[0, :cols]


@pytest.mark.parametrize("rows,cols", COLSUM_CASES)
def test_colsum_slabs(lib, rows, cols):
    """randn data within the bound; integer data exactly (the last two cases are the S cap: 512 slabs of 2049 rows, where
    one row too few or a slab twice would change the exact sums)."""
    ldx = cols + 3
    torch.manual_seed(rows + cols)
    X = torch.randn(rows, ldx, device=DEV)
    ref, cond = ref_colsum(X, rows, cols)
    _note("colsum", excess(_colsum(lib, X, rows, cols, ldx), ref, cond, rows), C_BOUND["colsum"])
    del X
    Xi = _ints(rows, ldx, seed=rows + cols)
    assert torch.equal(_colsum(lib, Xi, rows, cols, ldx).to(D), ref_colsum(Xi, rows, cols)[0])


def _small_out(lib, dout, Hm, rows, H, sf):
    scratch = _scratch(sf)
    got = _twice(lambda o: _check(lib.fsn_debug_small_out_wgrad(dout.data_ptr(), Hm.data_ptr(), rows, H, o.data_ptr(),
                                                                scratch.data_ptr(), sf, _st())), _sent(2 * H + 4))
    assert _untouched(got[2 * H:]) and _guard_ok(scratch), "dW or scratch written past its end"
    return got[:2 * H].view(2, H)


def _check_small_out(lib, rows, H, sf, seed):
    """randn data within the bound; integer data exactly."""
    torch.manual_seed(seed)
    dout, Hm = torch.randn(rows, 2, device=DEV), torch.randn(rows, H, device=DEV)
    ref, cond = ref_small_out(dout, Hm)
    _note("small_out", excess(_small_out(lib, dout, Hm, rows, H, sf), ref, cond, rows), C_BOUND["small_out"])
    dout, Hm = _ints(rows, 2, seed=seed), _ints(rows, H, seed=seed + 1)
    assert torch.equal(_small_out(lib, dout, Hm, rows, H, sf).to(D), ref_small_out(dout, Hm)[0])


@pytest.mark.parametrize("rows", [2045, 2046, 2047, 2048, 6001])    # rows per slab % 4 = 1, 2, 3, 0, and 1 over 3 slabs
@pytest.mark.parametrize("H", [1, 127, 128, 129, 512])
def test_small_out_wgrad(lib, rows, H):
    _check_small_out(lib, rows, H, 3 * 2 * H, seed=rows + H)


def test_small_out_wgrad_with_one_slab_of_scratch(lib):
    """6001 rows want 3 slabs; scratch for one makes it a single pass over all rows."""
    _check_small_out(lib, 6001, 129, 2 * 129, seed=1)


# ------------------------------------------------------------------ transposes
@pytest.mark.parametrize("rows,cols", [(1, 1), (31, 33), (32, 32), (33, 2048), (2048, 129), (1000, 257)])
def test_transpose_is_exact(lib, rows, cols):
    torch.manual_seed(rows)
    x = torch.randn(rows, cols, device=DEV)
    got = _twice(lambda o: _check(lib.fsn_debug_transpose(x.data_ptr(), rows, cols, o.data_ptr(), _st())),
                 _sent(rows * cols + 5))
    assert torch.equal(got[:rows * cols].view(cols, rows), x.T) and _untouched(got[rows * cols:])


def _blocked(lib, x, K, M, ld, max_slabs):
    """The blocked copy and, with max_slabs, the bias sums and the slab count; part carries a sentinel guard."""
    n = blocked_floats(K, M)
    part = _scratch(max_slabs * M) if max_slabs else None
    slabs = ctypes.c_int(0)
    init = torch.cat([_sent(n + 7), _sent(M + 1)])

    def run(o):
        _check(lib.fsn_debug_transpose_blocked(x.data_ptr(), K, M, ld, o.data_ptr(), None if part is None else part.data_ptr(),
                                               max_slabs, ctypes.byref(slabs),
                                               None if part is None else o[n + 7:].data_ptr(), _st()))
    got = _twice(run, init)
    assert _untouched(got[n:n + 7]) and _untouched(got[n + 7 + (M if max_slabs else 0):])
    assert part is None or _guard_ok(part), "slab sums written past max_slabs * M"
    return got[:n], got[n + 7:n + 7 + M], slabs.value


@pytest.mark.parametrize("K,M", [(1, 1), (33, 127), (300, 128), (5000, 129), (1000, 2048), (70001, 33)])
@pytest.mark.parametrize("max_slabs", [0, 1, 7, 512])
def test_transpose_blocked_layout_and_bias_sums(lib, K, M, max_slabs):
    """randn data: the layout bit for bit (zero padding included) and the bias sums within the bound; integer data: the
    bias sums exactly."""
    ld = M + 4
    torch.manual_seed(K + M)
    x = torch.randn(K, ld, device=DEV)
    blk, bias, slabs = _blocked(lib, x, K, M, ld, max_slabs)
    assert torch.equal(blk.cpu(), ref_blocked(x[:, :M].cpu())), "blocked layout or its zero padding differs"
    if not max_slabs:
        return
    nkb = (K + 31) // 32
    kb_per = 8 if (nkb + 7) // 8 <= max_slabs else -(-nkb // max_slabs)
    assert slabs == -(-nkb // kb_per) <= max_slabs
    ref, cond = ref_colsum(x, K, M)
    _note("colsum", excess(bias, ref, cond, K), C_BOUND["colsum"])
    xi = _ints(K, ld, seed=K + M)
    blk, bias, _ = _blocked(lib, xi, K, M, ld, max_slabs)
    assert torch.equal(bias.to(D), ref_colsum(xi, K, M)[0])


# ------------------------------------------------------------------ tgemm branches
def _tgemm(lib, M, N, K, acc=0, ldc_pad=0, sf=0, seed=0, chunk=None):
    g = torch.Generator(device=DEV).manual_seed(seed)
    ld = (K + 3) & ~3
    A, B = torch.randn(M, ld, device=DEV, generator=g), torch.randn(N, ld, device=DEV, generator=g)
    ldc = N + ldc_pad
    init = _sent(M + 3, ldc)
    if acc:
        init[:M, :N] = torch.randn(M, N, device=DEV, generator=g)
    C0 = init[:M, :N].clone() if acc else None
    scratch = _scratch(sf) if sf else None
    out = _twice(lambda o: _check(lib.fsn_debug_tgemm(A.data_ptr(), ld, B.data_ptr(), ld, o.data_ptr(), ldc, M, N, K, acc,
                                                      None if scratch is None else scratch.data_ptr(), sf, _st())), init)
    assert _untouched(out[M:]) and _untouched(out[:M, N:]), "rows past M or ldc padding written"
    assert scratch is None or _guard_ok(scratch), "split-K partials written past scratch_floats"
    At, Bt = tf32(A[:, :K]).to(D), tf32(B[:, :K]).to(D)
    out = out[:M]
    step = chunk or M
    for r0 in range(0, M, step):
        a = At[r0:r0 + step]
        ref, cond = a @ Bt.T, a.abs() @ Bt.abs().T
        if acc:
            ref, cond = ref + C0[r0:r0 + step].to(D), cond + C0[r0:r0 + step].to(D).abs()
        _note("tgemm", excess(out[r0:r0 + step, :N], ref, cond, K + (1 if acc else 0)), C_BOUND["tgemm"])


@pytest.mark.parametrize("M,N,K,sf,acc", [
    (64, 2048, 512, SPLIT, 0),            # per-step full-band GEMM, few tiles: S = 4 slices
    (64, 512, 2048, SPLIT, 1),            # S = 16, accumulate through the reduction
    (64, 512, 256, SPLIT, 0),             # K / 128 caps S at 2
    (64, 512, 383, SPLIT, 1),             # S = 2 with a short last slice
    (64, 512, 2048, 3 * 64 * 512, 0),     # scratch for 3 of the 16 slices
    (131072 + 5, 256, 32, 0, 0),          # short K, many tiles: BN = 128 although N % 256 == 0
    (200, 512, 100, 0, 1),                # BN = 256, partial M tile, accumulate
    (130, 130, 4, 0, 0),                  # K = 4, one k block
])
def test_tgemm_branches(lib, M, N, K, sf, acc):
    _tgemm(lib, M, N, K, acc, ldc_pad=4 if M < 100000 else 0, sf=sf, seed=N + K, chunk=8192)


# ------------------------------------------------------------------ gemm_tc
def _gemm_tc(lib, x3, K, N, B, T, mode, ldx_pad, offset, act, bias, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    rows, ldx = B * T, K + ldx_pad
    base = torch.randn(rows * ldx + offset, device=DEV, generator=g)
    xv = base[offset:].view(rows, ldx)
    W = torch.randn(N, K, device=DEV, generator=g) / math.sqrt(K)
    b = torch.randn(N, device=DEV, generator=g) if bias else None
    scale, rps, sB = None, 1, 0
    if mode == "clip":
        scale, rps = torch.rand(B, device=DEV, generator=g) + 0.5, T
    elif mode == "time":
        scale, rps, sB = torch.rand(T * B, device=DEV, generator=g) + 0.5, T, B
    ws_bytes = gemm_tc_ws_bytes(rows, K, N, x3)      # exactly what the hook carves
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=DEV)
    ldo = N + 3
    out = _twice(lambda o: _check(lib.fsn_debug_gemm_tc(xv.data_ptr(), ldx, K, None if scale is None else scale.data_ptr(), rps,
                                                        sB, W.data_ptr(), N, None if b is None else b.data_ptr(), act, x3,
                                                        o.data_ptr(), ldo, rows, ws.data_ptr(), ws_bytes, _st())),
                 _sent(rows + 2, ldo))
    assert _untouched(out[rows:]) and _untouched(out[:rows, N:])
    xs = xv[:, :K]
    if scale is not None:
        xs = xs * scale[torch.from_numpy(row_scale_index(np.arange(rows), rps, sB)).to(DEV)].unsqueeze(1)  # fp32, as the kernel
    a, w = (xs, W) if x3 else (tf32(xs), tf32(W))
    ref, cond = ref_linear(a, w, b, act)
    fam = "gemm_tc_x3" if x3 else "gemm_tc"
    _note(fam, excess(out[:rows, :N], ref, cond, K + 1, x3=bool(x3), rel_extra=TANH_ULP if act == ACT_TANH else None),
          C_BOUND[fam])


@pytest.mark.parametrize("x3", [0, 1])
@pytest.mark.parametrize("K,mode,ldx_pad,offset,act,bias", [
    (33, "clip", 0, 0, ACT_NONE, True),
    (257, "time", 3, 0, ACT_RELU, True),
    (257, None, 0, 1, ACT_TANH, False),        # unaligned x: the copy path without a scale
    (33, None, 7, 0, ACT_RELU6, False),        # ldx > K, no bias
    (257, "clip", 5, 1, ACT_NONE, False),
    (32, None, 4, 0, ACT_NONE, False),         # aligned, unscaled: the single pass reads x in place
])
def test_gemm_tc_operand_paths(lib, x3, K, mode, ldx_pad, offset, act, bias):
    _gemm_tc(lib, x3, K, 257, 3, 50, mode, ldx_pad, offset, act, bias, seed=K + ldx_pad + offset)


# ------------------------------------------------------------------ fused training-forward step
@pytest.mark.parametrize("R,H,K0,half,fold,first", [
    (200, 128, 12, 1, True, False),     # fp16 h, tf32 x in one k loop (K0 % 8 == 4)
    (130, 32, 36, 1, True, False),
    (1, 256, 260, 1, True, False),
    (129, 256, 36, 1, True, True),
    (200, 128, 16, 1, True, False),     # fp16 x and h
    (200, 128, 12, 0, True, False),     # tf32 throughout
    (257, 384, 64, 0, True, False),     # compile-time H
    (130, 512, 0, 1, False, False),     # hoisted projection in G
    (1, 32, 0, 0, False, False),
])
def test_lstm_fwd_step_against_rounded_operands(lib, R, H, K0, half, fold, first):
    g = torch.Generator(device=DEV).manual_seed(R + H + K0)
    k = 1.0 / H ** 0.5
    w_hh = (torch.rand(4 * H, H, device=DEV, generator=g) * 2 - 1) * k
    w_ih = (torch.rand(4 * H, max(K0, 4), device=DEV, generator=g) * 2 - 1) * k
    b_ih, b_hh = [(torch.rand(4 * H, device=DEV, generator=g) * 2 - 1) * k for _ in range(2)]
    hp, cp = torch.rand(R, H, device=DEV, generator=g) * 2 - 1, torch.randn(R, H, device=DEV, generator=g)
    x = torch.randn(R, max(K0, 4), device=DEV, generator=g)
    P = torch.randn(R, 4 * H, device=DEV, generator=g)
    G0 = _sent(R + 4, 4 * H)
    if not fold:
        G0[:R] = P
    scratch = torch.empty(2 * (2 * R * H + 4 * H * (H + K0) + R * K0) + 4096, dtype=torch.uint8, device=DEV)
    CH = _sent(2, R + 4, H)

    def run(o):
        Gx, CHx = o
        _check(lib.fsn_debug_lstm_fwd_step(None if first else hp.data_ptr(), w_hh.data_ptr(), x.data_ptr() if fold else None,
                                           w_ih.data_ptr() if fold else None, K0, Gx.data_ptr(), b_ih.data_ptr(), b_hh.data_ptr(),
                                           None if first else cp.data_ptr(), CHx[0].data_ptr(), CHx[1].data_ptr(), R, H, half,
                                           scratch.data_ptr(), scratch.numel(), _st()))
    outs = []
    for _ in range(2):
        o = (G0.clone(), CH.clone())
        run(o)
        outs.append(o)
    torch.cuda.synchronize()
    for a, b in zip(outs[0], outs[1]):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), "two runs differ"
    G, CHo = outs[0]
    rh = f16 if half else tf32
    rx = f16 if (half and K0 % 8 == 0) else tf32
    z = b_ih.to(D) + b_hh.to(D)
    z = z + (rx(x[:, :K0]).to(D) @ rx(w_ih[:, :K0]).to(D).T if fold else P.to(D))
    if not first:
        z = z + rh(hp).to(D) @ rh(w_hh).to(D).T
    i, f, gg, o_ = z[:, :H].sigmoid(), z[:, H:2 * H].sigmoid(), z[:, 2 * H:3 * H].tanh(), z[:, 3 * H:].sigmoid()
    c = i * gg if first else f * cp.to(D) + i * gg
    h = o_ * c.tanh()
    for name, got, ref in (("gates", G[:R], torch.cat([i, f, gg, o_], 1)), ("c", CHo[0, :R], c), ("h", CHo[1, :R], h)):
        _note("step_" + name, float((got.to(D) - ref).abs().max()), STEP_TOL[name])
    assert _untouched(G[R:]) and _untouched(CHo[:, R:])
