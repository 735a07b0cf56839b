"""The float64 references of the dense GEMM layer, pinned on the CPU, the error bound every GEMM check in
tests/test_gpu_gemm_kernels.py applies, a demonstration that the bound sees the bugs it is there to catch, and the
CPU-only argument checks of the GEMM-layer test hooks.

The kernels are the fp32 Linear (fc_gemm), the fp32 SIMT GEMM with its split-K reduction (sgemm), the column sums and the
two-output weight gradient of the backward pass (colsum, small_out_wgrad), the two transposes, and the tf32 tensor-core
GEMMs (tgemm, and the operand preparation + GEMM + epilogue of the full-band stacks, gemm_tc).

The bound, element by element, for C = A B^T over K terms:

    |C - C64|_ij <= c sqrt(K) 2^-24 (|A| |B|^T)_ij        (+ 2^-21 (|A| |B|^T)_ij for the x3 split)

C64 is the float64 product of exactly the operands the hardware multiplies: the fp32 values, their tf32 truncation
(bits & ~0x1FFF: the tensor core reads fp32 bits as tf32) or their fp16 round-to-nearest.  A bias, an accumulated C or
the partial sums of split-K are extra terms of the same sum.  The x3 split multiplies [hi | lo | hi] by [hi | hi | lo]
(hi = tf32(v), lo = v - hi, both read as tf32 again) and drops lo.lo: its 2^-21 term is pinned below."""
import math

import numpy as np
import pytest
import torch

D = torch.float64
U = 2.0 ** -24                       # fp32 unit roundoff
X3_TERM = 2.0 ** -21                 # the x3 split's dropped / truncated lo terms, relative to |A| |B|^T
ACT_NONE, ACT_RELU, ACT_TANH, ACT_RELU6 = 0, 1, 2, 3
TANH_ULP = 2.0 ** -21                # tanhf: 2 ulp of its result (CUDA math API), relative
# the bound's c for each family, about 4x the worst ratio measured on an H100 80GB HBM3 (700 W), which is in the comment.
# fc: the tiny-K Linears, where sqrt(K) undercounts the product, bias add and tanhf roundings; gemm_tc_x3: what is left
# after its 2^-21 term, an accumulation over 3K terms
C_BOUND = {
    "fc": 5.0,            # 1.23
    "sgemm": 1.5,         # 0.36
    "colsum": 1.5,        # 0.387
    "small_out": 0.35,    # 0.0844
    "tgemm": 3.5,         # 0.927
    "gemm_tc": 2.5,       # 0.626
    "gemm_tc_x3": 9.5,    # 2.29
}


# ------------------------------------------------------------------ operand rounding
def tf32(x: torch.Tensor) -> torch.Tensor:
    """The value the tensor core reads from fp32 bits: the 13 low mantissa bits dropped (truncation toward zero)."""
    x = x.float().contiguous()
    return (x.view(torch.int32) & ~0x1FFF).view(torch.float32)


def f16(x: torch.Tensor) -> torch.Tensor:
    """fp16 round-to-nearest (__float2half_rn), back in fp32."""
    return x.float().half().float()


def x3_split(v: torch.Tensor, operand: int) -> torch.Tensor:
    """split_tf32_kernel's compensated layout of v [rows, K]: A operand (1) [hi | lo | hi], B operand (2) [hi | hi | lo]."""
    v = v.float()
    hi = tf32(v)
    lo = v - hi                      # exact in fp32
    return torch.cat([hi, lo, hi] if operand == 1 else [hi, hi, lo], dim=1)


# ------------------------------------------------------------------ references
def act_ref(z: torch.Tensor, act: int) -> torch.Tensor:
    return {ACT_NONE: lambda v: v, ACT_RELU: torch.relu, ACT_TANH: torch.tanh,
            ACT_RELU6: lambda v: torch.clamp(v, 0.0, 6.0)}[act](z)


def ref_linear(A, W, bias=None, act=ACT_NONE, w_kmajor=False):
    """act(A W^T + bias) in float64 and its conditioning |A| |W|^T + |bias|; W [O,K] or, w_kmajor, [K,O]."""
    A, W = A.to(D), W.to(D)
    Wt = W if w_kmajor else W.T
    z = A @ Wt
    cond = A.abs() @ Wt.abs()
    if bias is not None:
        z = z + bias.to(D)
        cond = cond + bias.to(D).abs()
    return act_ref(z, act), cond


def ref_sgemm(ta, A, B, M, N, K, C0=None):
    """op(A) B (+ C0): op(A) = A[:M, :K] or, ta, A[:K, :M]^T; B [K, N]; returns (C, |op(A)| |B| + |C0|)."""
    a = (A[:K, :M].T if ta else A[:M, :K]).to(D)
    b = B[:K, :N].to(D)
    c, cond = a @ b, a.abs() @ b.abs()
    if C0 is not None:
        c, cond = c + C0.to(D), cond + C0.to(D).abs()
    return c, cond


def ref_colsum(X, rows, cols):
    x = X[:rows, :cols].to(D)
    return x.sum(0), x.abs().sum(0)


def ref_small_out(dout, Hm):
    """dW [2,H] = dout^T Hm of the two-output Linear."""
    d, h = dout.to(D), Hm.to(D)
    return d.T @ h, d.abs().T @ h.abs()


def row_scale_index(r, rows_per_scale, scale_B=0):
    """split_tf32_kernel's row-scale entry of row r: per clip r / rows_per_scale, or with scale_B > 0 the time-major entry
    (r % rows_per_scale) * scale_B + r / rows_per_scale of a [T', B] table."""
    r = np.asarray(r)
    if scale_B > 0:
        return (r % rows_per_scale) * scale_B + r // rows_per_scale
    return r // rows_per_scale


def blocked_index(k, m, K):
    """Where element (k, m) of in [K, M] lands in transpose_blocked_kernel's copy (fsn_tgemm.cu): tile (m / 128, k / 32)
    of 128 x 32 floats at ((mt * nkb + kb) * 128 + m % 128) * 32 + k % 32, nkb = ceil(K / 32)."""
    k, m = np.asarray(k), np.asarray(m)
    nkb = (K + 31) // 32
    return (((m // 128) * nkb + k // 32) * 128 + m % 128) * 32 + k % 32


def gemm_tc_ws_bytes(rows, K, N, x3):
    """fsn_debug_gemm_tc's workspace: the prepared A [rows, Kp p] and W [4 max(8, ceil(N/4)), Kp p] operands, each on a
    256-byte boundary (Kp = K rounded up to 4, p = 3 for x3)."""
    up = lambda n: (n + 255) // 256 * 256
    wa = ((K + 3) & ~3) * (3 if x3 else 1)
    return up(rows * wa * 4) + up(4 * max(8, -(-N // 4)) * wa * 4)


def blocked_floats(K, M):
    return ((M + 127) // 128) * 128 * ((K + 31) // 32) * 32


def ref_blocked(X):
    """The whole blocked copy of X [K, M] (zero padding included), built element by element from blocked_index."""
    K, M = X.shape
    out = torch.zeros(blocked_floats(K, M), dtype=X.dtype)
    kk, mm = np.meshgrid(np.arange(K), np.arange(M), indexing="ij")
    out[torch.from_numpy(blocked_index(kk, mm, K).reshape(-1))] = X.reshape(-1)
    return out


# ------------------------------------------------------------------ the bound
def excess(got, ref, cond, K, x3=False, rel_extra=None):
    """max over elements of |got - ref| / (sqrt(K) 2^-24 cond), after the x3 term 2^-21 cond (and rel_extra * |ref|,
    the ulp error of a final tanhf) are taken off; inf where cond == 0 and got != ref."""
    got, ref, cond = got.to(D), ref.to(D), cond.to(D)
    err = (got - ref).abs()
    if x3:
        err = err - X3_TERM * cond
    if rel_extra is not None:
        err = err - rel_extra * ref.abs()
    err = err.clamp(min=0.0)
    unit = math.sqrt(K) * U * cond
    r = torch.where(unit > 0, err / torch.where(unit > 0, unit, torch.ones_like(unit)),
                    torch.where(err > 0, torch.full_like(err, math.inf), torch.zeros_like(err)))
    return float(r.max()) if r.numel() else 0.0


# ------------------------------------------------------------------ pins
def test_tf32_truncation_rule():
    one = torch.tensor([1.0 + 2.0 ** -10, 1.0 + 2.0 ** -11, -(1.0 + 2.0 ** -11), 3.0 - 2.0 ** -22, 2.0 ** -140], dtype=torch.float32)
    got = tf32(one)
    assert got[0] == 1.0 + 2.0 ** -10        # 10 stored mantissa bits survive
    assert got[1] == 1.0 and got[2] == -1.0  # bit 11 dropped, toward zero on both signs
    assert got[3] == 3.0 - 2.0 ** -9         # truncation, not rounding up to 3
    assert got[4] == 0.0                     # a subnormal with no bit above the 13 dropped ones
    x = torch.randn(4096)
    t = tf32(x)
    assert bool(((x - t).abs() <= x.abs() * 2.0 ** -10).all()) and bool((t.abs() <= x.abs()).all())


def test_x3_split_is_exact_and_within_its_term():
    torch.manual_seed(0)
    a, b = torch.randn(40, 257) * 3, torch.randn(30, 257)
    A3, B3 = x3_split(a, 1), x3_split(b, 2)
    Kp = a.shape[1]
    assert torch.equal(A3[:, :Kp] + A3[:, Kp:2 * Kp], a)      # hi + lo == v exactly
    assert torch.equal(B3[:, :Kp] + B3[:, 2 * Kp:], b)
    assert torch.equal(A3[:, 2 * Kp:], A3[:, :Kp]) and torch.equal(B3[:, Kp:2 * Kp], B3[:, :Kp])
    # what the tensor core computes from the split (every part read as tf32 again) vs the exact product
    hw = tf32(A3).to(D) @ tf32(B3).to(D).T
    exact, cond = a.to(D) @ b.to(D).T, a.to(D).abs() @ b.to(D).abs().T
    assert float(((hw - exact).abs() / cond).max()) <= X3_TERM
    # the single pass sits far outside that term: the x3 bound does separate the two
    one = tf32(a).to(D) @ tf32(b).to(D).T
    assert float(((one - exact).abs() / cond).max()) > 16 * X3_TERM


@pytest.mark.parametrize("ta", [0, 1])
def test_references_match_torch_float64(ta):
    torch.manual_seed(1)
    M, N, K = 33, 17, 45
    A = torch.randn(K, M) if ta else torch.randn(M, K)
    B, C0 = torch.randn(K, N), torch.randn(M, N)
    c, cond = ref_sgemm(ta, A, B, M, N, K, C0)
    opA = A.to(D).T if ta else A.to(D)
    assert torch.allclose(c, torch.matmul(opA, B.to(D)) + C0.to(D), rtol=1e-14, atol=1e-14)
    assert torch.allclose(cond, torch.matmul(opA.abs(), B.to(D).abs()) + C0.to(D).abs(), rtol=1e-14, atol=1e-14)
    W, b = torch.randn(N, K), torch.randn(N)
    x = torch.randn(M, K)
    for act in (ACT_NONE, ACT_RELU, ACT_TANH, ACT_RELU6):
        want = torch.nn.functional.linear(x.to(D), W.to(D), b.to(D))
        want = {ACT_NONE: want, ACT_RELU: torch.nn.functional.relu(want), ACT_TANH: torch.tanh(want),
                ACT_RELU6: torch.nn.functional.relu6(want)}[act]
        assert torch.allclose(ref_linear(x, W, b, act)[0], want, rtol=1e-14, atol=1e-14)
        assert torch.allclose(ref_linear(x, W.T.contiguous(), b, act, w_kmajor=True)[0], want, rtol=1e-14, atol=1e-14)
    X = torch.randn(300, 20)
    s, cs = ref_colsum(X, 300, 20)
    assert torch.allclose(s, torch.sum(X.to(D), 0), rtol=1e-14, atol=1e-13)
    assert torch.allclose(cs, torch.sum(X.to(D).abs(), 0), rtol=1e-14)
    dout, Hm = torch.randn(300, 2), torch.randn(300, 7)
    dW, _ = ref_small_out(dout, Hm)
    lin = torch.nn.Linear(7, 2, dtype=D)
    y = lin(Hm.to(D))
    y.backward(dout.to(D))
    assert torch.allclose(dW, lin.weight.grad, rtol=1e-13, atol=1e-13)


def test_row_scale_index_reproduces_the_cumulative_norm():
    """Both row-scale modes against the oracle's cumulative_laplace_norm of a [B, 1, F, T] magnitude, rows clip-major
    (r = b T + t): per clip, one scale per (clip, frame) row (rows_per_scale = 1), and time-major, the [T, B] table of the
    streaming and tensor-core stacks (rows_per_scale = T, scale_B = B)."""
    from oracle import fullsubnet_oracle as O
    torch.manual_seed(2)
    B, F, T = 3, 9, 11
    mag = torch.rand(B, 1, F, T, dtype=D) + 0.1
    want = O.cumulative_laplace_norm(mag)[:, 0].permute(0, 2, 1).reshape(B * T, F)       # rows (b, t)
    cnt = torch.arange(1, T + 1, dtype=D) * F
    scale = 1.0 / (torch.cumsum(mag[:, 0].sum(1), -1) / cnt + O.EPSILON)              # [B, T]
    x = mag[:, 0].permute(0, 2, 1).reshape(B * T, F)
    r = np.arange(B * T)
    tm = scale.T.contiguous().reshape(-1)                                              # [T, B]
    got_tm = x * tm[torch.from_numpy(row_scale_index(r, T, B))].unsqueeze(1)
    got_rows = x * scale.reshape(-1)[torch.from_numpy(row_scale_index(r, 1))].unsqueeze(1)
    assert torch.allclose(got_tm, want, rtol=1e-13, atol=0)
    assert torch.allclose(got_rows, want, rtol=1e-13, atol=0)
    # per clip: one scale per clip of T rows (the offline norm)
    off = O.offline_laplace_norm(mag)[:, 0].permute(0, 2, 1).reshape(B * T, F)
    s_clip = 1.0 / (mag.mean(dim=(1, 2, 3)) + 1e-5)
    assert torch.allclose(x * s_clip[torch.from_numpy(row_scale_index(r, T))].unsqueeze(1), off, rtol=1e-13, atol=0)


@pytest.mark.parametrize("K,M", [(1, 1), (31, 127), (32, 128), (33, 129), (100, 300)])
def test_blocked_layout_is_a_padded_transpose(K, M):
    torch.manual_seed(3)
    X = torch.randn(K, M)
    blk = ref_blocked(X)
    MT, nkb = (M + 127) // 128, (K + 31) // 32
    # tile (mt, kb) is rows m of 128 floats... unfolded back: [MT, nkb, 128, 32] -> [MT*128, nkb*32] == padded X^T
    plain = blk.reshape(MT, nkb, 128, 32).permute(0, 2, 1, 3).reshape(MT * 128, nkb * 32)
    want = torch.zeros(MT * 128, nkb * 32)
    want[:M, :K] = X.T
    assert torch.equal(plain, want)
    assert len(set(blocked_index(*np.meshgrid(np.arange(K), np.arange(M), indexing="ij"), K).reshape(-1).tolist())) == K * M


# ------------------------------------------------------------------ the bound sees planted bugs
def _planted(M, N, K, seed):
    g = torch.Generator().manual_seed(seed)
    A, B = torch.randn(M, K, generator=g, dtype=D), torch.randn(N, K, generator=g, dtype=D)
    bias = torch.randn(N, generator=g, dtype=D)
    return A, B, bias


# the shapes of the GPU file where each mutation could hide: fc_gemm / gemm_tc Linears, sgemm at its split threshold,
# the per-step tgemm split-K (the column sums are checked exactly on integer data instead, see below)
PLANT_SHAPES = [(257, 257, 257), (65, 63, 17), (64, 2048, 512), (64, 512, 2048), (128, 64, 4096), (64, 64, 8192)]


@pytest.mark.parametrize("M,N,K", PLANT_SHAPES)
def test_bound_catches_planted_mutations(M, N, K):
    """Each mutation, applied to the float64 product, breaks the bound with the largest c of any family: one k term
    dropped, one 64-column tile shifted by one column, the bias applied to the neighbouring row, one split-K slab summed
    twice (four slabs)."""
    A, B, bias = _planted(M, N, K, seed=M + N + K)
    C = A @ B.T + bias
    cond = A.abs() @ B.abs().T + bias.abs()
    c = max(C_BOUND.values())
    assert excess(C, C, cond, K + 1) == 0.0
    mutations = {}
    k = K // 2
    mutations["dropped k term"] = C - torch.outer(A[:, k], B[:, k])
    if N > 64:
        shifted = C.clone()
        shifted[:, 64:min(128, N)] = C[:, 63:min(128, N) - 1]
        mutations["tile shifted by a column"] = shifted
    wrong = C.clone()
    wrong[0] -= bias
    wrong[1] += bias
    mutations["bias on the wrong row"] = wrong
    ks = (K + 3) // 4
    mutations["split-K slab twice"] = C + A[:, ks:2 * ks] @ B[:, ks:2 * ks].T
    for name, bad in mutations.items():
        for x3 in (False, True):
            assert excess(bad, C, cond, K + 1, x3=x3) > c, (name, x3)


@pytest.mark.parametrize("rows,cols", [(2049, 33), (512 * 2048 + 1, 1)])
def test_integer_column_sums_are_exact_and_see_one_row(rows, cols):
    """At the shapes the GPU file sums non-zero integers in [-8, 8], every fp32 partial sum is exact, in any slab order: the
    kernel's result must equal the float64 sum, and a slab cap that loses the last row (512 slabs of 2048 instead of 2049
    rows) or a slab summed twice changes it."""
    g = torch.Generator().manual_seed(rows)
    v = torch.randint(1, 9, (rows, cols), generator=g).float()
    X = torch.where(torch.rand(rows, cols, generator=g) < 0.5, -v, v)
    assert float(X.abs().sum(0).max()) < 2.0 ** 24
    exact = X.to(D).sum(0)
    S = min((rows + 2047) // 2048, 512)
    per = -(-rows // S)
    slabs = [X[z * per:(z + 1) * per].sum(0) for z in range(S)]       # fp32, as the kernel sums each slab
    total = torch.zeros(cols)
    for t in slabs:
        total = total + t
    assert torch.equal(total.to(D), exact)
    assert not torch.equal(X[:-1].to(D).sum(0), exact)                   # one row lost
    assert not torch.equal(exact + slabs[0].to(D), exact)                # one slab twice


# ------------------------------------------------------------------ argument checks (no GPU)
@pytest.fixture(scope="module")
def lib():
    from fullsubnet_b200 import _lib
    return _lib.load()


def test_gemm_hooks_refuse_before_any_cuda_call(lib):
    """Every new hook rejects null pointers, non-positive sizes, short leading dimensions and short scratch with its error
    class before any CUDA call: the stand-in pointers are never dereferenced and no device is touched."""
    from fullsubnet_b200 import _lib
    SH, WS = _lib.FSN_ERR_SHAPE, _lib.FSN_ERR_WORKSPACE
    p = 1 << 20
    # fc_gemm(A, W, bias, out, M, K, O, act, w_kmajor)
    fc = lambda A=p, W=p, out=p, M=4, K=4, O=4, act=0: lib.fsn_debug_fc_gemm(A, W, None, out, M, K, O, act, 0, None)
    for kw in ({"A": None}, {"W": None}, {"out": None}, {"M": 0}, {"K": -1}, {"O": 0}, {"act": 4}, {"act": -1},
               {"O": 65535 * 64 + 1}):
        assert fc(**kw) == SH, kw
    # sgemm(ta, A, lda, B, ldb, C, ldc, M, N, K, acc, scratch, scratch_floats)
    def sg(ta=0, A=p, lda=8, B=p, ldb=8, Cp=p, ldc=8, M=8, N=8, K=8, scratch=None, sf=0):
        return lib.fsn_debug_sgemm(ta, A, lda, B, ldb, Cp, ldc, M, N, K, 0, scratch, sf, None)
    for kw, code in (({"A": None}, SH), ({"B": None}, SH), ({"Cp": None}, SH), ({"M": 0}, SH), ({"N": -2}, SH),
                     ({"K": 0}, SH), ({"lda": 7}, SH), ({"ta": 1, "M": 9}, SH), ({"ldb": 7}, SH), ({"ldc": 7}, SH),
                     ({"N": 65535 * 64 + 1, "ldb": 65535 * 64 + 1, "ldc": 65535 * 64 + 1}, SH),
                     ({"sf": 100}, WS), ({"scratch": p, "sf": -1}, WS)):
        assert sg(**kw) == code, kw
    # colsum(X, rows, cols, ldx, out, out2, scratch, scratch_floats): S = min(ceil(rows / 2048), 512) slabs
    def cs(X=p, rows=4096, cols=3, ldx=3, out=p, scratch=p, sf=6):
        return lib.fsn_debug_colsum(X, rows, cols, ldx, out, None, scratch, sf, None)
    for kw, code in (({"X": None}, SH), ({"out": None}, SH), ({"rows": 0}, SH), ({"cols": 0}, SH), ({"ldx": 2}, SH),
                     ({"scratch": None}, WS), ({"sf": 5}, WS), ({"rows": 4097, "sf": 6}, WS),
                     ({"rows": 512 * 2048 + 1, "sf": 512 * 3 - 1}, WS)):
        assert cs(**kw) == code, kw
        if code == WS and kw.get("sf"):
            assert b"scratch" in lib.fsn_last_error()
    # small_out_wgrad(dout, Hm, rows, H, dW, scratch, scratch_floats): at least one slab of 2 H floats
    so = lambda d=p, h=p, rows=100, H=8, dW=p, scratch=p, sf=16: lib.fsn_debug_small_out_wgrad(d, h, rows, H, dW, scratch, sf, None)
    for kw, code in (({"d": None}, SH), ({"h": None}, SH), ({"dW": None}, SH), ({"rows": 0}, SH), ({"H": 0}, SH),
                     ({"scratch": None}, WS), ({"sf": 15}, WS), ({"sf": 0}, WS)):
        assert so(**kw) == code, kw
    # transpose(in, rows, cols, out)
    for args in ((None, 4, 4, p), (p, 4, 4, None), (p, 0, 4, p), (p, 4, 0, p), (p, 4, 65535 * 32 + 1, p)):
        assert lib.fsn_debug_transpose(*args, None) == SH, args
    # transpose_blocked(in, K, M, ld, out, colsum_part, max_slabs, slabs, bias_out)
    tb = lambda i=p, K=64, M=8, ld=8, out=p, part=None, ms=0, bo=None: lib.fsn_debug_transpose_blocked(i, K, M, ld, out, part,
                                                                                                      ms, None, bo, None)
    for kw in ({"i": None}, {"out": None}, {"K": 0}, {"M": 0}, {"ld": 7}, {"part": p, "ms": 4}, {"part": p, "bo": p},
               {"part": p, "ms": -1, "bo": p}):
        assert tb(**kw) == SH, kw
    # gemm_tc(x, ldx, K, row_scale, rps, scale_B, W, N, bias, act, x3, out, ldo, rows, ws, ws_bytes)
    need = gemm_tc_ws_bytes(100, 33, 20, 1)
    def gt(x=p, ldx=33, K=33, rs=None, rps=1, sB=0, W=p, N=20, act=0, out=p, ldo=20, rows=100, ws=p, nb=need):
        return lib.fsn_debug_gemm_tc(x, ldx, K, rs, rps, sB, W, N, None, act, 1, out, ldo, rows, ws, nb, None)
    for kw, code in (({"x": None}, SH), ({"W": None}, SH), ({"out": None}, SH), ({"K": 0}, SH), ({"N": 0}, SH),
                     ({"rows": 0}, SH), ({"rows": 1 << 31}, SH), ({"ldx": 32}, SH), ({"ldo": 19}, SH),
                     ({"rs": p, "rps": 0}, SH), ({"rs": p, "sB": -1}, SH), ({"act": 5}, SH), ({"ws": None}, WS),
                     ({"N": 65535 * 128 + 1}, SH), ({"nb": need - 1}, WS)):
        assert gt(**kw) == code, kw
