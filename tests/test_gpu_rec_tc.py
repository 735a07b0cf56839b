"""GPU: the tensor-core LSTM layer / Linear layer of the full-band stacks (fsn_lstm_rec_tc.cu: hoisted tf32 GEMM +
persistent wgmma recurrence) against float64 torch on the CPU (audio_zen/model/module/sequence_model.py:52-58,117), and
the recurrence alone (lstm_rec_tc_kernel / lstm_rec_tc_carry_kernel through fsn_debug_lstm_rec_tc, on a given input
projection P) against the float64 references of tests/test_cpu_rec_tc_kernels.py.
x3 = compensated arithmetic (fp32 error class), single pass = fp16 operands.

The recurrence runs in both modes over hidden sizes 64 (one k-block), 100, 257 (odd: scalar path, 33-CTA partial
slice), 384, 512, 1000 (3 x3 ring stages) and 8 x SMs (the largest: 2 x3 stages, one group on the whole chip); every
supported H at T = 2, R = 129; R at 1, 63-65, 127-129 and at rows-per-launch - 1 / + 0 / + 1 and a third launch (read
from the launcher, not assumed); T at 1, 2 and the ring's stage count and twice it, +-1, and T = 4000; contiguous,
NaN-padded and odd (scalar path) strides; carried state with a c / h_init row stride > H, restarts at none / 0 (NaN
h_init and c_init) / mid / T-1, fin_step -1 / 0 / mid / T-1, c in place and out of place; nn.LSTM-initialised and
saturating (x4 weights, large biases) weights; one scratch reused for H = 384 / 257 / 512.

Every case checks the step bound of reference (b) element by element (|h - h_b| <= c 2^-23 E_h, the same for c_fin),
the max-abs error against reference (a) per (mode, H), NaN guards before and after hall and c_fin and in every stride
gap, that every output element is written, that two runs give the same bits, and that a row gives the same bits alone
as in the batch (rows 0, 127, 128, the last row of a launch and the first of the next).

Worst measured on an H100 80GB HBM3 at its 700 W power limit (the inputs are seeded, the kernel is deterministic).
The step bound's ratio max |err| / (2^-23 E), over every case: x3 1.26, single pass 1.39.  Max-abs against (a):

    H                   64       100      257      384      512      1000     8 x SMs  (1056 on this card)
    x3                  2.4e-7   2.8e-7   6.7e-7   6.5e-7   1.2e-6   1.8e-6   1.5e-6
    single pass         1.6e-4   1.3e-4   2.6e-4   2.4e-4   3.3e-4   2.9e-4   3.0e-4

    saturating weights (H = 257 / 512): x3 6.8e-6 / 1.2e-5, single pass 4.0e-3 / 4.7e-3
    T = 4000 at H = 512:                x3 4.6e-7,          single pass 1.4e-4
    the sweep of every H at T = 2:      x3 6.0e-7,          single pass 9.0e-5

C_BOUND (test_cpu_rec_tc_kernels.py) and A_TOL sit about 4x above these.  The whole file runs in about a minute."""
import ctypes
import math

import pytest
import torch

from test_cpu_rec_tc_kernels import C_BOUND, make_carry, make_layer, ref_lstm, ref_step

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
GUARD = 64                  # NaN floats before and after every output region (a multiple of 2: bases stay 8-byte aligned)
NAN_BITS = 0x7FC00000
# max-abs error against (a), about 4x the worst measured (module docstring): (x3, H) with nn.LSTM initialisation,
# (x3, H, "sat") with saturating weights, (x3, "long") at T = 4000, (x3, "sweep") for the sweep at T = 2
# (x3, "max") at H = 8 x SMs
A_TOL = {(1, 64): 1e-6, (1, 100): 1.1e-6, (1, 257): 2.7e-6, (1, 384): 2.6e-6, (1, 512): 4.7e-6, (1, 1000): 7e-6,
         (1, "max"): 6.2e-6, (1, 257, "sat"): 2.7e-5, (1, 512, "sat"): 4.9e-5, (1, "long"): 1.9e-6, (1, "sweep"): 2.4e-6,
         (0, 64): 6.4e-4, (0, 100): 5.3e-4, (0, 257): 1e-3, (0, 384): 9.8e-4, (0, 512): 1.3e-3, (0, 1000): 1.1e-3,
         (0, "max"): 1.2e-3, (0, 257, "sat"): 1.6e-2, (0, 512, "sat"): 1.9e-2, (0, "long"): 5.4e-4, (0, "sweep"): 3.6e-4}
WORST = {}
ROWS_ALONE = (0, 127, 128)   # and the last row of a launch and the first of the next


def _note(key, v, tol):
    WORST[key] = max(WORST.get(key, 0.0), v)
    assert v <= tol, (key, v, tol)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k, v in sorted(WORST.items(), key=str):
        print(f"[rec_tc] {k} worst {v:.3g}")


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return DEV


@pytest.fixture(scope="module")
def lib(dev):
    from fullsubnet_b200 import _lib
    return _lib.load()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _hmax():
    return 8 * _sms()       # ceil(H / 8) CTAs of one group must fit on the chip


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ------------------------------------------------------------------------------------------------ buffers
class Strided:
    """A [R, T, n] view (or [R, n] with T = None) into a flat NaN buffer with GUARD NaN floats before and after, step
    stride n + t_pad and row stride (T - 1)(n + t_pad) + n + row_pad; everything outside the view must keep its bits."""

    def __init__(self, R, T, n, t_pad=0, row_pad=0):
        Tn = 1 if T is None else T
        self.t = n + t_pad
        self.row = (Tn - 1) * self.t + n + row_pad
        total = GUARD + (R - 1) * self.row + (Tn - 1) * self.t + n + GUARD
        shape, stride = ((R, n), (self.row, 1)) if T is None else ((R, T, n), (self.row, self.t, 1))
        self.buf = torch.full((total,), math.nan, device=DEV)
        self.view = self.buf.as_strided(shape, stride, GUARD)
        idx = torch.arange(total, device=DEV).as_strided(shape, stride, GUARD)
        self.outside = torch.ones(total, dtype=torch.bool, device=DEV)
        self.outside[idx.reshape(-1)] = False

    def ptr(self):
        return self.view.data_ptr()

    def fill(self, v):
        self.buf.fill_(math.nan)
        self.view.copy_(v)
        return self

    def untouched_outside(self):
        return bool((self.buf[self.outside].view(torch.int32) == NAN_BITS).all())


STRIDES = {  # (P t_pad, P row_pad, hall t_pad, hall row_pad); odd: the scalar path even where H is even
    "contig": (0, 0, 0, 0),
    "padded": (6, 10, 2, 4),
    "odd": (3, 2, 1, 2),
}


def _run(lib, W, bi, bh, Pb, hb, R, T, H, x3, carry=None, scratch=None):
    """One call of the recurrence hook; carry = (h_init Strided, c_init Strided, c_fin Strided, restart int32 tensor,
    fin_step).  Returns info [rows_per_launch, stages, launches, smem] (the return code is checked)."""
    from fullsubnet_b200 import _lib
    info = (ctypes.c_int * 4)()
    if scratch is None:
        scratch = torch.empty(lib.fsn_debug_lstm_rec_tc_scratch_bytes(H, x3), dtype=torch.uint8, device=DEV)
    if carry is None:
        hi = ci = cf = rs = None
        c_row, fin = 0, -1
    else:
        h0, c0, cfin, rs_t, fin = carry
        hi, ci, cf, rs, c_row = h0.ptr(), c0.ptr(), cfin.ptr(), rs_t.data_ptr(), h0.row
    _lib.check(lib.fsn_debug_lstm_rec_tc(W.data_ptr(), bi.data_ptr(), bh.data_ptr(), Pb.ptr(), Pb.row, Pb.t, hb.ptr(), hb.row,
                                         hb.t, R, T, H, x3, hi, ci, cf, c_row, rs, fin, info, scratch.data_ptr(),
                                         scratch.numel(), _stream()))
    return list(info)


def _probe(lib, H, x3):
    """What the launcher chooses at H (one row, one step)."""
    W, bi, bh, P = [t.to(DEV) for t in make_layer(1, 1, H, seed=0)]
    return _run(lib, W, bi, bh, Strided(1, 1, 4 * H).fill(P), Strided(1, 1, H), 1, 1, H, x3)


def case(lib, H, x3, R, T, strides="contig", carry=None, sat=False, seed=0, alone=ROWS_ALONE, akey=None, layer=None):
    """Run the recurrence on one configuration and check everything the module docstring lists.  carry: None or
    {"fin": fin_step, "inplace": bool, "c_pad": extra floats per c / h_init row}; alone: the rows run alone besides the
    launch edges (() for none); layer: (W, b_ih, b_hh, P) instead of make_layer's.  Returns the launcher's info."""
    W, bi, bh, P = [t.to(DEV) for t in (layer if layer is not None else make_layer(R, T, H, seed, sat=sat))]
    pt, pr, ht, hr = STRIDES[strides]
    Pb = Strided(R, T, 4 * H, pt, pr).fill(P)
    cargs, c_in, h0, c0, restart, fin = None, None, None, None, None, -1
    if carry is not None:
        h0, c0, restart = make_carry(R, H, T, seed + 1)
        h0, c0 = h0.to(DEV), c0.to(DEV)
        nan_rows = torch.as_tensor(restart == 0, device=DEV)
        h0[nan_rows], c0[nan_rows] = math.nan, math.nan     # ignored by a row that restarts at step 0
        fin = carry["fin"]
        pad = carry.get("c_pad", 6)
        hb0 = Strided(R, None, H, row_pad=pad).fill(h0)
        c_in = Strided(R, None, H, row_pad=pad).fill(c0)
        c_out = c_in if carry["inplace"] else Strided(R, None, H, row_pad=pad)
        rs_t = torch.as_tensor(restart, device=DEV)
        cargs = (hb0, c_in, c_out, rs_t, fin)

    def once():
        hb = Strided(R, T, H, ht, hr)
        if carry is not None:
            c_in.fill(c0)
            if not carry["inplace"]:
                c_out.buf.fill_(math.nan)
        info = _run(lib, W, bi, bh, Pb, hb, R, T, H, x3, cargs)
        torch.cuda.synchronize()
        return info, hb, (None if carry is None else c_out)

    info, hb, cb = once()
    hall = hb.view.clone()
    assert hb.untouched_outside(), "hall: a guard or a stride gap was written"
    assert bool(torch.isfinite(hall).all()), "hall: an element was not written (or is not finite)"
    c_fin = None
    if carry is not None:
        if fin < 0:
            want = c0 if carry["inplace"] else torch.full_like(c0, math.nan)
            assert torch.equal(cb.view.view(torch.int32), want.view(torch.int32)), "c_fin written with fin_step = -1"
        else:
            c_fin = cb.view.clone()
            assert bool(torch.isfinite(c_fin).all()), "c_fin: an element was not written"
        assert cb.untouched_outside(), "c_fin: a guard or a row gap was written"
        assert hb0_untouched(cargs[0], h0)
    # two runs, the same bits
    _, hb2, cb2 = once()
    assert torch.equal(hb2.view.view(torch.int32), hall.view(torch.int32)), "run-to-run difference in hall"
    if c_fin is not None:
        assert torch.equal(cb2.view.view(torch.int32), c_fin.view(torch.int32)), "run-to-run difference in c_fin"
    # (b): the step bound, element by element; (a): max-abs
    kw = {} if carry is None else dict(h_init=h0, c_init=c0, restart=restart)
    h, c, Eh, Ec = ref_step(P, W, bi, bh, hall, x3, **kw)
    err_h = (hall.double() - h).abs()
    r = float((err_h / (2.0 ** -23 * Eh)).max())
    if c_fin is not None:
        r = max(r, float(((c_fin.double() - c[:, fin]).abs() / (2.0 ** -23 * Ec[:, fin])).max()))
    _note(("step", x3), r, C_BOUND[x3])
    ha, ca = ref_lstm(P, W, bi, bh, **kw)
    ea = float((hall.double() - ha).abs().max())
    if c_fin is not None:
        ea = max(ea, float((c_fin.double() - ca[:, fin]).abs().max()))
    key = akey if akey is not None else ((x3, H, "sat") if sat else (x3, H))
    _note(("a",) + key, ea, A_TOL[key])
    # a row alone gives the bits it gives in the batch
    if alone:
        rpl = info[0]
        for row in sorted({q for q in (*alone, rpl - 1, rpl) if q < R}):
            Pa = Strided(1, T, 4 * H).fill(P[row:row + 1])
            ha1 = Strided(1, T, H)
            ca = None
            if carry is not None:
                ca1 = Strided(1, None, H).fill(c0[row:row + 1])
                ca = (Strided(1, None, H).fill(h0[row:row + 1]), ca1, ca1, rs_t[row:row + 1].clone(), fin)
            _run(lib, W, bi, bh, Pa, ha1, 1, T, H, x3, ca)
            torch.cuda.synchronize()
            assert torch.equal(ha1.view[0].view(torch.int32), hall[row].view(torch.int32)), f"row {row} alone differs"
            if c_fin is not None:
                assert torch.equal(ca[2].view[0].view(torch.int32), c_fin[row].view(torch.int32)), f"row {row} c alone"
    return info


def hb0_untouched(hb0, h0):
    """h_init is only read"""
    return bool((hb0.view.view(torch.int32) == h0.view(torch.int32)).all()) and hb0.untouched_outside()


# ------------------------------------------------------------------------------------------------ the recurrence alone
def _H(h, x3):
    """The hidden size and the key of its max-abs bound against (a)."""
    return (_hmax(), (x3, "max")) if h == "max" else (h, (x3, h))


@pytest.mark.parametrize("x3", [1, 0])
@pytest.mark.parametrize("H", [64, 100, 257, 384, 512, 1000, "max"])
def test_rec_hidden_sizes(lib, H, x3):
    H, key = _H(H, x3)
    case(lib, H, x3, 130, 9, akey=key)
    case(lib, H, x3, 130, 9, strides="padded", carry={"fin": 8, "inplace": True}, seed=1, akey=key)


@pytest.mark.parametrize("x3", [1, 0])
def test_rec_unsupported_hidden_sizes_leave_the_output(lib, x3):
    for H in (56, _hmax() + 8):
        W, bi, bh, P = [t.to(DEV) for t in make_layer(2, 3, H, seed=0)]
        hb = Strided(2, 3, H)
        with pytest.raises(NotImplementedError):
            _run(lib, W, bi, bh, Strided(2, 3, 4 * H).fill(P), hb, 2, 3, H, x3)
        torch.cuda.synchronize()
        assert bool((hb.buf.view(torch.int32) == NAN_BITS).all())


@pytest.mark.parametrize("x3", [1, 0])
def test_rec_every_hidden_size(lib, x3):
    """Every supported H from 64 up at T = 2, R = 129 (one launch each): every CTA count ceil(H/8), every k padding and
    every ring-stage choice.  The weights of each H are cut from one seeded pair of matrices; the references run on the
    GPU in float64."""
    Hm = _hmax()
    g = torch.Generator(device=DEV).manual_seed(7)
    Wbig = torch.rand(4, Hm, Hm, generator=g, device=DEV) * 2 - 1
    bbig = torch.rand(2, 4, Hm, generator=g, device=DEV) * 2 - 1
    Pbig = torch.randn(129, 2, 4, Hm, generator=g, device=DEV)
    stages = set()
    for H in range(64, Hm + 1):
        k = 1.0 / math.sqrt(H)
        W = (Wbig[:, :H, :H] * k).reshape(4 * H, H).contiguous()
        bi, bh = (bbig[0, :, :H] * k).reshape(-1).contiguous(), (bbig[1, :, :H] * k).reshape(-1).contiguous()
        P = Pbig[..., :H].reshape(129, 2, 4 * H).contiguous()
        info = case(lib, H, x3, 129, 2, layer=(W, bi, bh, P), akey=(x3, "sweep"), alone=(128,))
        stages.add(info[1])
    assert stages == ({2, 3, 4} if x3 else {6}) or Hm <= 1024, stages


@pytest.mark.parametrize("x3", [1, 0])
@pytest.mark.parametrize("H", [512, 1000])
def test_rec_row_counts(lib, H, x3):
    """R around the m64 halves and the 128-row groups, and around the rows one cooperative launch covers."""
    rpl = _probe(lib, H, x3)[0]
    assert rpl % 128 == 0 and rpl == (_sms() // ((H + 7) // 8)) * 128
    seen = set()
    for R in sorted({1, 63, 64, 65, 127, 128, 129, rpl - 1, rpl, rpl + 1, 2 * rpl + 1}):
        info = case(lib, H, x3, R, 4, seed=R)
        assert info[2] == -(-R // rpl)
        seen.add(info[2])
    assert max(seen) >= 3


@pytest.mark.parametrize("x3", [1, 0])
@pytest.mark.parametrize("H", [384, 1000, "max"])
def test_rec_step_counts(lib, H, x3):
    """T = 1, 2 and around one and two trips of the state ring (its stage count, read from the launcher)."""
    H, key = _H(H, x3)
    S = _probe(lib, H, x3)[1]
    for T in sorted({1, 2, S - 1, S, S + 1, 2 * S - 1, 2 * S + 1}):
        case(lib, H, x3, 65, T, seed=T, akey=key)
        case(lib, H, x3, 65, T, carry={"fin": T - 1, "inplace": False}, seed=T + 50, alone=(), akey=key)


@pytest.mark.parametrize("x3", [1, 0])
@pytest.mark.parametrize("strides", ["contig", "padded", "odd"])
@pytest.mark.parametrize("H", [100, 257, 384])
def test_rec_strides(lib, H, strides, x3):
    case(lib, H, x3, 129, 6, strides=strides, seed=H)


@pytest.mark.parametrize("x3", [1, 0])
@pytest.mark.parametrize("inplace", [True, False])
@pytest.mark.parametrize("fin", ["none", 0, "mid", "last"])
@pytest.mark.parametrize("H", [257, 512])
def test_rec_carry(lib, H, fin, inplace, x3):
    """The carried state as the stream slot passes it: c / h_init rows wider than H, restarts none / 0 / mid / T-1."""
    T = 7
    f = {"none": -1, "mid": T // 2, "last": T - 1}.get(fin, fin)
    case(lib, H, x3, 130, T, strides="padded", carry={"fin": f, "inplace": inplace, "c_pad": 3 * H}, seed=H + f)


@pytest.mark.parametrize("x3", [1, 0])
@pytest.mark.parametrize("H", [257, 512])
def test_rec_saturating_weights(lib, H, x3):
    case(lib, H, x3, 65, 16, sat=True, seed=3)
    case(lib, H, x3, 65, 16, sat=True, carry={"fin": 15, "inplace": True}, seed=4)


@pytest.mark.parametrize("x3", [1, 0])
def test_rec_long_sequence(lib, x3):
    """T = 4000 at H = 512: the ring wraps thousands of times; carried state with restarts none / 0 / mid / T-1."""
    case(lib, 512, x3, 4, 4000, carry={"fin": 3999, "inplace": True}, seed=9, alone=(), akey=(x3, "long"))


@pytest.mark.parametrize("x3", [1, 0])
def test_rec_scratch_reused_across_hidden_sizes(lib, x3):
    """One scratch for H = 384, 257, 512 back to back on one stream (fast_fullsubnet's encoder / decoder): each result
    equals its run on a fresh scratch, bit for bit."""
    R, T = 130, 5
    layers = {H: [t.to(DEV) for t in make_layer(R, T, H, seed=H)] for H in (384, 257, 512)}
    shared = torch.empty(lib.fsn_debug_lstm_rec_tc_scratch_bytes(384, x3), dtype=torch.uint8, device=DEV)
    outs = {}
    for H, (W, bi, bh, P) in layers.items():
        outs[H] = Strided(R, T, H)
        _run(lib, W, bi, bh, Strided(R, T, 4 * H).fill(P), outs[H], R, T, H, x3, scratch=shared)
    torch.cuda.synchronize()
    for H, (W, bi, bh, P) in layers.items():
        fresh = torch.full((lib.fsn_debug_lstm_rec_tc_scratch_bytes(H, x3),), 0xA5, dtype=torch.uint8, device=DEV)
        hb = Strided(R, T, H)
        _run(lib, W, bi, bh, Strided(R, T, 4 * H).fill(P), hb, R, T, H, x3, scratch=fresh)
        torch.cuda.synchronize()
        assert torch.equal(hb.view.view(torch.int32), outs[H].view.view(torch.int32)), H


def test_rec_launch_choices(lib):
    """The launcher's branches that the matrix relies on: the default x3 ring (4 stages) at H = 512, 3 stages above
    H = 768 and 2 above H = 1024 (the 227 KB shared-memory opt-in limit), 6 stages in single pass, more than one group per
    launch at H <= 8 x SMs / 2 and one group at the largest H."""
    Hm = _hmax()
    assert _probe(lib, 512, 1)[1] == 4 and _probe(lib, 1000, 1)[1] == 3
    if Hm > 1024:
        assert _probe(lib, Hm, 1)[1] == 2
    assert all(_probe(lib, H, 0)[1] == 6 for H in (64, 512, Hm))
    assert _probe(lib, 512, 1)[0] >= 256 and _probe(lib, Hm, 0)[0] == 128


# ------------------------------------------------------------------------------------------------ the layer hooks
def _layer(dev, R, T, K, H, x3, seed=0):
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    g = torch.Generator().manual_seed(seed)
    k = 1.0 / H ** 0.5
    w = [(torch.rand(*s, generator=g) * 2 - 1) * k for s in ((4 * H, K), (4 * H, H), (4 * H,), (4 * H,))]
    x = torch.randn(R, T, K, generator=g)
    lstm = torch.nn.LSTM(K, H, batch_first=True).double()
    with torch.no_grad():
        for p, v in zip((lstm.weight_ih_l0, lstm.weight_hh_l0, lstm.bias_ih_l0, lstm.bias_hh_l0), w):
            p.copy_(v)
        ref = lstm(x.double())[0]
    n = lib.fsn_debug_lstm_tc_workspace_bytes(R, T, K, H, x3)
    ws = torch.empty(n, dtype=torch.uint8, device=dev)
    d = [t.to(dev).contiguous() for t in w + [x]]
    outs = []
    for _ in range(2):
        out = torch.full((R, T, H), float("nan"), device=dev)
        _lib.check(lib.fsn_debug_lstm_layer_tc(*[t.data_ptr() for t in d], R, T, K, H, x3, out.data_ptr(), ws.data_ptr(), n,
                                               torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        outs.append(out.cpu())
    assert torch.equal(outs[0], outs[1]), "run-to-run difference"  # fixed-order arithmetic, no atomics in the data path
    return float((outs[0].double() - ref).abs().max())


@pytest.mark.parametrize("R,T,K,H", [(2, 26, 64, 384), (3, 253, 384, 257), (256, 60, 257, 512), (300, 12, 128, 512),
                                     (1, 9, 33, 64), (130, 5, 100, 200)])
def test_lstm_layer_tc_matches_float64(dev, R, T, K, H):
    """Rows beyond one 128-row group, partial groups, partial unit slices (H % 8 != 0), odd strides, launch chunking."""
    e3, e1 = _layer(dev, R, T, K, H, 1), _layer(dev, R, T, K, H, 0)
    print(f"lstm_layer_tc R={R} T={T} K={K} H={H}: max-abs error x3 {e3:.1e}, single pass {e1:.1e}")
    assert e3 < 5e-6 and e1 < 3e-3


@pytest.mark.parametrize("rows,K,N,act", [(52, 257, 64, 1), (506, 512, 514, 0), (64768, 512, 257, 1), (1000, 257, 2048, 0)])
def test_linear_tc_matches_float64(dev, rows, K, N, act):
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    g = torch.Generator().manual_seed(rows + K + N)
    x, W, b = torch.randn(rows, K, generator=g), torch.randn(N, K, generator=g) / K ** 0.5, torch.randn(N, generator=g)
    ref = x.double() @ W.double().T + b.double()
    if act:
        ref = ref.clamp_min(0)
    Hm = max(8, (N + 3) // 4)
    for x3, tol in ((1, 5e-6), (0, 3e-3)):
        n = lib.fsn_debug_lstm_tc_workspace_bytes(rows, 1, K, Hm, x3)
        ws = torch.empty(n, dtype=torch.uint8, device=dev)
        out = torch.full((rows, N), float("nan"), device=dev)
        xd, Wd, bd = x.to(dev), W.to(dev), b.to(dev)
        _lib.check(lib.fsn_debug_linear_tc(xd.data_ptr(), rows, K, Wd.data_ptr(), bd.data_ptr(), N, act, x3, out.data_ptr(),
                                           ws.data_ptr(), n, torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        e = (out.cpu().double() - ref)
        assert float(e.norm() / ref.norm()) < tol, (x3, float(e.norm() / ref.norm()))


def test_unsupported_hidden_size_is_reported(dev):
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    z = torch.zeros(16, device=dev)
    with pytest.raises(NotImplementedError):
        _lib.check(lib.fsn_debug_lstm_layer_tc(z.data_ptr(), z.data_ptr(), z.data_ptr(), z.data_ptr(), z.data_ptr(), 1, 2, 4, 8,
                                               1, z.data_ptr(), z.data_ptr(), 64, torch.cuda.current_stream().cuda_stream))
