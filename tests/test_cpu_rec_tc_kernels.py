"""The float64 references of the full-band tensor-core LSTM recurrence (lstm_rec_tc_kernel / lstm_rec_tc_carry_kernel,
fsn_lstm_rec_tc.cu), pinned on the CPU, the step bound every recurrence check in tests/test_gpu_rec_tc.py applies, a
demonstration that the bound sees the bugs it is there to catch, and the CPU-only argument checks of the recurrence and
layer hooks.

Two references of one layer, gates z_t = P_t + b_ih + b_hh + h_{t-1} W_hh^T (order i, f, g, o):

(a) ref_lstm: nn.LSTM in float64 from zero state or a carried (h, c), each row restarting from zero state at its restart
    step.  It compounds over T, so it only gives a max-abs error per (mode, H).
(b) ref_step: step t from the KERNEL's own h_{t-1} (hall[:, t-1], h_init at step 0 of the carried kernel, zero at a
    restart step and at step 0 of the plain kernel), rounded as the kernel feeds it to the MMA: fp16 rn hi, and under
    x3 lo = rn(h - hi); W_hh split the same way; under x3 the products hi.hi + hi.lo + lo.hi (lo.lo dropped, as the
    kernel drops it).  c is carried in float64 from these gates.  Nothing but c compounds, so (b) supports an
    element-wise bound per step:

        |h - h_b| <= c_mode 2^-23 E_h,      |c_fin - c_b| <= c_mode 2^-23 E_c

    E propagates, to first order through the cell, a gate error of cond = |P| + |b_ih| + |b_hh| + sum_k |W||h| (over the
    operands the MMA multiplies) plus one unit per activation (fast_sigmoid / fast_tanh with __expf / __fdividef in
    single pass, expf under x3) plus one unit of the cell's own fp32 roundings; E_c carries through f.  c_mode is
    C_BOUND, about 4x the worst ratio measured on an H100 80GB HBM3 at 700 W (tests/test_gpu_rec_tc.py gives the numbers).

The planted bugs, each injected into a float64 emulation of the kernel, break that bound by orders of magnitude (step t
reading h_{t-2}, a neighbour's bias, the last partial k-block dropped, a neighbour's P row, a restart one step late or
keeping c, c_fin one step off: ratios 5e4 and up); the x3 operand bugs (the h lo or the W lo product dropped) by 20x and
more (ratios above 100)."""
import math

import numpy as np
import pytest
import torch

D = torch.float64
S = 2.0 ** -23                        # one unit of the step bound
# the step bound's c per mode (x3), about 4x the worst ratio measured (tests/test_gpu_rec_tc.py, module docstring)
C_BOUND = {1: 5.0, 0: 5.5}        # measured 1.26 (x3), 1.39 (single pass)
# budget of (b) with faithful operands against (a), relative to sum_k |W||h|: the fp16 rn of h and W (2^-11 each) in
# single pass; the fp16 rn of the lo parts and the dropped lo.lo under x3
FP16_BUDGET = {0: 2.0 ** -10 + 2.0 ** -21, 1: 2.0 ** -20}


# ------------------------------------------------------------------ operands as the MMA sees them
def split16(v: torch.Tensor):
    """fp16 hi = rn(v) and lo = rn(v - hi) of fp32 values (v - hi is exact in fp32), as float64."""
    v = v.float()
    hi = v.half().float()
    lo = (v - hi).half().float()
    return hi.to(D), lo.to(D)


def rec_term(hprev: torch.Tensor, W: torch.Tensor, x3: int, drop=()):
    """h_{t-1} W_hh^T of the kernel's operands and its conditioning: hprev [..., H] fp32, W [4H, H] fp32 -> [..., 4H].
    drop (planted bugs only): "h_lo" / "w_lo" leaves that product out under x3."""
    hh, hl = split16(hprev)
    Wh, Wl = split16(W)
    term, cond = hh @ Wh.T, hh.abs() @ Wh.abs().T
    if x3:
        if "w_lo" not in drop:
            term, cond = term + hh @ Wl.T, cond + hh.abs() @ Wl.abs().T
        if "h_lo" not in drop:
            term, cond = term + hl @ Wh.T, cond + hl.abs() @ Wh.abs().T
    return term, cond


def restart_mask(restart, R, T, device="cpu"):
    """[R, T] bool: step t is row r's restart step (restart[r] outside [0, T): never)."""
    if restart is None:
        return torch.zeros(R, T, dtype=torch.bool, device=device)
    rs = torch.as_tensor(np.asarray(restart), device=device).long()
    return torch.arange(T, device=device)[None, :] == rs[:, None]


def step_inputs(hall, h_init=None, restart=None):
    """The h_{t-1} step t multiplies, [R, T, H] fp32: hall[:, t-1]; at step 0 h_init (carried kernel) or zero (plain);
    zero at a row's restart step."""
    R, T, H = hall.shape
    hp = torch.zeros(R, T, H, dtype=torch.float32, device=hall.device)
    hp[:, 1:] = hall[:, :-1]
    if h_init is not None:
        hp[:, 0] = h_init
    return torch.where(restart_mask(restart, R, T, hall.device)[..., None], torch.zeros((), device=hall.device), hp)


# ------------------------------------------------------------------ the cell and its error propagation
def ref_cell(z, c0=None, restart=None, dz=None, da=0.0, dr=0.0):
    """The LSTM cell over gates z [R, T, 4H] (float64, bias included) with c carried from c0 [R, H] (zero if None) and
    zeroed at each row's restart step.  Returns h, c [R, T, H] and, when dz (absolute gate error [R, T, 4H]) is given,
    the first-order bounds E_h, E_c: dz through the activations' derivatives, da per activation evaluation, dr relative
    per fp32 rounding of the cell; E_c carried through f."""
    R, T, H4 = z.shape
    H = H4 // 4
    i, f, g, o = torch.sigmoid(z[..., :H]), torch.sigmoid(z[..., H:2 * H]), torch.tanh(z[..., 2 * H:3 * H]), torch.sigmoid(z[..., 3 * H:])
    rs = restart_mask(restart, R, T, z.device)
    c = torch.zeros(R, H, dtype=D, device=z.device) if c0 is None else c0.to(D)
    E = torch.zeros_like(c)
    cs, Es = [], []
    if dz is not None:
        di, df, dg, do = dz[..., :H], dz[..., H:2 * H], dz[..., 2 * H:3 * H], dz[..., 3 * H:]
        # the parts of E_c that do not depend on c
        loc_ig = g.abs() * (i * (1 - i) * di + da) + i * ((1 - g * g) * dg + da) + dr * i * g.abs()
        loc_f = f * (1 - f) * df + da
    for t in range(T):
        keep = ~rs[:, t, None]
        cp = torch.where(keep, c, torch.zeros((), dtype=D, device=z.device))
        c = f[:, t] * cp + i[:, t] * g[:, t]
        cs.append(c)
        if dz is not None:
            Ep = torch.where(keep, E, torch.zeros((), dtype=D, device=z.device))
            E = f[:, t] * Ep + cp.abs() * (loc_f[:, t] + dr * f[:, t]) + loc_ig[:, t] + dr * c.abs()
            Es.append(E)
    C = torch.stack(cs, 1)
    tc = torch.tanh(C)
    h = o * tc
    if dz is None:
        return h, C, None, None
    Ec = torch.stack(Es, 1)
    Eh = tc.abs() * (o * (1 - o) * do + da) + o * ((1 - tc * tc) * Ec + da) + dr * h.abs()
    return h, C, Eh, Ec


def bias_of(b_ih, b_hh):
    return b_ih.to(D) + b_hh.to(D), b_ih.to(D).abs() + b_hh.to(D).abs()


def ref_step(P, W, b_ih, b_hh, hall, x3, h_init=None, c_init=None, restart=None):
    """Reference (b): every step from the kernel's own h_{t-1} (hall [R, T, H] fp32).  P [R, T, 4H] fp32.  Returns h, c
    [R, T, H] and the bounds E_h, E_c in units of S (see the module docstring)."""
    hp = step_inputs(hall, h_init, restart)
    term, cond = rec_term(hp, W, x3)
    b, bc = bias_of(b_ih, b_hh)
    z = P.to(D) + b + term
    cond = cond + P.to(D).abs() + bc
    return ref_cell(z, c_init, restart, dz=cond, da=1.0, dr=1.0)


def ref_lstm(P, W, b_ih, b_hh, h_init=None, c_init=None, restart=None):
    """Reference (a): the layer in float64 from zero state (or h_init / c_init), each row restarting from zero state at
    its restart step.  P [R, T, 4H]; returns h, c [R, T, H]."""
    R, T, H4 = P.shape
    H = H4 // 4
    Wd = W.to(D)
    b = b_ih.to(D) + b_hh.to(D)
    rs = restart_mask(restart, R, T, P.device)
    h = torch.zeros(R, H, dtype=D, device=P.device) if h_init is None else h_init.to(D)
    c = torch.zeros(R, H, dtype=D, device=P.device) if c_init is None else c_init.to(D)
    hs, cs = [], []
    zero = torch.zeros((), dtype=D, device=P.device)
    for t in range(T):
        keep = ~rs[:, t, None]
        h, c = torch.where(keep, h, zero), torch.where(keep, c, zero)
        z = P[:, t].to(D) + b + h @ Wd.T
        i, f, g, o = torch.sigmoid(z[:, :H]), torch.sigmoid(z[:, H:2 * H]), torch.tanh(z[:, 2 * H:3 * H]), torch.sigmoid(z[:, 3 * H:])
        c = f * c + i * g
        h = o * torch.tanh(c)
        hs.append(h)
        cs.append(c)
    return torch.stack(hs, 1), torch.stack(cs, 1)


def excess(got, ref, E):
    """max over elements of |got - ref| / (S E) (E > 0 everywhere); NaN if got has a NaN."""
    err = (got.to(D) - ref.to(D)).abs()
    if not bool(torch.isfinite(err).all()):
        return math.nan
    return float((err / (S * E)).max()) if err.numel() else 0.0


def step_excess(P, W, b_ih, b_hh, hall, x3, h_init=None, c_init=None, restart=None, c_fin=None, fin_step=-1):
    """The step bound's ratio of a kernel result (hall, and c_fin after fin_step): max of |err| / (S E)."""
    h, c, Eh, Ec = ref_step(P, W, b_ih, b_hh, hall, x3, h_init, c_init, restart)
    r = excess(hall, h, Eh)
    if c_fin is not None and fin_step >= 0:
        r = max(r, excess(c_fin, c[:, fin_step], Ec[:, fin_step]))
    return r


# ------------------------------------------------------------------ inputs
def make_layer(R, T, H, seed, sat=False, device="cpu", p_scale=1.0):
    """nn.LSTM initialisation U(-1/sqrt(H), 1/sqrt(H)), or (sat) x4 weights and biases of N(0, 3^2) that saturate the
    gates; P [R, T, 4H] ~ N(0, p_scale^2).  All fp32."""
    g = torch.Generator().manual_seed(seed)
    k = 1.0 / math.sqrt(H)
    W = (torch.rand(4 * H, H, generator=g) * 2 - 1) * k
    b_ih, b_hh = [(torch.rand(4 * H, generator=g) * 2 - 1) * k for _ in range(2)]
    if sat:
        W = W * 4
        b_ih, b_hh = torch.randn(4 * H, generator=g) * 3, torch.randn(4 * H, generator=g) * 3
    P = torch.randn(R, T, 4 * H, generator=g) * p_scale
    return [t.to(device) for t in (W, b_ih, b_hh, P)]


def make_carry(R, H, T, seed, device="cpu"):
    """h_init, c_init [R, H] and the restart table cycling through none (-1), 0, mid-sequence and T-1."""
    g = torch.Generator().manual_seed(seed)
    h0 = torch.rand(R, H, generator=g) * 2 - 1
    c0 = torch.randn(R, H, generator=g)
    pattern = [-1, 0, T // 2, T - 1]
    restart = np.array([pattern[r % 4] for r in range(R)], dtype=np.int32)
    return h0.to(device), c0.to(device), restart


# ------------------------------------------------------------------ a float64 emulation of the kernel, with planted bugs
def emulate(P, W, b_ih, b_hh, x3, h_init=None, c_init=None, restart=None, fin_step=-1, bug=None, bug_row=0, bug_unit=0):
    """What the kernel computes, step by step in float64 from its own fp32 h (the operand rules of (b)), or that with one
    planted bug.  Returns hall [R, T, H] fp32 and c after fin_step [R, H] fp32 (None if fin_step < 0)."""
    R, T, H4 = P.shape
    H = H4 // 4
    b_ih, b_hh = b_ih.clone(), b_hh.clone()
    P = P.clone()
    W = W.clone()
    if bug == "bias_neighbour":          # unit bug_unit of a partial slice takes unit bug_unit + 1's bias
        for q in range(4):
            b_ih[q * H + bug_unit], b_hh[q * H + bug_unit] = b_ih[q * H + bug_unit + 1], b_hh[q * H + bug_unit + 1]
    if bug == "kblock":                  # the last, partial 64-wide k-block of W_hh dropped
        W[:, (H - 1) // 64 * 64:] = 0
    if bug == "row":                     # row bug_row reads its neighbour's P row
        P[bug_row] = P[bug_row + 1]
    rst = None if restart is None else np.asarray(restart).copy()
    if bug == "restart_late":
        rst = np.where((rst >= 0) & (rst < T - 1), rst + 1, rst)
    drop = {"h_lo": ("h_lo",), "w_lo": ("w_lo",)}.get(bug, ())
    b = b_ih.to(D) + b_hh.to(D)
    hall = torch.zeros(R, T, H, dtype=torch.float32)
    h = torch.zeros(R, H) if h_init is None else h_init.float().clone()
    c = torch.zeros(R, H, dtype=D) if c_init is None else c_init.to(D).clone()
    c_fin = None
    for t in range(T):
        if t == 0:
            hp = h if h_init is not None else torch.zeros(R, H)
        elif bug == "parity":            # step t reads h_{t-2}: the other ping-pong buffer (zeros before step 1)
            hp = hall[:, t - 2] if t >= 2 else torch.zeros(R, H)
        else:
            hp = hall[:, t - 1]
        hp = hp.clone()
        if rst is not None:
            at = torch.as_tensor(rst == t)
            hp[at] = 0
            if bug != "restart_keeps_c":
                c[at] = 0
        term, _ = rec_term(hp, W, x3, drop)
        z = P[:, t].to(D) + b + term
        i, f, g, o = torch.sigmoid(z[:, :H]), torch.sigmoid(z[:, H:2 * H]), torch.tanh(z[:, 2 * H:3 * H]), torch.sigmoid(z[:, 3 * H:])
        c = f * c + i * g
        hall[:, t] = (o * torch.tanh(c)).float()
        store = fin_step + (1 if bug == "cfin_late" else 0)
        if t == store:
            c_fin = c.float().clone()
    if bug == "cfin_late" and fin_step == T - 1:
        c_fin = None
    return hall, c_fin


# ------------------------------------------------------------------ pins
def test_split16_is_round_to_nearest_and_exact_lo():
    v = torch.tensor([1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11, 1.0 + 2.0 ** -11 + 2.0 ** -20, -(1.0 + 3 * 2.0 ** -11)])
    hi, lo = split16(v)
    assert hi.tolist() == [1.0, 1.0 + 2.0 ** -9, 1.0 + 2.0 ** -10, -(1.0 + 2.0 ** -9)]  # ties to even, nearest otherwise
    x = torch.randn(20000) * 0.7
    hi, lo = split16(x)
    tiny = 2.0 ** -25                                                             # half an fp16 subnormal step
    assert bool(((hi - x.to(D)).abs() <= x.to(D).abs() * 2.0 ** -11 + tiny).all())
    assert bool(((hi + lo - x.to(D)).abs() <= x.to(D).abs() * 2.0 ** -22 + tiny).all())
    assert torch.equal((x - hi.float()), (x.to(D) - hi).float())                  # the fp32 difference is exact


@pytest.mark.parametrize("carry", [False, True])
def test_ref_lstm_is_torch_lstm(carry):
    """(a) is nn.LSTM in float64: with P = x W_ih^T, from zero state or a given (h, c), and (carry) every row restarting
    at its restart step = nn.LSTM over the steps before it from (h, c), then over the rest from zero state."""
    torch.manual_seed(0)
    R, T, K, H = 5, 9, 7, 16
    lstm = torch.nn.LSTM(K, H, batch_first=True).double()
    x = torch.randn(R, T, K, dtype=D)
    W, b_ih, b_hh = lstm.weight_hh_l0.detach(), lstm.bias_ih_l0.detach(), lstm.bias_hh_l0.detach()
    P = x @ lstm.weight_ih_l0.detach().T
    if not carry:
        got, _ = ref_lstm(P, W, b_ih, b_hh)
        with torch.no_grad():
            want = lstm(x)[0]
        assert torch.allclose(got, want, rtol=0, atol=1e-13)
        return
    h0, c0, restart = make_carry(R, H, T, 1)
    h0, c0 = h0.to(D), c0.to(D)
    got, gc = ref_lstm(P, W, b_ih, b_hh, h0, c0, restart)
    with torch.no_grad():
        for r in range(R):
            j = int(restart[r]) if 0 <= restart[r] < T else T
            parts = []
            if j > 0:
                y, (hn, cn) = lstm(x[r:r + 1, :j], (h0[r][None, None], c0[r][None, None]))
                parts.append(y)
            if j < T:
                parts.append(lstm(x[r:r + 1, j:])[0])
            want = torch.cat(parts, 1)[0]
            assert torch.allclose(got[r], want, rtol=0, atol=1e-13), r
        # c after the last step: nn.LSTM's final cell state of a row with no restart
        r = int(np.flatnonzero(restart == -1)[0])
        _, (hn, cn) = lstm(x[r:r + 1], (h0[r][None, None], c0[r][None, None]))
        assert torch.allclose(gc[r, -1], cn[0, 0], rtol=0, atol=1e-13)


@pytest.mark.parametrize("x3", [0, 1])
@pytest.mark.parametrize("carry", [False, True])
def test_ref_step_with_faithful_operands_is_ref_lstm(x3, carry):
    """(b) fed (a)'s own h (as fp32) is (a) within the fp16 rounding budget of the operands, propagated through the cell
    by the same E as the step bound; and that budget is tight enough to tell the two modes apart."""
    R, T, H = 6, 12, 100
    W, b_ih, b_hh, P = make_layer(R, T, H, seed=3)
    kw = {}
    if carry:
        h0, c0, restart = make_carry(R, H, T, 4)
        kw = dict(h_init=h0, c_init=c0, restart=restart)
    ha, ca = ref_lstm(P, W, b_ih, b_hh, **kw)
    hall = ha.float()
    hp = step_inputs(hall, kw.get("h_init"), kw.get("restart"))
    term, _ = rec_term(hp, W, x3)
    b, _ = bias_of(b_ih, b_hh)
    z = P.to(D) + b + term
    cond_exact = hp.to(D).abs() @ W.to(D).abs().T
    dz = FP16_BUDGET[x3] * cond_exact + 2.0 ** -24 * cond_exact
    hb, cb, Eh, Ec = ref_cell(z, kw.get("c_init"), kw.get("restart"), dz=dz)
    # first order: twice the propagated budget covers the second-order terms
    assert bool(((hb - ha).abs() <= 2 * Eh + 1e-15).all())
    assert bool(((cb - ca).abs() <= 2 * Ec + 1e-15).all())
    # hb is also what ref_step computes from the same hall
    hs, cs, _, _ = ref_step(P, W, b_ih, b_hh, hall, x3, **kw)
    assert torch.equal(hs, hb) and torch.equal(cs, cb)
    if not x3:
        assert float((hb - ha).abs().max()) > 1e-5          # single pass sits far outside the x3 budget
    else:
        assert float((hb - ha).abs().max()) < 1e-6


def test_ref_step_rules_at_step_zero_and_restart():
    """Step 0 of the plain kernel has no recurrent term; a restarting row enters its restart step with zero h and c."""
    R, T, H = 4, 6, 64
    W, b_ih, b_hh, P = make_layer(R, T, H, seed=5)
    hall = torch.randn(R, T, H)
    hp = step_inputs(hall)
    assert torch.equal(hp[:, 0], torch.zeros(R, H)) and torch.equal(hp[:, 1:], hall[:, :-1])
    h0, c0, restart = make_carry(R, H, T, 6)
    hp = step_inputs(hall, h0, restart)
    for r in range(R):
        j = int(restart[r])
        for t in range(T):
            want = torch.zeros(H) if t == j else (h0[r] if t == 0 else hall[r, t - 1])
            assert torch.equal(hp[r, t], want), (r, t)
    b, _ = bias_of(b_ih, b_hh)
    h, c, _, _ = ref_cell(P.to(D) + b, c0, restart)
    r = int(np.flatnonzero(restart == T // 2)[0])
    j = T // 2
    zz = P[r, j].to(D) + b
    i, g = torch.sigmoid(zz[:H]), torch.tanh(zz[2 * H:3 * H])
    assert torch.allclose(c[r, j], i * g, rtol=0, atol=1e-15)      # c_{j-1} dropped


# ------------------------------------------------------------------ the bound sees planted bugs
PLANTS = ["parity", "bias_neighbour", "kblock", "row", "restart_late", "restart_keeps_c", "cfin_late"]


@pytest.mark.parametrize("x3", [0, 1])
@pytest.mark.parametrize("H", [100, 257])
def test_step_bound_catches_planted_bugs(x3, H):
    """The emulated kernel passes its own step bound with room to spare; each planted bug breaks the bound with the
    largest c of either mode (the x3-only operand bugs: with the x3 c)."""
    R, T = 130, 8
    W, b_ih, b_hh, P = make_layer(R, T, H, seed=H + x3)
    h0, c0, restart = make_carry(R, H, T, 7)
    fin = T // 2
    carry = dict(h_init=h0, c_init=c0, restart=restart)
    ok_plain, _ = emulate(P, W, b_ih, b_hh, x3)
    assert step_excess(P, W, b_ih, b_hh, ok_plain, x3) <= 1.0
    ok, ok_c = emulate(P, W, b_ih, b_hh, x3, fin_step=fin, **carry)
    assert step_excess(P, W, b_ih, b_hh, ok, x3, c_fin=ok_c, fin_step=fin, **carry) <= 1.0
    c_max = max(C_BOUND.values())
    unit = H - 2                     # takes the bias of the last unit, in the last (partial) slice at H = 100
    for bug in PLANTS:
        if bug in ("restart_late", "restart_keeps_c", "cfin_late"):
            hall, cf = emulate(P, W, b_ih, b_hh, x3, fin_step=fin, bug=bug, **carry)
            r = step_excess(P, W, b_ih, b_hh, hall, x3, c_fin=cf, fin_step=fin, **carry)
        else:
            hall, _ = emulate(P, W, b_ih, b_hh, x3, bug=bug, bug_row=127, bug_unit=unit)
            r = step_excess(P, W, b_ih, b_hh, hall, x3)
        assert r > c_max, (bug, r)
    if x3:
        for bug in ("h_lo", "w_lo"):
            hall, _ = emulate(P, W, b_ih, b_hh, x3, bug=bug)
            r = step_excess(P, W, b_ih, b_hh, hall, x3)
            assert r > C_BOUND[1], (bug, r)


def test_cfin_one_step_early_is_caught():
    """c stored one step early (after fin_step - 1) breaks the c_fin bound."""
    R, T, H = 9, 6, 64
    W, b_ih, b_hh, P = make_layer(R, T, H, seed=11)
    h0, c0, restart = make_carry(R, H, T, 12)
    carry = dict(h_init=h0, c_init=c0, restart=restart)
    for x3 in (0, 1):
        hall, _ = emulate(P, W, b_ih, b_hh, x3, fin_step=T - 1, **carry)
        _, early = emulate(P, W, b_ih, b_hh, x3, fin_step=T - 2, **carry)
        assert step_excess(P, W, b_ih, b_hh, hall, x3, c_fin=early, fin_step=T - 1, **carry) > max(C_BOUND.values())


# ------------------------------------------------------------------ argument checks (no GPU)
@pytest.fixture(scope="module")
def lib():
    from fullsubnet_b200 import _lib
    return _lib.load()


def test_rec_tc_hooks_refuse_before_any_cuda_call(lib):
    """The recurrence hook, the layer hooks and the Linear hook reject null pointers, non-positive sizes, strides that do
    not cover their extent, a bad fin_step or c_row, carry pointers without a restart table, misaligned P / hall bases and
    short scratch with their error class before any CUDA call: the stand-in pointers are never dereferenced and no device
    is touched.  An unsupported H is reported only after those checks; the layer hooks report an H below the kernel's
    minimum before the workspace, as they always have."""
    from fullsubnet_b200 import _lib
    SH, WS, UN = _lib.FSN_ERR_SHAPE, _lib.FSN_ERR_WORKSPACE, _lib.FSN_ERR_UNSUPPORTED
    p = 1 << 20
    H, T, R = 64, 5, 3
    need = lib.fsn_debug_lstm_rec_tc_scratch_bytes(H, 1)
    assert need > 0 and need == lib.fsn_debug_lstm_rec_tc_scratch_bytes(1000, 0)     # the same for every H and mode

    def rec(w=p, bi=p, bh=p, P=p, p_row=T * 4 * H, p_t=4 * H, hall=p, h_row=T * H, h_t=H, R=R, T=T, H=H, hi=None, ci=None,
            cf=None, c_row=H, rs=None, fin=-1, ws=p, nb=need):
        return lib.fsn_debug_lstm_rec_tc(w, bi, bh, P, p_row, p_t, hall, h_row, h_t, R, T, H, 1, hi, ci, cf, c_row, rs, fin,
                                         None, ws, nb, None)
    carry = dict(hi=p, ci=p, cf=p, rs=p)
    for kw, code in (({"w": None}, SH), ({"bi": None}, SH), ({"bh": None}, SH), ({"P": None}, SH), ({"hall": None}, SH),
                     ({"R": 0}, SH), ({"T": 0}, SH), ({"H": 0}, SH), ({"H": -64}, SH),
                     ({"p_t": 4 * H - 1}, SH), ({"p_row": (T - 1) * 4 * H + 4 * H - 1}, SH), ({"h_t": H - 1}, SH),
                     ({"h_row": (T - 1) * H + H - 1}, SH), ({"p_t": 1 << 62, "p_row": 1 << 62}, SH),
                     ({"hi": p}, SH), ({"ci": p}, SH), ({"cf": p}, SH),
                     (dict(carry, hi=None), SH), (dict(carry, ci=None), SH), (dict(carry, cf=None), SH),
                     (dict(carry, c_row=H - 1), SH), (dict(carry, fin=-2), SH), (dict(carry, fin=T), SH),
                     ({"ws": None}, WS), ({"nb": need - 1}, WS),
                     ({"P": p + 4}, SH), ({"hall": p + 4}, SH),
                     ({"H": 56, "p_row": T * 4 * 56, "p_t": 4 * 56, "h_row": T * 56, "h_t": 56}, UN)):
        assert rec(**kw) == code, kw
    # the tight extents are accepted up to the unsupported-H report (H = 56: no CUDA call is needed to refuse it)
    h = 56
    assert rec(H=h, p_row=(T - 1) * (4 * h + 1) + 4 * h, p_t=4 * h + 1, h_row=(T - 1) * h + h, h_t=h, **carry,
               c_row=h, fin=T - 1) == UN
    assert rec(H=h, p_row=4 * h, p_t=4 * h, h_row=h, h_t=h, T=1) == UN
    # layer hooks: (w_ih, w_hh, b_ih, b_hh, x, R, T, K, H, x3, [h_init, c, restart, fin_step,] hall, ws, ws_bytes)
    K = 33
    lneed = lib.fsn_debug_lstm_tc_workspace_bytes(R, T, K, H, 1)

    def layer(wi=p, wh=p, bi=p, bh=p, x=p, R=R, T=T, K=K, H=H, hall=p, ws=p, nb=lneed):
        return lib.fsn_debug_lstm_layer_tc(wi, wh, bi, bh, x, R, T, K, H, 1, hall, ws, nb, None)

    def carry_layer(hi=p, c=p, rs=p, fin=-1, **kw):
        a = dict(wi=p, wh=p, bi=p, bh=p, x=p, R=R, T=T, K=K, H=H, hall=p, ws=p, nb=lneed)
        a.update(kw)
        return lib.fsn_debug_lstm_tc_carry(a["wi"], a["wh"], a["bi"], a["bh"], a["x"], a["R"], a["T"], a["K"], a["H"], 1, hi, c,
                                           rs, fin, a["hall"], a["ws"], a["nb"], None)
    shape_cases = ({"wi": None}, {"wh": None}, {"bi": None}, {"bh": None}, {"x": None}, {"hall": None}, {"R": 0}, {"T": 0},
                   {"K": 0}, {"H": 0}, {"R": 1 << 16, "T": 1 << 15})
    for kw in shape_cases:
        assert layer(**kw) == SH, kw
        assert carry_layer(**kw) == SH, kw
    for kw in ({"ws": None}, {"nb": lneed - 1}):
        assert layer(**kw) == WS, kw
        assert carry_layer(**kw) == WS, kw
    for kw in ({"hi": None}, {"c": None}, {"rs": None}, {"fin": -2}, {"fin": T}):
        assert carry_layer(**kw) == SH, kw
    small = lib.fsn_debug_lstm_tc_workspace_bytes(R, T, K, 8, 1)
    assert layer(H=8, nb=small) == UN and carry_layer(H=8, nb=small, fin=T - 1) == UN
    # an H below the kernel's minimum is unsupported whatever workspace comes with it; the pointers and shape come first
    for kw in ({"nb": 64}, {"ws": None}):
        assert layer(H=63, **kw) == UN and carry_layer(H=63, **kw) == UN, kw
    assert layer(H=63, x=None) == SH and carry_layer(H=63, R=0) == SH and carry_layer(H=63, hi=None) == SH
    # Linear hook: (x, rows, K, W, bias, N, act, x3, out, ws, ws_bytes)
    N = 20
    nneed = lib.fsn_debug_lstm_tc_workspace_bytes(100, 1, K, max(8, (N + 3) // 4), 1)

    def lin(x=p, rows=100, K=K, W=p, N=N, act=0, out=p, ws=p, nb=nneed):
        return lib.fsn_debug_linear_tc(x, rows, K, W, None, N, act, 1, out, ws, nb, None)
    for kw, code in (({"x": None}, SH), ({"W": None}, SH), ({"out": None}, SH), ({"rows": 0}, SH), ({"K": 0}, SH),
                     ({"N": 0}, SH), ({"act": 4}, SH), ({"act": -1}, SH), ({"N": 65535 * 128 + 1}, SH), ({"ws": None}, WS),
                     ({"nb": nneed - 1}, WS)):
        assert lin(**kw) == code, kw
