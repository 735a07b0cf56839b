"""The kernels around the training step alone against float64: fsn_clip_adam / fsn_clip_adam_steps and FusedClipAdam,
fsn_mse_loss, fsn_build_cirm / fsn_compress_cirm / fsn_decompress_cirm, fsn_drop_band, fsn_si_sdr, fsn_rir_convolve and
fsn_snr_mix, against the references of tests/test_cpu_train_kernels.py (each pinned there to torch, numpy / scipy or a
golden of the reference code).

Every call also checks: the guard floats past each output are untouched, every output element is written (outputs are
filled with a sentinel first; buffers updated in place are compared element by element), two runs give the same bits,
and for the one-CTA-per-clip kernels (rir_convolve, snr_mix, si_sdr) a clip inside a batch gives the bits it gives
alone.  drop_band and rir_convolve are bit-exact.  The
other bounds are about 4x the worst error measured on an H100 for each family (printed with -s as
`[train kernels] family worst`)."""
import copy
import ctypes as C

import numpy as np
import pytest
import torch

from test_cpu_train_kernels import (EPS_CIRM, ref_build_cirm, ref_cirm_ratio, ref_clip_adam, ref_compress,
                                    ref_decompress, ref_drop_band, ref_mse, ref_rir_convolve, ref_si_sdr, ref_snr_mix,
                                    torch_clip_adam_run)
from test_gpu_dsp import GUARD, SENT, Out, _bits

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
F32 = np.float32
# bounds about 4x the worst error measured on an H100 80GB HBM3 (700 W); units in the comment of each family
TOL = {
    "adam_norm": 4e-7,        # |norm - ref| / ref, and the same for the applied coefficient
    "adam_grad": 6e-7,        # |g - ref| / |ref| per element (the clipped gradient written back)
    "adam_m": 7e-7,           # |m - ref| / (b1 |m_prev| + (1 - b1) |g|) per element
    "adam_v": 1.5e-6,         # |v - ref| / (b2 v_prev + (1 - b2) g^2) per element
    "adam_dp": 1.5e-5,        # (|p - ref| - ulp(p) / 2) / lr per element
    "adam_traj50": 7e-3,      # |p - ref| / lr after 50 steps, each side from its own state
    "fused_vs_torch": 1e-3,   # |p - p_torch| / lr, FusedClipAdam against torch.optim.Adam + clip_grad_norm_ (CUDA fp32)
    "mse_loss": 3e-7,         # |loss - ref| / ref
    "mse_grad": 5e-7,         # |dcrm - ref| / |ref| per element
    "compress": 7e-7,         # |out - ref| / K
    "decompress": 6e-7,       # |out - ref| / (K + |ref|)
    "cirm": 2.5e-6,           # |out - ref| / (1 + kappa): kappa = (|a c| + |b d|) / (|noisy|^2 + eps), the ratio's scale
    "cirm_near_zero": 2.5e-6, # the same against the float32 evaluation of the formula, |noisy|^2 < 1e-4
    "si_sdr": 1.5e-5,         # |dB - ref dB|
    "snr_mix": 6e-7,          # |out - ref| / max|ref| of the row
}
WORST = {}
RECORD = {}


def _note(family, err):
    err = float(err)
    WORST[family] = max(WORST.get(family, 0.0), err)
    assert err < TOL[family], (family, err)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k, v in sorted(WORST.items()):
        print(f"[train kernels] {k} worst {v:.3e} (bound {TOL[k]:.1e})")
    for k, v in sorted(RECORD.items()):
        print(f"[train kernels] {k} {v:.3e} (recorded, not asserted)")


@pytest.fixture(scope="module")
def lib():
    from fullsubnet_b200 import _lib
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return _lib.load()


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, F32)).to(DEV)


def _stream():
    from fullsubnet_b200 import _lib
    return _lib.stream_ptr(DEV)


def _same_bits(a, b):
    return np.array_equal(_bits(np.asarray(a, F32)), _bits(np.asarray(b, F32)))


# ------------------------------------------------------------------ clip + Adam
class InPlace:
    """A device copy of a float32 array that a kernel updates in place, with GUARD sentinel floats behind it."""

    def __init__(self, a):
        self.n = a.size
        self.buf = torch.cat([torch.from_numpy(np.ascontiguousarray(a, F32).reshape(-1)),
                              torch.full((GUARD,), SENT, dtype=torch.float32)]).to(DEV)
        self.ptr = self.buf.data_ptr()

    def get(self):
        b = self.buf.cpu().numpy()
        assert np.all(_bits(b[self.n:]) == _bits(np.full(GUARD, SENT, F32))), "guard floats overwritten"
        return b[:self.n].copy()


def run_clip_adam(lib, p, g, m, v, steps, max_norm, grad_scale, lr, b1, b2, eps, single=False):
    """One call on float32 copies of the lists p, g, m, v (steps: one per tensor; single: fsn_clip_adam with steps[0]).
    Returns (norm_out [2], p, g, m, v) as float32 arrays."""
    from fullsubnet_b200 import _lib
    n = len(p)
    L = _lib.ParamList()
    L.n = n
    keep = []
    for i in range(n):
        t = [InPlace(x[i]) for x in (p, g, m, v)]
        keep.append(t)
        L.param[i], L.grad[i], L.exp_avg[i], L.exp_avg_sq[i] = (x.ptr for x in t)
        L.numel[i] = t[0].n
    scratch = torch.empty(lib.fsn_clip_adam_scratch_bytes(), dtype=torch.uint8, device=DEV)
    norm = Out((2,))
    args = (float(max_norm), float(grad_scale), float(lr), float(b1), float(b2), float(eps))
    if single:
        assert len(set(steps)) == 1
        rc = lib.fsn_clip_adam(C.byref(L), *args, int(steps[0]), norm.ptr, scratch.data_ptr(), scratch.numel(), _stream())
    else:
        st = (C.c_int * n)(*steps)
        rc = lib.fsn_clip_adam_steps(C.byref(L), *args, st, norm.ptr, scratch.data_ptr(), scratch.numel(), _stream())
    _lib.check(rc)
    torch.cuda.synchronize()
    out = [[t[k].get() for t in keep] for k in range(4)]
    return (norm.get(), *out)


def _f32(x):
    return float(F32(x))


def check_clip_adam_step(lib, p, g, m, v, steps, max_norm, grad_scale, lr, b1, b2, eps, single=False):
    """One kernel step against the float64 reference from the same (float32) state; returns the kernel's state."""
    got = run_clip_adam(lib, p, g, m, v, steps, max_norm, grad_scale, lr, b1, b2, eps, single)
    nk, pk, gk, mk, vk = got
    # the reference receives the float32 values the kernel receives
    fl, f1, f2, fe = _f32(lr), _f32(b1), _f32(b2), _f32(eps)
    norm, coef, gr, mr, vr, pr = ref_clip_adam(p, g, m, v, steps, _f32(max_norm), _f32(grad_scale), fl, f1, f2, fe)
    _note("adam_norm", abs(nk[0] - norm * 1.0) / norm)
    _note("adam_norm", abs(nk[1] - coef) / coef)
    if max_norm <= 0:
        assert nk[1] == F32(grad_scale)
    for i in range(len(p)):
        _note("adam_grad", (np.abs(gk[i] - gr[i]) / np.maximum(np.abs(gr[i]), 1e-38)).max())
        gi = np.abs(gr[i])
        _note("adam_m", (np.abs(mk[i] - mr[i]) / (f1 * np.abs(m[i]) + (1 - f1) * gi + 1e-38)).max())
        _note("adam_v", (np.abs(vk[i] - vr[i]) / (f2 * np.asarray(v[i], np.float64) + (1 - f2) * gi * gi + 1e-38)).max())
        ulp = np.spacing(np.abs(pk[i])).astype(np.float64)
        _note("adam_dp", (np.maximum(np.abs(pk[i] - pr[i]) - 0.5 * ulp, 0.0) / fl).max())
    return pk, gk, mk, vk, nk


POOL = [1, 255, 256, 257, 8191, 8192, 8193, 32769]
HYPER = [(1e-3, 0.9, 0.999, 1e-8), (3e-4, 0.8, 0.99, 1e-6)]


def _grads(rng, sizes):
    return [(rng.standard_normal(n) * 10 ** rng.uniform(-3, 1)).astype(F32) for n in sizes]


def _state(rng, sizes, g, start):
    """(p, m, v) for a tensor list about to take step `start`: zeros at step 1, else an Adam-like state (v >= m^2)."""
    p = [rng.standard_normal(n).astype(F32) for n in sizes]
    if start == 1:
        return p, [np.zeros(n, F32) for n in sizes], [np.zeros(n, F32) for n in sizes]
    m = [(gi * rng.uniform(-1, 1, gi.shape)).astype(F32) for gi in g]
    v = [(mi.astype(np.float64) ** 2 * rng.uniform(1, 4, mi.shape) + 1e-12).astype(F32) for mi in m]
    return p, m, v


def _total_norm(g, scale):
    return float(np.sqrt(sum(float((x.astype(np.float64) ** 2).sum()) for x in g))) * scale


CASES = [  # (tensor sizes, clip: active / inactive / off, grad_scale, first steps per tensor, hyper-parameter set)
    ([POOL[3]], "active", 1.0, [1], 0),
    ([POOL[0]], "off", 0.25, [2], 1),
    ([16 * 1024 * 1024 + 3], "active", 1 / 3, [10], 0),
    (POOL[1:], "inactive", 1.0, [1000] * 7, 1),
    (POOL[:7], "active", 0.25, [1, 2, 10, 1000, 1, 2, 10], 0),
    (POOL[1:], "off", 1 / 3, [10] * 7, 0),
    ([POOL[i % 8] for i in range(64)], "active", 1 / 3, [(1, 2, 10, 1000)[i % 4] for i in range(64)], 1),
    ([POOL[(i * 3) % 8] for i in range(64)], "inactive", 0.25, [1] * 64, 0),
    ([POOL[(i * 5) % 8] for i in range(64)], "off", 1.0, [1000] * 64, 1),
]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_clip_adam_matches_float64(lib, case):
    """Three consecutive steps, each from the kernel's own state; equal steps also through fsn_clip_adam, bit for bit
    the same as fsn_clip_adam_steps."""
    sizes, clip, scale, steps, h = CASES[case]
    lr, b1, b2, eps = HYPER[h]
    rng = np.random.default_rng(100 + case)
    g = _grads(rng, sizes)
    p, m, v = _state(rng, sizes, g, min(steps))
    equal = len(set(steps)) == 1
    for it in range(3):
        nrm = _total_norm(g, scale)
        max_norm = {"active": 0.3 * nrm, "inactive": 3.0 * nrm, "off": 0.0}[clip]
        st = [s + it for s in steps]
        if equal:
            a = run_clip_adam(lib, p, g, m, v, st, max_norm, scale, lr, b1, b2, eps, single=True)
            b = run_clip_adam(lib, p, g, m, v, st, max_norm, scale, lr, b1, b2, eps)
            for x, y in zip(a[1:], b[1:]):
                assert all(_same_bits(xi, yi) for xi, yi in zip(x, y))
            assert _same_bits(a[0], b[0])
        out = check_clip_adam_step(lib, p, g, m, v, st, max_norm, scale, lr, b1, b2, eps)
        again = run_clip_adam(lib, p, g, m, v, st, max_norm, scale, lr, b1, b2, eps)
        for x, y in zip(out[:4], again[1:]):
            assert all(_same_bits(xi, yi) for xi, yi in zip(x, y)), "two runs differ"
        p, _, m, v, _ = out
        g = _grads(rng, sizes)


def test_clip_adam_trajectory_50_steps(lib):
    """50 steps over 7 tensors with the clip active; kernel and float64 reference each carry their own state."""
    sizes = POOL[1:]
    lr, b1, b2, eps = HYPER[0]
    rng = np.random.default_rng(5)
    p = [rng.standard_normal(n).astype(F32) for n in sizes]
    m = [np.zeros(n, F32) for n in sizes]
    v = [np.zeros(n, F32) for n in sizes]
    pr, mr, vr = [x.astype(np.float64) for x in p], [x.astype(np.float64) for x in m], [x.astype(np.float64) for x in v]
    for s in range(1, 51):
        g = _grads(rng, sizes)
        max_norm = 0.5 * _total_norm(g, 1.0)
        _, p, _, m, v = run_clip_adam(lib, p, g, m, v, [s] * 7, max_norm, 1.0, lr, b1, b2, eps)
        *_, mr, vr, pr = ref_clip_adam(pr, g, mr, vr, [s] * 7, _f32(max_norm), 1.0, _f32(lr), _f32(b1), _f32(b2),
                                       _f32(eps))
    _note("adam_traj50", max(np.abs(p[i] - pr[i]).max() for i in range(7)) / _f32(lr))


def test_clip_adam_bias_correction_drift_is_recorded(lib):
    """The kernel takes beta1 / beta2 as floats and forms the bias corrections with powf; torch.optim.Adam uses the
    Python doubles.  Recorded: the largest relative difference of the step factor lr / bc1 / sqrt(bc2) over steps
    1..1000, and how far a 1000-step run of the kernel drifts from torch.optim.Adam (float64, double betas)."""
    lr, b1, b2, eps = 1e-3, 0.9, 0.999, 1e-8
    s = np.arange(1, 1001)
    f32 = F32(lr) / (F32(1) - np.power(F32(b1), s.astype(F32))) / np.sqrt(F32(1) - np.power(F32(b2), s.astype(F32)))
    f64 = lr / (1 - b1 ** s.astype(np.float64)) / np.sqrt(1 - b2 ** s.astype(np.float64))
    RECORD["bias_correction_drift_rel_1000"] = float(np.abs(f32 / f64 - 1).max())
    from fullsubnet_b200 import _lib
    rng = np.random.default_rng(9)
    n = 4096
    p0 = rng.standard_normal(n).astype(F32)
    gs = rng.standard_normal((1000, n)).astype(F32)
    p, m, v = _dev(p0), torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    gd = _dev(gs)
    L = _lib.ParamList()
    L.n = 1
    L.param[0], L.exp_avg[0], L.exp_avg_sq[0], L.numel[0] = p.data_ptr(), m.data_ptr(), v.data_ptr(), n
    scratch = torch.empty(lib.fsn_clip_adam_scratch_bytes(), dtype=torch.uint8, device=DEV)
    for k in range(1000):
        L.grad[0] = gd[k].data_ptr()
        _lib.check(lib.fsn_clip_adam(C.byref(L), 0.0, 1.0, lr, b1, b2, eps, k + 1, None, scratch.data_ptr(),
                                     scratch.numel(), _stream()))
    pt = torch.nn.Parameter(torch.from_numpy(p0.astype(np.float64)))
    opt = torch.optim.Adam([pt], lr=lr, betas=(b1, b2), eps=eps, foreach=False)
    for k in range(1000):
        pt.grad = torch.from_numpy(gs[k].astype(np.float64))
        opt.step()
    RECORD["adam_1000_steps_vs_torch_in_lr"] = float(np.abs(p.cpu().numpy() - pt.detach().numpy()).max() / lr)


@pytest.mark.parametrize("bad", [np.nan, np.inf])
@pytest.mark.parametrize("clip", [0.0, 1.0])
def test_clip_adam_nonfinite_gradient_pattern(lib, bad, clip):
    """A NaN or an inf in one gradient: the NaN / zero pattern of the gradients, moments and parameters is the one of
    clip_grad_norm_ + torch.optim.Adam (float64); no fault."""
    rng = np.random.default_rng(11)
    sizes = [300, 9000]
    g = _grads(rng, sizes)
    g[1][4321] = bad
    p = [rng.standard_normal(n).astype(F32) for n in sizes]
    z = [np.zeros(n, F32) for n in sizes]
    _, pk, gk, mk, vk = run_clip_adam(lib, p, g, z, z, [1, 1], clip, 1.0, 1e-3, 0.9, 0.999, 1e-8)
    traj, clipped, opt = torch_clip_adam_run(p, [g], clip, 1.0, 1e-3, 0.9, 0.999, 1e-8)
    for i in range(2):
        st = opt.state[opt.param_groups[0]["params"][i]]
        for got, want in ((gk[i], clipped[0][i]), (pk[i], traj[0][i]), (mk[i], st["exp_avg"].numpy()),
                          (vk[i], st["exp_avg_sq"].numpy())):
            assert np.array_equal(np.isnan(got), np.isnan(want))
            assert np.array_equal(got == 0, want == 0)
            assert np.array_equal(np.isinf(got), np.isinf(want)) and np.all(got[np.isinf(want)] == want[np.isinf(want)])
            ok = np.isfinite(want)
            assert np.abs(got[ok] - want[ok]).max(initial=0) <= 1e-5 * max(np.abs(want[ok]).max(initial=0), 1.0)


# ------------------------------------------------------------------ FusedClipAdam against torch.optim.Adam
def _fused_vs_torch(params, grad_seq, max_norm, torch_state=None, torch_pre=None):
    """FusedClipAdam and clip_grad_norm_ + torch.optim.Adam(foreach=False), both CUDA float32, over grad_seq; optional
    torch_pre steps of torch.optim.Adam first, whose state_dict FusedClipAdam then loads.  Returns the worst |dp| / lr."""
    from fullsubnet_b200.optim import FusedClipAdam
    lr = 1e-3
    tp = [torch.nn.Parameter(_dev(p)) for p in params]
    topt = torch.optim.Adam(tp, lr=lr, foreach=False)

    def torch_step(grads):
        for p, g in zip(tp, grads):
            p.grad = None if g is None else _dev(g)
        if max_norm:
            torch.nn.utils.clip_grad_norm_([p for p in tp if p.grad is not None], max_norm)
        topt.step()

    for grads in torch_pre or []:
        torch_step(grads)
    fp = [torch.nn.Parameter(p.detach().clone()) for p in tp]
    fopt = FusedClipAdam(fp, lr=lr, max_norm=max_norm)
    if torch_pre:  # a checkpoint written and read back: torch's state_dict() holds its live state tensors
        fopt.load_state_dict(copy.deepcopy(topt.state_dict()))
    worst = 0.0
    for grads in grad_seq:
        torch_step(grads)
        for p, g in zip(fp, grads):
            p.grad = None if g is None else _dev(g)
        fopt.step()
        torch.cuda.synchronize()
        for a, b in zip(fp, tp):
            x, y = a.detach().cpu().numpy(), b.detach().cpu().numpy()
            worst = max(worst, float((np.maximum(np.abs(x - y) - np.spacing(np.abs(y)), 0)).max() / lr))
        assert [int(fopt.state[a]["step"]) if fopt.state[a] else 0 for a in fp] == \
               [int(topt.state[b]["step"]) if topt.state[b] else 0 for b in tp]
    return worst


@pytest.mark.parametrize("where", ["first", "last"])
def test_fused_clip_adam_parameter_without_grad_in_first_step(where):
    """torch.optim.Adam skips a parameter whose grad is None and keeps its step count; FusedClipAdam must too.  With
    one step count for the whole call, the parameter that missed a step takes the others' bias correction (first in
    the list), or every other parameter takes its own (last in the list)."""
    rng = np.random.default_rng(21)
    sizes = [300, 17, 1000]
    k = 0 if where == "first" else 2
    params = [rng.standard_normal(n).astype(F32) for n in sizes]
    seq = [_grads(rng, sizes) for _ in range(5)]
    seq[0][k] = None
    for max_norm in (None, 1.0):
        _note("fused_vs_torch", _fused_vs_torch(params, seq, max_norm))


def test_fused_clip_adam_resumes_torch_checkpoint_with_unequal_steps():
    """A torch.optim.Adam state_dict whose parameters have different step counts (one had no grad for two steps)."""
    rng = np.random.default_rng(22)
    sizes = [64, 4097, 5]
    params = [rng.standard_normal(n).astype(F32) for n in sizes]
    pre = [_grads(rng, sizes) for _ in range(4)]
    pre[0][1] = pre[1][1] = None
    seq = [_grads(rng, sizes) for _ in range(4)]
    for max_norm in (None, 0.5):
        _note("fused_vs_torch", _fused_vs_torch(params, seq, max_norm, torch_pre=pre))


# ------------------------------------------------------------------ MSE
def run_mse(lib, cirm, crm, with_dcrm=True):
    from fullsubnet_b200 import _lib
    B, _, F, T = crm.shape
    loss = Out((1,))
    d = Out(crm.shape) if with_dcrm else None
    scratch = torch.empty(lib.fsn_mse_loss_scratch_bytes(), dtype=torch.uint8, device=DEV)
    a, b = _dev(cirm), _dev(crm)
    _lib.check(lib.fsn_mse_loss(a.data_ptr(), b.data_ptr(), B, F, T, loss.ptr, None if d is None else d.ptr,
                                scratch.data_ptr(), scratch.numel(), _stream()))
    torch.cuda.synchronize()
    assert _same_bits(a.cpu().numpy(), cirm) and _same_bits(b.cpu().numpy(), crm), "an input was written"
    return loss.get()[0], None if d is None else d.get()


@pytest.mark.parametrize("B,F,T", [(1, 3, 5), (2, 7, 9), (1, 1, 131071), (2, 256, 256), (1, 3, 43691), (32, 257, 193),
                                   (1, 1, 1), (300, 1, 1), (1, 257, 1), (4, 1, 777), (1, 1000, 3)])
def test_mse_loss_matches_float64(lib, B, F, T):
    """n = 2BFT below one CTA, at 262144 and 262144 +- 2 (the MSE_BLOCKS cap and its grid-stride loop), ~3.2 M, and B, F
    or T equal to 1"""
    rng = np.random.default_rng(B * 7 + F * 3 + T)
    cirm = rng.uniform(-10, 10, (B, F, T, 2)).astype(F32)
    crm = (cirm.transpose(0, 3, 1, 2) + rng.standard_normal((B, 2, F, T)) * 10 ** rng.uniform(-3, 0)).astype(F32)
    crm.reshape(-1)[::97] = cirm.transpose(0, 3, 1, 2).reshape(-1)[::97]  # exact zeros of the difference
    loss, d = run_mse(lib, cirm, crm)
    ref, dref = ref_mse(cirm, crm)
    _note("mse_loss", abs(loss - ref) / ref)
    assert np.all(_bits(d.reshape(-1)[::97]) == 0)
    _note("mse_grad", (np.abs(d - dref) / np.maximum(np.abs(dref), 1e-38)).max())
    loss2, d2 = run_mse(lib, cirm, crm)
    assert _same_bits(loss2, loss) and _same_bits(d2, d)
    loss3, _ = run_mse(lib, cirm, crm, with_dcrm=False)  # dcrm = NULL: the same loss, nothing else written
    assert _same_bits(loss3, loss)


# ------------------------------------------------------------------ compress / decompress / cIRM
EW_PASS = 132 * 16 * 256  # elements per pass of ew_grid
EW_SIZES = [0, 1, 257, EW_PASS, 3 * EW_PASS + 1]


def _unary(lib, fn, x, *args):
    xd = _dev(x) if x.size else torch.zeros(1, device=DEV)
    o = Out(x.shape)
    from fullsubnet_b200 import _lib
    _lib.check(fn(xd.data_ptr(), o.ptr, x.size, *args, _stream()))
    torch.cuda.synchronize()
    return o.get()


def _specials(x, vals):
    x = x.copy()
    k = min(len(vals), x.size)
    x[:k] = np.asarray(vals, F32)[:k]
    return x


@pytest.mark.parametrize("n", EW_SIZES)
@pytest.mark.parametrize("K,Cc", [(10.0, 0.1), (4.0, 0.5)])
def test_compress_cirm_matches_float64(lib, n, K, Cc):
    rng = np.random.default_rng(n + int(K))
    x = _specials(rng.uniform(-150, 150, n).astype(F32),
                  [-1e30, -100.0, np.nextafter(F32(-100), F32(0)), np.nextafter(F32(-100), F32(-200)), -99.0, 0.0,
                   1e-30, -1e-30, 1e30, np.inf, -np.inf, np.nan, 250.0, 1e-3])
    got = _unary(lib, lib.fsn_compress_cirm, x, K, Cc)
    ref = ref_compress(x, K, _f32(Cc))
    assert np.array_equal(np.isnan(got), np.isnan(ref))
    ok = ~np.isnan(ref)
    if ok.any():
        _note("compress", (np.abs(got[ok] - ref[ok]) / K).max())
    assert _same_bits(_unary(lib, lib.fsn_compress_cirm, x, K, Cc), got)


@pytest.mark.parametrize("n", EW_SIZES)
def test_decompress_cirm_matches_float64(lib, n):
    rng = np.random.default_rng(n + 1)
    lim = F32(9.9)
    x = _specials(rng.uniform(-12, 12, n).astype(F32),
                  [lim, -lim, np.nextafter(lim, F32(0)), np.nextafter(-lim, F32(0)), np.nextafter(lim, F32(20)),
                   np.nextafter(-lim, F32(-20)), np.nan, np.inf, -np.inf, 0.0, 1e30, -1e30, 1e-30, 9.0])
    got = _unary(lib, lib.fsn_decompress_cirm, x, 10.0, 9.9)
    ref = ref_decompress(x)
    assert not np.any(np.isnan(got))
    _note("decompress", (np.abs(got - ref) / (10.0 + np.abs(ref))).max(initial=0))
    if n >= 7:
        assert got[6] == 0  # NaN -> 0
        assert got[0] == got[4] and got[1] == got[5]  # beyond +-9.9: the value at +-9.9
        assert got[2] < got[0] and got[3] > got[1]  # just inside: less saturated
    assert _same_bits(_unary(lib, lib.fsn_decompress_cirm, x, 10.0, 9.9), got)


def _cirm_inputs(rng, n):
    mag = 10 ** rng.uniform(-4, 1, n)
    a, b = (mag * rng.standard_normal(n)).astype(F32), (mag * rng.standard_normal(n)).astype(F32)
    c, d = rng.standard_normal(n).astype(F32), rng.standard_normal(n).astype(F32)
    q = max(n // 8, 1)
    a[:q:4], b[:q:4] = 0, 0                                              # exactly zero noisy bins
    a[1:q:4], b[1:q:4] = (1e-5 * rng.standard_normal((2, len(a[1:q:4])))).astype(F32)  # near zero
    c[2:q:4], d[2:q:4] = -300 * a[2:q:4], -300 * b[2:q:4]                   # real ratio -300: the -100 clamp
    c[3:q:4], d[3:q:4] = 1e4 * a[3:q:4], 1e4 * b[3:q:4]                     # +1e4: saturated at +10
    return a, b, c, d


def _cirm_f32(a, b, c, d):
    """the float32 evaluation of the same formula (numpy, no fused multiply-adds)"""
    with np.errstate(all="ignore"):
        den = a * a + b * b + F32(EPS_CIRM)
        out = []
        for r in ((a * c + b * d) / den, (a * d - b * c) / den):
            r = np.where(r <= F32(-100), F32(-100), r)
            e = np.exp(F32(-0.1) * r)
            out.append(F32(10) * (F32(1) - e) / (F32(1) + e))
    return np.stack(out, -1)


@pytest.mark.parametrize("n", EW_SIZES)
def test_build_cirm_matches_float64(lib, n):
    from fullsubnet_b200 import _lib
    rng = np.random.default_rng(n + 2)
    a, b, c, d = _cirm_inputs(rng, n)
    ins = [_dev(x) if n else torch.zeros(1, device=DEV) for x in (a, b, c, d)]
    o = Out((n, 2))

    def run():
        _lib.check(lib.fsn_build_cirm(*(t.data_ptr() for t in ins), o.ptr, n, _stream()))
        torch.cuda.synchronize()
        return o.get()
    got = run()
    assert _same_bits(run(), got)
    if n == 0:
        return
    ref = ref_build_cirm(a, b, c, d)
    A, Bb, Cc, D = (np.abs(x.astype(np.float64)) for x in (a, b, c, d))
    den = A * A + Bb * Bb + EPS_CIRM
    kappa = np.stack([(A * Cc + Bb * D) / den, (A * D + Bb * Cc) / den], -1)
    err = np.abs(got - ref) / (1 + kappa)
    near = den < 1e-4
    _note("cirm", err[~near].max(initial=0))
    if near.any():
        _note("cirm_near_zero", (np.abs(got - _cirm_f32(a, b, c, d)) / (1 + kappa))[near].max())
    zero = (a == 0) & (b == 0)
    assert np.all(got[zero] == 0)
    re, _ = ref_cirm_ratio(a, b, c, d)
    assert np.all(np.abs(got[re <= -100, 0] - ref_compress(-100.0)) <= 1e-5)
    sat = re > 1e3
    assert np.all(np.abs(got[sat, 0] - 10) <= 1e-5)


# ------------------------------------------------------------------ drop_band
@pytest.mark.parametrize("G", [2, 3, 4, 7])
def test_drop_band_is_bit_exact(lib, G):
    from fullsubnet_b200 import _lib
    rng = np.random.default_rng(G)
    shapes = [(B, Cc, F, 5) for B in (G + 1, 2 * G + 1, 33) for Cc in (1, 2) for F in (3 * G, 3 * G + G - 1)]
    shapes.append((33, 2, 257, 193))  # beyond one ew_grid pass
    for B, Cc, F, T in shapes:
        x = rng.standard_normal((B, Cc, F, T)).astype(F32)
        xd = _dev(x)
        o = Out((B, Cc, F // G, T))
        for _ in range(2):
            _lib.check(lib.fsn_drop_band(xd.data_ptr(), o.ptr, B, Cc, F, T, G, _stream()))
            torch.cuda.synchronize()
            assert _same_bits(o.get(), ref_drop_band(x, G)), (B, Cc, F, T)
            o = Out((B, Cc, F // G, T))


# ------------------------------------------------------------------ SI-SDR
def run_si_sdr(lib, r, e):
    from fullsubnet_b200 import _lib
    B = r.shape[0]
    o = Out((B,))
    rd, ed = _dev(r), _dev(e)
    _lib.check(lib.fsn_si_sdr(rd.data_ptr(), ed.data_ptr(), B, r.shape[1], o.ptr, _stream()))
    torch.cuda.synchronize()
    return o.get()


def _si_sdr_pair(rng, B, L, snrs):
    r = rng.standard_normal((B, L)) * (0.2 + np.abs(np.sin(np.arange(L) / 500.0)))
    n = rng.standard_normal((B, L))
    s = np.asarray(snrs, np.float64)[:, None]
    n *= np.sqrt((r * r).sum(1, keepdims=True) / (n * n).sum(1, keepdims=True)) * 10 ** (-s / 20)
    return r.astype(F32), (r * rng.uniform(0.5, 2.0, (B, 1)) + n).astype(F32)


def check_si_sdr(lib, r, e):
    got = run_si_sdr(lib, r, e)
    ref = ref_si_sdr(r, e)
    fin = np.isfinite(ref)
    assert np.array_equal(got[~fin], ref[~fin].astype(F32))
    if fin.any():
        _note("si_sdr", np.abs(got[fin] - ref[fin]).max())
    assert _same_bits(run_si_sdr(lib, r, e), got)
    for b in sorted({0, r.shape[0] - 1}):
        assert _same_bits(run_si_sdr(lib, r[b:b + 1], e[b:b + 1]), got[b:b + 1]), b
    return got


@pytest.mark.parametrize("L", [255, 256, 257, 49152, 160000])
def test_si_sdr_matches_float64(lib, L):
    rng = np.random.default_rng(L)
    snrs = [-20, -10, 0, 10, 20, 30, 40]
    r, e = _si_sdr_pair(rng, len(snrs), L, snrs)
    e[3] = r[3]  # est = ref: +inf, as the reference gives
    got = check_si_sdr(lib, r, e)
    assert got[3] == np.inf


def test_si_sdr_one_sample_and_300_clips(lib):
    rng = np.random.default_rng(1)
    r = rng.standard_normal((3, 1)).astype(F32)
    got = check_si_sdr(lib, r, np.stack([r[0], 2 * r[1], r[2]]))  # one sample: est a multiple of ref, noise 0
    assert np.all(got == np.inf)
    snrs = np.linspace(-20, 40, 300)
    check_si_sdr(lib, *_si_sdr_pair(rng, 300, 4001, snrs))


# ------------------------------------------------------------------ RIR convolution
CT, CR = 128, 9
CO, CK = CT * CR, 128 * CR


def run_rir(lib, x, rir, lens):
    from fullsubnet_b200 import _lib
    B, L = x.shape
    o = Out((B, L))
    xd, rd = _dev(x), _dev(rir)
    ld = None if lens is None else torch.tensor(lens, dtype=torch.int32, device=DEV)
    _lib.check(lib.fsn_rir_convolve(xd.data_ptr(), rd.data_ptr(), _lib.ptr(ld), B, L, rir.shape[1], o.ptr, _stream()))
    torch.cuda.synchronize()
    return o.get()


def check_rir(lib, x, rir, lens):
    got = run_rir(lib, x, rir, lens)
    B, Lr = rir.shape
    for b in range(B):
        lr = Lr if lens is None else min(lens[b], Lr)
        assert _same_bits(got[b], ref_rir_convolve(x[b], rir[b], lr)[0]), (b, lr)
    assert _same_bits(run_rir(lib, x, rir, lens), got)
    for b in sorted({0, B - 1}):
        one = run_rir(lib, x[b:b + 1], rir[b:b + 1], None if lens is None else [lens[b]])
        assert _same_bits(one, got[b:b + 1]), b


def _rir(rng, B, Lr):
    return (rng.standard_normal((B, Lr)) * np.exp(-np.arange(Lr) / 400.0)).astype(F32)


@pytest.mark.parametrize("L", [5, CO - 1, CO, CO + 1, 3000])
def test_rir_convolve_is_bit_exact(lib, L):
    """rir_len 0 (copy), 1, CR, CK - 1, CK, CK + 1, 2 CK + 5, and beyond Lr_max (clamped); L below CR, at the CTA's CO
    outputs and either side, and shorter than the RIR"""
    rng = np.random.default_rng(L)
    lens = [0, 1, CR, CK - 1, CK, CK + 1, 2 * CK + 5, 5000]
    Lr = 2 * CK + 5
    x = rng.standard_normal((len(lens), L)).astype(F32)
    check_rir(lib, x, _rir(rng, len(lens), Lr), lens)
    check_rir(lib, x[:3], _rir(rng, 3, CK + 1), None)  # rir_len = NULL: Lr_max taps everywhere


def test_rir_convolve_mixed_clips(lib):
    rng = np.random.default_rng(77)
    lens = [300, 0, 16000, 2, 7000, 11, 16000, 1153]
    L = 6 * CO + 17
    x = (0.3 * rng.standard_normal((len(lens), L))).astype(F32)
    check_rir(lib, x, _rir(rng, len(lens), 16000), lens)


# ------------------------------------------------------------------ snr_mix
def run_snr_mix(lib, clean, noise, snr, nt, target=-25.0, eps=1e-6):
    from fullsubnet_b200 import _lib
    B, L = clean.shape
    y, c = Out((B, L)), Out((B, L))
    ins = [_dev(a) for a in (clean, noise, snr, nt)]
    _lib.check(lib.fsn_snr_mix(*(t.data_ptr() for t in ins), target, eps, B, L, y.ptr, c.ptr, _stream()))
    torch.cuda.synchronize()
    return y.get(), c.get()


def check_snr_mix(lib, clean, noise, snr, nt):
    y, c = run_snr_mix(lib, clean, noise, snr, nt)
    clipped = []
    for b in range(clean.shape[0]):
        yr, cr, peak = ref_snr_mix(clean[b], noise[b], float(snr[b]), -25.0, float(nt[b]))
        assert abs(peak - 0.999) >= 1e-4, (b, peak)  # a float / double difference cannot flip the branch
        clipped.append(peak > 0.999)
        if not np.any(clean[b]):
            assert np.all(_bits(y[b]) == 0) and np.all(_bits(c[b]) == 0)
            continue
        s = np.abs(yr).max()
        _note("snr_mix", max(np.abs(y[b] - yr).max(), np.abs(c[b] - cr).max()) / s)
    y2, c2 = run_snr_mix(lib, clean, noise, snr, nt)
    assert _same_bits(y2, y) and _same_bits(c2, c)
    for b in sorted({0, clean.shape[0] - 1}):
        y1, c1 = run_snr_mix(lib, clean[b:b + 1], noise[b:b + 1], snr[b:b + 1], nt[b:b + 1])
        assert _same_bits(y1, y[b:b + 1]) and _same_bits(c1, c[b:b + 1]), b
    return clipped


@pytest.mark.parametrize("L", [1, 1000, 1024, 1025, 49152, 160000])
def test_snr_mix_matches_float64(lib, L):
    """rows: smooth speech-like clips (no rescale), impulsive clips pushed to a loud target (rescale), an all-zero
    noise row and an all-zero clean row"""
    rng = np.random.default_rng(L)
    B = 6
    t = np.arange(L)
    clean = (0.2 * np.sin(2 * np.pi * 0.013 * t) * (1 + 0.5 * np.sin(2 * np.pi * 3e-4 * t))
             + 0.02 * rng.standard_normal((B, L))).astype(F32)
    noise = (0.3 * rng.standard_normal((B, L))).astype(F32)
    for b in (2, 3):
        clean[b] = (0.002 * rng.standard_normal(L)).astype(F32)
        clean[b, ::997] = 0.95
    noise[4] = 0
    clean[5] = 0
    snr = np.array([10, -5, 20, 15, 5, 0], F32)
    nt = np.array([-25, -35, -12, -15, -25, -20], F32)
    clipped = check_snr_mix(lib, clean, noise, snr, nt)
    if L >= 1000:
        assert clipped[2] and clipped[3] and not clipped[0] and not clipped[1]
