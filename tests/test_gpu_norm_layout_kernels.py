"""The norm and frequency-unfold kernels alone against float64: the statistics of the offline norms,
fsn_debug_norm_stats (frame_stats, clip_reduce with and without per-clip lengths, norm_scales) and fsn_debug_train_stats
(train_mag_stats, train_tm_stats), and the backward kernels of the second norm and the unfolds:
fsn_debug_norm_unfold_bwd (train_dot + train_dfbz, train_cum_unit_bwd + train_dfbz_cum), fsn_debug_fast_norm_unfold_bwd
(ftr_dbn, train_dot + ftr_denc<false>, ftr_cum_suffix + ftr_denc<true>) and fsn_debug_imp_unfold_bwd (train_dot +
imp_unfold_bwd, first and later sections), and the forward of the section unfold, fsn_debug_imp_section_input
(imp_section_input), against the torch.autograd references of tests/test_cpu_norm_layout_kernels.py.

The shapes are where the index arithmetic breaks: one bin or one frame, N = 0, 1 and F - 1 (M - 1, Fu - 1), drop_band
with G = 2, 3, 4, 7 not dividing F or B, S = 1, 2, 3 with a partial last block and a last shrunk step that feeds no
frame, improved sections at both edges and with lo > 0, grid-stride kernels past one pass, more than 64 clips and more
than 128 rows, and a 4000-frame cumulative norm.

Every call also checks: the guard floats past each output are untouched, every output element is written (sentinel
fill), two runs give the same bits, and a clip gives the same bits in a batch as alone.  Each error is normalised by
the conditioning of its sum (the sum of the absolute values of the terms, tests/test_cpu_norm_layout_kernels.py);
where that is 0 (an activation's zero derivative, a shrunk step no frame reads) the kernel must give exactly 0.  The
bounds are about 4x the worst error measured on an H100 for each family (printed with -s as
`[norm/unfold bwd] family worst`)."""
import numpy as np
import pytest
import torch

from test_cpu_norm_layout_kernels import (ACT_NONE, ACT_RELU, ACT_RELU6, ACT_TANH, fast_shrunk, imp_section,
                                          ref_fast_bwd, ref_frame_stats, ref_fsn_norm_bwd, ref_imp_bwd, ref_inv)
from test_gpu_dsp import Out, _bits

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
F32 = np.float32
# bounds about 4x the worst error measured on an H100 80GB HBM3 (700 W), |kernel - float64| / conditioning
TOL = {                      # worst measured
    "fsn_dot": 1e-7,         # 2.4e-8  dot[b'] of train_dot over Sum |dX X|
    "fsn_dz": 4.5e-7,        # 1.0e-7  train_dfbz
    "fsn_dz_cum": 5e-7,      # 1.3e-7  train_cum_unit_bwd + train_dfbz_cum
    "fast_dbn": 4.5e-7,      # 1.1e-7  ftr_dbn
    "fast_denc": 5.5e-7,     # 1.3e-7  train_dot + ftr_denc<false>
    "fast_denc_cum": 5.5e-7, # 1.3e-7  ftr_cum_suffix + ftr_denc<true>
    "imp_dfb": 4.5e-7,       # 1.0e-7  train_dot + imp_unfold_bwd over the sections
    "imp_fs": 5.5e-7,        # 1.4e-7  the (b, t) block sums of imp_section_input over Sum |terms|
    "frame_stats": 6e-7,     # 1.5e-7  frame_stats (both sums) over Sum |terms|
    "clip_sums": 4.5e-7,     # 1.0e-7  clip_reduce over Sum |terms|
    "inv": 7.5e-7,           # 1.9e-7  norm_scales' inv1 / inv2, relative
    "train_stats": 4.5e-7,   # 1.1e-7  train_mag_stats / train_tm_stats over Sum |terms|
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
        print(f"[norm/unfold bwd] {k} worst {v:.3e} (bound {TOL[k]:.1e})")
    for k, v in sorted(RECORD.items()):
        print(f"[norm/unfold bwd] {k} {v:.3e} (recorded, not asserted)")


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
    return np.array_equal(_bits(np.ascontiguousarray(a, F32)), _bits(np.ascontiguousarray(b, F32)))


def _cond_err(got, ref, cond):
    """max |got - ref| / cond; where cond is 0 the kernel must give exactly 0."""
    got, ref, cond = (np.asarray(a, np.float64) for a in (got, ref, cond))
    zero = cond == 0
    assert np.all(got[zero] == 0), "a gradient with no terms is not exactly 0"
    return float((np.abs(got - ref)[~zero] / cond[~zero]).max()) if np.any(~zero) else 0.0


def _f32(a):
    return np.asarray(a, np.float64).astype(F32)


# ------------------------------------------------------------------ fullsubnet
def run_fsn(lib, dX, X, fbz, scale, cum, B, F, G, Tp, Ns, act):
    R, K = X.shape[1], X.shape[2]
    d = [_dev(a) for a in (dX, X, fbz, scale)]
    mid, dz = Out((Tp, R) if cum else (B,)), Out((Tp, B, F))
    rc = lib.fsn_debug_norm_unfold_bwd(*[t.data_ptr() for t in d], int(cum), B, F, G, Tp, Ns, float(F * K * Tp), act,
                                       mid.ptr, dz.ptr, _stream())
    torch.cuda.synchronize()
    assert rc == 0, lib.fsn_last_error()
    assert lib.fsn_last_launch_count() == 2
    return mid.get(), dz.get()


def check_fsn(lib, B, F, Tp, Ns, G, act, cum, seed=0, family=None):
    rng = np.random.default_rng(seed)
    Fsub = F // G if G > 1 else F
    R, K = B * Fsub, 2 * Ns + 2
    mag = _f32(rng.random((B, F, Tp)) + 0.05)
    z = _f32(rng.standard_normal((B, F, Tp)) * (4.0 if act == ACT_RELU6 else 1.0))
    if act == ACT_TANH:  # the z whose tanh is a float32: the kernel's y then is the reference's, and so is 1 - y^2
        z = np.arctanh(np.tanh(z).astype(F32).astype(np.float64))
    dX = _f32(rng.standard_normal((Tp, R, K)))
    dz_ref, cond, X, y, scale = ref_fsn_norm_bwd(mag, z, dX, Ns, G, act, cum)
    X, y, scale = _f32(X), _f32(y), _f32(scale)
    mid, dz = run_fsn(lib, dX, X, y, scale, cum, B, F, G, Tp, Ns, act)
    mid2, dz2 = run_fsn(lib, dX, X, y, scale, cum, B, F, G, Tp, Ns, act)
    assert _same_bits(mid, mid2) and _same_bits(dz, dz2)
    err = _cond_err(dz, dz_ref, cond)
    _note(family or ("fsn_dz_cum" if cum else "fsn_dz"), err)
    if not cum:
        p = dX.astype(np.float64) * X.astype(np.float64)
        per = p.reshape(Tp, B, Fsub * K)
        _note("fsn_dot", np.max(np.abs(mid - per.sum(axis=(0, 2))) / np.abs(per).sum(axis=(0, 2))))
    if G <= 1 and B > 1:  # the last clip alone gives the same bits
        b = B - 1
        rows = slice(b * F, (b + 1) * F)
        sc = scale[:, rows] if cum else scale[b:b + 1]
        mid1, dz1 = run_fsn(lib, dX[:, rows], X[:, rows], y[:, b:b + 1], sc, cum, 1, F, G, Tp, Ns, act)
        assert _same_bits(dz1[:, 0], dz[:, b])
        assert _same_bits(mid1, mid[:, rows] if cum else mid[b:b + 1])
    return err


FSN_CASES = [  # B, F, Tp, Ns, G, act
    (1, 2, 1, 0, 1, ACT_NONE),      # two bins, one frame
    (3, 2, 1, 1, 1, ACT_RELU),      # N = F - 1
    (4, 31, 32, 30, 1, ACT_TANH),
    (5, 32, 33, 15, 2, ACT_RELU6),
    (7, 33, 31, 1, 3, ACT_RELU),    # G = 3 divides neither F nor B
    (9, 257, 3, 15, 4, ACT_NONE),   # G = 4, one bin dropped
    (8, 33, 5, 2, 7, ACT_TANH),     # G = 7: 5 bins of each clip dropped
    (70, 257, 33, 2, 2, ACT_RELU),  # 593 k elements: train_dfbz's grid-stride loop takes three passes; 70 CTAs
]


@pytest.mark.parametrize("B,F,Tp,Ns,G,act", FSN_CASES)
def test_fsn_offline_norm_bwd_matches_float64(lib, B, F, Tp, Ns, G, act):
    check_fsn(lib, B, F, Tp, Ns, G, act, cum=False)


@pytest.mark.parametrize("B,F,Tp,Ns,G,act", [
    (1, 2, 1, 1, 1, ACT_NONE),
    (3, 33, 33, 2, 1, ACT_RELU),
    (9, 31, 17, 30, 3, ACT_TANH),    # dropped units get no gradient
    (5, 257, 40, 15, 2, ACT_NONE),   # R = 640 rows: five CTAs of train_cum_unit_bwd
    (70, 64, 20, 1, 1, ACT_RELU6),   # R = 4480
])
def test_fsn_cumulative_norm_bwd_matches_float64(lib, B, F, Tp, Ns, G, act):
    check_fsn(lib, B, F, Tp, Ns, G, act, cum=True)


def test_fsn_dropped_units_keep_the_norm_mean_term(lib):
    """drop_band removes units after the offline norm, so a removed unit's full-band output still moves the clip's mean:
    its gradient is -inv2 dot / cnt2 times act', not 0."""
    B, F, Tp, Ns, G = 5, 9, 4, 1, 2
    rng = np.random.default_rng(7)
    dX = _f32(rng.standard_normal((Tp, B * (F // G), 2 * Ns + 2)))
    mag, z = _f32(rng.random((B, F, Tp)) + 0.1), _f32(rng.standard_normal((B, F, Tp)))
    dz_ref, _, X, y, scale = ref_fsn_norm_bwd(mag, z, dX, Ns, G, ACT_NONE, False)
    _, dz = run_fsn(lib, dX, _f32(X), _f32(y), _f32(scale), False, B, F, G, Tp, Ns, ACT_NONE)
    dropped = np.array([[f % G != b % G or f // G >= F // G for f in range(F)] for b in range(B)])
    assert np.all(np.abs(dz_ref[:, dropped]) > 0) and np.all(dz[:, dropped] != 0)
    np.testing.assert_allclose(dz[:, dropped], dz_ref[:, dropped], rtol=1e-4)


def test_fsn_cumulative_norm_over_4000_frames(lib):
    """60 s at hop 256: the float32 suffix sum of train_cum_unit_bwd over 4000 frames against float64, recorded next to
    torch's own float32 arithmetic (autograd through cumulative_laplace_norm, whose forward is torch.cumsum)."""
    B, F, Tp, Ns = 2, 16, 4000, 1
    rng = np.random.default_rng(11)
    mag, z = _f32(rng.random((B, F, Tp)) + 0.05), _f32(rng.standard_normal((B, F, Tp)))
    dX = _f32(rng.standard_normal((Tp, B * F, 2 * Ns + 2)))
    err = check_fsn(lib, B, F, Tp, Ns, 1, ACT_NONE, cum=True, seed=11)
    dz_ref, cond, *_ = ref_fsn_norm_bwd(mag, z, dX, Ns, 1, ACT_NONE, True)
    dz_t32 = ref_fsn_norm_bwd(mag, z, dX, Ns, 1, ACT_NONE, True, dtype=torch.float32)[0]
    RECORD["cum_4000_frames_kernel"] = err
    RECORD["cum_4000_frames_torch_float32"] = _cond_err(dz_t32, dz_ref, cond)


# ------------------------------------------------------------------ fast_fullsubnet
def run_fast(lib, ddec, dX, X, encT, bn_out, scale, cum, B, Tp, M, Nn, Ne, S):
    Ts, R, K = fast_shrunk(Tp, S), B * M, X.shape[2]
    d = [_dev(a) for a in (ddec, dX, X, encT, bn_out, scale)]
    mid, denc, dbn = Out((Ts, R) if cum else (B,)), Out((Tp, B, M)), Out((Ts, R))
    rc = lib.fsn_debug_fast_norm_unfold_bwd(*[t.data_ptr() for t in d], int(cum), B, Tp, M, Nn, Ne, S,
                                            float(M * K * Ts), mid.ptr, denc.ptr, dbn.ptr, _stream())
    torch.cuda.synchronize()
    assert rc == 0, lib.fsn_last_error()
    assert lib.fsn_last_launch_count() == 3
    return mid.get(), denc.get(), dbn.get()


def check_fast(lib, B, M, Tp, Nn, Ne, S, cum, seed=0):
    rng = np.random.default_rng(seed)
    Ts, K = fast_shrunk(Tp, S), (2 * Nn + 1) + (2 * Ne + 1)
    mel = _f32(rng.random((B, M, Tp)) + 0.05)
    z, zb = _f32(rng.standard_normal((B, M, Tp)) + 0.3), _f32(rng.standard_normal((B, M, Ts)))
    ddec = _f32(rng.standard_normal((Tp, B, 2 * M)))
    dX = _f32(rng.standard_normal((Ts, B * M, K)))
    dz_ref, cond, dzb_ref, condb, X, encT, bn_out, scale = ref_fast_bwd(mel, z, zb, ddec, dX, Nn, Ne, S, cum)
    X, encT, bn_out, scale = _f32(X), _f32(encT), _f32(bn_out), _f32(scale)
    args = (ddec, dX, X, encT, bn_out, scale, cum, B, Tp, M, Nn, Ne, S)
    out = run_fast(lib, *args)
    out2 = run_fast(lib, *args)
    assert all(_same_bits(a, b) for a, b in zip(out, out2))
    mid, denc, dbn = out
    _note("fast_denc_cum" if cum else "fast_denc", _cond_err(denc, dz_ref, cond))
    _note("fast_dbn", _cond_err(dbn, dzb_ref, condb))
    if B > 1:  # the last clip alone gives the same bits
        b = B - 1
        rows = slice(b * M, (b + 1) * M)
        sc = scale[:, rows] if cum else scale[b:b + 1]
        mid1, denc1, dbn1 = run_fast(lib, ddec[:, b:b + 1], dX[:, rows], X[:, rows], encT[:, b:b + 1], bn_out[:, rows],
                                     sc, cum, 1, Tp, M, Nn, Ne, S)
        assert _same_bits(denc1[:, 0], denc[:, b]) and _same_bits(dbn1, dbn[:, rows])
        assert _same_bits(mid1, mid[:, rows] if cum else mid[b:b + 1])
    return dbn, Ts


FAST_CASES = [  # B, M, Tp, Nn, Ne, S
    (1, 2, 2, 1, 1, 1),      # Nn = Ne = M - 1, no shrink
    (2, 5, 7, 1, 2, 3),      # (Tp - 1) % S == 0: full last block
    (2, 5, 5, 4, 0, 3),      # partial last block, and (Ts - 1) S >= Tp: the last shrunk step feeds no frame
    (3, 32, 33, 0, 31, 2),
    (2, 33, 32, 2, 5, 3),
    (65, 64, 140, 1, 3, 3),  # 582 k elements: ftr_denc's grid-stride loop takes a second pass; R = 4160
]


@pytest.mark.parametrize("B,M,Tp,Nn,Ne,S", FAST_CASES)
def test_fast_offline_norm_bwd_matches_float64(lib, B, M, Tp, Nn, Ne, S):
    check_fast(lib, B, M, Tp, Nn, Ne, S, cum=False)


@pytest.mark.parametrize("B,M,Tp,Nn,Ne,S", [
    (1, 2, 2, 1, 1, 1),
    (2, 5, 11, 2, 4, 3),     # the last shrunk step feeds no frame
    (3, 33, 64, 3, 5, 2),
    (5, 40, 31, 1, 1, 1),    # R = 200: two CTAs of ftr_cum_suffix
    (1, 8, 7999, 1, 2, 2),   # Ts = 4000 shrunk steps
])
def test_fast_cumulative_norm_bwd_matches_float64(lib, B, M, Tp, Nn, Ne, S):
    check_fast(lib, B, M, Tp, Nn, Ne, S, cum=True)


def test_fast_last_shrunk_step_without_frames_gets_exactly_zero(lib):
    B, M, Tp, S = 2, 5, 5, 3
    dbn, Ts = check_fast(lib, B, M, Tp, 1, 1, S, cum=False, seed=3)
    assert (Ts - 1) * S >= Tp
    assert np.all(_bits(dbn[Ts - 1]) == 0)


# ------------------------------------------------------------------ improved_fullsubnet
def run_imp(lib, dXs, Xs, invss, y, B, T, Fu, secs, act):
    dfb = Out((T, B, Fu))
    dots = []
    yd = _dev(y)
    for i, (sec, dX, X, inv) in enumerate(zip(secs, dXs, Xs, invss)):
        d = [_dev(a) for a in (dX, X, inv)]
        dot = Out((B,))
        last = i == len(secs) - 1
        rc = lib.fsn_debug_imp_unfold_bwd(*[t.data_ptr() for t in d], yd.data_ptr(), B, T, Fu, *sec, int(i == 0),
                                          act if last else ACT_NONE, dot.ptr, dfb.ptr, _stream())
        torch.cuda.synchronize()
        assert rc == 0, lib.fsn_last_error()
        dots.append(dot.get())
    return dots, dfb.get()


def check_imp(lib, B, Fu, T, secs, act, seed=0):
    rng = np.random.default_rng(seed)
    noisy, z = _f32(rng.random((B, Fu, T)) + 0.05), _f32(rng.standard_normal((B, Fu, T)))
    dXs = [_f32(rng.standard_normal((T, B * (hi - lo) // cs, cs + 2 * ns + cf + 2 * nf)))
           for lo, hi, cs, ns, cf, nf in secs]
    dz_ref, cond, y, per = ref_imp_bwd(noisy, z, dXs, secs, act)
    Xs, invss, y = [_f32(p[0]) for p in per], [_f32(p[1]) for p in per], _f32(y)
    dots, dfb = run_imp(lib, dXs, Xs, invss, y, B, T, Fu, secs, act)
    dots2, dfb2 = run_imp(lib, dXs, Xs, invss, y, B, T, Fu, secs, act)
    assert _same_bits(dfb, dfb2) and all(_same_bits(a, b) for a, b in zip(dots, dots2))
    _note("imp_dfb", _cond_err(dfb, dz_ref, cond))
    if B > 1:
        b = B - 1
        sl = [slice(b * X.shape[1] // B, (b + 1) * X.shape[1] // B) for X in Xs]
        dots1, dfb1 = run_imp(lib, [d[:, s] for d, s in zip(dXs, sl)], [X[:, s] for X, s in zip(Xs, sl)],
                              [v[b:b + 1] for v in invss], y[:, b:b + 1], 1, T, Fu, secs, act)
        assert _same_bits(dfb1[:, 0], dfb[:, b])
        assert all(_same_bits(a, d[b:b + 1]) for a, d in zip(dots1, dots))


IMP_CASES = [  # B, Fu, T, sections (lo, hi, cs, ns, cf, nf), act
    (1, 2, 1, [(0, 2, 1, 1, 1, 1)], ACT_NONE),                                    # two bins, ns = nf = Fu - 1
    (2, 12, 4, [(0, 4, 2, 1, 2, 3), (4, 12, 4, 2, 4, 11)], ACT_RELU),             # nf = Fu - 1 in a section with lo > 0
    (3, 32, 33, [(0, 32, 1, 31, 1, 31)], ACT_NONE),
    (2, 33, 31, [(0, 3, 3, 0, 3, 0), (3, 33, 3, 2, 3, 1)], ACT_RELU),
    (2, 256, 31, [(0, 32, 1, 15, 1, 15), (32, 128, 4, 15, 4, 15), (128, 256, 32, 15, 32, 15)], ACT_RELU),
    (66, 256, 33, [(0, 64, 2, 3, 2, 0), (64, 256, 8, 2, 8, 5)], ACT_RELU),       # 557 k elements: a second pass
]


@pytest.mark.parametrize("B,Fu,T,secs,act", IMP_CASES)
def test_imp_unfold_bwd_matches_float64(lib, B, Fu, T, secs, act):
    check_imp(lib, B, Fu, T, secs, act)


def run_section_input(lib, magc, fbT, B, T, Fu, sec, tm):
    lo, hi, cs, ns, cf, nf = sec
    N, W = (hi - lo) // cs, cs + 2 * ns + cf + 2 * nf
    d = [_dev(a) for a in (magc, fbT)]
    X, fs = Out((T, B * N, W)), Out((B * T, 2))
    rc = lib.fsn_debug_imp_section_input(d[0].data_ptr(), d[1].data_ptr(), B, T, Fu, *sec, int(tm), X.ptr, fs.ptr,
                                         _stream())
    torch.cuda.synchronize()
    assert rc == 0, lib.fsn_last_error()
    return X.get(), fs.get()


@pytest.mark.parametrize("tm", [False, True])
@pytest.mark.parametrize("B,Fu,T,secs", [c[:4] for c in IMP_CASES])
def test_imp_section_input_matches_float64(lib, B, Fu, T, secs, tm):
    """X is a bit-exact copy of the oracle's section unfold (reflection at both edges, lo > 0); fs holds each (b, t)
    block's sum."""
    rng = np.random.default_rng(5)
    noisy, y = _f32(rng.random((B, Fu, T))), _f32(rng.random((B, Fu, T)))
    lay = (lambda a: np.ascontiguousarray(a.transpose(2, 0, 1) if tm else a.transpose(0, 2, 1)))  # [T,B,Fu] / [B,T,Fu]
    for sec in secs:
        U = imp_section(torch.from_numpy(noisy.astype(np.float64)), torch.from_numpy(y.astype(np.float64)),
                        sec)[1].numpy()
        X, fs = run_section_input(lib, lay(noisy), lay(y), B, T, Fu, sec, tm)
        X2, fs2 = run_section_input(lib, lay(noisy), lay(y), B, T, Fu, sec, tm)
        assert _same_bits(X, X2) and _same_bits(fs, fs2)
        assert _same_bits(X, U.astype(F32))
        ref = U.reshape(T, B, -1).sum(axis=2).T.reshape(-1)  # [B*T], the terms are all positive
        assert _same_bits(fs[:, 0], fs[:, 1])
        _note("imp_fs", np.max(np.abs(fs[:, 0] - ref) / ref))


# ------------------------------------------------------------------ statistics of the offline norms
def run_stats(lib, x, B, T_pad, F, N, tm, lengths=None, hop=1, la=0, fb_sums=None, cnt1=1.0, cnt2=1.0):
    """x clip-major [B,T_pad,F] or time-major [T_pad,B,F]; returns fs [B*T_pad,2], sums [B,2], inv1, inv2 and the device
    sums (for a later call's fb_sums)."""
    bs, ts = (F, B * F) if tm else (T_pad * F, F)
    xd = _dev(x)
    fs, sums, inv1, inv2 = Out((B * T_pad, 2)), Out((B, 2)), Out((B,)), Out((B,))
    h = None if lengths is None else np.ascontiguousarray(lengths, np.int32)
    lens = torch.empty(B, dtype=torch.int32, device=DEV)
    rc = lib.fsn_debug_norm_stats(xd.data_ptr(), B, T_pad, F, N, bs, ts, None if h is None else h.ctypes.data,
                                  lens.data_ptr(), hop, la, None if fb_sums is None else fb_sums.data_ptr(), cnt1, cnt2,
                                  1e-5, fs.ptr, sums.ptr, inv1.ptr, inv2.ptr, _stream())
    torch.cuda.synchronize()
    assert rc == 0, lib.fsn_last_error()
    # frames past a clip's length are not reduced, but frame_stats still writes them
    return fs.get(), sums.get(), inv1.get(), inv2.get(), sums.buf


def _rel(got, ref, scale):
    return float(np.max(np.abs(np.asarray(got, np.float64) - ref) / scale))


STATS_CASES = [(F, N, T) for F, N in [(2, 0), (2, 1), (31, 30), (32, 0), (33, 1), (257, 15), (257, 256)]
               for T in (1, 31, 32, 33)] + [(33, 1, 300), (257, 15, 257)]  # more than 256 frames per clip_reduce CTA


@pytest.mark.parametrize("tm", [False, True])
@pytest.mark.parametrize("F,N,T", STATS_CASES)
def test_norm_stats_match_float64(lib, F, N, T, tm):
    """frame_stats (N = 0: .y == .x bit for bit), clip_reduce over more than 256 frames, and norm_scales' inv1 / inv2
    with a second tensor's sums, against the unfold sums and offline_laplace_norm's mean."""
    B, Nf = 3, min(2, F - 1)
    rng = np.random.default_rng(F * 1000 + T)
    mag, fb = _f32(rng.random((B, T, F)) + 0.01), _f32(rng.random((B, T, F)))
    lay = (lambda a: np.ascontiguousarray(a.transpose(1, 0, 2)) if tm else a)
    K = (2 * N + 1) + (2 * Nf + 1)
    _, _, _, _, fbs = run_stats(lib, lay(fb), B, T, F, Nf, tm)
    args = (lay(mag), B, T, F, N, tm)
    kw = dict(fb_sums=fbs, cnt1=float(F * T), cnt2=float(F * K * T))
    fs, sums, inv1, inv2, _ = run_stats(lib, *args, **kw)
    again = run_stats(lib, *args, **kw)[:4]
    assert all(_same_bits(a, b) for a, b in zip((fs, sums, inv1, inv2), again))
    s0, s1 = ref_frame_stats(mag, N)
    if N == 0:
        assert _same_bits(fs[:, 0], fs[:, 1])
    r0, r1 = s0.reshape(-1), s1.reshape(-1)
    _note("frame_stats", max(_rel(fs[:, 0], r0, r0), _rel(fs[:, 1], r1, r1)))
    _note("clip_sums", max(_rel(sums[:, 0], s0.sum(1), s0.sum(1)), _rel(sums[:, 1], s1.sum(1), s1.sum(1))))
    t = torch.from_numpy(mag.astype(np.float64)).permute(0, 2, 1)[:, None]
    u = torch.from_numpy(fb.astype(np.float64)).permute(0, 2, 1)[:, None]
    from oracle import fullsubnet_oracle as O
    ref1 = ref_inv([mag])
    ref2 = ref_inv([O.freq_unfold(t, N).numpy(), O.freq_unfold(u, Nf).numpy()])
    _note("inv", max(_rel(inv1, ref1, ref1), _rel(inv2, ref2, ref2)))


@pytest.mark.parametrize("tm", [False, True])
@pytest.mark.parametrize("hop,la,lengths", [
    (256, 0, [256 * 299, 0, 256 * 31, 256 * 31 + 255, 256 * 300 - 1]),  # 300, 1, 32, 32 and 300 frames of T_pad = 300
    (160, 2, [160 * 40, 160 * 297 + 7, 1, 160 * 255]),                  # la = 2
])
def test_norm_stats_with_lengths_give_each_clip_its_bits_alone(lib, tm, hop, la, lengths):
    """A clip in a padded batch gives, bit for bit, the sums and scales of a call on its own frames with T_pad = its
    frame count, and the frames past its length do not reach its sums."""
    B, F, N = len(lengths), 33, 4
    tp = [1 + n // hop + la for n in lengths]
    T_pad = max(tp)
    rng = np.random.default_rng(hop)
    x = _f32(rng.random((B, T_pad, F)))
    lay = (lambda a, Bq: np.ascontiguousarray(a.transpose(1, 0, 2)) if tm else a)
    fs, sums, inv1, inv2, _ = run_stats(lib, lay(x, B), B, T_pad, F, N, tm, lengths=lengths, hop=hop, la=la,
                                        cnt1=float(F), cnt2=float(F * (2 * N + 1)))
    for b in range(B):
        xb = x[b:b + 1, :tp[b]]
        fs1, sums1, inv11, inv21, _ = run_stats(lib, lay(xb, 1), 1, tp[b], F, N, tm,
                                                cnt1=float(np.float32(F) * np.float32(tp[b])),
                                                cnt2=float(np.float32(F * (2 * N + 1)) * np.float32(tp[b])))
        assert _same_bits(sums1[0], sums[b]) and _same_bits(inv11[0], inv1[b]) and _same_bits(inv21[0], inv2[b])
        assert _same_bits(fs1, fs[b * T_pad:b * T_pad + tp[b]])
        s0, s1 = ref_frame_stats(xb, N)
        _note("clip_sums", max(_rel(sums[b, 0], s0.sum(), s0.sum()), _rel(sums[b, 1], s1.sum(), s1.sum())))
        ref = ref_inv([xb])
        _note("inv", _rel(inv1[b], ref, ref))


@pytest.mark.parametrize("tm", [False, True])
@pytest.mark.parametrize("B,F,T,N", [(1, 2, 1, 0), (3, 2, 33, 1), (4, 33, 32, 32), (70, 257, 31, 15), (2, 161, 300, 0)])
def test_train_stats_match_float64(lib, B, F, T, N, tm):
    """train_mag_stats ([B,F,T]) and train_tm_stats ([T,B,F]): one CTA per clip, a clip alone gives the same bits."""
    rng = np.random.default_rng(B * F + T)
    x = _f32(rng.random((B, T, F)))
    lay = (lambda a: np.ascontiguousarray(a.transpose(1, 0, 2) if tm else a.transpose(0, 2, 1)))

    def run(a, Bq):
        xd, sums = _dev(a), Out((Bq, 2))
        rc = lib.fsn_debug_train_stats(xd.data_ptr(), int(tm), Bq, F, T, N, sums.ptr, _stream())
        torch.cuda.synchronize()
        assert rc == 0, lib.fsn_last_error()
        return sums.get()

    sums = run(lay(x), B)
    assert _same_bits(sums, run(lay(x), B))
    assert _same_bits(run(lay(x[B - 1:]), 1)[0], sums[B - 1])
    s0, s1 = ref_frame_stats(x, N)
    _note("train_stats", max(_rel(sums[:, 0], s0.sum(1), s0.sum(1)), _rel(sums[:, 1], s1.sum(1), s1.sum(1))))
    if N == 0:
        assert _same_bits(sums[:, 0], sums[:, 1])
