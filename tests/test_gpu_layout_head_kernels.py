"""The cumulative-norm forward scales, the layout kernels and the sub-band heads alone against the float64 references of
tests/test_cpu_layout_head_kernels.py, through the hooks fsn_debug_cum_clip_scale (frame_stats + cum_clip_scale),
fsn_debug_cum_unit_scale, fsn_debug_forget_unit_broadcast, fsn_debug_fast_bn (fast_bn_input, then fast_cum_bn_scale or
clip_reduce + norm_scales), fsn_debug_fast_dec_input, fsn_debug_transpose_mag, fsn_debug_crm_output,
fsn_debug_scale_rows, fsn_debug_imp_compress, fsn_debug_train_gather, fsn_debug_sb_head, fsn_debug_sb_head_bwd and
fsn_debug_train_dy.

Pure copies and single float32 products must match numpy's float32 bit for bit: the re-layouts, the scaled copies,
sqrtf (fdrc = 0.5; the build has no fast math), the head backward and train_dy for none / ReLU / ReLU6.  The tanh
derivative is fused in the SASS (FFMA d = 1 - y*y, then FMUL v*d), so it is bit exact where 1 - y^2 needs no rounding
and within 2 ulp of float64 elsewhere; powf (fdrc = 0.3, 1.0) is held in ulps of float64.  The sums (the cumulative
scales, the bottleneck block means and sums, the head's dot product) go against float64 over their conditioning, with
bounds about 4x the worst error measured on an H100 (printed with -s as `[layout/head] family worst`).

The shapes hit every 32 x 32 tile edge (F, T in 1, 2, 31, 32, 33, 257), look-ahead pads of 0..3 frames, clip-major and
time-major strides, B from 1 to more than 64, drop_band with G = 2, 3, 4, 7 dividing neither F nor B, S = 1, 2, 3 with a
partial last block, every head geometry the models use (fullsubnet, improved sections with lo > 0, the stream's
frame-major cRM, fast_fullsubnet's bottleneck with O = 1, the training call offset by la) with H % 32 != 0, and
grid-stride loops past one pass.  Every call also checks the guard floats behind its output, that every element is
written, that two runs give the same bits and, for the per-clip kernels, that a clip alone gives the bits it gets in a
batch."""
import numpy as np
import pytest
import torch

from test_cpu_layout_head_kernels import (ACT_NONE, ACT_RELU, ACT_RELU6, ACT_TANH, EPS_F32, EPS_OFF, TOL, act_grad32,
                                          act_grad64, act64, cum_err, fast_bottleneck, fast_shrunk, head_index,
                                          ref_clip_scale, ref_crm_output, ref_cum_scale, ref_dec_input, ref_imp_compress,
                                          ref_sb_head, ref_scale_rows, ref_train_dy, ref_transpose_mag, unit_inputs)
from test_gpu_dsp import SENT, Out, _bits
from test_gpu_norm_layout_kernels import _cond_err

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
F32 = np.float32
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
        bound = f" (bound {TOL[k]:.1e})" if k in TOL else ""
        print(f"[layout/head] {k} worst {v:.3e}{bound}")
    for k, v in sorted(RECORD.items()):
        print(f"[layout/head] {k} {v:.3e} (recorded, not asserted)")


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


def _same(a, b):
    return np.array_equal(_bits(np.ascontiguousarray(a, F32)), _bits(np.ascontiguousarray(b, F32)))


def _exact(got, ref):
    ref = np.asarray(ref, np.float64).astype(F32)
    assert _same(got, ref), float(np.max(np.abs(got.astype(np.float64) - ref.astype(np.float64))))


def _call(lib, fn, *args, launches=1):
    rc = fn(*args, _stream())
    torch.cuda.synchronize()
    assert rc == 0, lib.fsn_last_error()
    assert lib.fsn_last_launch_count() == launches


def _twice(run):
    """run() twice: the same bits both times; returns the first result."""
    a, b = run(), run()
    for x, y in zip(a if isinstance(a, tuple) else (a,), b if isinstance(b, tuple) else (b,)):
        assert _same(x, y), "two runs differ"
    return a


EDGES = [1, 2, 31, 32, 33, 257]


# ------------------------------------------------------------------ re-layouts
def run_transpose(lib, mag, Tp, tm, scale):
    B, F, T = mag.shape
    bs, ts = (F, B * F) if tm else (Tp * F, F)
    shape = (Tp, B, F) if tm else (B, Tp, F)
    d, s = _dev(mag), _dev(scale)
    out, sc = Out(shape), Out(shape)
    _call(lib, lib.fsn_debug_transpose_mag, d.data_ptr(), B, F, T, Tp, bs, ts, out.ptr, s.data_ptr(), sc.ptr)
    o, c = out.get(), sc.get()
    return (o.transpose(1, 0, 2), c.transpose(1, 0, 2)) if tm else (o, c)


@pytest.mark.parametrize("F", EDGES)
@pytest.mark.parametrize("T", EDGES)
def test_transpose_mag_exact(lib, F, T):
    rng = np.random.default_rng(F * 300 + T)
    for B, la, tm in [(3, T % 4, False), (2, (T + 1) % 4, True)]:
        mag = rng.random((B, F, T)).astype(F32)
        scale = (rng.random(B) + 0.5).astype(F32)
        Tp = T + la
        o, c = _twice(lambda: run_transpose(lib, mag, Tp, tm, scale))
        ref = ref_transpose_mag(mag, Tp)
        _exact(o, ref)
        _exact(c, (ref.astype(F32) * scale[:, None, None]).astype(F32))  # one float32 product
        assert not np.any(_bits(o[:, T:]))  # the pad frames are +0
        if not tm and B > 1:
            o1, c1 = run_transpose(lib, mag[1:2], Tp, tm, scale[1:2])
            assert _same(o1[0], o[1]) and _same(c1[0], c[1])


def test_transpose_mag_many_clips(lib):
    rng = np.random.default_rng(5)
    mag = rng.random((70, 33, 40)).astype(F32)
    scale = (rng.random(70) + 0.5).astype(F32)
    o, c = run_transpose(lib, mag, 43, True, scale)
    _exact(o, ref_transpose_mag(mag, 43))
    _exact(c, (ref_transpose_mag(mag, 43).astype(F32) * scale[:, None, None]).astype(F32))


def run_crm(lib, y, la, tm):
    """y [B,Tp,2F] laid out clip-major, or time-major [Tp,B,2F] when tm."""
    B, Tp, F2 = y.shape
    F = F2 // 2
    src = y.transpose(1, 0, 2) if tm else y
    bs, ts = (F2, B * F2) if tm else (Tp * F2, F2)
    d = _dev(src)
    out = Out((B, 2, F, Tp - la))
    _call(lib, lib.fsn_debug_crm_output, d.data_ptr(), bs, ts, B, Tp, F, la, out.ptr)
    return out.get()


@pytest.mark.parametrize("F", EDGES)
@pytest.mark.parametrize("T", EDGES)
def test_crm_output_exact(lib, F, T):
    rng = np.random.default_rng(F * 7 + T)
    for B, la, tm in [(2, T % 4, False), (3, 3 - T % 4, True), (1, 0, False)]:
        y = rng.standard_normal((B, T + la, 2 * F)).astype(F32)
        o = _twice(lambda: run_crm(lib, y, la, tm))
        _exact(o, ref_crm_output(y, la))
        if B > 1:
            assert _same(run_crm(lib, y[-1:], la, tm)[0], o[-1])


def test_crm_output_many_clips(lib):
    rng = np.random.default_rng(6)
    y = rng.standard_normal((66, 35, 2 * 33)).astype(F32)
    _exact(run_crm(lib, y, 2, True), ref_crm_output(y, 2))


@pytest.mark.parametrize("n,cols,rows,div", [(1, 1, 1, 1), (33 * 31, 33, 31, 1), (7 * 5 * 3 * 4, 4, 15, 5),
                                             (600 * 2049, 2049, 600, 1), (40 * 9 * 7 * 32, 32, 63, 7)])
def test_scale_rows_exact(lib, n, cols, rows, div):
    rng = np.random.default_rng(n)
    x = rng.standard_normal(n).astype(F32)
    scale = (rng.random(cdiv(rows, div)) + 0.5).astype(F32)
    ref = ref_scale_rows(x.astype(np.float64), scale, cols, rows, div)
    xs, s = _dev(x), _dev(scale)
    out = Out((n,))
    _call(lib, lib.fsn_debug_scale_rows, xs.data_ptr(), s.data_ptr(), n, cols, rows, div, out.ptr)
    _exact(out.get(), (x * scale[((np.arange(n) // cols) % rows) // div]).astype(F32))
    # in place, as the section norms and the fast bottleneck run it
    buf = Out((n,), fill=x)
    _call(lib, lib.fsn_debug_scale_rows, buf.ptr, s.data_ptr(), n, cols, rows, div, buf.ptr)
    _exact(buf.get(), ref.astype(F32))


def cdiv(a, b):
    return -(-a // b)


@pytest.mark.parametrize("F", [2, 3, 32, 33, 257])
@pytest.mark.parametrize("fdrc", [0.5, 0.3, 1.0])
def test_imp_compress(lib, F, fdrc):
    rng = np.random.default_rng(F)
    for B, T, tm in [(2, 33, False), (3, 31, True), (1, 257, False), (2, 1, True)]:
        mag = (rng.random((B, F, T)) * 3).astype(F32)
        mag[:, ::3, ::2] = 0  # exact zeros
        d = _dev(mag)

        def run(mag_d=d, B=B):
            out = Out((T, B, F - 1) if tm else (B, T, F - 1))
            _call(lib, lib.fsn_debug_imp_compress, mag_d.data_ptr(), B, F, T, fdrc, int(tm), out.ptr)
            o = out.get()
            return o.transpose(1, 0, 2) if tm else o

        o = _twice(run)
        ref = ref_imp_compress(mag, fdrc)
        if fdrc == 0.5:
            _exact(o, np.sqrt(mag)[:, :-1].transpose(0, 2, 1))  # sqrtf: correctly rounded
        else:
            assert np.all(o[ref == 0] == 0)
            ulp = np.spacing(np.abs(ref).astype(F32)).astype(np.float64)
            nz = ref != 0
            e = float(np.max(np.abs(o.astype(np.float64) - ref)[nz] / ulp[nz])) if np.any(nz) else 0.0
            WORST["powf_ulp"] = max(WORST.get("powf_ulp", 0.0), e)
            assert e <= 4.0, e  # CUDA's documented powf bound
        if B > 1 and not tm:
            assert _same(run(_dev(mag[1:2]), 1)[0], o[1])


# ------------------------------------------------------------------ causal scales
def run_clip_scale(lib, x, tm):
    B, Tp, F = x.shape
    src = x.transpose(1, 0, 2) if tm else x
    bs, ts = (F, B * F) if tm else (Tp * F, F)
    d = _dev(src)
    fs, sc = Out((B * Tp, 2)), Out((Tp, B))
    _call(lib, lib.fsn_debug_cum_clip_scale, d.data_ptr(), B, Tp, F, bs, ts, EPS_F32, fs.ptr, sc.ptr, launches=2)
    fs.get()
    return sc.get()


@pytest.mark.parametrize("F", EDGES)
@pytest.mark.parametrize("B,Tp,tm", [(1, 1, False), (3, 33, True), (70, 40, False), (2, 300, True)])
def test_cum_clip_scale(lib, F, B, Tp, tm):
    rng = np.random.default_rng(B * F + Tp)
    x = (rng.random((B, Tp, F)) + 0.01).astype(F32)
    s = _twice(lambda: run_clip_scale(lib, x, tm))
    _, m, cond = ref_clip_scale(x, EPS_F32)
    _note("cum_clip_scale", cum_err(s, m, cond, EPS_F32))
    if B > 1:
        assert _same(run_clip_scale(lib, x[-1:], tm)[:, 0], s[:, -1])


def run_unit_scale(lib, mag, fb, G, Ns, Nf, tm):
    """mag, fb [B,F,Tp] -> scaleT [Tp,R] with the inputs clip-major [B,Tp,F] or time-major [Tp,B,F]."""
    B, F, Tp = mag.shape
    lay = (lambda a: a.transpose(2, 0, 1)) if tm else (lambda a: a.transpose(0, 2, 1))
    dm, df = _dev(lay(mag)), _dev(lay(fb))
    R = B * (F // G if G > 1 else F)
    sc = Out((Tp, R))
    _call(lib, lib.fsn_debug_cum_unit_scale, dm.data_ptr(), df.data_ptr(), B, F, G, Tp, Ns, Nf, EPS_F32, int(tm), sc.ptr)
    return sc.get()


@pytest.mark.parametrize("B,F,Tp,Ns,Nf,G,tm", [
    (1, 1, 3, 0, 0, 1, False), (2, 2, 33, 1, 1, 1, True), (3, 31, 32, 15, 0, 2, False), (5, 33, 31, 2, 3, 3, True),
    (9, 257, 20, 15, 0, 4, True), (9, 33, 17, 5, 1, 7, False), (70, 32, 12, 3, 0, 1, False), (66, 33, 9, 2, 0, 2, True)])
def test_cum_unit_scale(lib, B, F, Tp, Ns, Nf, G, tm):
    rng = np.random.default_rng(B + F + Tp)
    mag, fb = (rng.random((B, F, Tp)) + 0.01).astype(F32), (rng.random((B, F, Tp)) * 2).astype(F32)
    s = _twice(lambda: run_unit_scale(lib, mag, fb, G, Ns, Nf, tm))
    _, m, cond = ref_cum_scale(unit_inputs(mag, fb, Ns, Nf, G), EPS_F32)
    _note("cum_unit_scale", cum_err(s, m, cond, EPS_F32))
    if G <= 1 and B > 1:
        assert _same(run_unit_scale(lib, mag[-1:], fb[-1:], G, Ns, Nf, tm), s[:, -F:])


@pytest.mark.parametrize("B,F,G,Tp", [(1, 1, 1, 4), (3, 9, 2, 5), (5, 10, 3, 33), (9, 33, 4, 7), (8, 16, 7, 3),
                                      (9, 257, 1, 300)])
def test_forget_unit_broadcast_exact(lib, B, F, G, Tp):
    from oracle import fullsubnet_oracle as O
    rng = np.random.default_rng(B * F)
    scaleT = rng.random((Tp, B)).astype(F32)
    src_b = np.repeat(O.drop_band_index_map(B, F, G)[0], F // G) if G > 1 else np.repeat(np.arange(B), F)
    d = _dev(scaleT)
    out = Out((Tp, len(src_b)))
    _call(lib, lib.fsn_debug_forget_unit_broadcast, d.data_ptr(), B, F, G, Tp, out.ptr)
    _exact(out.get(), scaleT[:, src_b])


# ------------------------------------------------------------------ fast_fullsubnet bottleneck and decoder input
def run_fast_bn(lib, mel, enc, Nn, Ne, S, cum, tm):
    """mel, enc [B,M,Tp] -> bn [Ts,B*M,K], fs [B,Ts], scale ([Ts,B*M] or [B])."""
    B, M, Tp = mel.shape
    Ts, K = fast_shrunk(Tp, S), 2 * Nn + 2 * Ne + 2
    lay = (lambda a: a.transpose(2, 0, 1)) if tm else (lambda a: a.transpose(0, 2, 1))
    bs, ts = (M, B * M) if tm else (Tp * M, M)
    dm, de = _dev(lay(mel)), _dev(lay(enc))
    bn, fs, sums = Out((Ts, B * M, K)), Out((B, Ts, 2)), Out((B, 2))
    sc = Out((Ts, B * M) if cum else (B,))
    _call(lib, lib.fsn_debug_fast_bn, dm.data_ptr(), de.data_ptr(), bs, ts, B, Tp, M, Nn, Ne, S, int(cum),
          EPS_F32 if cum else EPS_OFF, bn.ptr, fs.ptr, sums.ptr if not cum else None, sc.ptr, launches=2 if cum else 3)
    f = fs.get()
    assert _same(f[..., 0], f[..., 1])
    if not cum:
        sums.get()
    return bn.get(), f[..., 0], sc.get()


@pytest.mark.parametrize("cum", [False, True])
@pytest.mark.parametrize("B,M,Tp,Nn,Ne,S,tm", [
    (1, 2, 2, 1, 0, 1, False), (2, 5, 7, 1, 2, 3, True), (3, 33, 32, 5, 0, 2, False), (2, 31, 33, 3, 3, 3, True),
    (70, 8, 9, 1, 1, 2, False), (2, 64, 100, 5, 0, 2, True)])
def test_fast_bn(lib, cum, B, M, Tp, Nn, Ne, S, tm):
    rng = np.random.default_rng(B * M + Tp + S)
    mel, enc = (rng.random((B, M, Tp)) + 0.01).astype(F32), (rng.random((B, M, Tp)) * 2).astype(F32)
    bn, fs, sc = _twice(lambda: run_fast_bn(lib, mel, enc, Nn, Ne, S, cum, tm))
    X, U, m = fast_bottleneck(torch.as_tensor(mel, dtype=torch.float64), torch.as_tensor(enc, dtype=torch.float64),
                              Nn, Ne, S, cum)
    U = U.numpy()
    Ts = U.shape[0]
    _note("fast_bn", np.max(np.abs(bn - U) / np.abs(U)))  # block means of positive frames: cond is the mean itself
    blk = U.reshape(Ts, B, M * U.shape[2]).sum(-1).T  # [B, Ts]
    _note("fast_bn_sums", np.max(np.abs(fs - blk) / blk))
    if cum:
        _, mm, cond = ref_cum_scale(U, EPS_F32)
        _note("fast_cum_bn_scale", cum_err(sc, mm, cond, EPS_F32))
    else:
        inv = 1.0 / (U.reshape(Ts, B, -1).transpose(1, 0, 2).reshape(B, -1).mean(1) + EPS_OFF)
        _note("fast_inv2", np.max(np.abs(sc / inv - 1)))
    if B > 1:
        bn1, fs1, sc1 = run_fast_bn(lib, mel[-1:], enc[-1:], Nn, Ne, S, cum, tm)
        assert _same(bn1[:, 0 * M:M], bn[:, -M:]) and _same(fs1[0], fs[-1])
        assert _same(sc1, sc[:, -M:] if cum else sc[-1:])


@pytest.mark.parametrize("B,M,Tp,S,tm", [(1, 1, 1, 1, False), (2, 5, 7, 3, True), (3, 33, 32, 2, False),
                                         (70, 8, 9, 2, True), (3, 128, 1000, 3, False), (2, 31, 33, 1, True)])
def test_fast_dec_input_exact(lib, B, M, Tp, S, tm):
    """Inference: encT [B,Tp,M] clip-major, bn_out [B*M, Ts]; training: time-major [Tp,B,M], bn_out [Ts, B*M]."""
    rng = np.random.default_rng(B * M + Tp)
    Ts = fast_shrunk(Tp, S)
    enc = rng.standard_normal((B, Tp, M)).astype(F32)
    bn_out = rng.standard_normal((B, M, Ts)).astype(F32)
    if tm:
        e, n, strides, rows = enc.transpose(1, 0, 2), bn_out.transpose(2, 0, 1), (M, 1, B * M), (1, B)
    else:
        e, n, strides, rows = enc, bn_out, (M * Ts, Ts, 1), (Tp, 1)
    de, dn = _dev(e), _dev(n)

    def run():
        out = Out((Tp, B, 2 * M) if tm else (B, Tp, 2 * M))
        _call(lib, lib.fsn_debug_fast_dec_input, de.data_ptr(), dn.data_ptr(), *strides, B, Tp, M, S, Ts, *rows, out.ptr)
        o = out.get()
        return o.transpose(1, 0, 2) if tm else o

    _exact(_twice(run), ref_dec_input(enc, bn_out, S, Tp))


# ------------------------------------------------------------------ training gather
def run_gather(lib, raw, fbz, inv2, us, B, F, G, Ns, Nf):
    Tp = raw.shape[0]
    R = B * (F // G if G > 1 else F)
    d = [_dev(a) for a in (raw, fbz)]
    s2 = _dev(inv2) if inv2 is not None else None
    su = _dev(us) if us is not None else None
    X = Out((Tp, R, 2 * Ns + 2 * Nf + 2))
    _call(lib, lib.fsn_debug_train_gather, d[0].data_ptr(), d[1].data_ptr(), s2.data_ptr() if s2 is not None else None,
          su.data_ptr() if su is not None else None, B, F, G, Tp, Ns, Nf, X.ptr)
    return X.get()


@pytest.mark.parametrize("per_unit", [False, True])
@pytest.mark.parametrize("B,F,Tp,Ns,Nf,G", [(1, 1, 2, 0, 0, 1), (3, 9, 4, 2, 0, 2), (5, 10, 3, 9, 1, 3),
                                            (9, 33, 5, 15, 2, 4), (8, 16, 3, 3, 0, 7), (9, 257, 40, 15, 0, 1)])
def test_train_gather_exact(lib, per_unit, B, F, Tp, Ns, Nf, G):
    from oracle import fullsubnet_oracle as O
    rng = np.random.default_rng(B * F + Tp)
    raw, fbz = rng.random((Tp, B, F)).astype(F32), rng.standard_normal((Tp, B, F)).astype(F32)
    U = unit_inputs(raw.transpose(1, 2, 0), fbz.transpose(1, 2, 0), Ns, Nf, G).astype(F32)  # exact copies
    R = U.shape[1]
    inv2 = (rng.random(B) + 0.5).astype(F32)
    us = (rng.random((Tp, R)) + 0.5).astype(F32) if per_unit else None
    X = _twice(lambda: run_gather(lib, raw, fbz, None if per_unit else inv2, us, B, F, G, Ns, Nf))
    if per_unit:
        ref = U * us[:, :, None]
    else:
        src_b = np.repeat(O.drop_band_index_map(B, F, G)[0], F // G) if G > 1 else np.repeat(np.arange(B), F)
        ref = U * inv2[src_b][None, :, None]
    _exact(X, ref.astype(F32))


# ------------------------------------------------------------------ heads
def run_head(lib, h, W, bias, act, geom, t0, size, fill=None):
    steps, R, H = h.shape
    N, c, lo, rows, rs, bs = geom
    d = [_dev(a) for a in (h, W, bias)]
    out = Out((size,), fill=np.full(size, SENT, F32) if fill is None else fill)
    _call(lib, lib.fsn_debug_sb_head, d[0].data_ptr(), R, H, steps, d[1].data_ptr(), d[2].data_ptr(), W.shape[0], act,
          N, c, lo, rows, rs, bs, t0, out.ptr)
    return out.get(written=False)


# (name, B, N, c, lo, rows, O, frames, rs, bs, steps, t0, act)
HEADS = [
    ("fullsubnet", 3, 9, 1, 0, 9, 2, 20, 20, 0, 20, 0, ACT_NONE),           # N = Fsub, c = 1
    ("fullsubnet_step", 2, 33, 1, 0, 33, 2, 12, 12, 0, 1, 7, ACT_TANH),     # one frame t0 > 0 per call
    ("training", 4, 31, 1, 0, 31, 2, 9, 9, 0, 9, 0, ACT_RELU6),            # h offset by la, steps = Tp - la
    ("improved", 2, 4, 4, 4, 21, 8, 6, 6, 0, 6, 0, ACT_RELU),              # lo > 0, O = 2 cs, Nyquist row untouched
    ("improved_part", 3, 5, 3, 2, 33, 5, 5, 5, 0, 5, 0, ACT_TANH),         # O < 2c
    ("stream", 3, 17, 1, 0, 17, 2, 1, 1, (4 + 1) * 34, 1, 0, ACT_NONE),    # frame-major cRM: rs = 1, bs != 0
    ("fast_bottleneck", 1, 70, 1, 0, 0, 1, 13, 13, 0, 1, 5, ACT_RELU),      # O = 1, rows = 0, ReLU
    ("many_rows", 70, 33, 1, 0, 33, 2, 3, 3, 0, 3, 0, ACT_NONE),
]


def _head_size(B, rows, rs, bs, frames, R):
    return (B * bs if bs else B * 2 * rows * rs) if rows else R * rs


@pytest.mark.parametrize("H", [33, 100, 257])
@pytest.mark.parametrize("case", HEADS, ids=[c[0] for c in HEADS])
def test_sb_head(lib, H, case):
    name, B, N, c, lo, rows, O_, frames, rs, bs, steps, t0, act = case
    R = B * N
    rng = np.random.default_rng(H + R)
    h = rng.standard_normal((steps, R, H)).astype(F32)
    W = (rng.standard_normal((O_, H)) / np.sqrt(H)).astype(F32)
    bias = rng.standard_normal(O_).astype(F32)
    if act == ACT_RELU6:
        W *= 8
    size = _head_size(B, rows, rs, bs, frames, R)
    idx = head_index(R, O_, steps, t0, N, c, lo, rows, rs, bs)
    assert idx.max() < size and len(np.unique(idx)) == idx.size
    out = _twice(lambda: run_head(lib, h, W, bias, act, (N, c, lo, rows, rs, bs), t0, size))
    ref, cond, _ = ref_sb_head(h, W, bias, act)
    got = out[idx]
    assert not np.any(got == F32(SENT)), "a head output was not written"
    mask = np.ones(size, bool)
    mask[idx] = False
    assert np.all(out[mask] == F32(SENT)), "a head wrote outside its rows"
    _note("sb_head", _cond_err(got, ref, cond))
    # integer h and W: the dot product is exact, so the bias and the activation's edges (exactly 0 and 6) match bit
    # for bit
    hi = rng.integers(-3, 4, (steps, R, H)).astype(F32)
    Wi = rng.integers(-3, 4, (O_, H)).astype(F32)
    z = hi.astype(np.float64) @ Wi.T.astype(np.float64)
    bi = np.array([-z.reshape(-1, O_)[0, o] + (6.0 if o % 2 else 0.0) for o in range(O_)], F32)  # row 0 lands on 0 / 6
    oi = run_head(lib, hi, Wi, bi, act, (N, c, lo, rows, rs, bs), t0, size)
    if act != ACT_TANH:
        _exact(oi[idx], act64(z + bi, act))
    else:  # tanhf is not correctly rounded: within 2 ulp, and exactly 0 at 0
        t = np.tanh(z + bi)
        assert np.max(np.abs(oi[idx] - t) / np.spacing(np.abs(t).astype(F32))) <= 2
        assert np.all(oi[idx][t == 0] == 0)
    if bs == 0 and rows and B > 1:  # the last clip alone
        o1 = run_head(lib, h[:, -N:], W, bias, act, (N, c, lo, rows, rs, bs), t0, size // B)
        assert _same(o1, out[size - size // B:])


def run_head_bwd(lib, dcrm, y, act, R, O_, steps, la, geom):
    N, c, lo, rows, rs, bs = geom
    d = _dev(dcrm)
    dy = _dev(y) if y is not None else None
    out = Out((steps, R, O_))
    _call(lib, lib.fsn_debug_sb_head_bwd, d.data_ptr(), dy.data_ptr() if dy is not None else None, act, R, O_, steps, la,
          N, c, lo, rows, rs, bs, out.ptr)
    return out.get()


def _act_out(rng, shape, act):
    if act == ACT_TANH:  # float32 tanh outputs, half of them with 12 fraction bits (1 - y^2 exact)
        y = np.tanh(rng.standard_normal(shape)).astype(F32)
        grid = (rng.integers(-4095, 4096, shape) / 4096.0).astype(F32)
        return np.where(rng.random(shape) < 0.5, grid, y), np.abs(grid * 4096 - np.round(grid * 4096)) == 0
    y = act64(rng.standard_normal(shape) * 4, act).astype(F32)
    if act == ACT_RELU6:
        y.reshape(-1)[::7] = 6.0
    return y, None


def _check_grad(got, v, y, act):
    if act != ACT_TANH:
        _exact(got, act_grad64(v, y, act))
        return
    ref = act_grad64(v, y, act)
    _exact(got[_grid_mask(y)], ref[_grid_mask(y)])
    ulp = np.spacing(np.abs(ref).astype(F32)).astype(np.float64)
    nz = ref != 0
    e = float(np.max(np.abs(got.astype(np.float64) - ref)[nz] / ulp[nz]))
    WORST["tanh_grad_ulp"] = max(WORST.get("tanh_grad_ulp", 0.0), e)
    assert e <= 2.0, e
    _exact(got, act_grad32(v, y, act))  # the fused form the SASS has


def _grid_mask(y):
    g = np.asarray(y, np.float64) * 4096
    return g == np.round(g)


@pytest.mark.parametrize("act", [ACT_NONE, ACT_RELU, ACT_RELU6, ACT_TANH])
@pytest.mark.parametrize("case", HEADS, ids=[c[0] for c in HEADS])
def test_sb_head_bwd(lib, act, case):
    name, B, N, c, lo, rows, O_, frames, rs, bs, steps, t0, _ = case
    if t0:
        pytest.skip("the backward reads whole clips from frame 0")
    R = B * N
    rng = np.random.default_rng(R + O_ + act)
    size = _head_size(B, rows, rs, bs, frames, R)
    for la in sorted({0, min(3, steps - 1)}):
        idx = head_index(R, O_, steps - la, 0, N, c, lo, rows, rs, bs)
        dcrm = rng.standard_normal(size).astype(F32)
        y, _ = _act_out(rng, size, act)
        got = _twice(lambda: run_head_bwd(lib, dcrm, y if act else None, act, R, O_, steps, la, (N, c, lo, rows, rs, bs)))
        assert not np.any(_bits(got[:la]))
        _check_grad(got[la:], dcrm[idx], y[idx], act)


def test_sb_head_bwd_grid_stride(lib):
    """More elements than one pass of the 132 x 16 CTA grid covers."""
    B, N, T = 3, 257, 400
    R = B * N
    rng = np.random.default_rng(9)
    size = B * 2 * N * T
    dcrm = rng.standard_normal(size).astype(F32)
    y, _ = _act_out(rng, size, ACT_RELU)
    got = run_head_bwd(lib, dcrm, y, ACT_RELU, R, 2, T, 2, (N, 1, 0, N, T, 0))
    idx = head_index(R, 2, T - 2, 0, N, 1, 0, N, T, 0)
    _check_grad(got[2:], dcrm[idx], y[idx], ACT_RELU)


@pytest.mark.parametrize("act", [ACT_NONE, ACT_RELU, ACT_RELU6, ACT_TANH])
@pytest.mark.parametrize("B,F,T,la", [(1, 1, 1, 0), (2, 33, 31, 3), (3, 257, 400, 2), (70, 9, 5, 1)])
def test_train_dy(lib, act, B, F, T, la):
    rng = np.random.default_rng(B * F + T + act)
    Tp = T + la
    dout = rng.standard_normal((B, 2, F, T)).astype(F32)
    y, _ = _act_out(rng, (Tp, B, 2 * F), act)
    dd, dy = _dev(dout), _dev(y)

    def run():
        out = Out((Tp, B, 2 * F))
        _call(lib, lib.fsn_debug_train_dy, dd.data_ptr(), dy.data_ptr() if act else None, act, B, F, T, Tp, la, out.ptr)
        return out.get()

    got = _twice(run)
    v = ref_train_dy(dout, None, ACT_NONE, la)
    assert not np.any(_bits(got[:la]))
    _check_grad(got, v, y, act) if act != ACT_TANH else _check_grad(got[la:], v[la:], y[la:], act)


# ------------------------------------------------------------------ long clips
def _unit_sums(mag, fb, Ns, Nf):
    """sum over each unit's K features [Tp, B*F] without the unit tensor: reflect-count matrices of the oracle unfold."""
    from oracle import fullsubnet_oracle as O
    F = mag.shape[1]
    eye = torch.eye(F, dtype=torch.float64)[None, None]  # [1,1,F(rows),F(cols)]

    def cnt(N):
        return O.freq_unfold(eye, N).reshape(F, 2 * N + 1, F).sum(1).numpy()  # [unit f, source row]

    s = np.einsum("fg,bgt->tbf", cnt(Ns), mag.astype(np.float64)) + np.einsum("fg,bgt->tbf", cnt(Nf), fb.astype(np.float64))
    return s.reshape(s.shape[0], -1)


@pytest.mark.parametrize("Tp", [4000, 37500])
def test_long_clip_scans(lib, Tp):
    """The cumulative scans over 4 000 and 37 500 frames (10 min at hop 256): one float32 running sum per clip / row.
    torch's own float32 CPU path (cumsum accumulating in double) is recorded next to it."""
    rng = np.random.default_rng(Tp)
    B, F = 2, 257
    x = (rng.random((B, Tp, F)) + 0.01).astype(F32)
    s = run_clip_scale(lib, x, False)
    _, m, cond = ref_clip_scale(x, EPS_F32)
    _note("cum_long", cum_err(s, m, cond, EPS_F32))
    WORST[f"cum_clip_scale_T{Tp}"] = cum_err(s, m, cond, EPS_F32)
    xt = torch.from_numpy(x)
    m32 = (torch.cumsum(xt.sum(-1), dim=-1) / torch.arange(F, F * Tp + 1, F, dtype=torch.float32)).numpy().T
    RECORD[f"torch_f32_cum_clip_T{Tp}"] = float(np.max(np.abs(m32 - m) / cond))
    # second norm: every sub-band unit of a 33-bin clip, time-major as in training
    Fu, Ns = 33, 15
    mag, fb = (rng.random((B, Fu, Tp)) + 0.01).astype(F32), (rng.random((B, Fu, Tp)) + 0.01).astype(F32)
    su = run_unit_scale(lib, mag, fb, 1, Ns, 0, True)
    sums = _unit_sums(mag, fb, Ns, 0)
    K = 2 * Ns + 2
    mu = np.cumsum(sums, axis=0) / (K * np.arange(1, Tp + 1)[:, None])
    e = cum_err(su, mu, mu, EPS_F32)
    _note("cum_long", e)
    WORST[f"cum_unit_scale_T{Tp}"] = e
    # fast_fullsubnet's second norm over the shrunk steps
    M, S = 8, 2
    mel, enc = (rng.random((B, M, Tp)) + 0.01).astype(F32), (rng.random((B, M, Tp)) + 0.01).astype(F32)
    _, _, sc = run_fast_bn(lib, mel, enc, 1, 0, S, True, True)
    _, U, _ = fast_bottleneck(torch.as_tensor(mel, dtype=torch.float64), torch.as_tensor(enc, dtype=torch.float64), 1, 0, S,
                              True)
    _, mm, cc = ref_cum_scale(U.numpy(), EPS_F32)
    e = cum_err(sc, mm, cc, EPS_F32)
    _note("cum_long", e)
    WORST[f"fast_cum_bn_scale_T{Tp}"] = e
