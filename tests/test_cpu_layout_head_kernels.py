"""The float64 references of the cumulative-norm forward scales, the layout kernels and the sub-band heads, each pinned
to the oracle on the CPU, the proof that the GPU tests' bounds catch planted index bugs, and the CPU-only argument checks
of their hooks and of the entry points whose batch size the layout grids bound.  The references are shared with
tests/test_gpu_layout_head_kernels.py.

- The causal scales are cumulative_laplace_norm's 1 / (running mean + eps) (oracle/fullsubnet_oracle.py), of the noisy
  frame (first norm) and of every sub-band unit: the oracle's freq_unfold of the noisy and full-band rows, concatenated
  and reordered by drop_band (second norm).
- fast_fullsubnet's bottleneck input is the unfold, concat and real_time_downsampling of oracle/fast_fullsubnet_oracle.py
  (fast_bottleneck of tests/test_cpu_norm_layout_kernels.py), and its decoder input the encoder output next to
  real_time_upsampling of the bottleneck output.
- imp_compress is |X|^fdrc with the Nyquist bin dropped (improved_fullsubnet/model.py:564-565).
- The heads are the reshape / permute of fullsubnet/model.py:129-135 and the section scatter of the improved oracle
  (model.py:239-247), written as one index map, head_index, over a cRM geometry (N, c, lo, rows, rs, bs).

A scale's error is taken on the mean it inverts, m = 1 / scale - eps, over the mean of the absolute values of the terms
it sums (cum_err)."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import fast_fullsubnet_oracle as FO
from oracle import fullsubnet_oracle as O
from oracle import improved_fullsubnet_oracle as IO
from test_cpu_norm_layout_kernels import ACT_NONE, ACT_RELU, ACT_RELU6, ACT_TANH, EPS_F32, EPS_OFF, fast_bottleneck, fast_shrunk

D = torch.float64
F32 = np.float32
# bounds of the summing families on |kernel - float64| / conditioning, about 4x the worst error measured on an H100
# 80GB HBM3 (700 W) by tests/test_gpu_layout_head_kernels.py (printed with -s)
TOL = {                         # worst measured
    "cum_clip_scale": 2.5e-6,   # 6.1e-7  frame_stats + cum_clip_scale, up to 300 frames
    "cum_unit_scale": 1.2e-6,   # 2.9e-7  cum_unit_scale, up to 33 frames
    "fast_cum_bn_scale": 1.3e-6,  # 3.1e-7  fast_bn_input + fast_cum_bn_scale
    "fast_bn": 6e-7,            # 1.5e-7  the block means of fast_bn_input
    "fast_bn_sums": 5.5e-7,     # 1.3e-7  its (b, ts) block sums
    "fast_inv2": 6.5e-7,        # 1.6e-7  clip_reduce + norm_scales on the block sums, relative
    "sb_head": 3.5e-7,          # 8.5e-8  sb_head over sum |h||W| + |b|
    "cum_long": 3.6e-5,         # 9.0e-6  the three scans at 4 000 and 37 500 frames
}


# ------------------------------------------------------------------ references
def unit_inputs(mag, fb, Ns, Nf, G):
    """The sub-band units before their norm (fullsubnet/model.py:98-119) of mag, fb [B,F,Tp]: U [Tp, R, K] with
    K = 2Ns+1 + 2Nf+1, the oracle's freq_unfold of both, concatenated, then drop_band with G groups (G <= 1: none)."""
    mag, fb = torch.as_tensor(mag, dtype=D), torch.as_tensor(fb, dtype=D)
    B, F, Tp = mag.shape
    U = torch.cat([O.freq_unfold(mag[:, None], Ns).reshape(B, F, 2 * Ns + 1, Tp),
                   O.freq_unfold(fb[:, None], Nf).reshape(B, F, 2 * Nf + 1, Tp)], dim=2)
    K = U.shape[2]
    if G > 1:
        return O.drop_band(U.permute(0, 2, 1, 3), G).permute(3, 0, 2, 1).reshape(Tp, -1, K).numpy()
    return U.permute(3, 0, 1, 2).reshape(Tp, B * F, K).numpy()


def ref_cum_scale(U, eps):
    """cumulative_laplace_norm's scale of U [Tp, R, K] (mean over the K features and the frames so far): scale [Tp, R],
    its mean m and the mean of |terms| (the conditioning of m)."""
    U = np.asarray(U, np.float64)
    Tp, K = U.shape[0], U.shape[2]
    cnt = K * np.arange(1, Tp + 1, dtype=np.float64)[:, None]
    m = np.cumsum(U.sum(-1), axis=0) / cnt
    cond = np.cumsum(np.abs(U).sum(-1), axis=0) / cnt
    return 1.0 / (m + eps), m, cond


def cum_err(got, m, cond, eps):
    """max |m_got - m| / cond with m_got = 1 / got - eps: the scale's error on the mean it inverts."""
    mg = 1.0 / np.asarray(got, np.float64) - eps
    return float(np.max(np.abs(mg - m) / cond))


def ref_clip_scale(x, eps):
    """first cumulative norm of x [B,Tp,F]: scale1T [Tp,B], m, cond."""
    return ref_cum_scale(np.asarray(x, np.float64).transpose(1, 0, 2), eps)


def ref_transpose_mag(mag, Tp, scale=None):
    """mag [B,F,T] -> [B,Tp,F] with the look-ahead frames T.. zero (model.py:85), and times scale[b] (model.py:92)."""
    B, F, T = mag.shape
    out = np.zeros((B, Tp, F), np.float64)
    out[:, :T] = np.asarray(mag, np.float64).transpose(0, 2, 1)
    return out if scale is None else (out, out * np.asarray(scale, np.float64)[:, None, None])


def ref_crm_output(y, la):
    """y [B,Tp,2F] (channel c*F+f) -> [B,2,F,Tp-la] (fullsubnet/model.py:129-135)."""
    B, Tp, F2 = y.shape
    return np.asarray(y).reshape(B, Tp, 2, F2 // 2).transpose(0, 2, 3, 1)[..., la:]


def ref_scale_rows(x, scale, cols, rows, div):
    i = np.arange(x.size)
    return np.asarray(x, np.float64).reshape(-1) * np.asarray(scale, np.float64)[((i // cols) % rows) // div]


def ref_imp_compress(mag, fdrc):
    """|X|^fdrc without the Nyquist bin (model.py:564-565): [B,F,T] -> [B,T,F-1]."""
    return (np.asarray(mag, np.float64) ** fdrc)[:, :-1].transpose(0, 2, 1)


def ref_dec_input(enc, bn_out, S, Tp):
    """fast_fullsubnet decoder input (model.py:191-194) of enc [B,Tp,M] and bn_out [B,M,Ts]: [B,Tp,2M]."""
    up = FO.real_time_upsampling(torch.as_tensor(bn_out, dtype=D)[:, None], S, Tp)[:, 0]  # [B,M,Tp]
    return np.concatenate([np.asarray(enc, np.float64), up.numpy().transpose(0, 2, 1)], axis=2)


def head_index(R, O, steps, t0, N, c, lo, rows, rs, bs):
    """element of the cRM that output o of row r gets at step s, [steps, R, O] (HeadGeom of fsn_internal.cuh)."""
    s, r, o = np.meshgrid(np.arange(steps), np.arange(R), np.arange(O), indexing="ij")
    b, n, ch, j = r // N, r % N, o // c, o % c
    bstride = bs if bs else 2 * rows * rs
    return b * bstride + (ch * rows + lo + n * c + j) * rs + t0 + s


def act64(z, act):
    return {ACT_NONE: lambda v: v, ACT_RELU: lambda v: np.maximum(v, 0), ACT_TANH: np.tanh,
            ACT_RELU6: lambda v: np.clip(v, 0, 6)}[act](z)


def ref_sb_head(h, W, bias, act):
    """act(h W^T + b) of h [steps, R, H] in float64 and the conditioning sum |h||W| + |b| (both [steps, R, O])."""
    h, W, bias = (np.asarray(a, np.float64) for a in (h, W, bias))
    z = h @ W.T + bias
    return act64(z, act), np.abs(h) @ np.abs(W).T + np.abs(bias), z


def act_grad64(v, y, act):
    """v times the derivative of act from its output y (float64)."""
    v, y = np.asarray(v, np.float64), np.asarray(y, np.float64)
    if act == ACT_RELU:
        return np.where(y > 0, v, 0.0)
    if act == ACT_RELU6:
        return np.where((y > 0) & (y < 6), v, 0.0)
    if act == ACT_TANH:
        return v * (1.0 - y * y)
    return v


def act_grad32(v, y, act):
    """the kernels' float32 act_grad: the tanh form is fused, d = fmaf(-y, y, 1) rounded once, then v * d.  Exact for
    the y whose 1 - y^2 is a float64 without rounding (|y| of at most 12 fraction bits)."""
    v, y = np.asarray(v, F32), np.asarray(y, F32)
    if act == ACT_TANH:
        d = (1.0 - y.astype(np.float64) ** 2).astype(F32)
        return (v * d).astype(F32)
    return act_grad64(v, y, act).astype(F32)


def ref_train_dy(dout, y, act, la):
    """dY [Tp,B,2F] of dout [B,2,F,T]: frame t - la (0 before), times act'(y [Tp,B,2F])."""
    B, _, F, T = dout.shape
    v = np.zeros((T + la, B, 2 * F), np.float64)
    v[la:] = np.asarray(dout, np.float64).reshape(B, 2 * F, T).transpose(2, 0, 1)
    return v


# ------------------------------------------------------------------ pins
@pytest.mark.parametrize("B,F,Tp,Ns,Nf,G", [(3, 7, 5, 2, 0, 1), (5, 9, 4, 3, 1, 3), (7, 10, 3, 9, 2, 4), (4, 2, 6, 1, 1, 1)])
def test_cum_scales_are_cumulative_laplace_norm(B, F, Tp, Ns, Nf, G):
    """ref_cum_scale of the unit inputs is the scale the oracle's cumulative_laplace_norm applies, with drop_band's row
    order; ref_clip_scale is the first norm's."""
    g = torch.Generator().manual_seed(B * F)
    mag, fb = torch.rand(B, F, Tp, generator=g, dtype=D) + 0.1, torch.rand(B, F, Tp, generator=g, dtype=D) + 0.1
    U = unit_inputs(mag, fb, Ns, Nf, G)
    s, m, cond = ref_cum_scale(U, EPS_F32)
    K = U.shape[2]
    cat = torch.cat([O.freq_unfold(mag[:, None], Ns).reshape(B, F, 2 * Ns + 1, Tp),
                     O.freq_unfold(fb[:, None], Nf).reshape(B, F, 2 * Nf + 1, Tp)], dim=2)
    X = O.cumulative_laplace_norm(cat)
    if G > 1:
        X = O.drop_band(X.permute(0, 2, 1, 3), G).permute(3, 0, 2, 1).reshape(Tp, -1, K)
    else:
        X = X.permute(3, 0, 1, 2).reshape(Tp, B * F, K)
    np.testing.assert_allclose(X.numpy(), U * s[:, :, None], rtol=1e-13)
    np.testing.assert_allclose(cond, m, rtol=1e-13)  # positive inputs: the conditioning is the mean itself
    src_b, src_f = O.drop_band_index_map(B, F, G) if G > 1 else (np.arange(B), np.tile(np.arange(F), (B, 1)))
    Fsub = U.shape[1] // B
    np.testing.assert_allclose(U[:, :, Ns], mag.numpy()[np.repeat(src_b, Fsub), np.asarray(src_f).reshape(-1)].T,
                               rtol=0)  # the centre row of each unit
    x = mag.permute(0, 2, 1).numpy()
    s1, _, _ = ref_clip_scale(x, EPS_F32)
    np.testing.assert_allclose((O.cumulative_laplace_norm(mag[:, None]) / mag[:, None])[:, 0, 0].numpy().T, s1, rtol=1e-13)


def test_layout_references_follow_the_oracle():
    g = torch.Generator().manual_seed(7)
    B, F, T, la = 3, 5, 6, 2
    mag = torch.rand(B, F, T, generator=g, dtype=D)
    pad = torch.nn.functional.pad(mag[:, None], [0, la])[:, 0]  # model.py:85
    out, sc = ref_transpose_mag(mag.numpy(), T + la, scale=np.arange(1, B + 1))
    np.testing.assert_array_equal(out, pad.permute(0, 2, 1).numpy())
    np.testing.assert_array_equal(sc, out * np.arange(1, B + 1)[:, None, None])
    # the head Linear's rows (b,t) of 2F -> the cRM of fullband_baseline/model.py:58-62
    y = torch.rand(B, T + la, 2 * F, generator=g, dtype=D)
    crm = y.permute(0, 2, 1).reshape(B, 2, F, T + la)[..., la:]
    np.testing.assert_array_equal(ref_crm_output(y.numpy(), la), crm.numpy())
    # improved: |X|^fdrc without Nyquist, as the oracle forward computes it
    for fdrc in (0.5, 0.3, 1.0):
        np.testing.assert_allclose(ref_imp_compress(mag.numpy(), fdrc),
                                   (mag[:, None] ** fdrc)[..., :-1, :][:, 0].permute(0, 2, 1).numpy(), rtol=1e-15)
    # fast_fullsubnet: the bottleneck input means are real_time_downsampling's, the decoder reads real_time_upsampling
    M, Tp, S = 4, 8, 3
    mel, enc = torch.rand(B, M, Tp, generator=g, dtype=D), torch.rand(B, M, Tp, generator=g, dtype=D)
    X, U, m = fast_bottleneck(mel, enc, 1, 0, S, True)
    assert U.shape == (fast_shrunk(Tp, S), B * M, 4)
    np.testing.assert_allclose(U[1, :, 1].numpy(), mel[:, :, 1:1 + S].mean(-1).reshape(-1).numpy(), rtol=1e-14)
    bn_out = torch.rand(B, M, U.shape[0], generator=g, dtype=D)
    dec = ref_dec_input(enc.permute(0, 2, 1).numpy(), bn_out.numpy(), S, Tp)
    np.testing.assert_array_equal(dec[:, 4, M:], bn_out[:, :, 4 // S].numpy())
    np.testing.assert_array_equal(dec[:, :, :M], enc.permute(0, 2, 1).numpy())


@pytest.mark.parametrize("B,F,G,la", [(3, 6, 1, 0), (5, 9, 3, 2), (2, 4, 1, 1)])
def test_fullsubnet_head_index_is_the_reshape_permute(B, F, G, la):
    """fullsubnet's sub-band Linear output [B*Fsub, T, 2] through model.py:129-135 lands where head_index (N = Fsub,
    c = 1) puts it; the training call's geometry (offset by la, steps = Tp - la) drops the look-ahead frames."""
    Fsub = F // G if G > 1 else F
    R, Tp = B * Fsub, 7
    out = np.arange(R * Tp * 2, dtype=np.float64).reshape(R, Tp, 2)  # sequence_model output [R, Tp, 2]
    crm = torch.as_tensor(out).permute(0, 2, 1).reshape(B, Fsub, 2, Tp).permute(0, 2, 1, 3)[..., la:]
    T = Tp - la
    idx = head_index(R, 2, T, 0, Fsub, 1, 0, Fsub, T, 0)
    got = np.zeros(B * 2 * Fsub * T)
    got[idx] = out[:, la:].transpose(1, 0, 2)
    np.testing.assert_array_equal(got.reshape(B, 2, Fsub, T), crm.numpy())


def test_improved_head_index_is_the_section_scatter():
    """Each improved section's Linear(H -> 2c) output through model.py:239-247, concatenated and padded with the Nyquist
    row, is head_index with (N, c, lo) of the section and rows = F; rows outside the section stay untouched."""
    B, Fu, T = 2, 12, 3
    F = Fu + 1
    crm = np.zeros(B * 2 * F * T)
    outs = []
    for lo, hi, cs in [(0, 4, 2), (4, 12, 4)]:
        N = (hi - lo) // cs
        o = torch.randn(B * N, 2 * cs, T, dtype=D)  # seq_time_major output per unit [B*N, 2c, T]
        outs.append(o.reshape(B, N, 2, -1, T).permute(0, 2, 1, 3, 4).reshape(B, 2, -1, T))
        idx = head_index(B * N, 2 * cs, T, 0, N, cs, lo, F, T, 0)
        crm[idx] = o.permute(2, 0, 1).numpy()
    ref = torch.nn.functional.pad(torch.cat(outs, dim=-2), (0, 0, 0, 1))
    np.testing.assert_array_equal(crm.reshape(B, 2, F, T), ref.numpy())


def test_tanh_derivative_emulation():
    """The fused form 1 - y^2 (one rounding, then v * d) is exact on y with 12 fraction bits and within 2 ulp of the
    float64 product elsewhere."""
    rng = np.random.default_rng(0)
    y = (rng.integers(-4095, 4096, 1000) / 4096.0).astype(F32)
    v = rng.standard_normal(1000).astype(F32)
    exact = act_grad64(v, y, ACT_TANH)
    np.testing.assert_array_equal(act_grad32(v, y, ACT_TANH), exact.astype(F32))
    y = np.tanh(rng.standard_normal(1000)).astype(F32)
    got = act_grad32(v, y, ACT_TANH).astype(np.float64)
    ulp = np.spacing(np.abs(act_grad64(v, y, ACT_TANH)).astype(F32)).astype(np.float64)
    assert np.all(np.abs(got - act_grad64(v, y, ACT_TANH)) <= 2 * ulp)


# ------------------------------------------------------------------ the bounds catch planted bugs
def _seq32_scale(U, eps):
    """a float32 scan of the kernels' shape: one running float32 sum per row over the frames' float32 sums."""
    U = np.asarray(U, F32)
    Tp, R, K = U.shape
    run = np.zeros(R, F32)
    out = np.empty((Tp, R), F32)
    for t in range(Tp):
        run = (run + U[t].sum(-1, dtype=F32)).astype(F32)
        out[t] = F32(1.0) / (run / (F32(K) * F32(t + 1)) + F32(eps))
    return out


def test_bounds_catch_planted_bugs():
    rng = np.random.default_rng(3)
    B, F, Tp, Ns, Nf, G = 5, 33, 40, 3, 1, 2
    mag, fb = rng.random((B, F, Tp)) + 0.05, rng.random((B, F, Tp)) + 0.05
    U = unit_inputs(mag, fb, Ns, Nf, G)
    s, m, cond = ref_cum_scale(U, EPS_F32)
    ok = cum_err(_seq32_scale(U, EPS_F32), m, cond, EPS_F32)
    assert ok < TOL["cum_unit_scale"], ok
    # a dropped reflected neighbour (the last noisy row of each unit)
    drop = np.delete(U, 2 * Ns, axis=2)
    bad = _seq32_scale(np.concatenate([drop, drop[:, :, :1] * 0], axis=2), EPS_F32)
    assert cum_err(bad, m, cond, EPS_F32) > 100 * TOL["cum_unit_scale"]
    # the scale of the neighbouring clip
    x = rng.random((B, Tp, F)) + 0.05
    s1, m1, c1 = ref_clip_scale(x, EPS_F32)
    good = _seq32_scale(x.transpose(1, 0, 2), EPS_F32)
    assert cum_err(good, m1, c1, EPS_F32) < TOL["cum_clip_scale"]
    assert cum_err(np.roll(good, 1, axis=1), m1, c1, EPS_F32) > 100 * TOL["cum_clip_scale"]
    # the look-ahead off by one, in the cRM re-layout and the two backward re-layouts
    y = rng.standard_normal((B, Tp, 2 * F)).astype(F32)
    for la in (1, 2):
        n = Tp - la - 1
        assert not np.array_equal(ref_crm_output(y, la)[..., :n], ref_crm_output(y, la + 1)[..., :n])
        assert not np.array_equal(ref_crm_output(y, la)[..., :n], ref_crm_output(y, la - 1)[..., :n])
    dout = rng.standard_normal((B, 2, F, Tp - 2))
    assert not np.array_equal(ref_train_dy(dout, None, ACT_NONE, 2)[1:], ref_train_dy(dout, None, ACT_NONE, 1)[1:])
    # a 32-wide tile shifted by one frame
    mag32 = rng.random((2, 40, 70)).astype(F32)
    good = ref_transpose_mag(mag32, 72)
    bad = good.copy()
    bad[:, 32:64] = ref_transpose_mag(mag32, 72)[:, 33:65]
    assert not np.array_equal(good, bad)
    # the scale of clip b + 1 in the scaled copy
    sc = rng.random(2) + 0.5
    _, scaled = ref_transpose_mag(mag32, 72, sc)
    assert not np.array_equal(scaled.astype(F32), (good * np.roll(sc, 1)[:, None, None]).astype(F32))
    # a head row lo + n c + j off by one
    R, O_, T = 2 * 3, 4, 5
    a = head_index(R, O_, T, 0, 3, 2, 4, 12, T, 0)
    b = head_index(R, O_, T, 0, 3, 2, 5, 12, T, 0)
    vals = rng.standard_normal(a.shape)
    out_a, out_b = np.zeros(2 * 2 * 12 * T), np.zeros(2 * 2 * 12 * T)
    out_a[a] = vals
    out_b[b] = vals
    assert not np.array_equal(out_a, out_b)
    # a head sum with a dropped k term is far outside the sb_head bound
    h, W = rng.standard_normal((2, 8, 40)), rng.standard_normal((2, 40))
    yv, cnd, _ = ref_sb_head(h, W, np.zeros(2), ACT_NONE)
    got = (h[..., :-1] @ W[:, :-1].T)
    assert np.max(np.abs(got - yv) / cnd) > 100 * TOL["sb_head"]
    faithful = np.einsum("srh,oh->sro", h.astype(F32), W.astype(F32), dtype=F32)
    assert np.max(np.abs(faithful - yv) / cnd) < TOL["sb_head"]


# ------------------------------------------------------------------ refusals without a GPU
P = 1 << 20  # stand-in device pointer: every call below returns before it could be used


@pytest.fixture(scope="module")
def lib():
    from fullsubnet_b200 import _lib
    return _lib.load()


def _expect(lib, rc, code, text=None):
    assert rc == code, (rc, lib.fsn_last_error())
    assert lib.fsn_last_error_code() == code
    if text:
        assert text in lib.fsn_last_error(), lib.fsn_last_error()


def test_layout_head_hooks_refuse_before_any_cuda_call(lib):
    from fullsubnet_b200 import _lib
    SH, UN = _lib.FSN_ERR_SHAPE, _lib.FSN_ERR_UNSUPPORTED
    ex = (lambda rc, code, text=None: _expect(lib, rc, code, text))

    def clip(x=P, fs=P, B=2, Tp=5, F=9):
        return lib.fsn_debug_cum_clip_scale(x, B, Tp, F, Tp * F, F, 1e-7, fs, P, None)

    ex(clip(x=None), SH, b"null")
    ex(clip(fs=None), SH, b"null")
    ex(clip(B=0), SH)
    ex(clip(Tp=0), SH)
    ex(clip(B=70000, Tp=40000), SH, b"2^31")

    def unit(magT=P, B=5, F=9, G=2, Tp=4, Ns=2, Nf=0):
        return lib.fsn_debug_cum_unit_scale(magT, P, B, F, G, Tp, Ns, Nf, 1e-7, 0, P, None)

    ex(unit(magT=None), SH, b"null")
    ex(unit(G=5), SH, b"B > G")
    ex(unit(F=1, G=2), SH, b"B > G")
    ex(unit(Ns=9), SH, b"< F")
    ex(unit(Nf=-1), SH)
    ex(unit(Tp=0), SH)
    ex(lib.fsn_debug_forget_unit_broadcast(None, 5, 9, 2, 4, P, None), SH, b"null")
    ex(lib.fsn_debug_forget_unit_broadcast(P, 3, 9, 3, 4, P, None), SH, b"B > G")
    ex(lib.fsn_debug_forget_unit_broadcast(P, 3, 9, 1, 0, P, None), SH)

    def fbn(sums=P, cum=0, M=5, Nn=1, Ne=2, S=2, Tp=7):
        return lib.fsn_debug_fast_bn(P, P, Tp * M, M, 2, Tp, M, Nn, Ne, S, cum, 1e-5, P, P, sums, P, None)

    ex(fbn(sums=None), SH, b"null")   # the offline scale needs the clip sums
    ex(fbn(S=0), SH)
    ex(fbn(Nn=5), SH, b"< M")
    ex(fbn(Ne=5), SH, b"< M")

    def dec(rbs=7, rts=1, S=2, Ts=4):
        return lib.fsn_debug_fast_dec_input(P, P, 5 * Ts, Ts, 1, 2, 7, 5, S, Ts, rbs, rts, P, None)

    ex(dec(rbs=7, rts=2), SH, b"clip-major")
    ex(dec(S=0), SH)
    ex(dec(Ts=0), SH)
    ex(lib.fsn_debug_fast_dec_input(None, P, 1, 1, 1, 2, 7, 5, 2, 4, 7, 1, P, None), SH, b"null")

    def tm(B=2, F=9, T=5, Tp=7, scale=None, scaled=None):
        return lib.fsn_debug_transpose_mag(P, B, F, T, Tp, Tp * F, F, P, scale, scaled, None)

    ex(tm(scaled=P), SH, b"null")     # a scaled copy needs its scale
    ex(tm(Tp=4), SH)                  # Tp < T
    ex(tm(B=65536), UN, b"at most 65535")
    ex(tm(F=65535 * 32 + 1), UN, b"grid")

    def crm(B=2, Tp=7, F=9, la=2):
        return lib.fsn_debug_crm_output(P, Tp * 2 * F, 2 * F, B, Tp, F, la, P, None)

    ex(crm(la=7), SH)                 # no frame left
    ex(crm(la=-1), SH)
    ex(crm(B=32768), UN, b"at most 32767")
    ex(lib.fsn_debug_crm_output(None, 1, 1, 2, 7, 9, 2, P, None), SH, b"null")

    ex(lib.fsn_debug_scale_rows(P, None, 10, 5, 2, 1, P, None), SH, b"null")
    ex(lib.fsn_debug_scale_rows(P, P, 10, 5, 2, 0, P, None), SH)
    ex(lib.fsn_debug_scale_rows(P, P, 0, 5, 2, 1, P, None), SH)

    ex(lib.fsn_debug_imp_compress(None, 2, 9, 5, 0.5, 0, P, None), SH, b"null")
    ex(lib.fsn_debug_imp_compress(P, 2, 1, 5, 0.5, 0, P, None), SH)  # nothing left without the Nyquist bin
    ex(lib.fsn_debug_imp_compress(P, 65536, 9, 5, 0.5, 1, P, None), UN, b"at most 65535")

    def gat(inv2=P, us=None, B=5, F=9, G=2, Ns=2, Nf=0):
        return lib.fsn_debug_train_gather(P, P, inv2, us, B, F, G, 4, Ns, Nf, P, None)

    ex(gat(inv2=None), SH, b"null")   # a scale is needed: inv2 or the per-unit scales
    ex(gat(G=5), SH, b"B > G")
    ex(gat(Ns=9), SH, b"< F")
    ex(gat(Nf=9), SH, b"< F")

    def head(R=6, O=2, N=3, c=1, lo=0, rows=3, rs=5, bs=0, t0=0, steps=5, act=0, bias=P):
        return lib.fsn_debug_sb_head(P, R, 8, steps, P, bias, O, act, N, c, lo, rows, rs, bs, t0, P, None)

    ex(head(bias=None), SH, b"null")
    ex(head(R=7), SH, b"whole clips")
    ex(head(O=3), SH, b"2c")
    ex(head(lo=1), SH, b"exceed rows")
    ex(head(rows=0), SH, b"exceed rows")  # one-channel table with two outputs
    ex(head(rs=0), SH)
    ex(head(t0=-1), SH)
    ex(head(act=4), SH, b"act")
    ex(head(R=1 << 20, N=1 << 20, rows=1 << 20, steps=1 << 14), SH, b"grid")

    def hbwd(y=P, act=1, la=0, O=2, c=1):
        return lib.fsn_debug_sb_head_bwd(P, y, act, 6, O, 5, la, 3, c, 0, 3, 5, 0, P, None)

    ex(hbwd(y=None), SH, b"null")    # ReLU' needs the kept output
    ex(hbwd(la=-1), SH)
    ex(hbwd(O=3), SH, b"2c")
    ex(hbwd(act=7), SH, b"act")

    def dy(y=P, act=3, T=5, Tp=7, la=2):
        return lib.fsn_debug_train_dy(P, y, act, 2, 9, T, Tp, la, P, None)

    ex(dy(y=None), SH, b"null")
    ex(dy(Tp=8), SH, b"Tp = T + la")
    ex(dy(act=-1), SH, b"act")


def test_entry_points_refuse_batches_beyond_the_layout_grids(lib):
    """transpose_mag and imp_compress put the clip in gridDim.z, crm_output the (clip, channel) pair: every entry point
    that reaches them refuses a larger batch before any CUDA call (stand-in pointers, never read)."""
    from fullsubnet_b200 import _lib
    UN = _lib.FSN_ERR_UNSUPPORTED
    ex = (lambda rc, text: _expect(lib, rc, UN, text))
    d = _lib.ModelDesc(num_freqs=257, look_ahead=2, fb_num_neighbors=0, sb_num_neighbors=15, fb_hidden=512, sb_hidden=384,
                       fb_activation=1, sb_activation=0, norm_type=0, num_groups_in_drop_band=2, precision=0, cell_type=0)
    ex(lib.fsn_model_forward(C.byref(d), None, None, None, P, 65536, 10, P, P, 1 << 40, None), b"model: B=65536")
    assert lib.fsn_model_forward(C.byref(d), None, None, None, P, 65535, 10, P, None, 0, None) == _lib.FSN_ERR_WORKSPACE
    ex(lib.fsn_train_forward(C.byref(d), None, None, P, 65536, 10, P, P, 1 << 40, None), b"training: B=65536")
    fbb = _lib.FullbandDesc(num_freqs=257, hidden=512, num_layers=3, look_ahead=2, activation=0, norm_type=0, precision=0,
                            cell_type=0)
    ex(lib.fsn_fullband_forward(C.byref(fbb), P, P, P, P, 32768, 10, P, P, 1 << 40, None), b"fullband: B=32768")
    assert lib.fsn_fullband_forward(C.byref(fbb), P, P, P, P, 32767, 10, P, None, 0, None) == _lib.FSN_ERR_WORKSPACE
    # the STFT's own limit is 65535 clips: fullband_enhance used to pass its checks here and fail at crm_output's launch
    ex(lib.fsn_fullband_enhance(C.byref(fbb), P, P, P, P, None, 32768, 4000, 512, 256, 512, P, None, None, 1.0, P, 1 << 40,
                                None), b"fullband_enhance: B=32768")
    ex(lib.fsn_fullband_train_forward(C.byref(fbb), P, P, P, P, 32768, 10, P, P, 1 << 40, None), b"fullband training")
    fd = _lib.FastDesc(num_freqs=257, look_ahead=2, shrink_size=2, num_mels=64, enc1_hidden=384, enc2_hidden=257,
                       bn_hidden=384, bn_layers=2, dec_hidden=512, noisy_num_neighbors=5, enc_num_neighbors=0, precision=0,
                       cell_type=0)
    ex(lib.fsn_fast_model_forward(C.byref(fd), None, P, 32768, 10, P, P, 1 << 40, None), b"fast model: B=32768")
    ex(lib.fsn_fast_train_forward(C.byref(fd), None, P, 32768, 10, P, P, 1 << 40, None), b"fast training: B=32768")
