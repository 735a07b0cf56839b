"""The float64 references of the norm and frequency-unfold kernels, each pinned to an authority on the CPU, and the
CPU-only argument checks of their test hooks.  The references are shared with tests/test_gpu_norm_layout_kernels.py.
The kernels are the frame / clip statistics and scales of the offline norms, the improved section input (a pure
re-layout of the spectrogram rows), and the backward of the second norm and the unfolds of every training step.

The statistics reference sums each frame and its N-neighbour unfold (freq_unfold), and the scales are 1 / (mean + eps)
of offline_laplace_norm's mean.

Each reference is torch.autograd in float64 through the reference model's own forward, composed from the oracle ports:
- fullsubnet (fsn_debug_norm_unfold_bwd): the noisy magnitude unfolded with Ns neighbours next to the full-band output
  (freq_unfold of oracle/fullsubnet_oracle.py), offline_laplace_norm or cumulative_laplace_norm, then drop_band;
- fast_fullsubnet (fsn_debug_fast_norm_unfold_bwd): the noisy-mel and encoder-output unfolds, real_time_downsampling and
  the second norm, and real_time_upsampling of the bottleneck output (oracle/fast_fullsubnet_oracle.py);
- improved_fullsubnet (fsn_debug_imp_unfold_bwd): the section unfolds of oracle/improved_fullsubnet_oracle.py and its
  offline_laplace_norm, summed over the sections.

Each forward is also written out as U / (m + eps), with U the sub-band input before the norm and m the norm's mean laid
out like U.  That form gives each gradient's conditioning: the gradient of sum |dX| U s + sum |dX X| s m with
s = 1 / (m + eps) held constant, the sum of the absolute values of the terms the kernels add.  The tests pin it to the
oracle forward, the unfolds to reflect_count and drop_band_index_map, and each adjoint to torch.autograd.gradcheck at
small shapes."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import fast_fullsubnet_oracle as FO
from oracle import fullsubnet_oracle as O
from oracle import improved_fullsubnet_oracle as IO

D = torch.float64
EPS_OFF = 1e-5                                    # audio_zen/model/base_model.py:203-218
EPS_F32 = float(np.finfo(np.float32).eps)         # cumulative norm; improved_fullsubnet/model.py:23
ACT_NONE, ACT_RELU, ACT_TANH, ACT_RELU6 = 0, 1, 2, 3


def act_fn(act):
    return {ACT_NONE: lambda z: z, ACT_RELU: torch.relu, ACT_TANH: torch.tanh,
            ACT_RELU6: lambda z: torch.clamp(z, 0, 6)}[act]


def _cum_mean(U):
    """cumulative_laplace_norm's mean of U [..., K, T]: over the K features and the frames so far."""
    K, T = U.shape[-2], U.shape[-1]
    cnt = K * torch.arange(1, T + 1, dtype=U.dtype)
    return (torch.cumsum(U.sum(dim=-2), dim=-1) / cnt).unsqueeze(-2).expand_as(U)


def _clip_mean(U):
    return U.mean(dim=list(range(1, U.dim())), keepdim=True).expand_as(U)


def _grad(loss, z):
    return torch.autograd.grad(loss, z, retain_graph=True)[0]


# ------------------------------------------------------------------ fullsubnet
def fsn_sub_band(mag, y, Ns, G, cum):
    """Model.forward's sub-band input (fullsubnet/model.py:98-119) of mag, y [B,F,Tp]: X [Tp, B*Fsub, K] (oracle
    functions), and U, m in the same layout with X = U / (m + eps)."""
    B, F, Tp = mag.shape
    K = 2 * Ns + 2
    U = torch.cat([O.freq_unfold(mag[:, None], Ns).reshape(B, F, 2 * Ns + 1, Tp),
                   O.freq_unfold(y[:, None], 0).reshape(B, F, 1, Tp)], dim=2)  # [B,F,K,Tp]
    X = O.cumulative_laplace_norm(U) if cum else O.offline_laplace_norm(U)
    m = _cum_mean(U) if cum else _clip_mean(U)

    def lay(a):
        if G > 1 and B > 1:
            a = O.drop_band(a.permute(0, 2, 1, 3), G)  # [B, K, Fsub, Tp]
            return a.permute(3, 0, 2, 1).reshape(Tp, -1, K)
        return a.permute(3, 0, 1, 2).reshape(Tp, B * F, K)

    return lay(X), lay(U), lay(m)


def ref_fsn_norm_bwd(mag, z, dX, Ns, G, act, cum, dtype=D):
    """d <dX, X> / d z of the full-band output y = act(z) (all [B,F,Tp], float64, or torch's own arithmetic in dtype):
    returns dz, its conditioning (both [Tp,B,F]) and the kernel inputs X [Tp,R,K], fbz = y [Tp,B,F], scale (inv2 [B] or
    scaleT [Tp,R])."""
    z = torch.as_tensor(z, dtype=dtype).clone().requires_grad_(True)
    mag = torch.as_tensor(mag, dtype=dtype)
    dX = torch.as_tensor(dX, dtype=dtype)
    y = act_fn(act)(z)
    X, U, m = fsn_sub_band(mag, y, Ns, G, cum)
    dz = _grad((X * dX).sum(), z)
    eps = EPS_F32 if cum else EPS_OFF
    s = (1.0 / (m + eps)).detach()
    cond = _grad((dX.abs() * U * s).sum() + ((dX * X).abs().detach() * s * m).sum(), z)
    if cum:
        scale = s[:, :, 0]
    else:  # inv2 of each input clip (drop_band reorders the rows, not the clips' means)
        scale = (1.0 / (fsn_sub_band(mag, y, Ns, 1, False)[1].reshape(mag.shape[2], mag.shape[0], -1).mean(dim=(0, 2))
                        + eps)).detach()
    tm = (lambda a: a.permute(2, 0, 1).contiguous())
    return (tm(dz).detach().numpy(), tm(cond).detach().numpy(), X.detach().numpy(), tm(y).detach().numpy(),
            scale.detach().numpy())


# ------------------------------------------------------------------ fast_fullsubnet
def fast_shrunk(Tp, S):
    return 1 + -(-(Tp - 1) // S)


def fast_bottleneck(mel, enc, Nn, Ne, S, cum):
    """fast_fullsubnet's bottleneck input (model.py:174-187) of mel, enc [B,M,Tp]: X [Ts, B*M, K], U, m alike."""
    B, M, Tp = mel.shape
    U = torch.cat([O.freq_unfold(mel[:, None], Nn).reshape(B, M, 2 * Nn + 1, Tp),
                   O.freq_unfold(enc[:, None], Ne).reshape(B, M, 2 * Ne + 1, Tp)], dim=2)
    U = FO.real_time_downsampling(U, S)  # [B,M,K,Ts]
    X = O.cumulative_laplace_norm(U) if cum else O.offline_laplace_norm(U)
    m = _cum_mean(U) if cum else _clip_mean(U)
    K, Ts = U.shape[2], U.shape[3]
    lay = (lambda a: a.permute(3, 0, 1, 2).reshape(Ts, B * M, K))
    return lay(X), lay(U), lay(m)


def ref_fast_bwd(mel, z, zb, ddec, dX, Nn, Ne, S, cum):
    """fast_fullsubnet backward of L = <ddec, dec_in> + <dX, X_bn> (float64): the encoder output is relu(z) [B,M,Tp],
    the bottleneck output relu(zb) [B,M,Ts], ddec [Tp,B,2M], dX [Ts,B*M,K].  Returns d z [Tp,B,M], its conditioning,
    d zb [Ts,B*M] and its conditioning, and the kernel inputs X, encT [Tp,B,M], bn_out [Ts,B*M], scale."""
    mel = torch.as_tensor(mel, dtype=D)
    ddec = torch.as_tensor(ddec, dtype=D)
    dX = torch.as_tensor(dX, dtype=D)
    z = torch.as_tensor(z, dtype=D).clone().requires_grad_(True)
    zb = torch.as_tensor(zb, dtype=D).clone().requires_grad_(True)
    B, M, Tp = mel.shape
    enc = torch.relu(z)
    X, U, m = fast_bottleneck(mel, enc, Nn, Ne, S, cum)
    tm = (lambda a: a.permute(2, 0, 1))  # [B,M,T] -> [T,B,M]
    dz = _grad((X * dX).sum() + (ddec[:, :, :M] * tm(enc)).sum(), z)
    eps = EPS_F32 if cum else EPS_OFF
    s = (1.0 / (m + eps)).detach()
    cond = _grad((dX.abs() * U * s).sum() + ((dX * X).abs().detach() * s * m).sum()
                 + (ddec[:, :, :M].abs() * tm(enc)).sum(), z)
    bn_out = torch.relu(zb)
    up = FO.real_time_upsampling(bn_out[:, None], S, Tp)[:, 0]  # [B,M,Tp]
    dzb = _grad((ddec[:, :, M:] * tm(up)).sum(), zb)
    condb = _grad((ddec[:, :, M:].abs() * tm(up)).sum(), zb)
    Ts = bn_out.shape[2]
    rows = (lambda a: a.permute(2, 0, 1).reshape(Ts, B * M))
    scale = s[:, :, 0] if cum else s[0, ::M, 0]
    n = (lambda a: a.detach().contiguous().numpy())
    return (n(tm(dz)), n(tm(cond)), n(rows(dzb)), n(rows(condb)), n(X), n(tm(enc)), n(rows(bn_out)), n(scale))


# ------------------------------------------------------------------ improved_fullsubnet
def imp_section(noisy, y, sec):
    """Section input (model.py:321-443) of noisy, y [B,Fu,T] for sec = (lo, hi, cs, ns, cf, nf): X [T, B*N, W], U, m."""
    lo, hi, cs, ns, cf, nf = sec
    B, Fu, T = noisy.shape
    U = torch.cat([IO.freq_unfold(noisy[:, None], lo, hi, cs, ns), IO.freq_unfold(y[:, None], lo, hi, cf, nf)], dim=-2)
    X = IO.offline_laplace_norm(U)
    m = _clip_mean(U)
    N, W = U.shape[1], U.shape[3]
    lay = (lambda a: a[:, :, 0].permute(3, 0, 1, 2).reshape(T, B * N, W))
    return lay(X), lay(U), lay(m)


def ref_imp_bwd(noisy, z, dXs, secs, act):
    """d sum_s <dX_s, X_s> / d z of the full-band output y = act(z) [B,Fu,T] over the sections secs (float64).  Returns
    dz [T,B,Fu], its conditioning, y [T,B,Fu] and per section (X_s, invs_s [B])."""
    noisy = torch.as_tensor(noisy, dtype=D)
    z = torch.as_tensor(z, dtype=D).clone().requires_grad_(True)
    y = act_fn(act)(z)
    loss, closs, per = 0.0, 0.0, []
    for sec, dX in zip(secs, dXs):
        dX = torch.as_tensor(dX, dtype=D)
        X, U, m = imp_section(noisy, y, sec)
        s = (1.0 / (m + EPS_F32)).detach()
        loss = loss + (X * dX).sum()
        closs = closs + (dX.abs() * U * s).sum() + ((dX * X).abs().detach() * s * m).sum()
        N = X.shape[1] // noisy.shape[0]
        per.append((X.detach().numpy(), s[0, ::N, 0].numpy().copy()))
    dz, cond = _grad(loss, z), _grad(closs, z)
    tm = (lambda a: a.detach().permute(2, 0, 1).contiguous().numpy())
    return tm(dz), tm(cond), tm(y), per


# ------------------------------------------------------------------ statistics of the offline norms
def ref_frame_stats(x, N):
    """x [B,T,F] -> (sum_f x, the sum of the frame's N-neighbour unfold (fullsubnet/model.py:98-105)), both [B,T]."""
    x = torch.as_tensor(x, dtype=D)
    u = O.freq_unfold(x.permute(0, 2, 1)[:, None], N)  # [B,F,1,2N+1,T]
    return x.sum(-1).numpy(), u.sum(dim=(1, 2, 3)).numpy()


def ref_inv(parts, eps=EPS_OFF):
    """1 / (offline_laplace_norm's mean of the concatenation of parts + eps), parts [B, ...] each."""
    cat = torch.cat([torch.as_tensor(p, dtype=D).reshape(p.shape[0], -1) for p in parts], dim=1)
    return (1.0 / (cat.mean(dim=1) + eps)).numpy()


# ------------------------------------------------------------------ pins
@pytest.mark.parametrize("F,N", [(257, 15), (161, 15), (2, 1), (33, 0)])
def test_frame_stats_reference(F, N):
    """The unfold sum is the reflect_count-weighted sum, and ref_inv is offline_laplace_norm's scale."""
    g = torch.Generator().manual_seed(4)
    x = torch.rand(2, 3, F, generator=g, dtype=D)
    s0, s1 = ref_frame_stats(x, N)
    np.testing.assert_allclose(s1, (x.numpy() * O.reflect_count(F, N)).sum(-1), rtol=1e-13)
    np.testing.assert_allclose(s0, x.sum(-1).numpy(), rtol=1e-13)
    X = O.offline_laplace_norm(x)
    np.testing.assert_allclose(ref_inv([x.numpy()]), (X / x)[:, 0, 0].numpy(), rtol=1e-13)


def test_explicit_norm_forms_match_the_oracle_functions():
    """U / (m + eps) of each reference equals the oracle forward, including drop_band with G not dividing F."""
    g = torch.Generator().manual_seed(0)
    for cum in (False, True):
        eps = EPS_F32 if cum else EPS_OFF
        for (B, F, Tp, Ns, G) in [(5, 7, 4, 2, 2), (7, 10, 3, 9, 3), (3, 4, 2, 0, 1)]:
            mag, y = torch.rand(B, F, Tp, generator=g, dtype=D), torch.rand(B, F, Tp, generator=g, dtype=D)
            X, U, m = fsn_sub_band(mag, y, Ns, G, cum)
            torch.testing.assert_close(X, U / (m + eps), rtol=1e-13, atol=0)
        for (B, M, Tp, Nn, Ne, S) in [(2, 6, 7, 1, 2, 3), (3, 5, 5, 4, 0, 3), (2, 4, 9, 0, 3, 2)]:
            mel, enc = torch.rand(B, M, Tp, generator=g, dtype=D), torch.rand(B, M, Tp, generator=g, dtype=D)
            X, U, m = fast_bottleneck(mel, enc, Nn, Ne, S, cum)
            torch.testing.assert_close(X, U / (m + eps), rtol=1e-13, atol=0)
            assert X.shape[0] == fast_shrunk(Tp, S)
    for sec in [(0, 6, 2, 1, 2, 3), (6, 12, 3, 11, 3, 0)]:
        noisy, y = torch.rand(2, 12, 5, generator=g, dtype=D), torch.rand(2, 12, 5, generator=g, dtype=D)
        X, U, m = imp_section(noisy, y, sec)
        torch.testing.assert_close(X, U / (m + EPS_F32), rtol=1e-13, atol=0)


@pytest.mark.parametrize("F,N", [(2, 1), (7, 0), (7, 3), (7, 6), (33, 15), (257, 15), (161, 256 // 2 - 1)])
def test_unfold_multiplicity_is_reflect_count(F, N):
    """Every row of the unfolded sub-band input counted through the oracle freq_unfold equals O.reflect_count and the
    library's reflect_count (the multiplicity the closed-form norm means use)."""
    if N >= F:
        pytest.skip("reflection needs N < F")
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    idx = torch.arange(F, dtype=D).reshape(1, 1, F, 1)
    u = O.freq_unfold(idx, N).reshape(-1).long()
    cnt = np.bincount(u.numpy(), minlength=F)
    np.testing.assert_array_equal(cnt, O.reflect_count(F, N))
    np.testing.assert_array_equal(cnt, [lib.fsn_debug_reflect_count(r, F, N) for r in range(F)])


@pytest.mark.parametrize("B,F,G", [(3, 7, 2), (5, 9, 3), (9, 10, 4), (8, 16, 7), (66, 33, 4)])
def test_sub_band_rows_follow_drop_band_index_map(B, F, G):
    """Row r of the reference sub-band input is the unit the drop_band index map and the library's row_to_unit give."""
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    clip = torch.arange(B, dtype=D).reshape(B, 1, 1).expand(B, F, 1)
    freq = torch.arange(F, dtype=D).reshape(1, F, 1).expand(B, F, 1)
    Xb = fsn_sub_band(clip.contiguous(), clip.contiguous(), 0, G, False)[1][0, :, 0]
    Xf = fsn_sub_band(freq.contiguous(), freq.contiguous(), 0, G, False)[1][0, :, 0]
    src_b, src_f = O.drop_band_index_map(B, F, G)
    Fsub = F // G
    np.testing.assert_array_equal(Xb.numpy().astype(int), np.repeat(src_b, Fsub))
    np.testing.assert_array_equal(Xf.numpy().astype(int), src_f.reshape(-1))
    b, f = C.c_int(), C.c_int()
    for r in range(B * Fsub):
        assert lib.fsn_debug_row_to_unit(B, F, G, r, C.byref(b), C.byref(f)) == 0
        assert (b.value, f.value) == (int(Xb[r]), int(Xf[r]))


def test_real_time_resampling_blocks():
    """The down-sampling averages frame 0 alone and then blocks of S frames (the last one partial); up-sampling maps
    frame t to shrunk step t // S, so with (Ts - 1) S >= Tp the last shrunk step feeds no frame."""
    x = torch.arange(11, dtype=D).reshape(1, 11)
    d = FO.real_time_downsampling(x, 3)
    np.testing.assert_array_equal(d.numpy(), [[0, 2, 5, 8, 10]])  # 1-3, 4-6, 7-9, 10
    assert d.shape[-1] == fast_shrunk(11, 3)
    up = FO.real_time_upsampling(torch.arange(5, dtype=D).reshape(1, 5), 3, 11)
    np.testing.assert_array_equal(up.numpy(), [[0, 0, 0, 1, 1, 1, 2, 2, 2, 3, 3]])


def _gradcheck(fn, z):
    assert torch.autograd.gradcheck(fn, (z,), eps=1e-6, atol=1e-8, rtol=1e-6)


@pytest.mark.parametrize("cum", [False, True])
@pytest.mark.parametrize("G,act", [(1, ACT_TANH), (3, ACT_NONE)])
def test_fsn_reference_is_the_gradient(cum, G, act):
    """The autograd reference agrees with finite differences (gradcheck) through norm and drop_band, and the returned
    kernel inputs are the forward's."""
    g = torch.Generator().manual_seed(1)
    B, F, Tp, Ns = 4, 5, 3, 2
    mag = torch.rand(B, F, Tp, generator=g, dtype=D) + 0.1
    z = (torch.rand(B, F, Tp, generator=g, dtype=D) + 0.2).requires_grad_(True)
    R = B * (F // G if G > 1 else F)
    dX = torch.randn(Tp, R, 2 * Ns + 2, generator=g, dtype=D)
    _gradcheck(lambda zz: (fsn_sub_band(mag, act_fn(act)(zz), Ns, G, cum)[0] * dX).sum(), z)
    dz, cond, X, y, scale = ref_fsn_norm_bwd(mag, z.detach(), dX, Ns, G, act, cum)
    assert np.all(cond >= np.abs(dz) * (1 - 1e-12))
    if not cum:
        mean = torch.cat([O.freq_unfold(mag[:, None], Ns).reshape(B, F, -1, Tp),
                          act_fn(act)(z.detach()).reshape(B, F, 1, Tp)], dim=2).mean(dim=(1, 2, 3))
        np.testing.assert_allclose(scale, 1 / (mean.numpy() + EPS_OFF), rtol=1e-13)
    else:
        assert scale.shape == (Tp, R)


@pytest.mark.parametrize("cum", [False, True])
def test_fast_reference_is_the_gradient(cum):
    g = torch.Generator().manual_seed(2)
    B, M, Tp, Nn, Ne, S = 2, 5, 7, 1, 2, 3
    Ts = fast_shrunk(Tp, S)
    mel = torch.rand(B, M, Tp, generator=g, dtype=D)
    z = (torch.rand(B, M, Tp, generator=g, dtype=D) + 0.1).requires_grad_(True)
    zb = (torch.randn(B, M, Ts, generator=g, dtype=D)).requires_grad_(True)
    ddec = torch.randn(Tp, B, 2 * M, generator=g, dtype=D)
    dX = torch.randn(Ts, B * M, 2 * Nn + 2 * Ne + 2, generator=g, dtype=D)
    _gradcheck(lambda zz: (fast_bottleneck(mel, torch.relu(zz), Nn, Ne, S, cum)[0] * dX).sum()
               + (ddec[:, :, :M] * torch.relu(zz).permute(2, 0, 1)).sum(), z)
    _gradcheck(lambda zz: (ddec[:, :, M:] * FO.real_time_upsampling(torch.relu(zz)[:, None], S, Tp)[:, 0]
                           .permute(2, 0, 1)).sum(), zb)
    out = ref_fast_bwd(mel, z.detach(), zb.detach(), ddec, dX, Nn, Ne, S, cum)
    assert out[0].shape == (Tp, B, M) and out[2].shape == (Ts, B * M)


def test_imp_reference_is_the_gradient():
    g = torch.Generator().manual_seed(3)
    B, Fu, T = 2, 12, 4
    secs = [(0, 4, 2, 1, 2, 3), (4, 12, 4, 2, 4, 11)]
    noisy = torch.rand(B, Fu, T, generator=g, dtype=D)
    z = torch.randn(B, Fu, T, generator=g, dtype=D).requires_grad_(True)
    dXs = []
    for lo, hi, cs, ns, cf, nf in secs:
        dXs.append(torch.randn(T, B * (hi - lo) // cs, cs + 2 * ns + cf + 2 * nf, generator=g, dtype=D))
    _gradcheck(lambda zz: sum((imp_section(noisy, torch.tanh(zz), s)[0] * d).sum() for s, d in zip(secs, dXs)), z)
    dz, cond, y, per = ref_imp_bwd(noisy, z.detach(), dXs, secs, ACT_RELU)
    assert np.all(cond >= np.abs(dz) * (1 - 1e-12)) and len(per) == 2


# ------------------------------------------------------------------ refusals without a GPU
P = 1 << 20  # stand-in device pointer: every call below returns before it could be used


def test_norm_unfold_bwd_hooks_refuse_before_any_cuda_call():
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    SH, UN = _lib.FSN_ERR_SHAPE, _lib.FSN_ERR_UNSUPPORTED

    def expect(rc, code, text=None):
        assert rc == code, (rc, lib.fsn_last_error())
        assert lib.fsn_last_error_code() == code
        if text:
            assert text in lib.fsn_last_error(), lib.fsn_last_error()

    def fsn(dX=P, mid=P, B=4, F=9, G=2, Tp=3, Ns=2, cnt2=1.0, act=0, cum=0):
        return lib.fsn_debug_norm_unfold_bwd(dX, P, P, P, cum, B, F, G, Tp, Ns, cnt2, act, mid, P, None)

    expect(fsn(dX=None), SH, b"null")
    expect(fsn(mid=None), SH, b"null")
    expect(fsn(B=0), SH)
    expect(fsn(Tp=0), SH)
    expect(fsn(G=4), SH, b"B > G")   # drop_band needs more clips than groups
    expect(fsn(F=1, G=2), SH)
    expect(fsn(Ns=9), SH, b"Ns < F")   # N >= F
    expect(fsn(Ns=-1), SH)
    expect(fsn(act=4), SH, b"act")
    expect(fsn(cnt2=0.0), SH, b"cnt2")
    expect(fsn(B=40000, F=257, G=1, Tp=400, Ns=15), SH, b"2^31")

    def fast(ddec=P, bn_out=P, denc=P, dbn=P, dX=P, B=2, Tp=7, M=5, Nn=1, Ne=2, S=3, cnt2=1.0, cum=0):
        return lib.fsn_debug_fast_norm_unfold_bwd(ddec, dX, P, P, bn_out, P, cum, B, Tp, M, Nn, Ne, S, cnt2, P, denc,
                                                  dbn, None)

    expect(fast(ddec=None), SH, b"null")
    expect(fast(bn_out=None), SH, b"null")
    expect(fast(dX=None), SH, b"null")
    expect(fast(S=0), SH)
    expect(fast(M=0), SH)
    expect(fast(Nn=5), SH, b"< M")      # M - 1 is the largest reflection
    expect(fast(Ne=5), SH, b"< M")
    expect(fast(cnt2=0.0), SH, b"cnt2")

    def imp(dX=P, y=P, B=2, T=4, Fu=12, lo=4, hi=12, cs=4, ns=2, cf=4, nf=3, act=1):
        return lib.fsn_debug_imp_unfold_bwd(dX, P, P, y, B, T, Fu, lo, hi, cs, ns, cf, nf, 1, act, P, P, None)

    expect(imp(dX=None), SH, b"null")
    expect(imp(y=None), SH, b"null")      # ReLU' needs the kept output
    expect(imp(act=2), UN, b"ReLU")
    expect(imp(hi=13), SH)               # beyond Fu
    expect(imp(hi=11), SH, b"divisible")  # (hi - lo) % cs != 0
    expect(imp(cf=2), UN, b"match")       # SecGeom: sub-band and full-band centre widths must match
    expect(imp(ns=12), SH, b"neighbours")  # ns >= Fu
    expect(imp(nf=12), SH, b"neighbours")
    expect(imp(lo=-1), SH)
    expect(imp(lo=12), SH)                # empty section
    expect(imp(Fu=1, lo=0, hi=1, cs=1, cf=1, ns=0, nf=0), SH)

    def sec_in(magc=P, X=P, B=2, T=4, Fu=12, lo=4, hi=12, cs=4, ns=2, cf=4, nf=3):
        return lib.fsn_debug_imp_section_input(magc, P, B, T, Fu, lo, hi, cs, ns, cf, nf, 0, X, P, None)

    expect(sec_in(magc=None), SH, b"null")
    expect(sec_in(X=None), SH, b"null")
    expect(sec_in(T=0), SH)
    expect(sec_in(hi=10), SH, b"divisible")
    expect(sec_in(cf=2), UN, b"match")
    expect(sec_in(nf=12), SH, b"neighbours")

    def stats(x=P, fs=P, B=2, T_pad=5, F=9, N=2, lengths=None, lens=P, hop=4, la=0, inv1=None, cnt1=1.0):
        h = None if lengths is None else (C.c_int32 * len(lengths))(*lengths)
        return lib.fsn_debug_norm_stats(x, B, T_pad, F, N, T_pad * F, F, h, lens, hop, la, None, cnt1, 1.0, 1e-5, fs, P,
                                        inv1, None, None)

    expect(stats(x=None), SH, b"null")
    expect(stats(fs=None), SH, b"null")
    expect(stats(B=0), SH)
    expect(stats(N=9), SH, b"N < F")
    expect(stats(inv1=P, cnt1=0.0), SH, b"cnt1")
    expect(stats(lengths=[16, 12], lens=None), SH, b"lens_dev")
    expect(stats(lengths=[16, 12], hop=0), SH, b"hop")
    expect(stats(lengths=[16, 20]), SH, b"clip 1")  # 1 + 20/4 = 6 frames > T_pad
    expect(stats(lengths=[16, 12], la=1), SH, b"clip 0")  # 1 + 16/4 + 1 = 6
    expect(stats(lengths=[16, -1]), SH, b"clip 1")
    expect(lib.fsn_debug_train_stats(None, 0, 2, 9, 5, 2, P, None), SH, b"null")
    expect(lib.fsn_debug_train_stats(P, 1, 2, 9, 5, 9, P, None), SH, b"N < F")
    expect(lib.fsn_debug_train_stats(P, 1, 2, 9, 0, 2, P, None), SH)
