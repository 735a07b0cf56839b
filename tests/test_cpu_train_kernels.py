"""The float64 references of the kernels around the training step, each pinned to an authority on the CPU, and the
CPU-only argument checks of fsn_clip_adam_steps.  The references are shared with tests/test_gpu_train_kernels.py:

- clip + Adam (fsn_clip_adam, fsn_clip_adam_steps): clip_grad_norm_ then the single-tensor torch.optim.Adam formula, one
  step count per tensor; pinned to clip_grad_norm_ + torch.optim.Adam(foreach=False) in float64;
- the cIRM, compress and decompress (audio_zen/acoustics/mask.py:22-40, 58-63), pinned to tests/golden/dsp.npz;
- drop_band (audio_zen/acoustics/feature.py:309-345) as an index map, pinned to the same golden;
- the MSE loss and its gradient, pinned to torch.nn.functional.mse_loss and autograd;
- SI-SDR (audio_zen/metrics.py:6-31), pinned to its closed form on an orthogonal split;
- the RIR convolution as the plain float64 loop with k ascending (the bit-exact reference of rir_conv_kernel), pinned to
  np.convolve / scipy.signal.fftconvolve;
- snr_mix (feature.py:99-114, dataset_train.py:136-199) in float64, pinned to oracle/mix_oracle.py and to the items of
  tests/golden/dataset_train.npz."""
import ctypes as C

import numpy as np
import pytest
import scipy.signal
import torch

from test_cpu_dsp import ref_decompress  # noqa: F401  (re-exported for the GPU tests)

EPS_CIRM = float(np.float32(1.1920928955078125e-07))  # audio_zen/constant.py:9


# ------------------------------------------------------------------ clip + Adam
def ref_clip_adam(params, grads, exp_avgs, exp_avg_sqs, steps, max_norm, grad_scale, lr, b1, b2, eps):
    """clip_grad_norm_(max_norm) over the gradients times grad_scale, then one torch.optim.Adam step (no weight decay,
    no amsgrad) per tensor at its own step, all in float64.  A tensor whose grad is None is skipped.  max_norm <= 0 turns
    the clip off.  Returns (norm, coef, grads, exp_avgs, exp_avg_sqs, params): coef is the factor applied to the raw
    gradients (grad_scale times the clip coefficient), lists hold None where the grad was None."""
    f64 = [None if g is None else np.asarray(g, np.float64) * grad_scale for g in grads]
    with np.errstate(invalid="ignore", over="ignore"):
        norm = float(np.sqrt(sum(float((g * g).sum()) for g in f64 if g is not None)))
        clip = float(np.minimum(1.0, max_norm / (norm + 1e-6))) if max_norm > 0 else 1.0  # NaN propagates like clamp
    out_g, out_m, out_v, out_p = [], [], [], []
    for p, g, m, v, s in zip(params, f64, exp_avgs, exp_avg_sqs, steps):
        if g is None:
            out_g.append(None), out_m.append(None), out_v.append(None), out_p.append(None)
            continue
        with np.errstate(invalid="ignore", over="ignore"):
            g = g * clip
            m = np.asarray(m, np.float64) * b1 + (1 - b1) * g
            v = np.asarray(v, np.float64) * b2 + (1 - b2) * g * g
            bc1, bc2 = 1 - b1 ** s, 1 - b2 ** s
            p = np.asarray(p, np.float64) - lr / bc1 * (m / (np.sqrt(v) / np.sqrt(bc2) + eps))
        out_g.append(g), out_m.append(m), out_v.append(v), out_p.append(p)
    return norm, clip * grad_scale, out_g, out_m, out_v, out_p


def torch_clip_adam_run(params, grad_seq, max_norm, grad_scale, lr, b1, b2, eps, dtype=torch.float64, device="cpu",
                        opt_state=None):
    """clip_grad_norm_ + torch.optim.Adam(foreach=False) over the gradient lists of grad_seq (None = no grad that step);
    returns the parameters after every step, the clipped gradients of every step and the optimiser."""
    ps = [torch.nn.Parameter(torch.as_tensor(p, dtype=dtype, device=device).clone()) for p in params]
    opt = torch.optim.Adam(ps, lr=lr, betas=(b1, b2), eps=eps, foreach=False)
    if opt_state is not None:
        opt.load_state_dict(opt_state)
    traj, clipped = [], []
    for grads in grad_seq:
        for p, g in zip(ps, grads):
            p.grad = None if g is None else torch.as_tensor(g, dtype=dtype, device=device) * grad_scale
        live = [p for p in ps if p.grad is not None]
        if max_norm > 0:
            torch.nn.utils.clip_grad_norm_(live, max_norm)
        clipped.append([None if p.grad is None else p.grad.detach().cpu().numpy().copy() for p in ps])
        opt.step()
        traj.append([p.detach().cpu().numpy().copy() for p in ps])
    return traj, clipped, opt


def _adam_case(rng, sizes):
    params = [rng.standard_normal(n) for n in sizes]
    return params, [np.zeros(n) for n in sizes], [np.zeros(n) for n in sizes]


@pytest.mark.parametrize("max_norm,grad_scale", [(0.0, 1.0), (0.5, 1.0), (1e3, 0.25), (0.7, 1 / 3)])
def test_reference_clip_adam_matches_torch(max_norm, grad_scale):
    """Six steps over three tensors; tensor 1 has no grad in the first step, so from then on it is one step behind."""
    rng = np.random.default_rng(int(max_norm * 10) + 7)
    sizes = [17, 300, 5]
    lr, b1, b2, eps = 1e-3, 0.8, 0.99, 1e-6
    params, ms, vs = _adam_case(rng, sizes)
    seq = [[rng.standard_normal(n) * (3.0 if k == 0 else 1.0) for k, n in enumerate(sizes)] for _ in range(6)]
    seq[0][1] = None
    traj, clipped, _ = torch_clip_adam_run(params, seq, max_norm, grad_scale, lr, b1, b2, eps)
    steps = [0] * len(sizes)
    p = params
    for it, grads in enumerate(seq):
        steps = [s + (g is not None) for s, g in zip(steps, grads)]
        norm, coef, g, m, v, pn = ref_clip_adam(p, grads, ms, vs, steps, max_norm, grad_scale, lr, b1, b2, eps)
        for k in range(len(sizes)):
            if grads[k] is None:
                assert clipped[it][k] is None and np.array_equal(traj[it][k], p[k])
                continue
            assert np.abs(g[k] - clipped[it][k]).max() <= 1e-13 * np.abs(g[k]).max()
            assert np.abs(pn[k] - traj[it][k]).max() <= 1e-13
            ms[k], vs[k] = m[k], v[k]
        p = [pn[k] if pn[k] is not None else p[k] for k in range(len(sizes))]
        if max_norm > 0:
            assert abs(coef / grad_scale - min(1.0, max_norm / (norm + 1e-6))) < 1e-15
    assert steps == [6, 5, 6]


def test_reference_clip_adam_nonfinite_pattern_matches_torch():
    """A NaN or an inf gradient: the clip coefficient is NaN / 0, and the NaN / zero pattern follows torch."""
    rng = np.random.default_rng(3)
    for bad in (np.nan, np.inf):
        for max_norm in (0.0, 1.0):
            params, ms, vs = _adam_case(rng, [40, 9])
            grads = [rng.standard_normal(40), rng.standard_normal(9)]
            grads[0][7] = bad
            traj, clipped, _ = torch_clip_adam_run(params, [grads], max_norm, 1.0, 1e-3, 0.9, 0.999, 1e-8)
            _, _, g, _, _, p = ref_clip_adam(params, grads, ms, vs, [1, 1], max_norm, 1.0, 1e-3, 0.9, 0.999, 1e-8)
            for k in range(2):
                assert np.array_equal(np.isnan(g[k]), np.isnan(clipped[0][k]))
                assert np.array_equal(g[k] == 0, clipped[0][k] == 0)
                assert np.array_equal(np.isnan(p[k]), np.isnan(traj[0][k]))
                ok = ~np.isnan(p[k])
                assert np.abs(p[k][ok] - traj[0][k][ok]).max(initial=0) <= 1e-13


# ------------------------------------------------------------------ cIRM, compress, decompress
def ref_compress(m, K=10.0, C=0.1):
    """compress_cIRM (mask.py:38-40): m clamped below at -100, then K (1 - e^{-C m}) / (1 + e^{-C m})."""
    m = np.asarray(m, np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        m = np.where(m <= -100, -100.0, m)
        e = np.exp(-C * m)
        return K * (1 - e) / (1 + e)


def ref_cirm_ratio(nr, ni, cr, ci):
    """the uncompressed cIRM (mask.py:22-25) in float64 from the float32 spectra: (real, imag)"""
    a, b, c, d = (np.asarray(x, np.float64) for x in (nr, ni, cr, ci))
    den = a * a + b * b + EPS_CIRM
    return (a * c + b * d) / den, (a * d - b * c) / den


def ref_build_cirm(nr, ni, cr, ci):
    """build_complex_ideal_ratio_mask: [..., 2] (real, imag) of the compressed cIRM (K = 10, C = 0.1)"""
    re, im = ref_cirm_ratio(nr, ni, cr, ci)
    return np.stack([ref_compress(re), ref_compress(im)], -1)


def test_reference_masks_match_golden(golden):
    g = golden("dsp")
    assert np.abs(ref_compress(g["big"]) - g["comp"]).max() < 2e-6 * np.abs(g["comp"]).max()
    edge = ref_compress(np.array([-1e30, -100.0, -99.0, 0.0, 1e30, np.inf, -np.inf, np.nan]))
    sat = 10 * (1 - np.exp(10.0)) / (1 + np.exp(10.0))
    assert np.allclose(edge[:2], sat, rtol=1e-15, atol=0) and edge[2] > sat and edge[3] == 0 and edge[4] == edge[5] == 10
    assert edge[6] == sat and np.isnan(edge[7])
    # the cIRM from the golden's noisy spectrum and the float32 torch STFT of its clean signal (the reference's STFT)
    w = torch.hann_window(512)
    X = torch.stft(torch.from_numpy(g["yc"]), 512, 256, 512, window=w, center=True, pad_mode="reflect",
                   return_complex=True)
    cr, ci = X.real.numpy(), X.imag.numpy()
    got = ref_build_cirm(g["real"], g["imag"], cr, ci)
    assert got.shape == g["cirm"].shape
    # float32 rounding of the golden, amplified by the ratio's conditioning: (|a c| + |b d|) / (|noisy|^2 + eps)
    a, b = np.abs(g["real"]).astype(np.float64), np.abs(g["imag"]).astype(np.float64)
    den = a * a + b * b + EPS_CIRM
    kr = (a * np.abs(cr) + b * np.abs(ci)) / den
    ki = (a * np.abs(ci) + b * np.abs(cr)) / den
    err = np.abs(got - g["cirm"]) / (1.0 + np.stack([kr, ki], -1))
    assert err.max() < 1e-5
    well = np.stack([den, den], -1) > 1e-2
    assert well.mean() > 0.5 and np.abs(got - g["cirm"])[well].max() < 1e-5


# ------------------------------------------------------------------ drop_band
def ref_drop_band(x, G):
    """feature.py:309-345 as an index map: F truncated to a multiple of G, output group g = clips g, g+G, ... at bins
    g, g+G, ... (groups concatenated along the batch)"""
    x = np.asarray(x)
    F2 = x.shape[2] - x.shape[2] % G
    return np.concatenate([x[g::G, :, g:F2:G, :] for g in range(G)], 0)


def test_reference_drop_band_matches_golden(golden):
    g = golden("dsp")
    assert np.array_equal(ref_drop_band(g["xb"], 2), g["db2"])
    assert np.array_equal(ref_drop_band(g["xb"], 3), g["db3"])


# ------------------------------------------------------------------ MSE
def ref_mse(cirm, crm):
    """loss = mean((cirm - crm)^2) with cirm [B,F,T,2], crm [B,2,F,T]; dcrm = 2 (crm - cirm) / n in crm's layout"""
    c = np.asarray(cirm, np.float64).transpose(0, 3, 1, 2)
    r = np.asarray(crm, np.float64)
    d = r - c
    return float((d * d).mean()), 2.0 * d / d.size


@pytest.mark.parametrize("B,F,T", [(1, 1, 1), (3, 17, 29), (2, 1, 300), (1, 257, 1)])
def test_reference_mse_matches_torch(B, F, T):
    rng = np.random.default_rng(B * F * T)
    cirm = rng.uniform(-10, 10, (B, F, T, 2))
    crm = torch.from_numpy(rng.uniform(-10, 10, (B, 2, F, T))).requires_grad_()
    want = torch.nn.functional.mse_loss(torch.from_numpy(cirm), crm.permute(0, 2, 3, 1))
    want.backward()
    loss, d = ref_mse(cirm, crm.detach().numpy())
    assert abs(loss - float(want.detach())) <= 1e-14 * float(want.detach())
    assert np.abs(d - crm.grad.numpy()).max() <= 1e-15 * np.abs(d).max()


# ------------------------------------------------------------------ SI-SDR
def ref_si_sdr(reference, estimation):
    """audio_zen/metrics.py:6-31 in float64 over the last axis"""
    r = np.asarray(reference, np.float64)
    e = np.asarray(estimation, np.float64)
    alpha = (r * e).sum(-1, keepdims=True) / (r * r).sum(-1, keepdims=True)
    p = alpha * r
    n = e - p
    with np.errstate(divide="ignore"):
        return 10 * np.log10((p * p).sum(-1) / (n * n).sum(-1))


def test_reference_si_sdr_closed_form():
    """est = s ref + n with n orthogonal to ref: SI-SDR = 10 log10(|s ref|^2 / |n|^2); scale-invariant; est = ref: +inf"""
    rng = np.random.default_rng(0)
    r = rng.standard_normal((4, 3001))
    n = rng.standard_normal((4, 3001))
    n -= ((n * r).sum(-1, keepdims=True) / (r * r).sum(-1, keepdims=True)) * r
    for s in (0.3, 1.0, 7.0):
        n_s = n * np.array([[0.01], [0.1], [1.0], [10.0]])
        want = 10 * np.log10((s * s * (r * r).sum(-1)) / (n_s * n_s).sum(-1))
        assert np.abs(ref_si_sdr(r, s * r + n_s) - want).max() < 1e-9
        assert np.abs(ref_si_sdr(r, 5.0 * (s * r + n_s)) - want).max() < 1e-9
    assert np.all(ref_si_sdr(r, r) == np.inf)


# ------------------------------------------------------------------ RIR convolution
def ref_rir_convolve(x, rir, lr):
    """the first len(x) samples of x * rir[:lr]: each output summed k ascending in one float64 accumulator (float32
    inputs, so every product is exact), rounded to float32 once; lr = 0 copies x.  Returns (float32, float64 sums)."""
    x = np.asarray(x, np.float32)
    if lr <= 0:
        return x.copy(), x.astype(np.float64)
    xd = x.astype(np.float64)
    h = np.asarray(rir, np.float32).astype(np.float64)
    L = len(x)
    acc = np.zeros(L)
    for k in range(min(lr, L)):
        acc[k:] += h[k] * xd[:L - k]
    return acc.astype(np.float32), acc


@pytest.mark.parametrize("L,lr", [(1, 1), (5, 9), (1151, 1152), (1153, 1153), (3000, 2309), (700, 2309), (2000, 1)])
def test_reference_rir_convolve_matches_numpy(L, lr):
    rng = np.random.default_rng(L + lr)
    x = rng.standard_normal(L).astype(np.float32)
    h = (rng.standard_normal(lr) * np.exp(-np.arange(lr) / 300)).astype(np.float32)
    _, acc = ref_rir_convolve(x, h, lr)
    full = np.convolve(x.astype(np.float64), h.astype(np.float64))[:L]
    fft = scipy.signal.fftconvolve(x.astype(np.float64), h.astype(np.float64))[:L]
    scale = np.abs(x).max() * np.abs(h).sum()
    assert np.abs(acc - full).max() <= 1e-12 * scale
    assert np.abs(acc - fft).max() <= 1e-12 * scale
    assert np.array_equal(ref_rir_convolve(x, h, 0)[0], x)


# ------------------------------------------------------------------ snr_mix
def ref_snr_mix(clean, noise, snr, target_dB_FS, noisy_target_dB_FS, eps=1e-6):
    """Dataset.snr_mix (dataset_train.py:167-195, feature.py:99-114) in float64 after the reverberation; returns
    (noisy, clean, max|noisy| before the anti-clipping rescale)"""
    def rms(y):
        return np.sqrt(np.mean(y * y))

    def norm_tailor(y):
        y = y / (np.abs(y).max() + eps)
        return y * (10 ** (target_dB_FS / 20) / (rms(y) + eps))

    c = norm_tailor(np.asarray(clean, np.float64))
    n = norm_tailor(np.asarray(noise, np.float64))
    n = n * (rms(c) / 10 ** (snr / 20) / (rms(n) + eps))
    y = c + n
    k = 10 ** (noisy_target_dB_FS / 20) / (rms(y) + eps)
    y, c = y * k, c * k
    peak = float(np.abs(y).max())
    if peak > 0.999:
        s = peak / (0.99 - eps)
        y, c = y / s, c / s
    return y, c, peak


def test_reference_snr_mix_matches_oracle_and_golden(golden):
    """Within float32 rounding of the numpy pipelines (2e-5 of the row's peak, the bound of tests/golden/mix.npz)."""
    from conftest import rel_max
    from oracle import mix_oracle
    g = golden("dataset_train")
    clipped = 0
    for i in range(g["clean"].shape[0]):
        x = g["clean"][i]
        lr = int(g["rir_len"][i])
        if lr:
            x = ref_rir_convolve(x, g["rir"][i], lr)[1]
        y, c, peak = ref_snr_mix(x, g["noise"][i], float(g["snr"][i]), -25.0, float(g["noisy_target_dB_FS"][i]))
        clipped += peak > 0.999
        assert rel_max(y, g["noisy"][i]) < 2e-5 and rel_max(c, g["clean_out"][i]) < 2e-5, i
    assert clipped >= 1
    rng = np.random.default_rng(1)
    for snr, nt, spiky in ((-5.0, -25.0, False), (20.0, -12.0, True), (0.0, -35.0, False)):
        clean = (0.1 * rng.standard_normal(4000)).astype(np.float32)
        if spiky:
            clean[::501] = 0.9
        noise = (0.3 * rng.standard_normal(4000)).astype(np.float32)
        want = mix_oracle.snr_mix(clean, noise, snr, -25, nt)
        y, c, _ = ref_snr_mix(clean, noise, snr, -25, nt)
        assert rel_max(y, want[0]) < 2e-5 and rel_max(c, want[1]) < 2e-5


# ------------------------------------------------------------------ fsn_clip_adam_steps refusals without a GPU
P = 1 << 20  # stand-in device pointer: every call below returns before it could be used


def test_clip_adam_steps_refuses_before_any_cuda_call():
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    SH, WS = _lib.FSN_ERR_SHAPE, _lib.FSN_ERR_WORKSPACE

    def call(n=3, steps=(1, 2, 3), scratch=P, nbytes=None, L=True):
        pl = _lib.ParamList()
        pl.n = n
        for i in range(min(max(n, 0), _lib.MAX_PARAM_TENSORS)):
            pl.param[i] = pl.grad[i] = pl.exp_avg[i] = pl.exp_avg_sq[i] = P
            pl.numel[i] = 10
        st = None if steps is None else (C.c_int * max(len(steps), 1))(*steps)
        nb = lib.fsn_clip_adam_scratch_bytes() if nbytes is None else nbytes
        return lib.fsn_clip_adam_steps(C.byref(pl) if L else None, 10.0, 1.0, 1e-3, 0.9, 0.999, 1e-8, st, P, scratch, nb,
                                       None)

    def expect(rc, code, text=None):
        assert rc == code, (rc, lib.fsn_last_error())
        assert lib.fsn_last_error_code() == code
        if text:
            assert text in lib.fsn_last_error(), lib.fsn_last_error()

    expect(call(L=False), SH)
    expect(call(n=0, steps=()), SH)
    expect(call(n=_lib.MAX_PARAM_TENSORS + 1, steps=[1] * 65), SH, b"64")
    expect(call(steps=None), SH, b"step")
    expect(call(steps=(1, 0, 3)), SH, b"tensor 1")
    expect(call(steps=(1, 2, -4)), SH, b"tensor 2")
    expect(call(scratch=None), WS)
    expect(call(nbytes=lib.fsn_clip_adam_scratch_bytes() - 1), WS)
    # only the first n entries are read: valid arguments reach the scratch check, the last one before the first launch
    expect(call(n=2, steps=(5, 1, 0), scratch=None), WS)
    expect(call(n=_lib.MAX_PARAM_TENSORS, steps=list(range(1, 65)), scratch=None), WS)
    # fsn_clip_adam checks its single step, then runs the same launcher
    pl = _lib.ParamList()
    pl.n = 1
    assert lib.fsn_clip_adam(C.byref(pl), 10.0, 1.0, 1e-3, 0.9, 0.999, 1e-8, 0, P, P, 1 << 20, None) == SH
    assert lib.fsn_clip_adam(C.byref(pl), 10.0, 1.0, 1e-3, 0.9, 0.999, 1e-8, 1, P, None, 0, None) == WS


def test_fused_clip_adam_refuses_host_parameters():
    from fullsubnet_b200.optim import FusedClipAdam
    p = torch.nn.Parameter(torch.zeros(3))
    p.grad = torch.ones(3)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        FusedClipAdam([p], lr=1e-3, max_norm=1.0).step()
