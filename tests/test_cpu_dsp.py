"""The signal layer's float64 reference, pinned to torch.stft / torch.istft, and the CPU-only checks of its unit-test hooks
(fsn_debug_stft, fsn_debug_istft, fsn_debug_istft_mask_adjoint, fsn_debug_wav_epilogue in fsn_dsp.cu): every bad
argument and every shape the kernels cannot run is refused with its error class before any CUDA call (stand-in device
pointers, never dereferenced).  The reference functions are shared with tests/test_gpu_dsp.py."""
import ctypes as C

import numpy as np
import pytest
import torch

LIMIT = float(np.float32(9.9))  # decompress_cIRM's clip, compared in float32 like the kernels


# ------------------------------------------------------------------ float64 reference, straight from the definitions
def ref_window(n, W):
    """torch.hann_window(W) (periodic; [1] for W = 1) centred in n samples, left = (n - W) // 2."""
    w = np.zeros(n)
    h = np.ones(1) if W == 1 else 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(W) / W)
    left = (n - W) // 2
    w[left:left + W] = h
    return w


def ref_stft(x, n, hop, W):
    """x [L] -> X [n/2+1, 1 + L//hop]: reflect padding by n/2, windowed frames every hop samples, rfft."""
    x = np.asarray(x, np.float64)
    L = x.shape[0]
    T = 1 + L // hop
    idx = np.abs(np.arange(T)[:, None] * hop + np.arange(n)[None, :] - n // 2)
    idx = np.where(idx >= L, 2 * (L - 1) - idx, idx)
    return np.fft.rfft(x[idx] * ref_window(n, W), axis=1).T


def ref_istft(X, n, hop, W, length=None):
    """X [n/2+1, T] complex -> (y, env): irfft of every frame (Im of DC and Nyquist ignored), windowed overlap-add over
    the window-square envelope env (0 where env <= 1e-11), the n/2 centre padding cropped, then cut or zero-padded to
    length (default hop*(T-1)).  env is returned on the same samples."""
    X = np.array(X, np.complex128)
    X[0].imag = 0
    X[-1].imag = 0
    T = X.shape[1]
    w = ref_window(n, W)
    frames = np.fft.irfft(X.T, n=n, axis=1) * w
    full = n + hop * (T - 1)
    idx = (np.arange(T)[:, None] * hop + np.arange(n)[None, :]).ravel()
    acc = np.bincount(idx, frames.ravel(), minlength=full)
    env = np.bincount(idx, np.tile(w * w, T), minlength=full)
    y = np.where(env > 1e-11, acc / np.where(env > 1e-11, env, 1.0), 0.0)
    out_len = length if length else hop * (T - 1)
    out, oenv = np.zeros(out_len), np.zeros(out_len)
    m = min(out_len, full - n // 2)
    out[:m], oenv[:m] = y[n // 2:n // 2 + m], env[n // 2:n // 2 + m]
    return out, oenv


def ref_decompress(m, K=10.0):
    """decompress_cIRM: clip to +-9.9 (NaN -> 0), then -K log((K - m) / (K + m))."""
    m = np.asarray(m, np.float64)
    with np.errstate(invalid="ignore"):
        c = np.where(np.abs(m) < LIMIT, m, np.where(m >= LIMIT, LIMIT, np.where(m <= -LIMIT, -LIMIT, 0.0)))
    return -K * np.log((K - c) / (K + c))


def ref_mask(X, crm, mode):
    """X [..., F, T] complex, crm [..., 2, F, T] -> the masked spectrum: mode 1 the complex product with the decompressed
    cIRM, mode 2 Re * crm0 + i Im * crm1, mode 0 X itself."""
    if mode == 0:
        return X
    crm = np.asarray(crm, np.float64)
    if mode == 1:
        return (ref_decompress(crm[..., 0, :, :]) + 1j * ref_decompress(crm[..., 1, :, :])) * X
    return X.real * crm[..., 0, :, :] + 1j * X.imag * crm[..., 1, :, :]


def ref_mask_adjoint(g, X, n, hop, W, L):
    """d <istft(X (.) M, length=L), g> / d M of mask mode 2, in closed form: the per-sample gradient over the envelope,
    windowed into frames, rfft, irfft's adjoint c_k / n (c = 1 at DC, 2 inside; Im of DC gets none), times the spectrum.
    Returns [2, n/2+1, T]; the Nyquist row, a constant of the model, is left 0."""
    T = X.shape[1]
    F = n // 2 + 1
    w = ref_window(n, W)
    full = n + hop * (T - 1)
    idx = np.arange(T)[:, None] * hop + np.arange(n)[None, :]
    env = np.bincount(idx.ravel(), np.tile(w * w, T), minlength=full)
    s = np.arange(full)
    ok = (s >= n // 2) & (s < n // 2 + L) & (env > 1e-11)
    G = np.zeros(full)
    G[ok] = np.asarray(g, np.float64)[s[ok] - n // 2] / env[ok]
    H = np.fft.rfft(G[idx] * w, axis=1).T
    c = np.full((F, 1), 2.0 / n)
    c[0] = 1.0 / n
    d = np.zeros((2, F, T))
    d[0, :F - 1] = (c * H.real * X.real)[:F - 1]
    d[1, 1:F - 1] = (c * H.imag * X.imag)[1:F - 1]
    return d


# ------------------------------------------------------------------ the reference against torch (float64)
def _torch_window(W):
    return torch.hann_window(W, dtype=torch.float64)


@pytest.mark.parametrize("n,hop,W,L", [(16, 8, 16, 9), (16, 5, 15, 100), (64, 16, 32, 333), (64, 64, 1, 200),
                                       (96, 40, 95, 777), (256, 300, 128, 1999), (512, 128, 511, 4001),
                                       (960, 480, 960, 4800), (1200, 333, 600, 5000), (2048, 512, 1, 9000)])
def test_reference_stft_matches_torch(n, hop, W, L):
    x = np.random.default_rng(n + hop + W + L).standard_normal(L)
    got = ref_stft(x, n, hop, W)
    want = torch.stft(torch.from_numpy(x), n, hop, W, window=_torch_window(W), center=True, pad_mode="reflect",
                      return_complex=True).numpy()
    assert got.shape == want.shape
    assert np.abs(got - want).max() < 1e-12 * np.abs(want).max()


@pytest.mark.parametrize("n,hop,W,T,length", [(16, 8, 16, 9, None), (16, 4, 15, 40, 150), (64, 16, 32, 33, 500),
                                              (96, 24, 95, 17, 300), (120, 45, 120, 34, 1000), (512, 256, 511, 5, None),
                                              (512, 128, 256, 12, 900), (960, 480, 960, 10, 4000),
                                              (2048, 512, 2048, 9, 4096)])
def test_reference_istft_matches_torch(n, hop, W, T, length):
    rng = np.random.default_rng(n + hop + W + T)
    X = rng.standard_normal((n // 2 + 1, T)) + 1j * rng.standard_normal((n // 2 + 1, T))  # Im of DC / Nyquist != 0
    got, env = ref_istft(X, n, hop, W, length)
    Xt = X.copy()
    Xt[0].imag = 0
    Xt[-1].imag = 0
    want = torch.istft(torch.from_numpy(Xt), n, hop, W, window=_torch_window(W), center=True, length=length).numpy()
    assert got.shape == want.shape
    assert np.abs(got - want).max() < 1e-10 * np.abs(want).max()
    assert env.shape == got.shape


def test_reference_istft_writes_zero_where_torch_refuses():
    """win_length = hop = n/2: every n/2-th sample has a zero envelope.  torch.istft refuses; the reference (and the
    kernels) write exactly 0 there."""
    n, hop, W, T = 64, 32, 32, 9
    X = np.random.default_rng(0).standard_normal((n // 2 + 1, T)) + 0j
    with pytest.raises(RuntimeError):
        torch.istft(torch.from_numpy(X), n, hop, W, window=_torch_window(W), center=True)
    y, env = ref_istft(X, n, hop, W)
    zero = env == 0
    assert zero.sum() >= T - 2 and np.all(y[zero] == 0) and np.all(np.abs(y[~zero]) > 0)


@pytest.mark.parametrize("n,hop,W,T,L", [(16, 8, 16, 12, 90), (64, 16, 63, 20, 300), (96, 24, 48, 11, 200),
                                         (512, 128, 512, 10, 1100), (120, 60, 120, 9, 500)])
def test_reference_mask_adjoint_matches_torch_autograd(n, hop, W, T, L):
    rng = np.random.default_rng(n + T + L)
    F = n // 2 + 1
    X = rng.standard_normal((F, T)) + 1j * rng.standard_normal((F, T))
    M = torch.from_numpy(rng.standard_normal((2, F, T))).requires_grad_()
    g = rng.standard_normal(L)
    Xt = torch.from_numpy(X)
    Y = torch.complex(Xt.real * M[0], Xt.imag * M[1])
    y = torch.istft(Y, n, hop, W, window=_torch_window(W), center=True, length=L)
    (y * torch.from_numpy(g)).sum().backward()
    want = M.grad.numpy()
    got = ref_mask_adjoint(g, X, n, hop, W, L)
    assert np.abs(got[:, :F - 1] - want[:, :F - 1]).max() < 1e-10 * np.abs(want).max()
    assert np.all(want[1, 0] == 0)  # the imaginary part of DC gets no gradient


def test_reference_decompress_matches_golden(golden):
    g = golden("dsp")
    assert np.abs(ref_decompress(g["m"]) - g["dec"]).max() < 2e-6 * np.abs(g["dec"]).max()
    edge = np.array([np.nan, LIMIT, -LIMIT, 1e30, -np.inf, 0.0], np.float32)
    sat = -10 * np.log((10 - LIMIT) / (10 + LIMIT))
    assert np.array_equal(ref_decompress(edge), [0.0, sat, -sat, sat, -sat, 0.0])


# ------------------------------------------------------------------ hook refusals without a GPU
P = 1 << 20  # stand-in device pointer: every call below is refused before it could be used


@pytest.fixture(scope="module")
def lib():
    from fullsubnet_b200 import _lib
    return _lib.load()


def _lens(*v):
    return (C.c_int32 * len(v))(*v)


def _expect(lib, rc, code, text=None):
    assert rc == code, (rc, lib.fsn_last_error())
    assert lib.fsn_last_error_code() == code
    if text is not None:
        assert text in lib.fsn_last_error(), lib.fsn_last_error()


def test_stft_hook_refuses_without_gpu(lib):
    from fullsubnet_b200 import _lib
    SH, UN = _lib.FSN_ERR_SHAPE, _lib.FSN_ERR_UNSUPPORTED

    def call(wav=P, B=2, L=1000, n=64, hop=16, W=64, lengths=None, lens_dev=P, magT=None, T_pad=0):
        return lib.fsn_debug_stft(wav, B, L, n, hop, W, lengths, lens_dev, P, P, P, P, magT, T_pad, None)

    _expect(lib, call(B=65536), UN, b"65535")
    _expect(lib, call(B=70000, lengths=_lens(*([1000] * 70000))), UN, b"65535")
    for n in (8, 14, 17, 1202, 4096, 1536):
        _expect(lib, call(n=n, W=8), UN, b"unsupported")
    _expect(lib, call(B=0), SH)
    _expect(lib, call(hop=0), SH)
    _expect(lib, call(W=0), SH)
    _expect(lib, call(W=65), SH)
    _expect(lib, call(L=32), SH, b"reflect")
    _expect(lib, call(magT=P, T_pad=62), SH, b"T_pad")
    _expect(lib, call(wav=None), SH)
    _expect(lib, call(lengths=_lens(1000, 600), lens_dev=None), SH, b"length table")
    _expect(lib, call(lengths=_lens(1000, 32)), SH, b"clip 1")
    _expect(lib, call(lengths=_lens(999, 600)), SH, b"longest")
    _expect(lib, call(lengths=_lens(1001, 600)), SH)


def _smem_ok(n, hop):
    """shared-memory bytes of the iSTFT kernels' frame buffers <= the 227 KB opt-in of sm_90 (fsn_dsp*.cu layouts)"""
    is_pow2 = n & (n - 1) == 0
    np_max = (16 + -(-n // hop) + 2) // 2
    b = (np_max * (n + 1) * 8 + n // 2 * 8 + n * 4) if is_pow2 else (2 * np_max * n * 8 + n * 12)
    return b <= 227 * 1024


def test_istft_hook_refuses_without_gpu(lib):
    from fullsubnet_b200 import _lib
    SH, UN = _lib.FSN_ERR_SHAPE, _lib.FSN_ERR_UNSUPPORTED

    def call(real=P, imag=P, cstride=1, crm=None, mode=0, B=2, T=20, n=64, hop=16, W=64, length=0, lengths=None,
             lens_dev=P, wav=P, peak=P, pcm=None, crm_out=None):
        return lib.fsn_debug_istft(real, imag, cstride, crm, mode, B, T, n, hop, W, length, lengths, lens_dev, wav, peak,
                                   pcm, 26213.6, crm_out, None)

    # over-budget shared memory: refused before the peak memset, on both paths
    for n, hop in ((2048, 227), (1024, 27), (512, 5), (256, 1), (1200, 239), (960, 87)):
        assert not _smem_ok(n, hop) and _smem_ok(n, hop + 1)
        _expect(lib, call(n=n, W=n, hop=hop, T=40), UN, b"shared memory")
    _expect(lib, call(B=65536), UN, b"65535")
    for n in (8, 14, 17, 1202, 4096):
        _expect(lib, call(n=n, W=8, hop=4), UN, b"unsupported")
    _expect(lib, call(lengths=_lens(300, 200), length=0), UN, b"output length")
    _expect(lib, call(B=0), SH)
    _expect(lib, call(T=0), SH)
    _expect(lib, call(hop=65), SH)
    _expect(lib, call(W=65), SH)
    _expect(lib, call(cstride=3), SH, b"cstride")
    _expect(lib, call(T=1), SH, b"output length")
    _expect(lib, call(lengths=_lens(320, 200), length=320, T=20), SH, b"frames")  # 320 / 16 = 20 needs 21 frames
    _expect(lib, call(mode=3, crm=P), SH, b"mask mode")
    _expect(lib, call(mode=1), SH, b"mask")
    _expect(lib, call(mode=0, crm=P), SH, b"mask")
    _expect(lib, call(real=None), SH)
    _expect(lib, call(wav=None), SH)
    _expect(lib, call(pcm=P, peak=None), SH, b"peak")
    _expect(lib, call(crm_out=P), SH, b"lengths")
    _expect(lib, call(lengths=_lens(300, 200), length=300, lens_dev=None), SH, b"length table")
    _expect(lib, call(lengths=_lens(300, 32), length=300), SH, b"clip 1")
    _expect(lib, call(lengths=_lens(299, 200), length=300), SH, b"longest")


def test_adjoint_and_epilogue_hooks_refuse_without_gpu(lib):
    from fullsubnet_b200 import _lib
    SH, UN = _lib.FSN_ERR_SHAPE, _lib.FSN_ERR_UNSUPPORTED

    def adj(dwav=P, B=2, L=300, T=20, n=64, hop=16, W=64, dcrm=P):
        return lib.fsn_debug_istft_mask_adjoint(dwav, P, P, B, L, T, n, hop, W, dcrm, None)

    _expect(lib, adj(B=65536), UN, b"65535")
    _expect(lib, adj(n=1536, W=64), UN, b"unsupported")
    _expect(lib, adj(n=4096, W=64), UN, b"unsupported")
    for kw in ({"B": 0}, {"L": 0}, {"T": 0}, {"hop": 0}, {"hop": 65}, {"W": 0}, {"W": 65}, {"dwav": None},
               {"dcrm": None}):
        _expect(lib, adj(**kw), SH)

    def epi(enh=P, peak=P, B=2, L=300, lengths=None, lens_dev=P, pcm=P, crm_out=None, F=33, T=20, hop=16):
        return lib.fsn_debug_wav_epilogue(enh, peak, B, L, lengths, lens_dev, 26213.6, pcm, crm_out, F, T, hop, None)

    for kw in ({"B": 0}, {"L": 0}, {"F": 1}, {"T": 0}, {"hop": 0}, {"peak": None}, {"crm_out": P}, {"enh": None},
               {"lengths": _lens(300, 200), "lens_dev": None}, {"lengths": _lens(300, 32)}, {"lengths": _lens(299, 200)}):
        _expect(lib, epi(**kw), SH)
