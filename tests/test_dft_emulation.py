"""CPU emulation of the index arithmetic of the STFT / iSTFT kernels of fullsubnet_b200/csrc/fsn_dsp.cu on their
direct-DFT policy (the shared framing: two real frames packed into one complex direct DFT, un-packing, Hermitian
extension, overlap-add segments) against the oracle STFT / iSTFT.
It pins the ALGORITHM of the non-power-of-two path on the CPU; the kernels themselves are checked on the GPU
(tests/test_gpu_parity.py::test_non_power_of_two_stft_istft)."""
import numpy as np
import pytest
import torch

from oracle import fullsubnet_oracle as O

FR = 16


def reflect(i, n):
    i = np.abs(i)
    return np.where(i > n - 1, 2 * (n - 1) - i, i)


def tables(n, win_length):
    k = np.arange(n)
    tw = np.exp(-2j * np.pi * k / n)
    m = np.arange(n) - (n - win_length) // 2
    win = np.where((m >= 0) & (m < win_length), 0.5 - 0.5 * np.cos(2 * np.pi * m / win_length), 0.0)
    return tw, win


def dft(zin, tw, inverse):
    n = zin.shape[-1]
    idx = (np.arange(n)[:, None] * np.arange(n)[None, :]) % n  # [i, k] -> (i*k) mod n
    w = np.conj(tw) if inverse else tw
    return zin @ w[idx]


def emu_stft(x, n, hop, win_length):
    L = len(x)
    T = 1 + L // hop
    F = n // 2 + 1
    tw, win = tables(n, win_length)
    out = np.zeros((F, T), dtype=np.complex128)
    for t0 in range(0, T, FR):
        zin = np.zeros((FR // 2, n), dtype=np.complex128)
        for p in range(FR // 2):
            for q, t in enumerate((t0 + 2 * p, t0 + 2 * p + 1)):
                if t < T:
                    v = x[reflect(t * hop + np.arange(n) - n // 2, L)] * win
                    zin[p] += v if q == 0 else 1j * v
        z = dft(zin, tw, False)
        for j in range(FR):
            t = t0 + j
            if t >= T:
                continue
            k = np.arange(F)
            zk = z[j >> 1, k]
            zn = z[j >> 1, np.where(k == 0, 0, n - k)]
            if j & 1 == 0:
                out[:, t] = 0.5 * (zk.real + zn.real) + 1j * 0.5 * (zk.imag - zn.imag)
            else:
                out[:, t] = 0.5 * (zk.imag + zn.imag) - 1j * 0.5 * (zk.real - zn.real)
    return out


def emu_istft(E, n, hop, win_length, out_len):
    F, T = E.shape
    tw, win = tables(n, win_length)
    seg = FR * hop
    out = np.zeros(out_len)
    full = n + hop * (T - 1)
    for blk in range((out_len + seg - 1) // seg):
        s_begin = n // 2 + blk * seg
        s_end = min(s_begin + seg, n // 2 + out_len)
        t_min = (s_begin - n) // hop + 1 if s_begin >= n else 0
        t_max = min(T - 1, (s_end - 1) // hop)
        nframes = t_max - t_min + 1
        npairs = (nframes + 1) // 2 if nframes > 0 else 0
        zin = np.zeros((max(npairs, 1), n), dtype=np.complex128)
        for p in range(npairs):
            e = np.zeros((2, F), dtype=np.complex128)
            for q in range(2):
                t = t_min + 2 * p + q
                if t <= t_max:
                    e[q] = E[:, t]
            e.imag[:, 0] = 0.0
            e.imag[:, n // 2] = 0.0
            k = np.arange(F)
            zin[p, k] = (e[0].real - e[1].imag) + 1j * (e[0].imag + e[1].real)
            km = np.arange(1, n // 2)
            zin[p, n - km] = (e[0].real[km] + e[1].imag[km]) + 1j * (-e[0].imag[km] + e[1].real[km])
        z = dft(zin, tw, True)
        for s in range(s_begin, s_end):
            acc = env = 0.0
            if s < full:
                tl = max(t_min, (s - n) // hop + 1 if s >= n else 0)
                th = min(t_max, s // hop)
                for t in range(tl, th + 1):
                    i, q = s - t * hop, t - t_min
                    v = z[q >> 1, i]
                    acc += (v.imag if q & 1 else v.real) / n * win[i]
                    env += win[i] ** 2
            out[s - n // 2] = acc / env if env > 1e-11 else 0.0
    return out


@pytest.mark.parametrize("n,hop,L", [(960, 480, 5000), (96, 24, 1000), (120, 60, 777)])
def test_direct_dft_stft_istft_emulation_matches_oracle(n, hop, L):
    y = O.make_noisy(1, L, seed=n)[0]
    mag, _, re, im = O.stft(y[None], n, hop, n)
    got = emu_stft(y.numpy().astype(np.float64), n, hop, n)
    ref = re[0].numpy() + 1j * im[0].numpy()
    assert got.shape == ref.shape
    assert np.abs(got - ref).max() < 2e-5 * np.abs(ref).max()
    E = ref * (0.5 + 0.25j)  # arbitrary spectrum: Im of DC / Nyquist must be ignored like torch.istft
    want = O.istft((torch.from_numpy(E.real.astype(np.float32))[None], torch.from_numpy(E.imag.astype(np.float32))[None]),
                   n, hop, n, length=L, input_type="real_imag")[0].numpy()
    back = emu_istft(E, n, hop, n, L)
    n_ok = hop * (ref.shape[1] - 1)  # beyond that the window-square envelope tends to 0 (ill-conditioned in torch too)
    assert np.abs(back[:n_ok] - want[:n_ok]).max() < 2e-5 * max(1.0, np.abs(want).max())
