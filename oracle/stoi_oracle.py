"""Float64 oracle of the STOI intelligibility measure (Taal et al., 2011) as pystoi 0.3.3 computes
``stoi(x, y, fs_sig, extended=False)`` (audio_zen/metrics.py:STOI): clean ``x``, estimate ``y``.  Written from the
definition with numpy and ``scipy.signal.resample_poly``; the stage functions are exposed so that the tests can compare
the library's intermediate buffers (fsn_debug_stoi_stages) stage by stage."""
from __future__ import annotations

import math

import numpy as np
from scipy.signal import resample_poly

FS = 10000
N_FRAME = 256
NFFT = 512
NUMBAND = 15
MINFREQ = 150
N = 30
BETA = -15.0
DYN_RANGE = 40
EPS = np.finfo(float).eps
HOP = N_FRAME // 2


def window() -> np.ndarray:
    """The frame window: np.hanning(N_FRAME + 2)[1:-1] (MATLAB's hanning(256))."""
    return np.hanning(N_FRAME + 2)[1:-1]


def resample_filter(fs_sig: int):
    """(p, q, h, beta): the Octave-style Kaiser-windowed sinc of resample_oct(x, FS, fs_sig), before h / h.sum()."""
    g = math.gcd(FS, fs_sig)
    p, q = FS // g, fs_sig // g
    cutoff = 1.0 / (2 * max(p, q))
    roll_off = cutoff / 10
    rejection_db = 60.0
    L = int(np.ceil((rejection_db - 8) / (28.714 * roll_off)))
    t = np.arange(-L, L + 1)
    beta = 0.1102 * (rejection_db - 8.7)
    h = np.kaiser(2 * L + 1, beta) * 2 * p * cutoff * np.sinc(2 * cutoff * t)
    return p, q, h, beta


def resample(x: np.ndarray, fs_sig: int) -> np.ndarray:
    """x at fs_sig -> float64 at FS (the identity, widened, at FS)."""
    x = np.asarray(x, dtype=np.float64)
    if fs_sig == FS:
        return x
    p, q, h, _ = resample_filter(fs_sig)
    return resample_poly(x, p, q, window=h / h.sum())


def n_frames(n: int) -> int:
    """len(range(0, n - N_FRAME, HOP)): the frames of a signal of n samples (the last possible frame excluded)."""
    return len(range(0, n - N_FRAME, HOP))


def frames(x: np.ndarray) -> np.ndarray:
    w = window()
    return np.array([w * x[i:i + N_FRAME] for i in range(0, len(x) - N_FRAME, HOP)]).reshape(-1, N_FRAME)


def silent_mask(x: np.ndarray) -> np.ndarray:
    """Kept frames of the clean signal: energy within DYN_RANGE dB of the loudest frame."""
    xf = frames(x)
    if len(xf) == 0:
        raise ValueError("STOI: the clip is too short for one frame")
    energies = 20 * np.log10(np.linalg.norm(xf, axis=1) + EPS)
    return (np.max(energies) - DYN_RANGE - energies) < 0


def overlap_add(fr: np.ndarray) -> np.ndarray:
    out = np.zeros((len(fr) + 1) * HOP)
    for i, f in enumerate(fr):
        out[i * HOP:i * HOP + N_FRAME] += f
    return out


def remove_silent_frames(x: np.ndarray, y: np.ndarray):
    """(x_sil, y_sil, mask): both signals rebuilt by overlap-add from the frames the clean signal keeps."""
    mask = silent_mask(x)
    return overlap_add(frames(x)[mask]), overlap_add(frames(y)[mask]), mask


def band_edges():
    """[(lo, hi)] bins of the NUMBAND one-third-octave bands on the NFFT-point grid, band j = bins [lo, hi)."""
    f = np.linspace(0, FS, NFFT + 1)[:NFFT // 2 + 1]
    k = np.arange(NUMBAND, dtype=np.float64)
    lo = MINFREQ * np.power(2.0, (2 * k - 1) / 6)
    hi = MINFREQ * np.power(2.0, (2 * k + 1) / 6)
    return [(int(np.argmin(np.square(f - a))), int(np.argmin(np.square(f - b)))) for a, b in zip(lo, hi)]


def band_magnitudes(x_sil: np.ndarray) -> np.ndarray:
    """[NUMBAND, frames]: sqrt of the summed |rfft|^2 of each windowed, NFFT-padded frame over each band's bins."""
    fr = frames(x_sil)
    spec = np.fft.rfft(fr, n=NFFT, axis=1) if len(fr) else np.zeros((0, NFFT // 2 + 1), np.complex128)
    power = np.square(np.abs(spec)).T  # [bins, frames]
    return np.sqrt(np.stack([power[lo:hi].sum(axis=0) for lo, hi in band_edges()]))


def intermediate_intelligibility(x_tob: np.ndarray, y_tob: np.ndarray) -> float:
    """d over the segments of N frames, or 1e-5 when there are fewer than N frames."""
    T = x_tob.shape[1]
    if T < N:
        return 1e-5
    xs = np.array([x_tob[:, m - N:m] for m in range(N, T + 1)])
    ys = np.array([y_tob[:, m - N:m] for m in range(N, T + 1)])
    alpha = np.linalg.norm(xs, axis=2, keepdims=True) / (np.linalg.norm(ys, axis=2, keepdims=True) + EPS)
    yp = np.minimum(ys * alpha, xs * (1 + 10 ** (-BETA / 20)))
    yp = yp - np.mean(yp, axis=2, keepdims=True)
    xs = xs - np.mean(xs, axis=2, keepdims=True)
    yp /= np.linalg.norm(yp, axis=2, keepdims=True) + EPS
    xs /= np.linalg.norm(xs, axis=2, keepdims=True) + EPS
    J, M = xs.shape[0], xs.shape[1]
    return float(np.sum(yp * xs) / (J * M))


def stages(x, y, fs_sig: int = 16000) -> dict:
    """Every intermediate of stoi(x, y, fs_sig)."""
    if np.shape(x) != np.shape(y):
        raise ValueError("x and y should have the same length")
    xr, yr = resample(x, fs_sig), resample(y, fs_sig)
    xs, ys, mask = remove_silent_frames(xr, yr)
    xb, yb = band_magnitudes(xs), band_magnitudes(ys)
    return {"resampled": (xr, yr), "mask": mask, "compacted": (xs, ys), "bands": (xb, yb),
            "d": intermediate_intelligibility(xb, yb)}


def stoi(x, y, fs_sig: int = 16000) -> float:
    """STOI of the estimate y against the clean x (1-D arrays of the same length, fs_sig 16000 or 10000)."""
    return stages(x, y, fs_sig)["d"]


def min_length(fs_sig: int) -> int:
    """The shortest clip at fs_sig whose resampled signal holds one frame."""
    L = 1
    while n_frames(len(resample(np.zeros(L), fs_sig))) == 0:
        L += 1
    return L


def speechlike(n, seed, sr=16000):
    """A harmonic stack with vibrato and syllable-rate envelope plus a little noise."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / sr
    f0 = 120 + 30 * rng.random() + 8 * np.sin(2 * np.pi * 5 * t)
    phase = 2 * np.pi * np.cumsum(f0) / sr
    x = sum(np.sin(k * phase + rng.random() * 6.3) / k for k in range(1, 25) if k * 160 < sr / 2)
    env = 0.5 + 0.5 * np.sin(2 * np.pi * 3 * t + rng.random() * 6.3) ** 2
    return (0.1 * env * x + 1e-3 * rng.standard_normal(n)).astype(np.float32)
