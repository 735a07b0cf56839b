"""The signal layer alone against float64: the STFT, iSTFT and iSTFT-mask-adjoint kernels of fsn_dsp.cu on both transform
policies (radix-2 FFT and direct DFT) and the wav epilogue through their unit-test hooks, against the reference of
tests/test_cpu_dsp.py (itself pinned to torch.stft / torch.istft / autograd in float64).

Every call also checks: the guard floats past each output are untouched, every output element is written, two runs give
the same bits, and a clip inside a batch gives the bits it gives alone.  Error bounds are about 4x the worst error
measured on an H100 for each family (printed with -s as `[dsp] family worst`)."""
import ctypes as C

import numpy as np
import pytest
import torch

from test_cpu_dsp import ref_istft, ref_mask, ref_mask_adjoint, ref_stft, _smem_ok

pytestmark = pytest.mark.gpu

RADIX2 = [16, 32, 64, 128, 256, 512, 1024, 2048]
DFT = [18, 96, 120, 480, 960, 1200]
GAIN = np.float32(0.8 * 32767)
GUARD = 37
SENT = -3.0e38  # never written by a kernel
# bounds about 4x the worst |error| / scale measured on an H100 80GB HBM3 (700 W): STFT radix-2 3.9e-7, direct DFT
# 1.7e-6; iSTFT radix-2 2.4e-7, direct DFT 2.1e-6; mask mode 1 1.8e-6, mode 2 2.1e-6; adjoint 2.0e-6, and the
# dot-product identity between the iSTFT and adjoint kernels 3.6e-7
TOL = {"stft_radix2": 1.5e-6, "stft_dft": 7e-6, "istft_radix2": 1e-6, "istft_dft": 8e-6, "mask1": 7e-6, "mask2": 8e-6,
       "adjoint": 8e-6, "adjoint_identity": 1.5e-6}
WORST = {}


def _note(family, err):
    WORST[family] = max(WORST.get(family, 0.0), float(err))
    assert err < TOL[family], (family, err)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k, v in sorted(WORST.items()):
        print(f"[dsp] {k} worst {v:.3e} (bound {TOL[k]:.0e})")


@pytest.fixture(scope="module")
def lib():
    from fullsubnet_b200 import _lib
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return _lib.load()


DEV = torch.device("cuda:0")


def _bits(a):
    return np.ascontiguousarray(a).view(np.int32)


class Out:
    """A device output with GUARD sentinel floats behind it."""

    def __init__(self, shape, dtype=torch.float32, fill=None):
        n = int(np.prod(shape))
        self.shape, self.n = shape, n
        if fill is None:
            self.buf = torch.full((n + GUARD,), SENT, dtype=torch.float32, device=DEV)
        else:
            self.buf = torch.cat([torch.as_tensor(fill, dtype=torch.float32).reshape(-1),
                                  torch.full((GUARD,), SENT, dtype=torch.float32)]).to(DEV)
        self.ptr = self.buf.data_ptr()

    def get(self, written=True):
        b = self.buf.cpu().numpy()
        assert np.all(_bits(b[self.n:]) == _bits(np.full(GUARD, SENT, np.float32))), "guard floats overwritten"
        a = b[:self.n].reshape(self.shape)
        if written:
            assert not np.any(a == np.float32(SENT)), "output element not written"
        return a


def _lens_args(lengths, B):
    if lengths is None:
        return None, None, None
    h = np.ascontiguousarray(lengths, dtype=np.int32)
    return h, h.ctypes.data_as(C.c_void_p), torch.empty(B, dtype=torch.int32, device=DEV)


# ------------------------------------------------------------------ STFT
OUTS = ("mag", "phase", "real", "imag", "magT")


def run_stft(lib, x, n, hop, W, lengths=None, outs=OUTS, la=3):
    from fullsubnet_b200 import _lib
    B, L = x.shape
    F, T = n // 2 + 1, 1 + L // hop
    Tp = T + la
    o = {k: Out((B, Tp, F) if k == "magT" else (B, F, T)) for k in outs}
    xd = torch.from_numpy(np.ascontiguousarray(x, np.float32)).to(DEV)
    h, hp, ld = _lens_args(lengths, B)
    p = [o[k].ptr if k in o else None for k in OUTS]
    _lib.check(lib.fsn_debug_stft(xd.data_ptr(), B, L, n, hop, W, hp, _lib.ptr(ld), *p, Tp if "magT" in o else 0,
                                  _lib.stream_ptr(DEV)))
    torch.cuda.synchronize()
    return {k: v.get() for k, v in o.items()}


def check_stft(lib, x, n, hop, W, lengths=None):
    """One STFT case: every output against float64, DC / Nyquist exactly, frames past each clip 0, bits stable and equal
    to each clip alone."""
    family = "stft_radix2" if n in RADIX2 else "stft_dft"
    B, L = x.shape
    F, T = n // 2 + 1, 1 + L // hop
    Lb = [L] * B if lengths is None else list(lengths)
    got = run_stft(lib, x, n, hop, W, lengths)
    ref = np.zeros((B, F, T), np.complex128)
    for b in range(B):
        Xb = ref_stft(x[b, :Lb[b]], n, hop, W)
        ref[b, :, :Xb.shape[1]] = Xb
    scale = max(np.abs(ref).max(), 1e-30)
    re, im, mag, ph = got["real"], got["imag"], got["mag"], got["phase"]
    _note(family, max(np.abs(re - ref.real).max(), np.abs(im - ref.imag).max(), np.abs(mag - np.abs(ref)).max()) / scale)
    # phase compared directly (not modulo 2 pi), as |d phase| * |X|, away from the branch cut of atan2
    a = np.abs(ref)
    far = (ref.real > 0) | (np.abs(ref.imag) > 1e-4 * scale)
    far[:, [0, F - 1], :] = False
    _note(family, (np.abs(ph - np.angle(ref)) * a)[far].max() / scale if far.any() else 0.0)
    # DC and Nyquist: Im is +0 and the phase 0 or +pi, in every frame
    for k in (0, F - 1):
        assert np.all(_bits(im[:, k]) == 0), f"Im at bin {k} is not +0"
        assert np.array_equal(_bits(ph[:, k]), _bits(np.where(np.signbit(re[:, k]), np.float32(np.pi), np.float32(0))))
        sure = np.abs(ref[:, k].real) > 1e-4 * scale
        assert np.array_equal(np.signbit(re[:, k])[sure], (ref[:, k].real < 0)[sure])
    # magT: the time-major magnitude, look-ahead rows (and frames past each clip) exactly 0
    assert np.array_equal(_bits(got["magT"][:, :T]), _bits(mag.transpose(0, 2, 1)))
    assert np.all(_bits(got["magT"][:, T:]) == 0)
    for b in range(B):
        Tb = 1 + Lb[b] // hop
        for k in ("real", "imag", "mag", "phase"):
            assert np.all(_bits(got[k][b, :, Tb:]) == 0), (k, b)
    # the same bits again, and each clip alone
    again = run_stft(lib, x, n, hop, W, lengths)
    for k in OUTS:
        assert np.array_equal(_bits(again[k]), _bits(got[k])), k
    for b in sorted({0, B - 1}):
        Tb = 1 + Lb[b] // hop
        alone = run_stft(lib, x[b:b + 1, :Lb[b]], n, hop, W, outs=("real", "imag", "mag", "phase"))
        for k in alone:
            assert np.array_equal(_bits(alone[k][0]), _bits(got[k][b, :, :Tb])), (k, b)
    return got


def _hops(n, istft):
    h = [n // 2, n // 4, n // 3 + 1, n]
    if not istft:
        h.append(n + n // 2 + 1)
    return sorted(set(h))


def _length_for(n, hop, r):
    """a clip length whose frame count T = 1 + L//hop is r mod 16 (r = -1: the shortest clip, n/2 + 1)"""
    if r < 0:
        return n // 2 + 1
    T = 32 + r
    while (T - 1) * hop + hop // 2 <= n // 2:
        T += 16
    return (T - 1) * hop + hop // 2


@pytest.mark.parametrize("n", RADIX2 + DFT)
def test_stft_matches_float64(lib, n):
    rng = np.random.default_rng(n)
    case = 0
    for hop in _hops(n, istft=False):
        for W in (n, n - 1, n // 2, 1):
            L = _length_for(n, hop, (-1, 0, 1, 2)[case % 4])
            B = 3 if case % 2 else 1
            x = rng.standard_normal((B, L)).astype(np.float32)
            lengths = None
            if B == 3 and case % 4 == 1 and L > n // 2 + 2:
                lengths = [n // 2 + 1, L, (L + n // 2 + 1) // 2]
            check_stft(lib, x, n, hop, W, lengths)
            case += 1
    x = rng.standard_normal((1, 64000)).astype(np.float32)
    check_stft(lib, x, n, n // 4, n - 1)


@pytest.mark.parametrize("n", [16, 512, 2048, 18, 960, 1200])
def test_stft_outputs_requested_alone(lib, n):
    """each of mag / phase / real / imag / magT alone gives the bits it gives among all five"""
    x = np.random.default_rng(7).standard_normal((3, 5 * n + 3)).astype(np.float32)
    lengths = [5 * n + 3, n // 2 + 1, 2 * n]
    full = run_stft(lib, x, n, n // 4, n, lengths)
    for k in OUTS:
        one = run_stft(lib, x, n, n // 4, n, lengths, outs=(k,))
        assert np.array_equal(_bits(one[k]), _bits(full[k])), k


# ------------------------------------------------------------------ iSTFT
def run_istft(lib, X, n, hop, W, length=0, crm=None, mode=0, cstride=1, lengths=None, peak=False, pcm=False,
              crm_out=None):
    """X complex [B,F,T] -> dict(wav, peak bits, pcm, crm_out) through fsn_debug_istft"""
    from fullsubnet_b200 import _lib
    B, F, T = X.shape
    out_len = length if length > 0 else hop * (T - 1)
    if cstride == 1:
        spec = torch.from_numpy(np.stack([X.real, X.imag]).astype(np.float32)).to(DEV)
        rp, ip = spec[0].data_ptr(), spec[1].data_ptr()
    else:
        spec = torch.from_numpy(np.stack([X.real, X.imag], -1).astype(np.float32)).to(DEV)
        rp, ip = spec.data_ptr(), spec.data_ptr() + 4
    cd = None if crm is None else torch.from_numpy(np.ascontiguousarray(crm, np.float32)).to(DEV)
    wav = Out((B, out_len))
    pk = torch.full((B + 1,), 0x7f7f7f7f, dtype=torch.int32, device=DEV) if peak else None
    pc = torch.full((B * out_len + 16,), 12345, dtype=torch.int16, device=DEV) if pcm else None
    co = None if crm_out is None else Out(crm_out.shape, fill=crm_out)
    h, hp, ld = _lens_args(lengths, B)
    _lib.check(lib.fsn_debug_istft(rp, ip, cstride, _lib.ptr(cd), mode, B, T, n, hop, W, length, hp, _lib.ptr(ld),
                                   wav.ptr, _lib.ptr(pk), _lib.ptr(pc), float(GAIN), None if co is None else co.ptr,
                                   _lib.stream_ptr(DEV)))
    torch.cuda.synchronize()
    r = {"wav": wav.get()}
    if peak:
        p = pk.cpu().numpy()
        assert p[B] == 0x7f7f7f7f
        r["peak"] = p[:B].copy()
    if pcm:
        q = pc.cpu().numpy()
        assert np.all(q[B * out_len:] == 12345)
        r["pcm"] = q[:B * out_len].reshape(B, out_len)
    if co is not None:
        r["crm_out"] = co.get(written=False)
    return r


def _mask(rng, shape, mode):
    if mode == 0:
        return None
    if mode == 2:
        return rng.uniform(-2, 2, shape).astype(np.float32)
    m = rng.uniform(-12, 12, shape).astype(np.float32)  # beyond +-9.9 on both sides
    flat = m.reshape(-1)
    k = rng.choice(flat.size, size=min(flat.size, 60), replace=False)
    flat[k[0::5]] = np.float32(9.9)
    flat[k[1::5]] = -np.float32(9.9)
    flat[k[2::5]] = np.nan
    flat[k[3::5]] = 1e30
    flat[k[4::5]] = -np.inf
    return m


def check_istft(lib, X, n, hop, W, length=0, crm=None, mode=0, cstride=1, lengths=None):
    """One iSTFT case: every sample against float64 (error times the float64 envelope), exact 0 where the envelope is 0,
    the peak, the int16 output, bits stable and equal to each clip alone."""
    family = ("istft_radix2" if n in RADIX2 else "istft_dft") if mode == 0 else f"mask{mode}"
    B, F, T = X.shape
    out_len = length if length > 0 else hop * (T - 1)
    Lb = [out_len] * B if lengths is None else list(lengths)
    got = run_istft(lib, X, n, hop, W, length, crm, mode, cstride, lengths, peak=True, pcm=True)
    y = got["wav"]
    Y = ref_mask(X.astype(np.complex128), crm, mode)
    for b in range(B):
        Tb = 1 + Lb[b] // hop if lengths is not None else T
        yr, env = ref_istft(Y[b, :, :Tb], n, hop, W, Lb[b])
        Yd = Y[b, :, :Tb].copy()
        Yd[[0, -1]] = Yd[[0, -1]].real
        A = max(np.abs(np.fft.irfft(Yd.T, n=n, axis=1)).max(), 1e-30)
        _note(family, (np.abs(y[b, :Lb[b]] - yr) * env).max() / (A * max(env.max(), 1e-30)))
        assert np.all(_bits(y[b, :Lb[b]][env == 0]) == 0), "non-zero output where the envelope is 0"
        assert np.all(_bits(y[b, Lb[b]:]) == 0)
        # the peak is max|y| of the kernel's own output; int16 = float32 gain * y / peak, truncated
        pk = np.abs(y[b, :Lb[b]]).max()
        assert got["peak"][b] == _bits(np.float32(pk)), b
        want = np.zeros(out_len, np.int16)
        if pk > 0:
            want[:Lb[b]] = ((GAIN * y[b, :Lb[b]]) / np.float32(pk)).astype(np.int16)
        assert np.array_equal(got["pcm"][b], want), b
    again = run_istft(lib, X, n, hop, W, length, crm, mode, cstride, lengths, peak=True, pcm=True)
    for k in ("wav", "peak", "pcm"):
        assert np.array_equal(again[k].view(np.uint8), got[k].view(np.uint8)), k
    for b in sorted({0, B - 1}):
        Tb = 1 + Lb[b] // hop if lengths is not None else T
        ln = Lb[b] if lengths is not None else length
        alone = run_istft(lib, np.ascontiguousarray(X[b:b + 1, :, :Tb]), n, hop, W, ln,
                          None if crm is None else np.ascontiguousarray(crm[b:b + 1, :, :, :Tb]), mode, cstride, peak=True)
        assert np.array_equal(_bits(alone["wav"][0]), _bits(y[b, :Lb[b]])), b
        assert alone["peak"][0] == got["peak"][b]
    return got


def _spectrum(rng, B, F, T):
    return (rng.standard_normal((B, F, T)) + 1j * rng.standard_normal((B, F, T))).astype(np.complex64)  # Im(DC) != 0


def _small_hops(n):
    """the hop whose shared memory first crosses the 48 KB default, and the smallest hop that still fits the opt-in"""
    if n < 64:
        return []
    fits = [h for h in range(1, n + 1) if _smem_ok(n, h)]
    is_pow2 = n & (n - 1) == 0

    def smem(h):
        np_max = (16 + -(-n // h) + 2) // 2
        return (np_max * (n + 1) * 8 + n // 2 * 8 + n * 4) if is_pow2 else (2 * np_max * n * 8 + n * 12)
    over48 = [h for h in fits if smem(h) > 48 * 1024]
    return sorted({min(fits), max(over48)}) if over48 else [min(fits)]


@pytest.mark.parametrize("n", RADIX2 + DFT)
def test_istft_matches_float64(lib, n):
    rng = np.random.default_rng(1000 + n)
    F = n // 2 + 1
    case = 0
    for hop in _hops(n, istft=True) + _small_hops(n):
        for W in (n, n - 1, n // 2, 1):
            L = _length_for(n, hop, (0, 1, 2, -1)[case % 4])
            T = 1 + L // hop
            B = 3 if case % 2 else 1
            mode = case % 3
            lengths, length = None, (0, hop * (T - 1) - hop // 2 - 1, hop * (T - 1), n // 2 + hop * (T - 1) + 7, L)[case % 5]
            if length < 0 or (length == 0 and T == 1):
                length = L
            if B == 3 and case % 4 == 3 and L > n // 2 + 2:
                lengths, length = [L, n // 2 + 1, (L + n // 2 + 1) // 2], L
            X = _spectrum(rng, B, F, T)
            check_istft(lib, X, n, hop, W, length, _mask(rng, (B, 2, F, T), mode), mode, 1 + case % 2, lengths)
            case += 1
    X = _spectrum(rng, 1, F, 1 + 64000 // (n // 2))
    check_istft(lib, X, n, n // 2, n, 64000, _mask(rng, (1, 2, F, X.shape[2]), 1), 1)


@pytest.mark.parametrize("n", [64, 96])
def test_istft_zero_envelope_is_exactly_zero(lib, n):
    """win_length = hop = n/2: torch.istft refuses this shape; the kernels write 0 on the zero-envelope samples"""
    rng = np.random.default_rng(n)
    X = _spectrum(rng, 3, n // 2 + 1, 20)
    y = check_istft(lib, X, n, n // 2, n // 2, 0)["wav"]
    _, env = ref_istft(X[0], n, n // 2, n // 2)
    assert (env == 0).sum() >= 15 and np.all(_bits(y[:, env == 0]) == 0)


# ------------------------------------------------------------------ per-clip lengths, the epilogue
@pytest.mark.parametrize("n,hop,W", [(512, 256, 512), (256, 64, 255), (64, 24, 32), (960, 480, 960), (120, 45, 60)])
def test_per_clip_lengths_and_epilogue(lib, n, hop, W):
    """STFT -> mask -> iSTFT with per-clip lengths as the wav -> wav entry points run them: every row is the bits of its
    clip alone, the all-equal lengths give the bits of no lengths, and crm_out is zeroed exactly past each clip."""
    rng = np.random.default_rng(n + hop)
    L = 7 * n + 5
    F, T = n // 2 + 1, 1 + L // hop
    lengths = [n // 2 + 1, L, n + 3, 3 * n, L - 1, (L + n) // 2]
    B = len(lengths)
    x = rng.standard_normal((B, L)).astype(np.float32)
    st = check_stft(lib, x, n, hop, W, lengths)
    for b in range(B):  # rows past their clip hold garbage in a real batch: the kernels must not read them
        x[b, lengths[b]:] = 1e30
    assert np.array_equal(_bits(run_stft(lib, x, n, hop, W, lengths)["real"]), _bits(st["real"]))
    X = st["real"] + 1j * st["imag"]
    crm = _mask(rng, (B, 2, F, T), 1)
    check_istft(lib, X, n, hop, W, L, crm, 1, 1, lengths)
    # all lengths equal to L: the bits of the call without lengths
    same = run_istft(lib, X, n, hop, W, L, crm, 1, peak=True, pcm=True, lengths=[L] * B)
    none = run_istft(lib, X, n, hop, W, L, crm, 1, peak=True, pcm=True)
    for k in ("wav", "peak", "pcm"):
        assert np.array_equal(same[k].view(np.uint8), none[k].view(np.uint8)), k
    # zero_frames_past: frames t >= 1 + lengths[b]/hop of crm_out are 0, every other float untouched
    junk = rng.standard_normal((B, 2, F, T)).astype(np.float32)
    co = run_istft(lib, X, n, hop, W, L, crm, 1, lengths=lengths, crm_out=junk)["crm_out"]
    for b in range(B):
        Tb = 1 + lengths[b] // hop
        assert np.all(_bits(co[b, :, :, Tb:]) == 0) and np.array_equal(_bits(co[b, :, :, :Tb]), _bits(junk[b, :, :, :Tb]))


def test_wav_epilogue_on_any_signal(lib):
    """the int16 scaling keeps exactly lengths[b] samples of each row, even where the row is not 0 past its clip"""
    from fullsubnet_b200 import _lib
    rng = np.random.default_rng(5)
    B, L = 4, 3001
    lengths = [3001, 1000, 1001, 257]
    y = rng.uniform(-3, 3, (B, L)).astype(np.float32)
    peak = np.abs(y).max(1).astype(np.float32)
    peak[3] = 0.0  # an all-zero clip: 0 out
    yd = torch.from_numpy(y).to(DEV)
    pk = torch.from_numpy(_bits(peak).copy()).to(DEV)
    pc = torch.full((B * L + 16,), 12345, dtype=torch.int16, device=DEV)
    h, hp, ld = _lens_args(lengths, B)
    _lib.check(lib.fsn_debug_wav_epilogue(yd.data_ptr(), pk.data_ptr(), B, L, hp, ld.data_ptr(), float(GAIN), pc.data_ptr(),
                                          None, 257, 1 + L // 128, 128, _lib.stream_ptr(DEV)))
    torch.cuda.synchronize()
    q = pc.cpu().numpy()
    assert np.all(q[B * L:] == 12345)
    want = np.zeros((B, L), np.int16)
    for b in range(B):
        if peak[b] > 0:
            want[b, :lengths[b]] = ((GAIN * y[b, :lengths[b]]) / peak[b]).astype(np.int16)
    assert np.array_equal(q[:B * L].reshape(B, L), want)


# ------------------------------------------------------------------ the mask adjoint
def run_adjoint(lib, g, X, n, hop, W):
    from fullsubnet_b200 import _lib
    B, F, T = X.shape
    L = g.shape[1]
    spec = torch.from_numpy(np.stack([X.real, X.imag]).astype(np.float32)).to(DEV)
    gd = torch.from_numpy(np.ascontiguousarray(g, np.float32)).to(DEV)
    d = Out((B, 2, F, T))
    _lib.check(lib.fsn_debug_istft_mask_adjoint(gd.data_ptr(), spec[0].data_ptr(), spec[1].data_ptr(), B, L, T, n, hop, W,
                                                d.ptr, _lib.stream_ptr(DEV)))
    torch.cuda.synchronize()
    a = d.get(written=False)
    assert np.all(a[:, :, F - 1] == np.float32(SENT)), "the Nyquist row was written"
    assert not np.any(a[:, :, :F - 1] == np.float32(SENT))
    return a


@pytest.mark.parametrize("n", RADIX2 + DFT)
def test_mask_adjoint_matches_float64(lib, n):
    rng = np.random.default_rng(2000 + n)
    F = n // 2 + 1
    case = 0
    for hop in _hops(n, istft=True):
        for W in (n, n - 1, n // 2, 1):
            T = (17, 32, 33, 34)[case % 4]
            L = (hop * (T - 1), hop * (T - 1) - hop // 2 - 1, n // 2 + hop * (T - 1) + 5, n // 2 + 1)[case % 4]
            B = 3 if case % 2 else 1
            X = _spectrum(rng, B, F, T)
            # dwav shaped by the envelope: dwav / env is then bounded where the envelope nears 0 (it is a float32
            # cancellation there, in the kernels and in torch alike)
            _, env = ref_istft(np.zeros((F, T)), n, hop, W, L)
            # (no sample of the clip inside a frame's window, e.g. win_length 1 with hop = n: the gradient is 0)
            g = (rng.standard_normal((B, L)) * (env / env.max() if env.max() > 0 else 1.0)).astype(np.float32)
            d = run_adjoint(lib, g, X, n, hop, W)
            for b in range(B):
                ref = ref_mask_adjoint(g[b], X[b].astype(np.complex128), n, hop, W, L)
                _note("adjoint", np.abs(d[b, :, :F - 1] - ref[:, :F - 1]).max() / max(np.abs(ref).max(), 1e-30))
                assert np.all(_bits(d[b, 1, 0]) == 0)
            assert np.array_equal(_bits(run_adjoint(lib, g, X, n, hop, W)), _bits(d))
            b = B - 1
            alone = run_adjoint(lib, g[b:], np.ascontiguousarray(X[b:]), n, hop, W)
            assert np.array_equal(_bits(alone[0]), _bits(d[b]))
            # <istft(X (.) M), g> = <M, adj(g)> between the two kernels (the Nyquist row of M held at 0)
            M = rng.uniform(-2, 2, (B, 2, F, T)).astype(np.float32)
            M[:, :, F - 1] = 0
            y = run_istft(lib, X, n, hop, W, L, M, 2)["wav"].astype(np.float64)
            gg = g.astype(np.float64)
            lhs = float((y * gg).sum())
            rhs = float((M[:, :, :F - 1].astype(np.float64) * d[:, :, :F - 1].astype(np.float64)).sum())
            assert np.isfinite(lhs) and np.isfinite(rhs), (lhs, rhs, np.abs(y).max(), np.abs(gg).max())
            _note("adjoint_identity", abs(lhs - rhs) / max(np.abs(y).sum() * np.abs(gg).max(), 1e-30))
            case += 1
