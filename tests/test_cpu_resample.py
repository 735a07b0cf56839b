"""fsn_resample without a GPU: argument checks (each fails before any CUDA call), the workspace query, the library's
output length against the host resampler's, and the defaults of the new keyword."""
import ctypes as C
import inspect
from math import gcd

import numpy as np
import pytest

from fullsubnet_b200 import _lib
from fullsubnet_b200.acoustics.resample import resampled_length
from fullsubnet_b200.dataset import Dataset, _resampled_length
from fullsubnet_b200.inferencer import Inferencer

RATES = (8000, 11025, 16000, 22050, 24000, 32000, 44100, 48000, 96000)


@pytest.fixture(scope="module")
def lib():
    return _lib.load()


def _call(lib, lengths, N_max, sr_in=48000, sr_out=16000, zeros=24, B=None, x=16, y=16, N_out_max=None, ws=16,
          ws_bytes=0):
    """fsn_resample with stand-in device pointers (never read: every case fails before the first launch)."""
    arr = None if lengths is None else (C.c_int32 * len(lengths))(*lengths)
    B = (len(lengths) if lengths is not None else 2) if B is None else B
    if N_out_max is None:
        N_out_max = resampled_length(N_max, sr_in, sr_out) if sr_in > 0 and sr_out > 0 else N_max
    return lib.fsn_resample(x, arr, B, N_max, sr_in, sr_out, zeros, y, N_out_max, ws, ws_bytes, None)


def test_workspace_query_needs_no_gpu(lib):
    n1, n300 = lib.fsn_resample_workspace_bytes(1, 48000, 48000, 16000, 24), lib.fsn_resample_workspace_bytes(
        300, 48000, 48000, 16000, 24)
    assert 0 < n1 < n300 and n300 >= 300 * 4 and n300 % 256 == 0
    assert lib.fsn_resample_workspace_bytes(4, 16000, 16000, 16000, 1) == lib.fsn_resample_workspace_bytes(4, 1, 44100,
                                                                                                            8000, 8)
    for args, code in (((0, 100, 48000, 16000, 24), _lib.FSN_ERR_SHAPE), ((2, 0, 48000, 16000, 24), _lib.FSN_ERR_SHAPE),
                       ((2, 100, 0, 16000, 24), _lib.FSN_ERR_SHAPE), ((2, 100, 48000, -16000, 24), _lib.FSN_ERR_SHAPE),
                       ((2, 100, 48000, 16000, 0), _lib.FSN_ERR_SHAPE), ((65536, 100, 48000, 16000, 24),
                                                                         _lib.FSN_ERR_UNSUPPORTED),
                       ((2, 100, 1 << 30, 1, 24), _lib.FSN_ERR_UNSUPPORTED)):
        assert lib.fsn_resample_workspace_bytes(*args) == 0, args
        assert lib.fsn_last_error_code() == code, args
    assert lib.fsn_resample_workspace_bytes(65535, 100, 48000, 16000, 24) > 0
    assert lib.fsn_resample_workspace_bytes(2, 100, 1 << 24, 1, 24) > 0  # half = 24 * 2^24 = 2^28.6 taps: accepted


def test_rejects_bad_arguments_before_any_cuda_call(lib):
    assert _call(lib, [4800, 0, 3000], 4800) == _lib.FSN_ERR_SHAPE
    assert b"clip 1" in lib.fsn_last_error()
    assert _call(lib, [4800, 4801], 4800) == _lib.FSN_ERR_SHAPE  # longer than the row
    assert b"clip 1" in lib.fsn_last_error()
    assert _call(lib, [-1, 4800], 4800) == _lib.FSN_ERR_SHAPE
    assert _call(lib, None, 4800, B=0) == _lib.FSN_ERR_SHAPE
    assert _call(lib, None, 4800, B=-2) == _lib.FSN_ERR_SHAPE
    assert _call(lib, None, 0) == _lib.FSN_ERR_SHAPE
    assert _call(lib, None, 4800, sr_in=0) == _lib.FSN_ERR_SHAPE
    assert _call(lib, None, 4800, sr_out=-16000) == _lib.FSN_ERR_SHAPE
    assert _call(lib, None, 4800, zeros=0) == _lib.FSN_ERR_SHAPE
    assert _call(lib, None, 4800, x=None) == _lib.FSN_ERR_SHAPE
    assert _call(lib, None, 4800, y=None) == _lib.FSN_ERR_SHAPE
    assert _call(lib, None, 4800, B=65536) == _lib.FSN_ERR_UNSUPPORTED
    assert b"65535" in lib.fsn_last_error()
    assert _call(lib, None, 4800, sr_in=1 << 30, sr_out=1) == _lib.FSN_ERR_UNSUPPORTED
    # the output rows: at least the longest clip's resampled length, which the lengths (not N_max) decide
    assert _call(lib, None, 4800, N_out_max=1599) == _lib.FSN_ERR_SHAPE
    assert b"1600" in lib.fsn_last_error()
    assert _call(lib, [4800, 4800], 4800, N_out_max=1599) == _lib.FSN_ERR_SHAPE
    assert _call(lib, [4000, 3000], 4800, N_out_max=1333) == _lib.FSN_ERR_SHAPE
    # valid arguments reach the workspace check, the last one before the first launch
    assert _call(lib, [4000, 3000], 4800, N_out_max=1334) == _lib.FSN_ERR_WORKSPACE
    assert _call(lib, None, 4800) == _lib.FSN_ERR_WORKSPACE
    assert _call(lib, [1, 4800], 4800, sr_in=16000, sr_out=16000) == _lib.FSN_ERR_WORKSPACE
    need = lib.fsn_resample_workspace_bytes(2, 4800, 48000, 16000, 24)
    assert _call(lib, None, 4800, ws_bytes=need - 1) == _lib.FSN_ERR_WORKSPACE
    assert _call(lib, None, 4800, ws=None, ws_bytes=need) == _lib.FSN_ERR_WORKSPACE


def _library_out_len(lib, N, sr_in, sr_out):
    """The library's n_out for an N-sample clip: the N_out_max it accepts (workspace refusal) against the one below it
    (shape refusal); neither call reaches the device."""
    n = resampled_length(N, sr_in, sr_out)
    ok = _call(lib, [N], N, sr_in=sr_in, sr_out=sr_out, N_out_max=n)
    short = _call(lib, [N], N, sr_in=sr_in, sr_out=sr_out, N_out_max=n - 1)
    assert ok == _lib.FSN_ERR_WORKSPACE and short == _lib.FSN_ERR_SHAPE, (N, sr_in, sr_out, ok, short)
    return n


def test_output_length_matches_the_host_resampler(lib):
    rng = np.random.default_rng(0)
    pairs = [(a, b) for a in RATES for b in RATES if a != b] + [(16000, 16000), (7, 3), (3, 7), (1, 1000)]
    for sr_in, sr_out in pairs:
        Ns = [1, 2, 3, 5, 7, 159, 160, 161, 4799, 4800, 4801, 44099, 44100] + [int(v) for v in rng.integers(1, 200000, 6)]
        for N in Ns:
            n = _library_out_len(lib, N, sr_in, sr_out)
            assert n == _resampled_length(N, sr_in, sr_out), (N, sr_in, sr_out)
            if N <= 5000 and sr_in != sr_out and max(sr_in, sr_out) / min(sr_in, sr_out) < 20:
                assert n == len(Inferencer.resample(np.zeros(N, np.float32), sr_in, sr_out, zeros=2)), (N, sr_in, sr_out)
    # large clips: the host's float64 ceiling, evaluated as it is, up to 2^31 output samples
    for N, sr_in, sr_out in ((2_000_000_000, 48000, 16000), (700_000_000, 16000, 48000), (123_456_789, 44100, 16000)):
        g = gcd(sr_in, sr_out)
        assert _library_out_len(lib, N, sr_in, sr_out) == int(np.ceil(N * (sr_out // g) / (sr_in // g)))


def test_resample_on_device_defaults_to_false():
    assert inspect.signature(Inferencer.enhance_files).parameters["resample_on_device"].default is False
    params = list(inspect.signature(Dataset.__init__).parameters)
    assert params[-1] == "resample_on_device" and params[-2] == "num_workers"
    assert inspect.signature(Dataset.__init__).parameters["resample_on_device"].default is False
