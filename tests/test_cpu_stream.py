"""Chunked streaming of fullband_baseline without a GPU: the state, workspace and delay queries answer, every refusal
happens before any CUDA call with its error code, and the delay matches a numpy emulation of the framing schedule."""
import ctypes as C

import numpy as np
import pytest

from fullsubnet_b200 import _lib


def _desc(norm="cumulative_laplace_norm", la=2, cell="LSTM", prec="fp32", F=257, H=512):
    from fullsubnet_b200.fullband_baseline.model import Model
    return _lib.FullbandDesc(num_freqs=F, hidden=H, num_layers=3, look_ahead=la, activation=0,
                             norm_type=Model.NORM_TYPES[norm], precision=_lib.PREC[prec], cell_type=_lib.CELL[cell])


def _delay_emulated(n_fft, hop, la):
    """Smallest D with which every call can emit its K*hop samples: after N (a multiple of hop) input samples, step m
    (frame m) has run when its frame and the frame's pair partner (2k, 2k+1) are complete, frame t's cRM comes from
    step t + la, and output sample x reads the frames t with t*hop <= x + n/2 < t*hop + n_fft plus the partner of the
    last one in its iSTFT pair."""
    need = 0
    for N in range(0, 64 * hop, hop):
        # frames complete: the pair (2k, 2k+1) both inside [0, N); steps run at a fixed lag c behind N/hop
        c = -(-(n_fft // 2) // hop)
        steps = N // hop - c
        for m in range(max(steps, 0)):
            assert (m | 1) * hop + n_fft // 2 <= N  # the lag keeps every step's pair complete
        crm_frames = steps - la  # frames [0, crm_frames) have their cRM
        x = 0
        while (x + n_fft // 2) // hop + 1 < crm_frames:
            x += 1
        need = max(need, N - x)
    return need


@pytest.mark.parametrize("n_fft,hop,la", [(512, 256, 2), (512, 128, 0), (256, 256, 1), (512, 160, 3)])
def test_delay_formula_matches_emulation(n_fft, hop, la):
    lib = _lib.load()
    d = _desc(la=la, F=n_fft // 2 + 1)
    D = lib.fsn_fullband_stream_delay(C.byref(d), n_fft, hop)
    assert D == _delay_emulated(n_fft, hop, la)
    assert D == n_fft // 2 + (la + 1 + -(-(n_fft // 2) // hop)) * hop


def test_queries_answer():
    lib = _lib.load()
    for norm in ("cumulative_laplace_norm", "forgetting_norm"):
        d = _desc(norm)
        s1 = lib.fsn_fullband_stream_state_bytes(C.byref(d), 1, 512, 256)
        s4 = lib.fsn_fullband_stream_state_bytes(C.byref(d), 4, 512, 256)
        assert s1 > 2 * 3 * 512 * 4 and s4 == 4 * s1 and s1 % 256 == 0
        w1 = lib.fsn_fullband_stream_workspace_bytes(C.byref(d), 4, 1, 512, 256)
        w64 = lib.fsn_fullband_stream_workspace_bytes(C.byref(d), 4, 64, 512, 256)
        assert 0 < w1 < w64
        assert lib.fsn_fullband_stream_delay(C.byref(d), 512, 256) == 256 + 4 * 256


@pytest.mark.parametrize("kw,n_fft,code", [
    (dict(norm="offline_laplace_norm"), 512, _lib.FSN_ERR_UNSUPPORTED),
    (dict(cell="GRU"), 512, _lib.FSN_ERR_UNSUPPORTED),
    (dict(prec="f16_tc"), 512, _lib.FSN_ERR_UNSUPPORTED),
    (dict(F=481), 960, _lib.FSN_ERR_UNSUPPORTED),
    (dict(F=200), 512, _lib.FSN_ERR_SHAPE),
])
def test_refusals_before_any_cuda_call(kw, n_fft, code):
    lib = _lib.load()
    d = _desc(**kw)
    assert lib.fsn_fullband_stream_state_bytes(C.byref(d), 2, n_fft, 256) == 0
    assert lib.fsn_last_error_code() == code
    assert lib.fsn_fullband_stream_workspace_bytes(C.byref(d), 2, 4, n_fft, 256) == 0
    assert lib.fsn_last_error_code() == code
    assert lib.fsn_fullband_stream_delay(C.byref(d), n_fft, 256) == -code
    rc = lib.fsn_fullband_stream_step(C.byref(d), 1, 1, 1, 1, None, None, 2, 4, n_fft, 256, n_fft, 1, 1, 1 << 30, 1,
                                      1 << 30, None)
    assert rc == code
    assert lib.fsn_last_launch_count() == 0


def test_streamer_refuses_other_models():
    from fullsubnet_b200.stream import Streamer
    from fullsubnet_b200.fullsubnet.model import Model
    from oracle import fullsubnet_oracle as O
    m = Model(**dict(O.DEFAULT_MODEL_ARGS, norm_type="cumulative_laplace_norm"))
    with pytest.raises(NotImplementedError):
        Streamer(m, 2)


def _fbb_streamer(slots):
    from fullsubnet_b200.fullband_baseline.model import Model
    from fullsubnet_b200.stream import Streamer
    from oracle import fullband_baseline_oracle as BO
    return Streamer(Model(**dict(BO.DEFAULT_FBB_ARGS, norm_type="forgetting_norm")), slots)


def test_streamer_refuses_short_and_overlong_clips():
    """The host follows each slot's position and refuses, before the call, a clip of n_fft/2 samples or fewer and one
    past the library's position limit; a restored slot (position unknown) is not checked."""
    s = _fbb_streamer(2)
    assert s._check_lengths(1, [1, 1], [-1, 257]) == [256, None]
    with pytest.raises(AssertionError):
        s._check_lengths(1, [1, 0], [256, -1])
    s._pos = [1000, s.MAX_CLIP - 10]
    with pytest.raises(AssertionError):
        s._check_lengths(1, None, None)
    assert s._check_lengths(1, None, [0, 5]) == [None, None]
    s.slot_state(1)
    assert s._check_lengths(1, None, [-1, 0]) == [1256, None]
    s.copy_slot(0, 1)
    assert s._pos == [1000, 1000]
