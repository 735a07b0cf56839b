"""Chunked streaming of fast_fullsubnet without a GPU: the delay matches a numpy emulation of the schedule including the
bottleneck's down- and up-sampling (restated from the reference's real_time_downsampling / real_time_upsampling), the
state, workspace and delay queries answer, every refusal happens before any CUDA call with its error code, and the
Streamer refuses what the library cannot stream."""
import ctypes as C

import numpy as np
import pytest

from fullsubnet_b200 import _lib

CUM = "cumulative_laplace_norm"


def _args(**kw):
    from oracle import fast_fullsubnet_oracle as FO
    return dict(FO.DEFAULT_FAST_ARGS, **dict(dict(norm_type=CUM), **kw))


def _desc(norm=CUM, la=2, S=2, cell="LSTM", prec="fp32", F=257):
    return _lib.FastDesc(num_freqs=F, look_ahead=la, shrink_size=S, num_mels=64, enc1_hidden=384, enc2_hidden=257,
                         bn_hidden=384, bn_layers=2, dec_hidden=512, noisy_num_neighbors=5, enc_num_neighbors=0,
                         precision=_lib.PREC[prec], cell_type=_lib.CELL[cell],
                         norm_type={"offline_laplace_norm": 0, CUM: 1, "forgetting_norm": 4}[norm])


def _down_blocks(Tp, S):
    """The frames averaged into each shrunk step by real_time_downsampling: frame 0 alone, then torch.split of frames
    1.. into chunks of S (the last one possibly short), each chunk's mean."""
    rest = np.arange(1, Tp)
    return [np.array([0])] + [rest[i:i + S] for i in range(0, len(rest), S)]


def _up_index(Ts, S, Tp):
    """The shrunk step each frame reads after real_time_upsampling: every step repeated S times, truncated to Tp."""
    return np.repeat(np.arange(Ts), S)[:Tp]


@pytest.mark.parametrize("S", [2, 3])
def test_blocks_end_before_the_frames_that_read_them(S):
    """Frame t reads a block whose last frame is <= t, so a stream has it when it reaches frame t; a clip's short last
    block is never read."""
    for Tp in range(2, 40):
        blocks = _down_blocks(Tp, S)
        up = _up_index(len(blocks), S, Tp)
        for t in range(Tp):
            blk = blocks[up[t]]
            assert blk.max() <= t and blk.max() == up[t] * S
            assert len(blk) == (1 if up[t] == 0 else S)


def _delay_emulated(n_fft, hop, la, S):
    """Smallest D with which every call can emit its K*hop samples, with the bottleneck in the schedule: after N input
    samples (a multiple of hop), step m (frame m) has run when its frame and its pair partner are complete (a lag of
    c steps); the decoder frame t runs once frame t has run and the shrunk step it reads is complete; frame t's cRM is
    decoder frame t + la; output sample x reads the frames t with t*hop <= x + n/2 < t*hop + n_fft."""
    c = -(-(n_fft // 2) // hop)
    Tp = 80
    blocks = _down_blocks(Tp, S)
    up = _up_index(len(blocks), S, Tp)
    need = 0
    for N in range(0, 64 * hop, hop):
        steps = N // hop - c
        for m in range(max(steps, 0)):
            assert (m | 1) * hop + n_fft // 2 <= N
        dec = [t for t in range(min(max(steps, 0), Tp)) if blocks[up[t]].max() < steps]
        assert dec == list(range(min(max(steps, 0), Tp)))  # the bottleneck never holds a frame back
        crm_frames = len(dec) - la
        x = 0
        while (x + n_fft // 2) // hop + 1 < crm_frames:
            x += 1
        need = max(need, N - x)
    return need


@pytest.mark.parametrize("la", [0, 1, 2])
@pytest.mark.parametrize("S", [2, 3])
@pytest.mark.parametrize("hop", [256, 160, 128])
def test_delay_formula_matches_emulation(S, la, hop):
    lib = _lib.load()
    d = _desc(la=la, S=S)
    D = lib.fsn_fast_stream_delay(C.byref(d), 512, hop)
    assert D == _delay_emulated(512, hop, la, S)
    assert D == 256 + (la + 1 + -(-256 // hop)) * hop


def test_queries_answer():
    lib = _lib.load()
    d = _desc()
    s1 = lib.fsn_fast_stream_state_bytes(C.byref(d), 1, 512, 256)
    s4 = lib.fsn_fast_stream_state_bytes(C.byref(d), 4, 512, 256)
    bn = 2 * 2 * 64 * 384 * 4  # bottleneck h and c of both layers, every mel row
    assert bn < s1 < bn + 48 * 1024 and s4 == 4 * s1 and s1 % 256 == 0
    w1 = lib.fsn_fast_stream_workspace_bytes(C.byref(d), 4, 1, 512, 256)
    w64 = lib.fsn_fast_stream_workspace_bytes(C.byref(d), 4, 64, 512, 256)
    assert 0 < w1 < w64
    assert lib.fsn_fast_stream_delay(C.byref(d), 512, 256) == 1280
    assert lib.fsn_fast_stream_delay(C.byref(_desc(la=1, S=3)), 512, 256) == 256 + 3 * 256


@pytest.mark.parametrize("kw,n_fft,code", [
    (dict(norm="offline_laplace_norm"), 512, _lib.FSN_ERR_UNSUPPORTED),
    (dict(norm="forgetting_norm"), 512, _lib.FSN_ERR_UNSUPPORTED),
    (dict(cell="GRU"), 512, _lib.FSN_ERR_UNSUPPORTED),
    (dict(prec="f16_tc"), 512, _lib.FSN_ERR_UNSUPPORTED),
    (dict(prec="f16x3_tc"), 512, _lib.FSN_ERR_UNSUPPORTED),
    (dict(F=481), 960, _lib.FSN_ERR_UNSUPPORTED),
    (dict(), 256, _lib.FSN_ERR_SHAPE),
])
def test_refusals_before_any_cuda_call(kw, n_fft, code):
    lib = _lib.load()
    d = _desc(**kw)
    assert lib.fsn_fast_stream_state_bytes(C.byref(d), 2, n_fft, 256) == 0
    assert lib.fsn_last_error_code() == code
    assert lib.fsn_fast_stream_workspace_bytes(C.byref(d), 2, 4, n_fft, 256) == 0
    assert lib.fsn_last_error_code() == code
    assert lib.fsn_fast_stream_delay(C.byref(d), n_fft, 256) == -code
    w = _lib.FastWeights()
    rc = lib.fsn_fast_stream_step(C.byref(d), C.byref(w), 1, None, None, 2, 4, n_fft, 256, n_fft, 1, 1, 1 << 30, 1,
                                  1 << 30, None)
    assert rc == code
    assert lib.fsn_last_launch_count() == 0


def _fast_model(**kw):
    from fullsubnet_b200.fast_fullsubnet.model import Model
    precision = kw.pop("precision", "fp32")
    return Model(**_args(**kw), precision=precision)


@pytest.mark.parametrize("precision", ["auto", "f16x3_tc", "f16_tc"])
def test_streamer_refuses_other_precisions(precision):
    from fullsubnet_b200.stream import Streamer
    with pytest.raises(NotImplementedError, match='precision="fp32"'):
        Streamer(_fast_model(precision=precision), 2)


def test_streamer_refuses_the_offline_norm():
    from fullsubnet_b200.stream import Streamer
    with pytest.raises(NotImplementedError, match="offline norm"):
        Streamer(_fast_model(norm_type="offline_laplace_norm"), 2)


def test_streamer_accepts_fast_fullsubnet():
    from fullsubnet_b200.stream import Streamer
    s = Streamer(_fast_model(), 3)
    assert s.delay == 1280
    lib = _lib.load()
    assert s.state.numel() == lib.fsn_fast_stream_state_bytes(C.byref(_desc()), 3, 512, 256)
    assert int(s.state.abs().sum()) == 0


def test_streamer_refuses_short_and_overlong_clips():
    """As for fullband_baseline: the host follows each slot's position and refuses, before the call, a clip of n_fft/2
    samples or fewer and one past the library's position limit; a restored slot (position unknown) is not checked."""
    from fullsubnet_b200.stream import Streamer
    s = Streamer(_fast_model(), 2)
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
