"""Chunked streaming of fullsubnet without a GPU: the delay is fullband_baseline's, the state holds the layout computed
from the model's shapes, every refusal happens before any CUDA call with its error code, and the Streamer refuses what
the library cannot stream."""
import ctypes as C

import pytest

from fullsubnet_b200 import _lib

CUM, FGT = "cumulative_laplace_norm", "forgetting_norm"
NORM = {"offline_laplace_norm": 0, CUM: 1, FGT: 4}


def _desc(norm=CUM, la=2, cell="LSTM", prec="fp32", F=257, Hs=384, G=2):
    return _lib.ModelDesc(num_freqs=F, look_ahead=la, fb_num_neighbors=0, sb_num_neighbors=15, fb_hidden=512,
                          sb_hidden=Hs, fb_activation=_lib.ACT["ReLU"], sb_activation=_lib.ACT[False],
                          norm_type=NORM[norm], num_groups_in_drop_band=G, precision=_lib.PREC[prec],
                          cell_type=_lib.CELL[cell])


def _fbb_desc(la):
    return _lib.FullbandDesc(num_freqs=257, hidden=512, num_layers=3, look_ahead=la, activation=0, norm_type=1,
                             precision=_lib.PREC["fp32"], cell_type=_lib.CELL["LSTM"])


@pytest.mark.parametrize("la", [0, 1, 2])
@pytest.mark.parametrize("hop", [256, 160, 128])
def test_delay_is_fullband_baselines(hop, la):
    """The sub band adds no delay: frame t's cRM comes from step t + look_ahead as in fullband_baseline, whose delay
    tests/test_cpu_stream.py checks against an emulation of the schedule."""
    lib = _lib.load()
    D = lib.fsn_stream_delay(C.byref(_desc(la=la)), 512, hop)
    assert D == 256 + (la + 1 + -(-256 // hop)) * hop
    assert D == lib.fsn_fullband_stream_delay(C.byref(_fbb_desc(la)), 512, hop)
    assert lib.fsn_stream_delay(C.byref(_desc(FGT, la=la)), 512, hop) == D


def _align(x, a):
    return -(-x // a) * a


def _slot_bytes(norm, n_fft, hop, la, F=257, Hf=512, Hs=384):
    """meta, sample history, spectrum and cRM frames (fullband_baseline's sections), the second norm's accumulator,
    full-band (h | c), sub-band (h | c) of every frequency; 16-byte sections, 256-byte blocks"""
    c = -(-(n_fft // 2) // hop)
    Rc = -(-n_fft // hop) + 2
    floats = [(c + 1) * hop + n_fft // 2, (Rc + la) * 2 * F, Rc * 2 * F, F if norm == CUM else 1,
              2 * Hf, 2 * Hf, 2 * F * Hs, 2 * F * Hs]
    o = 16
    for n in floats:
        o = _align(o + 4 * n, 16)
    return _align(o, 256)


@pytest.mark.parametrize("norm", [CUM, FGT])
@pytest.mark.parametrize("hop,la", [(256, 2), (160, 1), (128, 0)])
def test_state_bytes_match_layout(norm, hop, la):
    lib = _lib.load()
    d = _desc(norm, la=la)
    s1 = lib.fsn_stream_state_bytes(C.byref(d), 1, 512, hop)
    assert s1 == _slot_bytes(norm, 512, hop, la)
    assert lib.fsn_stream_state_bytes(C.byref(d), 5, 512, hop) == 5 * s1
    if (norm, hop, la) == (CUM, 256, 2):  # the recipe: the sub-band rows are 1.58 MB of 1.61 MB
        assert s1 == 1612032 and 2 * 2 * 257 * 384 * 4 == 1579008


def test_queries_answer_and_ignore_drop_band():
    """Every slot is a B = 1 clip: num_groups_in_drop_band changes nothing."""
    lib = _lib.load()
    for norm in (CUM, FGT):
        d1, d2, d9 = _desc(norm, G=1), _desc(norm, G=2), _desc(norm, G=300)
        s = [lib.fsn_stream_state_bytes(C.byref(d), 3, 512, 256) for d in (d1, d2, d9)]
        w = [lib.fsn_stream_workspace_bytes(C.byref(d), 3, 4, 512, 256) for d in (d1, d2, d9)]
        assert s[0] > 0 and s == [s[0]] * 3 and w[0] > 0 and w == [w[0]] * 3
        w64 = lib.fsn_stream_workspace_bytes(C.byref(d1), 3, 64, 512, 256)
        assert w[0] < w64
        assert lib.fsn_stream_delay(C.byref(d9), 512, 256) == 1280


@pytest.mark.parametrize("kw,n_fft,code", [
    (dict(norm="offline_laplace_norm"), 512, _lib.FSN_ERR_UNSUPPORTED),
    (dict(cell="GRU"), 512, _lib.FSN_ERR_UNSUPPORTED),
    (dict(prec="f16_tc"), 512, _lib.FSN_ERR_UNSUPPORTED),
    (dict(prec="f16x3_tc"), 512, _lib.FSN_ERR_UNSUPPORTED),
    (dict(norm=FGT, prec="f16x3_tc"), 512, _lib.FSN_ERR_UNSUPPORTED),
    (dict(F=481), 960, _lib.FSN_ERR_UNSUPPORTED),
    (dict(), 256, _lib.FSN_ERR_SHAPE),
])
def test_refusals_before_any_cuda_call(kw, n_fft, code):
    lib = _lib.load()
    d = _desc(**kw)
    assert lib.fsn_stream_state_bytes(C.byref(d), 2, n_fft, 256) == 0
    assert lib.fsn_last_error_code() == code
    assert lib.fsn_stream_workspace_bytes(C.byref(d), 2, 4, n_fft, 256) == 0
    assert lib.fsn_last_error_code() == code
    assert lib.fsn_stream_delay(C.byref(d), n_fft, 256) == -code
    fb, sb = _lib.SeqWeights(), _lib.SeqWeights()
    rc = lib.fsn_stream_step(C.byref(d), C.byref(fb), C.byref(sb), 1, None, None, 2, 4, n_fft, 256, n_fft, 1, 1, 1 << 40,
                             1, 1 << 40, None)
    assert rc == code
    assert lib.fsn_last_launch_count() == 0


def _step(lib, d, start=None, tail=None, B=2, K=4, state_bytes=1 << 40, ws_bytes=1 << 40):
    s = (C.c_int32 * B)(*start) if start is not None else None
    t = (C.c_int32 * B)(*tail) if tail is not None else None
    fb, sb = _lib.SeqWeights(), _lib.SeqWeights()
    # non-null dummy pointers: a refusal must come before anything reads them
    return lib.fsn_stream_step(C.byref(d), C.byref(fb), C.byref(sb), 1, s, t, B, K, 512, 256, 512, 1, 1, state_bytes, 1,
                               ws_bytes, None)


def test_too_many_sub_band_rows_refused():
    """B x F x sb_hidden elements of sub-band state must stay int-indexable: 21 760 slots of the recipe fit, 21 761 not."""
    lib = _lib.load()
    assert 21760 * 257 * 384 < 2 ** 31 <= 21761 * 257 * 384
    assert _step(lib, _desc(), B=21761) == _lib.FSN_ERR_SHAPE
    assert lib.fsn_last_launch_count() == 0


def _fsn_model(**kw):
    from fullsubnet_b200.fullsubnet.model import Model
    from oracle import fullsubnet_oracle as O
    precision = kw.pop("precision", "fp32")
    return Model(**dict(O.DEFAULT_MODEL_ARGS, **dict(dict(norm_type=CUM), **kw)), precision=precision)


@pytest.mark.parametrize("norm", [CUM, FGT])
@pytest.mark.parametrize("precision", ["auto", "f16x3_tc", "f16_tc"])
def test_streamer_refuses_other_precisions(precision, norm):
    from fullsubnet_b200.stream import Streamer
    with pytest.raises(NotImplementedError, match='precision="fp32"'):
        Streamer(_fsn_model(precision=precision, norm_type=norm), 2)


def test_streamer_refuses_the_offline_norm():
    from fullsubnet_b200.stream import Streamer
    with pytest.raises(NotImplementedError, match="offline norm"):
        Streamer(_fsn_model(norm_type="offline_laplace_norm"), 2)


@pytest.mark.parametrize("norm", [CUM, FGT])
def test_streamer_accepts_fullsubnet(norm):
    from fullsubnet_b200.stream import Streamer
    s = Streamer(_fsn_model(norm_type=norm), 3)
    assert s.delay == 1280
    lib = _lib.load()
    assert s.state.numel() == lib.fsn_stream_state_bytes(C.byref(_desc(norm)), 3, 512, 256)
    assert int(s.state.abs().sum()) == 0
