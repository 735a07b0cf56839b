"""The call checks every chunked streaming step shares (stream_check / stream_check_sizes in fsn_stream.cu), without a
GPU, on the four step entry points: each refusal comes before any CUDA call with its error code.  The refusals by
descriptor and the model-specific argument checks are in each model's stream test file."""
import ctypes as C

import pytest

from fullsubnet_b200 import _lib
from test_cpu_fast_stream import _desc as _fast_desc
from test_cpu_fsn_stream import CUM, FGT, _desc as _fsn_desc
from test_cpu_stream import _desc as _fbb_desc

ENTRIES = ["fullband", "fast", "fsn", "fsn_tc"]
PREFIX = {"fullband": "fsn_fullband_stream", "fast": "fsn_fast_stream", "fsn": "fsn_stream", "fsn_tc": "fsn_stream_tc"}
# every descriptor each entry point streams: the norms it takes, and both precisions of the tensor-core stream
CONFIGS = [("fullband", CUM, "fp32"), ("fullband", FGT, "fp32"), ("fast", CUM, "fp32"), ("fsn", CUM, "fp32"),
           ("fsn", FGT, "fp32"), ("fsn_tc", CUM, "f16x3_tc"), ("fsn_tc", FGT, "f16x3_tc"), ("fsn_tc", CUM, "f16_tc"),
           ("fsn_tc", FGT, "f16_tc")]


def _desc(entry, norm=CUM, prec=None):
    if entry == "fullband":
        return _fbb_desc(norm)
    if entry == "fast":
        return _fast_desc(norm)
    return _fsn_desc(norm, prec=prec or ("f16x3_tc" if entry == "fsn_tc" else "fp32"))


def _weights(entry):
    """Non-null dummy weight arguments of each entry point: a refusal must come before anything reads them."""
    if entry == "fullband":
        return (1, 1, 1)
    if entry == "fast":
        return (C.byref(_lib.FastWeights()),)
    fb, sb = _lib.SeqWeights(), _lib.SeqWeights()
    return (C.byref(fb), C.byref(sb)) + ((1,) if entry == "fsn_tc" else ())


def _step(entry, d, start=None, tail=None, B=2, K=4, wav=1, out=1, state_bytes=1 << 40, ws_bytes=1 << 40):
    s = (C.c_int32 * B)(*start) if start is not None else None
    t = (C.c_int32 * B)(*tail) if tail is not None else None
    fn = getattr(_lib.load(), PREFIX[entry] + "_step")
    return fn(C.byref(d), *_weights(entry), wav, s, t, B, K, 512, 256, 512, out, 1, state_bytes, 1, ws_bytes, None)


def _refused(rc, code):
    assert rc == code
    assert _lib.load().fsn_last_launch_count() == 0


@pytest.mark.parametrize("tail", [[-2, -1], [0, 4 * 256 + 1]])
@pytest.mark.parametrize("entry", ENTRIES)
def test_tail_out_of_range_refused(entry, tail):
    _refused(_step(entry, _desc(entry), [1, 1], tail), _lib.FSN_ERR_SHAPE)


@pytest.mark.parametrize("entry", ENTRIES)
def test_zero_hops_refused(entry):
    _refused(_step(entry, _desc(entry), K=0), _lib.FSN_ERR_SHAPE)


@pytest.mark.parametrize("entry", ENTRIES)
def test_position_limit_refused(entry):
    """A call's end position K*hop + D must stay below 2^30 samples: the fewest hops that reach it are refused."""
    d = _desc(entry)
    D = getattr(_lib.load(), PREFIX[entry] + "_delay")(C.byref(d), 512, 256)
    assert D > 0
    _refused(_step(entry, d, K=-(-(2 ** 30 - D) // 256)), _lib.FSN_ERR_SHAPE)


@pytest.mark.parametrize("which", ["chunk", "output"])
@pytest.mark.parametrize("entry", ENTRIES)
def test_null_chunk_or_output_refused(entry, which):
    null = dict(wav=None) if which == "chunk" else dict(out=None)
    _refused(_step(entry, _desc(entry), **null), _lib.FSN_ERR_SHAPE)


@pytest.mark.parametrize("entry,norm,prec", CONFIGS)
def test_small_state_or_workspace_refused(entry, norm, prec):
    lib = _lib.load()
    d = _desc(entry, norm, prec)
    need_s = getattr(lib, PREFIX[entry] + "_state_bytes")(C.byref(d), 2, 512, 256)
    need_w = getattr(lib, PREFIX[entry] + "_workspace_bytes")(C.byref(d), 2, 4, 512, 256)
    assert need_s > 0 and need_w > 0
    _refused(_step(entry, d, state_bytes=need_s - 1), _lib.FSN_ERR_WORKSPACE)
    _refused(_step(entry, d, ws_bytes=need_w - 1), _lib.FSN_ERR_WORKSPACE)


@pytest.mark.parametrize("entry", ENTRIES)
def test_too_many_slots_refused(entry):
    """B = 65536 is FSN_ERR_UNSUPPORTED, also for fullsubnet, where it breaks the sub-band row bound (FSN_ERR_SHAPE) too."""
    _refused(_step(entry, _desc(entry), [0] * 65536, B=65536), _lib.FSN_ERR_UNSUPPORTED)
