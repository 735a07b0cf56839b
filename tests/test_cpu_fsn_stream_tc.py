"""Chunked streaming of fullsubnet on the fp16 tensor cores (fsn_stream_tc_*) without a GPU: the delay and the state are
the fp32 stream's, the workspace grows with K_max and ignores drop_band, every refusal happens before any CUDA call
with its error code, Streamer(tensor_cores=True) takes and refuses what the library does, and the carry instantiations
of the kernels keep the stack frames and stage-loop density the built library shows."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

from fullsubnet_b200 import _lib
from test_cpu_fsn_stream import CUM, FGT, _desc, _fsn_model
from test_cpu_subband_sass import _stage_loop

TC_PRECS = ["f16x3_tc", "f16_tc"]


@pytest.mark.parametrize("la", [0, 1, 2])
@pytest.mark.parametrize("hop", [256, 160, 128])
@pytest.mark.parametrize("prec", TC_PRECS)
def test_delay_is_the_fp32_streams(prec, hop, la):
    lib = _lib.load()
    for norm in (CUM, FGT):
        D = lib.fsn_stream_tc_delay(C.byref(_desc(norm, la=la, prec=prec)), 512, hop)
        assert D == lib.fsn_stream_delay(C.byref(_desc(norm, la=la)), 512, hop) > 0


@pytest.mark.parametrize("norm", [CUM, FGT])
@pytest.mark.parametrize("prec", TC_PRECS)
def test_state_is_the_fp32_streams(norm, prec):
    lib = _lib.load()
    for hop, la in ((256, 2), (160, 1), (128, 0)):
        for B in (1, 5):
            tc = lib.fsn_stream_tc_state_bytes(C.byref(_desc(norm, la=la, prec=prec)), B, 512, hop)
            assert tc == lib.fsn_stream_state_bytes(C.byref(_desc(norm, la=la)), B, 512, hop) > 0


@pytest.mark.parametrize("prec", TC_PRECS)
def test_workspace_grows_with_k_and_ignores_drop_band(prec):
    lib = _lib.load()
    for norm in (CUM, FGT):
        w = [lib.fsn_stream_tc_workspace_bytes(C.byref(_desc(norm, prec=prec, G=G)), 3, 4, 512, 256) for G in (1, 2, 300)]
        assert w[0] > 0 and w == [w[0]] * 3
        assert w[0] < lib.fsn_stream_tc_workspace_bytes(C.byref(_desc(norm, prec=prec)), 3, 64, 512, 256)


def _tc_step(lib, d, start=None, tail=None, B=2, K=4, n_fft=512, packed=1, state_bytes=1 << 40, ws_bytes=1 << 40):
    s = (C.c_int32 * B)(*start) if start is not None else None
    t = (C.c_int32 * B)(*tail) if tail is not None else None
    fb, sb = _lib.SeqWeights(), _lib.SeqWeights()
    # non-null dummy pointers: a refusal must come before anything reads them
    return lib.fsn_stream_tc_step(C.byref(d), C.byref(fb), C.byref(sb), packed, 1, s, t, B, K, n_fft, 256, n_fft, 1, 1,
                                  state_bytes, 1, ws_bytes, None)


@pytest.mark.parametrize("kw,n_fft,code", [
    (dict(prec="fp32"), 512, _lib.FSN_ERR_UNSUPPORTED),
    (dict(norm="offline_laplace_norm", prec="f16x3_tc"), 512, _lib.FSN_ERR_UNSUPPORTED),
    (dict(cell="GRU", prec="f16x3_tc"), 512, _lib.FSN_ERR_UNSUPPORTED),
    (dict(Hs=320, prec="f16x3_tc"), 512, _lib.FSN_ERR_UNSUPPORTED),   # sb_hidden not a multiple of 128
    (dict(Hs=512, prec="f16_tc"), 512, _lib.FSN_ERR_UNSUPPORTED),     # more than 3 slices of 128
    (dict(F=481, prec="f16x3_tc"), 960, _lib.FSN_ERR_UNSUPPORTED),
    (dict(prec="f16_tc"), 256, _lib.FSN_ERR_SHAPE),
])
def test_refusals_before_any_cuda_call(kw, n_fft, code):
    lib = _lib.load()
    d = _desc(**kw)
    assert lib.fsn_stream_tc_state_bytes(C.byref(d), 2, n_fft, 256) == 0
    assert lib.fsn_last_error_code() == code
    assert lib.fsn_stream_tc_workspace_bytes(C.byref(d), 2, 4, n_fft, 256) == 0
    assert lib.fsn_last_error_code() == code
    assert lib.fsn_stream_tc_delay(C.byref(d), n_fft, 256) == -code
    assert _tc_step(lib, d, n_fft=n_fft) == code
    assert lib.fsn_last_launch_count() == 0


def test_sub_band_input_too_wide_refused():
    """The tensor-core sub band gathers at most 32 inputs per row: sb_num_neighbors = 16 makes 33 + 1."""
    lib = _lib.load()
    d = _desc(prec="f16x3_tc")
    d.sb_num_neighbors = 16
    assert lib.fsn_stream_tc_state_bytes(C.byref(d), 2, 512, 256) == 0
    assert lib.fsn_last_error_code() == _lib.FSN_ERR_UNSUPPORTED
    assert _tc_step(lib, d) == _lib.FSN_ERR_UNSUPPORTED
    assert lib.fsn_last_launch_count() == 0


@pytest.mark.parametrize("prec", TC_PRECS)
def test_null_packed_weights_refused(prec):
    lib = _lib.load()
    assert _tc_step(lib, _desc(prec=prec), packed=None) == _lib.FSN_ERR_SHAPE
    assert lib.fsn_last_launch_count() == 0


@pytest.mark.parametrize("norm", [CUM, FGT])
@pytest.mark.parametrize("precision", ["auto", "f16x3_tc", "f16_tc"])
def test_streamer_tensor_cores_accepts_fullsubnet(precision, norm):
    from fullsubnet_b200.stream import Streamer
    m = _fsn_model(precision=precision, norm_type=norm)
    s = Streamer(m, 3, tensor_cores=True)
    assert s.delay == 1280
    lib = _lib.load()
    assert s.state.numel() == lib.fsn_stream_state_bytes(C.byref(_desc(norm)), 3, 512, 256)
    assert int(s.state.abs().sum()) == 0
    # "auto" streams the precision the whole-clip call resolves to
    assert m._stream_tc_desc().precision == _lib.PREC["f16x3_tc" if precision == "auto" else precision]


def test_streamer_tensor_cores_refuses_fp32():
    from fullsubnet_b200.stream import Streamer
    with pytest.raises(NotImplementedError, match="tensor_cores=False"):
        Streamer(_fsn_model(precision="fp32"), 2, tensor_cores=True)


def test_streamer_tensor_cores_refuses_the_offline_norm():
    from fullsubnet_b200.stream import Streamer
    with pytest.raises(NotImplementedError, match="offline norm"):
        Streamer(_fsn_model(precision="f16x3_tc", norm_type="offline_laplace_norm"), 2, tensor_cores=True)


def test_streamer_tensor_cores_refuses_other_models():
    from fullsubnet_b200.stream import Streamer
    from fullsubnet_b200.fullband_baseline.model import Model as Fbb
    from oracle import fullband_baseline_oracle as BO
    from test_cpu_fast_stream import _fast_model
    for m in (Fbb(**dict(BO.DEFAULT_FBB_ARGS, norm_type=CUM)), _fast_model()):
        with pytest.raises(NotImplementedError, match="tensor_cores=True"):
            Streamer(m, 2, tensor_cores=True)


# ---------------------------------------------------------------------------------------- carry instantiations' code
SB_X3 = "_ZN3fsn2tc23sb_carry_lstm_tc_kernelILb1EEEvNS0_5KArgsE"
SB_SINGLE = "_ZN3fsn2tc23sb_carry_lstm_tc_kernelILb0EEEvNS0_5KArgsE"
REC_X3 = "_ZN3fsn3rec24lstm_rec_tc_carry_kernelILb1EEEv14CUtensorMap_stNS0_4ArgsENS0_9CarryArgsE"
REC_SINGLE = "_ZN3fsn3rec24lstm_rec_tc_carry_kernelILb0EEEv14CUtensorMap_stNS0_4ArgsENS0_9CarryArgsE"
# CUDA 12.9, sm_90a: stack frames of the built library; lower is fine, higher fails
MAX_STACK = {SB_X3: 176, SB_SINGLE: 48, REC_X3: 0, REC_SINGLE: 0}
# instructions per HGMMA over the stage loop (8.3 / 8.4; the production kernels 7.8 / 8.4)
MAX_PER_HGMMA = {SB_X3: 8.5, SB_SINGLE: 8.5}


def _tool_and_lib():
    tool = next((c for c in (shutil.which("cuobjdump"), "/usr/local/cuda/bin/cuobjdump") if c and os.path.exists(c)), None)
    if tool is None:
        pytest.skip("no cuobjdump")
    if not os.path.exists(_lib.LIB_PATH):
        from fullsubnet_b200.csrc.build import build
        build()
    return tool, _lib.LIB_PATH


def test_carry_kernels_keep_their_stack_frames():
    tool, lib = _tool_and_lib()
    out = subprocess.run([tool, "--dump-resource-usage", lib], capture_output=True, text=True, check=True).stdout
    usage = dict(re.findall(r"Function (\S+):\s*\n\s*REG:\d+ STACK:(\d+)", out))
    for fn, limit in MAX_STACK.items():
        assert fn in usage, f"{fn} not found in the library"
        assert int(usage[fn]) <= limit, f"{fn}: {usage[fn]}-byte stack frame, at most {limit} expected"


@pytest.mark.parametrize("fn", [SB_X3, SB_SINGLE], ids=["f16x3_tc", "f16_tc"])
def test_carry_stage_loop_density(fn):
    tool, lib = _tool_and_lib()
    stages = _stage_loop(tool, lib, fn)
    assert stages, f"{fn}: no stage loop found"
    body = [s for st in stages for s in st]
    n_mma = sum(s.startswith("HGMMA") for s in body)
    assert n_mma > 0
    assert not [s for s in body if re.match(r"(@!?U?P\w+\s+)?(S2R|BSSY)\b", s)]
    per = len(body) / n_mma
    assert per <= MAX_PER_HGMMA[fn], f"{fn}: {per:.2f} instructions per HGMMA in the stage loop"
