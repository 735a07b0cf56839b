"""Chunked streaming of fast_fullsubnet on the fp16 tensor cores (fsn_fast_stream_tc_*) without a GPU: the delay and the
state are the fp32 stream's, the workspace grows with K_max, every refusal happens before any CUDA call with its error
code, Streamer(tensor_cores=True) takes and refuses what the library does, and the block-phased instantiation of the
bottleneck kernel keeps the stack frames and stage-loop density the built library shows."""
import ctypes as C
import re
import subprocess

import pytest

from fullsubnet_b200 import _lib
from test_cpu_fast_stream import _desc, _fast_model
from test_cpu_fsn_stream_tc import _tool_and_lib
from test_cpu_subband_sass import _stage_loop

TC_PRECS = ["f16x3_tc", "f16_tc"]


@pytest.mark.parametrize("S", [2, 3])
@pytest.mark.parametrize("la", [0, 1, 2])
@pytest.mark.parametrize("hop", [256, 160, 128])
@pytest.mark.parametrize("prec", TC_PRECS)
def test_delay_is_the_fp32_streams(prec, hop, la, S):
    lib = _lib.load()
    D = lib.fsn_fast_stream_tc_delay(C.byref(_desc(la=la, S=S, prec=prec)), 512, hop)
    assert D == lib.fsn_fast_stream_delay(C.byref(_desc(la=la, S=S)), 512, hop) > 0


@pytest.mark.parametrize("prec", TC_PRECS)
def test_state_is_the_fp32_streams(prec):
    lib = _lib.load()
    for hop in (256, 160, 128):
        for la in (0, 1, 2):
            for S in (2, 3):
                for B in (1, 5):
                    tc = lib.fsn_fast_stream_tc_state_bytes(C.byref(_desc(la=la, S=S, prec=prec)), B, 512, hop)
                    assert tc == lib.fsn_fast_stream_state_bytes(C.byref(_desc(la=la, S=S)), B, 512, hop) > 0


@pytest.mark.parametrize("prec", TC_PRECS)
def test_workspace_grows_with_k(prec):
    lib = _lib.load()
    d = _desc(prec=prec)
    w = [lib.fsn_fast_stream_tc_workspace_bytes(C.byref(d), 3, K, 512, 256) for K in (1, 4, 64)]
    assert 0 < w[0] < w[1] < w[2]
    assert lib.fsn_fast_stream_tc_delay(C.byref(d), 512, 256) == 1280


def _tc_step(lib, d, packed=1, n_fft=512, B=2, K=4):
    w = _lib.FastWeights()
    w.bn_packed = packed
    # non-null dummy pointers: a refusal must come before anything reads them
    return lib.fsn_fast_stream_tc_step(C.byref(d), C.byref(w), 1, None, None, B, K, n_fft, 256, n_fft, 1, 1, 1 << 40, 1,
                                       1 << 40, None)


def _wide():
    d = _desc(prec="f16x3_tc")
    d.noisy_num_neighbors = 15  # 31 + 1 = 32 inputs fit; 31 + 3 do not
    d.enc_num_neighbors = 1
    return d


def _bn(**kw):
    d = _desc(prec="f16_tc")
    for k, v in kw.items():
        setattr(d, k, v)
    return d


@pytest.mark.parametrize("d,n_fft,code", [
    (_desc(prec="fp32"), 512, _lib.FSN_ERR_UNSUPPORTED),
    (_desc(norm="offline_laplace_norm", prec="f16x3_tc"), 512, _lib.FSN_ERR_UNSUPPORTED),
    (_desc(norm="forgetting_norm", prec="f16x3_tc"), 512, _lib.FSN_ERR_UNSUPPORTED),
    (_desc(cell="GRU", prec="f16x3_tc"), 512, _lib.FSN_ERR_UNSUPPORTED),
    (_bn(bn_hidden=256), 512, _lib.FSN_ERR_UNSUPPORTED),
    (_bn(bn_layers=3), 512, _lib.FSN_ERR_UNSUPPORTED),
    (_wide(), 512, _lib.FSN_ERR_UNSUPPORTED),
    (_desc(F=481, prec="f16x3_tc"), 960, _lib.FSN_ERR_UNSUPPORTED),
    (_desc(prec="f16_tc"), 256, _lib.FSN_ERR_SHAPE),
], ids=["fp32", "offline", "forgetting", "gru", "bn_hidden", "bn_layers", "width", "n_fft960", "n_fft256"])
def test_refusals_before_any_cuda_call(d, n_fft, code):
    lib = _lib.load()
    assert lib.fsn_fast_stream_tc_state_bytes(C.byref(d), 2, n_fft, 256) == 0
    assert lib.fsn_last_error_code() == code
    assert lib.fsn_fast_stream_tc_workspace_bytes(C.byref(d), 2, 4, n_fft, 256) == 0
    assert lib.fsn_last_error_code() == code
    assert lib.fsn_fast_stream_tc_delay(C.byref(d), n_fft, 256) == -code
    assert _tc_step(lib, d, n_fft=n_fft) == code
    assert lib.fsn_last_launch_count() == 0


def test_input_width_32_accepted():
    lib = _lib.load()
    d = _wide()
    d.enc_num_neighbors = 0
    assert lib.fsn_fast_stream_tc_state_bytes(C.byref(d), 2, 512, 256) > 0


@pytest.mark.parametrize("prec", TC_PRECS)
def test_null_packed_weights_refused(prec):
    lib = _lib.load()
    assert _tc_step(lib, _desc(prec=prec), packed=None) == _lib.FSN_ERR_SHAPE
    assert lib.fsn_last_launch_count() == 0


@pytest.mark.parametrize("prec", TC_PRECS)
def test_too_many_slots_and_small_buffers_refused(prec):
    lib = _lib.load()
    assert _tc_step(lib, _desc(prec=prec), B=65536) == _lib.FSN_ERR_UNSUPPORTED
    assert lib.fsn_last_launch_count() == 0
    w = _lib.FastWeights()
    w.bn_packed = 1
    d = _desc(prec=prec)
    assert lib.fsn_fast_stream_tc_step(C.byref(d), C.byref(w), 1, None, None, 2, 4, 512, 256, 512, 1, 1, 16, 1, 1 << 40,
                                       None) == _lib.FSN_ERR_WORKSPACE
    assert lib.fsn_last_launch_count() == 0


@pytest.mark.parametrize("precision", ["auto", "f16x3_tc", "f16_tc"])
def test_streamer_tensor_cores_accepts_fast_fullsubnet(precision):
    from fullsubnet_b200.stream import Streamer
    m = _fast_model(precision=precision)
    s = Streamer(m, 3, tensor_cores=True)
    assert s.delay == 1280
    lib = _lib.load()
    assert s.state.numel() == lib.fsn_fast_stream_state_bytes(C.byref(_desc()), 3, 512, 256)
    assert int(s.state.abs().sum()) == 0
    # "auto" streams the precision the whole-clip call resolves to
    assert m._stream_tc_desc().precision == _lib.PREC["f16x3_tc" if precision == "auto" else precision]


def test_streamer_tensor_cores_refuses_fp32():
    from fullsubnet_b200.stream import Streamer
    with pytest.raises(NotImplementedError, match="tensor_cores=False"):
        Streamer(_fast_model(precision="fp32"), 2, tensor_cores=True)


def test_streamer_tensor_cores_refuses_the_offline_norm():
    from fullsubnet_b200.stream import Streamer
    with pytest.raises(NotImplementedError, match="offline norm"):
        Streamer(_fast_model(precision="f16x3_tc", norm_type="offline_laplace_norm"), 2, tensor_cores=True)


def test_streamer_without_tensor_cores_still_needs_fp32():
    from fullsubnet_b200.stream import Streamer
    for precision in ("auto", "f16x3_tc", "f16_tc"):
        with pytest.raises(NotImplementedError, match='precision="fp32"'):
            Streamer(_fast_model(precision=precision), 2)


# ------------------------------------------------------------------------------- block-phased instantiation's code
PH_X3 = "_ZN3fsn2tc24sb_phased_lstm_tc_kernelILb1EEEvNS0_5KArgsE"
PH_SINGLE = "_ZN3fsn2tc24sb_phased_lstm_tc_kernelILb0EEEvNS0_5KArgsE"
# CUDA 12.9, sm_90a: stack frames of the built library (sb_carry_lstm_tc_kernel: 176 / 48); lower is fine, higher fails
MAX_STACK = {PH_X3: 184, PH_SINGLE: 0}
# instructions per HGMMA over the stage loop (8.30 / 8.45; sb_carry_lstm_tc_kernel 8.3 / 8.4)
MAX_PER_HGMMA = {PH_X3: 8.5, PH_SINGLE: 8.5}


def test_phased_kernels_keep_their_stack_frames():
    tool, lib = _tool_and_lib()
    out = subprocess.run([tool, "--dump-resource-usage", lib], capture_output=True, text=True, check=True).stdout
    usage = dict(re.findall(r"Function (\S+):\s*\n\s*REG:\d+ STACK:(\d+)", out))
    for fn, limit in MAX_STACK.items():
        assert fn in usage, f"{fn} not found in the library"
        assert int(usage[fn]) <= limit, f"{fn}: {usage[fn]}-byte stack frame, at most {limit} expected"


@pytest.mark.parametrize("fn", [PH_X3, PH_SINGLE], ids=["f16x3_tc", "f16_tc"])
def test_phased_stage_loop_density(fn):
    tool, lib = _tool_and_lib()
    stages = _stage_loop(tool, lib, fn)
    assert stages, f"{fn}: no stage loop found"
    body = [s for st in stages for s in st]
    n_mma = sum(s.startswith("HGMMA") for s in body)
    assert n_mma > 0
    assert not [s for s in body if re.match(r"(@!?U?P\w+\s+)?(S2R|BSSY)\b", s)]
    per = len(body) / n_mma
    assert per <= MAX_PER_HGMMA[fn], f"{fn}: {per:.2f} instructions per HGMMA in the stage loop"
