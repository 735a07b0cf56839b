"""The two-pass sub-band stack (sb_l0_tc_kernel / sb_l1_tc_kernel) without a GPU: the stack frames of the built
kernels (cuobjdump --dump-resource-usage), the size of its h0 hand-over buffer, and its hook's argument checks.

Each consumer warpgroup of the two-pass kernels holds 4 x 24 accumulators and one layer's 24 cell states at 48 rows
(setmaxnreg: 152 registers, 160 in x3 layer 1).  With CUDA 12.9 for sm_90a the single pass does not spill; x3 has an
8-byte frame in layer 0 and 72 bytes in layer 1, whose spill loads all sit after the step's MMAs (once per step, none
in the stage loop).  A growth of these frames is a performance regression like that of the fused kernel's
(test_cpu_subband_resources.py)."""
from __future__ import annotations

import ctypes as C
import os
import re
import subprocess

import pytest

from test_cpu_subband_resources import _cuobjdump

# frame sizes of CUDA 12.9 for sm_90a; lower is fine, higher fails
MAX_STACK = {"_ZN3fsn2tc15sb_l0_tc_kernelILb1EEEvNS0_9SplitArgsE": 8,     # f16x3_tc, layer 0
             "_ZN3fsn2tc15sb_l0_tc_kernelILb0EEEvNS0_9SplitArgsE": 0,     # f16_tc, layer 0
             "_ZN3fsn2tc15sb_l1_tc_kernelILb1EEEvNS0_9SplitArgsE": 72,    # f16x3_tc, layer 1
             "_ZN3fsn2tc15sb_l1_tc_kernelILb0EEEvNS0_9SplitArgsE": 0}     # f16_tc, layer 1


def _lib():
    from fullsubnet_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        from fullsubnet_b200.csrc.build import build
        build()
    return _lib


def test_two_pass_kernels_keep_their_stack_frames():
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("no cuobjdump")
    out = subprocess.run([tool, "--dump-resource-usage", _lib().LIB_PATH], capture_output=True, text=True,
                         check=True).stdout
    usage = dict(re.findall(r"Function (\S+):\s*\n\s*REG:\d+ STACK:(\d+)", out))
    for fn, limit in MAX_STACK.items():
        assert fn in usage, f"{fn} not found in the library"
        assert int(usage[fn]) <= limit, f"{fn}: {usage[fn]}-byte stack frame, at most {limit} expected (spills grew)"


def test_h0_buffer_size():
    lib = _lib().load()
    # one pair's image per step: hi and lo k-blocks of 48 rows x H units (x3), hi only in the single pass
    assert lib.fsn_debug_sb_lstm_tc2_ws_bytes(48, 1, 384, 1, 0) == 48 * 384 * 4
    assert lib.fsn_debug_sb_lstm_tc2_ws_bytes(48, 1, 384, 0, 0) == 48 * 384 * 2
    assert lib.fsn_debug_sb_lstm_tc2_ws_bytes(49, 10, 128, 1, 0) == 2 * 10 * 48 * 128 * 4
    # rows beyond one chunk reuse the buffer: configs[1] (256 clips x 257 bins, 253 steps) holds 132 pairs, 2.46 GB
    assert lib.fsn_debug_sb_lstm_tc2_ws_bytes(256 * 257, 253, 384, 1, 0) == 132 * 253 * 48 * 384 * 4
    assert lib.fsn_debug_sb_lstm_tc2_ws_bytes(256 * 257, 253, 384, 1, 7) == 7 * 253 * 48 * 384 * 4
    assert lib.fsn_debug_sb_lstm_tc2_ws_bytes(48, 1, 192, 1, 0) == 0


def test_hook_rejects_bad_arguments_before_any_cuda_call():
    _l = _lib()
    lib = _l.load()
    s = _l.SeqWeights()
    p = C.c_void_p(16)

    def call(H=384, act=0, B=3, G=2, la=2, steps=10, stages=0, chunk=0, ws=p):
        return lib.fsn_debug_sb_lstm_tc2(C.byref(s), H, 15, 0, act, 1, p, p, B, 33, 10, G, p, None, la, steps, stages,
                                         chunk, p, ws, p, None)

    SH, UN = _l.FSN_ERR_SHAPE, _l.FSN_ERR_UNSUPPORTED
    for kw, code in ((dict(H=192), UN), (dict(act=7), SH), (dict(B=2, G=2), SH), (dict(la=10), SH),
                     (dict(steps=11), SH), (dict(stages=5), UN), (dict(stages=1), UN), (dict(chunk=-1), SH),
                     (dict(ws=None), SH)):
        assert call(**kw) == code, kw
        assert lib.fsn_last_error_code() == code, kw
