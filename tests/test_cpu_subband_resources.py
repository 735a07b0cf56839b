"""Stack frames of the production sub-band kernels in the built library (cuobjdump --dump-resource-usage, no GPU).

The x3 kernel's consumers need nearly all of their registers, so its local-memory spill traffic is a large share of
the headline step: taking the kernel arguments as a plain by-value struct (every field held in a register from kernel
entry) grew the x3 frame from 48 to 184 bytes and cost about 17 % of the step (DESIGN 4.1).  A growth of these frames
is a performance regression even when every result stays bit-identical."""
from __future__ import annotations

import os
import re
import shutil
import subprocess

import pytest

# frame sizes of CUDA 12.9 for sm_90a; lower is fine, higher fails
MAX_STACK = {"_ZN3fsn2tc17sb_lstm_tc_kernelILb1ELb0EEEvNS0_5KArgsE": 48,   # f16x3_tc
             "_ZN3fsn2tc17sb_lstm_tc_kernelILb0ELb0EEEvNS0_5KArgsE": 0}    # f16_tc


def _cuobjdump():
    for c in (shutil.which("cuobjdump"), "/usr/local/cuda/bin/cuobjdump"):
        if c and os.path.exists(c):
            return c
    return None


def test_production_subband_kernels_keep_their_stack_frames():
    from fullsubnet_b200 import _lib
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("no cuobjdump")
    if not os.path.exists(_lib.LIB_PATH):
        from fullsubnet_b200.csrc.build import build
        build()
    out = subprocess.run([tool, "--dump-resource-usage", _lib.LIB_PATH], capture_output=True, text=True,
                         check=True).stdout
    usage = dict(re.findall(r"Function (\S+):\s*\n\s*REG:\d+ STACK:(\d+)", out))
    for fn, limit in MAX_STACK.items():
        assert fn in usage, f"{fn} not found in the library"
        assert int(usage[fn]) <= limit, f"{fn}: {usage[fn]}-byte stack frame, at most {limit} expected (spills grew)"
