"""Instruction stream of the production sub-band kernels' stage loop in the built library (cuobjdump -sass, no GPU).

One consumer warpgroup issues the MMAs of a ring stage while the others wait for their turn, so the instructions it
issues per stage sit on the critical path.  With descriptors rebuilt per MMA in vector registers and moved over with
R2UR, per-stage S2R / LDC re-reads and divergent (BSSY) regions around the waits and arrives, the stage loop issued
14-22 instructions per HGMMA and the headline step was about 17 % slower at the same MMAs (DESIGN 4.1).  The stage
loop is taken as the instructions between consecutive `WARPGROUP.DEPBAR.LE gsb0, 0x1` (one per ring stage)."""
from __future__ import annotations

import os
import re
import shutil
import subprocess

import pytest

X3 = "_ZN3fsn2tc17sb_lstm_tc_kernelILb1ELb0EEEvNS0_5KArgsE"      # f16x3_tc
SINGLE = "_ZN3fsn2tc17sb_lstm_tc_kernelILb0ELb0EEEvNS0_5KArgsE"  # f16_tc
# CUDA 12.9, sm_90a: 7.8 (x3) and 8.4 (single pass) instructions per HGMMA over the stage loop; 14.4 / 22.5 before
MAX_PER_HGMMA = {X3: 9.0, SINGLE: 10.0}


def _cuobjdump():
    for c in (shutil.which("cuobjdump"), "/usr/local/cuda/bin/cuobjdump"):
        if c and os.path.exists(c):
            return c
    return None


def _stage_loop(tool, lib, fn):
    out = subprocess.run([tool, "-sass", "-fun", fn, lib], capture_output=True, text=True, check=True).stdout
    ins = [m.group(1).strip() for m in re.finditer(r"/\*[0-9a-f]{4,}\*/\s+([^;]*);", out)]
    marks = [i for i, s in enumerate(ins) if re.search(r"WARPGROUP\.DEPBAR\.LE\s+gsb0,\s*0x1\b", s)]
    return [ins[a + 1:b + 1] for a, b in zip(marks, marks[1:])]


@pytest.mark.parametrize("fn", [X3, SINGLE], ids=["f16x3_tc", "f16_tc"])
def test_stage_loop_issues_few_instructions_per_mma(fn):
    from fullsubnet_b200 import _lib
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("no cuobjdump")
    if not os.path.exists(_lib.LIB_PATH):
        from fullsubnet_b200.csrc.build import build
        build()
    stages = _stage_loop(tool, _lib.LIB_PATH, fn)
    assert stages, f"{fn}: no stage loop found"
    body = [s for st in stages for s in st]
    n_mma = sum(s.startswith("HGMMA") for s in body)
    n_r2ur = sum(s.startswith("R2UR") for s in body)
    assert n_mma > 0
    for op in ("S2R", "LDC", "BSSY"):
        hits = [s for s in body if re.match(rf"(@!?U?P\w+\s+)?{op}\b", s)]
        assert not hits, f"{fn}: {op} in the stage loop: {hits[:3]}"
    assert n_r2ur <= n_mma, f"{fn}: {n_r2ur} R2UR for {n_mma} HGMMA in the stage loop (descriptors built per MMA)"
    per = len(body) / n_mma
    assert per <= MAX_PER_HGMMA[fn], f"{fn}: {per:.1f} instructions per HGMMA in the stage loop"
