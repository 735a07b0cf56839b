"""improved_fullsubnet's fp16 tensor-core precisions without a GPU: the C ABI answers the workspace and packed-image
queries, refuses what is not built (training on f16, bad section indices, sub-band sizes the kernel lacks) before any
CUDA call, the model resolves its precisions, and the section kernel's stage loop stays free of GPU-scope fences."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

PROJ_KERNELS = {"_ZN3fsn2tc22sb_proj_lstm_tc_kernelILb1EEEvNS0_5KArgsE": "f16x3_tc",
                "_ZN3fsn2tc22sb_proj_lstm_tc_kernelILb0EEEvNS0_5KArgsE": "f16_tc"}


def _lib():
    from fullsubnet_b200 import _lib as L
    return L, L.load()


def _desc(args, precision):
    from fullsubnet_b200.improved_fullsubnet.model import Model
    return Model(**args)._desc(precision)


def _variants():
    from oracle import improved_fullsubnet_oracle as IO
    return {"k16": IO.DEFAULT_IMPROVED_ARGS, "k48": IO.ARGS_48K_1024, "k48_960": IO.ARGS_48K_960}


def test_abi_version_and_entry_points():
    L, lib = _lib()
    assert lib.fsn_version() == 102  # sb_packed is read only by precisions an older caller never selects
    for name in ("fsn_improved_packed_bytes", "fsn_improved_pack_sb_weights", "fsn_debug_imp_section_lstm_tc",
                 "fsn_debug_imp_section_lstm_tc_workspace_bytes"):
        assert hasattr(lib, name)
    assert C.sizeof(L.ImprovedWeights) == C.sizeof(L.SeqWeights) * (1 + L.IMP_MAX_SECTIONS) + 8 * L.IMP_MAX_SECTIONS


@pytest.mark.parametrize("tag", ["k16", "k48", "k48_960"])
def test_workspace_and_packed_size_queries(tag):
    L, lib = _lib()
    args = _variants()[tag]
    sr = 16000 if tag == "k16" else 48000
    ws = {p: lib.fsn_improved_workspace_bytes(C.byref(_desc(args, p)), 64, 10 * sr)
          for p in ("fp32", "tf32_tc", "f16x3_tc", "f16_tc")}
    assert all(v > 0 for v in ws.values()), ws
    # the f16 sections keep P and h1 of every step, not tf32_tc's gates, cell and hidden states of both layers
    assert ws["f16_tc"] < ws["f16x3_tc"] < ws["tf32_tc"], ws
    for p in ("f16x3_tc", "f16_tc"):
        e = lib.fsn_improved_enhance_workspace_bytes(C.byref(_desc(args, p)), 64, 10 * sr)
        assert e >= ws[p]
    # packed image per section: [hi (+ lo)] fp16 tiles of W_hh0 (4H x H), W_ih1 and W_hh1 for both halves, + biases
    H = args["sb_hidden_size"]
    for p, parts in (("f16x3_tc", 2), ("f16_tc", 1)):
        d = _desc(args, p)
        for s in range(d.num_sections):
            n = lib.fsn_improved_packed_bytes(C.byref(d), s)
            assert n == 2 * 4 * H * 3 * H * parts + 2 * 4 * H * 4 + 2 * H * 4 + 256, (p, s, n)
    for p in ("fp32", "tf32_tc"):  # no image for the other precisions
        assert lib.fsn_improved_packed_bytes(C.byref(_desc(args, p)), 0) == 0
        assert lib.fsn_last_error_code() == L.FSN_ERR_UNSUPPORTED


def test_bad_section_indices_are_refused():
    L, lib = _lib()
    d = _desc(_variants()["k16"], "f16x3_tc")
    w = L.ImprovedWeights()
    for s in (-1, d.num_sections, L.IMP_MAX_SECTIONS):
        assert lib.fsn_improved_packed_bytes(C.byref(d), s) == 0
        assert lib.fsn_last_error_code() == L.FSN_ERR_SHAPE
        rc = lib.fsn_improved_pack_sb_weights(C.byref(d), C.byref(w), s, 1 << 20, None)
        assert rc == L.FSN_ERR_SHAPE and lib.fsn_last_launch_count() == 0
    # a valid index with missing weights is refused before any CUDA call as well
    assert lib.fsn_improved_pack_sb_weights(C.byref(d), C.byref(w), 0, 1 << 20, None) == L.FSN_ERR_SHAPE
    assert lib.fsn_last_launch_count() == 0


def test_training_refuses_the_f16_precisions():
    L, lib = _lib()
    args = _variants()["k16"]
    for p in ("f16x3_tc", "f16_tc"):
        assert lib.fsn_improved_train_workspace_bytes(C.byref(_desc(args, p)), 2, 16000) == 0
        assert lib.fsn_last_error_code() == L.FSN_ERR_UNSUPPORTED
    assert lib.fsn_improved_train_workspace_bytes(C.byref(_desc(args, "tf32_tc")), 2, 16000) > 0


def test_unsupported_sub_band_sizes_are_refused():
    L, lib = _lib()
    for H in (64, 100, 512):
        args = dict(_variants()["k16"], sb_hidden_size=H)
        for p in ("f16x3_tc", "f16_tc"):
            assert lib.fsn_improved_workspace_bytes(C.byref(_desc(args, p)), 2, 16000) == 0
            assert lib.fsn_last_error_code() == L.FSN_ERR_UNSUPPORTED
        assert lib.fsn_debug_imp_section_lstm_tc_workspace_bytes(7, 3, 62, H, 1) == 0
    assert lib.fsn_debug_imp_section_lstm_tc_workspace_bytes(0, 3, 62, 384, 1) == 0
    assert lib.fsn_last_error_code() == L.FSN_ERR_SHAPE
    assert lib.fsn_debug_imp_section_lstm_tc_workspace_bytes(7, 3, 62, 384, 1) > 0
    w = L.SeqWeights()
    for stages, cluster in ((5, 0), (0, 3)):
        rc = lib.fsn_debug_imp_section_lstm_tc(C.byref(w), 62, 384, 1, 1 << 20, 7, 3, stages, cluster, 1 << 20,
                                               1 << 20, 1 << 20, 1 << 30, None)
        assert rc == L.FSN_ERR_UNSUPPORTED and lib.fsn_last_launch_count() == 0


def test_model_precisions():
    from fullsubnet_b200.improved_fullsubnet.model import Model
    m = Model(**_variants()["k16"])
    assert m._resolve_precision() == "tf32_tc"  # auto is unchanged
    for p in ("fp32", "tf32_tc", "f16x3_tc", "f16_tc"):
        m.precision = p
        assert m._resolve_precision() == p
    m.precision = "bf16"
    with pytest.raises(ValueError):
        m._resolve_precision()


def _cuobjdump():
    for c in (shutil.which("cuobjdump"), "/usr/local/cuda/bin/cuobjdump"):
        if c and os.path.exists(c):
            return c
    return None


@pytest.mark.parametrize("fn", list(PROJ_KERNELS), ids=list(PROJ_KERNELS.values()))
def test_section_kernel_stage_loop_has_no_gpu_scope_fence(fn):
    """The weight ring hands stages back with CTA-scope arrives only (DESIGN 4.1), in this instantiation too; the stage
    loop is the instructions between consecutive `WARPGROUP.DEPBAR.LE gsb0, 0x1`, as tests/test_cpu_subband_sass.py
    takes it."""
    from fullsubnet_b200 import _lib as L
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("no cuobjdump")
    if not os.path.exists(L.LIB_PATH):
        from fullsubnet_b200.csrc.build import build
        build()
    out = subprocess.run([tool, "-sass", "-fun", fn, L.LIB_PATH], capture_output=True, text=True, check=True).stdout
    ins = [m.group(1).strip() for m in re.finditer(r"/\*[0-9a-f]{4,}\*/\s+([^;]*);", out)]
    marks = [i for i, s in enumerate(ins) if re.search(r"WARPGROUP\.DEPBAR\.LE\s+gsb0,\s*0x1\b", s)]
    body = [s for a, b in zip(marks, marks[1:]) for s in ins[a + 1:b + 1]]
    assert sum(s.startswith("HGMMA") for s in body) > 0, f"{fn}: no stage loop found"
    fences = [s for s in body if re.search(r"\b(MEMBAR|FENCE)\b.*\bGPU\b|\bMEMBAR\.(SC|ALL)\b", s)]
    assert not fences, f"{fn}: GPU-scope fences in the stage loop: {fences[:3]}"
    for op in ("S2R", "LDC", "BSSY"):
        hits = [s for s in body if re.match(rf"(@!?U?P\w+\s+)?{op}\b", s)]
        assert not hits, f"{fn}: {op} in the stage loop: {hits[:3]}"
