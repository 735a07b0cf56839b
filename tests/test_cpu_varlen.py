"""CPU-only checks of the clips-of-different-lengths path: fsn_enhance's workspace query and argument checks
(both answer before any CUDA call), the file loop's batch planner, and the Python ``lengths`` argument."""
import ctypes as C
import random

import numpy as np
import pytest
import torch


def _desc(**kw):
    from fullsubnet_b200 import _lib
    a = dict(num_freqs=257, look_ahead=2, fb_num_neighbors=0, sb_num_neighbors=15, fb_hidden=512, sb_hidden=384,
             fb_activation=1, sb_activation=0, norm_type=0, num_groups_in_drop_band=2, precision=3, cell_type=0)
    a.update(kw)
    return _lib.ModelDesc(**a)


def _call(lib, d, lengths, L_max, n_fft=512, hop=256, enhanced=None):
    arr = (C.c_int32 * len(lengths))(*lengths)
    return lib.fsn_enhance(C.byref(d), None, None, None, None, arr, len(lengths), L_max, n_fft, hop, n_fft, enhanced, None,
                           None, 1.0, None, 0, None)


def test_enhance_workspace_query_needs_no_gpu():
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    d = _desc()
    n = lib.fsn_enhance_workspace_bytes(C.byref(d), 4, 64000, 512, 256)
    assert n > 0
    assert lib.fsn_enhance_workspace_bytes(C.byref(d), 8, 64000, 512, 256) > n
    # the query takes no lengths: at n_fft 960 it sizes the null-lengths call (lengths are refused at the call)
    assert lib.fsn_enhance_workspace_bytes(C.byref(_desc(num_freqs=481)), 4, 48000, 960, 480) > 0


def test_enhance_rejects_bad_lengths_before_any_cuda_call():
    """No workspace, no weights, no device: every one of these fails on its argument check."""
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    d = _desc()
    assert _call(lib, d, [4000, 256, 3000], 4000) == _lib.FSN_ERR_SHAPE  # too short: <= n_fft/2
    assert b"clip 1" in lib.fsn_last_error()
    assert _call(lib, d, [4000, 4001, 3000], 4000) == _lib.FSN_ERR_SHAPE  # longer than the row
    assert b"clip 1" in lib.fsn_last_error()
    assert _call(lib, d, [3900, 257, 3000], 4000) == _lib.FSN_ERR_SHAPE  # max(lengths) != L_max
    assert b"3900" in lib.fsn_last_error()
    assert _call(lib, _desc(num_freqs=481), [4800, 4000], 4800, 960, 480) == _lib.FSN_ERR_UNSUPPORTED
    assert b"n_fft=960" in lib.fsn_last_error()
    # valid lengths reach the workspace check, the last one before the first launch (a stand-in output pointer, never
    # written: the call returns before any CUDA call)
    assert _call(lib, d, [4000, 257, 3000], 4000, enhanced=16) == _lib.FSN_ERR_WORKSPACE


def _check_plan(lens, bs, mp):
    from fullsubnet_b200.inferencer import plan_batches
    plan = plan_batches(lens, bs, mp)
    flat = [i for b in plan for i in b]
    assert sorted(flat) == list(range(len(lens)))  # every clip exactly once
    for b in plan:
        assert 1 <= len(b) <= bs
        Lm = max(lens[i] for i in b)
        pad = len(b) * Lm - sum(lens[i] for i in b)
        assert pad <= mp * len(b) * Lm
        if mp == 0:
            assert len({lens[i] for i in b}) == 1
    return plan


def test_plan_batches_bounds_and_coverage():
    rng = random.Random(3)
    lens = [rng.randint(16000, 160000) for _ in range(300)] + [32000] * 7
    for bs in (1, 3, 64, 256):
        for mp in (0.0, 0.05, 0.2, 0.5):
            _check_plan(lens, bs, mp)
    # more padding allowed -> never more batches
    n = [len(_check_plan(lens, 64, mp)) for mp in (0.0, 0.05, 0.2, 0.5)]
    assert n == sorted(n, reverse=True) and n[-1] < n[0]


def test_plan_batches_exact_groups_at_zero_padding():
    """max_padding = 0 reproduces the equal-length grouping: ascending length, file order within a length."""
    from fullsubnet_b200.inferencer import plan_batches
    lens = [6000, 4000, 6000, 6000, 4000]
    assert plan_batches(lens, 2, 0.0) == [[1, 4], [0, 2], [3]]
    assert plan_batches(lens, 64, 0.0) == [[1, 4], [0, 2, 3]]
    assert plan_batches(lens, 64, 0.5) == [[1, 4, 0, 2, 3]]  # 2 * 2000 padded of 30000
    assert plan_batches([], 4, 0.1) == []
    with pytest.raises(ValueError):
        plan_batches(lens, 0, 0.0)
    with pytest.raises(ValueError):
        plan_batches(lens, 4, 1.0)


def test_python_lengths_argument_and_table_are_checked():
    from fullsubnet_b200 import _lib
    from fullsubnet_b200.fullsubnet.model import Model
    from oracle import fullsubnet_oracle as O
    m = Model(**O.DEFAULT_MODEL_ARGS)
    y = torch.zeros(3, 4000)
    for fn in (m.enhance, m.enhance_pcm):
        with pytest.raises(ValueError, match="entries"):
            fn(y, lengths=[4000, 3000])
        with pytest.raises(ValueError, match="exceeds"):
            fn(y, lengths=[4000, 4001, 300])
        with pytest.raises(ValueError):
            fn(y, lengths=torch.tensor([4000.0, 3000.0, 300.0]))
    lens = _lib.lengths_table(torch.tensor([4000, 3000, 300]), 3, 4000)
    assert lens.dtype == np.int32 and lens.tolist() == [4000, 3000, 300] and lens.flags["C_CONTIGUOUS"]


def test_models_without_the_varlen_entry_refuse_lengths():
    from fullsubnet_b200.fast_fullsubnet.model import Model as Fast
    from fullsubnet_b200.inferencer import Inferencer
    from oracle import fast_fullsubnet_oracle as FO
    inf = Inferencer.__new__(Inferencer)  # no device needed to reach the check
    inf.model, inf.n_fft = Fast(**FO.DEFAULT_FAST_ARGS), 512
    assert not inf.supports_lengths()
    with pytest.raises(NotImplementedError):
        inf.enhance_batch(torch.zeros(2, 4000), lengths=[4000, 3000])
    with pytest.raises(NotImplementedError):
        inf.enhance_to_pcm(torch.zeros(2, 4000), lengths=[4000, 3000])
