"""CPU checks of the fullband_baseline training step: the oracle's autograd reproduces the two golden optimisation steps of
the unmodified reference (tests/golden/train_fbb.npz, oracle/make_golden_train_fbb.py), and the workspace query of
fsn_fullband_train_* answers without a GPU, with the reference's error classes for descriptors that are not built."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import rel_l2, rel_max

SUB = 97  # oracle/make_golden_train_fbb.py:SUBSAMPLE


def oracle_two_steps(g):
    """Two steps of fullband_baseline/trainer.py:32-71 on the oracle: MSE, autograd, clip_grad_norm_(10), Adam(1e-3).  The
    target is the stored cIRM of the reference (see test_cpu_fast_train.oracle_two_steps)."""
    from oracle import fullband_baseline_oracle as BO
    from oracle import make_golden_train_fbb as MG
    from oracle import train_oracle as TO
    noisy, clean = MG.inputs()
    nm, cirm_oracle = TO.targets(noisy, clean, 1)
    cirm = torch.from_numpy(g["cirm"])
    params = BO.make_fbb_state_dict(seed=MG.SEEDS["weights"])
    state, steps = {}, []
    for _ in range(2):
        p = {k: v.clone().requires_grad_(True) for k, v in params.items()}
        crm = BO.fbb_forward(nm.unsqueeze(1), p).permute(0, 2, 3, 1)
        loss = torch.mean((cirm - crm) ** 2)
        loss.backward()
        grads = {k: v.grad for k, v in p.items()}
        gnorm, coef = TO.clip_coef(grads, 10.0)
        params, state = TO.adam_update(params, {k: g * coef for k, g in grads.items()}, state)
        steps.append(dict(loss=float(loss.detach()), gnorm=float(gnorm), grads=grads, params=params, cirm=cirm_oracle,
                          crm=crm.detach()))
    return noisy, clean, steps


def test_oracle_autograd_reproduces_golden_training_steps(golden):
    from oracle import make_golden_train_fbb as MG
    g = golden("train_fbb")
    noisy, clean, steps = oracle_two_steps(g)
    assert np.allclose(MG.fingerprint(noisy), g["noisy_fp"], rtol=1e-6) and np.allclose(MG.fingerprint(clean), g["clean_fp"], rtol=1e-6)
    assert rel_l2(steps[0]["cirm"], g["cirm"]) < 1e-2
    assert rel_max(steps[0]["crm"], g["crm"]) < 1e-5
    for it in range(2):
        assert abs(steps[it]["loss"] - g["loss"][it]) <= 1e-5 * g["loss"][it]
        # clip_grad_norm_ reduces 5.5 M float32 squares in float32, the oracle in float64: 1.1e-5 apart at step 0 while
        # every gradient's own L2 norm agrees to 4e-8
        assert abs(steps[it]["gnorm"] - g["gnorm"][it]) <= 3e-5 * g["gnorm"][it]
    assert len(steps[0]["grads"]) == 14
    for k, v in steps[0]["grads"].items():
        full = v.numpy().reshape(-1)
        assert rel_l2(full[::SUB], g["gsub." + k]) < 1e-5, k
        assert abs(np.sqrt((full.astype(np.float64) ** 2).sum()) - g["gl2." + k]) <= 1e-5 * g["gl2." + k], k
    for k, v in steps[1]["params"].items():
        assert np.abs(v.numpy().reshape(-1)[::SUB] - g["p1." + k]).max() < 1e-6, k


def recipe_desc(prec):
    from fullsubnet_b200 import _lib
    return _lib.FullbandDesc(num_freqs=257, hidden=512, num_layers=3, look_ahead=2, activation=0, norm_type=0,
                             precision=_lib.PREC[prec], cell_type=0)


def test_fbb_train_workspace_query_without_gpu():
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    d = recipe_desc("tf32_tc")
    n_tc = lib.fsn_fullband_train_workspace_bytes(C.byref(d), 100, 193)  # the recipe: 100 clips x 3.072 s
    assert 0.8e9 < n_tc < 2e9, n_tc
    d.precision = _lib.PREC["fp32"]
    n32 = lib.fsn_fullband_train_workspace_bytes(C.byref(d), 100, 193)
    assert 0 < n32 < n_tc  # no transposed weights / K-major copies / fp16 operands
    assert lib.fsn_fullband_train_workspace_bytes(C.byref(d), 1, 10) < n32
    d.norm_type = 1  # cumulative norm: frame sums and per-frame scales on top
    assert lib.fsn_fullband_train_workspace_bytes(C.byref(d), 100, 193) > n32
    d.norm_type = 0
    for field, value, code in (("cell_type", 1, _lib.FSN_ERR_UNSUPPORTED),
                               ("precision", _lib.PREC["f16_tc"], _lib.FSN_ERR_UNSUPPORTED),
                               ("precision", _lib.PREC["f16x3_tc"], _lib.FSN_ERR_UNSUPPORTED),
                               ("num_layers", 0, _lib.FSN_ERR_UNSUPPORTED), ("num_layers", 9, _lib.FSN_ERR_UNSUPPORTED),
                               ("norm_type", 2, _lib.FSN_ERR_UNSUPPORTED), ("num_freqs", 1, _lib.FSN_ERR_SHAPE),
                               ("hidden", 0, _lib.FSN_ERR_SHAPE), ("look_ahead", -1, _lib.FSN_ERR_SHAPE),
                               ("activation", 4, _lib.FSN_ERR_SHAPE)):
        bad = _lib.FullbandDesc.from_buffer_copy(d)
        setattr(bad, field, value)
        assert lib.fsn_fullband_train_workspace_bytes(C.byref(bad), 4, 100) == 0, field
        assert lib.fsn_last_error_code() == code, field
    for B, T in ((0, 100), (4, 0)):
        assert lib.fsn_fullband_train_workspace_bytes(C.byref(d), B, T) == 0
        assert lib.fsn_last_error_code() == _lib.FSN_ERR_SHAPE
    # the argument checks run before any CUDA call: a GRU descriptor fails on a machine without a GPU too
    bad = _lib.FullbandDesc.from_buffer_copy(d)
    bad.cell_type = 1
    assert lib.fsn_fullband_train_forward(C.byref(bad), None, None, None, None, 4, 100, None, None, 0, None) == \
        _lib.FSN_ERR_UNSUPPORTED
    assert lib.fsn_fullband_train_backward(C.byref(bad), None, None, None, None, 4, 100, None, None, 0, None) == \
        _lib.FSN_ERR_UNSUPPORTED
    assert lib.fsn_fullband_train_forward(C.byref(d), None, None, None, None, 4, 100, None, None, 0, None) == _lib.FSN_ERR_SHAPE
    assert lib.fsn_fullband_train_backward(C.byref(d), None, None, None, None, 4, 100, None, None, 0, None) == _lib.FSN_ERR_SHAPE


def test_fbb_model_train_precision():
    from fullsubnet_b200.fullband_baseline.model import Model
    from oracle import fullband_baseline_oracle as BO
    m = Model(**BO.DEFAULT_FBB_ARGS)
    m.train_precision = "auto"
    assert m._resolve_train_precision() == "tf32_tc"  # H = 512
    odd = Model(**dict(BO.DEFAULT_FBB_ARGS, num_freqs=33, hidden_size=30))
    odd.train_precision = "auto"
    assert odd._resolve_train_precision() == "fp32"
    m.train_precision = "fp32"
    assert m._resolve_train_precision() == "fp32"
    m.train_precision = "f16_tc"
    with pytest.raises(ValueError):
        m._resolve_train_precision()
    d = m._desc(2)
    assert (d.precision, d.cell_type, d.num_layers, d.look_ahead) == (2, 0, 3, 2)
    assert not hasattr(m, "num_groups_in_drop_band")  # the Trainer applies no drop_band to this model


def test_fbb_model_train_precision_default_from_environment(monkeypatch):
    from fullsubnet_b200.fullband_baseline.model import Model
    from oracle import fullband_baseline_oracle as BO
    monkeypatch.setenv("FSN_TRAIN_PRECISION", "fp32")
    assert Model(**BO.DEFAULT_FBB_ARGS)._resolve_train_precision() == "fp32"
    monkeypatch.delenv("FSN_TRAIN_PRECISION")
    assert Model(**BO.DEFAULT_FBB_ARGS).train_precision == "auto"
