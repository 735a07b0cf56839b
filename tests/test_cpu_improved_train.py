"""CPU checks of the improved_fullsubnet training step: the oracle's autograd (including the adjoint of the element-wise mask
and the iSTFT) reproduces the golden optimisation steps of the unmodified reference (tests/golden/train_imp*.npz,
oracle/make_golden_train_imp.py), and the workspace query of fsn_improved_train_* answers without a GPU, with the
reference's error classes for descriptors that are not built."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import rel_l2, rel_max


def oracle_steps(name, steps):
    """MSE(enhanced, clean) on the oracle, autograd, clip_grad_norm_(10), Adam(1e-3)."""
    from oracle import improved_fullsubnet_oracle as IO
    from oracle import make_golden_train_imp as MG
    from oracle import train_oracle as TO
    args = MG.args_of(name)
    noisy, clean = MG.inputs(name)
    params = IO.make_improved_state_dict(seed=MG.SEEDS["weights"], args=args)
    state, out = {}, []
    for _ in range(steps):
        p = {k: v.clone().requires_grad_(True) for k, v in params.items()}
        enhanced = IO.improved_forward(noisy, p, args)
        loss = torch.mean((enhanced - clean.unsqueeze(1)) ** 2)
        loss.backward()
        grads = {k: v.grad for k, v in p.items()}
        gnorm, coef = TO.clip_coef(grads, 10.0)
        params, state = TO.adam_update(params, {k: g * coef for k, g in grads.items()}, state)
        out.append(dict(loss=float(loss.detach()), gnorm=float(gnorm), grads=grads, params=params,
                        enhanced=enhanced.detach()))
    return noisy, clean, out


@pytest.mark.parametrize("name,steps", [("train_imp", 2), ("train_imp_960", 1)])
def test_oracle_autograd_reproduces_golden_training_steps(golden, name, steps):
    from oracle import make_golden_train_imp as MG
    g = golden(name)
    sub = MG.SUBSAMPLE
    noisy, clean, out = oracle_steps(name, steps)
    assert np.allclose(MG.fingerprint(noisy), g["noisy_fp"], rtol=1e-6) and np.allclose(MG.fingerprint(clean), g["clean_fp"], rtol=1e-6)
    if "enhanced" in g:
        assert rel_max(out[0]["enhanced"], g["enhanced"]) < 1e-5
    for it in range(steps):
        assert abs(out[it]["loss"] - g["loss"][it]) <= 1e-5 * g["loss"][it], (it, out[it]["loss"], g["loss"][it])
        assert abs(out[it]["gnorm"] - g["gnorm"][it]) <= 3e-5 * g["gnorm"][it], (it, out[it]["gnorm"], g["gnorm"][it])
    for k, v in out[0]["grads"].items():
        full = v.numpy().reshape(-1)
        assert rel_l2(full[::sub], g["gsub." + k]) < 1e-5, k
        assert abs(np.sqrt((full.astype(np.float64) ** 2).sum()) - g["gl2." + k]) <= 1e-5 * g["gl2." + k], k
    if steps > 1:
        for k, v in out[1]["params"].items():
            assert np.abs(v.numpy().reshape(-1)[::sub] - g["p1." + k]).max() < 1e-6, k


def default_desc(prec):
    from fullsubnet_b200.improved_fullsubnet.model import Model
    from oracle import improved_fullsubnet_oracle as IO
    m = Model(**IO.DEFAULT_IMPROVED_ARGS)
    return m._desc(prec)


def test_improved_train_workspace_query_without_gpu():
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    L = 49152  # 3.072 s at 16 kHz: T = 385
    d = default_desc("tf32_tc")
    n_tc = lib.fsn_improved_train_workspace_bytes(C.byref(d), 1, L)
    d.precision = _lib.PREC["fp32"]
    n32 = lib.fsn_improved_train_workspace_bytes(C.byref(d), 1, L)
    # the G / C / H of the section layers dominate: 57 sub-band rows per clip, 2 layers x 6 x 384 floats per row and step
    assert 0.4e9 < n32 < n_tc, (n32, n_tc)
    assert lib.fsn_improved_train_workspace_bytes(C.byref(d), 2, L) > n32
    for field, value, code in (("cell_type", _lib.CELL["GRU"], _lib.FSN_ERR_UNSUPPORTED),
                               ("precision", _lib.PREC["f16_tc"], _lib.FSN_ERR_UNSUPPORTED),
                               ("precision", _lib.PREC["f16x3_tc"], _lib.FSN_ERR_UNSUPPORTED),
                               ("fb_activation", _lib.ACT["Tanh"], _lib.FSN_ERR_UNSUPPORTED),
                               ("sb_activation", _lib.ACT["ReLU6"], _lib.FSN_ERR_UNSUPPORTED),
                               ("num_sections", 0, _lib.FSN_ERR_SHAPE), ("hop_length", 0, _lib.FSN_ERR_SHAPE),
                               ("sb_hidden", 0, _lib.FSN_ERR_SHAPE)):
        bad = _lib.ImprovedDesc.from_buffer_copy(d)
        setattr(bad, field, value)
        assert lib.fsn_improved_train_workspace_bytes(C.byref(bad), 4, 8000) == 0, field
        assert lib.fsn_last_error_code() == code, field
    bad = _lib.ImprovedDesc.from_buffer_copy(d)
    bad.fb_num_center[1] = 2  # cs != cf in section 1
    assert lib.fsn_improved_train_workspace_bytes(C.byref(bad), 4, 8000) == 0
    assert lib.fsn_last_error_code() == _lib.FSN_ERR_UNSUPPORTED
    for B, L in ((0, 8000), (4, 0)):
        assert lib.fsn_improved_train_workspace_bytes(C.byref(d), B, L) == 0
        assert lib.fsn_last_error_code() == _lib.FSN_ERR_SHAPE
    # the argument checks run before any CUDA call: they fail the same way on a machine without a GPU
    gru = _lib.ImprovedDesc.from_buffer_copy(d)
    gru.cell_type = _lib.CELL["GRU"]
    assert lib.fsn_improved_train_forward(C.byref(gru), None, None, 4, 8000, None, None, 0, None) == _lib.FSN_ERR_UNSUPPORTED
    assert lib.fsn_improved_train_backward(C.byref(gru), None, None, 4, 8000, None, None, 0, None) == _lib.FSN_ERR_UNSUPPORTED
    assert lib.fsn_improved_train_forward(C.byref(d), None, None, 4, 8000, None, None, 0, None) == _lib.FSN_ERR_SHAPE
    assert lib.fsn_improved_train_backward(C.byref(d), None, None, 4, 8000, None, None, 0, None) == _lib.FSN_ERR_SHAPE


def test_improved_model_train_precision(monkeypatch):
    from fullsubnet_b200.improved_fullsubnet.model import Model
    from oracle import improved_fullsubnet_oracle as IO
    m = Model(**IO.DEFAULT_IMPROVED_ARGS)
    assert m.train_precision == "auto" and m._resolve_train_precision() == "tf32_tc"  # 512 / 384
    assert Model(**dict(IO.DEFAULT_IMPROVED_ARGS, sb_hidden_size=30))._resolve_train_precision() == "fp32"
    assert Model(**dict(IO.DEFAULT_IMPROVED_ARGS, fb_hidden_size=30))._resolve_train_precision() == "fp32"
    m.train_precision = "fp32"
    assert m._resolve_train_precision() == "fp32"
    m.train_precision = "f16_tc"
    with pytest.raises(ValueError):
        m._resolve_train_precision()
    d = Model(**IO.DEFAULT_IMPROVED_ARGS)._train_desc()
    assert (d.precision, d.cell_type, d.num_sections) == (_prec("tf32_tc"), 0, 3)
    assert Model(**dict(IO.DEFAULT_IMPROVED_ARGS, sequence_model="GRU"))._train_desc().cell_type == 1
    monkeypatch.setenv("FSN_TRAIN_PRECISION", "fp32")
    assert Model(**IO.DEFAULT_IMPROVED_ARGS)._resolve_train_precision() == "fp32"


def _prec(name):
    from fullsubnet_b200 import _lib
    return _lib.PREC[name]
