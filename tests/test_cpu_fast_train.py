"""CPU checks of the fast_fullsubnet training step: the oracle's autograd reproduces the two golden optimisation steps of
the unmodified reference (tests/golden/train_fast.npz, oracle/make_golden_train_fast.py), and the workspace query of
fsn_fast_train_* answers without a GPU, with the reference's error classes for descriptors that are not built."""
import ctypes as C

import numpy as np
import torch

from conftest import rel_l2, rel_max

SUB = 97  # oracle/make_golden_train_fast.py:SUBSAMPLE


def oracle_two_steps(g):
    """Two steps of fast_fullsubnet/trainer.py:45-56 on the oracle: MSE, autograd, clip_grad_norm_(10), Adam(1e-3).  The
    target is the stored cIRM of the reference: at a few frame-0 bins the noisy magnitude is ~1e-4, where the ratio mask
    amplifies the rounding differences of two STFT implementations (checked separately, by relative L2)."""
    from oracle import fast_fullsubnet_oracle as FO
    from oracle import make_golden_train_fast as MG
    from oracle import train_oracle as TO
    noisy, clean = MG.inputs()
    nm, cirm_oracle = TO.targets(noisy, clean, 1)
    cirm = torch.from_numpy(g["cirm"])
    sd = FO.make_fast_state_dict(seed=MG.SEEDS["weights"])
    params = {k: v for k, v in sd.items() if k != "mel_scale.fb"}
    state, steps = {}, []
    for _ in range(2):
        p = {k: v.clone().requires_grad_(True) for k, v in params.items()}
        crm = FO.fast_model_forward(nm.unsqueeze(1), dict(p, **{"mel_scale.fb": sd["mel_scale.fb"]})).permute(0, 2, 3, 1)
        loss = torch.mean((cirm - crm) ** 2)
        loss.backward()
        grads = {k: v.grad for k, v in p.items()}
        gnorm, coef = TO.clip_coef(grads, 10.0)
        params, state = TO.adam_update(params, {k: g * coef for k, g in grads.items()}, state)
        steps.append(dict(loss=float(loss.detach()), gnorm=float(gnorm), grads=grads, params=params, cirm=cirm_oracle,
                          crm=crm.detach()))
    return noisy, clean, steps


def test_oracle_autograd_reproduces_golden_training_steps(golden):
    from oracle import make_golden_train_fast as MG
    g = golden("train_fast")
    noisy, clean, steps = oracle_two_steps(g)
    assert np.allclose(MG.fingerprint(noisy), g["noisy_fp"], rtol=1e-6) and np.allclose(MG.fingerprint(clean), g["clean_fp"], rtol=1e-6)
    assert rel_l2(steps[0]["cirm"], g["cirm"]) < 1e-2  # 13 of 49 344 bins, all at |noisy| < 0.01, differ by > 1e-4
    assert rel_max(steps[0]["crm"], g["crm"]) < 1e-5
    for it in range(2):
        assert abs(steps[it]["loss"] - g["loss"][it]) <= 1e-5 * g["loss"][it]
        assert abs(steps[it]["gnorm"] - g["gnorm"][it]) <= 1e-5 * g["gnorm"][it]
    assert len(steps[0]["grads"]) == 30
    for k, v in steps[0]["grads"].items():
        full = v.numpy().reshape(-1)
        assert rel_l2(full[::SUB], g["gsub." + k]) < 1e-5, k
        assert abs(np.sqrt((full.astype(np.float64) ** 2).sum()) - g["gl2." + k]) <= 1e-5 * g["gl2." + k], k
    for k, v in steps[1]["params"].items():
        assert np.abs(v.numpy().reshape(-1)[::SUB] - g["p1." + k]).max() < 1e-6, k


def test_fast_train_workspace_query_without_gpu():
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    d = _lib.FastDesc(num_freqs=257, look_ahead=2, shrink_size=2, num_mels=64, enc1_hidden=384, enc2_hidden=257, bn_hidden=384,
                      bn_layers=2, dec_hidden=512, noisy_num_neighbors=5, enc_num_neighbors=0, precision=_lib.PREC["tf32_tc"],
                      cell_type=0)
    n_tc = lib.fsn_fast_train_workspace_bytes(C.byref(d), 72, 193)  # the recipe: 72 clips x 3.072 s
    assert 4e9 < n_tc < 40e9, n_tc
    d.precision = _lib.PREC["fp32"]
    n32 = lib.fsn_fast_train_workspace_bytes(C.byref(d), 72, 193)
    assert 0 < n32 < n_tc  # no transposed weights / K-major copies / fp16 operands
    assert lib.fsn_fast_train_workspace_bytes(C.byref(d), 1, 10) < n32
    for field, value, code in (("cell_type", 1, _lib.FSN_ERR_UNSUPPORTED), ("bn_layers", 3, _lib.FSN_ERR_UNSUPPORTED),
                               ("precision", _lib.PREC["f16_tc"], _lib.FSN_ERR_UNSUPPORTED),
                               ("precision", _lib.PREC["f16x3_tc"], _lib.FSN_ERR_UNSUPPORTED),
                               ("enc_num_neighbors", 64, _lib.FSN_ERR_SHAPE)):
        bad = _lib.FastDesc.from_buffer_copy(d)
        setattr(bad, field, value)
        assert lib.fsn_fast_train_workspace_bytes(C.byref(bad), 4, 100) == 0, field
        assert lib.fsn_last_error_code() == code, field
    assert lib.fsn_fast_train_workspace_bytes(C.byref(d), 0, 100) == 0 and lib.fsn_last_error_code() == _lib.FSN_ERR_SHAPE
    # the argument checks run before any CUDA call: a GRU descriptor fails on a machine without a GPU too
    bad = _lib.FastDesc.from_buffer_copy(d)
    bad.cell_type = 1
    assert lib.fsn_fast_train_forward(C.byref(bad), None, None, 4, 100, None, None, 0, None) == _lib.FSN_ERR_UNSUPPORTED
    assert lib.fsn_fast_train_backward(C.byref(d), None, None, 4, 100, None, None, 0, None) == _lib.FSN_ERR_SHAPE


def test_fast_model_train_precision_and_frozen_parameters():
    from fullsubnet_b200.fast_fullsubnet.model import Model
    from oracle import fast_fullsubnet_oracle as FO
    m = Model(**FO.DEFAULT_FAST_ARGS)
    assert m._resolve_train_precision() == "tf32_tc"
    m.train_precision = "fp32"
    assert m._resolve_train_precision() == "fp32"
    m.train_precision = "f16_tc"
    try:
        m._resolve_train_precision()
        raise AssertionError("f16_tc is not a training precision")
    except ValueError:
        pass
    assert not hasattr(m, "num_groups_in_drop_band")  # the Trainer applies no drop_band to this model
