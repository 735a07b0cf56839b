"""fast_fullsubnet with norm_type="cumulative_laplace_norm", no GPU needed: the C ABI answers its workspace queries and refuses
what is not built before any CUDA call, and the oracle reproduces the unmodified reference built with that norm
(tests/golden/fast_cum.npz, oracle/make_golden_fast_cum.py), in inference and over two training steps."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import rel_l2, rel_max

SUB = 291  # oracle/make_golden_fast_cum.py:SUBSAMPLE


def _desc(prec, norm):
    from fullsubnet_b200 import _lib
    return _lib.FastDesc(num_freqs=257, look_ahead=2, shrink_size=2, num_mels=64, enc1_hidden=384, enc2_hidden=257,
                         bn_hidden=384, bn_layers=2, dec_hidden=512, noisy_num_neighbors=5, enc_num_neighbors=0,
                         precision=_lib.PREC[prec], cell_type=0, norm_type=norm)


def test_abi_version():
    from fullsubnet_b200 import _lib
    assert _lib.load().fsn_version() == 102


def test_workspace_queries_without_gpu():
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    for prec in ("fp32", "f16_tc", "f16x3_tc"):
        off = lib.fsn_fast_workspace_bytes(C.byref(_desc(prec, 0)), 512, 251)
        cum = lib.fsn_fast_workspace_bytes(C.byref(_desc(prec, 1)), 512, 251)
        assert 0 < off < cum, (prec, off, cum)
        assert lib.fsn_fast_packed_bytes(C.byref(_desc(prec, 1))) == lib.fsn_fast_packed_bytes(C.byref(_desc(prec, 0)))
    for prec in ("fp32", "tf32_tc"):
        off = lib.fsn_fast_train_workspace_bytes(C.byref(_desc(prec, 0)), 72, 193)
        cum = lib.fsn_fast_train_workspace_bytes(C.byref(_desc(prec, 1)), 72, 193)
        assert 0 < off < cum, (prec, off, cum)


@pytest.mark.parametrize("norm,cell", [(2, 0), (-1, 0), (1, 1)], ids=["norm2", "norm-1", "gru-cum"])
def test_unbuilt_descriptors_are_refused_before_any_cuda_call(norm, cell):
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    for prec in ("fp32", "f16x3_tc", "tf32_tc"):
        d = _desc(prec, norm)
        d.cell_type = cell
        assert lib.fsn_fast_workspace_bytes(C.byref(d), 4, 100) == 0
        assert lib.fsn_last_error_code() == _lib.FSN_ERR_UNSUPPORTED
        assert lib.fsn_fast_train_workspace_bytes(C.byref(d), 4, 100) == 0
        assert lib.fsn_last_error_code() == _lib.FSN_ERR_UNSUPPORTED
        assert lib.fsn_fast_model_forward(C.byref(d), None, None, 4, 100, None, None, 0, None) == _lib.FSN_ERR_UNSUPPORTED
        assert lib.fsn_fast_train_forward(C.byref(d), None, None, 4, 100, None, None, 0, None) == _lib.FSN_ERR_UNSUPPORTED
        assert lib.fsn_fast_train_backward(C.byref(d), None, None, 4, 100, None, None, 0, None) == _lib.FSN_ERR_UNSUPPORTED


def test_model_accepts_the_cumulative_norm():
    from fullsubnet_b200 import _lib
    from fullsubnet_b200.fast_fullsubnet.model import Model
    from oracle import fast_fullsubnet_oracle as FO
    m = Model(**dict(FO.DEFAULT_FAST_ARGS, norm_type="cumulative_laplace_norm"))
    assert m._desc(_lib.PREC["fp32"]).norm_type == 1
    assert Model(**FO.DEFAULT_FAST_ARGS)._desc(_lib.PREC["fp32"]).norm_type == 0
    for bad in ("offline_gaussian_norm", "cumulative_layer_norm", "forgetting_norm", "bogus"):
        with pytest.raises(NotImplementedError):
            Model(**dict(FO.DEFAULT_FAST_ARGS, norm_type=bad))
    with pytest.raises(RuntimeError):
        m.eval()(torch.zeros(1, 1, 257, 10))  # no CPU path


def test_oracle_matches_reference_inference(golden):
    from oracle import fast_fullsubnet_cum_oracle as CO
    from oracle import fast_fullsubnet_oracle as FO
    from oracle import make_golden_fast_cum as MG
    g = golden("fast_cum")
    args = MG.cum_args()
    sd = FO.make_fast_state_dict(seed=3, args=args)
    for T in MG.LENGTHS:
        mag = torch.from_numpy(g[f"mag_T{T}"]).unsqueeze(1)
        assert rel_max(CO.fast_model_forward(mag[:1], sd, args), g[f"out_b1_T{T}"]) < 2e-5, T
        out = CO.fast_model_forward(mag, sd, args)
        assert rel_max(out, g[f"out_b3_T{T}"]) < 2e-5, T
        # the offline norm gives another model: the fixture pins the cumulative one; with it, the restatement is the
        # recipe oracle's forward bit for bit
        off = FO.fast_model_forward(mag, sd)
        assert rel_max(off, g[f"out_b3_T{T}"]) > 1e-3, T
        assert torch.equal(CO.fast_model_forward(mag, sd, dict(args, norm_type="offline_laplace_norm")), off), T


def test_oracle_cumulative_norms_are_causal():
    """Each scale depends on the frames (encoder) and shrunk steps (bottleneck) up to its own: the outputs of frames whose
    down-sampling block is complete do not change when later frames do."""
    from oracle import fast_fullsubnet_cum_oracle as CO
    from oracle import fast_fullsubnet_oracle as FO
    from oracle import make_golden_fast_cum as MG
    args = MG.cum_args()
    sd = FO.make_fast_state_dict(seed=3, args=args)
    x = torch.rand(2, 1, 257, 14, generator=torch.Generator().manual_seed(0))
    y = x.clone()
    y[..., 9:] = torch.rand(2, 1, 257, 5, generator=torch.Generator().manual_seed(1))
    a, b = CO.fast_model_forward(x, sd, args), CO.fast_model_forward(y, sd, args)
    # padded frame t' = t + 2 reads shrunk step t' // 2, whose block ends at frame t' - t' % 2 <= t': frames t < 7 see
    # only input frames < 9
    assert torch.equal(a[..., :7], b[..., :7])
    assert not torch.equal(a[..., 7:], b[..., 7:])


def test_oracle_autograd_reproduces_golden_training_steps(golden):
    """Two steps of fast_fullsubnet/trainer.py:45-56 on the oracle with the cumulative norm: MSE against the reference's
    cIRM of train_fast.npz (same inputs), autograd, clip_grad_norm_(10), Adam(1e-3)."""
    from oracle import fast_fullsubnet_cum_oracle as CO
    from oracle import fast_fullsubnet_oracle as FO
    from oracle import make_golden_fast_cum as MG
    from oracle import make_golden_train_fast as MGT
    from oracle import train_oracle as TO
    g, g_fast = golden("fast_cum"), golden("train_fast")
    args = MG.cum_args()
    noisy, clean = MGT.inputs()
    nm, _ = TO.targets(noisy, clean, 1)
    cirm = torch.from_numpy(g_fast["cirm"])
    sd = FO.make_fast_state_dict(seed=MGT.SEEDS["weights"], args=args)
    params = {k: v for k, v in sd.items() if k != "mel_scale.fb"}
    state = {}
    for it in range(2):
        p = {k: v.clone().requires_grad_(True) for k, v in params.items()}
        crm = CO.fast_model_forward(nm.unsqueeze(1), dict(p, **{"mel_scale.fb": sd["mel_scale.fb"]}), args).permute(0, 2, 3, 1)
        loss = torch.mean((cirm - crm) ** 2)
        loss.backward()
        grads = {k: v.grad for k, v in p.items()}
        gnorm, coef = TO.clip_coef(grads, 10.0)
        assert abs(float(loss.detach()) - g["loss"][it]) <= 1e-5 * g["loss"][it], it
        assert abs(float(gnorm) - g["gnorm"][it]) <= 1e-5 * g["gnorm"][it], it
        if it == 0:
            assert rel_max(crm.detach(), g["crm"]) < 1e-5
            assert len(grads) == 30
            for k, v in grads.items():
                full = v.numpy().reshape(-1)
                assert rel_l2(full[::SUB], g["gsub." + k]) < 1e-5, k
                assert abs(np.sqrt((full.astype(np.float64) ** 2).sum()) - g["gl2." + k]) <= 1e-5 * g["gl2." + k], k
        params, state = TO.adam_update(params, {k: v * coef for k, v in grads.items()}, state)
        sub = SUB * (4 if it == 0 else 1)
        for k, v in params.items():
            assert np.abs(v.numpy().reshape(-1)[::sub] - g[f"p{it}." + k]).max() < 1e-6, (it, k)
