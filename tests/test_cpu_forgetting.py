"""forgetting_norm (audio_zen/model/base_model.py:102-151) without a GPU: the oracle against the unmodified reference
function (tests/golden/forgetting.npz), the coefficients at the edges of the t = 192 switch, the descriptors' refusals and
workspace queries, the hooks' argument checks, and the Python models' norm mapping."""
import ctypes as C

import numpy as np
import pytest
import torch


def _lib():
    from fullsubnet_b200 import _lib
    return _lib, _lib.load()


def test_coefficients_as_the_reference_rounds_them():
    from oracle import forgetting_oracle as FO
    a, b = FO.coefficients(200)
    assert a.dtype == np.float32 and b.dtype == np.float32
    assert a[0] == -1 and b[0] == 2 and a[1] == 0 and b[1] == 1
    alpha = 191 / 193
    assert a[191] == np.float32(190 / 192) and b[191] == np.float32(1) - np.float32(190 / 192)
    for t in (192, 193, 199):
        assert a[t] == np.float32(alpha) and b[t] == np.float32(1 - alpha)
    # the two halves round 1 - alpha differently: float32 subtraction before 192, the double rounded from 192 on
    assert np.float32(1) - np.float32(alpha) != np.float32(1 - alpha)
    for t in range(2, 192):
        assert a[t] == np.float32((t - 1) / (t + 1)) < np.float32(alpha)


@pytest.mark.parametrize("tag", ["n1", "n2"])
def test_oracle_matches_reference_function(golden, tag):
    """float32: the reference's bits at every frame, t = 0, 1, 191, 192, 193 included; float64 within 1e-6."""
    from oracle import forgetting_oracle as FO
    g = golden("forgetting")
    x, want = torch.from_numpy(g[tag + "_x"]), g[tag + "_y"]
    y32, mu32 = FO.forgetting_norm(x)
    assert y32.dtype == torch.float32 and mu32.shape == (x.shape[0], x.shape[-1])
    assert np.array_equal(y32.numpy().view(np.uint32), want.view(np.uint32))
    for t in (0, 1, 191, 192, 193):
        assert np.array_equal(y32.numpy()[..., t], want[..., t]), t
    y64, _ = FO.forgetting_norm(x.double())
    assert float(np.abs(y64.numpy() - want).max() / np.abs(want).max()) < 1e-6
    # mu_0 = 2 m_0 (a_0 = -1) and mu_1 = m_1 (a_1 = 0)
    m = FO.frame_means(x)
    assert torch.equal(mu32[:, 0], 2 * m[:, 0]) and torch.equal(mu32[:, 1], m[:, 1])


def _desc(norm):
    from fullsubnet_b200.fullsubnet.model import Model
    from oracle.make_golden_train import SMALL
    return Model(**dict(SMALL, norm_type=norm))._desc("fp32", 2)


def test_model_descriptor_accepts_forgetting_norm():
    _l, lib = _lib()
    for norm in ("offline_laplace_norm", "cumulative_laplace_norm", "forgetting_norm"):
        d = _desc(norm)
        assert lib.fsn_model_workspace_bytes(C.byref(d), 3, 40) > 0
        assert lib.fsn_train_workspace_bytes(C.byref(d), 5, 40) > 0
        assert lib.fsn_enhance_workspace_bytes(C.byref(d), 3, 1200, 64, 32) > 0
    assert _desc("forgetting_norm").norm_type == 4
    # the forgetting norm's workspace holds the cumulative norm's tables plus the full-band frame sums
    assert lib.fsn_model_workspace_bytes(C.byref(_desc("forgetting_norm")), 3, 40) > lib.fsn_model_workspace_bytes(
        C.byref(_desc("cumulative_laplace_norm")), 3, 40)
    d = _desc("forgetting_norm")
    for unbuilt in (2, 3, 5):  # offline_gaussian_norm, cumulative_layer_norm, no norm
        d.norm_type = unbuilt
        assert lib.fsn_model_workspace_bytes(C.byref(d), 3, 40) == 0 and lib.fsn_last_error_code() == 2
        assert lib.fsn_train_workspace_bytes(C.byref(d), 5, 40) == 0 and lib.fsn_last_error_code() == 2


def test_fullband_descriptor_accepts_forgetting_norm():
    _l, lib = _lib()
    from fullsubnet_b200.fullband_baseline.model import Model
    from oracle import fullband_baseline_oracle as BO
    m = Model(**dict(BO.DEFAULT_FBB_ARGS, num_freqs=33, hidden_size=32, norm_type="forgetting_norm"))
    assert m.norm == 4
    d = m._desc()
    assert d.norm_type == 4
    assert lib.fsn_fullband_workspace_bytes(C.byref(d), 2, 40) > 0
    assert lib.fsn_fullband_train_workspace_bytes(C.byref(d), 2, 40) > 0
    assert lib.fsn_fullband_enhance_workspace_bytes(C.byref(d), 2, 1200, 64, 32) > 0
    for unbuilt in (2, 3, 5):
        d.norm_type = unbuilt
        assert lib.fsn_fullband_workspace_bytes(C.byref(d), 2, 40) == 0 and lib.fsn_last_error_code() == 2
        assert lib.fsn_fullband_train_workspace_bytes(C.byref(d), 2, 40) == 0 and lib.fsn_last_error_code() == 2


def test_fast_descriptor_refuses_forgetting_norm():
    _l, lib = _lib()
    from fullsubnet_b200.fast_fullsubnet.model import Model
    from oracle import fast_fullsubnet_oracle as FO
    d = Model(**FO.DEFAULT_FAST_ARGS)._desc(_l.PREC["fp32"])
    d.norm_type = 4
    assert lib.fsn_fast_workspace_bytes(C.byref(d), 1, 20) == 0 and lib.fsn_last_error_code() == 2
    assert lib.fsn_fast_train_workspace_bytes(C.byref(d), 2, 20) == 0 and lib.fsn_last_error_code() == 2
    with pytest.raises(NotImplementedError):
        Model(**dict(FO.DEFAULT_FAST_ARGS, norm_type="forgetting_norm"))


def test_python_models_map_forgetting_norm():
    from fullsubnet_b200.fullband_baseline.model import Model as FBB
    from fullsubnet_b200.fullsubnet.model import Model as FSN
    from fullsubnet_b200.improved_fullsubnet.model import Model as IMP
    from oracle import fullband_baseline_oracle as BO
    from oracle.make_golden_train import SMALL
    m = FSN(**dict(SMALL, norm_type="forgetting_norm"))
    assert m.norm == 4
    assert FBB(**dict(BO.DEFAULT_FBB_ARGS, norm_type="forgetting_norm")).norm == 4
    with pytest.raises(NotImplementedError):
        IMP(norm_type="forgetting_norm")
    with pytest.raises(RuntimeError):
        m.eval()(torch.zeros(1, 1, 33, 10))  # no CPU path


def test_hooks_refuse_bad_arguments():
    """Every refusal returns before any CUDA call (no device here), with FSN_ERR_SHAPE."""
    _l, lib = _lib()
    p = C.c_void_p(16)  # never dereferenced: the checks fail first
    scale = lib.fsn_debug_forgetting_scale
    ok = dict(x=p, N=0, x2=None, N2=0, B=2, T=10, F=5, bs=50, ts=5, cnt=5.0, lengths=None, lens=None, hop=0, la=0,
              fs=p, fs2=None, scale=p, mu=None)

    def call(**kw):
        a = dict(ok, **kw)
        return scale(a["x"], a["N"], a["x2"], a["N2"], a["B"], a["T"], a["F"], a["bs"], a["ts"], a["cnt"], a["lengths"],
                     a["lens"], a["hop"], a["la"], a["fs"], a["fs2"], a["scale"], a["mu"], None)
    for bad in (dict(x=None), dict(fs=None), dict(scale=None), dict(x2=p, fs2=None), dict(B=0), dict(T=0), dict(F=0),
                dict(N=5), dict(N=-1), dict(x2=p, fs2=p, N2=5), dict(cnt=0.0), dict(bs=-1)):
        assert call(**bad) == 1, bad
    lens = (C.c_int32 * 2)(64, 9 * 32)
    assert call(lengths=lens, lens=None, hop=32) == 1          # no device table
    assert call(lengths=lens, lens=p, hop=0) == 1              # no hop
    assert call(lengths=lens, lens=p, hop=32, la=2) == 1       # clip 1 has 12 frames > T_pad
    bwd = lib.fsn_debug_forgetting_bwd
    okb = dict(dX=p, X=p, fbz=p, scale=p, B=3, F=6, G=2, Tp=5, Ns=1, act=1, mid=p, dz=p)

    def callb(**kw):
        a = dict(okb, **kw)
        return bwd(a["dX"], a["X"], a["fbz"], a["scale"], a["B"], a["F"], a["G"], a["Tp"], a["Ns"], a["act"], a["mid"],
                   a["dz"], None)
    for bad in (dict(dX=None), dict(X=None), dict(fbz=None), dict(scale=None), dict(mid=None), dict(dz=None), dict(B=0),
                dict(F=0), dict(Tp=0), dict(G=-1), dict(G=3), dict(F=1, G=2), dict(Ns=6), dict(Ns=-1), dict(act=9)):
        assert callb(**bad) == 1, bad
