"""CPU-only checks of fullband_baseline's wav -> wav entry point (fsn_fullband_enhance) and its inference precision:
the workspace queries and argument checks answer before any CUDA call, the Python ``lengths`` and ``precision``
arguments, the Inferencer's rules, and the oracle restatement against the wav fixture of the unmodified reference."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import rel_max


def _model(**kw):
    from fullsubnet_b200.fullband_baseline.model import Model
    from oracle import fullband_baseline_oracle as BO
    return Model(**dict(BO.DEFAULT_FBB_ARGS, **kw))


def _desc(prec="fp32", **kw):
    from fullsubnet_b200 import _lib
    a = dict(num_freqs=257, hidden=512, num_layers=3, look_ahead=2, activation=0, norm_type=0,
             precision=_lib.PREC[prec], cell_type=0)
    a.update(kw)
    return _lib.FullbandDesc(**a)


def _call(lib, d, lengths, L_max, n_fft=512, enhanced=None):
    arr = None if lengths is None else (C.c_int32 * len(lengths))(*lengths)
    B = 2 if lengths is None else len(lengths)
    return lib.fsn_fullband_enhance(C.byref(d), None, None, None, None, arr, B, L_max, n_fft, n_fft // 2, n_fft, enhanced,
                                    None, None, 1.0, None, 0, None)


def test_fbb_workspace_queries_need_no_gpu():
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    for norm in (0, 1):
        fp32 = lib.fsn_fullband_enhance_workspace_bytes(C.byref(_desc("fp32", norm_type=norm)), 4, 64000, 512, 256)
        # the forward's workspace (T = 1 + L/hop frames) plus the spectrum, cRM, peak and length table
        assert fp32 > lib.fsn_fullband_workspace_bytes(C.byref(_desc("fp32", norm_type=norm)), 4, 251) > 0
        # the training precision runs the fp32 kernels in inference; the tensor-core precisions are not built here
        assert lib.fsn_fullband_enhance_workspace_bytes(C.byref(_desc("tf32_tc", norm_type=norm)), 4, 64000, 512, 256) == fp32
        for prec in ("f16x3_tc", "f16_tc"):
            bad = _desc(prec, norm_type=norm)
            assert lib.fsn_fullband_enhance_workspace_bytes(C.byref(bad), 4, 64000, 512, 256) == 0
            assert lib.fsn_last_error_code() == _lib.FSN_ERR_UNSUPPORTED
            assert lib.fsn_fullband_workspace_bytes(C.byref(bad), 4, 251) == 0
            assert lib.fsn_last_error_code() == _lib.FSN_ERR_UNSUPPORTED
    # n_fft 960 (direct DFT) is accepted with null lengths; n_fft / 2 + 1 must match num_freqs
    assert lib.fsn_fullband_enhance_workspace_bytes(C.byref(_desc(num_freqs=481)), 2, 48000, 960, 480) > 0
    assert lib.fsn_fullband_enhance_workspace_bytes(C.byref(_desc()), 2, 48000, 960, 480) == 0
    assert lib.fsn_last_error_code() == _lib.FSN_ERR_SHAPE


def test_fbb_enhance_checks_arguments_before_any_cuda_call():
    """No workspace, no weights, no device: every one of these fails on its argument check."""
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    d = _desc("fp32")
    assert _call(lib, d, [16000, 256, 3000], 16000) == _lib.FSN_ERR_SHAPE  # too short: <= n_fft/2
    assert b"clip 1" in lib.fsn_last_error()
    assert _call(lib, d, [16000, 16001, 3000], 16000) == _lib.FSN_ERR_SHAPE  # longer than the row
    assert b"clip 1" in lib.fsn_last_error()
    assert _call(lib, d, [15000, 257, 3000], 16000) == _lib.FSN_ERR_SHAPE  # max(lengths) != L_max
    assert b"15000" in lib.fsn_last_error()
    # valid lengths reach the workspace check, the last one before the first launch (a stand-in output pointer, never
    # written: the call returns before any CUDA call)
    assert _call(lib, d, [16000, 257, 3000], 16000, enhanced=16) == _lib.FSN_ERR_WORKSPACE
    assert _call(lib, d, None, 16000, enhanced=16) == _lib.FSN_ERR_WORKSPACE
    # per-clip lengths are built for the power-of-two transform; null lengths take every n_fft
    d960 = _desc(num_freqs=481)
    assert _call(lib, d960, [48000, 30000], 48000, 960) == _lib.FSN_ERR_UNSUPPORTED
    assert _call(lib, d960, None, 48000, 960, enhanced=16) == _lib.FSN_ERR_WORKSPACE
    # the tensor-core precisions and the GRU cell are refused, as by fsn_fullband_forward
    for prec in ("f16x3_tc", "f16_tc"):
        assert _call(lib, _desc(prec), None, 16000) == _lib.FSN_ERR_UNSUPPORTED
        assert _call(lib, _desc(prec), [16000, 3000], 16000) == _lib.FSN_ERR_UNSUPPORTED
    gru = _desc(cell_type=1)
    assert _call(lib, gru, None, 16000) == _lib.FSN_ERR_UNSUPPORTED
    assert lib.fsn_fullband_enhance_workspace_bytes(C.byref(gru), 2, 16000, 512, 256) == 0
    assert lib.fsn_last_error_code() == _lib.FSN_ERR_UNSUPPORTED


def test_fbb_python_lengths_argument_is_checked():
    m = _model()
    y = torch.zeros(3, 4000)
    for fn in (m.enhance, m.enhance_pcm):
        with pytest.raises(ValueError, match="entries"):
            fn(y, lengths=[4000, 3000])
        with pytest.raises(ValueError, match="exceeds"):
            fn(y, lengths=[4000, 4001, 300])
        with pytest.raises(ValueError):
            fn(y, lengths=torch.tensor([4000.0, 3000.0, 300.0]))
        with pytest.raises(RuntimeError, match="CUDA tensor"):  # valid lengths reach the device check
            fn(y, lengths=torch.tensor([4000, 3000, 300]))


def test_fbb_inferencer_takes_the_fused_path():
    from fullsubnet_b200.inferencer import Inferencer
    for n_fft, ok in ((512, True), (960, False)):
        inf = Inferencer.__new__(Inferencer)
        inf.model, inf.n_fft = _model(), n_fft
        assert inf.supports_lengths() is ok, n_fft


def test_fbb_precision_resolution(monkeypatch):
    """fp32 only: the constructor refuses the tensor-core precisions, and the FSN_PRECISION of the other models is not
    read (a process that sets it for fullsubnet keeps running fullband_baseline at fp32)."""
    from fullsubnet_b200 import _lib
    monkeypatch.delenv("FSN_PRECISION", raising=False)
    for p in (None, "auto", "fp32"):
        m = _model(precision=p)
        assert m._resolve_precision() == "fp32" and m._infer_desc().precision == _lib.PREC["fp32"]
    for env in ("f16x3_tc", "f16_tc", "fp32"):
        monkeypatch.setenv("FSN_PRECISION", env)
        assert _model()._resolve_precision() == "fp32", env
    for bad in ("f16x3_tc", "f16_tc", "tf32_tc"):
        with pytest.raises(ValueError, match="not built"):
            _model(precision=bad)._resolve_precision()
    # the training step keeps its own switch
    assert _model()._train_desc().precision in (_lib.PREC["fp32"], _lib.PREC["tf32_tc"])


def test_fbb_wav_oracle_matches_reference(golden):
    """The oracle restatement, inside the reference's full_band_crm_mask flow, against tests/golden/fullband_baseline_wav.npz
    (oracle/make_golden_fbb_wav.py: the unmodified reference model, one clip at a time)."""
    from oracle import fullband_baseline_oracle as BO
    from oracle import fullsubnet_oracle as O
    g = golden("fullband_baseline_wav")
    small = dict(BO.DEFAULT_FBB_ARGS, num_freqs=33, hidden_size=32, output_activate_function="ReLU",
                 norm_type="cumulative_laplace_norm")
    assert np.abs(g["wb_crm"]).max() > 9.9  # wb exercises the clip of decompress_cIRM
    for tag, a, n_fft in (("small", small, 64), ("wa", dict(BO.DEFAULT_FBB_ARGS), 512), ("wb", dict(BO.DEFAULT_FBB_ARGS), 512)):
        sd = BO.make_fbb_state_dict(seed=11, args=a)
        if tag == "wb":
            for k in ("fullband_model.fc_output_layer.weight", "fullband_model.fc_output_layer.bias"):
                sd[k] = sd[k] * float(g["wb_gain"])
        hop = n_fft // 2
        for b, L in enumerate(g[tag + "_lengths"].tolist()):
            assert L % hop, (tag, L)
            y = torch.from_numpy(g[tag + "_y"][b:b + 1, :L])
            mag, _, real, imag = O.stft(y, n_fft, hop, n_fft)
            crm = BO.fbb_forward(mag.unsqueeze(1), sd, a)
            m = O.decompress_cIRM(crm.permute(0, 2, 3, 1))
            er = m[..., 0] * real - m[..., 1] * imag
            ei = m[..., 1] * real + m[..., 0] * imag
            wav = O.istft((er, ei), n_fft, hop, n_fft, length=L, input_type="real_imag")
            Tb = crm.shape[-1]
            assert rel_max(crm, g[tag + "_crm"][b:b + 1, :, :, :Tb]) < 2e-5, (tag, b)
            assert not g[tag + "_crm"][b, :, :, Tb:].any() and not g[tag + "_wav"][b, L:].any()
            ref = g[tag + "_wav"][b, :L]
            assert np.abs(wav.numpy()[0] - ref).max() < 2e-5 * max(1.0, np.abs(ref).max()), (tag, b)
