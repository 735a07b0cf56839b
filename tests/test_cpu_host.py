"""CPU-only checks: the C-ABI library builds, loads and exports every symbol declared in
include/fsn_b200.h; host-side logic (state_dict contract, error behaviour, sharding)."""
import os
import re
import shutil

import numpy as np
import pytest
import torch

from conftest import ROOT


@pytest.fixture(scope="module")
def lib():
    from fullsubnet_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        if shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"):
            pytest.skip("no nvcc and no prebuilt library")
        from fullsubnet_b200.csrc.build import build
        build()
    return _lib.load()


def test_library_exports_every_declared_symbol(lib):
    from fullsubnet_b200 import _lib
    header = open(os.path.join(ROOT, "include", "fsn_b200.h")).read()
    declared = set(re.findall(r"\b(fsn_[a-z0-9_]+)\s*\(", header))
    assert declared, "no declarations parsed"
    assert declared == set(_lib.EXPORTED_SYMBOLS), declared ^ set(_lib.EXPORTED_SYMBOLS)
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.fsn_version() >= 100
    assert lib.fsn_built_arch() == 90  # compiled for sm_90a


def test_workspace_queries_need_no_gpu(lib):
    import ctypes as C
    from fullsubnet_b200 import _lib
    d = _lib.ModelDesc(257, 2, 0, 15, 512, 384, 1, 0, 0, 2, 0, 0)
    n1 = lib.fsn_model_workspace_bytes(C.byref(d), 1, 251)
    n8 = lib.fsn_model_workspace_bytes(C.byref(d), 8, 251)
    assert 0 < n1 < n8
    assert lib.fsn_enhance_workspace_bytes(C.byref(d), 2, 64000, 512, 256) > n1
    # B == num_groups violates the reference's drop_band assertion (feature.py:317-319)
    assert lib.fsn_model_workspace_bytes(C.byref(d), 2, 251) == 0
    assert b"Batch size = 2" in lib.fsn_last_error()


def test_state_dict_contract_matches_reference():
    from fullsubnet_b200.fullsubnet.model import Model
    from oracle import fullsubnet_oracle as O
    m = Model(**O.DEFAULT_MODEL_ARGS)
    sd = m.state_dict()
    want = O.state_dict_shapes()
    assert list(sd.keys()) == [k for k, _ in want]
    assert [tuple(v.shape) for v in sd.values()] == [s for _, s in want]
    assert sum(v.numel() for v in sd.values()) == 5637635  # SURVEY: "5.6 M"
    # reference checkpoints (incl. DDP 'module.' prefix handling of base_inferencer.py:154-156) load strictly
    ref_sd = {"module." + k: v for k, v in O.make_state_dict(0).items()}
    m.load_state_dict({k.replace("module.", ""): v for k, v in ref_sd.items()}, strict=True)
    assert m.num_groups_in_drop_band == 2 and hasattr(m, "fb_model") and hasattr(m, "sb_model")
    # usable by the reference's optimizer / clip path (train.py:55-59, trainer.py:65-67)
    opt = torch.optim.Adam(m.parameters(), lr=1e-3, betas=(0.9, 0.999))
    assert len(opt.param_groups[0]["params"]) == 20


def test_host_error_behaviour_matches_reference():
    from fullsubnet_b200.fullsubnet.model import Model
    from fullsubnet_b200.acoustics import feature
    from oracle import fullsubnet_oracle as O
    with pytest.raises(AssertionError):
        Model(**dict(O.DEFAULT_MODEL_ARGS, sequence_model="SRU"))
    with pytest.raises(NotImplementedError):
        Model(**dict(O.DEFAULT_MODEL_ARGS, norm_type="bogus"))
    m = Model(**O.DEFAULT_MODEL_ARGS).eval()
    with pytest.raises(AssertionError):
        m(torch.zeros(1, 257, 5))  # model.py:84
    with pytest.raises(AssertionError):
        m(torch.zeros(1, 2, 257, 5))  # model.py:87-89
    with pytest.raises(RuntimeError, match="no CPU path"):
        m(torch.zeros(1, 1, 257, 5))  # no silent CPU fallback
    with pytest.raises(AssertionError):
        feature.stft(torch.zeros(4), 512, 256, 512)  # feature.py:25
    with pytest.raises(AssertionError):
        feature.drop_band(torch.zeros(2, 1, 8, 3), 2)  # feature.py:317-319
    with pytest.raises(NotImplementedError):
        feature.istft((torch.zeros(1, 257, 3), torch.zeros(1, 257, 3)), 512, 256, 512, input_type="bogus")


def test_initialize_module_plugin_mechanism():
    from fullsubnet_b200.utils import initialize_module
    from oracle import fullsubnet_oracle as O
    m = initialize_module("fullsubnet_b200.fullsubnet.model.Model", args=dict(O.DEFAULT_MODEL_ARGS))
    assert type(m).__name__ == "Model"
    cls = initialize_module("fullsubnet_b200.inferencer.Inferencer", initialize=False)
    assert cls.__name__ == "Inferencer"


def test_fast_fullsubnet_state_dict_contract():
    from fullsubnet_b200.fast_fullsubnet.model import Model
    from oracle import fast_fullsubnet_oracle as FO
    m = Model(**FO.DEFAULT_FAST_ARGS)
    sd = m.state_dict()
    want = FO.fast_state_dict_shapes()  # validated against the reference by oracle/make_golden.py (strict load)
    assert list(sd.keys()) == [k for k, _ in want] and [tuple(v.shape) for v in sd.values()] == [s for _, s in want]
    assert sum(p.numel() for p in m.parameters()) == 6842895  # SURVEY 8a row A13
    assert torch.allclose(sd["mel_scale.fb"], FO.melscale_fbanks(257, 64))
    m.load_state_dict(FO.make_fast_state_dict(3), strict=True)
    with pytest.raises(RuntimeError):
        m.eval()(torch.zeros(1, 1, 257, 4))  # no CPU path


def test_improved_fullsubnet_state_dict_contract():
    from fullsubnet_b200.improved_fullsubnet.model import Model
    from oracle import improved_fullsubnet_oracle as IO
    for args in (IO.DEFAULT_IMPROVED_ARGS, IO.ARGS_48K_1024):
        m = Model(**args)
        sd = m.state_dict()
        want = IO.improved_state_dict_shapes(args)  # validated against the reference by oracle/make_golden.py
        assert list(sd.keys()) == [k for k, _ in want]
        assert [tuple(v.shape) for v in sd.values()] == [s for _, s in want]
        m.load_state_dict(IO.make_improved_state_dict(5, args), strict=True)
        with pytest.raises(RuntimeError):
            m.eval()(torch.zeros(1, 2000))  # no CPU path
    with pytest.raises(NotImplementedError):
        Model(norm_type="cumulative_laplace_norm")


def test_training_host_objects_without_gpu():
    """Optimiser state is interchangeable with torch.optim.Adam; loss / optimiser / train forward refuse CPU tensors."""
    from fullsubnet_b200.fullsubnet.model import Model
    from fullsubnet_b200.loss import mse_loss, MSELoss
    from fullsubnet_b200.optim import FusedClipAdam
    from fullsubnet_b200.trainer import Trainer  # noqa: F401  (importable without CUDA)
    m = Model(num_freqs=9, look_ahead=1, sequence_model="LSTM", fb_num_neighbors=0, sb_num_neighbors=2,
              fb_output_activate_function="ReLU", sb_output_activate_function=False, fb_model_hidden_size=8,
              sb_model_hidden_size=4, weight_init=False)
    assert mse_loss is MSELoss
    opt = FusedClipAdam(m.parameters(), lr=1e-3, max_norm=10.0)
    ref = torch.optim.Adam(m.parameters(), lr=1e-3)
    assert set(opt.state_dict()["param_groups"][0]) >= {"lr", "betas", "eps", "weight_decay", "amsgrad", "params"}
    for p in m.parameters():
        p.grad = torch.ones_like(p)
    ref.step()
    opt.load_state_dict(ref.state_dict())  # torch -> fused
    assert int(opt.state[next(iter(m.parameters()))]["step"]) == 1
    with pytest.raises(RuntimeError):
        opt.step()  # no CPU path
    with pytest.raises(RuntimeError):
        mse_loss()(torch.zeros(1, 2, 3, 2), torch.zeros(1, 2, 3, 2))
    with pytest.raises(RuntimeError):
        m.train()(torch.zeros(3, 1, 9, 5))
    assert m._resolve_train_precision() == "tf32_tc"
    m.train_precision = "bf16"
    with pytest.raises(ValueError):
        m._resolve_train_precision()


def test_fullband_baseline_state_dict_contract():
    from fullsubnet_b200.fullband_baseline.model import Model
    from oracle import fullband_baseline_oracle as BO
    m = Model(**BO.DEFAULT_FBB_ARGS)
    want = BO.fbb_state_dict_shapes()  # validated against the reference by oracle/make_golden_fbb.py
    sd = m.state_dict()
    assert list(sd.keys()) == [k for k, _ in want] and [tuple(v.shape) for v in sd.values()] == [s for _, s in want]
    m.load_state_dict(BO.make_fbb_state_dict(11), strict=True)
    with pytest.raises(RuntimeError), torch.no_grad():
        m.eval()(torch.zeros(1, 1, 257, 4))  # no CPU path


def test_workspace_queries_report_error_class_without_gpu():
    """*_workspace_bytes() run no CUDA code: they can be exercised on the CPU box (sizes, error classes)."""
    import ctypes as C
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    d = _lib.ModelDesc(num_freqs=257, look_ahead=2, fb_num_neighbors=0, sb_num_neighbors=15, fb_hidden=512, sb_hidden=384,
                       fb_activation=1, sb_activation=0, norm_type=0, num_groups_in_drop_band=2, precision=2, cell_type=0)
    n = lib.fsn_train_workspace_bytes(C.byref(d), 64, 188)
    assert 40e9 < n < 50e9  # config 3: 28.7 GB of saved activations + transposed copies and scratch
    assert lib.fsn_train_workspace_bytes(C.byref(d), 2, 188) == 0  # B == G (feature.py:317-319)
    assert lib.fsn_last_error_code() == _lib.FSN_ERR_SHAPE and b"Batch size" in lib.fsn_last_error()
    d.norm_type = 1
    assert lib.fsn_train_workspace_bytes(C.byref(d), 64, 188) > n  # cumulative norm: + the per-step scale tables
    d.norm_type, d.cell_type, d.precision = 0, 1, 2
    assert lib.fsn_model_workspace_bytes(C.byref(d), 4, 100) == 0  # GRU is built for the fp32 inference kernels only
    assert lib.fsn_last_error_code() == _lib.FSN_ERR_UNSUPPORTED
    with pytest.raises(NotImplementedError):
        _lib.check_workspace(0)
    f = _lib.FullbandDesc(num_freqs=257, hidden=512, num_layers=3, look_ahead=2, activation=0, norm_type=0)
    assert lib.fsn_fullband_workspace_bytes(C.byref(f), 4, 100) > 0
    f.num_layers = 9
    assert lib.fsn_fullband_workspace_bytes(C.byref(f), 4, 100) == 0 and lib.fsn_last_error_code() == _lib.FSN_ERR_UNSUPPORTED
    # GRU: the fullband_baseline and fast_fullsubnet forwards have LSTM kernels only
    f.num_layers, f.cell_type = 3, 1
    assert lib.fsn_fullband_workspace_bytes(C.byref(f), 4, 100) == 0 and lib.fsn_last_error_code() == _lib.FSN_ERR_UNSUPPORTED
    fd = _lib.FastDesc(num_freqs=257, look_ahead=2, shrink_size=2, num_mels=64, enc1_hidden=384, enc2_hidden=257,
                       bn_hidden=384, bn_layers=2, dec_hidden=512, noisy_num_neighbors=5, enc_num_neighbors=0, precision=0,
                       cell_type=0)
    assert lib.fsn_fast_workspace_bytes(C.byref(fd), 4, 100) > 0 and lib.fsn_fast_packed_bytes(C.byref(fd)) > 0
    fd.cell_type = 1
    assert lib.fsn_fast_workspace_bytes(C.byref(fd), 4, 100) == 0 and lib.fsn_last_error_code() == _lib.FSN_ERR_UNSUPPORTED
    assert lib.fsn_fast_packed_bytes(C.byref(fd)) == 0


def test_write_wav_roundtrip(tmp_path):
    import wave
    from fullsubnet_b200.inferencer import Inferencer
    pcm = (np.arange(-500, 500) * 30).astype(np.int16)
    Inferencer.write_wav(tmp_path / "x.wav", pcm, 48000)
    with wave.open(str(tmp_path / "x.wav")) as f:
        assert (f.getnchannels(), f.getsampwidth(), f.getframerate(), f.getnframes()) == (1, 2, 48000, 1000)
        assert np.array_equal(np.frombuffer(f.readframes(1000), dtype="<i2"), pcm)


def test_c_abi_arguments_are_validated_without_gpu():
    """Every entry point validates its arguments before touching CUDA: the error classes of the reference's asserts can
    be checked on the CPU box (no kernel is launched by these calls)."""
    import ctypes as C
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    assert lib.fsn_stft(None, 1, 1000, 511, 256, 511, None, None, None, None, None, 0, None) == _lib.FSN_ERR_UNSUPPORTED
    assert b"n_fft=511" in lib.fsn_last_error()
    assert lib.fsn_stft(None, 1, 1000, 512, 0, 512, None, None, None, None, None, 0, None) == _lib.FSN_ERR_SHAPE
    assert lib.fsn_stft(None, 1, 100, 512, 256, 512, None, None, None, None, None, 0, None) == _lib.FSN_ERR_SHAPE  # pad >= L
    assert lib.fsn_stft(None, 0, 1000, 960, 480, 960, None, None, None, None, None, 0, None) == _lib.FSN_ERR_SHAPE
    assert lib.fsn_istft(None, None, 3, None, 1, 4, 512, 256, 512, 0, None, None) == _lib.FSN_ERR_SHAPE  # cstride
    assert lib.fsn_mse_loss(None, None, 0, 4, 4, None, None, None, 0, None) == _lib.FSN_ERR_SHAPE
    L = _lib.ParamList()
    L.n = 1
    assert lib.fsn_clip_adam(C.byref(L), 10.0, 1.0, 1e-3, 0.9, 0.999, 1e-8, 0, None, None, 0, None) == _lib.FSN_ERR_SHAPE
    L.n = _lib.MAX_PARAM_TENSORS + 1
    assert lib.fsn_clip_adam(C.byref(L), 10.0, 1.0, 1e-3, 0.9, 0.999, 1e-8, 1, None, None, 0, None) == _lib.FSN_ERR_SHAPE
    assert lib.fsn_peak_normalize_int16(None, 0, 10, 1.0, None, None) == _lib.FSN_ERR_SHAPE
    # entry points added in round 2
    assert lib.fsn_si_sdr(None, None, 0, 100, None, None) == _lib.FSN_ERR_SHAPE
    assert lib.fsn_snr_mix(None, None, None, None, -25.0, 1e-6, 4, 0, None, None, None) == _lib.FSN_ERR_SHAPE
    assert lib.fsn_rir_convolve(None, None, None, 2, 100, 0, None, None) == _lib.FSN_ERR_SHAPE
    d = _lib.ModelDesc(num_freqs=257, look_ahead=2, fb_num_neighbors=0, sb_num_neighbors=15, fb_hidden=512, sb_hidden=384,
                       fb_activation=1, sb_activation=0, norm_type=0, num_groups_in_drop_band=1, precision=3, cell_type=0)
    # the float output is required, also when only the int16 one is wanted (a stand-in pcm pointer, never written: each
    # call returns before any CUDA call)
    assert lib.fsn_enhance(C.byref(d), None, None, None, None, None, 2, 4000, 512, 256, 512, None, None, 16, 1.0, None, 0,
                           None) == _lib.FSN_ERR_SHAPE
    assert b"enhanced" in lib.fsn_last_error()
    fbb = _lib.FullbandDesc(num_freqs=257, hidden=512, num_layers=3, look_ahead=2, activation=0, norm_type=0, precision=0,
                            cell_type=0)
    assert lib.fsn_fullband_enhance(C.byref(fbb), None, None, None, None, None, 2, 4000, 512, 256, 512, None, None, 16, 1.0,
                                    None, 0, None) == _lib.FSN_ERR_SHAPE
    assert b"enhanced" in lib.fsn_last_error()
    from fullsubnet_b200.improved_fullsubnet.model import Model as Improved
    imp = Improved()._desc("fp32")
    assert lib.fsn_improved_enhance(C.byref(imp), None, None, None, 2, 4000, None, None, 16, 1.0, None, 0, None) \
        == _lib.FSN_ERR_SHAPE
    assert b"enhanced" in lib.fsn_last_error()
    assert lib.fsn_enhance_workspace_bytes(C.byref(d), 2, 4000, 512, 256) > 0
    d.cell_type = 1  # GRU with a tensor-core precision
    assert lib.fsn_enhance_workspace_bytes(C.byref(d), 2, 4000, 512, 256) == 0
    assert lib.fsn_last_error_code() == _lib.FSN_ERR_UNSUPPORTED and b"GRU" in lib.fsn_last_error()
    with pytest.raises(AssertionError):
        _lib.check(_lib.FSN_ERR_SHAPE)
    with pytest.raises(NotImplementedError):
        _lib.check(_lib.FSN_ERR_UNSUPPORTED)
    with pytest.raises(RuntimeError):
        _lib.check(_lib.FSN_ERR_CUDA)


def test_lstm_train_hook_checks_arguments_without_gpu():
    """fsn_debug_lstm_train (the shared training LSTM layer alone) rejects every bad argument with its error class before
    any CUDA call, and its workspace query needs no GPU: non-zero, growing with the layer count, the rows and the steps."""
    import ctypes as C
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    q = lib.fsn_debug_lstm_train_workspace_bytes
    fp32, tf32 = _lib.PREC["fp32"], _lib.PREC["tf32_tc"]
    for prec in (fp32, tf32):
        n = q(2, 31, 6, 20, 64, prec)
        assert n > 0
        assert q(3, 31, 6, 20, 64, prec) > n and q(2, 32, 6, 20, 64, prec) > n and q(2, 31, 7, 20, 64, prec) > n
        assert q(8, 31, 6, 20, 64, prec) > q(3, 31, 6, 20, 64, prec)
    assert q(2, 31, 6, 20, 64, tf32) > q(2, 31, 6, 20, 64, fp32)  # transposed weights, K-major and fp16 copies
    assert q(2, 31, 6, 20, 257, tf32) == q(2, 31, 6, 20, 257, fp32)  # H % 4 != 0: the fp32 kernels and layout
    for args, code in (((0, 4, 5, 8, 32, fp32), _lib.FSN_ERR_UNSUPPORTED), ((9, 4, 5, 8, 32, fp32), _lib.FSN_ERR_UNSUPPORTED),
                       ((2, 4, 5, 8, 32, _lib.PREC["f16_tc"]), _lib.FSN_ERR_UNSUPPORTED),
                       ((2, 0, 5, 8, 32, fp32), _lib.FSN_ERR_SHAPE), ((2, 4, 0, 8, 32, fp32), _lib.FSN_ERR_SHAPE),
                       ((2, 4, 5, 0, 32, fp32), _lib.FSN_ERR_SHAPE), ((2, 4, 5, 8, 0, fp32), _lib.FSN_ERR_SHAPE),
                       ((1, 1 << 16, 1 << 10, 8, 32, fp32), _lib.FSN_ERR_SHAPE)):  # 2^31 floats in one gate buffer
        assert q(*args) == 0, args
        assert lib.fsn_last_error_code() == code, (args, lib.fsn_last_error())

    # the hook itself: stand-in device pointers, never dereferenced because every check fails before the first launch
    n, R, T, K0, H = 2, 4, 5, 8, 32
    p = 1 << 20

    def layers():
        return (_lib.LstmLayer * n)(*[_lib.LstmLayer(p, p, p, p) for _ in range(n)])

    def grads():
        return (_lib.LstmGrads * n)(*[_lib.LstmGrads(p, p, p, p) for _ in range(n)])

    need = q(n, R, T, K0, H, fp32)

    def call(n=n, R=R, prec=fp32, x=p, dh=p, dout=None, fc_w=None, O=0, L=None, g=None, ws=p, nbytes=need):
        return lib.fsn_debug_lstm_train(L if L is not None else layers(), n, R, T, K0, H, prec, x, dh, dout, fc_w, O, p, p,
                                        g if g is not None else grads(), None, ws, nbytes, None)

    assert call(n=0) == _lib.FSN_ERR_UNSUPPORTED and call(n=9) == _lib.FSN_ERR_UNSUPPORTED
    assert call(prec=_lib.PREC["f16x3_tc"]) == _lib.FSN_ERR_UNSUPPORTED
    assert call(R=-1) == _lib.FSN_ERR_SHAPE
    assert call(x=None) == _lib.FSN_ERR_SHAPE
    assert call(dh=None) == _lib.FSN_ERR_SHAPE and b"no gradient on top" in lib.fsn_last_error()
    assert call(dout=p, O=2) == _lib.FSN_ERR_SHAPE  # a Linear on top without its weight
    assert call(dout=p, fc_w=p, O=0) == _lib.FSN_ERR_SHAPE
    assert call(O=1) == _lib.FSN_ERR_SHAPE  # O with no fc_w
    bad = grads()
    bad[1].b_hh = None
    assert call(g=bad) == _lib.FSN_ERR_SHAPE and b"layer 1" in lib.fsn_last_error()
    bad = layers()
    bad[0].w_ih = None
    assert call(L=bad) == _lib.FSN_ERR_SHAPE
    assert call(nbytes=need - 1) == _lib.FSN_ERR_WORKSPACE
    assert call(ws=None) == _lib.FSN_ERR_WORKSPACE
    assert call(prec=tf32, nbytes=need) == _lib.FSN_ERR_WORKSPACE  # the tensor-core layout is larger


def test_row_map_and_reflect_count_match_oracle():
    """The drop_band row map (feature.py:332-345) and its inverse as compiled into the library vs the oracle's index
    form; reflect multiplicity c[r] of the closed-form second norm (SURVEY A6) vs the oracle and its closed values."""
    import ctypes as C
    from hypothesis import given, settings, strategies as st
    from fullsubnet_b200 import _lib
    from oracle import fullsubnet_oracle as O
    lib = _lib.load()

    @settings(max_examples=60, deadline=None)
    @given(st.integers(1, 9), st.integers(2, 40), st.integers(1, 4))
    def check(B, F, G):
        if B > 1 and G > 1 and B <= G:
            return  # rejected by Model.forward (feature.py:317-319)
        if B > 1 and G > 1:
            sb_, sf_ = O.drop_band_index_map(B, F, G)
            want = [(int(sb_[i]), int(f)) for i in range(len(sb_)) for f in sf_[i]]
        else:
            want = [(b, f) for b in range(B) for f in range(F)]
        b, f = C.c_int(), C.c_int()
        seen = set()
        for r, (wb, wf) in enumerate(want):
            assert lib.fsn_debug_row_to_unit(B, F, G, r, C.byref(b), C.byref(f)) == 0
            assert (b.value, f.value) == (wb, wf)
            assert lib.fsn_debug_unit_to_row(B, F, G, wb, wf) == r  # inverse
            seen.add((wb, wf))
        assert lib.fsn_debug_row_to_unit(B, F, G, len(want), C.byref(b), C.byref(f)) == _lib.FSN_ERR_SHAPE
        for bb in range(B):
            for ff in range(F):
                if (bb, ff) not in seen:
                    assert lib.fsn_debug_unit_to_row(B, F, G, bb, ff) == -1  # dropped unit
    check()

    @settings(max_examples=40, deadline=None)
    @given(st.integers(2, 300), st.integers(0, 20))
    def check_count(F, N):
        if N >= F:
            return
        want = O.reflect_count(F, N)
        got = [lib.fsn_debug_reflect_count(r, F, N) for r in range(F)]
        assert got == list(want) and sum(got) == F * (2 * N + 1)
    check_count()
    c = [lib.fsn_debug_reflect_count(r, 257, 15) for r in range(257)]
    assert c[0] == c[256] == 16 and set(c[1:16]) == {32} and set(c[16:241]) == {31}  # SURVEY A6


def test_wav_load_resample_write_roundtrip(tmp_path):
    """Host loop pieces around the path (SURVEY 8f rank 2): stdlib wav I/O with librosa's int -> float scaling, channel
    mean, and the windowed-sinc resampler (48 kHz -> 16 kHz keeps an in-band tone to 1e-4)."""
    from fullsubnet_b200.inferencer import Inferencer
    t = np.arange(48000) / 48000.0
    y = (0.5 * np.sin(2 * np.pi * 440 * t)).astype(np.float32)
    pcm = np.round(y * 32767).astype(np.int16)
    Inferencer.write_wav(tmp_path / "a.wav", pcm, 48000)
    same = Inferencer.load_wav(tmp_path / "a.wav", 48000)
    assert same.dtype == np.float32 and np.array_equal(same, pcm.astype(np.float32) / 32768.0)
    z = Inferencer.load_wav(tmp_path / "a.wav", 16000)
    ref = 0.5 * np.sin(2 * np.pi * 440 * np.arange(len(z)) / 16000.0)
    assert len(z) == 16000 and np.abs(z[200:-200] - ref[200:-200]).max() < 2e-4
    import wave
    with wave.open(str(tmp_path / "st.wav"), "wb") as f:  # stereo: channels are averaged
        f.setnchannels(2); f.setsampwidth(2); f.setframerate(16000)
        f.writeframes(np.stack([pcm[:100], -pcm[:100]], 1).astype("<i2").tobytes())
    assert np.abs(Inferencer.load_wav(tmp_path / "st.wav", 16000)).max() == 0.0


def test_environment_switches_match_the_design_appendix():
    """Each FSN_* variable the library, the Python host or the bench scripts read appears in DESIGN.md (appendix
    "diagnostic switches"), so a maintainer can find what a switch does without reading the kernels; and every variable
    a row of that appendix names is still read somewhere, so the appendix lists no removed switch."""
    import glob
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    files = glob.glob(os.path.join(root, "fullsubnet_b200", "csrc", "*.cu")) + glob.glob(os.path.join(root, "fullsubnet_b200", "csrc", "*.cuh"))
    files += glob.glob(os.path.join(root, "fullsubnet_b200", "**", "*.py"), recursive=True)
    files += [os.path.join(root, "bench.py"), os.path.join(root, "bench_train.py")]
    names = set()
    for f in files:
        text = open(f).read()
        names |= set(re.findall(r'getenv\("(FSN_[A-Z0-9_]+)"', text))
        names |= set(re.findall(r'environ(?:\.get)?[\(\[]"(FSN_[A-Z0-9_]+)"', text))
    assert {"FSN_TC_STAGES", "FSN_TRAIN_PRECISION", "FSN_EXTRA_NVCC_FLAGS"} <= names, names  # the scanner finds all kinds
    doc = open(os.path.join(root, "DESIGN.md")).read()
    missing = sorted(n for n in names if n not in doc)
    assert not missing, missing
    appendix = doc.split("## Appendix: diagnostic switches", 1)[1].split("\n## ", 1)[0]
    rows = [line for line in appendix.splitlines() if line.startswith("| `")]
    listed = {n for line in rows for n in re.findall(r"`(FSN_[A-Z0-9_]+)", line)}
    assert {"FSN_TC_STAGES", "FSN_NO_REC_TC"} <= listed, listed
    stale = sorted(listed - names)
    assert not stale, stale
