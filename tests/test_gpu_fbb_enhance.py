"""fullband_baseline wav -> wav in one call (fsn_fullband_enhance).  Model.forward gives every clip the same bits at any
batch size with both norms; on that, the fused call with null lengths is the three-call path (fsn_stft -> Model.forward
-> fsn_istft) bit for bit, every clip of a mixed batch is bit-identical to the same clip enhanced alone, and the file
loop's mixed-length batches write the same files as equal-length batches.  Against the unmodified reference: cRM within
2e-5 relative, waveform within 1e-4 absolute, on every weight set."""
import numpy as np
import pytest
import torch

from conftest import rel_max

pytestmark = pytest.mark.gpu

NORMS = ["offline_laplace_norm", "cumulative_laplace_norm"]
CRM_GATE = 2e-5   # relative max-abs (test_fullband_baseline_matches_reference)
WAV_GATE = 1e-4   # absolute


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _args(norm="offline_laplace_norm", **kw):
    from oracle import fullband_baseline_oracle as BO
    return dict(BO.DEFAULT_FBB_ARGS, norm_type=norm, **kw)


def _small_args():
    return _args("cumulative_laplace_norm", num_freqs=33, hidden_size=32, output_activate_function="ReLU")


def _model(args, dev, fc_gain=1.0):
    from fullsubnet_b200.fullband_baseline.model import Model
    from oracle import fullband_baseline_oracle as BO
    sd = BO.make_fbb_state_dict(seed=11, args=args)
    for k in ("fullband_model.fc_output_layer.weight", "fullband_model.fc_output_layer.bias"):
        sd[k] = sd[k] * fc_gain
    m = Model(**args)
    m.load_state_dict(sd, strict=True)
    return m.to(dev).eval()


def _mixed_batch(lengths, seed):
    """[B, max(lengths)] rows of independent clips; the tail of every row is NaN or +-1e30 (never read)."""
    from oracle import fullsubnet_oracle as O
    y = O.make_noisy(len(lengths), max(lengths), seed=seed, speechlike=True)
    fills = (float("nan"), 1e30, -1e30)
    for b, Lb in enumerate(lengths):
        y[b, Lb:] = fills[b % 3]
    return y


def _three_calls(m, y, n_fft, hop):
    """The path Inferencer.enhance_batch took before the fused call: fsn_stft -> Model.forward -> fsn_istft."""
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    B, L = y.shape
    F, T = n_fft // 2 + 1, 1 + L // hop
    buf = torch.empty(3, B, F, T, dtype=torch.float32, device=y.device)
    out = torch.empty(B, L, dtype=torch.float32, device=y.device)
    st = _lib.stream_ptr(y.device)
    _lib.check(lib.fsn_stft(y.data_ptr(), B, L, n_fft, hop, n_fft, buf[0].data_ptr(), None, buf[1].data_ptr(),
                            buf[2].data_ptr(), None, 0, st))
    with torch.no_grad():
        crm = m(buf[0].unsqueeze(1)).contiguous()
    _lib.check(lib.fsn_istft(buf[1].data_ptr(), buf[2].data_ptr(), 1, crm.data_ptr(), B, T, n_fft, hop, n_fft, L,
                             out.data_ptr(), st))
    return out, crm, buf[0]


def _peak_int16(wav):
    from fullsubnet_b200 import _lib
    B, L = wav.shape
    want = torch.empty(B, L, dtype=torch.int16, device=wav.device)
    _lib.check(_lib.load().fsn_peak_normalize_int16(wav.data_ptr(), B, L, 0.8 * 32767.0, want.data_ptr(),
                                                    _lib.stream_ptr(wav.device)))
    return want


@pytest.mark.parametrize("norm", NORMS)
def test_forward_is_batch_invariant(dev, norm):
    """model(mag) on 3 equal-length clips gives each clip the bits of model(mag[i:i+1]), full size and small."""
    from oracle import fullsubnet_oracle as O
    for args, n_fft in ((_args(norm), 512), (_small_args(), 64)):
        m = _model(args, dev)
        y = O.make_noisy(3, n_fft // 2 * 60 + 11, seed=21, speechlike=True)
        mag = O.stft(y, n_fft, n_fft // 2, n_fft)[0].unsqueeze(1).to(dev)
        with torch.no_grad():
            out = m(mag)
            assert torch.isfinite(out).all()
            for i in range(3):
                assert torch.equal(out[i:i + 1], m(mag[i:i + 1])), (n_fft, i)


@pytest.mark.parametrize("norm", NORMS)
def test_null_lengths_equal_the_three_call_path(dev, norm):
    from oracle import fullsubnet_oracle as O
    m = _model(_args(norm), dev)
    L = 256 * 30 + 17
    y = O.make_noisy(3, L, seed=5, speechlike=True).to(dev)
    ref, ref_crm, _ = _three_calls(m, y, 512, 256)
    enh, crm = m.enhance(y, return_crm=True)
    assert torch.equal(enh, ref) and torch.equal(crm, ref_crm)
    enh2, pcm = m.enhance_pcm(y)
    assert torch.equal(enh2, ref) and torch.equal(pcm, _peak_int16(ref))
    # equal lengths given explicitly: the same bits
    enh3, crm3 = m.enhance(y, return_crm=True, lengths=[L] * 3)
    assert torch.equal(enh3, ref) and torch.equal(crm3, ref_crm)


def test_null_lengths_direct_dft(dev):
    """n_fft 960 (direct DFT) with null lengths: the three-call path's bits."""
    from oracle import fullsubnet_oracle as O
    m = _model(_args(num_freqs=481, hidden_size=128), dev)
    L = 480 * 20 + 33
    y = O.make_noisy(2, L, seed=6, speechlike=True, sr=48000).to(dev)
    ref, ref_crm, _ = _three_calls(m, y, 960, 480)
    enh, crm = m.enhance(y, 960, 480, 960, return_crm=True)
    assert torch.equal(enh, ref) and torch.equal(crm, ref_crm)


@pytest.mark.parametrize("norm", NORMS)
def test_mixed_batch_equals_single_clip_calls(dev, norm):
    hop, n_fft, F = 256, 512, 257
    m = _model(_args(norm), dev)
    L_max = 16000
    lengths = [n_fft // 2 + 1, hop * 20, hop * 25 - 1, hop * 15 + 5, L_max // 2 + 7, L_max]
    yd = _mixed_batch(lengths, seed=3).to(dev)
    B = len(lengths)
    T_max = 1 + L_max // hop
    enh, crm = m.enhance(yd, lengths=lengths, return_crm=True)
    enh2, pcm = m.enhance_pcm(yd, lengths=lengths)
    assert enh.shape == (B, L_max) and crm.shape == (B, 2, F, T_max) and pcm.shape == (B, L_max)
    assert torch.isfinite(enh).all() and torch.isfinite(crm).all()
    assert torch.equal(enh, enh2)
    for b, Lb in enumerate(lengths):
        Tb = 1 + Lb // hop
        one, crm1 = m.enhance(yd[b:b + 1, :Lb], return_crm=True)
        one2, pcm1 = m.enhance_pcm(yd[b:b + 1, :Lb])
        assert torch.equal(enh[b, :Lb], one[0]), (b, Lb)
        assert torch.equal(crm[b, :, :, :Tb], crm1[0]), (b, Lb)
        assert torch.equal(one2, one) and torch.equal(pcm[b, :Lb], pcm1[0]), (b, Lb)
        assert torch.equal(pcm1, _peak_int16(one)), (b, Lb)
        assert not enh[b, Lb:].any() and not crm[b, :, :, Tb:].any() and not pcm[b, Lb:].any(), (b, Lb)


def test_small_mixed_batch_equals_single_clip_calls(dev):
    """The small cumulative-norm configuration (n_fft 64, hidden 32: fp32 only)."""
    m = _model(_small_args(), dev)
    lengths = [33, 1201, 900, 64 * 10 - 1]
    yd = _mixed_batch(lengths, seed=8).to(dev)
    enh, crm = m.enhance(yd, 64, 32, 64, return_crm=True, lengths=lengths)
    for b, Lb in enumerate(lengths):
        one, crm1 = m.enhance(yd[b:b + 1, :Lb], 64, 32, 64, return_crm=True)
        assert torch.equal(enh[b, :Lb], one[0]) and torch.equal(crm[b, :, :, :1 + Lb // 32], crm1[0]), b


def _golden_sets():
    return [("small", _small_args(), 64), ("wa", _args(), 512), ("wb", _args(), 512)]


def test_matches_reference_wav(golden, dev):
    """One mixed batch per weight set of tests/golden/fullband_baseline_wav.npz (the unmodified reference model in
    Inferencer.full_band_crm_mask, one clip at a time): small cumulative-norm, W-a, and W-b past the +-9.9 clip."""
    g = golden("fullband_baseline_wav")
    for tag, args, n_fft in _golden_sets():
        m = _model(args, dev, float(g["wb_gain"]) if tag == "wb" else 1.0)
        lengths = g[tag + "_lengths"].tolist()
        enh, crm = m.enhance(torch.from_numpy(g[tag + "_y"]).to(dev), n_fft, n_fft // 2, n_fft, return_crm=True,
                             lengths=lengths)
        enh, crm = enh.cpu().numpy(), crm.cpu().numpy()
        wav_err, crm_err = float(np.abs(enh - g[tag + "_wav"]).max()), rel_max(crm, g[tag + "_crm"])
        print(f"fullband_baseline {tag}: cRM rel max {crm_err:.2e}, waveform max-abs {wav_err:.2e}")
        assert crm_err < CRM_GATE and wav_err < WAV_GATE, tag


def test_large_mixed_batch(dev):
    """64 clips of 1 - 10 s in one call: finite outputs, and the shortest, a middle and the longest clip equal their
    single-clip calls."""
    from oracle import fullsubnet_oracle as O
    m = _model(_args(), dev)
    rng = np.random.default_rng(64)
    lengths = rng.integers(16000, 160001, size=64).tolist()
    y = O.make_noisy(64, max(lengths), seed=64)
    for b, Lb in enumerate(lengths):
        y[b, Lb:] = float("nan")
    yd = y.to(dev)
    out, pcm = m.enhance_pcm(yd, lengths=lengths)
    torch.cuda.synchronize()
    assert torch.isfinite(out).all()
    for i in (int(np.argmin(lengths)), 32, int(np.argmax(lengths))):
        Lb = lengths[i]
        single, pcm1 = m.enhance_pcm(yd[i:i + 1, :Lb])
        assert torch.equal(single[0], out[i, :Lb]) and torch.equal(pcm1[0], pcm[i, :Lb]), i


def test_file_loop_mixed_length_batches(dev, tmp_path, monkeypatch):
    """Inferencer(model=fullband_baseline): enhance_files(max_padding=0.5) writes the same bytes as equal-length batches
    (max_padding=0), within 1 LSB of the reference host loop, with one library call per planned batch."""
    import wave
    from fullsubnet_b200.inferencer import Inferencer, plan_batches
    from oracle import fullsubnet_oracle as O
    m = _model(_args(), dev)
    inf = Inferencer(model=m, device=dev)
    assert inf.supports_lengths()
    lens = [6000, 4000, 7777, 5120, 4999, 9000]
    paths = []
    for i, L in enumerate(lens):
        y = O.make_noisy(1, L, seed=50 + i, speechlike=True)[0].numpy()
        p = tmp_path / f"n{i}.wav"
        inf.write_wav(p, np.round(y / np.abs(y).max() * 20000).astype(np.int16), 16000)
        paths.append(p)
    calls = []
    orig = m._enhance_call
    monkeypatch.setattr(m, "_enhance_call", lambda *a: calls.append(a[4]) or orig(*a))
    mixed = inf.enhance_files(paths, tmp_path / "mixed", batch_size=3, max_padding=0.5)
    plan = plan_batches(lens, 3, 0.5)
    assert len(calls) == len(plan) < len(lens) and any(c is not None for c in calls)
    calls.clear()
    exact = inf.enhance_files(paths, tmp_path / "exact", batch_size=3, max_padding=0.0)
    assert len(calls) == len(lens) and all(c is None for c in calls)
    amp = np.iinfo(np.int16).max
    for p, q, r in zip(paths, mixed, exact):
        assert q.name == r.name == p.name and q.read_bytes() == r.read_bytes()
        noisy = torch.from_numpy(inf.load_wav(p, 16000))[None].to(dev)
        enhanced = inf.full_band_crm_mask(noisy, {})
        ref = np.int16(0.8 * amp * enhanced / np.max(np.abs(enhanced)))
        with wave.open(str(q)) as f:
            got = np.frombuffer(f.readframes(f.getnframes()), dtype="<i2")
        assert got.shape == ref.shape
        assert np.abs(got.astype(np.int32) - ref).max() <= 1
