"""Clips of different lengths in one improved_fullsubnet call (fsn_improved_enhance).  The existing forward gives every
clip the same bits at any batch size; on that, every clip of a mixed batch is bit-identical to the same clip enhanced
alone, whatever its length, its neighbours or the samples past its end, at every precision and n_fft (radix-2 and
direct DFT); the file loop's mixed-length batches write the same files as equal-length batches."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

WAV_TOL = 1e-4
PRECISIONS = ["fp32", "tf32_tc"]


def _variants():
    from oracle import improved_fullsubnet_oracle as IO
    return {"k16": IO.DEFAULT_IMPROVED_ARGS, "k48": IO.ARGS_48K_1024, "k48_960": IO.ARGS_48K_960}


VARIANTS = ["k16", "k48", "k48_960"]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _model(tag, precision, dev):
    from fullsubnet_b200.improved_fullsubnet.model import Model
    from oracle import improved_fullsubnet_oracle as IO
    args = _variants()[tag]
    m = Model(**args)
    m.load_state_dict(IO.make_improved_state_dict(seed=5, args=args), strict=True)
    m.precision = precision
    return m.to(dev).eval()


def _lengths(hop, n_fft, L_max):
    """The shortest clip (n_fft/2 + 1), a multiple of hop, hop*k - 1, odd and even frame counts, L_max."""
    return [n_fft // 2 + 1, hop * 20, hop * 25 - 1, hop * 15 + 5, hop * 21 + 3, L_max // 2 + 7, L_max]


def _mixed_batch(lengths, seed, sr):
    """[B, max(lengths)] rows of independent clips; the tail of every row is NaN or +-1e30 (never read)."""
    from oracle import fullsubnet_oracle as O
    y = O.make_noisy(len(lengths), max(lengths), seed=seed, speechlike=True, sr=sr)
    fills = (float("nan"), 1e30, -1e30)
    for b, Lb in enumerate(lengths):
        y[b, Lb:] = fills[b % 3]
    return y


@pytest.mark.parametrize("tag", ["k16", "k48_960"])
@pytest.mark.parametrize("precision", PRECISIONS)
def test_forward_is_batch_invariant(dev, tag, precision):
    """model(y) on 3 equal-length clips gives each clip the bits of model(y[i:i+1])."""
    from oracle import fullsubnet_oracle as O
    m = _model(tag, precision, dev)
    y = O.make_noisy(3, 3 * m.hop_length * 40 + 11, seed=21, speechlike=True).to(dev)
    with torch.no_grad():
        out = m(y)
        for i in range(3):
            assert torch.equal(out[i:i + 1], m(y[i:i + 1])), i


@pytest.mark.parametrize("tag", VARIANTS)
@pytest.mark.parametrize("precision", PRECISIONS)
def test_mixed_batch_equals_single_clip_calls(dev, tag, precision):
    m = _model(tag, precision, dev)
    hop, n_fft, F = m.hop_length, m.n_fft, m.num_freqs
    sr = 16000 if tag == "k16" else 48000
    lengths = _lengths(hop, n_fft, sr)
    yd = _mixed_batch(lengths, seed=3, sr=sr).to(dev)
    B, L_max = yd.shape
    T_max = 1 + L_max // hop
    enh, crm = m.enhance(yd, lengths=lengths, return_crm=True)
    enh2, pcm = m.enhance_pcm(yd, lengths=lengths)
    assert enh.shape == (B, L_max) and crm.shape == (B, 2, F, T_max) and pcm.shape == (B, L_max)
    assert torch.isfinite(enh).all() and torch.isfinite(crm).all()
    assert torch.equal(enh, enh2)
    assert not crm[:, :, F - 1].any()  # Nyquist row
    for b, Lb in enumerate(lengths):
        Tb = 1 + Lb // hop
        with torch.no_grad():
            one, crm1 = m(yd[b:b + 1, :Lb], return_crm=True)
        one2, pcm1 = m.enhance_pcm(yd[b:b + 1, :Lb])
        assert torch.equal(enh[b, :Lb], one[0, 0]), (b, Lb)
        assert torch.equal(crm[b, :, :, :Tb], crm1[0]), (b, Lb)
        assert torch.equal(one2[0], one[0, 0]) and torch.equal(pcm[b, :Lb], pcm1[0]), (b, Lb)
        assert not enh[b, Lb:].any() and not crm[b, :, :, Tb:].any() and not pcm[b, Lb:].any(), (b, Lb)


@pytest.mark.parametrize("tag", VARIANTS)
def test_equal_lengths_give_the_forward(dev, tag):
    from fullsubnet_b200 import _lib
    from oracle import fullsubnet_oracle as O
    m = _model(tag, "auto", dev)
    L = m.hop_length * 30 + 17
    y = O.make_noisy(3, L, seed=5, speechlike=True).to(dev)
    with torch.no_grad():
        ref, ref_crm = m(y, return_crm=True)
    for lengths in (None, [L] * 3, torch.tensor([L] * 3)):
        enh, crm = m.enhance(y, lengths=lengths, return_crm=True)
        assert torch.equal(enh, ref[:, 0]) and torch.equal(crm, ref_crm), lengths
        enh2, pcm = m.enhance_pcm(y, lengths=lengths)
        assert torch.equal(enh2, ref[:, 0]), lengths
        want = torch.empty_like(pcm)
        _lib.check(_lib.load().fsn_peak_normalize_int16(enh2.data_ptr(), 3, L, 0.8 * 32767.0, want.data_ptr(),
                                                        _lib.stream_ptr(dev)))
        assert torch.equal(pcm, want), lengths


@pytest.mark.parametrize("precision", PRECISIONS)
def test_mixed_batch_matches_reference(dev, precision):
    """Two clips of a mixed batch against the CPU oracle on each clip alone (as test_improved_fullsubnet_matches_reference:
    waveform max-abs < 1e-4, < 1e-6 on fp32)."""
    from oracle import improved_fullsubnet_oracle as IO
    m = _model("k16", precision, dev)
    lengths = [12000, 7001, 9472]
    y = _mixed_batch(lengths, seed=13, sr=16000)
    enh = m.enhance(y.to(dev), lengths=lengths)
    sd = IO.make_improved_state_dict(seed=5, args=IO.DEFAULT_IMPROVED_ARGS)
    for b in (0, 1):
        Lb = lengths[b]
        ref = IO.improved_forward(y[b:b + 1, :Lb], sd, IO.DEFAULT_IMPROVED_ARGS)[0, 0].numpy()
        err = np.abs(enh[b, :Lb].cpu().numpy() - ref).max()
        print(f"improved mixed batch {precision} clip {b}: waveform max-abs {err:.2e}")
        assert err < (1e-6 if precision == "fp32" else WAV_TOL), (b, err)


def test_large_mixed_batch(dev):
    """128 clips of 0.5 - 2 s at 48 kHz (n_fft 960) in one call: finite outputs, one clip placed twice among neighbours
    of different lengths gives the same bits both times, and the shortest / longest / a middle clip equal their
    single-clip calls."""
    from oracle import fullsubnet_oracle as O
    m = _model("k48_960", "auto", dev)
    rng = np.random.default_rng(77)
    lengths = rng.integers(24000, 96001, size=128).tolist()
    lengths[7] = lengths[100] = 50001
    y = O.make_noisy(128, max(lengths), seed=77, sr=48000)
    y[100] = y[7]
    for b, Lb in enumerate(lengths):
        y[b, Lb:] = float("nan")
    yd = y.to(dev)
    out, pcm = m.enhance_pcm(yd, lengths=lengths)
    torch.cuda.synchronize()
    assert torch.isfinite(out).all()
    assert torch.equal(out[7], out[100]) and torch.equal(pcm[7], pcm[100])
    assert lengths[6] != lengths[99] and lengths[8] != lengths[101]
    for i in (int(np.argmin(lengths)), int(np.argmax(lengths)), 64):
        Lb = lengths[i]
        single, pcm1 = m.enhance_pcm(yd[i:i + 1, :Lb])
        assert torch.equal(single[0], out[i, :Lb]) and torch.equal(pcm1[0], pcm[i, :Lb]), i


def test_file_loop_mixed_length_batches(dev, tmp_path, monkeypatch):
    """Inferencer(model=improved) at 48 kHz: enhance_files(max_padding=0.5) writes the same bytes as equal-length batches
    (max_padding=0), within 1 LSB of the reference host loop on model(y), with one library call per planned batch."""
    import wave
    from fullsubnet_b200.inferencer import Inferencer, plan_batches
    from oracle import fullsubnet_oracle as O
    m = _model("k48_960", "auto", dev)
    inf = Inferencer(model=m, device=dev)
    assert (inf.n_fft, inf.hop_length) == (960, 480) and inf.supports_lengths()
    lens = [24000, 16000, 31111, 20480, 19999, 36000]
    paths = []
    for i, L in enumerate(lens):
        y = O.make_noisy(1, L, seed=50 + i, speechlike=True, sr=48000)[0].numpy()
        p = tmp_path / f"n{i}.wav"
        inf.write_wav(p, np.round(y / np.abs(y).max() * 20000).astype(np.int16), 48000)
        paths.append(p)
    calls = []
    orig = m._enhance_call
    monkeypatch.setattr(m, "_enhance_call", lambda *a: calls.append(a[1]) or orig(*a))
    mixed = inf.enhance_files(paths, tmp_path / "mixed", batch_size=3, sr=48000, max_padding=0.5)
    plan = plan_batches(lens, 3, 0.5)
    assert len(calls) == len(plan) < len(lens) and any(c is not None for c in calls)
    calls.clear()
    exact = inf.enhance_files(paths, tmp_path / "exact", batch_size=3, sr=48000, max_padding=0.0)
    assert len(calls) == len(lens) and all(c is None for c in calls)
    amp = np.iinfo(np.int16).max
    for p, q, r in zip(paths, mixed, exact):
        assert q.name == r.name == p.name and q.read_bytes() == r.read_bytes()
        noisy = torch.from_numpy(inf.load_wav(p, 48000))[None].to(dev)
        with torch.no_grad():
            enhanced = m(noisy)[0, 0].cpu().numpy()
        assert np.array_equal(inf.full_band_crm_mask(noisy, {}), enhanced)
        ref = np.int16(0.8 * amp * enhanced / np.max(np.abs(enhanced)))
        with wave.open(str(q)) as f:
            assert f.getframerate() == 48000
            got = np.frombuffer(f.readframes(f.getnframes()), dtype="<i2")
        assert got.shape == ref.shape
        assert np.abs(got.astype(np.int32) - ref).max() <= 1
