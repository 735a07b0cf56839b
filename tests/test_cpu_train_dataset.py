"""fullsubnet_b200.dataset.Dataset against the unmodified training Dataset of the reference (tests/golden/dataset_train.npz,
oracle/make_golden_dataset.py): with the golden seeds, every item carries bit for bit the arguments the reference passes
to snr_mix, with and without preloading; the default collate stacks the items under the reference's DataLoader set-up;
the constructor refuses what the reference refuses.  No GPU."""
import random
import wave

import numpy as np
import pytest
import torch
from torch.utils.data import DataLoader, DistributedSampler

from fullsubnet_b200.dataset import Dataset, load_wav
from oracle import make_golden_dataset as MG


@pytest.fixture(scope="module")
def corpus(tmp_path_factory):
    return MG.write_corpus(str(tmp_path_factory.mktemp("corpus")))


@pytest.mark.parametrize("preload", [False, True])
def test_items_equal_reference_snr_mix_arguments(golden, corpus, preload):
    g = golden("dataset_train")
    ds = Dataset(**MG.with_preload(corpus, preload))
    L = int(g["L"])
    assert len(ds) == len(g["clean"]) and ds.rir_length == g["rir"].shape[1]
    random.seed(int(g["seed"]))
    np.random.seed(int(g["seed"]))
    for i in range(len(ds)):
        it = ds[i]
        assert it["clean"].dtype == np.float32 and it["clean"].shape == (L,)
        assert np.array_equal(it["clean"], g["clean"][i]), i
        assert np.array_equal(it["noise"], g["noise"][i]), i
        n = int(g["rir_len"][i])
        assert int(it["rir_len"]) == n, i
        assert np.array_equal(it["rir"][:n], g["rir"][i, :n]) and not it["rir"][n:].any(), i
        assert float(it["snr"]) == g["snr"][i] and float(it["noisy_target_dB_FS"]) == g["noisy_target_dB_FS"][i], i
        assert float(it["target_dB_FS"]) == -25.0
    # the streams end where the reference's ended: the next draws agree with a fresh replay of the same items
    nxt = (random.random(), np.random.random())
    random.seed(int(g["seed"]))
    np.random.seed(int(g["seed"]))
    for i in range(len(ds)):
        ds[i]
    assert (random.random(), np.random.random()) == nxt


def test_items_against_reference_arithmetic(golden):
    """The golden's own consistency: the CPU restatement of snr_mix on the recorded arguments gives the reference's
    (noisy, clean) - the arguments are the whole input of the mixing."""
    from oracle.mix_oracle import snr_mix
    g = golden("dataset_train")
    for i in range(len(g["clean"])):
        n = int(g["rir_len"][i])
        noisy, clean = snr_mix(g["clean"][i], g["noise"][i], float(g["snr"][i]), -25, float(g["noisy_target_dB_FS"][i]),
                               rir=g["rir"][i, :n] if n else None)
        scale = np.abs(g["noisy"][i]).max()
        assert np.abs(noisy - g["noisy"][i]).max() < 2e-5 * scale, i
        assert np.abs(clean - g["clean_out"][i]).max() < 2e-5 * scale, i


@pytest.mark.parametrize("num_workers", [0, 2])
def test_default_collate_batches(corpus, num_workers):
    ds = Dataset(**corpus)
    L, Lr = int(0.075 * 16000), ds.rir_length
    sampler = DistributedSampler(dataset=ds, num_replicas=2, rank=1, shuffle=True)
    sampler.set_epoch(0)
    dl = DataLoader(dataset=ds, sampler=sampler, shuffle=False, batch_size=5, num_workers=num_workers, drop_last=True,
                    pin_memory=False)
    batches = list(dl)
    assert len(batches) == len(dl) == (len(ds) // 2) // 5
    for b in batches:
        assert set(b) == {"clean", "noise", "rir", "rir_len", "snr", "noisy_target_dB_FS", "target_dB_FS"}
        assert b["clean"].shape == b["noise"].shape == (5, L) and b["rir"].shape == (5, Lr)
        assert b["clean"].dtype == b["noise"].dtype == b["rir"].dtype == torch.float32
        assert b["rir_len"].shape == (5,) and b["rir_len"].dtype == torch.int32
        for k in ("snr", "noisy_target_dB_FS", "target_dB_FS"):
            assert b[k].shape == (5,) and b[k].dtype == torch.float32, k
        assert ((b["rir_len"] >= 0) & (b["rir_len"] <= Lr)).all()
        assert ((b["snr"] >= -5) & (b["snr"] <= 20)).all()
        assert ((b["noisy_target_dB_FS"] >= -35) & (b["noisy_target_dB_FS"] < -15)).all()


def _write(path, y, sr=16000, width=2):
    y = np.atleast_2d(y)
    scale = {1: 128.0, 2: 32768.0, 3: 8388608.0, 4: 2147483648.0}[width]
    v = np.clip(np.round(y * scale), -scale, scale - 1).astype(np.int64).T.reshape(-1)
    if width == 1:
        raw = (v + 128).astype(np.uint8).tobytes()
    elif width == 3:
        u = (v & 0xFFFFFF).astype(np.uint32)
        raw = np.stack([u & 0xFF, (u >> 8) & 0xFF, (u >> 16) & 0xFF], axis=1).astype(np.uint8).tobytes()
    else:
        raw = v.astype("<i2" if width == 2 else "<i4").tobytes()
    with wave.open(str(path), "wb") as f:
        f.setnchannels(y.shape[0])
        f.setsampwidth(width)
        f.setframerate(sr)
        f.writeframes(raw)


def _list(path, files):
    path.write_text("\n".join(str(f) for f in files) + "\n")
    return str(path)


def test_constructor_refusals(corpus, tmp_path):
    with pytest.raises(AssertionError):
        Dataset(**dict(corpus, snr_range=[5]))
    with pytest.raises(AssertionError):
        Dataset(**dict(corpus, snr_range=[10, 5]))
    for p in (-0.1, 1.5):
        with pytest.raises(AssertionError):
            Dataset(**dict(corpus, reverb_proportion=p))
    # offset and limit select from the lists like the reference
    ds = Dataset(**dict(corpus, clean_dataset_offset=3, clean_dataset_limit=5, rir_dataset_offset=2))
    assert len(ds) == 5 and ds.clean_dataset_list[0].endswith("clean_03.wav") and len(ds.rir_dataset_list) == 1
    assert ds.rir_length == 800
    assert len(Dataset(**dict(corpus, clean_dataset_offset=20)).clean_dataset_list) == 4
    # a multi-channel clean or noise file is refused: when preloaded at construction, otherwise when it is read
    stereo = tmp_path / "stereo.wav"
    _write(stereo, 0.1 * np.ones((2, 2000)))
    for key, pre in (("clean_dataset", "pre_load_clean_dataset"), ("noise_dataset", "pre_load_noise")):
        lst = _list(tmp_path / f"{key}.txt", [stereo])
        with pytest.raises(ValueError, match="channels"):
            Dataset(**dict(corpus, **{key: lst, pre: True}))
        ds = Dataset(**dict(corpus, **{key: lst}))
        with pytest.raises(ValueError, match="channels"):
            ds[0]


def test_paths_expand_home(corpus, tmp_path, monkeypatch):
    monkeypatch.setenv("HOME", str(tmp_path))
    (tmp_path / "lists").mkdir()
    for k in ("clean", "noise", "rir"):
        src = corpus[f"{k}_dataset"]
        (tmp_path / "lists" / f"{k}.txt").write_text(open(src).read())
    ds = Dataset(**dict(corpus, clean_dataset="~/lists/clean.txt", noise_dataset="~/lists/noise.txt",
                        rir_dataset="~/lists/rir.txt"))
    assert len(ds) == len(Dataset(**corpus))


def test_load_wav_keeps_channels_and_resamples(tmp_path):
    from fullsubnet_b200.inferencer import Inferencer
    y = 0.3 * np.sin(np.arange(2 * 4410).reshape(2, 4410) * 0.01)
    _write(tmp_path / "a.wav", y, sr=44100)
    w = load_wav(tmp_path / "a.wav", 16000)
    n = int(np.ceil(4410 * 160 / 441))
    assert w.shape == (2, n) and w.dtype == np.float32
    raw = np.round(y * 32768.0) / 32768.0
    assert np.array_equal(w[1], Inferencer.resample(raw[1].astype(np.float32), 44100, 16000))


def _old_load_wav(path, sr=16000):
    """Inferencer.load_wav as it was before it moved onto utils.read_wav."""
    from fullsubnet_b200.inferencer import Inferencer
    with wave.open(str(path), "rb") as f:
        nch, width, rate, n = f.getnchannels(), f.getsampwidth(), f.getframerate(), f.getnframes()
        raw = f.readframes(n)
    if width == 2:
        y = np.frombuffer(raw, dtype="<i2").astype(np.float32) / 32768.0
    elif width == 1:
        y = (np.frombuffer(raw, dtype=np.uint8).astype(np.float32) - 128.0) / 128.0
    elif width == 4:
        y = np.frombuffer(raw, dtype="<i4").astype(np.float32) / 2147483648.0
    else:
        b = np.frombuffer(raw, dtype=np.uint8).reshape(-1, 3).astype(np.int32)
        v = b[:, 0] | (b[:, 1] << 8) | (b[:, 2] << 16)
        y = (np.where(v >= 1 << 23, v - (1 << 24), v)).astype(np.float32) / 8388608.0
    if nch > 1:
        y = y.reshape(-1, nch).mean(axis=1).astype(np.float32)
    if rate != sr:
        y = Inferencer.resample(y, rate, sr)
    return np.ascontiguousarray(y, dtype=np.float32)


@pytest.mark.parametrize("width", [1, 2, 3, 4])
@pytest.mark.parametrize("channels", [1, 2, 3, 9])
@pytest.mark.parametrize("sr", [16000, 48000])
def test_inferencer_load_wav_unchanged(tmp_path, width, channels, sr):
    from fullsubnet_b200.inferencer import Inferencer
    rng = np.random.default_rng(width * 10 + channels)
    p = tmp_path / "x.wav"
    _write(p, 0.9 * rng.uniform(-1, 1, (channels, 3001)), sr=sr, width=width)
    got, want = Inferencer.load_wav(p, 16000), _old_load_wav(p, 16000)
    assert got.dtype == want.dtype and got.shape == want.shape and np.array_equal(got, want)
