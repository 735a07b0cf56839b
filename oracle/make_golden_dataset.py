"""TEST INFRASTRUCTURE ONLY.  ``tests/golden/dataset_train.npz``: the UNMODIFIED training ``Dataset``
(recipes/dns_interspeech_2020/dataset_train.py) on CPU over a small synthetic int16 corpus (``write_corpus``), items
0..N-1 in order after seeding ``random`` and ``np.random``, once with every ``pre_load_*`` false and once with them true.
``librosa.load`` is stubbed by a wav reader (``mono=False``, the corpus is at the target rate, so nothing resamples).
``Dataset.snr_mix`` is wrapped and still called, so every draw happens; per item the golden keeps the arguments it
receives (the RIR channel it draws is replayed from the saved ``np.random`` state), the noisy target dBFS it draws and
the (noisy, clean) it returns.
Run:  python oracle/make_golden_dataset.py
"""
from __future__ import annotations

import os
import random
import sys
import tempfile
import wave

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

SR = 16000
SEED = 11
N_CLEAN = 24
# clip lengths of the clean files (samples): shorter than, equal to and longer than the 1200-sample crop
CLEAN_LENGTHS = [700, 1200, 3000, 5000, 1200, 2500, 900, 4000, 1500, 6000, 1201, 2000] * 2
NOISE_LENGTHS = [250, 250, 300, 4000, 1200]   # three short files: noise assembled from three or more
RIR_SHAPES = [(1, 300), (2, 500), (1, 800)]   # (channels, taps)
SPIKY = (3, 15)                               # clean files with an impulsive peak: the anti-clipping rescale


def write_pcm16(path, y):
    """[C, N] float in [-1, 1) -> 16-bit PCM wav."""
    y = np.atleast_2d(y)
    pcm = np.clip(np.round(y * 32768.0), -32768, 32767).astype("<i2")
    with wave.open(str(path), "wb") as f:
        f.setnchannels(y.shape[0])
        f.setsampwidth(2)
        f.setframerate(SR)
        f.writeframes(np.ascontiguousarray(pcm.T).tobytes())


def write_corpus(root) -> dict:
    """Writes the seeded corpus and its three list files under ``root``; returns the Dataset arguments (pre_load_*
    false)."""
    rng = np.random.default_rng(2024)
    lists = {"clean": [], "noise": [], "rir": []}
    for i in range(N_CLEAN):
        n = CLEAN_LENGTHS[i]
        t = np.arange(n) / SR
        y = 0.2 * np.sin(2 * np.pi * (180 + 40 * i) * t) * (0.6 + 0.4 * np.sin(2 * np.pi * 3 * t)) + \
            0.02 * rng.standard_normal(n)
        if i in SPIKY:
            y = 0.002 * rng.standard_normal(n)
            y[::997] = 0.95
        lists["clean"].append(os.path.join(root, f"clean_{i:02d}.wav"))
        write_pcm16(lists["clean"][-1], y)
    for i, n in enumerate(NOISE_LENGTHS):
        lists["noise"].append(os.path.join(root, f"noise_{i}.wav"))
        write_pcm16(lists["noise"][-1], 0.3 * rng.standard_normal(n))
    for i, (c, n) in enumerate(RIR_SHAPES):
        r = rng.standard_normal((c, n)) * np.exp(-np.arange(n) / (n / 5.0))
        r[:, 0] = 0.9
        lists["rir"].append(os.path.join(root, f"rir_{i}.wav"))
        write_pcm16(lists["rir"][-1], 0.5 * r)
    args = {}
    for k, paths in lists.items():
        lst = os.path.join(root, f"{k}.txt")
        with open(lst, "w") as f:
            f.write("\n".join(paths) + "\n")
        args[k] = lst
    return dict(clean_dataset=args["clean"], clean_dataset_limit=False, clean_dataset_offset=0,
                noise_dataset=args["noise"], noise_dataset_limit=False, noise_dataset_offset=0,
                rir_dataset=args["rir"], rir_dataset_limit=False, rir_dataset_offset=0,
                snr_range=[-5, 20], reverb_proportion=0.6, silence_length=0.01, target_dB_FS=-25,
                target_dB_FS_floating_value=10, sub_sample_length=0.075, sr=SR,
                pre_load_clean_dataset=False, pre_load_noise=False, pre_load_rir=False, num_workers=2)


def with_preload(args: dict, on: bool) -> dict:
    return dict(args, pre_load_clean_dataset=on, pre_load_noise=on, pre_load_rir=on)


def run_reference(args: dict):
    """Items 0..N-1 of the unmodified Dataset after seeding; per item a dict of the snr_mix arguments and outputs."""
    import librosa

    import dataset_train
    from fullsubnet_b200.utils import read_wav

    def fake_load(path, mono=True, sr=SR):
        y, rate = read_wav(path)
        assert rate == sr and not mono
        return (y[0] if len(y) == 1 else y), rate
    librosa.load = fake_load

    loads, records = [], []
    orig_load = dataset_train.load_wav
    dataset_train.load_wav = lambda f, sr=SR: loads.append(orig_load(f, sr=sr)) or loads[-1]
    orig_mix = dataset_train.Dataset.__dict__["snr_mix"].__func__

    def wrapped(clean_y, noise_y, snr, target_dB_FS, target_dB_FS_floating_value, rir=None, eps=1e-6):
        state = np.random.get_state()
        rec = {"clean": np.array(clean_y, dtype=np.float32), "noise": np.array(noise_y, dtype=np.float32),
               "snr": snr, "loads": list(loads)}
        noisy, clean = orig_mix(clean_y, noise_y, snr, target_dB_FS, target_dB_FS_floating_value, rir=rir, eps=eps)
        replay = np.random.RandomState()
        replay.set_state(state)
        if rir is not None and rir.ndim > 1:
            ch = replay.randint(0, rir.shape[0])
            rec["rir"], rec["rir_channels"] = np.array(rir[ch], dtype=np.float32), rir.shape[0]
        elif rir is not None:
            rec["rir"], rec["rir_channels"] = np.array(rir, dtype=np.float32), 1
        else:
            rec["rir"], rec["rir_channels"] = np.zeros(0, np.float32), 0
        rec["noisy_target_dB_FS"] = replay.randint(target_dB_FS - target_dB_FS_floating_value,
                                                   target_dB_FS + target_dB_FS_floating_value)
        assert all(np.array_equal(a, b) for a, b in zip(replay.get_state()[1:3], np.random.get_state()[1:3]))  # every draw replayed
        rec["noisy"], rec["clean_out"] = noisy.astype(np.float32), clean.astype(np.float32)
        records.append(rec)
        return noisy, clean
    dataset_train.Dataset.snr_mix = staticmethod(wrapped)
    try:
        import joblib
        with joblib.parallel_backend("threading"):  # worker processes would not see the librosa stub
            ds = dataset_train.Dataset(**args)
        loads.clear()
        random.seed(SEED)
        np.random.seed(SEED)
        out = []
        for i in range(len(ds)):
            loads.clear()
            noisy, clean = ds[i]
            rec = records[-1]
            assert np.array_equal(noisy, rec["noisy"].astype(np.float32)) and np.array_equal(clean, rec["clean_out"])
            out.append(rec)
        return out
    finally:
        dataset_train.Dataset.snr_mix = staticmethod(orig_mix)
        dataset_train.load_wav = orig_load


def coverage(recs, L, silence):
    seen = set()
    for r in recs:
        clean_len = len(r["loads"][0])
        seen.add("clean<" if clean_len < L else "clean=" if clean_len == L else "clean>")
        noise_lens = [len(y) for y in r["loads"][1:1 + 64] if y.ndim == 1][:64]
        n_files, remaining, total, partial = 0, L, 0, False
        for n in noise_lens:
            n_files += 1
            remaining -= n
            total += n
            if remaining <= 0:
                break
            k = min(remaining, silence)
            partial |= k < silence
            remaining -= k
            total += k
        if n_files == 1:
            seen.add("noise:1 file")
        if n_files >= 3 and partial:
            seen.add("noise:3+ files, partial silence")
        if total == L:
            seen.add("noise=L")
        seen.add("reverb" if r["rir_channels"] else "dry")
        if r["rir_channels"] == 2:
            seen.add("2-channel rir")
        if abs(float(np.abs(r["noisy"]).max()) - 0.99) < 1e-4:
            seen.add("anti-clipping")
    return seen


def main():
    from make_golden import import_reference
    import_reference()
    with tempfile.TemporaryDirectory() as tmp:
        args = write_corpus(tmp)
        L = int(args["sub_sample_length"] * SR)
        runs = [run_reference(with_preload(args, on)) for on in (False, True)]
    for a, b in zip(*runs):  # preloading changes nothing
        for k in ("clean", "noise", "rir", "noisy", "clean_out"):
            assert np.array_equal(a[k], b[k]), k
        assert (a["snr"], a["noisy_target_dB_FS"]) == (b["snr"], b["noisy_target_dB_FS"])
    recs = runs[0]
    want = {"clean<", "clean=", "clean>", "noise:1 file", "noise:3+ files, partial silence", "noise=L", "reverb",
            "dry", "2-channel rir", "anti-clipping"}
    seen = coverage(recs, L, int(SR * args["silence_length"]))
    assert want <= seen, sorted(want - seen)
    Lr = max(c[1] for c in RIR_SHAPES)
    rir = np.zeros((len(recs), Lr), np.float32)
    for i, r in enumerate(recs):
        rir[i, :len(r["rir"])] = r["rir"]
    res = {"seed": np.int64(SEED), "L": np.int64(L),
           "clean": np.stack([r["clean"] for r in recs]), "noise": np.stack([r["noise"] for r in recs]),
           "rir": rir, "rir_len": np.array([len(r["rir"]) for r in recs], np.int32),
           "rir_channels": np.array([r["rir_channels"] for r in recs], np.int32),
           "snr": np.array([r["snr"] for r in recs], np.int64),
           "noisy_target_dB_FS": np.array([r["noisy_target_dB_FS"] for r in recs], np.int64),
           "noisy": np.stack([r["noisy"] for r in recs]), "clean_out": np.stack([r["clean_out"] for r in recs])}
    out = os.path.join(ROOT, "tests", "golden", "dataset_train.npz")
    np.savez_compressed(out, **res)
    print("covered:", sorted(seen))
    print(out, os.path.getsize(out))


if __name__ == "__main__":
    main()
