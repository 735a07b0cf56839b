"""fsn_stoi on the GPU against the float64 oracle (oracle/stoi_oracle.py), stage by stage through fsn_debug_stoi_stages;
per-clip lengths (bit-identical to the call on each clip alone, whatever the batch, its order or the samples past each
clip); STOI in Trainer validation behind the recipes' [trainer.visualization] metrics; the metrics CLI."""
import csv

import numpy as np
import pytest
import torch

from oracle import stoi_oracle as S
from oracle.stoi_oracle import speechlike

pytestmark = pytest.mark.gpu

OUT_TOL = 1e-6     # |out - oracle|, absolute
STAGE_TOL = 1e-12  # resampled, compacted and band magnitudes, relative to the clip's largest value


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _length_for_frames(T, sr):
    """The shortest clip whose resampled signal has T + 1 frames: T STFT frames when every frame is kept."""
    L = S.min_length(sr)
    while S.n_frames(len(S.resample(np.zeros(L), sr))) < T + 1:
        L += 1
    return L


def _cases(sr):
    """(clean, estimate) pairs at sr: speech-like clips at several SNRs, stretches 30-60 dB down and exactly zero,
    estimates far louder than the clean clip in some bands, all-zero clips, 29 / 30 / 31 STFT frames after removal and
    the minimum legal length."""
    rng = np.random.default_rng(sr)
    out = []
    for k, snr in enumerate((-5.0, 0.0, 10.0, 30.0)):
        n = int(sr * (1.0 + 0.7 * k)) + 37 * k
        x = speechlike(n, seed=10 * k + 1, sr=sr)
        x[n // 5:n // 5 + sr // 4] *= 10 ** (-(30 + 10 * k) / 20)  # 30 - 60 dB down: dropped frames
        if k % 2:
            x[n // 2:n // 2 + sr // 5] = 0.0
        noise = rng.standard_normal(n).astype(np.float32)
        y = x + noise * np.float32(np.sqrt(np.mean(x ** 2)) * 10 ** (-snr / 20))
        out.append((x, y.astype(np.float32)))
    # an estimate 40 dB louder than the clean clip in a narrow band (the -15 dB clip of step 5 bites)
    n = int(1.6 * sr)
    x = speechlike(n, seed=99, sr=sr)
    t = np.arange(n) / sr
    out.append((x, (x + 100 * np.std(x) * np.sin(2 * np.pi * 1000 * t)).astype(np.float32)))
    out.append((x, np.zeros_like(x)))
    out.append((np.zeros_like(x), x))
    for T in (29, 30, 31):
        L = _length_for_frames(T, sr)
        x = speechlike(L, seed=T, sr=sr) + np.float32(0.05)
        out.append((x, (x + 0.02 * rng.standard_normal(L)).astype(np.float32)))
    L = S.min_length(sr)
    x = speechlike(L, seed=5, sr=sr)
    out.append((x, (0.5 * x + 0.01 * rng.standard_normal(L)).astype(np.float32)))
    return out


def _threshold_case():
    """A 10 kHz clip whose single-sample bumps sit one float32 step either side of the 40 dB threshold: the float64
    keep / drop decision separates them, a float32 one cannot."""
    n = 40 * 128
    x = np.zeros(n, np.float32)
    w = S.window()
    x[:512] = 0.5 * np.sin(2 * np.pi * np.arange(512) / 37)
    top = S.silent_mask(x.astype(np.float64))  # the loud frames alone
    e = 20 * np.log10(np.linalg.norm(S.frames(x.astype(np.float64)), axis=1) + S.EPS)
    target = 10 ** ((e.max() - S.DYN_RANGE) / 20)
    assert top.sum() >= 1
    for m, pos in enumerate(range(1024, n - 256, 512)):
        i = pos % 128 + 128  # the bump is sample i of frame pos // 128 - 1 (the frame where its weight is larger)
        a = np.float32(target / w[i])
        keep_side = m % 2 == 0
        for _ in range(4):  # step to the float32 value on the wanted side of the threshold
            x[pos] = a
            kept = S.silent_mask(x.astype(np.float64))[pos // 128 - 1]
            if kept == keep_side:
                break
            a = np.nextafter(a, np.float32(np.inf) if keep_side else np.float32(0))
        x[pos] = a
        assert S.silent_mask(x.astype(np.float64))[pos // 128 - 1] == keep_side
    return x, (x + np.float32(1e-4) * np.random.default_rng(3).standard_normal(n).astype(np.float32)).astype(np.float32)


def _batch(pairs, tail=np.nan):
    lens = [len(x) for x, _ in pairs]
    L = max(lens)
    c = np.full((len(pairs), L), tail, np.float32)
    e = np.full((len(pairs), L), tail, np.float32)
    for b, (x, y) in enumerate(pairs):
        c[b, :len(x)] = x
        e[b, :len(y)] = y
    return torch.from_numpy(c), torch.from_numpy(e), lens


def _stages(clean, est, lens, sr, dev):
    """fsn_debug_stoi_stages on one batch: (out, resampled, keep, n_kept, compacted, bands) on the host."""
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    B, L = clean.shape
    Lr = len(S.resample(np.zeros(L), sr))
    nf = S.n_frames(Lr)
    rs = torch.empty(2, B, Lr, dtype=torch.float64, device=dev)
    cs = torch.empty_like(rs)
    keep = torch.empty(B, nf, dtype=torch.int32, device=dev)
    nk = torch.empty(B, dtype=torch.int32, device=dev)
    bands = torch.empty(2, B, 15, nf, dtype=torch.float64, device=dev)
    out = torch.empty(B, dtype=torch.float32, device=dev)
    nbytes = lib.fsn_stoi_workspace_bytes(B, L, sr)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    c, e = clean.to(dev), est.to(dev)
    arr = _lib.lengths_table(lens, B, L)
    _lib.check(lib.fsn_debug_stoi_stages(c.data_ptr(), e.data_ptr(), arr.ctypes.data, B, L, sr, rs.data_ptr(),
                                         keep.data_ptr(), nk.data_ptr(), cs.data_ptr(), bands.data_ptr(), out.data_ptr(),
                                         ws.data_ptr(), nbytes, _lib.stream_ptr(dev)))
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in (out, rs, keep, nk, cs, bands)]


def _rel(a, b):
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)) if b.size else 0.0


@pytest.mark.parametrize("sr", [16000, 10000])
def test_stoi_matches_the_float64_oracle_stage_by_stage(dev, sr):
    pairs = _cases(sr) + ([_threshold_case()] if sr == 10000 else [])
    clean, est, lens = _batch(pairs)
    out, rs, keep, nk, cs, bands = _stages(clean, est, lens, sr, dev)
    worst = {"out": 0.0, "resampled": 0.0, "compacted": 0.0, "bands": 0.0}
    for b, (x, y) in enumerate(pairs):
        st = S.stages(x, y, sr)
        Lr, nf, n_kept = len(st["resampled"][0]), len(st["mask"]), int(st["mask"].sum())
        assert np.array_equal(keep[b, :nf].astype(bool), st["mask"]), (sr, b)
        assert nk[b] == n_kept, (sr, b)
        for s in range(2):
            worst["resampled"] = max(worst["resampled"], _rel(rs[s, b, :Lr], st["resampled"][s]))
            assert not rs[s, b, Lr:].any()
            m = len(st["compacted"][s])
            assert m == (n_kept + 1) * 128
            worst["compacted"] = max(worst["compacted"], _rel(cs[s, b, :m], st["compacted"][s]))
            assert not cs[s, b, m:].any()
            T = st["bands"][s].shape[1]
            assert T == n_kept - 1
            worst["bands"] = max(worst["bands"], _rel(bands[s, b, :, :T], st["bands"][s]))
        err = abs(float(out[b]) - st["d"])
        worst["out"] = max(worst["out"], err)
        assert err <= OUT_TOL, (sr, b, float(out[b]), st["d"])
    print(f"[stoi {sr} Hz] worst: out {worst['out']:.2e} abs; resampled {worst['resampled']:.2e}, compacted "
          f"{worst['compacted']:.2e}, bands {worst['bands']:.2e} rel")
    assert max(worst["resampled"], worst["compacted"], worst["bands"]) <= STAGE_TOL, worst
    # the edge cases: x vs 0 and 0 vs x give 0, 29 frames give 1e-5, 30 and 31 a score
    d = [S.stoi(x, y, sr) for x, y in pairs]
    assert 0.0 in d and 1e-5 in d


def test_identity_and_scale_give_one(dev):
    from fullsubnet_b200.metrics import stoi
    x = torch.from_numpy(speechlike(32000, seed=7)).reshape(1, -1).to(dev)
    for y in (x, 3.7 * x):
        assert abs(float(stoi(x, y)[0]) - 1.0) <= 1e-6


@pytest.mark.parametrize("sr", [16000, 10000])
def test_per_clip_lengths_are_bit_exact_single_calls(dev, sr):
    from fullsubnet_b200.metrics import stoi
    pairs = _cases(sr)
    clean, est, lens = _batch(pairs)
    c, e = clean.to(dev), est.to(dev)
    got = stoi(c, e, lens, sr)
    again = stoi(c, e, lens, sr)
    assert torch.equal(got, again)  # two runs, same bits
    for b, Lb in enumerate(lens):
        one = stoi(c[b:b + 1, :Lb].contiguous(), e[b:b + 1, :Lb].contiguous(), sr=sr)
        assert torch.equal(got[b:b + 1], one), (b, float(got[b]), float(one[0]))
    # the samples past each clip are never read: zeros instead of NaN give the same bits
    c0, e0, _ = _batch(pairs, tail=0.0)
    assert torch.equal(stoi(c0.to(dev), e0.to(dev), lens, sr), got)
    # a permuted batch gives the permuted outputs
    perm = np.random.default_rng(1).permutation(len(pairs))
    pc, pe, pl = _batch([pairs[i] for i in perm])
    assert torch.equal(stoi(pc.to(dev), pe.to(dev), pl, sr), got[torch.from_numpy(perm).to(dev)])
    # no lengths = every clip L_max
    eq = [(x[:lens[-1]], y[:lens[-1]]) for x, y in pairs if len(x) >= lens[-1]]
    ec, ee, el = _batch(eq)
    assert torch.equal(stoi(ec.to(dev), ee.to(dev), sr=sr), stoi(ec.to(dev), ee.to(dev), el, sr))


# ---------------------------------------------------------------------------------------------- validation
LENGTHS = [12345, 16000, 8005, 16000, 4097, 12345, 9999, 16000, 6000]


def _items(seed):
    rng = np.random.default_rng(seed)
    out = []
    for i, L in enumerate(LENGTHS):
        clean = speechlike(L, seed=seed * 100 + i)
        noisy = clean + np.float32(0.05) * rng.standard_normal(L).astype(np.float32)
        out.append((torch.from_numpy(noisy).reshape(1, -1), torch.from_numpy(clean).reshape(1, -1), [f"clip{i}"],
                    ["With_reverb" if i % 3 else "No_reverb"]))
    return out


def _trainer(model, items, tmp_path, metrics=("WB_PESQ", "NB_PESQ", "STOI", "SI_SDR"), batch_size=32,
             max_padding=0.25):
    from fullsubnet_b200.loss import mse_loss
    from fullsubnet_b200.trainer import Trainer
    trainer = {"train": {"epochs": 1, "save_checkpoint_interval": 1, "clip_grad_norm_value": 10},
               "validation": {"validation_interval": 1, "save_max_metric_score": True, "batch_size": batch_size,
                              "max_padding": max_padding}}
    if metrics is not None:
        trainer["visualization"] = {"n_samples": 10, "num_workers": 36, "metrics": list(metrics)}
    cfg = {"meta": {"use_amp": False, "save_dir": str(tmp_path), "experiment_name": "v"},
           "acoustics": {"n_fft": 512, "hop_length": 256, "win_length": 512}, "trainer": trainer}
    return Trainer(None, 0, cfg, False, False, model, mse_loss(), torch.optim.SGD(model.parameters(), lr=0.0), [],
                   items)


def _model(dev):
    from fullsubnet_b200.fullsubnet.model import Model
    from oracle import fullsubnet_oracle as O
    m = Model(**O.DEFAULT_MODEL_ARGS, precision="f16x3_tc")
    m.load_state_dict(O.make_state_dict(seed=0), strict=True)
    return m.to(dev)


def test_validation_stoi_per_item_and_per_type(dev, tmp_path):
    from fullsubnet_b200.inferencer import Inferencer
    m = _model(dev)
    items = _items(3)
    tr = _trainer(m, items, tmp_path)
    score = tr._validation_epoch(1)
    st, v = tr.last_validation_stoi, tr.last_validation
    types = [it[3][0] for it in items]
    inf = Inferencer(config={"acoustics": {"n_fft": 512, "hop_length": 256, "win_length": 512}}, model=m, device=dev)
    worst = 0.0
    for i, (noisy, clean, _, _) in enumerate(items):
        x = clean.numpy()[0]
        assert abs(float(st["noisy"][i]) - S.stoi(x, noisy.numpy()[0])) <= OUT_TOL, i
        with torch.no_grad():
            enhanced = inf.enhance_batch(noisy.to(dev)).cpu().numpy()[0]
        worst = max(worst, abs(float(st["enhanced"][i]) - S.stoi(x, enhanced)))
    print(f"[stoi validation] enhanced vs oracle on the B = 1 waveform: {worst:.2e}")
    assert worst <= 1e-4
    sums = {}
    for i, t in enumerate(types):
        s = sums.setdefault(t, {"noisy": np.float32(0), "enhanced": np.float32(0)})
        s["noisy"] += st["noisy"][i]
        s["enhanced"] += st["enhanced"][i]
    assert v["stoi"] == {t: {w: float(sums[t][w]) / types.count(t) for w in ("noisy", "enhanced")}
                         for t in ("With_reverb", "No_reverb")}
    assert score == v["si_sdr"]["With_reverb"]


def test_validation_stoi_does_not_depend_on_grouping(dev, tmp_path):
    m = _model(dev)
    items = _items(4)
    ref = None
    for batch_size in (1, 3, len(items)):
        for max_padding in (0.0, 0.25):
            tr = _trainer(m, items, tmp_path, batch_size=batch_size, max_padding=max_padding)
            tr._validation_epoch(1)
            got = (tr.last_validation, tr.last_validation_stoi)
            if ref is None:
                ref = got
                continue
            assert got[0] == ref[0], (batch_size, max_padding)
            assert all(np.array_equal(got[1][k], ref[1][k]) for k in ("noisy", "enhanced"))


def test_validation_without_the_key_is_unchanged(dev, tmp_path):
    m = _model(dev)
    items = _items(5)
    plain = _trainer(m, items, tmp_path, metrics=None)
    no_stoi = _trainer(m, items, tmp_path, metrics=("SI_SDR", "WB_PESQ"))
    with_stoi = _trainer(m, items, tmp_path)
    results = []
    for tr in (plain, no_stoi, with_stoi):
        s = tr._validation_epoch(1)
        results.append((s, tr._validation_items(), tr.last_validation))
    for s, its, v in results[:2]:
        assert set(v) == {"loss_total", "loss", "si_sdr", "items"}
    assert plain.last_validation_stoi is None and no_stoi.last_validation_stoi is None
    s, its, v = results[2]
    assert set(v) == {"loss_total", "loss", "si_sdr", "items", "stoi"}
    for other in results[:2]:  # the same loss, SI-SDR and score with STOI on
        assert s == other[0] and all(np.array_equal(a, b) for a, b in zip(its[:2], other[1][:2]))
        assert {k: v[k] for k in other[2]} == other[2]


# ---------------------------------------------------------------------------------------------- the CLI
def test_cli_values_equal_the_library_calls(dev, tmp_path):
    from fullsubnet_b200 import metrics
    from fullsubnet_b200.inferencer import Inferencer
    from fullsubnet_b200.trainer import si_sdr
    rng = np.random.default_rng(6)
    ref_dir, est_dir = tmp_path / "clean", tmp_path / "enhanced"
    ref_dir.mkdir()
    est_dir.mkdir()
    for i, n in enumerate((16000, 12000, 16000, 9000, 20000)):
        x = speechlike(n, seed=200 + i)
        y = x + np.float32(0.03) * rng.standard_normal(n).astype(np.float32)
        Inferencer.write_wav(ref_dir / f"f{i}.wav", (x * 32767).astype(np.int16))
        Inferencer.write_wav(est_dir / f"f{i}.wav", (np.clip(y, -1, 1) * 32767).astype(np.int16))
    out_csv = tmp_path / "m.csv"
    assert metrics.main(["-R", str(ref_dir), "-E", str(est_dir), "-M", "SI_SDR,STOI", "--batch-size", "3",
                         "--csv", str(out_csv)]) == 0
    with open(out_csv) as f:
        rows = list(csv.DictReader(f))
    assert [r["Speech"] for r in rows] == [f"f{i}" for i in range(5)]
    for r in rows:
        x = torch.from_numpy(Inferencer.load_wav(ref_dir / f"{r['Speech']}.wav")).reshape(1, -1).to(dev)
        y = torch.from_numpy(Inferencer.load_wav(est_dir / f"{r['Speech']}.wav")).reshape(1, -1).to(dev)
        assert np.float32(float(r["STOI"])) == metrics.stoi(x, y).cpu().numpy()[0], r
        assert np.float32(float(r["SI_SDR"])) == si_sdr(x, y).cpu().numpy()[0], r
        assert metrics.STOI(x.cpu().numpy()[0], y.cpu().numpy()[0]) == float(metrics.stoi(x, y)[0])
