"""fsn_resample against the host resampler (Inferencer.resample): every rate of the gate, zeros 8 and 24, clip lengths
from 1 sample to 60 s at 48 kHz; batches and copies; a CUDA-graph replay; and the two users of the device path,
enhance_files(resample_on_device=True) and Dataset(resample_on_device=True)."""
import random
import wave
from math import gcd

import numpy as np
import pytest
import torch

from fullsubnet_b200 import _lib
from fullsubnet_b200.acoustics.resample import resample_batch, resampled_length
from fullsubnet_b200.inferencer import Inferencer

pytestmark = pytest.mark.gpu

GATE = 1e-7              # |device - host| <= GATE * max|x| per clip
BIT_IDENTICAL_FLOOR = 0.99999  # share of samples with the host's bits over the sweep; first measured on an H100: 1.0
PAIRS = [(r, 16000) for r in (8000, 11025, 22050, 24000, 32000, 44100, 48000, 96000)] + [(16000, 8000), (16000, 48000)]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _half(sr_in, sr_out, zeros):
    g = gcd(sr_in, sr_out)
    return int(np.ceil(zeros / min(1.0, (sr_out // g) / (sr_in // g))))


def _host_rows(y, sr_in, sr_out, zeros, n0, n1):
    """Outputs [n0, n1) of Inferencer.resample(y, sr_in, sr_out, zeros), its lines evaluated on those rows only (each
    output is its own row there), so that a 60 s clip needs no 6 GB of temporaries."""
    g = gcd(int(sr_in), int(sr_out))
    up, down = sr_out // g, sr_in // g
    cutoff = min(1.0, up / down)
    half = int(np.ceil(zeros / cutoff))
    t_out = np.arange(n0, n1, dtype=np.float64) * down / up
    base = np.floor(t_out).astype(np.int64)
    k = np.arange(-half + 1, half + 1)
    idx = base[:, None] + k[None, :]
    d = t_out[:, None] - idx
    w = cutoff * np.sinc(cutoff * d) * (0.5 + 0.5 * np.cos(np.pi * np.clip(d / half, -1, 1)))
    ok = (idx >= 0) & (idx < len(y))
    vals = np.where(ok, y[np.clip(idx, 0, len(y) - 1)], 0.0)
    return (vals * w).sum(axis=1).astype(np.float32)


def _host(y, sr_in, sr_out, zeros, rows=20000):
    n = resampled_length(len(y), sr_in, sr_out)
    if n <= rows:
        return Inferencer.resample(y, sr_in, sr_out, zeros)
    return np.concatenate([_host_rows(y, sr_in, sr_out, zeros, a, min(a + rows, n)) for a in range(0, n, rows)])


def _clip(n, seed, peak=0.7):
    """Speech-band noise scaled to max|x| = peak (< 1: a one-step rounding difference stays inside the gate)."""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(n) + 0.2 * np.sin(np.arange(n) * 0.01) + 0.05 * np.cumsum(rng.standard_normal(n)) / np.sqrt(
        np.arange(1, n + 1))
    return (peak * x / max(np.abs(x).max(), 1e-12)).astype(np.float32)


def _call(dev, xs, sr_in, sr_out, zeros, N_out_max=None, lengths=True):
    """fsn_resample on the rows of xs (a list of 1-D float32 arrays) in one call: y [B, N_out_max] on the host."""
    lib = _lib.load()
    B, N = len(xs), max(len(v) for v in xs)
    x = torch.full((B, N), float("nan"), dtype=torch.float32)
    for b, v in enumerate(xs):
        x[b, :len(v)] = torch.from_numpy(v)
    x = x.to(dev)
    need = max(resampled_length(len(v), sr_in, sr_out) for v in xs)
    N_out_max = need if N_out_max is None else N_out_max
    y = torch.full((B, N_out_max), float("nan"), dtype=torch.float32, device=dev)
    lens = np.array([len(v) for v in xs], dtype=np.int32)
    n = _lib.check_workspace(lib.fsn_resample_workspace_bytes(B, N, sr_in, sr_out, zeros))
    ws = torch.empty(n, dtype=torch.uint8, device=dev)
    _lib.check(lib.fsn_resample(x.data_ptr(), lens.ctypes.data if lengths else None, B, N, sr_in, sr_out, zeros,
                                y.data_ptr(), N_out_max, ws.data_ptr(), n, _lib.stream_ptr(dev)))
    return y.cpu().numpy()


def test_matches_host_resampler(dev):
    """Every clip within GATE * max|x| of the host, and the share of bit-identical samples over the sweep."""
    same = total = 0
    worst = 0.0
    for zeros in (8, 24):
        for sr_in, sr_out in PAIRS:
            h = _half(sr_in, sr_out, zeros)
            lengths = [1, 2, max(1, h - 1), 4801, 12345, sr_in + 1]
            xs = [_clip(n, seed=n + sr_in + zeros) for n in lengths]
            y = _call(dev, xs, sr_in, sr_out, zeros)
            for x, row in zip(xs, y):
                ref = _host(x, sr_in, sr_out, zeros)
                got = row[:len(ref)]
                err = float(np.abs(got.astype(np.float64) - ref).max() / np.abs(x).max())
                worst = max(worst, err)
                assert err <= GATE, (sr_in, sr_out, zeros, len(x), err)
                assert (row[len(ref):] == 0).all()
                same += int((got.view(np.int32) == ref.view(np.int32)).sum())
                total += len(ref)
    # 60 s at 48 kHz, both filters
    x = _clip(48000 * 60, seed=60)
    for zeros in (8, 24):
        got = _call(dev, [x], 48000, 16000, zeros)[0]
        ref = _host(x, 48000, 16000, zeros)
        err = float(np.abs(got.astype(np.float64) - ref).max() / np.abs(x).max())
        worst = max(worst, err)
        assert got.shape == ref.shape and err <= GATE, (zeros, err)
        same += int((got.view(np.int32) == ref.view(np.int32)).sum())
        total += len(ref)
    frac = same / total
    print(f"[resample] {same} of {total} samples bit-identical to the host ({frac:.7f}); worst |d| / max|x| {worst:.2e}")
    assert frac >= BIT_IDENTICAL_FLOOR, frac


def test_batch_rows_are_each_clip_alone_and_copies_keep_bits(dev):
    lengths = [1, 7, 4801, 30000, 12345, 2]
    xs = [_clip(n, seed=100 + n) for n in lengths]
    for sr_in, sr_out, zeros in ((44100, 16000, 24), (16000, 48000, 8), (22050, 16000, 24)):
        N_out_max = resampled_length(30000, sr_in, sr_out) + 37  # longer rows than needed: zero there too
        y = _call(dev, xs, sr_in, sr_out, zeros, N_out_max=N_out_max)
        for b, x in enumerate(xs):
            alone = _call(dev, [x], sr_in, sr_out, zeros, lengths=False)[0]
            n = len(alone)
            assert n == resampled_length(len(x), sr_in, sr_out)
            assert np.array_equal(y[b, :n].view(np.int32), alone.view(np.int32)), (sr_in, b)
            assert (y[b, n:] == 0).all() and not np.signbit(y[b, n:]).any()
    # the same rate: the input bits, rows 0 past each clip
    y = _call(dev, xs, 16000, 16000, 24, N_out_max=30005)
    for b, x in enumerate(xs):
        assert np.array_equal(y[b, :len(x)].view(np.int32), x.view(np.int32))
        assert (y[b, len(x):] == 0).all()
    # resample_batch: several rates in one list, one call per rate, results equal to the calls above
    rates = [44100, 16000, 48000, 44100, 16000, 48000]
    out = resample_batch(xs, rates, 16000, dev, zeros=24)
    for x, r, t in zip(xs, rates, out):
        want = _call(dev, [x], r, 16000, 24, lengths=False)[0]
        assert np.array_equal(t.cpu().numpy().view(np.int32), want.view(np.int32))


def test_graph_replay_matches_eager_call(dev):
    """One fsn_resample captured in a CUDA graph (no allocation, no host synchronisation inside the call) and replayed
    with new input gives the eager call's bits."""
    lib = _lib.load()
    lens = np.array([48000, 31111, 1], dtype=np.int32)
    B, N = len(lens), int(lens.max())
    N_out = resampled_length(N, 48000, 16000)
    x = torch.zeros(B, N, device=dev)
    y = torch.zeros(B, N_out, device=dev)
    n = _lib.check_workspace(lib.fsn_resample_workspace_bytes(B, N, 48000, 16000, 24))
    ws = torch.empty(n, dtype=torch.uint8, device=dev)
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(side):  # warm the module on the capture stream's device
        _lib.check(lib.fsn_resample(x.data_ptr(), lens.ctypes.data, B, N, 48000, 16000, 24, y.data_ptr(), N_out,
                                    ws.data_ptr(), n, _lib.stream_ptr(dev)))
    torch.cuda.current_stream(dev).wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        _lib.check(lib.fsn_resample(x.data_ptr(), lens.ctypes.data, B, N, 48000, 16000, 24, y.data_ptr(), N_out,
                                    ws.data_ptr(), n, _lib.stream_ptr(dev)))
    lens[:] = 5  # the lengths travelled in the captured launch, not through this buffer
    fresh = torch.from_numpy(np.stack([_clip(N, seed=s) for s in range(B)])).to(dev)
    x.copy_(fresh)
    g.replay()
    torch.cuda.synchronize(dev)
    want = _call(dev, [fresh[b, :v].cpu().numpy() for b, v in enumerate((48000, 31111, 1))], 48000, 16000, 24,
                 N_out_max=N_out)
    assert np.array_equal(y.cpu().numpy().view(np.int32), want.view(np.int32))


def _write(path, y, sr):
    """16-bit PCM wav, [C, N] or [N]."""
    y = np.atleast_2d(y)
    v = np.clip(np.round(y * 32768.0), -32768, 32767).astype("<i2")
    with wave.open(str(path), "wb") as f:
        f.setnchannels(y.shape[0])
        f.setsampwidth(2)
        f.setframerate(sr)
        f.writeframes(np.ascontiguousarray(v.T).tobytes())


def _pcm(path):
    with wave.open(str(path)) as f:
        return np.frombuffer(f.readframes(f.getnframes()), dtype="<i2").astype(np.int32)


@pytest.mark.parametrize("max_padding", [0.0, 0.5])
def test_enhance_files_resample_on_device(dev, tmp_path, max_padding):
    """16 kHz files byte-identical to the default run, resampled ones within one int16 step of it."""
    from fullsubnet_b200.fullsubnet.model import Model
    from oracle import fullsubnet_oracle as O
    m = Model(**O.DEFAULT_MODEL_ARGS, precision="auto")
    m.load_state_dict(O.make_state_dict(seed=0), strict=True)
    inf = Inferencer(model=m.to(dev).eval(), device=dev)
    files = [(16000, 1, 6000), (44100, 1, 16538), (48000, 2, 18000), (16000, 2, 6000), (44100, 2, 22050),
             (48000, 1, 18000), (16000, 1, 9000), (48000, 1, 29999)]
    paths = []
    for i, (sr, ch, n) in enumerate(files):
        p = tmp_path / f"f{i}_{sr}.wav"
        _write(p, np.stack([_clip(n, seed=200 + 7 * i + c, peak=0.6) for c in range(ch)]), sr)
        paths.append(p)
    host = inf.enhance_files(paths, tmp_path / "host", batch_size=3, max_padding=max_padding)
    devc = inf.enhance_files(paths, tmp_path / "dev", batch_size=3, max_padding=max_padding, resample_on_device=True)
    identical = 0
    for (sr, _, _), a, b in zip(files, host, devc):
        assert a.name == b.name
        if sr == 16000:
            assert a.read_bytes() == b.read_bytes(), a.name
        else:
            pa, pb = _pcm(a), _pcm(b)
            assert pa.shape == pb.shape and np.abs(pa - pb).max() <= 1, (a.name, np.abs(pa - pb).max())
            identical += a.read_bytes() == b.read_bytes()
    print(f"[resample] enhance_files max_padding={max_padding}: {identical} of "
          f"{sum(sr != 16000 for sr, _, _ in files)} resampled files byte-identical to the host path")


def test_dataset_preload_resample_on_device(dev, tmp_path):
    from fullsubnet_b200.dataset import Dataset, mix_batch
    rng = np.random.default_rng(7)
    lists = {"clean": [], "noise": [], "rir": []}
    for i, (sr, n) in enumerate([(48000, 9000), (44100, 7000), (16000, 3000), (48000, 4801), (22050, 5001)]):
        lists["clean"].append(tmp_path / f"clean_{i}.wav")
        _write(lists["clean"][-1], _clip(n, seed=300 + i, peak=0.5), sr)
    for i, (sr, n) in enumerate([(44100, 6000), (48000, 2500), (16000, 1500)]):
        lists["noise"].append(tmp_path / f"noise_{i}.wav")
        _write(lists["noise"][-1], _clip(n, seed=400 + i, peak=0.4), sr)
    for i, (sr, c, n) in enumerate([(48000, 2, 900), (16000, 1, 300), (44100, 3, 701)]):
        r = rng.standard_normal((c, n)) * np.exp(-np.arange(n) / (n / 5.0))
        r[:, 0] = 0.9
        lists["rir"].append(tmp_path / f"rir_{i}.wav")
        _write(lists["rir"][-1], 0.5 * r / np.abs(r).max(), sr)
    args = {}
    for k, paths in lists.items():
        (tmp_path / f"{k}.txt").write_text("\n".join(map(str, paths)) + "\n")
        args[k] = str(tmp_path / f"{k}.txt")
    common = dict(clean_dataset=args["clean"], clean_dataset_limit=False, clean_dataset_offset=0,
                  noise_dataset=args["noise"], noise_dataset_limit=False, noise_dataset_offset=0,
                  rir_dataset=args["rir"], rir_dataset_limit=False, rir_dataset_offset=0, snr_range=[-5, 20],
                  reverb_proportion=0.6, silence_length=0.01, target_dB_FS=-25, target_dB_FS_floating_value=10,
                  sub_sample_length=0.2, sr=16000, pre_load_clean_dataset=True, pre_load_noise=True, pre_load_rir=True,
                  num_workers=2)
    host, devd = Dataset(**common), Dataset(**common, resample_on_device=True)
    for kind in ("clean_dataset_list", "noise_dataset_list", "rir_dataset_list"):
        for (pa, wa), (pb, wb) in zip(getattr(host, kind), getattr(devd, kind)):
            assert pa == pb and wa.shape == wb.shape and wa.dtype == wb.dtype == np.float32
            assert np.abs(wa.astype(np.float64) - wb).max() <= GATE * np.abs(wa).max(), (kind, pa)
    assert host.rir_length == devd.rir_length
    items = {}
    for name, ds in (("host", host), ("dev", devd)):
        random.seed(11)
        np.random.seed(11)
        items[name] = [ds[i % len(ds)] for i in range(3 * len(ds))]
        items[name + "_state"] = (random.getstate(), np.random.get_state()[1].copy())
    assert items["host_state"][0] == items["dev_state"][0]
    assert np.array_equal(items["host_state"][1], items["dev_state"][1])  # the same draws, in the same number
    for a, b in zip(items["host"], items["dev"]):
        for k in ("rir_len", "snr", "noisy_target_dB_FS", "target_dB_FS"):
            assert a[k] == b[k], k
        for k in ("clean", "noise", "rir"):  # the same crop starts and RIR channel: equal within the gate
            assert a[k].shape == b[k].shape
            assert np.abs(a[k].astype(np.float64) - b[k]).max() <= GATE * max(np.abs(a[k]).max(), 1e-30), k
    collate = torch.utils.data.default_collate
    na, ca = mix_batch(collate(items["host"]), dev)
    nb, cb = mix_batch(collate(items["dev"]), dev)
    for u, v in ((na, nb), (ca, cb)):
        u, v = u.cpu().double(), v.cpu().double()
        assert ((u - v).abs().amax(dim=1) <= 2 * GATE * u.abs().amax(dim=1)).all()
