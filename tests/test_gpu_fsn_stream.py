"""Chunked streaming of fullsubnet (fsn_stream_step through fullsubnet_b200.stream.Streamer): every clip, under any
chunking schedule and alongside any other streams, concatenates to the whole-clip output (Model(precision="fp32")
.enhance on the clip alone, fsn_enhance with B = 1) bit for bit, on both causal norms and both weight sets; a start in
one slot leaves the others' bits alone; a slot's state moved to another slot carries the stream on; a captured step
replays to the same bits; the clips of the causal-norm fixtures stream within the gates their whole-clip tests hold."""
import random

import numpy as np
import pytest
import torch

from conftest import WB_GAIN
from test_gpu_stream import Runner

pytestmark = pytest.mark.gpu

NORMS = ["cumulative_laplace_norm", "forgetting_norm"]
HOP = 256
KS = (1, 2, 3, 7, 64)
WAV_TOL = 1e-4


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _model(norm, dev, gain=1.0, seed=11):
    """The recipe's shape, fp32, seeded weights; gain > 1 (W-b) drives the cRM past the +-9.9 clip of decompress_cIRM."""
    from fullsubnet_b200.fullsubnet.model import Model
    from oracle import fullsubnet_oracle as O
    args = dict(O.DEFAULT_MODEL_ARGS, norm_type=norm)
    m = Model(**args, precision="fp32")
    m.load_state_dict(O.make_state_dict(seed=seed, args=args, sb_fc_gain=gain), strict=True)
    return m.to(dev).eval()


def _clip(L, seed, dev):
    from oracle import fullsubnet_oracle as O
    return O.make_noisy(1, L, seed=seed, speechlike=True)[0].to(dev)


def _whole(m, clip, hop=HOP):
    return m.enhance(clip[None], hop_length=hop)[0]


def _run_mixed(m, dev, seed, lengths, slots=4, hop=HOP):
    """Clips queued on `slots` slots, K drawn from KS at random, starts delayed at random: each clip against its whole-clip
    output."""
    from fullsubnet_b200.stream import Streamer
    rng = random.Random(seed)
    s = Streamer(m, slots, hop=hop)
    assert s.delay == 256 + (m.look_ahead + 1 + -(-256 // hop)) * hop
    r = Runner(s, dev)
    clips = {i: _clip(L, seed * 100 + i, dev) for i, L in enumerate(lengths)}
    for i, clip in clips.items():
        r.add(i % slots, i, clip)
    while r.busy():
        r.call(rng.choice(KS), rng)
    for cid, clip in clips.items():
        ref = _whole(m, clip, hop)
        got = r.result(cid)
        assert got.shape == ref.shape, (cid, got.shape, ref.shape)
        assert torch.equal(got, ref), (cid, float((got - ref).abs().max()))


@pytest.mark.parametrize("gain", [1.0, WB_GAIN], ids=["Wa", "Wb"])
@pytest.mark.parametrize("norm", NORMS)
def test_stream_bit_identical_to_whole_clip(norm, gain, dev):
    m = _model(norm, dev, gain)
    # 0.3 s .. 5 s, on and off hop multiples; 80000 samples = 313 frames cross the forgetting norm's t = 192
    lengths = [4800, 16000 + 77, 7 * HOP, 80000, 64 * HOP, 3 * 16000 + 129, 6000, 25 * HOP + 1]
    _run_mixed(m, dev, 1 + NORMS.index(norm) * 2 + int(gain > 1), lengths)


@pytest.mark.parametrize("norm", NORMS)
def test_stream_20s_clip(norm, dev):
    """A 20 s clip alone, K = 64 and then K = 1 for its last 2 s."""
    from fullsubnet_b200.stream import Streamer
    m = _model(norm, dev, WB_GAIN)
    long = _clip(20 * 16000, 7, dev)
    r = Runner(Streamer(m, 1), dev)
    r.add(0, 0, long)
    while r.busy():
        r.call(64 if r.cur.get(0, [0, 0, 0])[2] < 18 * 16000 else 1)
    assert torch.equal(r.result(0), _whole(m, long))


@pytest.mark.parametrize("hop", [128, 160])
@pytest.mark.parametrize("norm", NORMS)
def test_stream_other_hops(norm, hop, dev):
    """hop 128: two steps of framing lag; hop 160: n_fft/2 not a multiple of hop."""
    m = _model(norm, dev, WB_GAIN)
    _run_mixed(m, dev, hop + NORMS.index(norm), [4800, 3 * 16000 + 129, 40 * hop, 7 * hop + 3, 20000], slots=3, hop=hop)


def test_clip_ending_on_a_chunk_boundary(dev):
    """tail = 0: the clip's last chunk was full and its end comes with the next call."""
    from fullsubnet_b200.stream import Streamer
    m = _model("cumulative_laplace_norm", dev)
    s = Streamer(m, 2)
    clips = {"a": _clip(12 * HOP, 21, dev), "b": _clip(3 * 16000 + 55, 22, dev), "c": _clip(8 * HOP, 23, dev)}
    r = Runner(s, dev, late=("a", "c"))
    r.add(0, "a", clips["a"])
    r.add(1, "b", clips["b"])
    r.add(0, "c", clips["c"])
    while r.busy():
        r.call(4)
    assert r.tails == {"a": 0, "b": 3 * 16000 + 55 - 46 * 4 * HOP, "c": 0}
    for cid, clip in clips.items():
        assert torch.equal(r.result(cid), _whole(m, clip)), cid


@pytest.mark.parametrize("norm", NORMS)
def test_stream_alone_and_among_63(norm, dev):
    from fullsubnet_b200.stream import Streamer
    m = _model(norm, dev)
    clip = _clip(12345, 3, dev)
    alone = Runner(Streamer(m, 1), dev)
    alone.add(0, "x", clip)
    many = Runner(Streamer(m, 64), dev)
    rng = random.Random(5)
    for b in range(64):
        if b == 17:
            many.add(b, "x", clip)
        else:
            many.add(b, b, _clip(rng.randint(4800, 20000), 200 + b, dev))
    ks = [3, 1, 7, 2, 64, 1, 1, 3]
    i = 0
    while alone.busy() or "x" not in many.out or 17 in many.cur:
        K = ks[i % len(ks)]
        i += 1
        if alone.busy():
            alone.call(K)
        many.call(K)
    ref = _whole(m, clip)
    assert torch.equal(alone.result("x"), ref)
    assert torch.equal(many.result("x"), ref)


@pytest.mark.parametrize("norm", NORMS)
def test_start_leaves_other_slots(norm, dev):
    from fullsubnet_b200.stream import Streamer
    m = _model(norm, dev)
    a, b = Streamer(m, 3), Streamer(m, 3)
    g = torch.Generator(device="cpu").manual_seed(9)
    for i in range(12):
        x = (0.1 * torch.randn(3, 2 * HOP, generator=g)).to(dev)
        st = [1, 1, 1] if i == 0 else [0, 0, 0]
        ya = a.step(x, st)
        yb = b.step(x, [0, 1, 0] if i == 5 else st)
        assert torch.equal(ya[0], yb[0]) and torch.equal(ya[2], yb[2]), i
    assert not torch.equal(ya[1], yb[1])


@pytest.mark.parametrize("move", ["slot_state", "copy_slot"])
@pytest.mark.parametrize("norm", NORMS)
def test_state_moves_between_slots(norm, move, dev):
    from fullsubnet_b200.stream import Streamer
    m = _model(norm, dev, WB_GAIN)
    clip = _clip(9000, 4, dev)
    ref = _whole(m, clip)
    s = Streamer(m, 3)
    D, Kh = s.delay, 3 * HOP
    outs, pos, slot = [], 0, 0
    while pos < clip.numel():
        if pos == 4 * Kh:  # mid-clip: carry the stream on in slot 2, slot 0's block cleared
            if move == "slot_state":
                saved = s.slot_state(0).clone()
                s.slot_state(0).zero_()
                s.slot_state(2).copy_(saved)
            else:
                s.copy_slot(0, 2)
                s.slot_state(0).zero_()
            slot = 2
        x = torch.zeros(3, Kh, device=dev)
        n = min(Kh, clip.numel() - pos)
        x[slot, :n] = clip[pos:pos + n]
        st, tl = [0] * 3, [-1] * 3
        st[slot] = int(pos == 0)
        if clip.numel() - pos <= Kh:
            tl[slot] = n
        y = s.step(x, st, tl)[slot]
        row0 = pos - D
        end = pos + n if tl[slot] >= 0 else row0 + Kh
        if end > max(row0, 0):
            outs.append(y[max(row0, 0) - row0:end - row0])
        pos += Kh
    assert torch.equal(torch.cat(outs), ref)


def test_enhance_stream_generator(dev):
    from fullsubnet_b200.stream import Streamer
    m = _model("forgetting_norm", dev, WB_GAIN)
    clip = _clip(10 * HOP + 99, 8, dev)
    s = Streamer(m, 2)
    pieces = [clip[:4 * HOP], clip[4 * HOP:5 * HOP], clip[5 * HOP:]]
    got = torch.cat(list(s.enhance_stream(pieces, slot=1)))
    assert torch.equal(got, _whole(m, clip))


def test_graph_capture_replays(dev):
    from fullsubnet_b200.stream import Streamer
    m = _model("cumulative_laplace_norm", dev)
    eager, cap = Streamer(m, 4), Streamer(m, 4)
    g = torch.Generator(device="cpu").manual_seed(2)
    xs = [(0.1 * torch.randn(4, 3 * HOP, generator=g)).to(dev) for _ in range(6)]
    ye = [eager.step(xs[0], [1] * 4)] + [eager.step(x) for x in xs[1:]]
    yc = [cap.step(xs[0], [1] * 4).clone()]  # also sizes the K = 3 workspace before the capture
    static_x = xs[1].clone()
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            static_y = cap.step(static_x)
    torch.cuda.current_stream(dev).wait_stream(side)
    for x in xs[1:]:
        static_x.copy_(x)
        graph.replay()
        yc.append(static_y.clone())
    torch.cuda.synchronize()
    for i, (a, b) in enumerate(zip(ye, yc)):
        assert torch.equal(a, b), i


def _stream_clips(m, ys, dev, seed):
    """Clips [N, L] streamed on N slots at once with mixed K -> [N, L]"""
    from fullsubnet_b200.stream import Streamer
    rng = random.Random(seed)
    r = Runner(Streamer(m, ys.shape[0]), dev)
    for i in range(ys.shape[0]):
        r.add(i, i, ys[i])
    while r.busy():
        r.call(rng.choice(KS))
    return torch.stack([r.result(i) for i in range(ys.shape[0])])


def test_fixture_cumulative_norm(golden, dev):
    """tests/golden/model_cum.npz: two 0.5 s clips of the unmodified reference with the cumulative norm, W-b (x60)."""
    from oracle import fullsubnet_oracle as O
    g = golden("model_cum")
    args = dict(O.DEFAULT_MODEL_ARGS, norm_type="cumulative_laplace_norm")
    from fullsubnet_b200.fullsubnet.model import Model
    m = Model(**args, precision="fp32")
    m.load_state_dict(O.make_state_dict(seed=0, args=args, sb_fc_gain=60.0), strict=True)
    m = m.to(dev).eval()
    y = torch.from_numpy(g["full_y"]).to(dev)
    got = _stream_clips(m, y, dev, 3)
    for i in range(y.shape[0]):
        assert torch.equal(got[i], _whole(m, y[i])), i
    assert np.abs(got.cpu().numpy() - g["full_wav"]).max() < WAV_TOL


@pytest.mark.parametrize("tag", ["wa", "wb"])
def test_fixture_forgetting_norm(golden, dev, tag):
    """tests/golden/model_forget_{wa,wb}.npz: one clip of T = 202 frames (both sides of t = 192) of the unmodified
    reference with the forgetting norm."""
    from fullsubnet_b200.fullsubnet.model import Model
    from oracle import fullsubnet_oracle as O
    from oracle.make_golden_forgetting import FULL_LEN
    from oracle.make_golden_long import fingerprint
    g = golden(f"model_forget_{tag}")
    y = O.make_noisy(1, FULL_LEN, seed=73, speechlike=True)
    assert np.allclose(fingerprint(y), g["y_fp"], rtol=1e-6)
    args = dict(O.DEFAULT_MODEL_ARGS, norm_type="forgetting_norm")
    m = Model(**args, precision="fp32")
    m.load_state_dict(O.make_state_dict(seed=0, args=args, sb_fc_gain=1.0 if tag == "wa" else WB_GAIN), strict=True)
    m = m.to(dev).eval()
    got = _stream_clips(m, y.to(dev), dev, 4 + len(tag))
    assert torch.equal(got[0], _whole(m, y[0].to(dev)))
    assert np.abs(got.cpu().numpy() - g["wav"]).max() < WAV_TOL
