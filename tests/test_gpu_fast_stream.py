"""Chunked streaming of fast_fullsubnet (fsn_fast_stream_step through fullsubnet_b200.stream.Streamer): every clip, under
any chunking schedule, at any block phase and alongside any other streams, concatenates to the whole-clip output
(Inferencer.enhance_batch: fsn_stft -> fsn_fast_model_forward -> fsn_istft) bit for bit, with the decoder on the
persistent kernel and, in a subprocess with FSN_FB_STEPWISE=1, on the per-step kernels; a start in one slot leaves the
others' bits alone; a slot's state moved to another slot carries the stream on; a captured step replays to the same
bits."""
import os
import random
import subprocess
import sys

import pytest
import torch

from test_gpu_stream import Runner

pytestmark = pytest.mark.gpu

HOP = 256
KS = (1, 2, 3, 7, 64)
# fast_fullsubnet/inference.toml (S = 2, look_ahead 2, no encoder-output neighbours) and an odd one
SHAPES = {"recipe": {}, "odd": dict(shrink_size=3, look_ahead=1, encoder_output_num_neighbors=1)}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _model(dev, shape="recipe", fc_gain=1.0, seed=11):
    """fp32, cumulative norm, seeded weights; fc_gain scales the decoder's Linear so that the cRM reaches the clip of
    decompress_cIRM."""
    from fullsubnet_b200.fast_fullsubnet.model import Model
    from oracle import fast_fullsubnet_oracle as FO
    args = dict(FO.DEFAULT_FAST_ARGS, norm_type="cumulative_laplace_norm", **SHAPES[shape])
    sd = FO.make_fast_state_dict(seed=seed, args=args)
    for k in ("decoder_lstm.1.fc_output_layer.weight", "decoder_lstm.1.fc_output_layer.bias"):
        sd[k] = sd[k] * fc_gain
    m = Model(**args, precision="fp32")
    m.load_state_dict(sd, strict=True)
    return m.to(dev).eval()


def _clip(L, seed, dev):
    from oracle import fullsubnet_oracle as O
    return O.make_noisy(1, L, seed=seed, speechlike=True)[0].to(dev)


def _whole(m, clip, hop=HOP):
    from fullsubnet_b200.inferencer import Inferencer
    acoustics = {"n_fft": 512, "hop_length": hop, "win_length": 512, "sr": 16000}
    return Inferencer(config={"acoustics": acoustics}, model=m, device=clip.device).enhance_batch(clip[None])[0]


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


@pytest.mark.parametrize("fc_gain", [1.0, 8.0], ids=["Wa", "Wb"])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_stream_bit_identical_to_whole_clip(shape, fc_gain, dev):
    m = _model(dev, shape, fc_gain)
    # 0.3 s .. 5 s, on and off hop multiples
    lengths = [4800, 16000 + 77, 7 * HOP, 80000, 64 * HOP, 3 * 16000 + 129, 6000, 25 * HOP + 1]
    _run_mixed(m, dev, 1 + list(SHAPES).index(shape) * 2 + int(fc_gain), lengths)


def test_stream_20s_clip(dev):
    """A 20 s clip alone, K = 64 and then K = 1 for its last 2 s."""
    from fullsubnet_b200.stream import Streamer
    m = _model(dev, "recipe", 8.0)
    long = _clip(20 * 16000, 7, dev)
    r = Runner(Streamer(m, 1), dev)
    r.add(0, 0, long)
    while r.busy():
        r.call(64 if r.cur.get(0, [0, 0, 0])[2] < 18 * 16000 else 1)
    assert torch.equal(r.result(0), _whole(m, long))


@pytest.mark.parametrize("hop", [128, 160])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_stream_other_hops(shape, hop, dev):
    """hop 128: two steps of framing lag; hop 160: n_fft/2 not a multiple of hop."""
    m = _model(dev, shape, 8.0)
    _run_mixed(m, dev, hop + len(shape), [4800, 3 * 16000 + 129, 40 * hop, 7 * hop + 3, 20000], slots=3, hop=hop)


def test_clip_ending_on_a_chunk_boundary(dev):
    """tail = 0: the clip's last chunk was full and its end comes with the next call."""
    from fullsubnet_b200.stream import Streamer
    m = _model(dev, "odd")
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


@pytest.mark.parametrize("shape", list(SHAPES))
def test_slots_out_of_block_phase(shape, dev):
    """Two slots started one hop apart with K = 1: their frames are never at the same block phase, so every call ends a
    block in one slot and not in the other (S = 2), or in at most one of them (S = 3)."""
    from fullsubnet_b200.stream import Streamer
    m = _model(dev, shape, 8.0)
    r = Runner(Streamer(m, 2), dev)
    clips = {"a": _clip(9000, 31, dev), "b": _clip(7 * HOP, 32, dev)}
    r.add(0, "a", clips["a"])
    r.call(1)
    r.add(1, "b", clips["b"])
    while r.busy():
        r.call(1)
    for cid, clip in clips.items():
        assert torch.equal(r.result(cid), _whole(m, clip)), cid


def test_stream_alone_and_among_63(dev):
    from fullsubnet_b200.stream import Streamer
    m = _model(dev, "recipe")
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


def test_start_leaves_other_slots(dev):
    from fullsubnet_b200.stream import Streamer
    m = _model(dev, "odd")
    a, b = Streamer(m, 3), Streamer(m, 3)
    g = torch.Generator(device="cpu").manual_seed(9)
    for i in range(12):
        x = (0.1 * torch.randn(3, 2 * HOP, generator=g)).to(dev)
        st = [1, 1, 1] if i == 0 else [0, 0, 0]
        ya = a.step(x, st)
        yb = b.step(x, [0, 1, 0] if i == 5 else st)
        assert torch.equal(ya[0], yb[0]) and torch.equal(ya[2], yb[2]), i
    assert not torch.equal(ya[1], yb[1])


def test_state_moves_between_slots(dev):
    from fullsubnet_b200.stream import Streamer
    m = _model(dev, "odd", 8.0)
    clip = _clip(9000, 4, dev)
    ref = _whole(m, clip)
    s = Streamer(m, 3)
    D, Kh = s.delay, 1 * HOP
    outs, pos, slot = [], 0, 0
    while pos < clip.numel():
        if pos == 7 * Kh:  # mid-clip, mid-block (S = 3): checkpoint slot 0, then carry the stream on in slot 2
            saved = s.slot_state(0).clone()
            s.slot_state(0).zero_()
            s.slot_state(2).copy_(saved)
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
    m = _model(dev, "recipe", 8.0)
    clip = _clip(10 * HOP + 99, 8, dev)
    s = Streamer(m, 2)
    pieces = [clip[:4 * HOP], clip[4 * HOP:5 * HOP], clip[5 * HOP:]]
    got = torch.cat(list(s.enhance_stream(pieces, slot=1)))
    assert torch.equal(got, _whole(m, clip))


def test_graph_capture_replays(dev):
    from fullsubnet_b200.stream import Streamer
    m = _model(dev, "recipe")
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


def _stepwise_check():
    """The mixed-schedule identity on both shapes, run by test_stream_decoder_per_step in a process with
    FSN_FB_STEPWISE=1 (the whole-clip decoder then runs the per-step kernels, and so must the stream)."""
    dev = torch.device("cuda:0")
    for i, shape in enumerate(SHAPES):
        _run_mixed(_model(dev, shape, 8.0), dev, 40 + i, [4800, 16000 + 77, 9 * HOP, 3 * 16000 + 129], slots=3)
    print("stepwise ok")


def test_stream_decoder_per_step(dev):
    here = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(here)
    env = dict(os.environ, FSN_FB_STEPWISE="1", PYTHONPATH=os.pathsep.join([here, root]))
    code = "import test_gpu_fast_stream as T; T._stepwise_check()"
    p = subprocess.run([sys.executable, "-c", code], env=env, cwd=root, capture_output=True, text=True, timeout=1800)
    assert p.returncode == 0 and "stepwise ok" in p.stdout, p.stdout[-3000:] + p.stderr[-3000:]
