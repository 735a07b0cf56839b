"""Chunked streaming of fullband_baseline (fsn_fullband_stream_step through fullsubnet_b200.stream.Streamer): every clip,
under any chunking schedule and any mix of other streams, concatenates to the whole-clip fsn_fullband_enhance output bit
for bit; a start in one slot leaves the others' bits alone; a slot's state moved to another slot carries the stream on;
a step captured in a CUDA graph replays with new data to the same bits."""
import random

import pytest
import torch

pytestmark = pytest.mark.gpu

NORMS = ["cumulative_laplace_norm", "forgetting_norm"]
HOP = 256
KS = (1, 2, 3, 7, 64)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _model(norm, dev, fc_gain=1.0, layers=3):
    from fullsubnet_b200.fullband_baseline.model import Model
    from fullsubnet_b200.model.module.sequence_model import SequenceModel
    from oracle import fullband_baseline_oracle as BO
    args = dict(BO.DEFAULT_FBB_ARGS, norm_type=norm)
    sd = BO.make_fbb_state_dict(seed=11, args=args)
    m = Model(**args)
    if layers != 3:  # the recipe's Model fixes 3 layers; the library reads the depth from its SequenceModel
        F, H = args["num_freqs"], args["hidden_size"]
        m.fullband_model = SequenceModel(input_size=F, output_size=2 * F, hidden_size=H, num_layers=layers,
                                         bidirectional=False, sequence_model=args["sequence_model"],
                                         output_activate_function=args["output_activate_function"])
        g = torch.Generator().manual_seed(11 + layers)
        sd = {k: (torch.rand(v.shape, generator=g) * 2 - 1) / H ** 0.5 for k, v in m.state_dict().items()}
    for k in ("fullband_model.fc_output_layer.weight", "fullband_model.fc_output_layer.bias"):
        sd[k] = sd[k] * fc_gain
    m.load_state_dict(sd, strict=True)
    return m.to(dev).eval()


def _clip(L, seed, dev):
    from oracle import fullsubnet_oracle as O
    return O.make_noisy(1, L, seed=seed, speechlike=True)[0].to(dev)


class Runner:
    """Drives a Streamer with per-slot clip queues and collects each clip's output samples."""

    def __init__(self, streamer, dev, late=()):
        self.s, self.dev = streamer, dev
        self.late = set(late)  # clips that end on a chunk boundary and are announced (tail = 0) on the next call
        self.queue = {b: [] for b in range(streamer.slots)}
        self.cur = {}  # slot -> [clip id, clip, pos]
        self.out = {}
        self.tails = {}  # clip id -> the tail its last call carried

    def add(self, b, cid, clip):
        self.queue[b].append((cid, clip))

    def busy(self):
        return bool(self.cur) or any(self.queue.values())

    def call(self, K, rng=None):
        S, D, Kh = self.s.slots, self.s.delay, K * self.s.hop
        chunk = torch.zeros(S, Kh, device=self.dev)
        start, tail = [0] * S, [-1] * S
        for b in range(S):
            if b not in self.cur and self.queue[b] and (rng is None or rng.random() < 0.7):
                cid, clip = self.queue[b].pop(0)
                self.cur[b] = [cid, clip, 0]
                self.out[cid] = []
                start[b] = 1
            if b in self.cur:
                cid, clip, pos = self.cur[b]
                n = min(Kh, clip.numel() - pos)
                chunk[b, :n] = clip[pos:pos + n]
                if clip.numel() - pos < Kh or (clip.numel() - pos == Kh and cid not in self.late) or n == 0:
                    tail[b] = self.tails[cid] = n
        y = self.s.step(chunk, start, tail)
        for b in list(self.cur):
            cid, clip, pos = self.cur[b]
            row0 = pos - D
            end = pos + tail[b] if tail[b] >= 0 else row0 + Kh
            lo = max(row0, 0)
            if end > lo:
                self.out[cid].append(y[b, lo - row0:end - row0])
            if tail[b] >= 0:
                del self.cur[b]
            else:
                self.cur[b][2] = pos + Kh
        return y

    def result(self, cid):
        return torch.cat(self.out[cid]) if self.out[cid] else torch.zeros(0, device=self.dev)


def _whole(m, clip):
    return m.enhance(clip[None])[0]


@pytest.mark.parametrize("norm,fc_gain,layers", [
    pytest.param(norm, gain, 3, id=f"{norm}-{w}") for norm in NORMS for gain, w in ((1.0, "Wa"), (8.0, "Wb"))
] + [
    # depth 1 runs one layer alone; depth 4 puts the top layer in the other half of the layer-output ping-pong
    pytest.param("cumulative_laplace_norm", 1.0, n, id=f"cumulative_laplace_norm-Wa-depth{n}") for n in (1, 4)
])
def test_stream_bit_identical_to_whole_clip(norm, fc_gain, layers, dev):
    from fullsubnet_b200.stream import Streamer
    m = _model(norm, dev, fc_gain, layers)
    assert m.fullband_model.num_layers == layers
    rng = random.Random(NORMS.index(norm) * 10 + int(fc_gain) + (0 if layers == 3 else 100 * layers))
    slots = 4
    s = Streamer(m, slots)
    assert s.delay == 256 + (m.look_ahead + 2) * HOP
    r = Runner(s, dev)
    clips = {}
    # 0.3 s .. 5 s, multiples of hop and not; 5 s = 313 frames crosses the forgetting norm's t = 192
    lengths = [4800, 16000 + 77, 7 * HOP, 80000, 64 * HOP, 3 * 16000 + 129, 6000, 25 * HOP]
    for i, L in enumerate(lengths):
        clips[i] = _clip(L, 100 + i, dev)
        r.add(i % slots, i, clips[i])
    while r.busy():
        r.call(rng.choice(KS), rng)
    for cid, clip in clips.items():
        ref = _whole(m, clip)
        got = r.result(cid)
        assert got.shape == ref.shape, (cid, got.shape, ref.shape)
        assert torch.equal(got, ref), (cid, float((got - ref).abs().max()))
    # a 20 s clip alone, K = 64 and then K = 1 for its last 2 s
    long = _clip(20 * 16000, 7, dev)
    r2 = Runner(Streamer(m, 1), dev)
    r2.add(0, 0, long)
    while r2.busy():
        r2.call(64 if r2.cur.get(0, [0, 0, 0])[2] < 18 * 16000 else 1)
    assert torch.equal(r2.result(0), _whole(m, long))


@pytest.mark.parametrize("hop", [128, 160])
@pytest.mark.parametrize("norm", NORMS)
def test_stream_other_hops(norm, hop, dev):
    """hop 128: two steps of framing lag; hop 160: n_fft/2 not a multiple of hop (c = 2, Rc = 6)."""
    from fullsubnet_b200.stream import Streamer
    m = _model(norm, dev, 8.0)
    rng = random.Random(hop + NORMS.index(norm))
    s = Streamer(m, 3, hop=hop)
    assert s.delay == 256 + (m.look_ahead + 1 + -(-256 // hop)) * hop
    r = Runner(s, dev)
    lengths = [4800, 3 * 16000 + 129, 40 * hop, 7 * hop + 3, 20000]
    clips = {i: _clip(L, 300 + i, dev) for i, L in enumerate(lengths)}
    for i, clip in clips.items():
        r.add(i % 3, i, clip)
    while r.busy():
        r.call(rng.choice(KS), rng)
    for cid, clip in clips.items():
        ref = m.enhance(clip[None], hop_length=hop)[0]
        assert torch.equal(r.result(cid), ref), (hop, cid)


def test_clip_ending_on_a_chunk_boundary(dev):
    """tail = 0: the clip's last chunk was full and its end comes with the next call, so its last frames come from the
    carried history and the reflection at the end."""
    from fullsubnet_b200.stream import Streamer
    m = _model("forgetting_norm", dev)
    s = Streamer(m, 2)
    clips = {"a": _clip(12 * HOP, 21, dev), "b": _clip(3 * 16000 + 55, 22, dev), "c": _clip(8 * HOP, 23, dev)}
    r = Runner(s, dev, late=("a", "c"))
    r.add(0, "a", clips["a"])
    r.add(1, "b", clips["b"])
    r.add(0, "c", clips["c"])
    while r.busy():  # K = 4: "a" and "c" are whole numbers of chunks
        r.call(4)
    assert r.tails == {"a": 0, "b": 3 * 16000 + 55 - 46 * 4 * HOP, "c": 0}
    for cid, clip in clips.items():
        assert torch.equal(r.result(cid), _whole(m, clip)), cid


def test_stream_alone_and_among_63(dev):
    from fullsubnet_b200.stream import Streamer
    m = _model("cumulative_laplace_norm", dev)
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
    m = _model("forgetting_norm", dev)
    a, b = Streamer(m, 3), Streamer(m, 3)
    g = torch.Generator(device="cpu").manual_seed(9)
    start0 = [1, 1, 1]
    for i in range(12):
        x = (0.1 * torch.randn(3, 2 * HOP, generator=g)).to(dev)
        st = start0 if i == 0 else [0, 0, 0]
        ya = a.step(x, st)
        yb = b.step(x, [0, 1, 0] if i == 6 else st)
        assert torch.equal(ya[0], yb[0]) and torch.equal(ya[2], yb[2]), i
    assert not torch.equal(ya[1], yb[1])


def test_state_moves_between_slots(dev):
    from fullsubnet_b200.stream import Streamer
    m = _model("cumulative_laplace_norm", dev)
    clip = _clip(9000, 4, dev)
    ref = _whole(m, clip)
    s = Streamer(m, 3)
    D, Kh = s.delay, 3 * HOP
    outs, pos, slot = [], 0, 0
    while pos < clip.numel():
        if pos == 4 * Kh:  # mid-clip: checkpoint slot 0, then carry the stream on in slot 2
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
    m = _model("forgetting_norm", dev)
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
    xs = [(0.1 * torch.randn(4, 4 * HOP, generator=g)).to(dev) for _ in range(6)]
    ye = [eager.step(xs[0], [1] * 4)] + [eager.step(x) for x in xs[1:]]
    yc = [cap.step(xs[0], [1] * 4).clone()]  # also sizes the K = 4 workspace before the capture
    static_x = xs[1].clone()
    side = torch.cuda.Stream(dev)
    side.wait_stream(torch.cuda.current_stream(dev))
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            static_y = cap.step(static_x)
    torch.cuda.current_stream(dev).wait_stream(side)
    # capture does not run the work: the state is still after call 0
    for x in xs[1:]:
        static_x.copy_(x)
        graph.replay()
        yc.append(static_y.clone())
    torch.cuda.synchronize()
    for i, (a, b) in enumerate(zip(ye, yc)):
        assert torch.equal(a, b), i
