"""Chunked streaming of fullsubnet on the fp16 tensor cores (fsn_stream_tc_step through Streamer(tensor_cores=True)).

Kernels alone: a run split into two launches with carried state is bit-identical to one launch, rows restarted at step
j match a fresh run from j, and the carried results stay within each precision's class of a float64 LSTM.  Model: every
clip, under any chunking schedule and alongside any other streams, concatenates to Model(precision=p).enhance on the
clip alone bit for bit, for p in f16x3_tc / f16_tc, both causal norms and both weight sets; the fixtures' clips stream
within their whole-clip gates; a call's launch count does not grow with K."""
import ctypes as C
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import WB_GAIN
from test_gpu_stream import Runner
from test_gpu_subband_tc import TOLERANCES, _weights, gather, stack

from fullsubnet_b200 import _lib

pytestmark = pytest.mark.gpu

NORMS = ["cumulative_laplace_norm", "forgetting_norm"]
PRECS = ["f16x3_tc", "f16_tc"]
HOP = 256
KS = (1, 2, 3, 7, 64)
WAV_TOL = 1e-4
NONE = 1 << 30  # a restart step no call reaches


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _ptr(t):
    return t.data_ptr()


def _sync_check(rc):
    _lib.check(rc)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------ sub-band carry kernel alone
def _sb_setup(dev, H=256, B=2, F=40, T=10, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    Ns, Nf = 15, 0
    K0 = 2 * Ns + 1 + 2 * Nf + 1
    k = 1.0 / H ** 0.5
    u = lambda *s: ((torch.rand(*s, generator=g) * 2 - 1) * k).to(dev).contiguous()
    w = dict(w_ih0=u(4 * H, K0), w_hh0=u(4 * H, H), w_ih1=u(4 * H, H), w_hh1=u(4 * H, H), b_ih0=u(4 * H), b_hh0=u(4 * H),
             b_ih1=u(4 * H), b_hh1=u(4 * H), fc_w=u(2, H), fc_b=u(2))
    magT = torch.rand(B, T, F, generator=g).to(dev)
    fbT = torch.rand(B, T, F, generator=g).to(dev)
    scale = (0.5 + torch.rand(T, B * F, generator=g)).to(dev)
    return dict(H=H, B=B, F=F, T=T, Ns=Ns, Nf=Nf, w=w, magT=magT, fbT=fbT, scale=scale)


def _sb_run(s, x3, t0, t1, h, c, restart, store_step):
    """steps [t0, t1) continued from h / c (updated in place) -> crm [B, t1 - t0, 2F]"""
    lib = _lib.load()
    w = s["w"]
    sw = _lib.SeqWeights()
    sw.w_ih[0], sw.w_ih[1] = _ptr(w["w_ih0"]), _ptr(w["w_ih1"])
    sw.w_hh[0], sw.w_hh[1] = _ptr(w["w_hh0"]), _ptr(w["w_hh1"])
    sw.b_ih[0], sw.b_ih[1] = _ptr(w["b_ih0"]), _ptr(w["b_ih1"])
    sw.b_hh[0], sw.b_hh[1] = _ptr(w["b_hh0"]), _ptr(w["b_hh1"])
    sw.fc_w, sw.fc_b = _ptr(w["fc_w"]), _ptr(w["fc_b"])
    B, F, H, n = s["B"], s["F"], s["H"], t1 - t0
    magT = s["magT"][:, t0:t1].contiguous()
    fbT = s["fbT"][:, t0:t1].contiguous()
    scale = s["scale"][t0:t1].contiguous()
    packed = torch.empty(lib.fsn_debug_sb_lstm_tc_packed_bytes(H, int(x3)), dtype=torch.uint8, device=magT.device)
    crm = torch.full((B, n, 2 * F), float("nan"), device=magT.device)
    rst = torch.as_tensor(restart, dtype=torch.int32, device=magT.device)
    _sync_check(lib.fsn_debug_sb_lstm_tc_carry(C.byref(sw), H, s["Ns"], s["Nf"], 0, int(x3), _ptr(magT), _ptr(fbT), B, F, n,
                                               _ptr(scale), n, _ptr(rst), store_step, _ptr(h), _ptr(c), _ptr(packed),
                                               _ptr(crm), None))
    return crm


@pytest.mark.parametrize("x3", [True, False], ids=PRECS)
def test_sb_carry_split_equals_one_launch(dev, x3):
    s = _sb_setup(dev)
    R, H, T = s["B"] * s["F"], s["H"], s["T"]
    none = [NONE] * R
    h1, c1 = torch.zeros(2, R, H, device=dev), torch.zeros(2, R, H, device=dev)
    one = _sb_run(s, x3, 0, T, h1, c1, none, T - 1)
    assert torch.isfinite(one).all()
    h2, c2 = torch.zeros(2, R, H, device=dev), torch.zeros(2, R, H, device=dev)
    a = _sb_run(s, x3, 0, 4, h2, c2, none, 3)
    b = _sb_run(s, x3, 4, T, h2, c2, none, T - 5)
    assert torch.equal(torch.cat([a, b], 1), one)
    assert torch.equal(h2, h1) and torch.equal(c2, c1)
    # a restart at step 0 ignores whatever state the buffers hold
    h3, c3 = torch.randn(2, R, H, device=dev), torch.randn(2, R, H, device=dev)
    assert torch.equal(_sb_run(s, x3, 0, T, h3, c3, [0] * R, -1), one)


@pytest.mark.parametrize("x3", [True, False], ids=PRECS)
def test_sb_carry_restart_equals_fresh_run(dev, x3):
    s = _sb_setup(dev, H=128, seed=1)
    B, F, R, H, T, j = s["B"], s["F"], s["B"] * s["F"], s["H"], s["T"], 3
    restart = [j if (r // F) == 1 else NONE for r in range(R)]  # clip 1's rows restart at step j
    h, c = torch.randn(2, R, H, device=dev) * 0.5, torch.randn(2, R, H, device=dev) * 0.5
    h0, c0 = h.clone(), c.clone()
    got = _sb_run(s, x3, 0, T, h, c, restart, -1)
    fresh = _sb_run(s, x3, j, T, torch.zeros_like(h), torch.zeros_like(c), [NONE] * R, -1)
    assert torch.equal(got[1, j:], fresh[1])
    cont = _sb_run(s, x3, 0, T, h0.clone(), c0.clone(), [NONE] * R, -1)
    assert torch.equal(got[0], cont[0])


# ------------------------------------------------------------------------------------------ full-band carry layer alone
def _rec_setup(dev, R=5, T=9, K=257, H=512, seed=3):
    g = torch.Generator(device="cpu").manual_seed(seed)
    k = 1.0 / H ** 0.5
    u = lambda *s: ((torch.rand(*s, generator=g) * 2 - 1) * k).to(dev).contiguous()
    return dict(R=R, T=T, K=K, H=H, w_ih=u(4 * H, K), w_hh=u(4 * H, H), b_ih=u(4 * H), b_hh=u(4 * H),
                x=torch.randn(R, T, K, generator=g).to(dev))


def _rec_run(s, x3, t0, t1, h_init, c, restart, fin_step):
    lib = _lib.load()
    R, K, H, n = s["R"], s["K"], s["H"], t1 - t0
    x = s["x"][:, t0:t1].contiguous()
    hall = torch.full((R, n, H), float("nan"), device=x.device)
    nb = lib.fsn_debug_lstm_tc_workspace_bytes(R, n, K, H, int(x3))
    ws = torch.empty(nb, dtype=torch.uint8, device=x.device)
    rst = torch.as_tensor(restart, dtype=torch.int32, device=x.device)
    _sync_check(lib.fsn_debug_lstm_tc_carry(_ptr(s["w_ih"]), _ptr(s["w_hh"]), _ptr(s["b_ih"]), _ptr(s["b_hh"]), _ptr(x), R, n,
                                            K, H, int(x3), _ptr(h_init.contiguous()), _ptr(c), _ptr(rst), fin_step,
                                            _ptr(hall), _ptr(ws), nb, None))
    return hall


def _lstm64(s, h0, c0, t0=0):
    """float64 nn.LSTM semantics from (h0, c0) over steps t0.."""
    H = s["H"]
    w_ih, w_hh = s["w_ih"].double(), s["w_hh"].double()
    b = (s["b_ih"] + 0.0).double() + s["b_hh"].double()
    h, c, out = h0.double(), c0.double(), []
    for t in range(t0, s["T"]):
        gates = s["x"][:, t].double() @ w_ih.T + h @ w_hh.T + b
        i, f, gg, o = gates.split(H, 1)
        c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(gg)
        h = torch.sigmoid(o) * torch.tanh(c)
        out.append(h)
    return torch.stack(out, 1), c


@pytest.mark.parametrize("x3", [True, False], ids=PRECS)
def test_rec_carry_split_equals_one_launch(dev, x3):
    s = _rec_setup(dev)
    R, H, T = s["R"], s["H"], s["T"]
    none = [NONE] * R
    c1 = torch.zeros(R, H, device=dev)
    one = _rec_run(s, x3, 0, T, torch.zeros(R, H, device=dev), c1, none, T - 1)
    c2 = torch.zeros(R, H, device=dev)
    a = _rec_run(s, x3, 0, 4, torch.zeros(R, H, device=dev), c2, none, 3)
    b = _rec_run(s, x3, 4, T, a[:, -1], c2, none, T - 5)
    assert torch.equal(torch.cat([a, b], 1), one)
    assert torch.equal(c2, c1)
    # entering step 0 with zero state is the whole-sequence layer, bit for bit
    lib = _lib.load()
    ref = torch.empty_like(one)
    nb = lib.fsn_debug_lstm_tc_workspace_bytes(R, T, s["K"], H, int(x3))
    ws = torch.empty(nb, dtype=torch.uint8, device=dev)
    _sync_check(lib.fsn_debug_lstm_layer_tc(_ptr(s["w_ih"]), _ptr(s["w_hh"]), _ptr(s["b_ih"]), _ptr(s["b_hh"]), _ptr(s["x"]),
                                            R, T, s["K"], H, int(x3), _ptr(ref), _ptr(ws), nb, None))
    assert torch.equal(ref, one)
    assert torch.equal(_rec_run(s, x3, 0, T, torch.randn(R, H, device=dev), torch.randn(R, H, device=dev), [0] * R, -1), one)


@pytest.mark.parametrize("x3", [True, False], ids=PRECS)
def test_rec_carry_restart_and_float64(dev, x3):
    s = _rec_setup(dev, seed=4)
    R, H, T, j = s["R"], s["H"], s["T"], 2
    # a carried state an LSTM can hold: |h| < 1
    h0, c0 = 0.9 * torch.tanh(torch.randn(R, H, device=dev)), torch.randn(R, H, device=dev)
    restart = [j if r % 2 else NONE for r in range(R)]
    got = _rec_run(s, x3, 0, T, h0, c0.clone(), restart, -1)
    fresh = _rec_run(s, x3, j, T, torch.zeros(R, H, device=dev), torch.zeros(R, H, device=dev), [NONE] * R, -1)
    for r in range(1, R, 2):
        assert torch.equal(got[r, j:], fresh[r])
    ref, _ = _lstm64(s, h0, c0)
    tol = 5e-6 if x3 else 3e-3  # the max-abs gates tests/test_gpu_rec_tc.py holds the whole-sequence layer to
    kept = [r for r in range(R) if r % 2 == 0]
    err = (got[kept].double() - ref[kept]).abs().max().item()
    print(f"lstm_rec_tc carry {'x3' if x3 else 'single pass'}: max-abs error {err:.1e}")
    assert err < tol


@pytest.mark.parametrize("H", [128, 256, 384])
def test_sb_carry_matches_float64(dev, H):
    """Two launches with the state carried between them against the float64 statement of the stack in
    tests/test_gpu_subband_tc.py (gather, per-(step, row) scale, 2 LSTM layers, Linear), within its per-H tolerances of
    the whole-sequence kernel, relative to max(1, max |ref|) as there."""
    B, F, T, Ns, Nf, t1 = 2, 33, 12, 15, 0, 5
    g = torch.Generator().manual_seed(H)
    w = _weights(H, (2 * Ns + 1) + (2 * Nf + 1), 2, "std", H + 1)
    magT = torch.randn(B, T, F, generator=g).abs()
    fbT = torch.relu(torch.randn(B, T, F, generator=g))
    unit = torch.rand(T, B * F, generator=g) + 0.3
    ref = stack(gather(magT.double(), fbT.double(), torch.ones(B, dtype=torch.float64), unit.double(), Ns, Nf, 1, T, 1),
                {k: v.double() for k, v in w.items()}, 0, 0)  # [B*F, 2, T]
    scale = max(1.0, float(ref.abs().max()))
    s = dict(H=H, B=B, F=F, T=T, Ns=Ns, Nf=Nf, magT=magT.to(dev), fbT=fbT.to(dev), scale=unit.to(dev),
             w={f"{n}{l}": w[f"{m}_l{l}"].to(dev).contiguous() for l in range(2)
                for n, m in (("w_ih", "weight_ih"), ("w_hh", "weight_hh"), ("b_ih", "bias_ih"), ("b_hh", "bias_hh"))})
    s["w"]["fc_w"], s["w"]["fc_b"] = w["fc_w"].to(dev).contiguous(), w["fc_b"].to(dev).contiguous()
    R = B * F
    for x3 in (1, 0):
        h, c = torch.zeros(2, R, H, device=dev), torch.zeros(2, R, H, device=dev)
        out = torch.cat([_sb_run(s, x3, 0, t1, h, c, [NONE] * R, t1 - 1), _sb_run(s, x3, t1, T, h, c, [NONE] * R, -1)], 1)
        got = out.cpu().double().view(B, T, 2, F).permute(0, 3, 2, 1).reshape(R, 2, T)
        err = float((got - ref).abs().max()) / scale
        print(f"sb_carry_lstm_tc H={H} {'x3' if x3 else 'single pass'}: error {err:.2e} (scale {scale:.3g})")
        assert err < TOLERANCES[(x3, H)], (H, x3, err)


# ------------------------------------------------------------------------------------------------------- whole model
def _model(norm, dev, prec, gain=1.0, seed=11):
    from fullsubnet_b200.fullsubnet.model import Model
    from oracle import fullsubnet_oracle as O
    args = dict(O.DEFAULT_MODEL_ARGS, norm_type=norm)
    m = Model(**args, precision=prec)
    m.load_state_dict(O.make_state_dict(seed=seed, args=args, sb_fc_gain=gain), strict=True)
    return m.to(dev).eval()


def _clip(L, seed, dev):
    from oracle import fullsubnet_oracle as O
    return O.make_noisy(1, L, seed=seed, speechlike=True)[0].to(dev)


def _whole(m, clip, hop=HOP):
    return m.enhance(clip[None], hop_length=hop)[0]


def _streamer(m, slots, hop=HOP):
    from fullsubnet_b200.stream import Streamer
    return Streamer(m, slots, hop=hop, tensor_cores=True)


def _run_mixed(m, dev, seed, lengths, slots=4, hop=HOP):
    rng = random.Random(seed)
    s = _streamer(m, slots, hop)
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
@pytest.mark.parametrize("prec", PRECS)
def test_stream_bit_identical_to_whole_clip(prec, norm, gain, dev):
    m = _model(norm, dev, prec, gain)
    lengths = [4800, 16000 + 77, 7 * HOP, 80000, 64 * HOP, 3 * 16000 + 129, 6000, 25 * HOP + 1]
    _run_mixed(m, dev, 1 + NORMS.index(norm) * 2 + int(gain > 1) + 10 * PRECS.index(prec), lengths)


@pytest.mark.parametrize("prec", PRECS)
def test_stream_20s_clip(prec, dev):
    m = _model("forgetting_norm", dev, prec, WB_GAIN)
    long = _clip(20 * 16000, 7, dev)
    r = Runner(_streamer(m, 1), dev)
    r.add(0, 0, long)
    while r.busy():
        r.call(64 if r.cur.get(0, [0, 0, 0])[2] < 18 * 16000 else 1)
    assert torch.equal(r.result(0), _whole(m, long))


@pytest.mark.parametrize("hop", [128, 160])
@pytest.mark.parametrize("prec", PRECS)
def test_stream_other_hops(prec, hop, dev):
    m = _model("cumulative_laplace_norm", dev, prec, WB_GAIN)
    _run_mixed(m, dev, hop + PRECS.index(prec), [4800, 3 * 16000 + 129, 40 * hop, 7 * hop + 3, 20000], slots=3, hop=hop)


def test_clip_ending_on_a_chunk_boundary(dev):
    m = _model("cumulative_laplace_norm", dev, "f16x3_tc")
    clips = {"a": _clip(12 * HOP, 21, dev), "b": _clip(3 * 16000 + 55, 22, dev), "c": _clip(8 * HOP, 23, dev)}
    r = Runner(_streamer(m, 2), dev, late=("a", "c"))
    r.add(0, "a", clips["a"])
    r.add(1, "b", clips["b"])
    r.add(0, "c", clips["c"])
    while r.busy():
        r.call(4)
    assert r.tails["a"] == 0 and r.tails["c"] == 0
    for cid, clip in clips.items():
        assert torch.equal(r.result(cid), _whole(m, clip)), cid


@pytest.mark.parametrize("prec", PRECS)
def test_stream_alone_and_among_63(prec, dev):
    m = _model("forgetting_norm", dev, prec)
    clip = _clip(12345, 3, dev)
    alone = Runner(_streamer(m, 1), dev)
    alone.add(0, "x", clip)
    many = Runner(_streamer(m, 64), dev)
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
    m = _model(norm, dev, "f16x3_tc")
    a, b = _streamer(m, 3), _streamer(m, 3)
    g = torch.Generator(device="cpu").manual_seed(9)
    for i in range(12):
        x = (0.1 * torch.randn(3, 2 * HOP, generator=g)).to(dev)
        st = [1, 1, 1] if i == 0 else [0, 0, 0]
        ya = a.step(x, st)
        yb = b.step(x, [0, 1, 0] if i == 5 else st)
        assert torch.equal(ya[0], yb[0]) and torch.equal(ya[2], yb[2]), i
    assert not torch.equal(ya[1], yb[1])


@pytest.mark.parametrize("move", ["slot_state", "copy_slot"])
def test_state_moves_between_slots(move, dev):
    m = _model("cumulative_laplace_norm", dev, "f16_tc", WB_GAIN)
    clip = _clip(9000, 4, dev)
    ref = _whole(m, clip)
    s = _streamer(m, 3)
    D, Kh = s.delay, 3 * HOP
    outs, pos, slot = [], 0, 0
    while pos < clip.numel():
        if pos == 4 * Kh:
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


def test_enhance_stream_and_graph_replay(dev):
    m = _model("forgetting_norm", dev, "f16x3_tc", WB_GAIN)
    clip = _clip(10 * HOP + 99, 8, dev)
    pieces = [clip[:4 * HOP], clip[4 * HOP:5 * HOP], clip[5 * HOP:]]
    assert torch.equal(torch.cat(list(_streamer(m, 2).enhance_stream(pieces, slot=1))), _whole(m, clip))
    eager, cap = _streamer(m, 4), _streamer(m, 4)
    g = torch.Generator(device="cpu").manual_seed(2)
    xs = [(0.1 * torch.randn(4, 3 * HOP, generator=g)).to(dev) for _ in range(6)]
    ye = [eager.step(xs[0], [1] * 4)] + [eager.step(x) for x in xs[1:]]
    yc = [cap.step(xs[0], [1] * 4).clone()]
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


def test_launch_count_does_not_grow_with_k(dev):
    lib = _lib.load()
    m = _model("cumulative_laplace_norm", dev, "f16x3_tc")
    s = _streamer(m, 4)
    counts = {}
    for K in (1, 4, 64):
        s.step(torch.zeros(4, K * HOP, device=dev), [1] * 4)
        counts[K] = lib.fsn_last_launch_count()
    torch.cuda.synchronize()
    assert counts[1] == counts[4] == counts[64] > 0, counts


def test_full_band_stepwise_branch(dev):
    """FSN_FB_STEPWISE=1: the whole-clip call runs the full band on the per-step kernels, and so does the stream."""
    code = (
        "import torch, random, sys\n"
        "sys.path.insert(0, 'tests')\n"
        "from test_gpu_fsn_stream_tc import _model, _run_mixed\n"
        "dev = torch.device('cuda:0')\n"
        "for p in ('f16x3_tc', 'f16_tc'):\n"
        "    _run_mixed(_model('forgetting_norm', dev, p, 60.0), dev, 31, [4800, 16000 + 77, 30 * 256 + 5], slots=2)\n"
        "print('ok')\n")
    env = dict(os.environ, FSN_FB_STEPWISE="1")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-c", code], cwd=root, env=env, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and out.stdout.strip().endswith("ok"), out.stdout[-2000:] + out.stderr[-4000:]


def _stream_clips(m, ys, dev, seed):
    rng = random.Random(seed)
    r = Runner(_streamer(m, ys.shape[0]), dev)
    for i in range(ys.shape[0]):
        r.add(i, i, ys[i])
    while r.busy():
        r.call(rng.choice(KS))
    return torch.stack([r.result(i) for i in range(ys.shape[0])])


def test_fixture_cumulative_norm(golden, dev):
    from oracle import fullsubnet_oracle as O
    from fullsubnet_b200.fullsubnet.model import Model
    g = golden("model_cum")
    args = dict(O.DEFAULT_MODEL_ARGS, norm_type="cumulative_laplace_norm")
    m = Model(**args, precision="f16x3_tc")
    m.load_state_dict(O.make_state_dict(seed=0, args=args, sb_fc_gain=60.0), strict=True)
    m = m.to(dev).eval()
    y = torch.from_numpy(g["full_y"]).to(dev)
    got = _stream_clips(m, y, dev, 3)
    for i in range(y.shape[0]):
        assert torch.equal(got[i], _whole(m, y[i])), i
    assert np.abs(got.cpu().numpy() - g["full_wav"]).max() < WAV_TOL


@pytest.mark.parametrize("tag", ["wa", "wb"])
def test_fixture_forgetting_norm(golden, dev, tag):
    from fullsubnet_b200.fullsubnet.model import Model
    from oracle import fullsubnet_oracle as O
    from oracle.make_golden_forgetting import FULL_LEN
    from oracle.make_golden_long import fingerprint
    g = golden(f"model_forget_{tag}")
    y = O.make_noisy(1, FULL_LEN, seed=73, speechlike=True)
    assert np.allclose(fingerprint(y), g["y_fp"], rtol=1e-6)
    args = dict(O.DEFAULT_MODEL_ARGS, norm_type="forgetting_norm")
    m = Model(**args, precision="f16x3_tc")
    m.load_state_dict(O.make_state_dict(seed=0, args=args, sb_fc_gain=1.0 if tag == "wa" else WB_GAIN), strict=True)
    m = m.to(dev).eval()
    got = _stream_clips(m, y.to(dev), dev, 4 + len(tag))
    assert torch.equal(got[0], _whole(m, y[0].to(dev)))
    assert np.abs(got.cpu().numpy() - g["wav"]).max() < WAV_TOL
