"""Chunked streaming of fast_fullsubnet on the fp16 tensor cores (fsn_fast_stream_tc_step through
Streamer(tensor_cores=True)).

Bottleneck kernel alone (sb_phased_lstm_tc_kernel through fsn_debug_sb_lstm_tc_phased): from zero state, or restarted
at step 0 over any state, it is bit-identical to the whole-clip sb_lstm_tc_kernel with `shrink`; a run split into two
launches with the state carried and each slot at its own block phase is bit-identical to one launch; the carried result
stays within each precision's class of a float64 LSTM.  Model: every clip, under any chunking schedule, at any block
phase and alongside any other streams, concatenates to the whole-clip call of the same precision (Inferencer.
enhance_batch: fsn_stft -> fsn_fast_model_forward -> fsn_istft) bit for bit, for f16x3_tc and f16_tc, and in a
subprocess with FSN_FB_STEPWISE=1 for the encoder / decoder per-step branch; a call's launch count does not depend on K."""
import ctypes as C
import os
import random
import subprocess
import sys

import pytest
import torch

from test_gpu_stream import Runner
from test_gpu_subband_tc import TOLERANCES, _weights, gather, stack

from fullsubnet_b200 import _lib

pytestmark = pytest.mark.gpu

PRECS = ["f16x3_tc", "f16_tc"]
HOP = 256
KS = (1, 2, 3, 7, 64)
SHAPES = {"recipe": {}, "odd": dict(shrink_size=3, look_ahead=1, encoder_output_num_neighbors=1)}
RELU = 1


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _ptr(t):
    return t.data_ptr()


# ------------------------------------------------------------------------------------------ bottleneck kernel alone
def _setup(dev, H=384, B=4, M=40, S=2, Ns=5, Nf=1, n_frames=40, seed=0):
    """Weights (fc_out 1, its bias keeping most outputs above the ReLU's zero) and per-slot frames: mel / enc [B, OFF + n_frames, M], frame f of slot b at index OFF + f; one
    scale per (block, row), scale_whole [n_frames, B*M]."""
    g = torch.Generator().manual_seed(seed)
    w = _weights(H, (2 * Ns + 1) + (2 * Nf + 1), 1, "std", seed + 7, fc_bias=0.1)
    off = 8
    mel = torch.randn(B, off + n_frames, M, generator=g).abs()
    enc = torch.relu(torch.randn(B, off + n_frames, M, generator=g))
    scale = 0.5 + torch.rand(n_frames, B * M, generator=g)
    d = {k: v.to(dev).contiguous() for k, v in w.items()}
    return dict(H=H, B=B, M=M, S=S, Ns=Ns, Nf=Nf, off=off, w=w, dw=d, mel=mel.to(dev), enc=enc.to(dev),
                scale=scale.to(dev))


def _seq_weights(d):
    sw = _lib.SeqWeights()
    for l in range(2):
        sw.w_ih[l], sw.w_hh[l] = _ptr(d[f"weight_ih_l{l}"]), _ptr(d[f"weight_hh_l{l}"])
        sw.b_ih[l], sw.b_hh[l] = _ptr(d[f"bias_ih_l{l}"]), _ptr(d[f"bias_hh_l{l}"])
    sw.fc_w, sw.fc_b = _ptr(d["fc_w"]), _ptr(d["fc_b"])
    return sw


def _first_end(m0, S):
    m = max(m0, 0)
    return (m + S - 1) // S * S - m0


def _ends_before(jf, S, lim):
    return (lim - 1 - jf) // S + 1 if lim > jf else 0


def _phased(s, x3, m0, St, h, c, restart, store):
    """One launch: slot b's call steps are frames m0[b] .. m0[b] + St - 1 -> out [B, nb, 2M]; h / c updated in place"""
    lib = _lib.load()
    B, M, S, H = s["B"], s["M"], s["S"], s["H"]
    dev = h.device
    nb = -(-St // S)
    idx = torch.stack([torch.arange(St + S - 1) + s["off"] + m - (S - 1) for m in m0])  # [B, S-1+St]
    bi = torch.arange(B)[:, None]
    catM = s["mel"][bi, idx].contiguous()
    catE = s["enc"][bi, idx].contiguous()
    # the scale of the block each step ends: block (m0 + j) / S of the slot's clip
    sc = torch.ones(nb, B * M, device=dev)
    for b in range(B):
        jf = _first_end(m0[b], S)
        for i in range(nb):
            j = jf + i * S
            if j < St:
                sc[i, b * M:(b + 1) * M] = s["scale"][(m0[b] + j) // S, b * M:(b + 1) * M]
    t = lambda v: torch.as_tensor(v, dtype=torch.int32, device=dev)
    m0t, rst, sto = t(m0), t(restart), t(store)
    packed = torch.empty(lib.fsn_debug_sb_lstm_tc_packed_bytes(H, int(x3)), dtype=torch.uint8, device=dev)
    x = torch.empty(nb, B * M, (2 * s["Ns"] + 1) + (2 * s["Nf"] + 1), device=dev)
    out = torch.full((B, nb, 2 * M), float("nan"), device=dev)
    _lib.check(lib.fsn_debug_sb_lstm_tc_phased(C.byref(_seq_weights(s["dw"])), H, s["Ns"], s["Nf"], int(x3), _ptr(catM),
                                               _ptr(catE), B, M, S, St, _ptr(m0t), _ptr(sc), _ptr(rst), _ptr(sto), _ptr(h),
                                               _ptr(c), _ptr(packed), _ptr(x), _ptr(out), None))
    torch.cuda.synchronize()
    return out


def _whole_kernel(s, x3, Tp):
    """The whole-clip bottleneck: sb_lstm_tc_kernel with shrink over frames 0 .. Tp-1, per-clip scale (the blocks'
    scale_whole rows set to it) -> [B, M, Ts]"""
    lib = _lib.load()
    B, M, S, H = s["B"], s["M"], s["S"], s["H"]
    Ts = 1 + -(-(Tp - 1) // S)
    magT = s["mel"][:, s["off"]:s["off"] + Tp].contiguous()
    fbT = s["enc"][:, s["off"]:s["off"] + Tp].contiguous()
    packed = torch.empty(lib.fsn_debug_sb_lstm_tc_packed_bytes(H, int(x3)), dtype=torch.uint8, device=magT.device)
    crm = torch.full((B, 2, M, Ts), float("nan"), device=magT.device)
    _lib.check(lib.fsn_debug_sb_lstm_tc(C.byref(_seq_weights(s["dw"])), H, s["Ns"], s["Nf"], 1, RELU, int(x3), _ptr(magT),
                                        _ptr(fbT), B, M, Tp, 1, _ptr(s["inv2"]), None, 0, Ts, S, 0, 0, _ptr(packed),
                                        _ptr(crm), None))
    torch.cuda.synchronize()
    return crm[:, 0]


def _per_clip_scale(s, dev):
    """scale_whole constant over the blocks of a clip (the offline form the whole-clip hook takes with shrink)"""
    g = torch.Generator().manual_seed(3)
    s["inv2"] = (0.5 + torch.rand(s["B"], generator=g)).to(dev)
    s["scale"] = s["inv2"].repeat_interleave(s["M"])[None].expand(s["scale"].shape[0], -1).contiguous()


@pytest.mark.parametrize("S", [2, 3])
@pytest.mark.parametrize("x3", [True, False], ids=PRECS)
def test_phased_from_zero_state_equals_whole_clip_kernel(dev, x3, S):
    s = _setup(dev, S=S, seed=S)
    _per_clip_scale(s, dev)
    B, M, H = s["B"], s["M"], s["H"]
    Tp = 1 + 6 * S  # full blocks only: the whole clip's steps are exactly the stream's block ends
    ref = _whole_kernel(s, x3, Tp)  # [B, M, Ts]
    assert float((ref > 0).float().mean()) > 0.5
    R = B * M
    zeros = lambda: (torch.zeros(2, R, H, device=dev), torch.zeros(2, R, H, device=dev))
    h, c = zeros()
    got = _phased(s, x3, [0] * B, Tp, h, c, [-1] * B, [-1] * B)
    assert got.shape[1] == ref.shape[2]
    assert torch.equal(got[:, :, :M].permute(0, 2, 1), ref)
    assert torch.equal(got[:, :, M:], torch.zeros_like(got[:, :, M:]))  # the packer's zero second output, after ReLU
    # a restart at step 0 ignores whatever state the buffers hold
    h, c = torch.randn(2, R, H, device=dev), torch.randn(2, R, H, device=dev)
    assert torch.equal(_phased(s, x3, [0] * B, Tp, h, c, [0] * B, [-1] * B), got)
    # a slot whose frame 0 lies later in the call restarts at its first block end, block 0, all the same
    h, c = torch.randn(2, R, H, device=dev), torch.randn(2, R, H, device=dev)
    late = _phased(s, x3, [-2] * B, Tp + 2, h, c, [0] * B, [-1] * B)
    assert torch.equal(late[:, :got.shape[1]], got)


@pytest.mark.parametrize("S", [2, 3])
@pytest.mark.parametrize("x3", [True, False], ids=PRECS)
def test_phased_split_equals_one_launch(dev, x3, S):
    """Slots at different block phases (one fresh, the others carried from a random state), split after K1 steps: the
    first launch stores each slot's state after its last block end before K1, and its rows run on past that step."""
    s = _setup(dev, S=S, B=4, seed=10 + S)
    B, M, H, R = s["B"], s["M"], s["H"], s["B"] * s["M"]
    m0 = [-1, 1, 2, 4]
    fresh = lambda ms, St: [0 if m <= 0 and -m < St else -1 for m in ms]  # the slot's block 0 lies in the call
    T = 23
    h0, c0 = 0.5 * torch.randn(2, R, H, device=dev), 0.5 * torch.randn(2, R, H, device=dev)
    n = [_ends_before(_first_end(m, S), S, T) for m in m0]
    h1, c1 = h0.clone(), c0.clone()
    one = _phased(s, x3, m0, T, h1, c1, fresh(m0, T), [k - 1 for k in n])
    assert float((one[:, :, :M] > 0).float().mean()) > 0.5
    for K1 in (1, S, 7):
        n1 = [_ends_before(_first_end(m, S), S, K1) for m in m0]
        h2, c2 = h0.clone(), c0.clone()
        a = _phased(s, x3, m0, K1, h2, c2, fresh(m0, K1), [k - 1 for k in n1])
        m0b = [m + K1 for m in m0]
        n2 = [_ends_before(_first_end(m, S), S, T - K1) for m in m0b]
        b = _phased(s, x3, m0b, T - K1, h2, c2, fresh(m0b, T - K1), [k - 1 for k in n2])
        for sl in range(B):
            assert n1[sl] + n2[sl] == n[sl]
            assert torch.equal(torch.cat([a[sl, :n1[sl]], b[sl, :n2[sl]]]), one[sl, :n[sl]]), (K1, sl)
        assert torch.equal(h2, h1) and torch.equal(c2, c1), K1


@pytest.mark.parametrize("H", [128, 256, 384])
def test_phased_matches_float64(dev, H):
    """Two launches with the state carried between them against the float64 statement of the stack with the down-sampled
    gather (tests/test_gpu_subband_tc.py), within its per-H tolerances of the whole-sequence kernel, relative to
    max(1, max |ref|) as there."""
    S, Tp, K1 = 2, 1 + 2 * 9, 8
    s = _setup(dev, H=H, B=2, M=33, S=S, Ns=15, Nf=0, seed=H)
    _per_clip_scale(s, dev)
    B, M, R = s["B"], s["M"], s["B"] * s["M"]
    Ts = 1 + (Tp - 1) // S
    magT = s["mel"][:, s["off"]:s["off"] + Tp].cpu().double()
    fbT = s["enc"][:, s["off"]:s["off"] + Tp].cpu().double()
    ref = stack(gather(magT, fbT, s["inv2"].cpu().double(), None, s["Ns"], s["Nf"], 1, Ts, S),
                {k: v.double() for k, v in s["w"].items()}, RELU, 0)[:, 0]  # [R, Ts]
    scale = max(1.0, float(ref.abs().max()))
    assert float((ref > 0).double().mean()) > 0.5
    for x3 in (1, 0):
        h, c = torch.zeros(2, R, H, device=dev), torch.zeros(2, R, H, device=dev)
        n1 = _ends_before(0, S, K1)
        a = _phased(s, x3, [0] * B, K1, h, c, [0] * B, [n1 - 1] * B)[:, :n1]
        b = _phased(s, x3, [K1] * B, Tp - K1, h, c, [-1] * B, [-1] * B)[:, :Ts - n1]
        got = torch.cat([a, b], 1)[:, :, :M].permute(0, 2, 1).reshape(R, Ts).cpu().double()
        err = float((got - ref).abs().max()) / scale
        print(f"sb_phased_lstm_tc H={H} {'x3' if x3 else 'single pass'}: error {err:.2e} (scale {scale:.3g})")
        assert err < TOLERANCES[(x3, H)], (H, x3, err)


# ------------------------------------------------------------------------------------------------------- whole model
def _model(dev, prec, shape="recipe", fc_gain=1.0, seed=11):
    """cumulative norm, seeded weights, precision `prec`; fc_gain scales the decoder's Linear so that the cRM reaches the
    clip of decompress_cIRM."""
    from fullsubnet_b200.fast_fullsubnet.model import Model
    from oracle import fast_fullsubnet_oracle as FO
    args = dict(FO.DEFAULT_FAST_ARGS, norm_type="cumulative_laplace_norm", **SHAPES[shape])
    sd = FO.make_fast_state_dict(seed=seed, args=args)
    for k in ("decoder_lstm.1.fc_output_layer.weight", "decoder_lstm.1.fc_output_layer.bias"):
        sd[k] = sd[k] * fc_gain
    m = Model(**args, precision=prec)
    m.load_state_dict(sd, strict=True)
    return m.to(dev).eval()


def _clip(L, seed, dev):
    from oracle import fullsubnet_oracle as O
    return O.make_noisy(1, L, seed=seed, speechlike=True)[0].to(dev)


def _whole(m, clip, hop=HOP):
    from fullsubnet_b200.inferencer import Inferencer
    acoustics = {"n_fft": 512, "hop_length": hop, "win_length": 512, "sr": 16000}
    return Inferencer(config={"acoustics": acoustics}, model=m, device=clip.device).enhance_batch(clip[None])[0]


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


@pytest.mark.parametrize("fc_gain", [1.0, 8.0], ids=["Wa", "Wb"])
@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("prec", PRECS)
def test_stream_bit_identical_to_whole_clip(prec, shape, fc_gain, dev):
    m = _model(dev, prec, shape, fc_gain)
    lengths = [4800, 16000 + 77, 7 * HOP, 80000, 64 * HOP, 3 * 16000 + 129, 6000, 25 * HOP + 1]
    _run_mixed(m, dev, 1 + list(SHAPES).index(shape) * 2 + int(fc_gain > 1) + 10 * PRECS.index(prec), lengths)


@pytest.mark.parametrize("prec", PRECS)
def test_stream_20s_clip(prec, dev):
    """A 20 s clip alone, K = 64 and then K = 1 for its last 2 s."""
    m = _model(dev, prec, "recipe", 8.0)
    long = _clip(20 * 16000, 7, dev)
    r = Runner(_streamer(m, 1), dev)
    r.add(0, 0, long)
    while r.busy():
        r.call(64 if r.cur.get(0, [0, 0, 0])[2] < 18 * 16000 else 1)
    assert torch.equal(r.result(0), _whole(m, long))


@pytest.mark.parametrize("hop", [128, 160])
@pytest.mark.parametrize("prec", PRECS)
def test_stream_other_hops(prec, hop, dev):
    """hop 128: two steps of framing lag; hop 160: n_fft/2 not a multiple of hop."""
    m = _model(dev, prec, "odd" if hop == 160 else "recipe", 8.0)
    _run_mixed(m, dev, hop + PRECS.index(prec), [4800, 3 * 16000 + 129, 40 * hop, 7 * hop + 3, 20000], slots=3, hop=hop)


def test_clip_ending_on_a_chunk_boundary(dev):
    """tail = 0: the clip's last chunk was full and its end comes with the next call."""
    m = _model(dev, "f16_tc", "odd")
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


@pytest.mark.parametrize("shape", list(SHAPES))
@pytest.mark.parametrize("prec", PRECS)
def test_slots_out_of_block_phase(prec, shape, dev):
    """Two slots started one hop apart with K = 1: their frames are never at the same block phase."""
    m = _model(dev, prec, shape, 8.0)
    r = Runner(_streamer(m, 2), dev)
    clips = {"a": _clip(9000, 31, dev), "b": _clip(7 * HOP, 32, dev)}
    r.add(0, "a", clips["a"])
    r.call(1)
    r.add(1, "b", clips["b"])
    while r.busy():
        r.call(1)
    for cid, clip in clips.items():
        assert torch.equal(r.result(cid), _whole(m, clip)), cid


@pytest.mark.parametrize("prec", PRECS)
def test_stream_alone_and_among_63(prec, dev):
    m = _model(dev, prec)
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


def test_start_leaves_other_slots(dev):
    m = _model(dev, "f16x3_tc", "odd")
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
    m = _model(dev, "f16x3_tc", "odd", 8.0)
    clip = _clip(9000, 4, dev)
    ref = _whole(m, clip)
    s = _streamer(m, 3)
    D, Kh = s.delay, 1 * HOP
    outs, pos, slot = [], 0, 0
    while pos < clip.numel():
        if pos == 7 * Kh:  # mid-clip, mid-block (S = 3)
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
    m = _model(dev, "f16_tc", "recipe", 8.0)
    clip = _clip(10 * HOP + 99, 8, dev)
    pieces = [clip[:4 * HOP], clip[4 * HOP:5 * HOP], clip[5 * HOP:]]
    assert torch.equal(torch.cat(list(_streamer(m, 2).enhance_stream(pieces, slot=1))), _whole(m, clip))
    eager, cap = _streamer(m, 4), _streamer(m, 4)
    g = torch.Generator(device="cpu").manual_seed(2)
    xs = [(0.1 * torch.randn(4, 3 * HOP, generator=g)).to(dev) for _ in range(6)]
    ye = [eager.step(xs[0], [1] * 4)] + [eager.step(x) for x in xs[1:]]
    yc = [cap.step(xs[0], [1] * 4).clone()]  # also sizes the K = 3 workspace and packs the weights before the capture
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


@pytest.mark.parametrize("prec", PRECS)
def test_launch_count_does_not_depend_on_k(prec, dev):
    lib = _lib.load()
    m = _model(dev, prec)
    s = _streamer(m, 4)
    counts = {}
    for K in (1, 2, 4, 64):
        s.step(torch.zeros(4, K * HOP, device=dev), [1] * 4)
        counts[K] = lib.fsn_last_launch_count()
    torch.cuda.synchronize()
    print(f"fast_fullsubnet tensor-core stream, {prec}: {counts[1]} launches per call")
    assert counts[1] == counts[2] == counts[4] == counts[64] > 0, counts


def _stepwise_check():
    """The mixed-schedule identity on both shapes and precisions, run by test_stream_encoder_decoder_per_step in a process
    with FSN_FB_STEPWISE=1 (the whole-clip encoder and decoder then run the per-step kernels, and so must the stream)."""
    dev = torch.device("cuda:0")
    for i, shape in enumerate(SHAPES):
        for prec in PRECS:
            _run_mixed(_model(dev, prec, shape, 8.0), dev, 40 + i, [4800, 16000 + 77, 9 * HOP], slots=3)
    print("stepwise ok")


def test_stream_encoder_decoder_per_step(dev):
    here = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(here)
    env = dict(os.environ, FSN_FB_STEPWISE="1", PYTHONPATH=os.pathsep.join([here, root]))
    code = "import test_gpu_fast_stream_tc as T; T._stepwise_check()"
    p = subprocess.run([sys.executable, "-c", code], env=env, cwd=root, capture_output=True, text=True, timeout=1800)
    assert p.returncode == 0 and "stepwise ok" in p.stdout, p.stdout[-3000:] + p.stderr[-3000:]
