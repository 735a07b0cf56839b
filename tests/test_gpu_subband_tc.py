"""The sub-band tensor-core LSTM stack (`sb_lstm_tc_kernel<X3>`, fsn_subband_tc.cu) through its unit-test hook
`fsn_debug_sb_lstm_tc`, against a float64 statement of the same operation (model.py:98-135: reflect unfold, norm scale,
drop_band, 2 x nn.LSTM, Linear, activation, look-ahead slice; fast_fullsubnet/model.py:108-129 for the time
down-sampling of the bottleneck).

The GPU matrix covers every value of every axis the kernel accepts at least once under the compensated arithmetic
(X3, f16x3_tc): hidden size 128 / 256 / 384 (1-3 consumer warpgroups), cluster 1 / 2 / 4 x ring depth 2 / 3 / 4
(full cross at H = 384 and H = 128), partial, exact and multi-wave grids, output staging lengths, input widths
2 ... 32 with full-band neighbours, every output activation, drop_band with 1-3 groups, per-clip and per-(step, row)
scales, the bottleneck's down-sampling with a one-output Linear, and weights that saturate the gates or amplify the
output x200.  Each case also runs the single-pass fp16 variant (f16_tc).

Error = max-abs / max(1, max|ref|) over the checked rows.  Worst measured on an H100 80GB HBM3, the same bits at 400 W
and 700 W power limits (the inputs are seeded and the kernel is deterministic):

    H      x3 (f16x3_tc)   single pass (f16_tc)
    128    3.8e-7          1.2e-4
    256    6.0e-7          1.4e-4
    384    3.8e-6          4.1e-4   (both from the cases with the x200 Linear gain)

TOLERANCES sit about 4x above these, so a subtle error still fails.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import rel_max
from oracle import fast_fullsubnet_oracle as FO
from oracle import fullsubnet_oracle as O

ACT_NAMES = {0: None, 1: "ReLU", 2: "Tanh", 3: "ReLU6"}
# (x3, H) -> bound on the error, ~4x the worst measured (module docstring)
TOLERANCES = {(1, 128): 1.5e-6, (1, 256): 2.4e-6, (1, 384): 1.5e-5,
              (0, 128): 5e-4, (0, 256): 5.6e-4, (0, 384): 1.6e-3}
GUARD = 256  # NaN floats before and after crm that the kernel must not touch
FULL = [(cl, st) for cl in (1, 2, 4) for st in (2, 3, 4)]
EDGE = [(1, 2), (4, 4)]


# ------------------------------------------------------------------------------------------------ float64 reference
def _reflect(i, n):
    i = np.abs(i)
    return np.where(i >= n, 2 * (n - 1) - i, i)


def _row_map(B, F, G):
    """drop_band as Model.forward applies it (G only when B > 1): source clip and frequency of every sub-band row."""
    g = G if B > 1 and G > 1 else 1
    if g > 1:
        src_b, src_f = O.drop_band_index_map(B, F, g)
    else:
        src_b, src_f = np.arange(B), np.tile(np.arange(F), (B, 1))
    return g, F // g, src_b, src_f


def gather(magT, fbT, inv2, unit_scale, Ns, Nf, G, steps, shrink, rows=None):
    """Sub-band input [n, Ksb, steps] of the sub-band rows `rows` (default: all B*Fsub): 2Ns+1 reflected magnitude rows
    and 2Nf+1 reflected full-band rows of the row's source clip and frequency, down-sampled in time when shrink > 1,
    times inv2[clip] or unit_scale[t, row].  magT, fbT [B, src_T, F]."""
    B, _, F = magT.shape
    _, Fsub, src_b, src_f = _row_map(B, F, G)
    rows = np.arange(B * Fsub) if rows is None else np.asarray(rows)
    b, f = src_b[rows // Fsub], src_f[rows // Fsub, rows % Fsub]
    bb, b = torch.as_tensor(b)[:, None], torch.as_tensor(b)
    cm = torch.as_tensor(_reflect(f[:, None] + np.arange(-Ns, Ns + 1)[None], F))
    cf = torch.as_tensor(_reflect(f[:, None] + np.arange(-Nf, Nf + 1)[None], F))
    x = torch.cat([magT[bb, :, cm], fbT[bb, :, cf]], dim=1)  # [n, Ksb, src_T]
    if shrink > 1:
        return FO.real_time_downsampling(x, shrink)[..., :steps] * inv2[b][:, None, None]
    x = x[..., :steps]
    if unit_scale is not None:
        return x * unit_scale[:steps, torch.as_tensor(rows)].T[:, None, :]
    return x * inv2[b][:, None, None]


def stack(x, w, act, la, dtype=torch.float64):
    """2 x nn.LSTM(K -> H) + Linear(H -> fc_out) + activation over x [n, K, T] -> [n, fc_out, T - la]."""
    H = w["weight_hh_l0"].shape[1]
    lstm = torch.nn.LSTM(x.shape[1], H, num_layers=2, batch_first=True).to(dtype)
    with torch.no_grad():
        for name, p in lstm.named_parameters():
            p.copy_(w[name])
        o = lstm(x.to(dtype).transpose(1, 2))[0] @ w["fc_w"].to(dtype).T + w["fc_b"].to(dtype)
    name = ACT_NAMES[act]
    if name == "ReLU":
        o = torch.relu(o)
    elif name == "Tanh":
        o = torch.tanh(o)
    elif name == "ReLU6":
        o = torch.clamp(o, 0, 6)
    return o[:, la:].transpose(1, 2)


def _sd_weights(sd, prefix):
    w = {k: sd[f"{prefix}sequence_model.{k}"] for k in
         (f"{n}_l{l}" for l in range(2) for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"))}
    w["fc_w"], w["fc_b"] = sd[f"{prefix}fc_output_layer.weight"], sd[f"{prefix}fc_output_layer.bias"]
    return w


# ------------------------------------------------------------------------------------------------ CPU: the reference
@pytest.mark.parametrize("norm", ["offline_laplace_norm", "cumulative_laplace_norm"])
def test_reference_matches_oracle_model_forward(norm):
    """The reference above, run in float32, is the sub-band half of oracle.model_forward: its gather equals `sb_input`
    (unfold, norm, drop_band with B not a multiple of G, full-band neighbours) and its stack the model's output."""
    args = dict(O.DEFAULT_MODEL_ARGS, num_freqs=17, look_ahead=2, fb_num_neighbors=1, sb_num_neighbors=3,
                fb_model_hidden_size=16, sb_model_hidden_size=24, sb_output_activate_function="Tanh", norm_type=norm,
                num_groups_in_drop_band=2)
    sd = O.make_state_dict(seed=4, args=args)
    mag = O.stft(O.make_noisy(3, 2000, seed=9, speechlike=True), 32, 16, 32)[0].unsqueeze(1)  # [3, 1, 17, 126]
    out, inter = O.model_forward(mag, sd, args, return_intermediates=True)
    B, F, la, Ns, Nf = 3, 17, 2, 3, 1
    magT = torch.nn.functional.pad(mag, [0, la])[:, 0].transpose(1, 2).contiguous()
    fbT = inter["fb_output"][:, 0].transpose(1, 2).contiguous()
    Tp = magT.shape[1]
    raw = gather(magT, fbT, torch.ones(B), None, Ns, Nf, 1, Tp, 1)  # every (clip, frequency) unit, unscaled
    inv2, unit_scale = None, None
    if norm == "offline_laplace_norm":  # model.py:110-111: mean of the clip's whole unfolded input
        inv2 = 1.0 / (raw.reshape(B, -1).mean(1) + 1e-5)
    else:  # base_model.py:220-251: running mean of the unit's rows over the frames so far
        K = raw.shape[1]
        mean = torch.cumsum(raw.sum(1), -1) / (K * torch.arange(1, Tp + 1, dtype=raw.dtype))
        per_unit = 1.0 / (mean + O.EPSILON)  # [B*F, Tp]
        _, Fsub, src_b, src_f = _row_map(B, F, 2)
        r = np.arange(B * Fsub)
        unit_scale = per_unit[src_b[r // Fsub] * F + src_f[r // Fsub, r % Fsub]].T.contiguous()  # [Tp, R]
        inv2 = torch.ones(B)
    x = gather(magT, fbT, inv2, unit_scale, Ns, Nf, 2, Tp, 1)
    assert x.shape == inter["sb_input"].shape
    assert rel_max(x, inter["sb_input"]) < 1e-5
    ref = stack(x, _sd_weights(sd, "sb_model."), 2, la, dtype=torch.float32)  # [R, 2, T]
    ref = ref.reshape(B, F // 2, 2, -1).permute(0, 2, 1, 3)
    assert ref.shape == out.shape
    assert float((ref - out).abs().max()) < 1e-5


def test_reference_shrink_matches_fast_bottleneck():
    """With shrink > 1 the gather is the fast_fullsubnet bottleneck input (first frame alone, blocks of 2, a short last
    block) and the stack with a one-output Linear + ReLU its output."""
    sd = FO.make_fast_state_dict(seed=1)
    mag = O.stft(O.make_noisy(2, 3000, seed=5, speechlike=True), 512, 256, 512)[0].unsqueeze(1)  # T = 12
    out, inter = FO.fast_model_forward(mag, sd, return_intermediates=True)
    a = FO.DEFAULT_FAST_ARGS
    B, S, M, Nn, Ne = 2, a["shrink_size"], a["num_mels"], a["noisy_input_num_neighbors"], a["encoder_output_num_neighbors"]
    magT = inter["mel"][:, 0].transpose(1, 2).contiguous()
    fbT = inter["enc_out"][:, 0].transpose(1, 2).contiguous()
    Tp = magT.shape[1]
    assert (Tp - 1) % S != 0  # the last block is short
    Ts = 2 + (Tp - 2) // S
    raw = gather(magT, fbT, torch.ones(B), None, Nn, Ne, 1, Ts, S)
    inv2 = 1.0 / (raw.reshape(B, -1).mean(1) + 1e-5)
    x = gather(magT, fbT, inv2, None, Nn, Ne, 1, Ts, S)
    bn_shr = inter["bn_shr"].reshape(B * M, -1, Ts)
    assert x.shape == bn_shr.shape and rel_max(x, bn_shr) < 1e-5
    ref = stack(x, _sd_weights(sd, "bottleneck."), 1, 0, dtype=torch.float32)  # [B*M, 1, Ts]
    up = FO.real_time_upsampling(ref.reshape(B, M, -1), S, mag.shape[-1] + 2)
    assert float((up - inter["bn_up"][:, 0]).abs().max()) < 1e-5


# ------------------------------------------------------------------------------------------------ CPU: argument checks
def test_hook_argument_checks_need_no_gpu():
    """fsn_debug_sb_lstm_tc validates everything before its first CUDA call: these calls return on a machine without a
    GPU, with the documented error classes."""
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    host = torch.zeros(64)
    p = host.data_ptr()
    s = _lib.SeqWeights()
    ok = dict(H=384, Ns=15, Nf=0, fc_out=2, act=0, x3=1, B=3, F=33, src_T=10, G=2, la=2, steps=10, shrink=1, stages=0,
              cluster=0, unit=None)

    def call(**kw):
        a = dict(ok, **kw)
        return lib.fsn_debug_sb_lstm_tc(C.byref(s), a["H"], a["Ns"], a["Nf"], a["fc_out"], a["act"], a["x3"], p, p, a["B"],
                                        a["F"], a["src_T"], a["G"], p, a["unit"], a["la"], a["steps"], a["shrink"],
                                        a["stages"], a["cluster"], p, p, None)

    unsupported = [dict(cluster=3), dict(cluster=8), dict(cluster=-1), dict(stages=1), dict(stages=5),
                   dict(H=64), dict(H=192), dict(H=512), dict(Ns=16), dict(Ns=14, Nf=2),  # H, Ksb = 34
                   dict(shrink=2, steps=5, la=0, unit=p)]  # per-step scales with down-sampling
    shape = [dict(B=0), dict(F=1, Ns=0), dict(Ns=33), dict(Nf=33), dict(Ns=-1), dict(src_T=0), dict(steps=11),
             dict(steps=0, la=0), dict(la=10), dict(la=-1), dict(fc_out=0), dict(fc_out=3), dict(act=4), dict(G=0),
             dict(B=2, G=2), dict(B=3, G=3), dict(F=33, G=34, B=35, Ns=0), dict(shrink=0),
             dict(shrink=2, steps=7, la=0)]  # 10 source frames give 1 + ceil(9 / 2) = 6 down-sampled steps
    for kw in unsupported:
        assert call(**kw) == _lib.FSN_ERR_UNSUPPORTED, kw
        assert lib.fsn_last_error_code() == _lib.FSN_ERR_UNSUPPORTED
    for kw in shape:
        assert call(**kw) == _lib.FSN_ERR_SHAPE, kw
        assert lib.fsn_last_error_code() == _lib.FSN_ERR_SHAPE
    assert lib.fsn_debug_sb_lstm_tc(None, 384, 15, 0, 2, 0, 1, p, p, 3, 33, 10, 2, p, None, 2, 10, 1, 0, 0, p, p,
                                    None) == _lib.FSN_ERR_SHAPE  # no weights
    n3, n1 = lib.fsn_debug_sb_lstm_tc_packed_bytes(384, 1), lib.fsn_debug_sb_lstm_tc_packed_bytes(384, 0)
    assert n3 > n1 > lib.fsn_debug_sb_lstm_tc_packed_bytes(128, 0) > 0
    assert lib.fsn_debug_sb_lstm_tc_packed_bytes(192, 1) == 0 and lib.fsn_debug_sb_lstm_tc_packed_bytes(512, 0) == 0


# ------------------------------------------------------------------------------------------------ GPU: the matrix
def _case(name, **kw):
    c = dict(name=name, H=384, B=1, F=33, G=1, steps=10, la=2, Ns=15, Nf=0, act=0, unit=False, shrink=1, src_T=None,
             fc_out=2, weights="std", fc_bias=None, configs=EDGE)
    c.update(kw)
    if c["src_T"] is None:
        c["src_T"] = c["steps"]
    return pytest.param(c, id=name)


CASES = [
    # H = 384 (3 warpgroups): 3 CTAs of 16 rows (3 mod 4 != 0: clusters 2 and 4 pad the grid), drop_band G = 2 with
    # B = 3, 17 steps (two full OUT_T blocks + one frame), Linear gain 200 with ReLU6 (outputs span -2.9 ... 7.2, both
    # clamps active); every (cluster, stages)
    _case("h384_cross", H=384, B=3, F=33, G=2, steps=17, la=2, act=3, weights="gain", configs=FULL),
    # H = 128 (1 warpgroup: turn[] hands off to itself): 13 rows (one partial CTA, 3 padding CTAs at cluster 4),
    # Ksb 8, 9 steps (one-over OUT_T), saturated gates, ReLU; every (cluster, stages)
    _case("h128_cross", H=128, B=1, F=13, steps=9, la=0, Ns=3, act=1, weights="saturated", configs=FULL),
    # H = 256 (2 warpgroups): full-band neighbours (Ksb 15 + 5 = 20), G = 3 with B = 5, per-(step, row) scales, Tanh
    _case("h256_nf2_unit", H=256, B=5, F=31, G=3, steps=8, la=0, Ns=7, Nf=2, act=2, unit=True),
    # several waves of CTAs (6168 rows = 386 CTAs), Ksb 27 + 3 = 30, one output frame, Linear gain 200
    _case("h384_waves", H=384, B=24, F=257, steps=3, la=2, Ns=13, Nf=1, act=0, weights="gain"),
    # exactly one CTA (4 clips x 4 bins with G = 2), Ksb = 2 (30 zero lanes), a single step
    _case("h128_ksb2", H=128, B=4, F=9, G=2, steps=1, la=0, Ns=0, act=0),
    # H = 384, per-(step, row) scales, G = 3 with B = 4 (20 rows: 2 CTAs), saturated gates, ReLU
    _case("h384_unit_g3", H=384, B=4, F=17, G=3, steps=10, la=2, Ns=15, act=1, unit=True, weights="saturated"),
    # the fast_fullsubnet bottleneck: shrink 2 over 10 source frames (short last block), one-output Linear, ReLU
    # (the bias centres the outputs, -0.019 ... -0.009 without it, on the ReLU knee)
    _case("bn_shrink2", H=384, B=2, F=64, steps=6, la=0, Ns=5, act=1, shrink=2, src_T=10, fc_out=1, fc_bias=0.014),
    # shrink 3 over 12 source frames (last block of 2), full-band neighbours, H = 256, Tanh, saturated gates
    _case("bn_shrink3", H=256, B=3, F=21, steps=5, la=0, Ns=2, Nf=1, act=2, shrink=3, src_T=12, fc_out=1,
          weights="saturated"),
]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def worst():
    w = {}
    yield w
    for (x3, H), e in sorted(w.items()):
        print(f"sb_lstm_tc worst error {'x3' if x3 else 'single pass'} H={H}: {e:.2e}")


def _weights(H, Ksb, fc_out, mode, seed, fc_bias=None):
    g = torch.Generator().manual_seed(seed)
    k = 1.0 / H ** 0.5
    lstm_gain = 4.0 if mode == "saturated" else 1.0
    fc_gain = 200.0 if mode == "gain" else 1.0

    def u(*shape):
        return (torch.rand(*shape, generator=g) * 2 - 1) * k

    w = {}
    for l in range(2):
        w[f"weight_ih_l{l}"] = u(4 * H, Ksb if l == 0 else H) * lstm_gain
        w[f"weight_hh_l{l}"] = u(4 * H, H) * lstm_gain
        w[f"bias_ih_l{l}"] = u(4 * H) * lstm_gain
        w[f"bias_hh_l{l}"] = u(4 * H) * lstm_gain
    w["fc_w"], w["fc_b"] = u(fc_out, H) * fc_gain, u(fc_out) * fc_gain
    if fc_bias is not None:
        w["fc_b"] = torch.full((fc_out,), fc_bias)
    return w


def _inputs(c, seed):
    """magnitude-like inputs; clip 0 duplicated at the last position of its drop_band group (another CTA)."""
    g = torch.Generator().manual_seed(seed)
    B, F, src_T = c["B"], c["F"], c["src_T"]
    magT = torch.randn(B, src_T, F, generator=g).abs()
    fbT = torch.relu(torch.randn(B, src_T, F, generator=g))
    inv2 = torch.rand(B, generator=g) + 0.3
    gr, Fsub, src_b, _ = _row_map(B, F, c["G"])
    unit = torch.rand(c["steps"], B * Fsub, generator=g) + 0.3 if c["unit"] else None
    dup = None
    if B > 1:
        dst = max(b for b in range(1, B) if b % gr == 0)
        magT[dst], fbT[dst], inv2[dst] = magT[0], fbT[0], inv2[0]
        pos = [int(np.flatnonzero(src_b == b)[0]) for b in (0, dst)]
        if unit is not None:
            unit[:, pos[1] * Fsub:(pos[1] + 1) * Fsub] = unit[:, pos[0] * Fsub:(pos[0] + 1) * Fsub]
        dup = pos
    return magT, fbT, inv2, unit, dup


def _check_rows(R):
    """all rows of small grids; else first and last row of the first, second, middle, last-but-one and last CTA"""
    if R <= 512:
        return np.arange(R)
    nct = -(-R // 16)
    rows = set()
    for cta in (0, 1, nct // 2, nct - 2, nct - 1):
        rows |= {16 * cta, min(16 * cta + 15, R - 1)}
    return np.array(sorted(rows))


def _launch(dev, c, wd, d_in, x3, stages, cluster):
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    magT, fbT, inv2, unit = d_in
    s = _lib.SeqWeights()
    for l in range(2):
        s.w_ih[l], s.w_hh[l] = wd[f"weight_ih_l{l}"].data_ptr(), wd[f"weight_hh_l{l}"].data_ptr()
        s.b_ih[l], s.b_hh[l] = wd[f"bias_ih_l{l}"].data_ptr(), wd[f"bias_hh_l{l}"].data_ptr()
    s.fc_w, s.fc_b = wd["fc_w"].data_ptr(), wd["fc_b"].data_ptr()
    packed = torch.empty(lib.fsn_debug_sb_lstm_tc_packed_bytes(c["H"], x3), dtype=torch.uint8, device=dev)
    _, Fsub, _, _ = _row_map(c["B"], c["F"], c["G"])
    shape = (c["B"], 2, Fsub, c["steps"] - c["la"])
    n = int(np.prod(shape))
    buf = torch.full((n + 2 * GUARD,), float("nan"), device=dev)
    _lib.check(lib.fsn_debug_sb_lstm_tc(
        C.byref(s), c["H"], c["Ns"], c["Nf"], c["fc_out"], c["act"], x3, magT.data_ptr(), fbT.data_ptr(), c["B"],
        c["F"], c["src_T"], c["G"], inv2.data_ptr(), None if unit is None else unit.data_ptr(), c["la"], c["steps"],
        c["shrink"], stages, cluster, packed.data_ptr(), buf[GUARD:].data_ptr(), torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    buf = buf.cpu()
    assert torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[GUARD + n:]).all(), (x3, stages, cluster, "write outside crm")
    out = buf[GUARD:GUARD + n].view(shape)
    assert not torch.isnan(out).any(), (x3, stages, cluster, f"{int(torch.isnan(out).sum())} crm elements never written")
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("c", CASES)
def test_sb_lstm_tc_matches_float64(dev, worst, c):
    """Accuracy against float64, full coverage of crm (and nothing written outside it), run-to-run determinism,
    bit-identical results for every (cluster, stages), and row independence (a duplicated clip in another CTA gives the
    same bits)."""
    Ksb = (2 * c["Ns"] + 1) + (2 * c["Nf"] + 1)
    seed = sum(map(ord, c["name"]))
    w = _weights(c["H"], Ksb, c["fc_out"], c["weights"], seed, c["fc_bias"])
    magT, fbT, inv2, unit, dup = _inputs(c, seed)
    _, Fsub, _, _ = _row_map(c["B"], c["F"], c["G"])
    R = c["B"] * Fsub
    rows = _check_rows(R)
    x = gather(magT.double(), fbT.double(), inv2.double(), None if unit is None else unit.double(), c["Ns"], c["Nf"],
               c["G"], c["steps"], c["shrink"], rows)
    ref = stack(x, {k: v.double() for k, v in w.items()}, c["act"], c["la"])  # [n, fc_out, T]
    wd = {k: v.to(dev).contiguous() for k, v in w.items()}
    d_in = [None if t is None else t.to(dev).contiguous() for t in (magT, fbT, inv2, unit)]
    scale = max(1.0, float(ref.abs().max()))
    for x3 in (1, 0):
        outs = [_launch(dev, c, wd, d_in, x3, st, cl) for cl, st in c["configs"]]
        again = _launch(dev, c, wd, d_in, x3, c["configs"][0][1], c["configs"][0][0])
        assert torch.equal(again, outs[0]), "run-to-run difference"
        for (cl, st), o in zip(c["configs"], outs):
            assert torch.equal(o, outs[0]), f"cluster {cl}, stages {st} differ from {c['configs'][0]}"
        out = outs[0]
        if dup is not None:
            assert torch.equal(out[dup[0]], out[dup[1]]), "duplicated clip differs"
        if c["fc_out"] == 1:
            assert torch.equal(out[:, 1], torch.zeros_like(out[:, 1]))  # act(0 . h + 0)
        r = torch.as_tensor(rows)
        got = out[r // Fsub, :c["fc_out"], r % Fsub].double()  # [n, fc_out, T]
        err = float((got - ref).abs().max()) / scale
        print(f"{c['name']} {'x3' if x3 else 'single pass'}: error {err:.2e} (scale {scale:.3g}, {len(rows)} of {R} rows)")
        worst[(x3, c["H"])] = max(worst.get((x3, c["H"]), 0.0), err)
        assert err < TOLERANCES[(x3, c["H"])], (c["name"], x3, err)


@pytest.mark.gpu
@pytest.mark.parametrize("Hs", [128, 256])
def test_model_auto_resolves_to_x3_at_small_hidden_sizes(dev, Hs):
    """Model(precision="auto") with sb hidden 128 / 256 packs its weights (fsn_pack_sb_weights), resolves to f16x3_tc
    and matches both the fp32 kernels and oracle.model_forward, for B = 1 and for B = 3 with drop_band."""
    from fullsubnet_b200.fullsubnet.model import Model
    args = dict(O.DEFAULT_MODEL_ARGS, num_freqs=65, fb_model_hidden_size=64, sb_model_hidden_size=Hs)
    sd = O.make_state_dict(seed=Hs, args=args)
    mag = O.stft(O.make_noisy(3, 3000, seed=Hs, speechlike=True), 128, 64, 128)[0].unsqueeze(1)  # [3, 1, 65, 47]
    models = {}
    for prec in ("auto", "fp32"):
        m = Model(**args, precision=prec)
        m.load_state_dict(sd, strict=True)
        models[prec] = m.to(dev).eval()
    assert models["auto"]._resolve_precision() == "f16x3_tc"
    for x in (mag[:1], mag):
        ref = O.model_forward(x, sd, args)
        with torch.no_grad():
            got, f32 = (models[p](x.to(dev)).cpu() for p in ("auto", "fp32"))
        assert got.shape == ref.shape == f32.shape
        e_ref, e_f32 = rel_max(got, ref), rel_max(got, f32)
        print(f"model sb hidden {Hs} B={x.shape[0]}: auto vs oracle {e_ref:.2e}, vs fp32 {e_f32:.2e}")
        assert e_ref < 5e-5 and e_f32 < 5e-5
