"""The float64 references of the two-pass sub-band stack's passes (`sb_l0_tc_kernel` / `sb_l1_tc_kernel`,
fsn_subband_tc.cu, DESIGN 4.1.1), pinned on the CPU, with the image codec of the h0 hand-over buffer, a demonstration
that each bound sees the bugs it is there to catch, and the argument checks of the pass hook `fsn_debug_sb_tc2_pass`.
tests/test_gpu_subband_two_pass_layers.py applies them to the kernels.

h0ws image.  Layer 0 stores h0_t of the launch's pair p (48 rows) at byte (p Tp + t) img, img = PARTS nkh 6144: for
part (hi, then lo under x3), k-block s (units 64 s ... 64 s + 63) and row n, unit u at part nkh 6144 + s 6144 +
swz128_off(n, u mod 64), the 128B-swizzled K-major layout the MMA reads back as its B operand.  `encode` / `decode`
state that layout; the pins below hold it to a restatement of swz128_off and of the kernel's store expression.

Layer 0, step bound.  Step t starts from the kernel's own h0_{t-1} (the decoded image of step t - 1: hi, and lo under
x3; zero at t = 0) and carries only c in float64.  x_t is formed as the gather warp forms it: v = src * scale in fp32
(scale inv2[clip], or unit_scale[t R + row]), hi = rn16(v), lo = rn16(v - hi); W_ih0 and W_hh0 are split the same way;
the products are the ones the kernel issues (hi.hi + hi.lo + lo.hi under x3, hi.hi in the single pass).  With E the
first-order gate conditioning of test_cpu_rec_tc_kernels.py propagated through the cell,

    x3:          |hi + lo - h_ref| <= C0 2^-23 E + 2^-22 |h_ref| + 2^-25    (the last two: the image's representation)
    single pass: hi is rn16 of a value within C0 2^-23 E of h_ref

element-wise, every step.  Layer 1 exposes only the cRM: its reference is nn.LSTM (one layer) in float64 over the exact
operand values of a given image (hi + lo, or hi), then Linear, activation and look-ahead slice, and its bound is the
max-abs / max(1, max|ref|) error TOL1.  The bounds are about 4x the worst measured on an H100
(tests/test_gpu_subband_two_pass_layers.py gives the numbers)."""
import ctypes as C
import math

import pytest
import torch

import test_cpu_rec_tc_kernels as RT
from test_cpu_rec_tc_kernels import D, S, split16

NB2 = 48                  # rows per CTA pair
KB = 64                   # units per k-block
S_KBLK2 = NB2 * KB * 2    # 6144 bytes: one k-block of one part
# layer 0's step bound: c per mode (x3), about 4x the worst ratio measured (tests/test_gpu_subband_two_pass_layers.py)
C0 = {1: 11.0, 0: 3.0}           # measured 2.76 (x3), 0.715 (single pass)
# layer 1's end-to-end bound per (x3, H), about 4x the worst error measured (same place)
TOL1 = {(1, 128): 4e-7, (1, 256): 2e-6, (1, 384): 4.5e-5,      # measured 9.3e-8, 4.7e-7, 1.1e-5
        (0, 128): 3e-4, (0, 256): 1.5e-4, (0, 384): 4.5e-3}      # measured 7.2e-5, 3.6e-5, 1.1e-3
ACT = {0: lambda v: v, 1: torch.relu, 2: torch.tanh, 3: lambda v: torch.clamp(v, 0, 6)}


# ------------------------------------------------------------------ the h0ws image codec
def swz128_off(row, k):
    """fsn_tc_ptx.cuh swz128_off: byte offset of (row, k < 64) in a 128B-swizzled block of 64 k (rows of 128 B)."""
    return (row >> 3) * 1024 + (row & 7) * 128 + ((((k >> 3) ^ (row & 7)) & 7) << 4) + (k & 7) * 2


def img_bytes(H, x3):
    return (2 if x3 else 1) * (H // KB) * S_KBLK2


def image_index(H, x3, device="cpu"):
    """[PARTS, 48, H] int64: fp16 element offset (bytes / 2) of (part, row n, unit u) within one image."""
    parts, nkh = (2 if x3 else 1), H // KB
    n = torch.arange(NB2)[:, None]
    u = torch.arange(H)[None, :]
    k = u % KB
    off = (n >> 3) * 1024 + (n & 7) * 128 + ((((k >> 3) ^ (n & 7)) & 7) << 4) + (k & 7) * 2 + (u // KB) * S_KBLK2
    idx = torch.stack([off + p * nkh * S_KBLK2 for p in range(parts)])
    return (idx // 2).to(device)


def encode(hi, lo, x3):
    """hi, lo [pairs, steps, 48, H] (fp16-representable; lo ignored in the single pass) -> the uint8 image bytes of
    pairs x steps images, pair-major."""
    P, T, _, H = hi.shape
    idx = image_index(H, x3, hi.device)
    words = torch.empty(P, T, img_bytes(H, x3) // 2, dtype=torch.float16, device=hi.device)
    words[..., idx[0]] = hi.half()
    if x3:
        words[..., idx[1]] = lo.half()
    return words.view(torch.uint8).reshape(-1)


def decode_bits(buf, steps, H, x3, pair=None, n=None):
    """The fp16 bits (int16) of an image buffer: [pairs, steps, PARTS, 48, H], or with `pair` / `n` (equal-length
    index lists) only those rows: [rows, steps, PARTS, H]."""
    idx = image_index(H, x3, buf.device)
    W = img_bytes(H, x3) // 2
    w = buf.view(torch.int16)
    if pair is None:
        return w.reshape(-1, steps, W)[:, :, idx]
    pair = torch.as_tensor(pair, device=buf.device).long()
    n = torch.as_tensor(n, device=buf.device).long()
    base = (pair[:, None] * steps + torch.arange(steps, device=buf.device)[None, :]) * W  # [rows, steps]
    return w[base[:, :, None, None] + idx[:, n].permute(1, 0, 2)[:, None]]


def decode(buf, steps, H, x3, pair=None, n=None):
    """decode_bits as float32 values: (hi, lo), lo None in the single pass."""
    bits = decode_bits(buf, steps, H, x3, pair, n)
    v = bits.view(torch.float16).float()
    hi, lo = v.select(-3, 0), (v.select(-3, 1) if x3 else None)
    return hi, lo


# ------------------------------------------------------------------ layer 0: the step reference
def _dev(w, device):
    return {k: v.to(device) for k, v in w.items()}


def l0_ref(x, w, hi, lo, x3):
    """Layer 0 from the kernel's own h0_{t-1}: x [n, Ksb, T] fp32 as the gather warp forms it, hi / lo [n, T, H] the
    decoded image of the same rows (lo None in the single pass; step T - 1's image is not read).  Returns h [n, T, H]
    and its bound E [n, T, H] in units of S, both float64."""
    w = _dev(w, x.device)
    n, _, T = x.shape
    H = w["weight_hh_l0"].shape[1]
    xh, xl = split16(x.transpose(1, 2))
    Wih, Wil = split16(w["weight_ih_l0"])
    Whh, Whl = split16(w["weight_hh_l0"])
    hp_h = torch.zeros(n, T, H, dtype=D, device=x.device)
    hp_l = torch.zeros_like(hp_h)
    hp_h[:, 1:] = hi[:, :-1].to(D)
    if x3:
        hp_l[:, 1:] = lo[:, :-1].to(D)
    pairs = [(xh, Wih), (hp_h, Whh)]
    if x3:
        pairs += [(xh, Wil), (xl, Wih), (hp_h, Whl), (hp_l, Whh)]
    b, bc = RT.bias_of(w["bias_ih_l0"], w["bias_hh_l0"])
    z, cond = b.expand(n, T, 4 * H).clone(), bc.expand(n, T, 4 * H).clone()
    for s_, W_ in pairs:
        z += s_ @ W_.T
        cond += s_.abs() @ W_.abs().T
    h, _, Eh, _ = RT.ref_cell(z, dz=cond, da=1.0, dr=1.0)
    return h, Eh


def _ulp16(a):
    """fp16 spacing at magnitude a >= 0 (float64): 2^(e - 10) for a in [2^e, 2^(e+1)), 2^-24 below 2^-14."""
    e = torch.floor(torch.log2(a.clamp_min(2.0 ** -24))).clamp_min(-14)
    return torch.exp2(e - 10)


def l0_excess(h, E, hi, lo, x3):
    """The step bound's ratio: max over elements of (distance of the image from h beyond its representation error) /
    (S E).  x3: |hi + lo - h| less 2^-22 |h| + 2^-25; single pass: the distance from h of the interval of reals that
    round to hi.  inf if the image holds a NaN."""
    hi = hi.to(D)
    if not bool(torch.isfinite(hi).all()) or (x3 and not bool(torch.isfinite(lo).all())):
        return math.inf
    if x3:
        gap = ((hi + lo.to(D) - h).abs() - 2.0 ** -22 * h.abs() - 2.0 ** -25).clamp_min(0)
    else:
        away, toward = _ulp16(hi.abs()), _ulp16(hi.abs() * (1 - 2.0 ** -12))
        neg = hi < 0
        lower = hi - torch.where(neg, away, toward) / 2
        upper = hi + torch.where(neg, toward, away) / 2
        gap = (lower - h).clamp_min(0) + (h - upper).clamp_min(0)
    return float((gap / (S * E)).max()) if gap.numel() else 0.0


# ------------------------------------------------------------------ layer 1: the end-to-end reference
def l1_operands(hi, lo, x3):
    """The values layer 1's MMAs read from an image: hi + lo under x3, hi in the single pass (float64)."""
    return hi.to(D) + lo.to(D) if x3 else hi.to(D)


def l1_ref(v, w, act, la):
    """nn.LSTM (one layer, layer 1's weights) in float64 over v [n, T, H], Linear(H -> 2), activation, look-ahead
    slice: [n, 2, T - la]."""
    H = v.shape[-1]
    lstm = torch.nn.LSTM(H, H, batch_first=True).to(device=v.device, dtype=D)
    with torch.no_grad():
        for name in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"):
            getattr(lstm, f"{name}_l0").copy_(w[f"{name}_l1"])
        o = lstm(v.to(D))[0] @ w["fc_w"].to(device=v.device, dtype=D).T + w["fc_b"].to(device=v.device, dtype=D)
    return ACT[act](o)[:, la:].transpose(1, 2)


def l1_error(got, ref):
    """max-abs / max(1, max|ref|); inf if got holds a NaN."""
    err = (got.to(D) - ref).abs()
    if not bool(torch.isfinite(err).all()):
        return math.inf
    return float(err.max()) / max(1.0, float(ref.abs().max()))


# ------------------------------------------------------------------ a float64 emulation of both passes, with planted bugs
def _mm(s, W, x3, drop=()):
    """s W^T as the kernel issues it over fp32 s [n, K] and W [4H, K] fp32: hi.hi, and under x3 + hi.lo (state lo,
    drop "s_lo") + lo.hi (weight lo, drop "w_lo")."""
    sh, sl = split16(s)
    Wh, Wl = split16(W)
    z = sh @ Wh.T
    if x3 and "s_lo" not in drop:
        z = z + sl @ Wh.T
    if x3 and "w_lo" not in drop:
        z = z + sh @ Wl.T
    return z


def _cell(z, c):
    H = z.shape[-1] // 4
    i, f, g, o = torch.sigmoid(z[:, :H]), torch.sigmoid(z[:, H:2 * H]), torch.tanh(z[:, 2 * H:3 * H]), torch.sigmoid(z[:, 3 * H:])
    c = f * c + i * g
    return (o * torch.tanh(c)).float(), c


def emulate_l0(u, scale, w, x3, bug=None):
    """Layer 0 of pairs = R / 48 full pairs in float64 from fp32 h, as the kernel runs it, to the image bytes it stores.
    u [R, Ksb, T] the gathered (unscaled) inputs, scale [T, R] per-(step, row) scales, both fp32."""
    R, K, T = u.shape
    H = w["weight_hh_l0"].shape[1]
    rows = torch.arange(R)
    src = {"scale_row": rows ^ 1, "scale_pair": (rows + NB2) % R}.get(bug, rows)  # whose scale each row reads
    x = u * scale[:, src].T[:, None, :]
    drop = (bug,) if bug in ("w_lo", "s_lo") else ()
    b = w["bias_ih_l0"].to(D) + w["bias_hh_l0"].to(D)
    hall = torch.zeros(R, T, H)
    c = torch.zeros(R, H, dtype=D)
    for t in range(T):
        back = 2 if bug == "parity" else 1          # "parity": step t reads h0_{t-2}, the other buffer
        hp = hall[:, t - back] if t >= back else torch.zeros(R, H)
        z = b + _mm(x[:, :, t], w["weight_ih_l0"], x3, drop) + _mm(hp, w["weight_hh_l0"], x3, drop)
        hall[:, t], c = _cell(z, c)
    hi, lo = split16(hall)
    img = [v.reshape(R // NB2, NB2, T, H).transpose(1, 2).clone() for v in (hi, lo)]
    for v in img:
        if bug == "kblock":                          # the last k-block also stored at s = 0, over k-block 0
            v[..., :KB] = v[..., H - KB:]
        if bug == "pair_shift":                      # pair p's image at p + 1
            v[:] = v.roll(1, 0)
    return encode(img[0], img[1], x3), x


def emulate_l1(buf, steps, w, x3, act, la, bug=None):
    """Layer 1 in float64 from fp32 h1 as the kernel runs it over an image buffer of full pairs: [R, 2, T - la]."""
    H = w["weight_hh_l1"].shape[1]
    hi, lo = decode(buf, steps, H, x3)
    R = hi.shape[0] * NB2
    hi, lo = [None if v is None else v.transpose(1, 2).reshape(R, steps, H) for v in (hi, lo)]
    b = w["bias_ih_l1"].to(D) + w["bias_hh_l1"].to(D)
    h1 = torch.zeros(R, H)
    c = torch.zeros(R, H, dtype=D)
    out = []
    for t in range(steps):
        tt = t - 1 if bug == "lag" else t             # "lag": step t reads the image of step t - 1
        xh = hi[:, tt].to(D) if tt >= 0 else torch.zeros(R, H, dtype=D)
        xl = lo[:, tt].to(D) if (x3 and tt >= 0 and bug != "no_lo") else torch.zeros(R, H, dtype=D)
        if bug == "last_kblock":                      # the last k-block of h0_t never reaches the MMA
            xh[:, H - KB:], xl[:, H - KB:] = 0, 0
        Wh, Wl = split16(w["weight_ih_l1"])
        z = b + xh @ Wh.T + (xl @ Wh.T + xh @ Wl.T if x3 else 0) + _mm(h1, w["weight_hh_l1"], x3)
        h1, c = _cell(z, c)
        out.append(h1.to(D) @ w["fc_w"].to(D).T + w["fc_b"].to(D))
    return ACT[act](torch.stack(out, 2))[..., la:]


def chosen_image(pairs, steps, H, x3, seed, device="cpu"):
    """h0-like values in (-1, 1) for every row of `pairs` pairs, split as the kernel splits h: (hi, lo) [pairs, steps,
    48, H] float32."""
    g = torch.Generator(device=device).manual_seed(seed)
    v = torch.tanh(torch.randn(pairs, steps, NB2, H, generator=g, device=device) * 0.8)
    v = v.float()
    hi = v.half().float()
    return hi, (v - hi).half().float()


def _weights(H, Ksb, seed, mode="std"):
    import test_gpu_subband_tc as TG
    return TG._weights(H, Ksb, 2, mode, seed)


# ------------------------------------------------------------------ pins: the codec
@pytest.mark.parametrize("x3", [0, 1])
@pytest.mark.parametrize("H", [128, 256, 384])
def test_codec_is_the_kernel_layout_and_a_bijection(H, x3):
    """image_index is swz128_off of (row, unit mod 64) in k-block unit / 64 of part (hi, then lo); that offset is what
    the kernel's store computes (ub + (n >> 3) 1024 + (n & 7) 128 + ((chunk ^ (n & 7)) << 4), ub = (u & 7) 2, chunk =
    u >> 3); it covers every fp16 word of the image exactly once; and encode / decode invert each other."""
    idx = image_index(H, x3)
    nkh, parts = H // KB, (2 if x3 else 1)
    assert idx.shape == (parts, NB2, H)
    for part in range(parts):
        for n in range(NB2):
            for u in range(H):
                s, k = divmod(u, KB)
                store = (k & 7) * 2 + (n >> 3) * 1024 + (n & 7) * 128 + (((k >> 3) ^ (n & 7)) << 4)
                assert store == swz128_off(n, k)
                assert int(idx[part, n, u]) * 2 == part * nkh * S_KBLK2 + s * S_KBLK2 + swz128_off(n, k)
    assert torch.equal(idx.flatten().sort().values, torch.arange(img_bytes(H, x3) // 2))
    g = torch.Generator().manual_seed(H + x3)
    buf = torch.randint(0, 256, (3 * 2 * img_bytes(H, x3),), generator=g, dtype=torch.uint8)
    buf.view(torch.int16)[(buf.view(torch.int16) & 0x7C00) == 0x7C00] = 0   # no inf / NaN words: values round-trip
    hi, lo = decode(buf, 2, H, x3)
    assert torch.equal(encode(hi, lo, x3), buf)
    bits = decode_bits(buf, 2, H, x3)
    for p, t, n in ((0, 0, 0), (2, 1, 47), (1, 0, 13)):
        r = decode_bits(buf, 2, H, x3, pair=[p], n=[n])
        assert torch.equal(r[0, t], bits[p, t, :, n])


# ------------------------------------------------------------------ pins: the references
@pytest.mark.parametrize("x3", [0, 1])
def test_l0_ref_is_the_layer_from_its_own_state(x3):
    """Fed the split of nn.LSTM's own float64 h0 (as fp32), l0_ref is nn.LSTM's layer 0 within the fp16 operand
    budget (2^-20 relative to the conditioning under x3; the single pass is far off it), step 0 ignores the image, and
    the last step's image is never read."""
    H, K, T, n = 128, 31, 7, 5
    w = _weights(H, K, 7)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(n, K, T, generator=g).abs()
    lstm = torch.nn.LSTM(K, H, batch_first=True).double()
    with torch.no_grad():
        for name, p in lstm.named_parameters():
            p.copy_(w[name])
        h_exact = lstm(x.to(D).transpose(1, 2))[0]
    hi, lo = split16(h_exact.float())
    h, E = l0_ref(x, w, hi, lo, x3)
    err = float((h - h_exact).abs().max())
    if x3:
        assert err < 1e-6
    else:
        assert 1e-5 < err < 1e-2
    junk = torch.randn(n, T, H)
    h2, _ = l0_ref(x, w, junk, junk, x3)
    h3, _ = l0_ref(x, w, torch.cat([hi[:, :-1], junk[:, -1:]], 1), torch.cat([lo[:, :-1], junk[:, -1:]], 1), x3)
    assert torch.equal(h2[:, 0], h[:, 0]) and torch.equal(h3, h)
    assert bool((E > 0).all())


def test_l0_excess_single_pass_is_the_rounding_interval():
    """The single-pass ratio is zero exactly for values that round to hi, and measures the distance beyond the
    rounding interval otherwise, at a normal value, at a power of two and in the subnormal range."""
    E = torch.ones(1, dtype=D)
    for v in (0.3, 0.5, -0.5, 2.0 ** -15, 0.0):
        hi = torch.tensor([v]).half().float()
        ulp_up = float(_ulp16(hi.abs().to(D)))   # the spacing away from zero
        h_in = torch.tensor([float(hi) + 0.49 * ulp_up * (1 if v >= 0 else -1)], dtype=D)
        assert l0_excess(h_in, E, hi, None, 0) == 0.0
        h_out = torch.tensor([float(hi) + (0.5 * ulp_up + 3 * S) * (1 if v >= 0 else -1)], dtype=D)
        assert 2.9 < l0_excess(h_out, E, hi, None, 0) < 3.1
    # below a power of two the spacing halves
    hi = torch.tensor([0.5])
    assert l0_excess(torch.tensor([0.5 - 2.0 ** -13 + 1e-12], dtype=D), E, hi, None, 0) == 0.0
    assert l0_excess(torch.tensor([0.5 - 2.0 ** -12], dtype=D), E, hi, None, 0) > 1.0
    assert l0_excess(torch.tensor([0.5], dtype=D), E, torch.tensor([math.nan]), None, 0) == math.inf


def test_l1_ref_is_layer_1_of_the_stack_reference():
    """l1_ref over layer 0's exact float64 output is the two-layer float64 stack of test_gpu_subband_tc."""
    import test_gpu_subband_tc as TG
    H, K, T, n = 128, 9, 6, 4
    w = _weights(H, K, 3)
    x = torch.randn(n, K, T, generator=torch.Generator().manual_seed(2), dtype=torch.float32).to(D)
    lstm = torch.nn.LSTM(K, H, batch_first=True).double()
    with torch.no_grad():
        for name, p in lstm.named_parameters():
            p.copy_(w[name])
        h0 = lstm(x.transpose(1, 2))[0]
    for act, la in ((0, 0), (2, 2), (3, 1)):
        want = TG.stack(x, {k: v.double() for k, v in w.items()}, act, la)  # [n, 2, T - la]
        got = l1_ref(h0, w, act, la)
        assert got.shape == want.shape == (n, 2, T - la)
        assert torch.allclose(got, want, rtol=0, atol=1e-13)


# ------------------------------------------------------------------ the bounds see planted bugs
def _l0_inputs(H, T, seed, pairs=2):
    R, K = pairs * NB2, 31
    g = torch.Generator().manual_seed(seed)
    u = torch.randn(R, K, T, generator=g).abs()
    scale = torch.rand(T, R, generator=g) + 0.3
    return u, scale, _weights(H, K, seed)


def _l0_ratio(buf, x, w, T, H, x3):
    hi, lo = decode(buf, T, H, x3)
    R = hi.shape[0] * NB2
    hi, lo = [None if v is None else v.transpose(1, 2).reshape(R, T, H) for v in (hi, lo)]
    h, E = l0_ref(x, w, hi, lo, x3)
    return l0_excess(h, E, hi, lo, x3)


L0_BUGS = ["parity", "scale_row", "scale_pair", "kblock", "pair_shift"]


@pytest.mark.parametrize("x3", [0, 1])
@pytest.mark.parametrize("H", [128, 384])
def test_layer0_step_bound_catches_planted_bugs(H, x3):
    """The emulated layer 0 passes its step bound; each planted bug breaks it with the larger c of either mode: h0 read
    from the wrong double buffer, a row scaled by its neighbour's or the neighbouring pair's row's scale, one k-block
    stored at the wrong s, a pair's image stored at p + 1; under x3 also the W_lo.S_hi or the S_lo products dropped."""
    T = 6
    u, scale, w = _l0_inputs(H, T, H + x3)
    x = u * scale.T[:, None, :]
    buf, xe = emulate_l0(u, scale, w, x3)
    assert torch.equal(xe, x)
    assert _l0_ratio(buf, x, w, T, H, x3) <= 0.5
    c_max = max(C0.values())
    for bug in L0_BUGS + (["w_lo", "s_lo"] if x3 else []):
        bad, _ = emulate_l0(u, scale, w, x3, bug=bug)
        r = _l0_ratio(bad, x, w, T, H, x3)
        assert r > c_max, (bug, r)


@pytest.mark.parametrize("x3", [0, 1])
@pytest.mark.parametrize("H, mode, act", [(128, "std", 2), (384, "gain", 0)])
def test_layer1_bound_catches_planted_bugs(H, mode, act, x3):
    """The emulated layer 1 over an encoded image is well within TOL1 of its float64 reference; reading the image of
    step t - 1 at step t, missing the last k-block of h0 and (x3) ignoring the lo image each break TOL1.  H = 384 runs
    the x200 Linear gain, the weights that set TOL1 there."""
    T, la = 8, 2
    w = _weights(H, 31, 5 + H + x3, mode)
    hi, lo = chosen_image(2, T, H, x3, seed=H)
    buf = encode(hi, lo, x3)
    v = l1_operands(*[None if a is None else a.transpose(1, 2).reshape(-1, T, H) for a in (hi, lo)], x3)
    ref = l1_ref(v, w, act, la)
    tol = TOL1[(x3, H)]
    assert l1_error(emulate_l1(buf, T, w, x3, act, la), ref) < tol / 2
    for bug in ["lag", "last_kblock"] + (["no_lo"] if x3 else []):
        e = l1_error(emulate_l1(buf, T, w, x3, act, la, bug=bug), ref)
        assert e > tol, (bug, e)


# ------------------------------------------------------------------ argument checks (no GPU)
def test_pass_hook_refuses_before_any_cuda_call():
    """fsn_debug_sb_tc2_pass rejects a bad layer, a chunk beyond the rows, a short or missing h0ws, a bad ring depth
    and every shape fsn_debug_sb_lstm_tc2 rejects, with its error class and before any CUDA call (no GPU here: a CUDA
    call would report FSN_ERR_CUDA)."""
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    SH, WS, UN = _lib.FSN_ERR_SHAPE, _lib.FSN_ERR_WORKSPACE, _lib.FSN_ERR_UNSUPPORTED
    host = torch.zeros(64)
    p = host.data_ptr()
    s = _lib.SeqWeights()
    # B = 7 clips x 33 bins, G = 2: 16 sub-band bins, 112 rows = 3 pairs (the last partial)
    ok = dict(sb=C.byref(s), H=384, Ns=15, Nf=0, act=0, x3=1, B=7, F=33, src_T=12, G=2, unit=None, la=2, steps=10,
              stages=0, layer=0, pair0=1, pairs=2, h0ws=p, crm=p)
    img = 2 * 6 * 6144
    ok["nb"] = 2 * 10 * img

    def call(**kw):
        a = dict(ok, **kw)
        return lib.fsn_debug_sb_tc2_pass(a["sb"], a["H"], a["Ns"], a["Nf"], a["act"], a["x3"], p, p, a["B"], a["F"],
                                         a["src_T"], a["G"], p, a["unit"], a["la"], a["steps"], a["stages"], a["layer"],
                                         a["pair0"], a["pairs"], p, a["h0ws"], a["nb"], a["crm"], None)
    cases = [(dict(layer=2), SH), (dict(layer=-1), SH),
             (dict(pair0=2, pairs=2), SH), (dict(pair0=0, pairs=4), SH), (dict(pair0=3, pairs=1), SH),
             (dict(pair0=-1), SH), (dict(pairs=0), SH), (dict(pair0=1 << 30, pairs=1 << 30), SH),
             (dict(h0ws=None), WS), (dict(nb=2 * 10 * img - 1), WS), (dict(x3=0, nb=2 * 10 * img // 2 - 1), WS),
             (dict(steps=11, src_T=12, nb=2 * 11 * img - 1), WS),
             (dict(stages=1), UN), (dict(stages=5), UN), (dict(stages=5, layer=2), UN),
             (dict(H=192), UN), (dict(H=64), UN), (dict(Ns=16), UN), (dict(Ns=14, Nf=2), UN),
             (dict(sb=None), SH), (dict(crm=None), SH), (dict(act=4), SH), (dict(act=-1), SH), (dict(B=0), SH),
             (dict(B=2, G=2), SH), (dict(G=0), SH), (dict(F=1, Ns=0), SH), (dict(steps=13), SH), (dict(steps=0, la=0), SH),
             (dict(la=10), SH), (dict(la=-1), SH), (dict(src_T=0), SH)]
    for kw, code in cases:
        assert call(**kw) == code, kw
        assert lib.fsn_last_error_code() == code, kw
    # a chunk that ends exactly at the last (partial) pair is accepted up to the ring depth check
    assert call(pair0=0, pairs=3, nb=3 * 10 * img, stages=1) == UN
