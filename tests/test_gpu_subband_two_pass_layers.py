"""The two passes of the whole-clip sub-band stack (`sb_l0_tc_kernel`, `sb_l1_tc_kernel`, fsn_subband_tc.cu, DESIGN
4.1.1) one at a time, chunk by chunk, through `fsn_debug_sb_tc2_pass`, against the float64 references of
tests/test_cpu_subband_two_pass_layers.py.

Every case runs both arithmetics and checks, per chunk of CTA pairs:
  * layer 0: its decoded h0 image against the step bound, element by element and step by step (all rows of small
    chunks, else the first and last row of the first, second, middle and last pair); every image byte of every row < R
    written (h0ws prefilled with 0xFF, an fp16 NaN); guard bytes around h0ws and the whole crm untouched; the same bits
    from a second run and from every other ring depth of the case;
  * layer 1, fed by encode() of chosen h0 values: its cRM against nn.LSTM in float64 over the image's operand values;
    h0ws unchanged; only the chunk's rows of crm written, NaN guards around crm untouched;
  * a clip duplicated into another pair or chunk gives the same image and cRM bits;
  * layer 0 then layer 1 per chunk gives the bits of fsn_debug_sb_lstm_tc2, the production sequence.
The cases cover H = 128 / 256 / 384, ring depths 0 (the default), 2, 3 and 4 at H = 128 and H = 384, 1, 2, 17, 253 and
1000 steps, R < 48, R not a multiple of 48 and an exact pair, several chunks (pair0 > 0) with drop_band G = 2 and
G = 3 and per-(step, row) scales, src_T > steps, look-ahead 0 and 2, every activation, saturated gates and a Linear
gain of 200.  The 1000-step case runs the production chunk of 132 pairs, so pair 131's image starts at 131 x 1000 x img
bytes, past 2^32 in both arithmetics.  A last case runs fsn_debug_sb_lstm_tc2 with the production chunk over 140 pairs
(a full chunk and a partial one) and 253 steps against the float64 stack of test_gpu_subband_tc.py.

Worst measured on an H100 80GB HBM3 at 700 W (the inputs are seeded and the kernels deterministic), with the bounds:

                                              x3 (f16x3_tc)        single pass (f16_tc)
    layer 0 step-bound ratio (C0)             2.76   (11)          0.715  (3.0)
    layer 1 error (TOL1)           H = 128    9.3e-8 (4e-7)        7.2e-5 (3e-4)
                                   H = 256    4.7e-7 (2e-6)        3.6e-5 (1.5e-4)
                                   H = 384    1.1e-5 (4.5e-5)      1.1e-3 (4.5e-3)   (the x200 Linear gain case)
    production chunks, 253 steps, H = 384     1.7e-7 (7e-7)        1.1e-5 (4.5e-5)   (E2E_TOL)

The largest x3 step ratios come from the 253-step case with saturated gates (2.4-2.8); up to 17 steps they are
0.6-1.6, at 1000 steps 1.9.  Each bound is about 4x the worst measured; the whole file runs in about 20 s."""
import ctypes as C

import numpy as np
import pytest
import torch

import test_cpu_subband_two_pass_layers as L
import test_gpu_subband_tc as T

GUARD = 256           # NaN floats before and after crm
GUARD_B = 4096        # guard bytes before and after h0ws
GUARD_V = 0x5A
# the production-chunk case's error per x3, about 4x the worst measured (module docstring)
E2E_TOL = {1: 7e-7, 0: 4.5e-5}      # measured 1.7e-7 (x3), 1.1e-5 (single pass)


def _case(name, **kw):
    c = dict(name=name, H=384, B=1, F=33, G=1, steps=10, src_T=None, la=2, Ns=15, Nf=0, act=0, unit=False,
             weights="std", chunk=132, stages=[0])
    c.update(kw)
    if c["src_T"] is None:
        c["src_T"] = c["steps"]
    return pytest.param(c, id=name)


CASES = [
    # 13 rows (one partial pair), one step (layer 0 sends no h0 to the peer at all), H = 128, every ring depth, ReLU,
    # saturated gates, 3 source frames
    _case("h128_r13_t1", H=128, B=1, F=13, steps=1, src_T=3, la=0, Ns=3, act=1, weights="saturated", stages=[2, 3, 4, 0]),
    # 40 rows, two steps (the only exchange is step 0's), H = 384, every ring depth
    _case("h384_r40_t2", H=384, B=1, F=40, steps=2, la=0, act=0, stages=[0, 2, 3, 4]),
    # 48 rows: exactly one pair (3 clips x 16 bins, G = 2), 17 steps, Linear gain 200 with ReLU6, ring depth 3
    _case("h384_exact_g2", H=384, B=3, F=33, G=2, steps=17, src_T=20, la=2, act=3, weights="gain", stages=[3]),
    # 100 rows (G = 3, B = 10) = 3 pairs, the last partial, in chunks of one pair; per-(step, row) scales, full-band
    # neighbours, Tanh, 17 steps of 19 source frames, ring depth 4
    _case("h256_g3_chunks", H=256, B=10, F=31, G=3, steps=17, src_T=19, la=0, Ns=7, Nf=2, act=2, unit=True, chunk=1,
          stages=[4]),
    # configs[1]'s 253 steps: 1152 rows (G = 2, B = 9) = 24 pairs in chunks of 10 (the last of 4), per-(step, row)
    # scales, saturated gates, ring depth 2
    _case("h384_t253_g2_chunks", H=384, B=9, F=257, G=2, steps=253, src_T=256, la=2, act=0, unit=True,
          weights="saturated", chunk=10, stages=[2]),
    # 1000 steps, 6682 rows = 140 pairs in the production chunks (132, then 8): h0ws of 4.9 / 9.7 GB
    _case("h384_t1000_production_chunk", H=384, B=26, F=257, steps=1000, la=2, Ns=13, Nf=1, act=2, stages=[0]),
]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def worst():
    w = {}
    yield w
    for k, e in sorted(w.items()):
        print(f"two-pass worst {k}: {e:.3g}")


def _seq(wd):
    from fullsubnet_b200 import _lib
    s = _lib.SeqWeights()
    for l in range(2):
        s.w_ih[l], s.w_hh[l] = wd[f"weight_ih_l{l}"].data_ptr(), wd[f"weight_hh_l{l}"].data_ptr()
        s.b_ih[l], s.b_hh[l] = wd[f"bias_ih_l{l}"].data_ptr(), wd[f"bias_hh_l{l}"].data_ptr()
    s.fc_w, s.fc_b = wd["fc_w"].data_ptr(), wd["fc_b"].data_ptr()
    return s


def _fingerprint(buf):
    """buf itself (a copy) when small, else a position-weighted int64 checksum of its 32-bit words."""
    if buf.numel() <= 1 << 28:
        return buf.clone()
    w = buf.view(torch.int32)
    total, step = 0, 1 << 26
    for i in range(0, w.numel(), step):
        part = w[i:i + step].long()
        pos = torch.arange(i, i + part.numel(), device=buf.device) % 65521 + 1
        total += int((part * pos).sum())
    return total


def _same(a, b):
    return torch.equal(a, b) if isinstance(a, torch.Tensor) else a == b


def _sample_rows(pair0, pairs, R):
    """The chunk's rows < R: all of a chunk of at most 4 pairs, else the first and last row of its first, second,
    middle and last pair."""
    lo, hi = L.NB2 * pair0, min(L.NB2 * (pair0 + pairs), R)
    if pairs <= 4:
        return list(range(lo, hi))
    rows = set()
    for p in (pair0, pair0 + 1, pair0 + pairs // 2, pair0 + pairs - 1):
        rows |= {L.NB2 * p, min(L.NB2 * p + L.NB2 - 1, R - 1)}
    return sorted(r for r in rows if r < R)


class Run:
    """One case in one arithmetic on the GPU: inputs, weights, the guarded h0ws and crm buffers and the hook calls."""

    def __init__(self, dev, c, x3):
        from fullsubnet_b200 import _lib
        self._lib, self.lib = _lib, _lib.load()
        self.dev, self.c, self.x3 = dev, c, x3
        Ksb = (2 * c["Ns"] + 1) + (2 * c["Nf"] + 1)
        seed = sum(map(ord, c["name"]))
        self.w = T._weights(c["H"], Ksb, 2, c["weights"], seed)
        self.wd = {k: v.to(dev).contiguous() for k, v in self.w.items()}
        self.s = _seq(self.wd)
        self.host = T._inputs(c, seed + 1)   # magT, fbT, inv2, unit, dup
        self.d_in = [None if t is None else t.to(dev).contiguous() for t in self.host[:4]]
        _, self.Fsub, _, _ = T._row_map(c["B"], c["F"], c["G"])
        self.R = c["B"] * self.Fsub
        self.total = -(-self.R // L.NB2)
        size = c["chunk"] or 132                     # 0: the production chunk
        self.chunks = [(p0, min(size, self.total - p0)) for p0 in range(0, self.total, size)]
        self.img = L.img_bytes(c["H"], x3)
        self.ws_bytes = self.chunks[0][1] * c["steps"] * self.img
        assert self.ws_bytes == self.lib.fsn_debug_sb_lstm_tc2_ws_bytes(self.R, c["steps"], c["H"], x3, c["chunk"])
        self.ws_all = torch.full((self.ws_bytes + 2 * GUARD_B,), GUARD_V, dtype=torch.uint8, device=dev)
        self.ws = self.ws_all[GUARD_B:GUARD_B + self.ws_bytes]
        self.packed = torch.empty(self.lib.fsn_debug_sb_lstm_tc_packed_bytes(c["H"], x3), dtype=torch.uint8,
                                  device=dev)
        self.shape = (c["B"], 2, self.Fsub, c["steps"] - c["la"])
        self.n = int(np.prod(self.shape))

    def crm_buffer(self):
        return torch.full((self.n + 2 * GUARD,), float("nan"), device=self.dev)

    def crm_of(self, buf):
        return buf[GUARD:GUARD + self.n].view(self.shape)

    def check_guards(self, crm_buf):
        g = self.ws_all
        assert bool((g[:GUARD_B] == GUARD_V).all()) and bool((g[GUARD_B + self.ws_bytes:] == GUARD_V).all()), \
            "write outside h0ws"
        assert bool(torch.isnan(crm_buf[:GUARD]).all()) and bool(torch.isnan(crm_buf[GUARD + self.n:]).all()), \
            "write outside crm"

    def run_pass(self, layer, pair0, pairs, crm_buf, stages):
        c = self.c
        magT, fbT, inv2, unit = self.d_in
        self._lib.check(self.lib.fsn_debug_sb_tc2_pass(
            C.byref(self.s), c["H"], c["Ns"], c["Nf"], c["act"], self.x3, magT.data_ptr(), fbT.data_ptr(), c["B"],
            c["F"], c["src_T"], c["G"], inv2.data_ptr(), None if unit is None else unit.data_ptr(), c["la"], c["steps"],
            stages, layer, pair0, pairs, self.packed.data_ptr(), self.ws.data_ptr(), self.ws_bytes,
            crm_buf[GUARD:].data_ptr(), torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        self.check_guards(crm_buf)

    def run_tc2(self, crm_buf):
        c = self.c
        magT, fbT, inv2, unit = self.d_in
        self._lib.check(self.lib.fsn_debug_sb_lstm_tc2(
            C.byref(self.s), c["H"], c["Ns"], c["Nf"], c["act"], self.x3, magT.data_ptr(), fbT.data_ptr(), c["B"],
            c["F"], c["src_T"], c["G"], inv2.data_ptr(), None if unit is None else unit.data_ptr(), c["la"], c["steps"],
            c["stages"][0], c["chunk"], self.packed.data_ptr(), self.ws.data_ptr(), crm_buf[GUARD:].data_ptr(),
            torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        self.check_guards(crm_buf)

    def rows_out(self, crm, rows):
        """crm rows [n, 2, T - la]"""
        r = torch.as_tensor(rows, device=crm.device)
        return crm[r // self.Fsub, :, r % self.Fsub]

    def gather(self, rows):
        """x [n, Ksb, steps] fp32 of the rows, formed as the gather warp forms it (fp32 products with the scale)."""
        magT, fbT, inv2, unit, _ = self.host
        c = self.c
        x = T.gather(magT, fbT, inv2, unit, c["Ns"], c["Nf"], c["G"], c["steps"], 1, rows)
        assert x.dtype == torch.float32
        return x.to(self.dev)


def _chosen(run, pair_global):
    return L.chosen_image(1, run.c["steps"], run.c["H"], run.x3, seed=1000 + pair_global, device=run.dev)


def _dup_rows(run):
    """(row, row) pairs of the duplicated clip: the same source in another pair, often another chunk."""
    dup = run.host[4]
    if dup is None:
        return []
    F = run.Fsub
    return [(dup[0] * F + f, dup[1] * F + f) for f in sorted({0, F // 2, F - 1})]


@pytest.mark.gpu
@pytest.mark.parametrize("x3", [1, 0], ids=["x3", "single"])
@pytest.mark.parametrize("c", CASES)
def test_two_pass_layers_against_float64(dev, worst, c, x3):
    run = Run(dev, c, x3)
    H, steps, R = c["H"], c["steps"], run.R
    dup = _dup_rows(run)
    dup_rows = {r for d in dup for r in d}
    img_bits = {}
    crm0 = run.crm_buffer()
    # ---------------- layer 0, chunk by chunk
    for pair0, pairs in run.chunks:
        rows = sorted(set(_sample_rows(pair0, pairs, R)) | {r for r in dup_rows if pair0 * L.NB2 <= r < (pair0 + pairs) * L.NB2})
        region = run.ws[:pairs * steps * run.img]
        region.fill_(0xFF)
        before = crm0.clone()
        run.run_pass(0, pair0, pairs, crm0, c["stages"][0])
        assert torch.equal(crm0.view(torch.int32), before.view(torch.int32)), "layer 0 wrote crm"
        # every image byte of every row < R written
        full = min(pairs, (R - pair0 * L.NB2) // L.NB2)
        w16 = run.ws.view(torch.int16)
        for i in range(0, full * steps * run.img // 2, 1 << 28):
            assert not bool((w16[i:min(i + (1 << 28), full * steps * run.img // 2)] == -1).any()), \
                f"unwritten image bytes in the chunk at pair {pair0}"
        if full < pairs:
            nval = R - (pair0 + full) * L.NB2
            bits = L.decode_bits(run.ws, steps, H, x3, pair=[full] * nval, n=list(range(nval)))
            assert not bool((bits == -1).any()), f"unwritten image bytes of the partial pair {pair0 + full}"
        fp = _fingerprint(region)
        for st in c["stages"][1:] + [c["stages"][0]]:   # every other ring depth, then the same run again
            region.fill_(0xFF)
            run.run_pass(0, pair0, pairs, crm0, st)
            assert _same(fp, _fingerprint(region)), f"layer 0 image differs with ring depth {st} (or run to run)"
        # the step bound on the sampled rows
        pr = [r // L.NB2 - pair0 for r in rows]
        nr = [r % L.NB2 for r in rows]
        bits = L.decode_bits(run.ws, steps, H, x3, pair=pr, n=nr)
        for r, b in zip(rows, bits):
            if r in dup_rows:
                img_bits[r] = b.clone()
        v = bits.view(torch.float16).float()
        hi, lo = v[:, :, 0], (v[:, :, 1] if x3 else None)
        h, E = L.l0_ref(run.gather(rows), run.w, hi, lo, x3)
        ratio = L.l0_excess(h, E, hi, lo, x3)
        print(f"{c['name']} x3={x3} chunk {pair0}+{pairs}: layer 0 step-bound ratio {ratio:.3g} ({len(rows)} rows)")
        worst[("layer0 ratio", x3)] = max(worst.get(("layer0 ratio", x3), 0.0), ratio)
        assert ratio <= L.C0[x3], (pair0, ratio)
    for a, b in dup:
        assert torch.equal(img_bits[a], img_bits[b]), f"rows {a} and {b} of a duplicated clip: different images"
    # ---------------- layer 1 fed by encode() of chosen values
    crm1 = run.crm_buffer()
    done = torch.zeros(R, dtype=torch.bool)
    for pair0, pairs in run.chunks:
        for p in range(pairs):
            hi, lo = _chosen(run, pair0 + p)
            run.ws[p * steps * run.img:(p + 1) * steps * run.img] = L.encode(hi, lo, x3)
        fp = _fingerprint(run.ws_all)
        run.run_pass(1, pair0, pairs, crm1, c["stages"][0])
        assert _same(fp, _fingerprint(run.ws_all)), "layer 1 wrote h0ws"
        done[pair0 * L.NB2:min((pair0 + pairs) * L.NB2, R)] = True
        out = run.crm_of(crm1)
        nan = torch.isnan(run.rows_out(out, torch.arange(R, device=dev))).flatten(1).cpu()
        assert bool((~nan[done]).all()), f"layer 1 of the chunk at pair {pair0} left crm elements of its rows unwritten"
        assert bool(nan[~done].all()), f"layer 1 of the chunk at pair {pair0} wrote rows of other chunks"
        rows = _sample_rows(pair0, pairs, R)
        vals = []
        for r in rows:
            hi, lo = _chosen(run, r // L.NB2)
            n = r % L.NB2
            vals.append(L.l1_operands(hi[0, :, n], None if lo is None else lo[0, :, n], x3))
        ref = L.l1_ref(torch.stack(vals), run.wd, c["act"], c["la"])
        err = L.l1_error(run.rows_out(out, rows), ref)
        print(f"{c['name']} x3={x3} chunk {pair0}+{pairs}: layer 1 error {err:.3g} (scale {float(ref.abs().max()):.3g})")
        worst[("layer1 error", x3, H)] = max(worst.get(("layer1 error", x3, H), 0.0), err)
        assert err < L.TOL1[(x3, H)], (pair0, err)
    # ---------------- composition: layer 0 then layer 1 per chunk = fsn_debug_sb_lstm_tc2
    comp = run.crm_buffer()
    for pair0, pairs in run.chunks:
        run.run_pass(0, pair0, pairs, comp, c["stages"][0])
        run.run_pass(1, pair0, pairs, comp, c["stages"][0])
    tc2 = run.crm_buffer()
    run.run_tc2(tc2)
    assert not bool(torch.isnan(run.crm_of(comp)).any()), "crm elements never written"
    nbits = int((comp.view(torch.int32) != tc2.view(torch.int32)).sum())
    assert nbits == 0, f"{nbits} crm elements differ from fsn_debug_sb_lstm_tc2"
    out = run.crm_of(comp)
    for a, b in dup:
        assert torch.equal(run.rows_out(out, [a]), run.rows_out(out, [b])), f"rows {a} and {b}: different crm"


@pytest.mark.gpu
@pytest.mark.parametrize("x3", [1, 0], ids=["x3", "single"])
def test_production_chunks_against_float64(dev, worst, x3):
    """fsn_debug_sb_lstm_tc2 with the production chunk over 140 pairs (132, then 8) and 253 steps, against the float64
    stack on the first and last row of the first, second, middle and last pair of each chunk."""
    c = dict(name="production", H=384, B=26, F=257, G=1, steps=253, src_T=253, la=2, Ns=13, Nf=1, act=0,
             unit=False, weights="std", chunk=0, stages=[0])
    run = Run(dev, c, x3)
    assert run.chunks == [(0, 132), (132, 8)]
    crm = run.crm_buffer()
    run.run_tc2(crm)
    out = run.crm_of(crm)
    assert not bool(torch.isnan(out).any()), "crm elements never written"
    rows = sorted(set(_sample_rows(0, 132, run.R)) | set(_sample_rows(132, 8, run.R)))
    x = run.gather(rows).cpu().double()
    ref = T.stack(x, {k: v.double() for k, v in run.w.items()}, c["act"], c["la"])
    got = run.rows_out(out, rows).cpu().double()
    err = float((got - ref).abs().max()) / max(1.0, float(ref.abs().max()))
    print(f"production chunks x3={x3}: error {err:.3g} over {len(rows)} rows")
    worst[("production error", x3)] = max(worst.get(("production error", x3), 0.0), err)
    assert err < E2E_TOL[x3], err
