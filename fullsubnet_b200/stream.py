"""Chunked streaming enhancement (DESIGN 4.14): ``Streamer`` advances many streams by K hops per call and returns, for
each clip, the samples of the whole-clip ``enhance`` call bit for bit, ``delay`` samples later.

Built for fullband_baseline with ``cumulative_laplace_norm`` or ``forgetting_norm`` (LSTM, fp32), for fullsubnet with
``cumulative_laplace_norm`` or ``forgetting_norm`` (LSTM, ``precision="fp32"``) and for fast_fullsubnet with
``cumulative_laplace_norm`` (LSTM, ``precision="fp32"``).  Each model names its library calls in
``STREAM_ENTRY_POINTS`` and gives their arguments through ``_stream_desc()`` and ``_stream_weights()``.

``tensor_cores=True`` streams fullsubnet and fast_fullsubnet on their fp16 tensor-core precision (``f16x3_tc`` or
``f16_tc``, what the model resolves to, so ``precision="auto"`` too), bit for bit the whole-clip call of that precision,
through ``STREAM_TC_ENTRY_POINTS``, ``_stream_tc_desc()`` and ``_stream_tc_weights()``."""
from __future__ import annotations

import ctypes as C
from typing import Iterable, Iterator, Optional

import numpy as np
import torch

from . import _lib


class Streamer:
    """Owns the stream state of ``slots`` slots and a workspace per chunk length of the model ``model``.

    ``step(chunk [slots, K*hop], start=None, tail=None) -> enhanced [slots, K*hop + delay]`` on the current CUDA stream:
    ``start[b]`` truthy begins a new clip in slot b with this chunk; ``tail[b] >= 0`` ends slot b's clip after that many
    samples of the chunk (-1 or None: it goes on).  Row b's first K*hop samples are the clip's samples [pos - delay,
    pos - delay + K*hop), pos being the clip's position before the call (negative positions as 0); on the call that
    ends the clip the row holds the samples from pos - delay to the clip's end, then 0.

    ``tensor_cores=False`` (default): the fp32 kernels, for models built with ``precision="fp32"`` (fullsubnet,
    fast_fullsubnet) and for fullband_baseline.  ``tensor_cores=True``: fullsubnet and fast_fullsubnet on the fp16 tensor
    cores, for models that resolve to ``f16x3_tc`` or ``f16_tc`` (``precision="auto"`` included); the output matches the
    whole-clip call of that precision, the delay and the state size are those of the fp32 stream."""

    def __init__(self, model, slots: int, n_fft: int = 512, hop: int = 256, win_length: int = 512,
                 tensor_cores: bool = False):
        if tensor_cores:
            names = getattr(type(model), "STREAM_TC_ENTRY_POINTS", ())
            if not names:
                raise NotImplementedError("fullsubnet_b200: tensor-core streaming (tensor_cores=True) is built for "
                                          "fullsubnet and fast_fullsubnet; stream this model with tensor_cores=False")
            self._desc_of, self._weights_of = model._stream_tc_desc, model._stream_tc_weights
        else:
            names = getattr(type(model), "STREAM_ENTRY_POINTS", ())
            if not names:
                raise NotImplementedError("fullsubnet_b200: chunked streaming is built for fullband_baseline, fullsubnet "
                                          "and fast_fullsubnet")
            self._desc_of, self._weights_of = model._stream_desc, model._stream_weights
        self.model, self.slots, self.n_fft, self.hop, self.win_length = model, int(slots), n_fft, hop, win_length
        self.device = next(model.parameters()).device
        lib = _lib.load()
        self._state_bytes, self._workspace_bytes, self._delay, self._step = (getattr(lib, n) for n in names)
        d = self._desc_of()
        delay = self._delay(C.byref(d), n_fft, hop)
        if delay < 0:
            _lib.check(-delay)
        self.delay = int(delay)
        n = _lib.check_workspace(self._state_bytes(C.byref(d), self.slots, n_fft, hop))
        self.state = torch.zeros(n, dtype=torch.uint8, device=self.device)
        self._ws = None
        self._pos = [None] * self.slots  # each slot's clip position as far as the host knows it

    # the library's limit on a clip's position (an int32 sample count on the device)
    MAX_CLIP = 1 << 30

    def slot_state(self, b: int) -> torch.Tensor:
        """View of slot b's block of the state, to checkpoint a stream (copy it out) or restore one (copy it back, or
        into another slot).  The host then no longer knows slot b's position, so ``step`` skips its clip-length checks
        for that slot until it starts a new clip; ``copy_slot`` keeps them."""
        n = self.state.numel() // self.slots
        self._pos[b] = None
        return self.state[b * n:(b + 1) * n]

    def copy_slot(self, src: int, dst: int) -> None:
        """Move the stream of slot ``src`` to slot ``dst`` (a device copy of its block); ``src`` keeps its copy."""
        n = self.state.numel() // self.slots
        self.state[dst * n:(dst + 1) * n].copy_(self.state[src * n:(src + 1) * n])
        self._pos[dst] = self._pos[src]

    def _workspace(self, d, K: int) -> torch.Tensor:
        """One workspace, sized for the largest K so far: a workspace for K_max serves every K <= K_max."""
        n = _lib.check_workspace(self._workspace_bytes(C.byref(d), self.slots, K, self.n_fft, self.hop))
        if self._ws is None or self._ws.numel() < n:
            self._ws = None
            self._ws = torch.empty(n, dtype=torch.uint8, device=self.device)
        return self._ws

    def _check_lengths(self, K: int, st, tl):
        """Positions the host can follow: a clip must end after more than n_fft/2 samples, and stay within MAX_CLIP
        (the call itself cannot check either).  Returns the positions after the call."""
        Kh, pos = K * self.hop, list(self._pos)
        for b in range(self.slots):
            if st is not None and st[b]:
                pos[b] = 0
            if pos[b] is None:
                continue
            t = -1 if tl is None else int(tl[b])
            if t >= 0:
                assert pos[b] + t > self.n_fft // 2, (
                    f"slot {b}: a clip of {pos[b] + t} samples; streaming needs more than n_fft/2 = {self.n_fft // 2}")
                pos[b] = None
            else:
                pos[b] += Kh
                assert pos[b] <= self.MAX_CLIP, f"slot {b}: a clip longer than {self.MAX_CLIP} samples"
        return pos

    def _table(self, v, fill: int) -> Optional[np.ndarray]:
        if v is None:
            return None
        t = np.ascontiguousarray([fill if x is None else int(x) for x in v], dtype=np.int32)
        if t.shape != (self.slots,):
            raise ValueError(f"{t.size} entries for {self.slots} slots")
        return t

    @torch.no_grad()
    def step(self, chunk: torch.Tensor, start=None, tail=None) -> torch.Tensor:
        assert chunk.dim() == 2 and chunk.shape[0] == self.slots, f"chunk must be [{self.slots}, K*hop]"
        assert chunk.shape[1] % self.hop == 0, f"a chunk is a whole number of hops ({self.hop} samples)"
        K = chunk.shape[1] // self.hop
        x = _lib.require_cuda(chunk, "chunk")
        d, weights = self._desc_of(), self._weights_of()
        ws = self._workspace(d, K)
        st, tl = self._table(start, 0), self._table(tail, -1)
        pos = self._check_lengths(K, st, tl)
        out = torch.empty(self.slots, K * self.hop + self.delay, dtype=torch.float32, device=self.device)
        _lib.check(self._step(
            C.byref(d), *weights, x.data_ptr(),
            None if st is None else st.ctypes.data_as(C.c_void_p), None if tl is None else tl.ctypes.data_as(C.c_void_p),
            self.slots, K, self.n_fft, self.hop, self.win_length, out.data_ptr(), self.state.data_ptr(),
            self.state.numel(), ws.data_ptr(), ws.numel(), _lib.stream_ptr(self.device)))
        self._pos = pos
        return out

    def enhance_stream(self, chunks: Iterable[torch.Tensor], slot: int = 0) -> Iterator[torch.Tensor]:
        """One clip through slot ``slot`` while the other slots idle: 1-D chunks, each a whole number of hops but the
        last -> the enhanced clip in pieces whose concatenation is the whole-clip ``enhance`` output."""
        it = iter(chunks)
        cur = next(it, None)
        pos, emitted = 0, 0
        while cur is not None:
            nxt = next(it, None)
            n = cur.numel()
            assert nxt is None or n % self.hop == 0, "only the last chunk may end inside a hop"
            K = max(1, -(-n // self.hop))
            buf = torch.zeros(self.slots, K * self.hop, dtype=torch.float32, device=self.device)
            buf[slot, :n] = cur.to(self.device, torch.float32)
            start, tail = [0] * self.slots, [-1] * self.slots
            start[slot] = int(pos == 0)
            if nxt is None:
                tail[slot] = n
            out = self.step(buf, start, tail)[slot]
            row0 = pos - self.delay  # clip sample of out[0]
            end = pos + n if nxt is None else row0 + K * self.hop
            if end > emitted:
                yield out[emitted - row0:end - row0]
                emitted = end
            pos += K * self.hop
            cur = nxt
