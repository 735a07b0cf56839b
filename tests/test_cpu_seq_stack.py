"""CPU-only checks of the inference SequenceModel's unit-test hook (fsn_debug_seq_stack, fsn_fullband.cu): the workspace
query needs no GPU and grows with the stack, and every bad argument is rejected with its error class before any CUDA
call (stand-in device pointers, never dereferenced)."""
import ctypes as C

import pytest


@pytest.fixture(scope="module")
def lib():
    from fullsubnet_b200 import _lib
    return _lib.load()


def _H(*h):
    return (C.c_int * len(h))(*h)


def test_seq_stack_workspace_query_needs_no_gpu(lib):
    from fullsubnet_b200 import _lib

    def q(n=2, H=64, R=5, Tp=7, K0=33, gru=0, step_scale=0, tc=0, x3=0, O=20):
        return lib.fsn_debug_seq_stack_workspace_bytes(n, _H(*([H] * n)), R, Tp, K0, gru, step_scale, tc, x3, O)

    base = q()
    assert base > 0
    assert q(n=1) < base < q(n=3)  # layer 1's state and the persistent kernel's scratch; the second layer-output buffer
    assert q(R=6) > base and q(Tp=8) > base and q(H=96) > base
    assert q(tc=1) > base and q(tc=1, x3=1) > q(tc=1)  # tensor-core operands ([hi | lo | hi] with x3) and projection
    assert q(step_scale=1) < base and q(gru=1) < base  # neither takes the persistent kernel: no scratch for it
    uneven = lib.fsn_debug_seq_stack_workspace_bytes(2, _H(96, 64), 5, 7, 33, 0, 0, 0, 0, 20)
    assert q() < uneven < q(H=96)  # sized per layer, not for the widest one everywhere
    for kw, code in (({"n": 0}, _lib.FSN_ERR_UNSUPPORTED), ({"n": 9}, _lib.FSN_ERR_UNSUPPORTED),
                     ({"H": 0}, _lib.FSN_ERR_SHAPE), ({"R": 0}, _lib.FSN_ERR_SHAPE), ({"Tp": 0}, _lib.FSN_ERR_SHAPE),
                     ({"K0": 0}, _lib.FSN_ERR_SHAPE), ({"O": 0}, _lib.FSN_ERR_SHAPE),
                     ({"R": 1 << 16, "Tp": 1 << 12}, _lib.FSN_ERR_SHAPE),  # 2^31 floats in one buffer
                     ({"gru": 1, "tc": 1}, _lib.FSN_ERR_UNSUPPORTED)):
        assert q(**kw) == 0, kw
        assert lib.fsn_last_error_code() == code, (kw, lib.fsn_last_error())
    assert lib.fsn_debug_seq_stack_workspace_bytes(2, None, 5, 7, 33, 0, 0, 0, 0, 20) == 0
    assert lib.fsn_last_error_code() == _lib.FSN_ERR_SHAPE


def test_seq_stack_hook_checks_arguments_without_gpu(lib):
    from fullsubnet_b200 import _lib
    n, R, Tp, K0, O = 2, 4, 5, 8, 6
    p = 1 << 20
    need = lib.fsn_debug_seq_stack_workspace_bytes(n, _H(32, 32), R, Tp, K0, 0, 0, 0, 0, O)
    assert need > 0

    def layers(k=n):
        return (_lib.LstmLayer * k)(*[_lib.LstmLayer(p, p, p, p) for _ in range(k)])

    path = C.c_int(-1)

    def call(n=n, H=(32, 32), R=R, gru=0, tc=0, x3=0, x=p, scale=p, fc_w=p, fc_b=p, O=O, act=1, out=p, L=None, ws=p,
             nbytes=need, Hptr=True):
        Hs = _H(*H) if Hptr else None
        return lib.fsn_debug_seq_stack(L if L is not None else layers(max(n, 1)), n, Hs, R, Tp, K0, gru, 0, tc, x3, 0, x, scale,
                                       fc_w, fc_b, O, act, out, ws, nbytes, C.byref(path), None)

    def err(code, text=None, **kw):
        assert call(**kw) == code, (kw, lib.fsn_last_error())
        if text is not None:
            assert text in lib.fsn_last_error(), (kw, lib.fsn_last_error())

    err(_lib.FSN_ERR_UNSUPPORTED, n=0, H=(32,))
    err(_lib.FSN_ERR_UNSUPPORTED, b"1..8 layers", n=9, H=(32,) * 9)
    err(_lib.FSN_ERR_SHAPE, Hptr=False)
    err(_lib.FSN_ERR_SHAPE, b"layer 1", H=(32, 0))
    err(_lib.FSN_ERR_SHAPE, H=(-4, 32))
    err(_lib.FSN_ERR_SHAPE, R=0)
    err(_lib.FSN_ERR_SHAPE, O=0)
    err(_lib.FSN_ERR_SHAPE, b"activation", act=4)
    err(_lib.FSN_ERR_UNSUPPORTED, b"GRU", gru=1, tc=1, H=(64, 64))
    err(_lib.FSN_ERR_UNSUPPORTED, b"tensor cores", tc=1)  # H = 32 < 64: never on the wgmma recurrence
    err(_lib.FSN_ERR_UNSUPPORTED, b"tensor cores", tc=1, x3=1)
    for name in ("x", "fc_w", "fc_b", "out"):
        err(_lib.FSN_ERR_SHAPE, b"null argument", **{name: None})
    bad = layers()
    bad[1].b_hh = None
    err(_lib.FSN_ERR_SHAPE, b"layer 1", L=bad)
    bad = layers()
    bad[0].w_ih = None
    err(_lib.FSN_ERR_SHAPE, b"layer 0", L=bad)
    err(_lib.FSN_ERR_WORKSPACE, nbytes=need - 1)
    err(_lib.FSN_ERR_WORKSPACE, ws=None)
    err(_lib.FSN_ERR_WORKSPACE, H=(32, 48))  # a wider layer needs more than the query of (32, 32)
    assert path.value == -1  # no failed call reports a path
    # the scale is nullable (no norm): the call then fails only at the workspace
    assert call(scale=None, nbytes=need - 1) == _lib.FSN_ERR_WORKSPACE
