"""fsn_debug_sb_lstm_tc_max_clusters (the resident-cluster query of the sub-band kernel, used by tools/tc_sweep.py)
validates its launch configuration before any CUDA call, like the kernel's own hook."""
import ctypes as C


def test_max_clusters_argument_checks_need_no_gpu():
    from fullsubnet_b200 import _lib
    lib = _lib.load()
    n = C.c_int(-7)
    for H, x3, stages, cluster in ((384, 1, 4, 3), (384, 1, 4, 8), (384, 1, 4, 0), (384, 0, 1, 2), (384, 0, 5, 2),
                                   (384, 1, 0, 2), (192, 1, 4, 2), (512, 0, 4, 2), (64, 0, 4, 1)):
        assert lib.fsn_debug_sb_lstm_tc_max_clusters(H, x3, stages, cluster, C.byref(n)) == _lib.FSN_ERR_UNSUPPORTED
        assert lib.fsn_last_error_code() == _lib.FSN_ERR_UNSUPPORTED
    assert lib.fsn_debug_sb_lstm_tc_max_clusters(384, 1, 4, 2, None) == _lib.FSN_ERR_SHAPE
    assert n.value == -7  # untouched on error
