"""Every path of the inference SequenceModel (`seq_stack_forward`, DESIGN §4.7) against the reference goldens.

By default the full-band / encoder / decoder stacks take the tensor-core layers or the persistent fp32 kernel wherever
those fit, so the per-step branch, and the persistent kernel under the tensor-core precisions, would go untested.  The
golden parity tests of all four models (fullsubnet incl. cumulative norm and GRU, fast_fullsubnet, improved_fullsubnet
incl. n_fft = 960, fullband_baseline) are rerun here with the switches that force those branches, at the tolerances of
the default run.  One pytest process per switch group, all started together."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

PARITY_TESTS = ["test_small_model_matches_reference", "test_full_model_and_inferencer_match_reference",
                "test_cumulative_laplace_norm_matches_reference", "test_gru_model_matches_reference",
                "test_fast_fullsubnet_matches_reference", "test_improved_fullsubnet_matches_reference",
                "test_improved_fullsubnet_960_matches_reference", "test_fullband_baseline_matches_reference"]
N_CASES = 18  # with their parameter sets

SWITCH_GROUPS = {
    "stepwise": {"FSN_FB_STEPWISE": "1"},  # per-step kernels + fc_gemm for every stack
    "no_rec_tc": {"FSN_NO_REC_TC": "1"},   # no wgmma recurrence: persistent kernel where it fits, else per-step
}


@pytest.fixture(scope="module")
def switch_runs():
    procs = {g: subprocess.Popen([sys.executable, "-m", "pytest", os.path.join(ROOT, "tests", "test_gpu_parity.py"), "-m",
                                  "gpu", "-q", "-k", " or ".join(PARITY_TESTS)],
                                 env=dict(os.environ, **env), stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True,
                                 cwd=ROOT)
             for g, env in SWITCH_GROUPS.items()}
    yield procs
    for p in procs.values():
        if p.poll() is None:
            p.kill()
            p.wait()


@pytest.mark.parametrize("group", list(SWITCH_GROUPS))
def test_golden_parity_under_path_switches(switch_runs, group):
    stdout, stderr = switch_runs[group].communicate(timeout=1200)
    assert switch_runs[group].returncode == 0, stdout[-3000:] + stderr[-1000:]
    assert f"{N_CASES} passed" in stdout and "failed" not in stdout, stdout[-1000:]
