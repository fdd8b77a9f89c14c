"""The integer (XOR + POPC) form of the matcher under the matcher and pose suites.  PLSTVO_K1=popc is documented as giving the
same results as the tensor-core form, and it is the only form that leaves several partials per row and column, i.e. the only
one that reaches the general merge loop of match_finalize_block (shared by the finalize kernel, K2 and the streamed solver's
prepare step).  The switch is read once per process, hence the subprocess; test_selected_matcher_form, which must pass in it,
proves the integer form was in use.  PLSTVO_K1_VARIANT=452 adds the 4-queries-per-thread kernel and its coarser plan."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.gpu
@pytest.mark.parametrize("variant", [None, "452"], ids=["default", "qpt4"])
def test_integer_matcher_passes_match_and_pose_suites(variant):
    env = dict(os.environ, PLSTVO_K1="popc")
    env.pop("PLSTVO_K1_VARIANT", None)
    if variant:
        env["PLSTVO_K1_VARIANT"] = variant
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-rA", "-m", "gpu", "-p", "no:cacheprovider",
                        "tests/test_gpu_match.py", "tests/test_gpu_pose.py"],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=1500)
    tail = (r.stdout + r.stderr)[-6000:]
    assert r.returncode == 0, tail
    assert "PASSED tests/test_gpu_match.py::test_selected_matcher_form" in r.stdout, tail
