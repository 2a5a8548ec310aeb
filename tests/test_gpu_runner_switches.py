"""The ResNet runner under each of its documented A/B switches (README): the batch-16 64x64 layerwise training
forward, the shallow teacher-forced backward and the folded-BN eval forward of tests/test_gpu_resnet.py, with their
own tolerances.  The switches are read once per process, so each one runs those tests in a subprocess."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = [
    "tests/test_gpu_resnet.py::test_resnet50_layerwise_forward_teacher_forced[b16_64]",
    "tests/test_gpu_resnet.py::test_backward_vs_oracle_teacher_forced[shallow_b16_64]",
    "tests/test_gpu_resnet.py::test_eval_forward_folded_bn_layerwise_vs_oracle[b16_64]",
    "tests/test_gpu_resnet.py::test_eval_mode_and_no_grad_paths",
]
SWITCHES = ["DIRB200_IM2COL", "DIRB200_ATMA", "DIRB200_FUSED_STATS", "DIRB200_FUSED_BWD_MOMENTS",
            "DIRB200_FOLDED_EVAL", "DIRB200_GRAPH"]


@pytest.mark.parametrize("switch", SWITCHES, ids=[s[len("DIRB200_"):].lower() for s in SWITCHES])
def test_runner_parity_with_switch_off(switch):
    e = dict(os.environ)
    e[switch] = "0"
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider"] + TESTS, env=e, cwd=ROOT,
                       capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, f"{switch}=0\n" + r.stdout[-5000:] + r.stderr[-2000:]
    assert f"{len(TESTS)} passed" in r.stdout, r.stdout[-2000:]
