"""The non-default GEMM feeding paths of the conv kernel -- the cp.async gather for the 3x3 / strided convs
(DIRB200_IM2COL=0) and for every conv (DIRB200_ATMA=0) -- against torch on the shapes of tests/cta2_check.py (the
defaults, tiled / im2col TMA, are what test_gpu_conv*.py exercise).
The switches are read once per process, so each variant runs tests/cta2_check.py in a subprocess."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("env", [{"DIRB200_IM2COL": "0"}, {"DIRB200_ATMA": "0"}],
                         ids=["gather_for_3x3", "cp_async_gather_only"])
def test_conv_variant_parity(env):
    e = dict(os.environ)
    e.update(env)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "cta2_check.py"), "parity"], env=e,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "15/15 ok" in r.stdout
