"""The non-default GEMM feeding paths of the conv kernel -- the cp.async gather for the 3x3 / strided convs
(DIRB200_IM2COL=0) and for every conv (DIRB200_ATMA=0) -- against float64 on the shapes of tests/cta2_check.py,
including the BN-statistics and folded-BN epilogues (the defaults, tiled / im2col TMA, are what test_gpu_conv*.py
exercise).
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
    import cta2_check
    import test_gpu_conv_epilogues as E
    total = len(cta2_check.PARITY) + 2 * len(E.SHAPES)
    assert f"{total}/{total} ok" in r.stdout
