"""Parity at the benchmark's own size (VERDICT r1, weak #3): every distinct convolution of the batch-256 ResNet-50 step
(SURVEY.md section 8d: 22 shapes + the stem) through the DEFAULT kernel selection -- tiled / im2col TMA,
stride-2 parity classes, wgrad split-K over up to 802 816 pixels -- fprop, dgrad and wgrad against torch fp32
convolutions (TF32 off) on the same bf16-rounded operands.  Tolerances as tests/test_gpu_conv.py."""
import pytest
import torch

from cta2_check import LAYERS
from test_gpu_conv import run_conv

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("layer", LAYERS, ids=[l[0].split()[0] + "_" + l[0].split()[1].replace("->", "to") + "_" +
                                               l[0].split()[2].replace("/", "s") for l in LAYERS])
def test_batch256_conv_shapes(layer):
    name, n, h, w, cin, cout, k, stride, pad, count = layer
    run_conv(n, h, w, cin, cout, k, stride, pad, seed=7, device_rng=True)
    torch.cuda.empty_cache()
