"""``ops.attention_qkv`` refuses a softmax scale that is not finite and > 0 on the CPU path too, as the kernels'
binding does on the GPU: scale 0 would turn every output into NaN and a negative scale picks the wrong row max."""
import math

import pytest
import torch

from distributed_training_guide_b200 import ops


def test_attention_qkv_refuses_bad_scale_on_cpu():
    qkv = torch.randn(1, 16, 4, 8)
    for bad in (0.0, -0.0, -0.5, float("nan"), float("inf"), -float("inf"), True):
        with pytest.raises(ValueError, match="scale"):
            ops.attention_qkv(qkv, 2, 1, scale=bad)
    for good in (None, 1.0 / math.sqrt(8), 0.05, 1.0):
        assert torch.isfinite(ops.attention_qkv(qkv, 2, 1, scale=good)).all()
