"""CPU tests of the shape predicate of GPI-PD's tensor-core plan (tc_mlp.TCProductMlp): QNet stacks of Linear [Dropout] [LayerNorm] ReLU with
one hidden width (a multiple of 64 for f16x2, of 32 for bf16x3, at most 256) and an output layer of at most 256 columns are accepted;
image features, unequal or wider layers, other activations and LayerNorm without affine parameters are not."""

import pytest
from torch import nn

from morl_baselines_b200 import ops
from morl_baselines_b200.multi_policy.gpi_pd.gpi_pd import QNet
from morl_baselines_b200.tc_mlp import TCPairMlp, TCProductMlp

F16, BF16 = ops.FMT_F16X2, ops.FMT_BF16X3


@pytest.mark.parametrize("fmt", [F16, BF16])
@pytest.mark.parametrize("arch", [(256,) * 4, (128,) * 3, (64,) * 2, (192,) * 3])
@pytest.mark.parametrize("drop,ln", [(0.01, True), (0.0, False), (0.5, False), (0.0, True)])
def test_accepted_stacks(fmt, arch, drop, ln):
    assert TCProductMlp.supported(QNet((8,), 6, 3, arch, drop_rate=drop, layer_norm=ln), fmt)


@pytest.mark.parametrize("width", [32, 96, 160, 224])
def test_bf16x3_only_widths(width):
    q = QNet((8,), 4, 3, (width,) * 3)
    assert TCProductMlp.supported(q, BF16)
    assert not TCProductMlp.supported(q, F16)


@pytest.mark.parametrize("fmt", [F16, BF16])
def test_rejected_stacks(fmt):
    assert not TCProductMlp.supported(QNet((1, 84, 84), 4, 3, (256, 256)), fmt)  # NatureCNN image features
    for arch in ((512, 512), (320,) * 3, (256, 128, 256), (128, 256)):  # wider than one column unit, or unequal widths
        assert not TCProductMlp.supported(QNet((8,), 4, 3, arch), fmt)
    assert not TCProductMlp.supported(QNet((8,), 18, 15, (128,) * 2), fmt)  # 270 output columns
    assert not TCProductMlp.supported(QNet((8,), 4, 3, (100,) * 2), fmt)
    q = QNet((8,), 4, 3, (128,) * 3)
    q.net[2] = nn.LayerNorm(128, elementwise_affine=False)
    assert not TCProductMlp.supported(q, fmt)
    q = QNet((8,), 4, 3, (128,) * 3)
    q.net[3] = nn.Tanh()
    assert not TCProductMlp.supported(q, fmt)
    q = QNet((8,), 4, 3, (128,) * 3, drop_rate=0.0, layer_norm=False)
    q.state_features = nn.Sequential(nn.Linear(8, 128), nn.Tanh())
    assert not TCProductMlp.supported(q, fmt)


def test_pair_plan_predicate_unchanged():
    # the Envelope plan still rejects anything but Linear / ReLU stacks
    q = QNet((8,), 4, 3, (128,) * 3)
    assert not TCPairMlp.supported(q.net, F16)
