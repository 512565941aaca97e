"""CPU tests of the tensor-core Q-network's shape predicates (morl_baselines_b200/tc_mlp.py): hidden widths up to 512 and up to 256
scalarising weights per update are accepted; unequal widths, widths beyond 512, training widths that are not multiples of 64 and more
than 256 weights are not."""

import pytest
from torch import nn

from morl_baselines_b200 import ops
from morl_baselines_b200.tc_mlp import TCPairMlp

F16, BF16 = ops.FMT_F16X2, ops.FMT_BF16X3


def _net(hidden, inp=35, out=24):
    layers, d = [], inp
    for h in hidden:
        layers += [nn.Linear(d, h), nn.ReLU()]
        d = h
    layers.append(nn.Linear(d, out))
    return nn.Sequential(*layers)


@pytest.mark.parametrize("fmt", [F16, BF16])
@pytest.mark.parametrize("hidden", [(512,) * 2, (512,) * 4, (320,) * 3, (448,) * 2, (256,) * 4])
@pytest.mark.parametrize("n_w", [1, 64, 65, 96, 128, 256])
def test_new_shapes_accepted(fmt, hidden, n_w):
    net = _net(hidden)
    assert TCPairMlp.supported(net, fmt)
    assert TCPairMlp.trainable_supported(net, n_w, fmt)


@pytest.mark.parametrize("fmt", [F16, BF16])
def test_rejected_shapes(fmt):
    assert not TCPairMlp.trainable_supported(_net((512, 256, 512)), 64, fmt)  # unequal widths
    assert not TCPairMlp.trainable_supported(_net((256, 512)), 64, fmt)
    for hidden in ((576,) * 2, (576,) * 4, (1024,) * 2):  # wider than 512
        assert not TCPairMlp.supported(_net(hidden), fmt)
        assert not TCPairMlp.trainable_supported(_net(hidden), 64, fmt)
    assert not TCPairMlp.trainable_supported(_net((512,) * 4), 257, fmt)
    assert not TCPairMlp.trainable_supported(_net((256,) * 4), 257, fmt)
    assert not TCPairMlp.supported(_net((512,) * 2, out=288), fmt)  # the output layer stays <= 256 wide


def test_training_widths_must_be_multiples_of_64():
    for h in (96, 160, 288, 480):
        # bf16x3 runs multiples of 32 forward only; f16x2 needs multiples of 64 even forward
        assert TCPairMlp.supported(_net((h,) * 3), BF16)
        assert not TCPairMlp.trainable_supported(_net((h,) * 3), 8, BF16)
        assert not TCPairMlp.supported(_net((h,) * 3), F16)
        assert not TCPairMlp.trainable_supported(_net((h,) * 3), 8, F16)
    assert not TCPairMlp.supported(_net((500,) * 2), BF16)


def test_shapes_the_existing_suite_marks_unsupported_stay_unsupported():
    # tests/test_tc_mlp_grad_gpu.py: bf16x3 widths 96 / 160 are forward-only
    assert TCPairMlp.supported(_net((96, 96)), BF16) and not TCPairMlp.trainable_supported(_net((96, 96)), 5, BF16)
    assert TCPairMlp.supported(_net((160,) * 3), BF16) and not TCPairMlp.trainable_supported(_net((160,) * 3), 8, BF16)
    # not a Linear / ReLU stack, or a single Linear
    assert not TCPairMlp.supported(nn.Sequential(nn.Linear(35, 256), nn.Tanh(), nn.Linear(256, 24)), F16)
    assert not TCPairMlp.supported(nn.Sequential(nn.Linear(35, 24)), F16)


def test_relu_bit_mask_layout():
    assert ops.relu_bits_words(24) == 8 and ops.relu_bits_words(256) == 8
    assert ops.relu_bits_words(288) == 16 and ops.relu_bits_words(512) == 16
    # within each 256-column half: word (c & 1) * 4 + (c >> 1) of the half's chunk c; the second half after the first
    assert [ops.relu_bits_word(c) for c in range(8)] == [0, 4, 1, 5, 2, 6, 3, 7]
    assert [ops.relu_bits_word(c) for c in range(8, 16)] == [8, 12, 9, 13, 10, 14, 11, 15]
