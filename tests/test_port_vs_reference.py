"""Pin the PyTorch-CPU port of Envelope.update (oracle/envelope_update_port.py -- the CPU baseline and the whole-update
checker) against the UNMODIFIED reference: tests/golden/port_vs_reference.npz holds the reference Envelope's initial parameters, the
replay indices and weight sets of three of its ``update()`` calls and its parameters afterwards
(tests/golden/make_golden_reference_pins.py)."""

import os

import numpy as np
import pytest
import torch as th

from oracle.envelope_update_port import EnvelopeUpdatePort, synthetic_store

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "port_vs_reference.npz")


@pytest.mark.parametrize("per", [False, True])
def test_port_reproduces_reference_update(per):
    gold = np.load(GOLD, allow_pickle=False)
    OBS, A, D, N = 12, 5, 3, 512
    tag = f"per{int(per)}"
    init = {k[len(tag) + 6:]: th.from_numpy(gold[k]) for k in gold.files if k.startswith(tag + "/init/")}
    store = synthetic_store(N, OBS, A, D, seed=1)
    port = EnvelopeUpdatePort(OBS, A, D, [32, 32], seed=0, state_dict=init)
    for step in range(3):
        idx, wset = gold[f"{tag}/idx{step}"], th.from_numpy(gold[f"{tag}/wset{step}"])
        port.update(th.from_numpy(store["obs"][idx]), th.from_numpy(store["actions"][idx]), th.from_numpy(store["rewards"][idx]),
                    th.from_numpy(store["next_obs"][idx]), th.from_numpy(store["dones"][idx]), wset)
    final = port.q_net.state_dict()
    want = [k for k in gold.files if k.startswith(tag + "/final/")]  # (same order as the reference's state_dict; the port names its layers itself)
    assert len(final) == len(want)
    for (k, v), kw in zip(final.items(), want):
        # the same ops in the same order: bit-identical on the machine that froze the fixture; another CPU's GEMM may round the last bit
        # differently, which three Adam steps (lr 3e-4) can carry to ~1e-7 absolute
        np.testing.assert_allclose(v.numpy(), gold[kw], rtol=1e-6, atol=2e-7, err_msg=k)
