"""Inputs shared by tests/golden/make_golden_envelope_update.py (run against the unmodified reference in the build container) and
tests/test_envelope_update_golden_gpu.py (run on the GPU): everything derives from numpy PCG64 / MT19937 streams, which are
bit-reproducible across machines, so the fixture stores the reference's initial parameters and outputs only."""

from __future__ import annotations

import numpy as np
import torch as th

from morl_baselines_b200.testing import synthetic_store

CASES = {
    # BASELINE.json metric shape
    "north_star": dict(obs=32, A=8, D=3, W=64, B=1024, N=16384, net=[256, 256, 256, 256], seed=7, np_seed=100, steps=2, global_step0=1, kwargs={}),
    # BASELINE.json configs[1]: minecart-v0 dims (obs 7, 6 actions, 3 objectives), |W| = 32, batch 256
    "config2": dict(obs=7, A=6, D=3, W=32, B=256, N=8192, net=[256, 256, 256, 256], seed=11, np_seed=200, steps=3, global_step0=1, kwargs={}),
    # homotopy schedule live (lambda changes every update, envelope.py:309-313, 351-358); 2 x 256 net
    "homotopy": dict(obs=7, A=6, D=3, W=32, B=256, N=4096, net=[256, 256], seed=13, np_seed=300, steps=3, global_step0=3,
                     kwargs=dict(initial_homotopy_lambda=0.2, final_homotopy_lambda=1.0, homotopy_decay_steps=10, learning_starts=0)),
}


def fill_agent(agent, c):
    """Load the synthetic transitions into ``agent.replay_buffer`` (reference or engine class) with NON-uniform priorities, so the
    sum-tree walk matters."""
    store = synthetic_store(c["N"], c["obs"], c["A"], c["D"], seed=c["seed"])
    rb = agent.replay_buffer
    n = c["N"]
    rb.obs[:n], rb.next_obs[:n], rb.actions[:n], rb.rewards[:n], rb.dones[:n] = (store[k] for k in ("obs", "next_obs", "actions", "rewards", "dones"))
    rb.size, rb.ptr = n, 0
    if hasattr(rb, "mark_all_dirty"):
        rb.mark_all_dirty()
    prio = np.random.default_rng(c["seed"] + 1).random(n) * 0.5 + 0.01
    rb.tree.batch_set(np.arange(n), prio)
    return store


def perturbed_target(init_sd):
    """target = online + 0.01 N(0,1) (numpy stream, float32): online and target nets differ from the first update on."""
    rng = np.random.default_rng(12345)
    return {k: v + th.from_numpy((0.01 * rng.standard_normal(tuple(v.shape))).astype(np.float32)) for k, v in init_sd.items()}
