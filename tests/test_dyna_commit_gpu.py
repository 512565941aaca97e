"""morl_dyna_commit_f32 (csrc/dyna.cu, ``ops.dyna_commit``) against the numpy oracle (tests/dyna_commit_oracle.py) and against the composition it
replaces (``ModelEnv.step_device`` -> boolean masks -> ``ReplayBuffer.add_batch``).

The sample and uncertainty must be bit-identical to morl_ensemble_sample_f32 on the same inputs (one shared per-row function); the oracle's
rule, gate and row-by-row ring append are applied to that sample, so every stored byte, count and alive row must match exactly."""

import numpy as np
import pytest
import torch as th

pytestmark = pytest.mark.gpu

RULES = (0, 1, 2, 3, 4)  # NONE, HOPPER, HUMANOID, MOUNTAINCAR, LUNARLANDER


def _inputs(rng, E, N, rew, S, A, noise, special=None):
    O = rew + S
    out = (rng.standard_normal((E, N, 2 * O)) * 0.05).astype(np.float32)
    out[..., O:] = (rng.standard_normal((E, N, O)) * 3 - 6).astype(np.float32)
    obs = (rng.standard_normal((N, S)) * 0.5).astype(np.float32)
    # state columns around every rule's thresholds, so that each rule has both outcomes
    obs[:, 0] = rng.uniform(-1.3, 2.3, N)
    if S > 1:
        obs[:, 1] = rng.uniform(-0.5, 0.5, N)
    if S > 7:
        obs[:, 6:8] = rng.uniform(0.85, 1.05, (N, 2))
    if rew > 0 and not noise:
        out[:, rng.random(N) < 0.3, 0] = 0.0  # r[0] == 0 exactly on some rows (LUNARLANDER's landed test)
    if special == "nonfinite" and S > 2:
        bad = rng.random(N) < 0.2
        obs[bad, 2] = np.where(rng.random(bad.sum()) < 0.5, np.inf, np.nan)   # s' non-finite, uncertainty finite: kept and terminal
        out[:, rng.random(N) < 0.05, rew + 1] = np.nan                         # NaN in the model output: uncertainty NaN, never kept
    if special == "all_done":
        obs[:, 0:2] = 5.0  # HUMANOID (s'[0] >= 2) and HOPPER (|s'[1]| >= 0.2): every row terminal
    act = rng.uniform(-1, 1, (N, A)).astype(np.float32)
    hi, lo = rng.uniform(-1, 0.5, O).astype(np.float32), rng.uniform(-7, -3, O).astype(np.float32)
    idx = rng.integers(0, E, N).astype(np.int32)
    nz = rng.standard_normal((E, N, O)).astype(np.float32) if noise else None
    return out, hi, lo, idx, nz, obs, act


def _run(dev, rng, E, N, rew, S, A, rule, noise, thr_mode, cap, ptr, special=None):
    from morl_baselines_b200 import ops
    from tests import dyna_commit_oracle as do

    out, hi, lo, idx, nz, obs, act = _inputs(rng, E, N, rew, S, A, noise, special)
    T = lambda a: None if a is None else th.from_numpy(a).to(dev)  # noqa: E731
    s, _, u = ops.ensemble_sample(T(out), T(hi), T(lo), T(idx), T(nz), T(obs), rew)
    s_np, u_np = s.cpu().numpy(), u.cpu().numpy()
    fin = u_np[np.isfinite(u_np)]
    thr = {"none": -1.0, "all": 1e30, "some": float(np.median(fin)) if len(fin) else 0.0}[thr_mode]
    init = [rng.standard_normal((cap, c)).astype(np.float32) for c in (S, S, A, rew, 1)]
    stores_np = [a.copy() for a in init]
    stores = tuple(T(a) for a in init)
    size0 = cap // 2
    next_alive = th.full((N, S), -7.0, device=dev)
    unc, counts = th.empty(N, device=dev), th.empty(2, dtype=th.int32, device=dev)
    ops.dyna_commit(T(out), T(hi), T(lo), T(idx), T(nz), T(obs), T(act), rew, rule, thr, stores, ptr, next_alive, unc, counts)
    p1, z1, alive_rows, _, done, keep = do.commit_rows(s_np, u_np, obs, act, rew, rule, thr, stores_np, ptr, size0)
    kept, alive = counts.cpu().tolist()
    assert kept == int(keep.sum()) and alive == int((~done).sum())
    assert (ptr + kept) % cap == p1 and min(size0 + kept, cap) == z1
    assert np.array_equal(unc.cpu().numpy().view(np.uint32), u_np.view(np.uint32))  # bit-identical to morl_ensemble_sample_f32
    for got, want in zip(stores, stores_np):
        assert np.array_equal(got.cpu().numpy().view(np.uint32), want.view(np.uint32))
    na = next_alive.cpu().numpy()
    assert np.array_equal(na[:alive].view(np.uint32), alive_rows.view(np.uint32))
    assert (na[alive:] == -7.0).all()
    return kept, alive, done


@pytest.mark.parametrize("E", [1, 5, 7])
@pytest.mark.parametrize("N", [1, 31, 32, 1000, 10007])
def test_commit_matches_oracle(cuda, N, E):
    rng = np.random.default_rng(N * 10 + E)
    S, rew, A = 11, 3, 3
    outcomes = set()
    for rule in RULES:
        for noise in (False, True):
            for thr_mode in ("none", "all", "some"):
                # rings: ptr at the last slot of a ring smaller than the step (kept > capacity wraps more than once), or a roomy ring
                cap, ptr = ((max(1, N // 3), max(1, N // 3) - 1) if (rule + (thr_mode == "all")) % 2 else (2 * N + 5, int(rng.integers(0, 2 * N + 5))))
                kept, alive, done = _run(cuda, rng, E, N, rew, S, A, rule, noise, thr_mode, cap, ptr)
                if thr_mode == "all":
                    assert kept == N
                if thr_mode == "none":
                    assert kept == 0
                if rule and N >= 1000:
                    outcomes.add((rule, bool(done.any()), bool((~done).any())))
    if N >= 1000:
        assert {(r, True, True) for r in RULES[1:]} <= outcomes


@pytest.mark.parametrize("rule", [1, 2])
def test_commit_every_row_terminal(cuda, rule):
    kept, alive, done = _run(cuda, np.random.default_rng(3), 5, 1000, 3, 11, 3, rule, True, "all", 4000, 17, special="all_done")
    assert alive == 0 and done.all() and kept == 1000


def test_commit_nonfinite_state_under_hopper(cuda):
    rng = np.random.default_rng(4)
    for noise in (False, True):
        for thr_mode in ("all", "some"):
            _, _, done = _run(cuda, rng, 5, 1000, 3, 11, 3, 1, noise, thr_mode, 300, 299, special="nonfinite")
            assert done.any()


def test_commit_other_shapes(cuda):
    """O wider than a warp, no reward columns, one state column, a single-column action."""
    rng = np.random.default_rng(5)
    for (rew, S, A, rule) in ((2, 45, 6, 4), (0, 5, 1, 1), (1, 1, 2, 2), (4, 8, 17, 3), (3, 40, 3, 0)):
        for N in (33, 777):
            _run(cuda, rng, 5, N, rew, S, A, rule, True, "some", 100, 99)
            _run(cuda, rng, 3, N, rew, S, A, rule, False, "all", 2 * N, 5)


class _StubModel:
    """Stands in for the ensemble inside ModelEnv: sample_device runs the existing sampling kernel on a fixed raw output."""

    def __init__(self, out, hi, lo, idx, noise):
        self.out, self.hi, self.lo, self.idx, self.noise, self.device = out, hi, lo, idx, noise, out.device

    def sample_device(self, inputs, deterministic=False, obs=None, rew_dim=0):
        from morl_baselines_b200 import ops

        return ops.ensemble_sample(self.out, self.hi, self.lo, self.idx, None if deterministic else self.noise, obs, rew_dim)


def test_commit_equals_step_device_masks_add_batch(cuda):
    from morl_baselines_b200 import ops
    from morl_baselines_b200.common.buffer import ReplayBuffer
    from morl_baselines_b200.common.model_based.utils import ModelEnv

    rng = np.random.default_rng(6)
    E, N, rew, S, A, cap = 5, 3000, 3, 11, 3, 2000
    for env_id, rule in (("mo-hopper-v4", 1), ("mo-mountaincar-v0", 3), ("mo-lunar-lander-continuous-v2", 4), ("mo-humanoid-v4", 2)):
        out, hi, lo, idx, nz, obs, act = (th.from_numpy(a).to(cuda) for a in _inputs(rng, E, N, rew, S, A, True))
        u = ops.ensemble_sample(out, hi, lo, idx, nz, obs, rew)[2]
        thr = float(u.median())
        a, b = (ReplayBuffer((S,), A, rew_dim=rew, max_size=cap, device=cuda) for _ in range(2))
        a.ptr = b.ptr = 1500
        a.size = b.size = 1700
        # the composition: ModelEnv.step_device, boolean masks, add_batch
        env = ModelEnv(_StubModel(out, hi, lo, idx, nz), env_id, rew_dim=rew)
        nobs, r, d, info = env.step_device(obs, act)
        keep = info["uncertainty"] < thr
        a.add_batch(obs[keep], act[keep], r[keep], nobs[keep], d[keep].float())
        alive_ref = nobs[~d.squeeze(-1)]
        # the fused step
        na, unc, counts = th.empty(N, S, device=cuda), th.empty(N, device=cuda), th.empty(2, dtype=th.int32, device=cuda)
        ops.dyna_commit(out, hi, lo, idx, nz, obs, act, rew, rule, thr, b._dev, b.ptr, na, unc, counts)
        kept, alive = counts.cpu().tolist()
        b.ptr, b.size = (b.ptr + kept) % cap, min(b.size + kept, cap)
        assert (a.ptr, a.size) == (b.ptr, b.size) and alive == alive_ref.shape[0]
        for x, y in zip(a._dev, b._dev):
            assert th.equal(x.view(th.int32), y.view(th.int32)), env_id
        assert th.equal(na[:alive].view(th.int32), alive_ref.view(th.int32))


def test_commit_graph_replay_equals_eager(cuda):
    from morl_baselines_b200 import ops

    rng = np.random.default_rng(7)
    E, N, rew, S, A, cap = 5, 5000, 3, 11, 3, 3000
    ins = [th.from_numpy(a).to(cuda) for a in _inputs(rng, E, N, rew, S, A, True)]
    thr = float(ops.ensemble_sample(*ins[:5], ins[5], rew)[2].median())

    def fresh():
        return (tuple(th.zeros(cap, c, device=cuda) for c in (S, S, A, rew, 1)), th.zeros(N, S, device=cuda), th.zeros(N, device=cuda),
                th.zeros(2, dtype=th.int32, device=cuda))

    st_e, na_e, u_e, c_e = fresh()
    ops.dyna_commit(*ins, rew, 1, thr, st_e, 2990, na_e, u_e, c_e)
    st_g, na_g, u_g, c_g = fresh()
    ws = ops.dyna_commit_workspace(N, cuda)
    side = th.cuda.Stream()
    side.wait_stream(th.cuda.current_stream())
    with th.cuda.stream(side):  # warm-up outside the capture
        ops.dyna_commit(*ins, rew, 1, thr, st_g, 2990, na_g, u_g, c_g, ws)
    th.cuda.current_stream().wait_stream(side)
    for t in list(st_g) + [na_g, u_g, c_g]:
        t.zero_()
    g = th.cuda.CUDAGraph()
    with th.cuda.graph(g):
        ops.dyna_commit(*ins, rew, 1, thr, st_g, 2990, na_g, u_g, c_g, ws)
    g.replay()
    th.cuda.synchronize()
    for x, y in zip(list(st_e) + [na_e, u_e, c_e], list(st_g) + [na_g, u_g, c_g]):
        assert th.equal(x, y) or th.equal(x.view(th.int32), y.view(th.int32))


def test_commit_refuses_bad_arguments(cuda):
    from morl_baselines_b200 import _lib, ops

    rng = np.random.default_rng(8)
    E, N, A = 3, 40, 3
    for rew, S, rule in ((3, 11, 9), (3, 1, 1), (3, 7, 4), (0, 11, 4), (3, 1, 3)):
        out, hi, lo, idx, nz, obs, act = (None if a is None else th.from_numpy(a).to(cuda) for a in _inputs(rng, E, N, rew, S, A, True))
        stores = tuple(th.zeros(10, c, device=cuda) for c in (S, S, A, rew, 1))
        with pytest.raises(_lib.MorlB200Error):
            ops.dyna_commit(out, hi, lo, idx, nz, obs, act, rew, rule, 1.0, stores, 0, th.empty(N, S, device=cuda), th.empty(N, device=cuda),
                            th.empty(2, dtype=th.int32, device=cuda))
