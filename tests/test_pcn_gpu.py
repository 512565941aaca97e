"""PCN / LCN on the GPU: the fused update and forward kernels against the float64 restatement (tests/pcn_f64.py) and torch autograd,
determinism and graph replays, and the learners against the reference's golden vectors (tests/golden/pcn.npz) on both the kernel path
and the eager fallback."""

import os
import tempfile

import numpy as np
import pytest
import torch as th

from morl_baselines_b200 import ops
from morl_baselines_b200.multi_policy.lcn.lcn import LCN
from morl_baselines_b200.multi_policy.pcn import pcn as pcn_mod
from morl_baselines_b200.multi_policy.pcn.pcn import PCN, ContinuousActionsDefaultModel, DiscreteActionsDefaultModel, Transition
from tests import pcn_f64
from tests.golden import make_golden_pcn as mg
from tests.pcn_standin import VarLengthEnv

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "pcn.npz"))
RTOL, ATOL = 1e-4, 2e-6  # on parameters, as the MOSAC tests


def _model(S, d, H, A, continuous, seed, dev):
    th.manual_seed(seed)
    cls = ContinuousActionsDefaultModel if continuous else DiscreteActionsDefaultModel
    scaling = np.random.default_rng(seed).uniform(0.05, 1.0, d + 1).astype(np.float32)
    return cls(S, A, d, scaling, H).to(dev)


def _kernel_case(S, d, H, A, B, continuous, seed, dev):
    rng = np.random.default_rng(seed)
    m = _model(S, d, H, A, continuous, seed, dev)
    N = max(2 * B, 50)
    ld = S + d + (A if continuous else 1)
    store = np.zeros((N, ld), np.float32)
    store[:, :S] = rng.standard_normal((N, S))
    store[:, S:S + d] = rng.standard_normal((N, d)) * 3
    if continuous:
        store[:, S + d:] = rng.uniform(-1, 1, (N, A))
    else:
        store.view(np.int32)[:, S + d] = rng.integers(0, A, N)
    rows = rng.integers(0, N, B).astype(np.int32)
    hor = rng.integers(1, 300, B).astype(np.int32)
    return m, store, rows, hor


def _run_kernel(m, store_d, rows_d, hor_d, B, continuous, out=None):
    ts = pcn_mod.default_model_tensors(m)
    grads = out if out is not None else [th.full_like(t, float("nan")) for t in ts]
    stats = th.zeros(2, device=store_d.device)
    pred = th.zeros((B, m.action_dim), device=store_d.device)
    ws = ops.pcn_workspace(m.state_dim, m.reward_dim, m.hidden_dim, m.action_dim, B, store_d.device)
    ops.pcn_update(ops.pcn_pointer_table(ts), ops.pcn_pointer_table(grads), m.scaling_factor, store_d, m.state_dim, m.reward_dim, rows_d, hor_d,
                   B, m.hidden_dim, m.action_dim, continuous, stats[0:1], None if continuous else stats[1:2], pred, ws)
    return grads, stats, pred


SHAPES = [  # (S, d, H, A, B, continuous)
    (7, 3, 64, 6, 256, False), (2, 6, 64, 2, 32, False), (11, 3, 64, 3, 256, True), (4, 2, 32, 3, 1, False), (5, 8, 128, 5, 37, True),
    (3, 4, 256, 32, 17, False), (9, 5, 256, 4, 300, True), (1, 7, 32, 1, 100, True), (256, 2, 128, 7, 40, False), (6, 8, 64, 9, 4096, False),
]


@pytest.mark.parametrize("shape", SHAPES, ids=[f"S{s}-d{d}-H{h}-A{a}-B{b}-{'c' if c else 'd'}" for s, d, h, a, b, c in SHAPES])
def test_update_kernel_matches_f64_and_autograd(shape, cuda):
    S, d, H, A, B, cont = shape
    assert ops.pcn_supported(S, d, H, A, B)
    m, store, rows, hor = _kernel_case(S, d, H, A, B, cont, 7, cuda)
    store_d, rows_d, hor_d = th.from_numpy(store).to(cuda), th.from_numpy(rows).to(cuda), th.from_numpy(hor).to(cuda)
    grads, stats, pred = _run_kernel(m, store_d, rows_d, hor_d, B, cont)
    th.cuda.synchronize()
    p = {k: v.detach().cpu().numpy() for k, v in m.state_dict().items()}
    act = store[rows, S + d:] if cont else store.view(np.int32)[rows, S + d]
    loss, ent, y, g = pcn_f64.loss_and_grads(p, m.scaling_factor.cpu().numpy(), store[rows, :S], store[rows, S:S + d], hor, act, cont)
    np.testing.assert_allclose(pred.cpu().numpy(), y, rtol=1e-4, atol=1e-5)
    assert abs(stats[0].item() - loss) <= 1e-5 * max(1.0, abs(loss))
    if not cont:
        assert abs(stats[1].item() - ent) <= 1e-5 * max(1.0, abs(ent))
    for k, gk in zip(pcn_f64.KEYS, grads):
        ref = g[k]
        np.testing.assert_allclose(gk.cpu().numpy(), ref, rtol=1e-3, atol=1e-5 * max(1e-3, np.abs(ref).max()), err_msg=k)
    # torch autograd in fp32 on the same rows
    sd = store_d[rows_d.long()]
    out = m(sd[:, :S], sd[:, S:S + d], hor_d.float().unsqueeze(1))
    if cont:
        l = th.nn.functional.mse_loss(sd[:, S + d:], out)
    else:
        l = -out.gather(1, sd[:, S + d].contiguous().view(th.int32).long().unsqueeze(1)).mean()
    tg = th.autograd.grad(l, pcn_mod.default_model_tensors(m))
    for k, a, b in zip(pcn_f64.KEYS, grads, tg):
        scale = b.abs().max().item()
        assert (a - b).abs().max().item() <= 1e-4 * max(scale, 1e-3), k


def test_update_kernel_is_deterministic_and_graph_replays_match(cuda):
    S, d, H, A, B, cont = 7, 3, 64, 6, 256, False
    m, store, rows, hor = _kernel_case(S, d, H, A, B, cont, 3, cuda)
    store_d, rows_d, hor_d = th.from_numpy(store).to(cuda), th.from_numpy(rows).to(cuda), th.from_numpy(hor).to(cuda)
    g1, s1, p1 = _run_kernel(m, store_d, rows_d, hor_d, B, cont)
    g2, s2, p2 = _run_kernel(m, store_d, rows_d, hor_d, B, cont)
    bufs = [th.zeros_like(t) for t in pcn_mod.default_model_tensors(m)]
    stats = th.zeros(2, device=cuda)
    pred = th.zeros((B, A), device=cuda)
    ws = ops.pcn_workspace(S, d, H, A, B, cuda)
    tables = (ops.pcn_pointer_table(pcn_mod.default_model_tensors(m)), ops.pcn_pointer_table(bufs))
    graph = th.cuda.CUDAGraph()
    side = th.cuda.Stream()
    side.wait_stream(th.cuda.current_stream())
    with th.cuda.stream(side), th.cuda.graph(graph):
        ops.pcn_update(*tables, m.scaling_factor, store_d, S, d, rows_d, hor_d, B, H, A, cont, stats[0:1], stats[1:2], pred, ws)
    th.cuda.current_stream().wait_stream(side)
    graph.replay()
    th.cuda.synchronize()
    for a, b, c in zip(g1, g2, bufs):
        assert th.equal(a, b) and th.equal(a, c)
    assert th.equal(s1, s2) and th.equal(s1, stats) and th.equal(p1, p2) and th.equal(p1, pred)


@pytest.mark.parametrize("shape", [(7, 3, 64, 6, False), (11, 3, 64, 3, True), (3, 8, 256, 32, False), (2, 2, 32, 1, True)])
def test_forward_kernel_rows_argmax_and_pinned(shape, cuda):
    S, d, H, A, cont = shape
    m = _model(S, d, H, A, cont, 1, cuda)
    rng = np.random.default_rng(2)
    N = 45
    obs, ret = rng.standard_normal((N, S)).astype(np.float32), (rng.standard_normal((N, d)) * 5).astype(np.float32)
    hor = rng.integers(1, 100, N).astype(np.float32)
    table = ops.pcn_pointer_table(pcn_mod.default_model_tensors(m))
    out = th.zeros((N, A), device=cuda)
    am = th.zeros(N, dtype=th.int32, device=cuda)
    ops.pcn_forward(table, m.scaling_factor, th.from_numpy(obs).to(cuda), th.from_numpy(ret).to(cuda), th.from_numpy(hor).to(cuda), H, not cont, out, am)
    th.cuda.synchronize()
    p = {k: v.detach().cpu().numpy() for k, v in m.state_dict().items()}
    y, _ = pcn_f64.forward(p, m.scaling_factor.cpu().numpy(), obs, ret, hor, cont)
    np.testing.assert_allclose(out.cpu().numpy(), y, rtol=1e-4, atol=1e-5)
    assert np.array_equal(am.cpu().numpy(), np.argmax(out.cpu().numpy(), axis=1))
    # one row through pinned host memory
    pin = [th.from_numpy(a[:1].copy()).pin_memory() for a in (obs, ret, hor)]
    out_h = th.zeros((1, A)).pin_memory()
    ops.pcn_forward(table, m.scaling_factor, *pin, H, not cont, out_h)
    th.cuda.current_stream().synchronize()
    assert th.equal(out_h, out[:1].cpu())


# ---- learners against the reference --------------------------------------------------------------------------------------------------
def _agent(name, cuda, model_class=None, use_cuda_graph=True):
    c = mg.UPDATE_CASES[name]
    env = VarLengthEnv(**c["env"], seed=c["seed"])
    agent = PCN(env, np.array(c["scaling"], np.float32), learning_rate=c["lr"], batch_size=c["batch"], hidden_dim=c["hidden"], log=False,
                seed=c["seed"], device=cuda, model_class=model_class, use_cuda_graph=use_cuda_graph)
    init = {k.split("/", 2)[2]: th.from_numpy(v) for k, v in GOLDEN.items() if k.startswith(f"update_{name}/init/")}
    agent.model.load_state_dict(init)
    mg.fill(agent, env, c["seed"], Transition)
    return agent


def _assert_params(model, prefix):
    for k, v in model.state_dict().items():
        np.testing.assert_allclose(v.cpu().numpy(), GOLDEN[f"{prefix}/{k}"], rtol=RTOL, atol=ATOL, err_msg=f"{prefix}/{k}")


class MyModel(DiscreteActionsDefaultModel):
    """A user-supplied model class (here with the default layers), which runs the eager torch path."""


class MyContinuousModel(ContinuousActionsDefaultModel):
    pass


def _user_class(name):
    return MyContinuousModel if name == "cont" else MyModel


@pytest.mark.parametrize("path", ["graph", "eager", "fallback", "out-of-range"])
@pytest.mark.parametrize("name", list(mg.UPDATE_CASES))
def test_update_block_matches_reference(name, path, cuda, monkeypatch):
    if path == "out-of-range":
        monkeypatch.setattr(pcn_mod.ops, "pcn_supported", lambda *a, **k: False)
    model_class = _user_class(name) if path.startswith("fallback") else None
    agent = _agent(name, cuda, model_class, use_cuda_graph=path != "eager")
    assert agent.fused == (path in ("graph", "eager"))
    assert [e[1] for e in agent.experience_replay] == list(GOLDEN[f"update_{name}/heap_steps"])
    loss, pred = agent.update()
    _assert_params(agent.model, f"update_{name}/after1")
    np.testing.assert_allclose(pred.cpu().numpy(), GOLDEN[f"update_{name}/pred1"], rtol=1e-4, atol=1e-5)
    assert abs(loss.item() - GOLDEN[f"update_{name}/loss"][0]) <= 1e-5 * abs(GOLDEN[f"update_{name}/loss"][0])
    v = agent._run_block(mg.N_UPDATES - 1)
    stats = v.stats.cpu().numpy()
    _assert_params(agent.model, f"update_{name}/afterU")
    np.testing.assert_allclose(stats[0], GOLDEN[f"update_{name}/loss"][1:], rtol=1e-5)
    if name == "disc":
        np.testing.assert_allclose(stats[1], GOLDEN[f"update_{name}/entropy"][1:], rtol=1e-5)


def test_graph_replay_is_bit_identical_to_eager(cuda):
    a = _agent("disc", cuda, use_cuda_graph=True)
    b = _agent("disc", cuda, use_cuda_graph=False)
    for n in (mg.N_UPDATES, 1, mg.N_UPDATES):
        va, vb = a._run_block(n), b._run_block(n)
        assert th.equal(va.stats, vb.stats)
    for (k, x), y in zip(a.model.state_dict().items(), b.model.state_dict().values()):
        assert th.equal(x, y), k


def test_act_log_probs_match_f64(cuda):
    agent = _agent("disc", cuda)
    p = {k: v.cpu().numpy() for k, v in agent.model.state_dict().items()}
    rng = np.random.default_rng(0)
    for _ in range(5):
        obs, ret, hor = rng.standard_normal(4).astype(np.float32), rng.standard_normal(2).astype(np.float32) * 4, np.float32(rng.integers(1, 20))
        lp = agent._predict_row(obs, ret, hor)
        y, _ = pcn_f64.forward(p, p["scaling_factor"], obs[None], ret[None], np.array([hor]), False)
        np.testing.assert_allclose(lp, y[0], rtol=1e-5, atol=1e-6)
        agent.set_desired_return_and_horizon(ret, hor)
        assert agent.eval(obs) == np.argmax(y[0])


def _run_train(algo, cuda, use_cuda_graph):
    c = mg.TRAIN[algo]
    env, eval_env = VarLengthEnv(**c["env"], seed=31), VarLengthEnv(**c["env"], seed=32)
    cls = PCN if algo == "pcn" else LCN
    agent = cls(env, np.array(c["scaling"], np.float32), log=False, device=cuda, use_cuda_graph=use_cuda_graph, **c["ctor"])
    agent.model.load_state_dict({k.split("/", 2)[2]: th.from_numpy(v) for k, v in GOLDEN.items() if k.startswith(f"train_{algo}/init/")})
    cmds = []
    choose = agent._choose_commands

    def recording(n):
        r, h = choose(n)
        cmds.append(np.concatenate([r, [h]]).astype(np.float32))
        return r, h

    agent._choose_commands = recording
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)
        try:
            agent.train(eval_env=eval_env, **c["train"])
            assert os.listdir(os.path.join(tmp, "weights"))
        finally:
            os.chdir(cwd)
    return agent, np.array(cmds)


@pytest.mark.parametrize("graph", [True, False])
@pytest.mark.parametrize("algo", ["pcn", "lcn"])
def test_train_matches_reference(algo, graph, cuda):
    agent, cmds = _run_train(algo, cuda, graph)
    assert agent.global_step == int(GOLDEN[f"train_{algo}/global_step"])
    np.testing.assert_allclose(cmds, GOLDEN[f"train_{algo}/commands"], rtol=1e-5, atol=1e-5)
    heap = agent.experience_replay
    assert [e[1] for e in heap] == list(GOLDEN[f"train_{algo}/heap_steps"])
    assert np.array_equal(agent._heap.episode_lengths(), GOLDEN[f"train_{algo}/heap_lengths"])
    np.testing.assert_allclose(agent._heap.episode_returns(), GOLDEN[f"train_{algo}/heap_returns"], rtol=1e-5, atol=1e-5)
    _assert_params(agent.model, f"train_{algo}/final")


def test_out_of_range_shape_selects_the_eager_path(cuda):
    env = VarLengthEnv(obs_dim=4, n_actions=3, reward_dim=2, seed=0)
    agent = PCN(env, np.ones(3, np.float32), hidden_dim=96, batch_size=16, log=False, seed=0, device=cuda)
    assert not agent.fused and not ops.pcn_supported(4, 2, 96, 3, 16)
    mg.fill(agent, env, 0, Transition)
    before = [t.clone() for t in agent.model.parameters()]
    loss, pred = agent.update()
    assert np.isfinite(loss.item()) and pred.shape == (16, 3)
    assert any(not th.equal(a, b) for a, b in zip(before, agent.model.parameters()))


def test_save_load_round_trip(cuda):
    a = _agent("disc", cuda)
    a.update()
    b = _agent("disc", cuda)
    b.update()
    assert len(b._graphs) == 1
    with tempfile.TemporaryDirectory() as tmp:
        a.save(save_dir=tmp)
        b.load(os.path.join(tmp, "PCN_model.pt"))
    assert len(b._graphs) == 0 and b.fused
    for (k, x), y in zip(a.model.state_dict().items(), b.model.state_dict().values()):
        assert th.equal(x, y), k
    b.update()
    b.model.load_state_dict(a.model.state_dict())
    assert len(b._graphs) == 0
    obs, ret = np.zeros(4, np.float32), np.ones(2, np.float32)
    assert np.array_equal(a._predict_row(obs, ret, 3.0), a._predict_row(obs, ret, 3.0))
