"""The argument contract of the ops bindings: every tensor a binding hands to libmorl_b200.so is checked before anything is launched.

One small valid call per binding, and for each of its tensor arguments the mutations the contract must refuse: a CPU tensor, the wrong
dtype, the wrong shape, a non-contiguous output, a workspace one element short, a two-element device scalar.  Each refusal is a
MorlB200Error naming the argument, launches nothing (ops.launch_count unchanged) and leaves the sentinel-filled outputs untouched.  A
coverage case keeps the table in step with the entry points ops.py launches."""

import os
import re

import numpy as np
import pytest
import torch as th

from morl_baselines_b200 import _lib, ops

pytestmark = pytest.mark.gpu

DEV = th.device("cuda:0")
F16 = ops.FMT_F16X2
ROWS = {}  # binding -> (entry points, make)


def row(*entries):
    def deco(make):
        ROWS[make.__name__] = (entries, make)
        return make

    return deco


def rn(*shape, scale=1.0):
    return th.randn(*shape, device=DEV) * scale


def sentinel(*shape, dtype=th.float32, pinned=False):
    t = th.full(shape, -7, dtype=dtype) if pinned else th.full(shape, -7, dtype=dtype, device=DEV)
    return t.pin_memory() if pinned else t


def ws_bytes(nbytes):
    return th.zeros(int(nbytes), dtype=th.uint8, device=DEV)


def planes(rows, ld, scale=None):
    return ops.split_planes(rn(rows, ld).relu_(), F16, rows_pad=rows, ldp=ld, scale=scale)


# Each make() returns (call, kwargs, kinds): kinds maps an argument (every tensor under it, for lists) to what the contract checks:
# "in" input, "out" output, "ws" workspace, "scalar" device scalar, "planes"/"planes_out" plane tensors; a "+free" suffix marks an input
# whose extent is free (it sets a size), so a shorter one is a valid call; "@name": the binding's own name for the argument.
@row("morl_envelope_td_f32")
def envelope_td():
    B, W, A, D = 4, 8, 3, 2
    kw = dict(q_online=rn(B, W, A, D), q_target=rn(B, W, A, D), wset=th.rand(W, D, device=DEV), reward=rn(B, D), done=th.zeros(B, device=DEV),
              gamma=0.9, out=sentinel(W * B, D), pref_out=sentinel(W * B, dtype=th.int32), act_out=sentinel(W * B, dtype=th.int32))
    return ops.envelope_td, kw, dict(q_online="in", q_target="in", wset="in", reward="in", done="in", out="out", pref_out="out", act_out="out")


@row("morl_greedy_td_f32")
def greedy_td():
    N, A, D = 24, 4, 3
    kw = dict(q_select=rn(N, A, D), q_eval=rn(N, A, D), w=th.rand(8, D, device=DEV), reward=rn(3, D), done=th.zeros(3, device=DEV), gamma=0.9)
    return ops.greedy_td, kw, dict(q_select="in", q_eval="in", w="in", reward="in", done="in")


@row("morl_critic_min_td_f32")
def critic_min_td():
    kw = dict(q_nets=rn(2, 24, 4, 3), w=th.rand(24, 3, device=DEV), reward=rn(24, 3), done=th.zeros(24, device=DEV), gamma=0.9)
    return ops.critic_min_td, kw, dict(q_nets="in", w="in", reward="in", done="in")


@row("morl_gpi_envelope_f32")
def gpi_envelope():
    kw = dict(q_nets=rn(2, 24, 5, 4, 3), w=th.rand(24, 3, device=DEV))
    return ops.gpi_envelope, kw, dict(q_nets="in", w="in")


@row("morl_actor_critic_td_f32")
def actor_critic_td():
    kw = dict(q_nets=rn(2, 24, 3), w=th.rand(3, device=DEV), reward=rn(24, 3), done=th.zeros(24, 1, device=DEV), logp=rn(24, 1), alpha=0.2, gamma=0.9,
              variant=ops.AC_SCALAR_MIN)
    return ops.actor_critic_td, kw, dict(q_nets="in", w="in", reward="in", done="in", logp="in")


@row("morl_discrete_sac_target_f32")
def discrete_sac_target():
    kw = dict(q_nets=rn(2, 40, 6, 3), logits=rn(40, 6), w=th.rand(3, device=DEV), reward=rn(40, 3), done=th.zeros(40, device=DEV),
              alpha=th.full((1,), 0.2, device=DEV), gamma=0.9, out=sentinel(40))
    return ops.discrete_sac_target, kw, dict(q_nets="in", logits="in", w="in", reward="in", done="in", alpha="scalar", out="out")


@row("morl_discrete_sac_actor_loss_f32")
def discrete_sac_actor_loss():
    lib = _lib.load()
    kw = dict(logits=rn(40, 6), q_nets=rn(2, 40, 6, 3), w=th.rand(3, device=DEV), alpha=th.full((1,), 0.2, device=DEV),
              log_alpha=th.full((1,), -0.5, device=DEV), target_entropy=0.9, workspace=ws_bytes(lib.morl_discrete_sac_workspace_bytes(40)))
    return ops.discrete_sac_actor_loss, kw, dict(logits="in", q_nets="in", w="in", alpha="scalar", log_alpha="scalar", workspace="ws")


@row("morl_vector_gae_f32")
def vector_gae():
    T, E, D = 6, 5, 3
    kw = dict(rewards=rn(T, E, D), values=rn(T, E, D), dones=th.zeros(T, E, device=DEV), next_value=rn(E, D), next_done=th.ones(E, device=DEV),
              weights=th.rand(D, device=DEV), gamma=0.99, gae_lambda=0.95, returns_out=sentinel(T, E, D), adv_out=sentinel(T, E))
    kinds = dict(rewards="in", values="in", dones="in", next_value="in", next_done="in", weights="in", returns_out="out", adv_out="out")
    return ops.vector_gae, kw, kinds


@row("morl_ppo_loss_f32")
def ppo_loss():
    M, A, D = 20, 3, 2
    kw = dict(mean=rn(M, A), logstd=rn(A, scale=0.3), value=rn(M, D), actions=rn(M, A), old_logprob=rn(M), advantages=rn(M), returns=rn(M, D),
              old_values=rn(M, D), clip_coef=0.2, ent_coef=0.01, vf_coef=0.5, norm_adv=True, clip_vloss=True, stats=sentinel(6),
              out=(sentinel(1), sentinel(M, A), sentinel(A), sentinel(M, D)))
    kinds = dict(mean="in", logstd="in", value="in", actions="in", old_logprob="in", advantages="in", returns="in", old_values="in", stats="out",
                 out="out")
    return ops.ppo_loss, kw, kinds


@row("morl_td_mse_priority_f32")
def td_mse_priority():
    B, W, A, D = 6, 4, 4, 3
    kw = dict(q_values=rn(B * W, A, D), action=th.randint(0, A, (B,), device=DEV, dtype=th.int32), target_q=rn(B * W, D), wset=th.rand(W, D, device=DEV),
              homotopy_lambda=0.0, B=B, W=W, workspace=ws_bytes(_lib.load().morl_td_workspace_bytes(B * W)), loss_out=sentinel(1),
              grad_out=sentinel(B * W, A, D), prio_out=sentinel(B), q_taken_out=sentinel(B * W, D), lambda_dev=th.full((1,), 0.3, device=DEV))
    kinds = dict(q_values="in", action="in", target_q="in", wset="in", workspace="ws", loss_out="out", grad_out="out", prio_out="out",
                 q_taken_out="out", lambda_dev="scalar")
    return ops.td_mse_priority, kw, kinds


@row("morl_td_huber_priority_f32")
def td_huber_priority():
    kw = dict(q_values=rn(2, 24, 4, 3, scale=0.02), action=th.randint(0, 4, (12,), device=DEV, dtype=th.int32), target_q=rn(24, 3), target_q_gpi=rn(24, 3),
              w=th.rand(24, 3, device=DEV), min_priority=0.01, p_rows=12, workspace=ws_bytes(_lib.load().morl_td_workspace_bytes(24)))
    return ops.td_huber_priority, kw, dict(q_values="in", action="in+free", target_q="in", target_q_gpi="in", w="in", workspace="ws")


@row("morl_replay_gather")
def replay_gather():
    N, B = 50, 8
    kw = dict(obs_store=rn(N, 7), next_obs_store=rn(N, 7), act_store=th.randint(0, 4, (N, 1), device=DEV, dtype=th.uint8), rew_store=rn(N, 3),
              done_store=th.zeros(N, 1, device=DEV), idx=th.randint(0, N, (B,), device=DEV),
              outs=(sentinel(B, 7), sentinel(B, 1, dtype=th.int32), sentinel(B, 3), sentinel(B, 7), sentinel(B, 1)))
    kinds = dict(obs_store="in", next_obs_store="in", act_store="in", rew_store="in", done_store="in", idx="in+free", outs="out")
    return ops.replay_gather, kw, kinds


def _pareto(dtype):
    kw = dict(points=th.randn(60, 3, device=DEV, dtype=dtype), remove_duplicates=True, raw=True, out=sentinel(60, dtype=th.uint8))
    return ops.pareto_mask, kw, dict(points="in", out="out")


@row("morl_pareto_mask_f32")
def pareto_mask_f32():
    return _pareto(th.float32)


@row("morl_pareto_mask_f64")
def pareto_mask_f64():
    return _pareto(th.float64)


@row("morl_front_pack_f64")
def front_pack():
    pts = th.randn(40, 3, device=DEV, dtype=th.float64)
    kw = dict(points=pts, keep=ops.pareto_mask(pts, True, raw=True), cap=16, rec=sentinel(1 + 16 * 3 + 2, dtype=th.float64),
              extras=th.ones(2, dtype=th.float64, device=DEV))
    return ops.front_pack, kw, dict(points="in", keep="in", rec="out", extras="in+free")


@row("morl_front_unpack_f64")
def front_unpack():
    world, d, cap, n_extra = 2, 3, 16, 2
    gathered = th.full((world, 1 + cap * d + n_extra), -1.0, dtype=th.float64, device=DEV)
    gathered[:, 0] = 3.0
    kw = dict(gathered=gathered, world=world, d=d, cap=cap, n_extra=n_extra, pts_out=sentinel(world * cap, d, dtype=th.float64),
              meta_out=sentinel(world, 1 + n_extra, dtype=th.float64))
    return ops.front_unpack, kw, dict(gathered="in", pts_out="out", meta_out="out")


@row("morl_hypervolume_f64")
def hypervolume():
    pts = th.rand(30, 3, device=DEV, dtype=th.float64)
    kw = dict(points=pts, ref_point=th.zeros(3, dtype=th.float64, device=DEV), keep=ops.pareto_mask(pts, True, raw=True),
              out=sentinel(1, dtype=th.float64))
    return ops.hypervolume, kw, dict(points="in", keep="in", out="out")  # ref_point: any array, converted (documented)


@row("morl_corner_weights_f64")
def corner_weights():
    return ops.corner_weights, dict(V=th.randint(0, 3, (6, 3), device=DEV).double(), cap=64), dict(V="in")


@row("morl_polyak_f32")
def polyak():
    kw = dict(params=[rn(16, 5), rn(16)], targets=[rn(16, 5), rn(16)])
    return (lambda params, targets: ops.PolyakPlan(params, targets).run(0.5)), kw, dict(params="in+free", targets="in")


@row("morl_amax_scale_f32")
def amax_scale():
    kw = dict(x=rn(500, scale=1e-3), target_exp=9, scale_out=sentinel(1), workspace=th.zeros(2, device=DEV, dtype=th.int32))
    return ops.amax_scale, kw, dict(x="in+free", scale_out="scalar", workspace="ws")


@row("morl_split_planes")
def split_planes():
    kw = dict(x=rn(50, 13), fmt=F16, ldp=64, out=ops.empty_planes(F16, 50, 64, DEV).fill_(-7), scale=ops.scale_tensor(2.0, DEV))
    return ops.split_planes, kw, dict(x="in", out="planes_out", scale="scalar")


@row("morl_split_planes_multi")
def split_planes_multi():
    s = ops.scale_tensor(1.0, DEV)
    jobs = [(rn(64, 64, scale=0.1), ops.empty_planes(F16, 64, 64, DEV).fill_(-7), False, s, 14),
            (rn(24, 64), ops.empty_planes(F16, 32, 64, DEV).fill_(-7), False, ops.scale_tensor(1.0, DEV), None)]
    kinds = {(0, 0): "in", (0, 1): "planes_out", (0, 3): "scalar", (1, 0): "in", (1, 1): "planes_out", (1, 3): "scalar"}
    return ops.split_planes_multi, dict(jobs=jobs, fmt=F16), dict(jobs=kinds)


def _gemm_operands(M=256, K=128, N=64):
    sa, sw = ops.scale_tensor(8.0, DEV), ops.scale_tensor(512.0, DEV)
    return planes(M, K, sa), ops.split_planes(rn(N, K, scale=1 / 8), F16, scale=sw), sa, sw


@row("morl_gemm_planes_f32")
def gemm_planes():
    ap, bp, sa, sw = _gemm_operands()
    kw = dict(a_planes=ap, b_planes=bp, n_out=64, bias=rn(64), relu=True, out_f32=True, out_planes=True,
              c_f32=sentinel(256, 64), c_planes=ops.empty_planes(F16, 256, 64, DEV).fill_(-7), a_scale=sa, b_scale=sw, c_scale=sa,
              relu_bits_in=th.full((256, 8), -1, dtype=th.int32, device=DEV), relu_bits_out=sentinel(256, 8, dtype=th.int32))
    kinds = dict(a_planes="planes", b_planes="planes", bias="in", c_f32="out", c_planes="planes_out", a_scale="scalar",
                 b_scale="scalar", c_scale="scalar", relu_bits_in="in", relu_bits_out="out")
    return ops.gemm_planes, kw, kinds


@row("morl_gemm_planes_ln_f32")
def gemm_planes_ln():
    ap, bp, sa, sw = _gemm_operands()
    kw = dict(a_planes=ap, b_planes=bp, n_out=64, bias=rn(64), ln_weight=rn(64), ln_bias=rn(64), ln_eps=1e-5, drop_p=0.1,
              drop_seed=th.tensor([7], dtype=th.int64, device=DEV), drop_offset=th.zeros(1, dtype=th.int32, device=DEV), out_f32=True,
              c_f32=sentinel(256, 64), c_planes=ops.empty_planes(F16, 256, 64, DEV).fill_(-7), a_scale=sa, b_scale=sw, c_scale=sa,
              drop_bits_out=sentinel(256, 8, dtype=th.int32))
    kinds = dict(a_planes="planes", b_planes="planes", bias="in", ln_weight="in", ln_bias="in", drop_seed="scalar", drop_offset="scalar", c_f32="out",
                 c_planes="planes_out", a_scale="scalar", b_scale="scalar", c_scale="scalar", drop_bits_out="out")
    return ops.gemm_planes_ln, kw, kinds


@row("morl_philox_advance")
def philox_advance():
    return ops.philox_advance, dict(offset=th.zeros(1, dtype=th.int32, device=DEV)), dict(offset="scalar")


def _ensemble(E=3, N=20, O=9):
    return dict(out=rn(E, N, 2 * O), max_logvar=th.zeros(O, device=DEV), min_logvar=th.full((O,), -5.0, device=DEV),
                model_idx=th.randint(0, E, (N,), device=DEV, dtype=th.int32), noise=rn(E, N, O))


_ENSEMBLE_KINDS = dict(out="in", max_logvar="in", min_logvar="in", model_idx="in", noise="in")


@row("morl_ensemble_sample_f32")
def ensemble_sample():
    return ops.ensemble_sample, dict(_ensemble(), obs=rn(20, 6), rew_dim=3), dict(_ENSEMBLE_KINDS, obs="in")


@row("morl_dyna_commit_f32")
def dyna_commit():
    N, S, A, cap = 20, 6, 2, 16
    kw = dict(_ensemble(), obs=rn(N, S), act=rn(N, A), rew_dim=3, rule=ops.TERM_NONE, max_uncertainty=1e30,
              stores=tuple(sentinel(cap, c) for c in (S, S, A, 3, 1)), ptr=3, next_alive=sentinel(N, S), uncertainty_out=sentinel(N),
              counts_out=sentinel(2, dtype=th.int32), workspace=ws_bytes(_lib.load().morl_dyna_commit_workspace_bytes(N)))
    kinds = dict(_ENSEMBLE_KINDS, obs="in", act="in", stores="out", next_alive="out", uncertainty_out="out", counts_out="out", workspace="ws")
    return ops.dyna_commit, kw, kinds


@row("morl_qhead_envelope_td_f32")
def qhead_envelope_td():
    B, W, A, D, K = 8, 32, 6, 3, 128
    M, N = B * W, A * D
    s_a, s_w = ops.scale_tensor(2.0, DEV), ops.scale_tensor(1024.0, DEV)
    p = [ops.split_planes(rn(N, K, scale=0.1), F16, rows_pad=32, ldp=K, scale=s_w) for _ in range(2)]
    kw = dict(a_on=planes(M, K, s_a), a_tg=planes(M, K, s_a), w_on=p[0], w_tg=p[1], bias_on=rn(N), bias_tg=rn(N), wset=th.rand(W, D, device=DEV),
              reward=rn(B, D), done=th.zeros(B, device=DEV), gamma=0.99, B=B, W=W, A=A, D=D, a_scale_on=s_a, a_scale_tg=s_a, w_scale_on=s_w,
              w_scale_tg=s_w, want_indices=True, out=sentinel(W * B, D), pref_out=sentinel(W * B, dtype=th.int32), act_out=sentinel(W * B, dtype=th.int32),
              q_on_out=sentinel(M, N), q_tg_out=sentinel(M, N))
    kinds = dict(a_on="planes", a_tg="planes", w_on="planes", w_tg="planes", bias_on="in", bias_tg="in", wset="in", reward="in", done="in",
                 a_scale_on="scalar", a_scale_tg="scalar", w_scale_on="scalar", w_scale_tg="scalar", out="out", pref_out="out", act_out="out",
                 q_on_out="out", q_tg_out="out")
    return ops.qhead_envelope_td, kw, kinds


def _chain_layers(M, n_layers=2):
    sw = ops.scale_tensor(1024.0, DEV)
    return dict(weights=[[ops.split_planes(rn(256, 256, scale=0.06), F16, rows_pad=256, ldp=256, scale=sw) for _ in range(n_layers)]],
                biases=[[rn(256, scale=0.1) for _ in range(n_layers)]], w_scales=[[sw] * n_layers],
                bits=[[sentinel(M, 8, dtype=th.int32) for _ in range(n_layers)]])


_CHAIN_KINDS = dict(weights="planes", biases="in", w_scales="scalar", bits="out")


@row("morl_gemm_chain_f32")
def gemm_chain():
    M = 512
    sa = ops.scale_tensor(2.0, DEV)
    kw = dict(_chain_layers(M), acts=[[planes(M, 256, sa)] + [ops.empty_planes(F16, M, 256, DEV).fill_(-7) for _ in range(2)]], act_scale=sa,
              bits_in=[[th.full((M, 8), -1, dtype=th.int32, device=DEV) for _ in range(2)]])
    call = lambda **k: ops.GemmChain(**k)()  # noqa: E731  (the checks run at construction, the launch at the call)
    return call, kw, dict(_CHAIN_KINDS, acts="planes", act_scale="scalar", bits_in="in")


@row("morl_gemm_chain_pairs_f32")
def gemm_chain_pairs():
    B, W = 64, 8
    M = B * W
    kw = dict(_chain_layers(M), outs=[[ops.empty_planes(F16, M, 256, DEV).fill_(-7) for _ in range(2)]], B=B, W=W,
              act_scale=ops.scale_tensor(2.0, DEV), us=[rn(B, 256)], vs=[rn(W, 256)])
    call = lambda us, vs, **k: ops.GemmChainPairs(**k)(us, vs)  # noqa: E731
    return call, kw, dict(_CHAIN_KINDS, outs="planes_out", act_scale="scalar", us="in", vs="in")


@row("morl_qhead_gemm_f32")
def qhead_gemm():
    sa, sw = ops.scale_tensor(2.0, DEV), ops.scale_tensor(1024.0, DEV)
    kw = dict(a_planes=planes(256, 128, sa), w_planes=ops.split_planes(rn(24, 128, scale=0.1), F16, rows_pad=32, ldp=128, scale=sw), n_out=24,
              bias=rn(24), out=sentinel(256, 24), a_scale=sa, w_scale=sw)
    return ops.qhead_gemm, kw, dict(a_planes="planes", w_planes="planes", bias="in", out="out", a_scale="scalar", w_scale="scalar")


@row("morl_pairs_relu_split_planes")
def pairs_relu_split():
    kw = dict(u=rn(6, 64), v=rn(5, 64), out=ops.empty_planes(F16, 30, 64, DEV).fill_(-7), scale=ops.scale_tensor(2.0, DEV),
              relu_bits_out=sentinel(30, 8, dtype=th.int32))
    return ops.pairs_relu_split, kw, dict(u="in", v="in", out="planes_out", scale="scalar", relu_bits_out="out")


@row("morl_pairs_product_split_planes")
def pairs_product_split():
    kw = dict(u=rn(6, 64), v=rn(5, 64), out=ops.empty_planes(F16, 30, 64, DEV).fill_(-7), scale=ops.scale_tensor(2.0, DEV))
    return ops.pairs_product_split, kw, dict(u="in", v="in", out="planes_out", scale="scalar")


@row("morl_product_layer1_uv_f32")
def product_layer1_uv():
    kw = dict(s=rn(7, 11), s_weight=rn(64, 11), s_bias=rn(64), m=rn(5, 3), w_weight=rn(64, 3), w_bias=rn(64), u=sentinel(7, 64), v=sentinel(5, 64))
    return ops.product_layer1_uv, kw, dict(s="in", s_weight="in", s_bias="in", m="in", w_weight="in", w_bias="in", u="out", v="out")


@row("morl_pair_layer1_uv_f32")
def pair_layer1_uv():
    kw = dict(feats=rn(7, 11), wset=th.rand(5, 2, device=DEV), weight=rn(64, 13), bias=rn(64), u=sentinel(7, 64), v=sentinel(5, 64))
    return ops.pair_layer1_uv, kw, dict(feats="in", wset="in", weight="in", bias="in", u="out", v="out")


@row("morl_pair_layer1_grad_f32")
def pair_layer1_grad():
    kw = dict(dU=rn(7, 64), dV=rn(5, 64), feats=rn(7, 11), wset=th.rand(5, 2, device=DEV), dW1=sentinel(64, 13), db1=sentinel(64),
              workspace=ws_bytes(_lib.load().morl_pair_layer1_grad_workspace_bytes(11, 2, 64)))
    return ops.pair_layer1_grad, kw, dict(dU="in", dV="in", feats="in", wset="in", dW1="out", db1="out", workspace="ws")


@row("morl_gemm_planes_mn_f32")
def gemm_planes_mn():
    sg, sa = ops.scale_tensor(2.0 ** 16, DEV), ops.scale_tensor(8.0, DEV)
    kw = dict(g_planes=ops.split_planes(rn(300, 24, scale=1e-3), F16, ldp=64, scale=sg), g_cols=24, h_planes=planes(300, 128, sa), h_cols=128,
              out=sentinel(24, 128), workspace=ws_bytes(ops.gemm_mn_workspace_bytes(300, 24, 128)), colsum=sentinel(24), g_scale=sg, h_scale=sa)
    kinds = dict(g_planes="planes", h_planes="planes", out="out", workspace="ws", colsum="out", g_scale="scalar", h_scale="scalar")
    return ops.gemm_planes_mn, kw, kinds


@row("morl_pairs_grad_reduce_planes")
def pairs_grad_reduce():
    B, W, H = 6, 70, 64  # the two-pass form
    kw = dict(planes=planes(B * W, H), B=B, W=W, workspace=ws_bytes(_lib.load().morl_pairs_grad_reduce_workspace_bytes(B, W, H)), dU=sentinel(B, H),
              dV=sentinel(W, H), scale=ops.scale_tensor(2.0, DEV))
    return ops.pairs_grad_reduce, kw, dict(planes="planes", workspace="ws", dU="out", dV="out", scale="scalar")


def _pcn(S=7, d=3, H=64, A=6):
    from morl_baselines_b200.multi_policy.pcn import pcn as pcn_mod

    m = pcn_mod.DiscreteActionsDefaultModel(S, A, d, np.ones(d + 1, np.float32), H).to(DEV)
    return m, pcn_mod.default_model_tensors(m)


@row("morl_pcn_update_f32")
def pcn_update():
    S, d, H, A, B, N = 7, 3, 64, 6, 12, 40
    m, ts = _pcn(S, d, H, A)
    store = rn(N, S + d + 1)
    store[:, S + d] = th.randint(0, A, (N,), device=DEV).int().view(th.float32)
    kw = dict(params=ts, grads=[th.empty_like(t) for t in ts], scaling=m.scaling_factor.detach(), store=store, obs_dim=S, d=d,
              rows=th.randint(0, N, (B,), device=DEV).int(), horizons=th.randint(1, 50, (B,), device=DEV).int(), batch=B, hidden=H, n_out=A,
              continuous=False, loss_out=sentinel(1), entropy_out=sentinel(1), pred_out=sentinel(B, A),
              workspace=ws_bytes(_lib.load().morl_pcn_workspace_bytes(S, d, H, A, B)))
    kinds = dict(params="in+free@tensors", grads="in+free@tensors", scaling="in", store="in", rows="in", horizons="in", loss_out="out", entropy_out="out",
                 pred_out="out", workspace="ws")

    def call(params, grads, **k):
        return ops.pcn_update(ops.pcn_pointer_table(params), ops.pcn_pointer_table(grads), **k)

    return call, kw, kinds


@row("morl_pcn_forward_f32")
def pcn_forward():
    m, ts = _pcn()
    kw = dict(params=ts, scaling=m.scaling_factor.detach(), obs=th.ones(1, 7).pin_memory(), ret=th.ones(1, 3).pin_memory(), hor=th.ones(1).pin_memory(),
              hidden=64, log_softmax=True, out=sentinel(1, 6, pinned=True), argmax_out=sentinel(1, dtype=th.int32, pinned=True))
    kinds = dict(params="in+free@tensors", scaling="in", obs="in", ret="in", hor="in", out="out", argmax_out="out")
    return (lambda params, **k: ops.pcn_forward(ops.pcn_pointer_table(params), **k)), kw, kinds


def _eupg(S=3, d=2, arch=(50,), A=4):
    from morl_baselines_b200.single_policy.esr.eupg import PolicyNet, policy_tensors

    return policy_tensors(PolicyNet((S,), A, d, list(arch)).to(DEV))


@row("morl_eupg_returns_f32")
def eupg_returns():
    block = rn(9, 6)
    return ops.eupg_returns, dict(rewards=block[:, 4:], gamma=0.99, out=sentinel(9, 2)), dict(rewards="in", out="out")


@row("morl_eupg_update_f32")
def eupg_update():
    S, d, A, T = 3, 2, 4, 9
    ts = _eupg(S, d, (50,), A)
    block = rn(T, S + 2 * d + 1)
    block[:, :S] = th.randint(-3, 4, (T, S), device=DEV).int().view(th.float32)
    block[:, S + d] = th.randint(0, A, (T,), device=DEV).int().view(th.float32)
    kw = dict(params=ts, grads=[th.empty_like(t) for t in ts], obs=block[:, :S].view(th.int32), acc=block[:, S:S + d],
              actions=block[:, S + d].view(th.int32), v=rn(T), loss_out=sentinel(1),
              workspace=ws_bytes(ops.eupg_workspace_bytes(S, d, [50], A)))
    kinds = dict(params="in+free", grads="in+free", obs="in", acc="in", actions="in", v="in", loss_out="out", workspace="ws")

    def call(params, grads, **k):
        return ops.eupg_update(ops.EupgNet(S, d, [50], A, params, grads), **k)

    return call, kw, kinds


@row("morl_eupg_probs_f32")
def eupg_probs():
    ts = _eupg()
    kw = dict(params=ts, x=th.ones(1, 5).pin_memory(), out=sentinel(1, 4, pinned=True))
    return (lambda params, **k: ops.eupg_probs(ops.EupgNet(3, 2, [50], 4, params), **k)), kw, dict(params="in+free", x="in", out="out")


# ------------------------------------------------------------------------------------------------ mutations
def _leaves(value, path=()):
    if isinstance(value, th.Tensor):
        yield path, value
    elif isinstance(value, (list, tuple)):
        for i, v in enumerate(value):
            yield from _leaves(v, path + (i,))


def _replace(value, path, new):
    if not path:
        return new
    items = list(value)
    items[path[0]] = _replace(items[path[0]], path[1:], new)
    return type(value)(items)


def _kind(kinds, key, sub):
    k = kinds.get(key)
    return k.get(sub) if isinstance(k, dict) else k


def _non_contiguous(t):
    """Same shape and dtype, every other element along the last dimension of size > 1 (refused by every output layout rule)."""
    dims = [i for i, n in enumerate(t.shape) if n > 1]
    if not dims:
        return None
    shape = list(t.shape)
    shape[dims[-1]] *= 2
    buf = sentinel(*shape, dtype=t.dtype, pinned=not t.is_cuda)
    return buf[(slice(None),) * dims[-1] + (slice(None, None, 2),)]


def _mutations(kind, t):
    base, _, flag = kind.partition("+")
    yield "cpu", th.zeros_like(t, device="cpu")
    if base == "ws":
        yield "short", t.reshape(-1)[:-1]
        return
    yield "dtype", t.to(th.int16)  # no argument of any binding takes int16
    if base == "scalar":
        yield "two-element", th.cat([t.reshape(-1), t.reshape(-1)])
        return
    if flag != "free":
        yield "shape", t.reshape(-1)[:-1]
    if base in ("out", "planes_out"):
        v = _non_contiguous(t)
        if v is not None:
            yield "non-contiguous", v


def _expected_name(kind, key, sub):
    """The argument a refusal names: the keyword, or the binding's own name for it (``kind@name``), with the list indices."""
    return (kind.partition("@")[2] or key) + "".join(f"[{i}]" for i in sub)


@pytest.mark.parametrize("binding", list(ROWS))
def test_binding_refuses_bad_arguments_before_launch(cuda, binding):
    th.manual_seed(0)
    call, kw, kinds = ROWS[binding][1]()
    outputs = [t for key, v in kw.items() for sub, t in _leaves(v) if (_kind(kinds, key, sub) or "").startswith(("out", "planes_out"))]
    for key, value in kw.items():
        for sub, t in _leaves(value):
            kind = _kind(kinds, key, sub)
            if kind is None:
                continue
            name = _expected_name(kind, key, sub)
            for what, bad in _mutations(kind.partition("@")[0], t):
                th.cuda.synchronize()
                before, launches = [o.clone() for o in outputs], ops.launch_count
                with pytest.raises(_lib.MorlB200Error) as err:
                    call(**dict(kw, **{key: _replace(value, sub, bad)}))
                assert f": {name} " in str(err.value), (binding, name, what, str(err.value))
                assert ops.launch_count == launches, (binding, name, what)
                th.cuda.synchronize()
                assert all(th.equal(o, b) for o, b in zip(outputs, before)), (binding, name, what, "an output was written")
                if what == "non-contiguous":
                    assert bool((bad == -7).all()), (binding, name, "the refused output was written")
    launches = ops.launch_count
    call(**kw)
    th.cuda.synchronize()
    assert ops.launch_count > launches


def test_every_launched_entry_point_has_a_row():
    src = open(os.path.join(os.path.dirname(ops.__file__), "ops.py")).read()
    launched = set()
    for m in re.finditer(r"_launch\(([^,]+),", src):
        launched |= set(re.findall(r'"(morl_\w+)"', m.group(1)))
    covered = {e for entries, _ in ROWS.values() for e in entries}
    assert launched and launched == covered, (launched - covered, covered - launched)
