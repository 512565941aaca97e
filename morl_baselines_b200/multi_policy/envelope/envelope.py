"""Envelope Q-Learning on the CUDA update engine (drop-in for reference
morl_baselines/multi_policy/envelope/envelope.py: same constructor, attributes, ``update / eval / act / max_action /
envelope_target / ddqn_target / train / save / load / get_config``).

What changes under the API (SURVEY.md section 8, rows a1-a6, a14-a17, a20):
  * the envelope target is evaluated on the B*|W| DISTINCT (s'_b, w_j) rows, not on the reference's B*|W|^2 tiled rows
    (envelope.py:284-291, 416-418) -- bit-identical result, |W| times fewer MLP rows;
  * the first dense layer is applied separably, h1[b, j] = relu(W1_s s_b + (W1_w w_j + b1)), so the [s || w] concat
    (envelope.py:75) is never materialised;
  * einsum -> max -> argmax -> gather x2 -> Bellman (envelope.py:422-440, 298) is ONE kernel (morl_envelope_td_f32);
    gather -> MSE -> homotopy loss -> d loss/d q -> PER priorities (envelope.py:301-313, 329-331) is ONE kernel
    (morl_td_mse_priority_f32); the minibatch gather reads a replay store resident in HBM (morl_replay_gather);
    the target sync is one multi-tensor launch (morl_polyak_f32);
  * the dense layers (forward on the three passes, hand-written backward) run on the tensor cores (wgmma) with fp32-accurate split
    operands (tc_mlp.py, csrc/gemm_bf16x3.cu); the update does not go through autograd: the loss kernel emits d loss / d Q, the
    backward GEMMs write straight into persistent ``.grad`` buffers, clip + Adam is one fused multi-tensor step;
  * the whole gradient update is captured in a CUDA graph and replayed (no host sync inside, no library kernel in the graph); the
    homotopy lambda is read from device memory, so the graph stays valid while the schedule decays it.
``use_tensor_cores=False`` is an explicit validation path (torch autograd + cuBLAS FP32 dense layers around the same fused operators);
network shapes the tensor-core path does not cover raise instead of silently taking it.  Everything requires a CUDA device.
"""

from __future__ import annotations

import os
from typing import List, Optional, Union

import numpy as np
import torch as th
import torch.nn as nn
import torch.optim as optim

from ... import ops
from ...tc_mlp import TCPairMlp, TCPairMlpFn
from ...common.buffer import ReplayBuffer
from ...common.fused_adam import FusedClipAdam
from ...common.morl_algorithm import MOAgent, MOPolicy
from ...common.networks import NatureCNN, get_grad_norm, layer_init, mlp, polyak_update
from ...common.prioritized_buffer import PrioritizedReplayBuffer
from ...common.utils import linearly_decaying_value
from ...common.weights import equally_spaced_weights, random_weights

# output layers + envelope operator + Bellman line as one kernel (csrc/qhead_envelope.cu; bit-identical to the
# three-launch chain, tests/test_qhead_envelope_gpu.py); MORL_FUSED_HEAD=0 keeps the three-launch chain (A/B runs)
_FUSED_HEAD = os.environ.get("MORL_FUSED_HEAD", "1") != "0"
_PRE_REFRESH = os.environ.get("MORL_PRE_REFRESH", "1") == "1"  # weight-plane refresh on a side branch, under the tree walk + gather (+1.4 %)
_HEAD_REVERSE = os.environ.get("MORL_HEAD_REVERSE", "1") == "1"  # the fused head walks the tiles from the last one after a chained pass (L2; +1.2 %)
# device PER: fork the priority / sum-tree branch after the backward GEMMs instead of right after the loss (MORL_DEFER_TREE=0: the earlier order)
_DEFER_TREE = os.environ.get("MORL_DEFER_TREE", "1") != "0"
# the online-net and target-net no-grad chains as two branches of the captured graph: one chain's kernels fill the launch gaps and tile
# tails of the other's (+2 % on the update; MORL_TWO_STREAMS=0: one stream; needs the fused head)
_TWO_STREAMS = os.environ.get("MORL_TWO_STREAMS", "1") == "1"
# ... and the training pass's forward as a third branch (+1 %; MORL_THREE_STREAMS=0 disables it)
_THREE_STREAMS = os.environ.get("MORL_THREE_STREAMS", "1") == "1"


class QNet(nn.Module):
    """Weight-conditioned vector Q-network; parameter names equal the reference's (envelope.py:33-77)."""

    def __init__(self, obs_shape, action_dim, rew_dim, net_arch):
        super().__init__()
        self.obs_shape = obs_shape
        self.action_dim = action_dim
        self.rew_dim = rew_dim
        if len(obs_shape) == 1:
            self.feature_extractor = None
            self.feat_dim = obs_shape[0]
        else:
            self.feature_extractor = NatureCNN(self.obs_shape, features_dim=512)
            self.feat_dim = self.feature_extractor.features_dim
        self.net = mlp(self.feat_dim + rew_dim, action_dim * rew_dim, net_arch)
        self.apply(layer_init)

    def forward(self, obs, w):
        """Q(s, w) for paired rows, the reference's calling convention: [N, A, D]."""
        feats = self.feature_extractor(obs) if self.feature_extractor is not None else obs
        if w.dim() == 1 and feats.dim() > 1:
            w = w.unsqueeze(0)
        x = th.cat((feats, w), dim=w.dim() - 1)
        return self.net(x).view(-1, self.action_dim, self.rew_dim)

    def forward_pairs(self, obs, wset):
        """Q(s_b, w_j) for every pair: obs [B, ...], wset [W, D] -> [B, W, A, D] (row b*W + j of the flattened batch).
        The first Linear is split column-wise: W1 [s || w] + b1 = W1_s s + (W1_w w + b1)."""
        feats = self.feature_extractor(obs) if self.feature_extractor is not None else obs
        first = self.net[0]
        B, W = feats.shape[0], wset.shape[0]
        u = feats @ first.weight[:, : self.feat_dim].t()  # [B, H]
        v = th.addmm(first.bias, wset, first.weight[:, self.feat_dim :].t())  # [W, H]
        h = (u.unsqueeze(1) + v.unsqueeze(0)).view(B * W, -1)
        h = self.net[1:](h)
        return h.view(B, W, self.action_dim, self.rew_dim)


class _FusedTDLoss(th.autograd.Function):
    """critic loss of envelope.py:301-313 as one kernel; backward hands the precomputed d loss / d q_values upstream."""

    @staticmethod
    def forward(ctx, q_values, action, target_q, wset, lam_dev, B, W, workspace, prio_out, loss_out):
        loss, grad, _ = ops.td_mse_priority(q_values.detach(), action, target_q, wset, 0.0, B, W, ops.ROWS_BMAJOR, want_grad=True,
                                            want_prio=prio_out is not None, workspace=workspace, prio_out=prio_out, loss_out=loss_out,
                                            lambda_dev=lam_dev)
        ctx.save_for_backward(grad)
        return loss.squeeze(0).clone()

    @staticmethod
    def backward(ctx, grad_out):
        (grad,) = ctx.saved_tensors
        return grad * grad_out, None, None, None, None, None, None, None, None, None


class Envelope(MOPolicy, MOAgent):
    """Envelope Q-Learning (R. Yang, X. Sun, K. Narasimhan, NeurIPS 2019) -- see the module docstring."""

    def __init__(
        self,
        env,
        learning_rate: float = 3e-4,
        initial_epsilon: float = 0.01,
        final_epsilon: float = 0.01,
        epsilon_decay_steps: int = None,
        tau: float = 1.0,
        target_net_update_freq: int = 200,
        buffer_size: int = int(1e6),
        net_arch: List = [256, 256, 256, 256],
        batch_size: int = 256,
        learning_starts: int = 100,
        gradient_updates: int = 1,
        gamma: float = 0.99,
        max_grad_norm: Optional[float] = 1.0,
        envelope: bool = True,
        num_sample_w: int = 4,
        per: bool = True,
        per_alpha: float = 0.6,
        initial_homotopy_lambda: float = 0.0,
        final_homotopy_lambda: float = 1.0,
        homotopy_decay_steps: int = None,
        project_name: str = "MORL-Baselines",
        experiment_name: str = "Envelope",
        wandb_entity: Optional[str] = None,
        log: bool = True,
        seed: Optional[int] = None,
        device: Union[th.device, str] = "auto",
        group: Optional[str] = None,
        use_cuda_graph: bool = True,
        replay_on_device: bool = True,
        use_tensor_cores: bool = True,
        tensor_core_format: Optional[str] = None,
        per_on_device: bool = True,
        tensor_core_accumulators: str = "single",
        dp_group=None,
    ):
        MOAgent.__init__(self, env, device=device, seed=seed)
        MOPolicy.__init__(self, device=device)
        if self.device.type != "cuda":
            raise ops._lib.MorlB200Error("morl_baselines_b200.Envelope needs a CUDA device: the update path is CUDA-only (no CPU fallback)")
        ops._lib.load()
        # DP-Envelope (SURVEY 8(e)): ``dp_group`` (True = the default process group, or a torch.distributed group) shards the scalarising
        # weight set of every update over the ranks -- each rank evaluates the targets of ALL weights (the envelope maximum needs Q for every
        # preference row; recomputed, no communication), back-propagates the loss rows of ITS num_sample_w / world weights, and ONE
        # all-reduce per update (parallel.DPFlat: gradients + the owner's priorities + loss) keeps the conditioned network identical on all
        # ranks.  Every rank must be constructed and seeded identically and see the same transitions.
        self._dp = None
        if dp_group is not None and dp_group is not False:
            import torch.distributed as dist

            grp = None if dp_group is True else dp_group
            world = dist.get_world_size(grp) if dist.is_initialized() else 1
            if world > 1:
                if num_sample_w % world != 0:
                    raise ValueError(f"dp_group: num_sample_w ({num_sample_w}) must be a multiple of the group size ({world})")
                self._dp = {"group": grp, "world": world, "rank": dist.get_rank(grp), "w_loc": num_sample_w // world, "flat": None}
        self.learning_rate = learning_rate
        self.initial_epsilon = initial_epsilon
        self.epsilon = initial_epsilon
        self.epsilon_decay_steps = epsilon_decay_steps
        self.final_epsilon = final_epsilon
        self.tau = tau
        self.target_net_update_freq = target_net_update_freq
        self.gamma = gamma
        self.max_grad_norm = max_grad_norm
        self.buffer_size = buffer_size
        self.net_arch = net_arch
        self.learning_starts = learning_starts
        self.batch_size = batch_size
        self.per = per
        self.per_alpha = per_alpha
        self.gradient_updates = gradient_updates
        self.initial_homotopy_lambda = initial_homotopy_lambda
        self.final_homotopy_lambda = final_homotopy_lambda
        self.homotopy_decay_steps = homotopy_decay_steps

        self.q_net = QNet(self.observation_shape, self.action_dim, self.reward_dim, net_arch=net_arch).to(self.device)
        self.target_q_net = QNet(self.observation_shape, self.action_dim, self.reward_dim, net_arch=net_arch).to(self.device)
        self.target_q_net.load_state_dict(self.q_net.state_dict())
        for p in self.target_q_net.parameters():
            p.requires_grad = False
        self.q_optim = FusedClipAdam(self.q_net.parameters(), lr=self.learning_rate)  # an optim.Adam with a fused clip+step

        self.envelope = envelope
        self.num_sample_w = num_sample_w
        self.homotopy_lambda = self.initial_homotopy_lambda
        if self.per:
            # with the transitions mirrored in HBM the sum tree lives there too (common/prioritized_buffer.DeviceSumTree, bit-identical to the
            # reference's numpy tree): sample -> gather -> update -> priorities -> tree is then ONE CUDA graph with no host round trip
            self.replay_buffer = PrioritizedReplayBuffer(self.observation_shape, 1, rew_dim=self.reward_dim, max_size=buffer_size, action_dtype=np.uint8,
                                                         device=self.device if replay_on_device else None,
                                                         tree_on_device=bool(replay_on_device and per_on_device and use_cuda_graph))
        else:
            self.replay_buffer = ReplayBuffer(self.observation_shape, 1, rew_dim=self.reward_dim, max_size=buffer_size, action_dtype=np.uint8,
                                              device=self.device if replay_on_device else None)
        self.dot_mode = ops.DOT_UNFUSED
        self.use_cuda_graph = use_cuda_graph
        # dense layers of all three passes on the tensor cores (wgmma, split operands, fp32-accurate).  No silent library fallback: a
        # network the tensor-core path does not cover is an error unless the caller explicitly opts into the validation path.
        # operand format of the tensor-core dense layers: "f16x2" (default: 3 MMAs / 4 B per element, fp16 exponent range with device-resident
        # power-of-two scales) or "bf16x3" (6 MMAs / 6 B per element, fp32 exponent range) -- tc_mlp.py
        fmt_name = tensor_core_format or os.environ.get("MORL_TC_FMT", "f16x2")
        if fmt_name not in ("f16x2", "bf16x3"):
            raise ValueError(f"tensor_core_format must be 'f16x2' or 'bf16x3', got {fmt_name!r}")
        if tensor_core_accumulators not in ("single", "split"):
            raise ValueError(f"tensor_core_accumulators must be 'single' or 'split', got {tensor_core_accumulators!r}")
        # "split": leading and correction products of the forward GEMMs in separate register accumulators (csrc/gemm_planes.cu), added
        # once with a correctly rounded fp32 add: fewer accumulations at full magnitude; a 256-wide layer then runs as two column units
        self.tensor_core_accumulators = tensor_core_accumulators
        self.tensor_core_format = fmt_name
        self._tc_fmt = ops.FMT_F16X2 if fmt_name == "f16x2" else ops.FMT_BF16X3
        if self._dp is not None and not use_tensor_cores:
            raise ops._lib.MorlB200Error("morl_baselines_b200.Envelope: dp_group needs the tensor-core update path (use_tensor_cores=True)")
        if use_tensor_cores and (self.q_net.feature_extractor is not None
                                 or not TCPairMlp.trainable_supported(self.q_net.net, num_sample_w, self._tc_fmt)):
            raise ops._lib.MorlB200Error(
                "morl_baselines_b200.Envelope: the tensor-core update path needs a flat observation, equal hidden widths that are multiples "
                f"of 64 and <= 512, and num_sample_w <= 256 (got obs {self.observation_shape}, net_arch {net_arch}, num_sample_w {num_sample_w}); "
                "pass use_tensor_cores=False to run the (slow) library-GEMM validation path explicitly")
        self.use_tensor_cores = bool(use_tensor_cores)
        self._tc_on = self._tc_tg = self._tc_train = None
        self._nograd_chain = None
        self._dq = self._grad_bufs = None
        self._last_lazy, self._last_inds_v, self._last_priority_v, self._updates_done = False, None, None, 0
        self._side_pending = False
        self._graphs = {}
        self._static = None
        self._last_loss = None
        self.log = log
        if log:
            self.setup_wandb(project_name, experiment_name, wandb_entity, group)

    # ------------------------------------------------------------------------------------------ config / io
    def get_config(self):
        return {
            "env_id": self.env.unwrapped.spec.id,
            "learning_rate": self.learning_rate,
            "initial_epsilon": self.initial_epsilon,
            "epsilon_decay_steps": self.epsilon_decay_steps,
            "batch_size": self.batch_size,
            "tau": self.tau,
            "clip_grand_norm": self.max_grad_norm,
            "target_net_update_freq": self.target_net_update_freq,
            "gamma": self.gamma,
            "use_envelope": self.envelope,
            "num_sample_w": self.num_sample_w,
            "net_arch": self.net_arch,
            "per": self.per,
            "gradient_updates": self.gradient_updates,
            "buffer_size": self.buffer_size,
            "initial_homotopy_lambda": self.initial_homotopy_lambda,
            "final_homotopy_lambda": self.final_homotopy_lambda,
            "homotopy_decay_steps": self.homotopy_decay_steps,
            "learning_starts": self.learning_starts,
            "seed": self.seed,
        }

    def save(self, save_replay_buffer: bool = True, save_dir: str = "weights/", filename: Optional[str] = None):
        """Checkpoint with the reference's keys (envelope.py:230-247)."""
        os.makedirs(save_dir, exist_ok=True)
        params = {"q_net_state_dict": self.q_net.state_dict(), "q_net_optimizer_state_dict": self.q_optim.state_dict()}
        if save_replay_buffer:
            params["replay_buffer"] = self.replay_buffer
        filename = getattr(self, "experiment_name", "Envelope") if filename is None else filename
        th.save(params, save_dir + "/" + filename + ".tar")

    def load(self, path: str, load_replay_buffer: bool = True):
        """Load a checkpoint written by this class or by the reference (envelope.py:249-261).  Tensors are overwritten in
        place so a captured CUDA graph stays valid."""
        params = th.load(path, weights_only=False, map_location=self.device)
        with th.no_grad():
            for net in (self.q_net, self.target_q_net):
                sd = net.state_dict()
                for k, v in params["q_net_state_dict"].items():
                    sd[k].copy_(v)
        self._load_optimizer_inplace(params["q_net_optimizer_state_dict"])
        if load_replay_buffer and "replay_buffer" in params:
            self.replay_buffer = params["replay_buffer"]
            if hasattr(self.replay_buffer, "to"):
                self.replay_buffer.to(self.device)
            self._graphs = {}  # a captured step gathers from the PREVIOUS buffer's device stores: re-capture against the new mirror

    def _load_optimizer_inplace(self, sd):
        cur = self.q_optim.state_dict()
        if len(cur["state"]) == 0 or not self._graphs:
            self.q_optim.load_state_dict(sd)
            self._graphs = {}  # state tensors were re-created: re-capture lazily
            return
        for gi, g in enumerate(sd["param_groups"]):
            for k, v in g.items():
                if k != "params":
                    self.q_optim.param_groups[gi][k] = v
        params = [p for g in self.q_optim.param_groups for p in g["params"]]
        for pid, st in sd["state"].items():
            dst = self.q_optim.state[params[pid]]
            for k, v in st.items():
                if th.is_tensor(v):
                    dst[k].copy_(v)
                else:
                    dst[k] = v

    # ------------------------------------------------------------------------------------------ the update
    def _ensure_static(self):
        """Static tensors of the update.  All per-step host inputs live in ONE pinned buffer mirrored by one device buffer:
            [ replay indices int64 B | homotopy lambda | weight vectors W x D | obs | next_obs | rewards | dones | actions int32 ]
        so a step issues a single host->device copy: indices + weights when the replay store is mirrored in HBM, weights +
        minibatch when it is host-resident (the reference makes six synchronous pageable copies, buffer.py:93-94)."""
        if self._static is not None:
            return self._static
        dev, B, W, D = self.device, self.batch_size, self.num_sample_w, self.reward_dim
        obs_n = int(np.prod(self.observation_shape))
        seg = lambda n: (n + 3) // 4 * 4  # noqa: E731  (16-byte aligned segments)
        sizes = [("idx", 2 * B), ("lam", 4), ("wset", W * D), ("obs", B * obs_n), ("nobs", B * obs_n), ("rew", B * D), ("done", B), ("act", B)]
        off, o = {}, 0
        for k, n in sizes:
            off[k] = (o, n)
            o += seg(n)
        total = o
        pin = th.zeros(total, dtype=th.float32).pin_memory()
        pdev = th.zeros(total, dtype=th.float32, device=dev)
        pnp = pin.numpy()
        cut = lambda buf, k: buf[off[k][0] : off[k][0] + off[k][1]]  # noqa: E731
        shp = {"wset": (W, D), "obs": (B,) + tuple(self.observation_shape), "nobs": (B,) + tuple(self.observation_shape), "rew": (B, D),
               "done": (B, 1), "act": (B, 1)}
        host = {k: cut(pnp, k).reshape(shp[k]) for k in shp if k != "act"}
        host["act"] = cut(pnp, "act").view(np.int32).reshape(B, 1)
        host["idx"] = cut(pnp, "idx").view(np.int64)
        host["lam"] = cut(pnp, "lam")
        # the captured step reads a PRIVATE copy (`work`, refreshed by the first node of the graph), so the next step's host->device
        # copy may overwrite `pdev` while the backward half of this step is still running
        work = th.zeros(total, dtype=th.float32, device=dev)
        stage = {k: cut(work, k).view(shp[k]) for k in ("obs", "nobs", "rew", "done")}
        stage["act"] = cut(work, "act").view(th.int32).view(B, 1)
        head_end = off["wset"][0] + seg(off["wset"][1])
        s = {
            "idx": cut(work, "idx").view(th.int64),
            "wset": cut(work, "wset").view(W, D),
            "lam": cut(work, "lam")[:1],  # device-resident homotopy lambda, refreshed with the per-step pack
            "work": work,
            # [priorities (B) | loss | pad | sampled indices as int64 (2 B floats)]: one device->host copy per step
            "result": th.zeros(seg(B + 1) + 2 * B, dtype=th.float32, device=dev),
            "ws": ops.td_workspace(B * W, dev),
            "pack_pin": pin, "pack_dev": pdev, "host": host, "stage": stage,
            # (device slice, pinned slice) of the one copy a step makes
            "copy_device": (pdev[:head_end], pin[:head_end]),
            "copy_host": (pdev[off["lam"][0] :], pin[off["lam"][0] :]),
            "result_pin": th.zeros(seg(B + 1) + 2 * B, dtype=th.float32).pin_memory(),
            "h2d_done": th.cuda.Event(),  # guards the pinned staging buffer against being overwritten while a copy is pending
            # recorded INSIDE the captured step right after the fused TD-loss kernel (external event node): the host waits for the
            # priorities only, writes them back to the sum-tree and prepares the next minibatch while the GPU runs backward + Adam
            "prio_ready": th.cuda.Event(external=True),
            "copy_stream": th.cuda.Stream(device=dev),
            "side_stream": th.cuda.Stream(device=dev),
            "side_stream2": th.cuda.Stream(device=dev),
            "side_stream3": th.cuda.Stream(device=dev),
        }
        # where a caller that stages inputs on the device itself (bench.py's `value` arm) must write them: the staging buffer, not the
        # private copy the graph refreshes from it
        s["in"] = {"idx": cut(pdev, "idx").view(th.int64), "wset": cut(pdev, "wset").view(W, D)}
        s["in"]["wset"].fill_(1.0 / D)
        s["wset"].fill_(1.0 / D)
        for buf in (pdev, work):
            cut(buf, "lam").fill_(float(self.homotopy_lambda))
        host["lam"][:] = np.float32(self.homotopy_lambda)
        s["prio"], s["loss"], s["loss1"] = s["result"][:B], s["result"][B], s["result"][B : B + 1]
        s["prio_np"] = s["result_pin"].numpy()[:B]
        s["loss_pin"] = s["result_pin"][B]
        # device-resident PER (mode "device_per"): the idx segment of the pack carries B uniform doubles instead of B int64 indices
        s["u"] = cut(work, "idx").view(th.float64)
        s["idx_out"] = s["result"][seg(B + 1) :].view(th.int64)  # the walk writes the sampled indices straight into the result record
        s["inds_np"] = s["result_pin"].numpy()[seg(B + 1) :].view(np.int64)
        s["host"]["u"] = cut(pnp, "idx").view(np.float64)
        s["raw_prio"] = th.zeros(B, dtype=th.float32, device=dev)
        s["prio64"] = th.zeros(B, dtype=th.float64, device=dev)
        # recorded INSIDE the captured step right after its first node: the staging buffer may be overwritten by the next step's copy
        s["consumed"] = th.cuda.Event(external=True)
        self._static = s
        return s

    def _gradient_step(self, obs, act, rew, nobs, done, wset, device_per: bool = False):
        """One gradient update on device tensors (everything between sampling and the priority write-back)."""
        s = self._static
        B, W, A, D = obs.shape[0], wset.shape[0], self.action_dim, self.reward_dim
        with th.no_grad():
            if self.use_tensor_cores and B == self.batch_size and W == self.num_sample_w:
                if self._tc_on is None:
                    split = self.tensor_core_accumulators == "split"
                    self._tc_on = TCPairMlp(self.q_net.net, self.q_net.feat_dim, B, W, fmt=self._tc_fmt, split_acc=split)
                    self._tc_tg = TCPairMlp(self.target_q_net.net, self.target_q_net.feat_dim, B, W, fmt=self._tc_fmt, split_acc=split)
                    if TCPairMlp.trainable_supported(self.q_net.net, W, self._tc_fmt):
                        self._tc_train = TCPairMlp(self.q_net.net, self.q_net.feat_dim, B, W if self._dp is None else self._dp["w_loc"],
                                                   share_weights_with=self._tc_on, trainable=True, split_acc=split)
                # every weight plane this step needs (online, target, transposed-for-backward) in one launch (unless _step already did it on a
                # side branch)
                if getattr(self, "_planes_fresh", False):
                    self._planes_fresh = False
                else:
                    TCPairMlp.refresh_many([self._tc_on, self._tc_tg], transposed_of=[self._tc_train] if self._tc_train is not None else [])
                early_q = None
                if _THREE_STREAMS and self._tc_train is not None:
                    # the training pass's forward (online net on s) does not depend on the targets: a third branch of the captured graph
                    main, side3 = th.cuda.current_stream(), s["side_stream3"]
                    side3.wait_stream(main)
                    with th.cuda.stream(side3):
                        dp_ = self._dp
                        ws_ = wset if dp_ is None else wset[dp_["rank"] * dp_["w_loc"] : (dp_["rank"] + 1) * dp_["w_loc"]]
                        early_q = self._tc_train.forward_pairs(obs, ws_)
                fused_head = self.envelope and _FUSED_HEAD and self.tensor_core_accumulators != "split" and self._tc_on.head_operands() is not None \
                    and ops.qhead_envelope_supported(self._tc_fmt, B, W, A, D, self._tc_on.lin[-1].in_features)
                self.fused_head_active = bool(fused_head)
                head_reverse = False
                if fused_head:
                    # output layers of both nets + envelope operator + Bellman line in ONE kernel: Q_on / Q_tg (envelope.py:420, :429) exist
                    # in tensor / shared memory only (csrc/qhead_envelope.cu; bit-identical to the three-launch chain below)
                    if self._tc_on.chain_supported() and self._tc_tg.chain_supported():
                        # hidden layers 2.. of BOTH nets in one persistent launch: a CTA takes each of its row tiles through all layers of
                        # both nets, re-reading every intermediate activation from L2 (csrc/gemm_planes.cu: gemm_chain_kernel)
                        if self._nograd_chain is None:
                            self._nograd_chain = TCPairMlp.make_chain([self._tc_on, self._tc_tg])
                        self._tc_on.layer1(nobs, wset)
                        self._tc_tg.layer1(nobs, wset)
                        self._nograd_chain()
                        h_on, h_tg = self._tc_on.h[-1], self._tc_tg.h[-1]
                        head_reverse = _HEAD_REVERSE  # the chain wrote its highest tiles last: start the head on them (still in L2)
                    elif _TWO_STREAMS:
                        # the two no-grad chains are independent: fork the target-net chain onto a side stream (a parallel branch of the
                        # captured graph) so that its kernels fill the launch gaps and tile tails of the online-net chain
                        main, side = th.cuda.current_stream(), s["side_stream2"]
                        side.wait_stream(main)
                        with th.cuda.stream(side):
                            h_tg = self._tc_tg.forward_hidden(nobs, wset)
                        h_on = self._tc_on.forward_hidden(nobs, wset)
                        main.wait_stream(side)
                    else:
                        h_on = self._tc_on.forward_hidden(nobs, wset)
                        h_tg = self._tc_tg.forward_hidden(nobs, wset)
                    (w_on, sw_on, b_on), (w_tg, sw_tg, b_tg) = self._tc_on.head_operands(), self._tc_tg.head_operands()
                    target_q, _, _ = ops.qhead_envelope_td(h_on, h_tg, w_on, w_tg, b_on.detach(), b_tg.detach(), wset, rew, done.reshape(-1), self.gamma,
                                                           B, W, A, D, self.dot_mode, ops.ROWS_BMAJOR, a_scale_on=self._tc_on.s_act,
                                                           a_scale_tg=self._tc_tg.s_act, w_scale_on=sw_on, w_scale_tg=sw_tg, reverse_tiles=head_reverse)
                    q_on = q_tg = None
                else:
                    q_on = self._tc_on.forward_pairs(nobs, wset).view(B, W, A, D)  # online net selects   (envelope.py:420)
                    q_tg = self._tc_tg.forward_pairs(nobs, wset).view(B, W, A, D)  # target net evaluates (envelope.py:429)
            else:
                fused_head, early_q = False, None
                q_on = self.q_net.forward_pairs(nobs, wset)
                q_tg = self.target_q_net.forward_pairs(nobs, wset)
            done1 = done.reshape(-1)
            if fused_head:
                pass
            elif self.envelope:
                target_q, _, _ = ops.envelope_td(q_on, q_tg, wset, rew, done1, self.gamma, self.dot_mode, ops.ROWS_BMAJOR, want_indices=False)
            else:
                target_q, _ = ops.greedy_td(q_on.view(B * W, A, D), q_tg.view(B * W, A, D), wset, rew, done1, self.gamma, self.dot_mode,
                                            ops.MAP_TILE, ops.MAP_BLOCK)
        dp = self._dp
        if self._tc_train is not None and B == self.batch_size and W == self.num_sample_w:
            # training pass on the tensor cores, without autograd: forward, fused loss (emits d loss / d Q, the loss and the priorities),
            # hand-written backward straight into the persistent .grad buffers; weight planes were refreshed above
            with th.no_grad():
                Wt, wset_t = W, wset
                if dp is not None:
                    # DP-Envelope: this rank's loss rows are those of its own scalarising weights i in [lo, hi) (all transitions); the targets
                    # above were formed for every i because the envelope maximum runs over all preference rows j
                    Wt, lo = dp["w_loc"], dp["rank"] * dp["w_loc"]
                    wset_t = wset[lo : lo + Wt]
                    target_q = target_q.view(B, W, D)[:, lo : lo + Wt].reshape(B * Wt, D)
                if early_q is not None:
                    th.cuda.current_stream().wait_stream(s["side_stream3"])
                    q_values = early_q.view(B * Wt, A, D)
                else:
                    q_values = self._tc_train.forward_pairs(obs, wset_t).view(B * Wt, A, D)
                if self._dq is None:
                    self._dq = th.empty_like(q_values)
                    self._grad_bufs = []
                    if dp is not None:
                        from ...parallel import DPFlat

                        dp["flat"] = DPFlat([p for l in self._tc_train.lin for p in (l.weight, l.bias)], B, dp["group"])
                        self._grad_bufs = list(dp["flat"].grads)
                        for prm, gbuf in zip([p for l in self._tc_train.lin for p in (l.weight, l.bias)], self._grad_bufs):
                            prm.grad = gbuf
                    else:
                        for l in self._tc_train.lin:
                            for p in (l.weight, l.bias):
                                p.grad = th.zeros_like(p)
                                self._grad_bufs.append(p.grad)
                raw = (s["raw_prio"] if device_per else s["prio"]) if self.per else None
                ops.td_mse_priority(q_values, act.reshape(-1), target_q, wset_t, 0.0, B, Wt, ops.ROWS_BMAJOR, want_grad=True, want_prio=self.per,
                                    workspace=s["ws"], loss_out=s["loss1"], grad_out=self._dq, prio_out=raw, lambda_dev=s["lam"])
                # device-resident PER: the priority / sum-tree branch (a single-block kernel with 45 KB of shared memory) is forked only
                # AFTER the last persistent GEMM of the backward pass -- forked right here it keeps one SM, hence one persistent CTA of every GEMM
                # that overlaps it, waiting; the host-tree modes keep the early hand-off
                defer_ship = dp is None and device_per and _DEFER_TREE
                if dp is None and not defer_ship:
                    self._ship_results(raw, device_per)
                for l, (gw, gb) in zip(self._tc_train.lin, zip(self._grad_bufs[0::2], self._grad_bufs[1::2])):
                    if l.weight.grad is not gw or l.bias.grad is not gb:  # (someone called zero_grad(set_to_none=True) in between)
                        l.weight.grad, l.bias.grad = gw, gb
                self._tc_train.backward(obs, wset_t, self._dq.view(B * Wt, A * D), grads_out=self._grad_bufs,
                                        after_gemms=(lambda: self._ship_results(raw, device_per)) if defer_ship else None)
            if dp is not None:
                return  # the collective and the optimiser step follow the captured half (_dp_finish)
        else:
            # explicit validation path (use_tensor_cores=False): torch autograd + library GEMMs around the same fused operators
            q_values = self.q_net.forward_pairs(obs, wset).view(B * W, A, D)
            raw = (s["raw_prio"] if device_per else s["prio"]) if self.per else None
            loss = _FusedTDLoss.apply(q_values, act.reshape(-1), target_q, wset, s["lam"], B, W, s["ws"], raw, s["loss1"])
            self._ship_results(raw, device_per)
            self.q_optim.zero_grad(set_to_none=True)
            loss.backward()
        self.q_optim.step_fused(self.max_grad_norm)  # clip_grad_norm_ + Adam.step (envelope.py:324-326) in two launches

    def _dp_finish(self):
        """Second half of a DP-Envelope update, after the (captured) forward / backward half: ONE all-reduce -- mean gradients into the
        parameters' .grad views, the owner rank's raw priorities and the mean loss into the result record --, then the hand-off of loss and
        priorities to the host and clip + Adam, identical on every rank."""
        s, dp = self._static, self._dp
        device_per = bool(self.per and getattr(self.replay_buffer, "tree_on_device", False) and self.use_cuda_graph)
        raw = (s["raw_prio"] if device_per else s["prio"]) if self.per else None  # where the captured half left |w . td| of the local rows
        prio, loss = dp["flat"].allreduce(raw, s["loss1"], owns_priorities=(dp["rank"] == 0))
        if self.per:
            raw.copy_(prio)
        s["loss1"].copy_(loss)
        # loss + priorities to the host; with the sum tree in HBM the priority power, the ratchet and the tree write-back run here as well
        # (stream-ordered, no host wait), so every rank's tree is updated with the same values before its next walk
        self._ship_results(raw, device_per)  # (side stream: runs under Adam; joined before the next step's tree walk, in update())
        self.q_optim.step_fused(self.max_grad_norm)

    def _ship_results(self, raw, device_per: bool):
        """Loss and priorities are final (the loss kernel wrote them): ship them to the host before the backward half starts.  With
        device-resident PER the priority power, the min_priority ratchet and SumTree.batch_set (envelope.py:329-334, prioritized_buffer.py:
        186-195) run here too, on a side stream -- a parallel branch of the captured graph, off the critical path of backward + Adam; it is
        joined again at the end of the step, so the tree is up to date for the next step's walk."""
        s = self._static
        if not device_per:
            s["result_pin"].copy_(s["result"], non_blocking=True)
            s["prio_ready"].record()
            return
        main, side = th.cuda.current_stream(), s["side_stream"]
        side.wait_stream(main)
        with th.cuda.stream(side):
            self.replay_buffer.update_priorities_dev(s["idx_out"], raw, self.per_alpha, s["prio64"], prio32_dev=s["prio"])
            s["result_pin"].copy_(s["result"], non_blocking=True)
            s["prio_ready"].record()
        self._side_pending = True

    def _step(self, mode: str):
        """What one CUDA graph captures.  mode "device": gather from the HBM-resident store by the static index buffer, then
        the gradient step; mode "host": the gradient step on the static staging tensors the host minibatch was copied into."""
        s = self._static
        src = s["copy_" + ("device" if mode == "device_per" else mode)][0]  # the segment of the staging buffer this mode's host->device copy fills
        s["work"][src.storage_offset() : src.storage_offset() + src.numel()].copy_(src)
        s["consumed"].record()  # the staging buffer may now be refilled for the next step
        pre = _PRE_REFRESH and self._tc_on is not None and self.use_tensor_cores
        if pre:
            # the weight planes of this step (online, target, transposed) depend only on the parameters: split them on a side branch while the
            # main branch walks the tree and gathers the minibatch
            main, side = th.cuda.current_stream(), s["side_stream2"]
            side.wait_stream(main)
            with th.cuda.stream(side):
                TCPairMlp.refresh_many([self._tc_on, self._tc_tg], transposed_of=[self._tc_train] if self._tc_train is not None else [])
            self._planes_fresh = True
        if mode == "device_per":
            # SumTree.sample on the device (prioritized_buffer.py:30-54): the host only supplied B uniform doubles from the numpy stream
            self.replay_buffer.tree.walk_into(s["u"], s["idx_out"], scale_by_root=True)
            obs_s, nobs_s, act_s, rew_s, done_s = self.replay_buffer.device_stores()
            obs, act, rew, nobs, done = ops.replay_gather(obs_s, nobs_s, act_s, rew_s, done_s, s["idx_out"])
        elif mode == "device":
            obs_s, nobs_s, act_s, rew_s, done_s = self.replay_buffer.device_stores()
            obs, act, rew, nobs, done = ops.replay_gather(obs_s, nobs_s, act_s, rew_s, done_s, s["idx"])
            s["idx_out"].copy_(s["idx"])
        else:
            st = s["stage"]
            obs, act, rew, nobs, done = st["obs"], st["act"], st["rew"], st["nobs"], st["done"]
        if pre:
            th.cuda.current_stream().wait_stream(s["side_stream2"])
        self._gradient_step(obs, act, rew, nobs, done, s["wset"], device_per=(mode == "device_per"))
        if self._side_pending:  # join the priority / tree branch
            th.cuda.current_stream().wait_stream(s["side_stream"])
            self._side_pending = False

    def _snapshot(self):
        snap = {"p": [p.detach().clone() for p in self.q_net.parameters()], "o": []}
        for p in self.q_net.parameters():
            st = self.q_optim.state.get(p, None)
            snap["o"].append(None if not st else {k: (v.clone() if th.is_tensor(v) else v) for k, v in st.items()})
        rb = self.replay_buffer
        if getattr(rb, "tree_on_device", False):  # the captured step also writes the device sum tree and min_priority
            snap["tree"] = (rb.tree.flat.clone(), rb._min_p_dev.clone())
        return snap

    def _restore(self, snap):
        with th.no_grad():
            for p, saved, st_saved in zip(self.q_net.parameters(), snap["p"], snap["o"]):
                p.copy_(saved)
                st = self.q_optim.state.get(p, None)
                if st:
                    for k, v in st.items():
                        if th.is_tensor(v):
                            v.copy_(st_saved[k]) if st_saved is not None else v.zero_()
            if "tree" in snap:
                self.replay_buffer.tree.flat.copy_(snap["tree"][0])
                self.replay_buffer._min_p_dev.copy_(snap["tree"][1])

    def _capture(self, mode: str):
        """Warm up on a side stream, capture one step into a CUDA graph, then restore parameters and optimiser state IN
        PLACE so the warm-up iterations leave no trace (parity with the reference's update count)."""
        self._ensure_static()
        if mode == "device":
            self.replay_buffer.flush()
        snap = self._snapshot()
        side = th.cuda.Stream()
        side.wait_stream(th.cuda.current_stream())
        with th.cuda.stream(side):
            for _ in range(3):
                self._step(mode)
        th.cuda.current_stream().wait_stream(side)
        g = th.cuda.CUDAGraph()
        before = ops.launch_count
        with th.cuda.graph(g):
            self._step(mode)
        self.launches_per_step = ops.launch_count - before
        self._restore(snap)
        self._graphs[mode] = g
        return g

    def __sample_indices(self):
        if self.per:
            return self.replay_buffer.tree.sample(self.batch_size)
        return self.replay_buffer._draw(self.batch_size)

    def update(self):
        """``gradient_updates`` gradient steps + target sync + schedules (reference envelope.py:266-367)."""
        s = self._ensure_static()
        rb = self.replay_buffer
        has_mirror = getattr(rb, "_dev", None) is not None
        # device-resident PER: the host's share of a step is B uniform doubles (the numpy stream SumTree.sample consumes) and the weight set;
        # walk, gather, update, priorities and the tree write-back are one graph replay and the host never waits for the GPU
        dev_per = bool(self.per and has_mirror and getattr(rb, "tree_on_device", False) and self.use_cuda_graph)
        critic_losses = []
        priority = None
        for _ in range(self.gradient_updates):
            # RNG consumption order of the reference: replay indices (global numpy RNG) first, then the weights (self.np_random)
            s["h2d_done"].synchronize()
            host = s["host"]
            b_inds = None
            if dev_per:
                host["u"][:] = np.random.random_sample(self.batch_size)  # np.random.uniform(0, root, B) = root * these, formed on the device
            else:
                b_inds = self.__sample_indices()
                if has_mirror:
                    host["idx"][:] = b_inds
                else:  # host-resident buffer: the minibatch crosses PCIe every update, packed into the pinned staging buffer
                    self._stage_host_batch(b_inds)
            w_np = random_weights(dim=self.reward_dim, n=self.num_sample_w, dist="gaussian", rng=self.np_random)
            host["wset"][:] = np.asarray(w_np).reshape(self.num_sample_w, -1)  # float64 -> float32, as th.tensor(w).float() (envelope.py:278)
            host["lam"][0] = np.float32(self.homotopy_lambda)  # read by the loss kernel from device memory: the graph survives the schedule
            mode = "device_per" if dev_per else ("device" if has_mirror else "host")
            dst, src = s["copy_" + ("device" if has_mirror else "host")]
            # the copy runs on its own stream and waits (on the device) until the previous step's graph has consumed the staging buffer
            # (`consumed`, recorded right after the graph's first node), so it overlaps that step's forward / backward
            if self.per:
                cs = s["copy_stream"]
                with th.cuda.stream(cs):
                    cs.wait_event(s["consumed"])
                    dst.copy_(src, non_blocking=True)
                    s["h2d_done"].record(cs)
                th.cuda.current_stream().wait_event(s["h2d_done"])
            else:
                dst.copy_(src, non_blocking=True)
                s["h2d_done"].record()

            if self._dp is not None and self._side_pending:  # the previous update's tree write-back (forked after its all-reduce)
                th.cuda.current_stream().wait_stream(s["side_stream"])
                self._side_pending = False
            if self.use_cuda_graph:
                g = self._graphs.get(mode) or self._capture(mode)
                if has_mirror:
                    rb.flush()
                g.replay()
            else:
                self._step(mode)
            if self._dp is not None:
                self._dp_finish()
            # (the static loss scalar is overwritten by the next gradient update: keep a copy when several are averaged)
            critic_losses.append(s["loss"].clone() if self.gradient_updates > 1 else s["loss"])
            self._updates_done += 1

            if dev_per:
                self._last_lazy = True  # indices / priorities of this step sit in the pinned result record: fetched on demand
                if self._updates_done % 256 == 0:
                    self._fetch_last()  # periodic health check: non-finite priorities must not poison the tree silently
            elif self.per:
                s["prio_ready"].synchronize()  # the priorities of THIS step have landed in pinned memory; backward + Adam still run
                if not np.isfinite(s["prio_np"]).all():
                    self._raise_non_finite()
                priority = (s["prio_np"] + rb.min_priority) ** self.per_alpha  # envelope.py:333 (float32, as the reference's tensor math)
                rb.update_priorities(b_inds, priority)
            if not dev_per:
                self._last_lazy, self._last_inds_v, self._last_priority_v = False, b_inds, priority

        if self.tau != 1 or self.global_step % self.target_net_update_freq == 0:
            polyak_update(self.q_net.parameters(), self.target_q_net.parameters(), self.tau)
        if self.epsilon_decay_steps is not None:
            self.epsilon = linearly_decaying_value(self.initial_epsilon, self.epsilon_decay_steps, self.global_step, self.learning_starts,
                                                   self.final_epsilon)
        if self.homotopy_decay_steps is not None:
            self.homotopy_lambda = linearly_decaying_value(self.initial_homotopy_lambda, self.homotopy_decay_steps, self.global_step,
                                                           self.learning_starts, self.final_homotopy_lambda)
        self._last_loss = critic_losses[-1] if critic_losses else None
        if self.log and self.global_step % 100 == 0:
            import wandb

            wandb.log({"losses/critic_loss": float(th.stack(critic_losses).mean()), "metrics/epsilon": self.epsilon,
                       "metrics/homotopy_lambda": self.homotopy_lambda, "global_step": self.global_step})
            wandb.log({"losses/grad_norm": get_grad_norm(self.q_net.parameters()).item(), "global_step": self.global_step})
            if self.per:
                wandb.log({"metrics/mean_priority": np.mean(self._last_priority)})

    def _fetch_last(self):
        """Device PER: wait for the last step's result record (sampled indices, powered priorities, loss) and check it."""
        s = self._static
        s["prio_ready"].synchronize()
        self._last_inds_v, self._last_priority_v = s["inds_np"].copy(), s["prio_np"].copy()
        self._last_lazy = False
        if not np.isfinite(self._last_priority_v).all():
            self._raise_non_finite()
        self.replay_buffer.tree.check()

    @property
    def _last_inds(self):
        """Replay indices of the most recent gradient update (numpy int64 [B])."""
        if self._last_lazy:
            self._fetch_last()
        return self._last_inds_v

    @property
    def _last_priority(self):
        """Priorities (|w . td| + min_priority) ** alpha written by the most recent gradient update (numpy float32 [B]); None without PER."""
        if self._last_lazy:
            self._fetch_last()
        return self._last_priority_v

    def _raise_non_finite(self):
        """The priorities of an update came back Inf / NaN: say why (the reference would silently write NaN priorities into its sum-tree)."""
        n = ops.plane_overflow_count() if self.use_tensor_cores and self._tc_fmt == ops.FMT_F16X2 else 0
        if n:
            raise ops._lib.MorlB200Error(
                f"Envelope.update: non-finite TD errors; {n} kernel launch(es) saw an activation or a back-propagated gradient outside the fp16 "
                "range of the 'f16x2' tensor-core operand format (|activation| >= 32752, or a backward gain beyond 2^13; see tc_mlp.py) -- "
                "construct the agent with tensor_core_format='bf16x3' (fp32 exponent range) for this problem")
        raise FloatingPointError("Envelope.update: non-finite TD errors (diverged Q-network or non-finite rewards / observations in the replay buffer)")

    def last_loss_host(self, wait: bool = True) -> float:
        """Critic loss of the most recent gradient update as a python float (the reference reads ``critic_loss.item()`` every update,
        envelope.py:327).  The value is copied to pinned host memory INSIDE the captured step right after the loss kernel, so reading it
        waits for the forward half of the step only, not for backward + Adam."""
        s = self._static
        if wait:
            s["prio_ready"].synchronize()
        return float(s["loss_pin"])

    def _stage_host_batch(self, inds):
        """Gather the host-resident minibatch for ``inds`` straight into the pinned staging buffer (C row gathers,
        csrc/host_replay.cu); replaces the reference's fancy-index temporaries + six synchronous th.tensor(x, device) copies
        (buffer.py:84-94)."""
        rb, host = self.replay_buffer, self._static["host"]
        lib = ops._lib.load()
        idx = np.ascontiguousarray(inds, dtype=np.int64)
        n = idx.shape[0]
        for key, arr in (("obs", rb.obs), ("nobs", rb.next_obs), ("rew", rb.rewards), ("done", rb.dones)):
            if arr.dtype != np.float32 or not arr.flags.c_contiguous:
                host[key][:] = arr[idx].reshape(host[key].shape)
                continue
            row_bytes = arr.strides[0]
            ops._lib.check(lib.morl_host_gather_rows(arr.ctypes.data, row_bytes, idx.ctypes.data, n, host[key].ctypes.data), "morl_host_gather_rows")
        act = rb.actions
        if act.dtype == np.uint8 and act.flags.c_contiguous:
            ops._lib.check(lib.morl_host_gather_u8_to_i32(act.ctypes.data, act.shape[1], idx.ctypes.data, n, host["act"].ctypes.data),
                           "morl_host_gather_u8_to_i32")
        else:
            host["act"][:] = act[idx].astype(np.int32).reshape(host["act"].shape)

    # ------------------------------------------------------------------------------------------ acting
    def eval(self, obs: np.ndarray, w: np.ndarray) -> int:
        obs = th.as_tensor(obs).float().to(self.device)
        w = th.as_tensor(w).float().to(self.device)
        return self.max_action(obs, w)

    def act(self, obs: th.Tensor, w: th.Tensor) -> int:
        """Epsilon-greedy action (reference envelope.py:375-387)."""
        if self.np_random.random() < self.epsilon:
            return self.env.action_space.sample()
        return self.max_action(obs, w)

    @th.no_grad()
    def max_action(self, obs: th.Tensor, w: th.Tensor) -> int:
        """argmax_a w . Q(obs, w)[a] (reference envelope.py:389-402); scalarise + argmax is one kernel."""
        q = self.q_net(obs, w)  # [1, A, D]
        _, _, act = ops.gpi_envelope(q.view(1, 1, 1, self.action_dim, self.reward_dim), w.reshape(1, -1), dot_mode=self.dot_mode)
        return int(act.item())

    @th.no_grad()
    def eval_batch(self, obs: np.ndarray, w: np.ndarray) -> np.ndarray:
        """Greedy actions for N (observation, weight) pairs at once -- the batched form of ``eval`` used by the lockstep evaluation round
        (common/evaluation.policy_evaluation_mo_batched): one network call + one scalarise/argmax kernel + one device->host copy."""
        obs_t = th.as_tensor(np.asarray(obs)).float().to(self.device)
        w_t = th.as_tensor(np.asarray(w)).float().to(self.device)
        n = obs_t.shape[0]
        q = self.q_net(obs_t, w_t)  # [N, A, D]
        _, _, act = ops.gpi_envelope(q.view(1, n, 1, self.action_dim, self.reward_dim), w_t, dot_mode=self.dot_mode)
        return act.cpu().numpy()

    @th.no_grad()
    def envelope_target(self, obs: th.Tensor, w: th.Tensor, sampled_w: th.Tensor) -> th.Tensor:
        """Reference calling convention (envelope.py:404-440): ``obs`` is the |W|-times tiled next-observation batch
        [W*B, ...], ``w`` the repeat_interleaved weights [W*B, D]; returns max_next_q [W*B, D] in the reference row order.
        Only the first B rows of ``obs`` are distinct; Q is evaluated on B*W rows."""
        W = sampled_w.size(0)
        B = obs.size(0) // W
        nobs = obs[:B]
        q_on = self.q_net.forward_pairs(nobs, sampled_w)
        q_tg = self.target_q_net.forward_pairs(nobs, sampled_w)
        zeros_r = th.zeros(B, self.reward_dim, device=obs.device)
        out, _, _ = ops.envelope_td(q_on, q_tg, sampled_w, zeros_r, th.zeros(B, device=obs.device), 1.0, self.dot_mode, ops.ROWS_REFERENCE,
                                    want_indices=False)
        return out  # 0 + ((1 - 0) * 1) * q == q exactly

    @th.no_grad()
    def ddqn_target(self, obs: th.Tensor, w: th.Tensor) -> th.Tensor:
        """Double-DQN target for paired rows (reference envelope.py:442-463)."""
        q_sel = self.q_net(obs, w)
        q_eval = self.target_q_net(obs, w)
        out, _ = ops.greedy_td(q_sel, q_eval, w, dot_mode=self.dot_mode)
        return out

    # ------------------------------------------------------------------------------------------ training loop
    def train(
        self,
        total_timesteps: int,
        eval_env=None,
        ref_point: Optional[np.ndarray] = None,
        known_pareto_front: Optional[List[np.ndarray]] = None,
        weight: Optional[np.ndarray] = None,
        total_episodes: Optional[int] = None,
        reset_num_timesteps: bool = True,
        eval_freq: int = 10000,
        num_eval_weights_for_front: int = 100,
        num_eval_episodes_for_front: int = 5,
        num_eval_weights_for_eval: int = 50,
        reset_learning_starts: bool = False,
        verbose: bool = False,
    ):
        """Interact with the (host) environment, one update per step after ``learning_starts`` (reference envelope.py:465-572)."""
        if eval_env is not None:
            assert ref_point is not None, "Reference point must be provided for the hypervolume computation."
        if self.log:
            self.register_additional_config({
                "total_timesteps": total_timesteps, "ref_point": ref_point.tolist() if ref_point is not None else None,
                "known_front": known_pareto_front, "weight": weight.tolist() if weight is not None else None,
                "total_episodes": total_episodes, "reset_num_timesteps": reset_num_timesteps, "eval_freq": eval_freq,
                "num_eval_weights_for_front": num_eval_weights_for_front, "num_eval_episodes_for_front": num_eval_episodes_for_front,
                "num_eval_weights_for_eval": num_eval_weights_for_eval, "reset_learning_starts": reset_learning_starts})
        self.global_step = 0 if reset_num_timesteps else self.global_step
        self.num_episodes = 0 if reset_num_timesteps else self.num_episodes
        if reset_learning_starts:
            self.learning_starts = self.global_step
        num_episodes = 0
        eval_weights = equally_spaced_weights(self.reward_dim, n=num_eval_weights_for_front) if eval_env is not None else None
        obs, _ = self.env.reset()
        w = weight if weight is not None else random_weights(self.reward_dim, 1, dist="gaussian", rng=self.np_random)
        tensor_w = th.tensor(w).float().to(self.device)

        for _ in range(1, total_timesteps + 1):
            if total_episodes is not None and num_episodes == total_episodes:
                break
            if self.global_step < self.learning_starts:
                action = self.env.action_space.sample()
            else:
                action = self.act(th.as_tensor(obs).float().to(self.device), tensor_w)
            next_obs, vec_reward, terminated, truncated, info = self.env.step(action)
            self.global_step += 1
            self.replay_buffer.add(obs, action, vec_reward, next_obs, terminated)
            if self.global_step >= self.learning_starts:
                self.update()
            if eval_env is not None and self.log and self.global_step % eval_freq == 0:
                from ...common.evaluation import log_all_multi_policy_metrics

                front = [self.policy_eval(eval_env, weights=ew, num_episodes=num_eval_episodes_for_front, log=self.log)[3] for ew in eval_weights]
                log_all_multi_policy_metrics(current_front=front, hv_ref_point=ref_point, reward_dim=self.reward_dim,
                                             global_step=self.global_step, n_sample_weights=num_eval_weights_for_eval,
                                             ref_front=known_pareto_front)
            if terminated or truncated:
                obs, _ = self.env.reset()
                num_episodes += 1
                self.num_episodes += 1
                if self.log and "episode" in info.keys():
                    from ...common.evaluation import log_episode_info

                    log_episode_info(info["episode"], np.dot, w, self.global_step, verbose=verbose)
                if weight is None:
                    w = random_weights(self.reward_dim, 1, dist="gaussian", rng=self.np_random)
                    tensor_w = th.tensor(w).float().to(self.device)
            else:
                obs = next_obs
