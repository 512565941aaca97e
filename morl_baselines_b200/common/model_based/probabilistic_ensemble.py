"""Probabilistic ensemble of dynamics networks for GPI-PD's Dyna path (SURVEY 8(f)3; mirrors reference
common/model_based/probabilistic_ensemble.py: same class / parameter / state_dict names, same constructor and ``fit`` arguments, same
numpy RNG consumption).

Device form: the training set, the bootstrap index table and the hold-out set live in HBM for the whole ``fit`` (the reference slices
numpy arrays and copies every minibatch to the device); a minibatch is a device gather; the five hold-out losses of an epoch come back in ONE
device-to-host copy (the reference calls ``.item()`` per network); ``sample`` is one batched forward plus ONE fused kernel
(``morl_ensemble_sample_f32``: logvar clamps, exp, reparameterised sample of the drawn elite, ensemble moments, uncertainty, + obs) instead
of three [E, N, O] device-to-host copies and a dozen numpy passes.  The dense layers are plain batched library GEMMs (``th.baddbmm``),
as in the reference on CUDA.
"""

from __future__ import annotations

import os

import numpy as np
import torch as th
from torch import nn as nn
from torch.nn import functional as F

from ... import ops
from ..graphed import GraphedStep

# minibatch steps of ``fit`` as CUDA-graph replays (MORL_DYNA_FIT_GRAPH=0: eager steps, the reference's op-by-op form)
_FIT_GRAPH = os.environ.get("MORL_DYNA_FIT_GRAPH", "1") != "0"


class EnsembleLayer(nn.Module):
    """One dense layer of every ensemble member: W [E, in, out], b [E, 1, out] (reference probabilistic_ensemble.py:11-25)."""

    def __init__(self, ensemble_size, input_dim, output_dim):
        super().__init__()
        self.W = nn.Parameter(th.empty((ensemble_size, input_dim, output_dim)), requires_grad=True).float()
        nn.init.orthogonal_(self.W, gain=nn.init.calculate_gain("relu"))
        self.b = nn.Parameter(th.zeros((ensemble_size, 1, output_dim)), requires_grad=True).float()

    def forward(self, x):  # x: [E, batch, in]
        return th.baddbmm(self.b, x, self.W)


class ProbabilisticEnsemble(nn.Module):
    """Ensemble of Gaussian dynamics models (reference probabilistic_ensemble.py:28-290)."""

    def __init__(self, input_dim, output_dim, ensemble_size=5, arch=[200, 200, 200, 200], activation=F.relu, learning_rate=0.001, num_elites=2,
                 normalize_inputs=True, device="auto"):
        super().__init__()
        self.ensemble_size = ensemble_size
        self.input_dim = input_dim
        self.output_dim = output_dim * 2  # mean and (log) variance
        self.activation = activation
        self.arch = arch
        self.num_elites = num_elites
        self.elites = [i for i in range(self.ensemble_size)]
        self.normalize_inputs = normalize_inputs
        self.learning_rate = learning_rate
        self.layers = nn.ModuleList()
        in_size = input_dim
        for hidden_size in self.arch:
            self.layers.append(EnsembleLayer(ensemble_size, in_size, hidden_size))
            in_size = hidden_size
        self.layers.append(EnsembleLayer(ensemble_size, self.arch[-1], self.output_dim))
        if self.normalize_inputs:
            self.inputs_mu = nn.Parameter(th.zeros((1, input_dim)), requires_grad=False)
            self.inputs_sigma = nn.Parameter(th.zeros((1, input_dim)), requires_grad=False)
        self.max_logvar = nn.Parameter(th.ones(1, output_dim, dtype=th.float32) / 2.0)
        self.min_logvar = nn.Parameter(-th.ones(1, output_dim, dtype=th.float32) * 10.0)
        if device == "auto":
            self.device = th.device("cuda") if th.cuda.is_available() else th.device("cpu")
        else:
            self.device = th.device(device)
        if self.device.type != "cuda":
            raise ops._lib.MorlB200Error("morl_baselines_b200.ProbabilisticEnsemble needs a CUDA device (no CPU fallback)")
        self.to(self.device)
        # test hook: a callable (shape, device) -> standard normal tensor replacing th.randn (CPU and CUDA generators differ, so parity
        # tests inject the reference's draws)
        self.noise_fn = None

    # ------------------------------------------------------------------------------------------ forward
    def _raw(self, input):
        """Raw output [E, N, 2*O] of the last layer (reference :87-111 up to the chunk)."""
        dim = len(input.shape)
        h = (input - self.inputs_mu) / self.inputs_sigma if self.normalize_inputs else input
        if dim < 3:
            h = h.unsqueeze(0)
            if dim == 1:
                h = h.unsqueeze(0)
            h = h.repeat(self.ensemble_size, 1, 1)
        for layer in self.layers[:-1]:
            h = self.activation(layer(h))
        return self.layers[-1](h)

    def forward(self, input, deterministic=False, return_dist=False):
        """Same contract as the reference's forward (:87-134)."""
        dim = len(input.shape)
        output = self._raw(input)
        if dim == 1:
            output = output.squeeze(1)
        mean, logvar = th.chunk(output, 2, dim=-1)
        logvar = self.max_logvar - F.softplus(self.max_logvar - logvar)
        logvar = self.min_logvar + F.softplus(logvar - self.min_logvar)
        if deterministic:
            return (mean, logvar) if return_dist else mean
        std = th.exp(0.5 * logvar)
        samples = mean + std * self._randn(std.shape)
        return (samples, mean, logvar) if return_dist else samples

    def _randn(self, shape):
        if self.noise_fn is not None:
            return self.noise_fn(tuple(shape), self.device)
        return th.randn(shape, device=self.device)

    @th.no_grad()
    def sample_device(self, input: th.Tensor, deterministic=False, obs: th.Tensor = None, rew_dim: int = 0):
        """``sample`` (reference :136-154) with everything after the last layer fused into one kernel and the results left on the
        device: (samples [N, O], vars [N, O], uncertainties [N]).  ``obs`` (optional) is added to the state part of the samples
        (ModelEnv.step, reference utils.py:165).  The elite of every row is drawn on the host from numpy's global RNG exactly like the
        reference's ``np.random.choice(self.elites, size=batch_size)``."""
        out = self._raw(input)  # [E, N, 2 O]
        E, N, O2 = out.shape
        model_inds = np.random.choice(self.elites, size=N)
        idx = th.from_numpy(np.ascontiguousarray(model_inds, dtype=np.int32)).to(self.device, non_blocking=True)
        noise = None if deterministic else self._randn((E, N, O2 // 2)).contiguous()
        return ops.ensemble_sample(out.contiguous(), self.max_logvar, self.min_logvar, idx, noise, obs, rew_dim)

    def sample(self, input, deterministic=False):
        """Reference signature (:136-154): numpy results."""
        s, v, u = self.sample_device(input, deterministic)
        return s.cpu().numpy(), v.cpu().numpy(), u.cpu().numpy()

    # ------------------------------------------------------------------------------------------ losses
    def _compute_loss(self, x, y):
        mean, logvar = self.forward(x, deterministic=True, return_dist=True)
        if len(y.shape) < 3:
            y = y.unsqueeze(0).repeat(self.ensemble_size, 1, 1)
        # F.gaussian_nll_loss(mean, y, exp(logvar), reduction="none") written out with its own arithmetic (eps = 1e-6, full = False): the library
        # function validates `var >= 0` with a host synchronisation, which is illegal inside a captured step
        var = th.exp(logvar).clone()
        with th.no_grad():
            var.clamp_(min=1e-6)
        total_losses = (0.5 * (th.log(var) + (mean - y) ** 2 / var)).mean()
        total_losses = total_losses + 0.01 * self.max_logvar.sum() - 0.01 * self.min_logvar.sum()
        return total_losses

    def _compute_mse_losses(self, x, y):
        mean = self.forward(x, deterministic=True, return_dist=False)
        if len(y.shape) < 3:
            y = y.unsqueeze(0).repeat(self.ensemble_size, 1, 1)
        return ((mean - y) ** 2).mean(-1).mean(-1)

    def save(self, path):
        save_dir = "weights/"
        if not os.path.isdir(save_dir):
            os.makedirs(save_dir)
        th.save({"ensemble_state_dict": self.state_dict()}, path + ".tar")

    def load(self, path):
        params = th.load(path, map_location=self.device)
        self.load_state_dict(params["ensemble_state_dict"])

    def _fit_input_stats(self, data):
        mu = np.mean(data, axis=0, keepdims=True)
        sigma = np.std(data, axis=0, keepdims=True)
        sigma[sigma < 1e-12] = 1.0
        self.inputs_mu.data = th.tensor(mu).to(self.device).float()
        self.inputs_sigma.data = th.tensor(sigma).to(self.device).float()

    # ------------------------------------------------------------------------------------------ training
    _WEIGHT_DECAYS = (0.000025, 0.00005, 0.000075, 0.000075, 0.0001)  # per layer, as the reference (:224)

    def _make_optimizer(self, capturable: bool):
        self.decays = list(self._WEIGHT_DECAYS)
        groups = [{"params": list(layer.parameters()), "weight_decay": self.decays[i]} for i, layer in enumerate(self.layers)]
        groups += [{"params": [self.max_logvar]}, {"params": [self.min_logvar]}]
        self.optim = th.optim.Adam(groups, lr=self.learning_rate, capturable=capturable)
        if capturable:
            # the state a captured step mutates must exist (and be snapshot) before the capture: Adam creates it lazily otherwise
            for grp in self.optim.param_groups:
                for prm in grp["params"]:
                    self.optim.state[prm] = {"step": th.zeros((), dtype=th.float32, device=prm.device), "exp_avg": th.zeros_like(prm),
                                             "exp_avg_sq": th.zeros_like(prm)}
                    prm.grad = th.zeros_like(prm)

    def _fit_mutated(self):
        out = []
        for grp in self.optim.param_groups:
            for prm in grp["params"]:
                st = self.optim.state[prm]
                out += [prm, prm.grad, st["step"], st["exp_avg"], st["exp_avg_sq"]]
        return out

    def _upload_split(self, X, Y, num_holdout):
        """Training set and hold-out set as device tensors: ONE upload of X and Y, the split is a device gather by the host permutation
        (``np.random.permutation``: first draw of the reference's ``fit``)."""
        order = th.from_numpy(np.random.permutation(X.shape[0])).to(self.device)
        Xd = th.from_numpy(np.ascontiguousarray(X)).to(self.device).float()
        Yd = th.from_numpy(np.ascontiguousarray(Y)).to(self.device).float()
        held, kept = order[:num_holdout], order[num_holdout:]
        return (Xd[kept], Yd[kept]), (Xd[held], Yd[held])

    def _train_step(self, xs, ys, pick):
        loss = self._compute_loss(xs[pick], ys[pick])
        self.optim.zero_grad(set_to_none=False)
        loss.backward()
        self.optim.step()

    def _train_epoch(self, train, table, batch_size, graph_state):
        """One pass over the bootstrap table [E, n]: member e of minibatch k sees rows table[e, k*bs:(k+1)*bs] (device gathers).  Full
        minibatches replay ONE captured step (gather, likelihood, backward, Adam over a static index buffer: ~40 launches -> one graph
        replay); a ragged last minibatch runs the same step eagerly."""
        xs, ys = train
        rows = th.from_numpy(table).to(self.device)
        self.train()
        for lo in range(0, table.shape[-1], batch_size):
            pick = rows[:, lo:lo + batch_size]
            if graph_state is not None and pick.shape[1] == batch_size:
                if "step" not in graph_state:
                    graph_state["idx"] = pick.clone()
                    graph_state["step"] = GraphedStep(lambda: self._train_step(xs, ys, graph_state["idx"]), self._fit_mutated)
                graph_state["idx"].copy_(pick)
                graph_state["step"]()
            else:
                self._train_step(xs, ys, pick)

    def fit(self, X, Y, batch_size=256, holdout_ratio=0.1, max_holdout_size=5000, max_epochs_no_improvement=5, max_epochs=200):
        """Maximum-likelihood training with bootstrapped minibatches and hold-out early stopping (reference :197-290).  numpy's global RNG is
        consumed in the reference's order: the split permutation, the bootstrap table, one uniform table per epoch (row shuffles)."""
        if self.normalize_inputs:
            self._fit_input_stats(X)
        use_graph = _FIT_GRAPH
        self._make_optimizer(capturable=use_graph)
        graph_state = {} if use_graph else None
        num_holdout = min(int(X.shape[0] * holdout_ratio), max_holdout_size)
        train, held = self._upload_split(X, Y, num_holdout)
        n_train = train[0].shape[0]
        table = np.random.randint(n_train, size=[self.ensemble_size, n_train])
        best = [float("inf")] * self.ensemble_size
        holdout_losses = list(best)
        stale, epoch = 0, 0
        while stale < max_epochs_no_improvement and epoch < max_epochs:
            self._train_epoch(train, table, batch_size, graph_state)
            # every member's row is permuted independently for the next epoch (argsort of one uniform table, :243-245)
            table = np.take_along_axis(table, np.argsort(np.random.uniform(size=table.shape), axis=-1), axis=-1)
            self.eval()
            with th.no_grad():
                holdout_losses = self._compute_mse_losses(*held).cpu().tolist()  # the E losses in one device-to-host copy
            self.elites = np.argsort(holdout_losses)[: self.num_elites]
            # a member "improves" when its hold-out loss drops by more than 1 % (always in the first epoch); any improvement resets the counter
            improved = False
            for e, cur in enumerate(holdout_losses):
                if epoch == 0 or (best[e] - cur) / best[e] > 0.01:
                    best[e], improved = cur, True
            stale = 0 if improved else stale + 1
            epoch += 1
        print("Epoch:", epoch, "Holdout losses:", ", ".join(["%.4f" % hl for hl in holdout_losses]))
        return np.mean(holdout_losses)
