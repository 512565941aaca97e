"""Linear Support weight selection (OLS and GPI-LS) -- drop-in for reference morl_baselines/multi_policy/linear_support/linear_support.py
(same constructor and defaults, same methods and return types).  Needs neither cvxpy nor pycddlib.

* The corner weights (reference :295-349, cdd vertex enumeration) are ONE device launch: ``ops.corner_weights`` enumerates the
  vertices of { V w <= u, w >= 0, sum w = 1 } exactly in float64 (csrc/linear_support.cu); a degenerate vertex comes out once.
* OLS's optimistic bound ``max_value_lp`` (reference :258-293, cvxpy) is ``scipy.optimize.linprog`` (HiGHS) on the host: d variables
  and one row per visited weight, not device-shaped work.  An unbounded LP (before every extremum has been visited) returns +inf.
* GPI-LS's expanded set is evaluated once per ``next_weight`` call for all corner weights at once with
  ``policy_evaluation_mo_batched`` (one batched ``eval_batch`` call per environment step); agents without ``eval_batch`` are
  evaluated with the serial ``policy_evaluation_mo``, once per corner weight.
* Everything else -- queue, ``visited_weights``, ``ccs``, ``weight_support``, dominance and obsolescence tests (the reference's exact
  ``==``), the stable descending priority sort, ``random.shuffle`` on python's global ``random`` when the top priority is 0, the
  ``epsilon is None`` rule -- is float64 numpy with the reference's expressions.

Deliberate deviations from the reference:
* Corner order: cdd's vertex order cannot be reproduced without cdd, so corners come in a canonical order (lexicographic on the
  values rounded to 1e-9, after |w| / sum |w| and snapping values within 1e-9 of 0 to 0).  That order breaks ties in the stable
  priority sort and is what ``random.shuffle`` permutes.
* Expanded set: the reference re-evaluates the GPI agent at all |W_c| corner weights inside its loop over the corner weights
  (|W_c|^2 x rep_eval episodes); here it is evaluated once (|W_c| x rep_eval episodes).  Identical for a deterministic environment and
  agent.
* Stochastic environments: the batched evaluation runs on deep copies of ``env``, whose episodes share its RNG state (see
  ``policy_evaluation_mo_batched``).
"""

from __future__ import annotations

import random
from copy import deepcopy
from typing import List, Optional

import numpy as np
import torch as th

from ... import ops
from ...common.evaluation import policy_evaluation_mo, policy_evaluation_mo_batched
from ...common.weights import extrema_weights

SNAP_TOL = 1e-9      # corner coordinates within this of 0 become exactly 0 (the kernel's tolerance on w)
ORDER_DECIMALS = 9   # canonical order: lexicographic on the values rounded to 1e-9


def canonical_corners(w: np.ndarray) -> np.ndarray:
    """Host post-processing of the vertex weights w [K, d] (reference :342-347 plus the canonical order): |w| / sum |w|, values within
    SNAP_TOL of 0 snapped to 0, rows sorted lexicographically on the values rounded to ORDER_DECIMALS."""
    w = np.abs(np.asarray(w, dtype=np.float64))
    if w.shape[0] == 0:
        return w
    w = w / w.sum(axis=1, keepdims=True)
    w[w <= SNAP_TOL] = 0.0
    key = np.round(w, ORDER_DECIMALS)
    return w[np.lexsort(key.T[::-1])]


class LinearSupport:
    """Linear Support for computing corner weights when using linear utility functions: Optimistic Linear Support (OLS; Roijers,
    thesis section 3.3) and Generalized Policy Improvement Linear Support (GPI-LS; Alegre et al., AAMAS 2023)."""

    def __init__(self, num_objectives: int, epsilon: float = 0.0, verbose: bool = True):
        """Args: num_objectives: number of objectives; epsilon: minimum improvement per iteration (None: keep every corner weight);
        verbose: print progress."""
        self.num_objectives = num_objectives
        self.epsilon = epsilon
        self.visited_weights = []
        self.ccs = []
        self.weight_support = []  # weight vector at which each CCS value vector was found
        self.iteration = 0
        self.ols_ended = False
        self.verbose = verbose
        self.queue = [(float("inf"), w) for w in extrema_weights(self.num_objectives)]

    def next_weight(self, algo: str = "ols", gpi_agent=None, env=None, rep_eval: int = 1) -> Optional[np.ndarray]:
        """The queued weight vector with the highest priority, or None once the queue is empty (``ended()`` is then True).

        algo: 'ols' or 'gpi-ls'; gpi_agent, env, rep_eval: the GPI agent, environment and episodes per weight of GPI-LS's priority."""
        if algo not in ("ols", "gpi-ls"):
            raise ValueError(f"Unknown algorithm {algo}.")
        if len(self.ccs) > 0:
            W_corner = self.compute_corner_weights()
            if self.verbose:
                print("W_corner:", W_corner, "W_corner size:", len(W_corner))
            gpi_expanded_set = None
            if algo == "gpi-ls" and len(W_corner) > 0:
                if gpi_agent is None:
                    raise ValueError("GPI-LS requires passing a GPI agent.")
                gpi_expanded_set = self._gpi_expanded_set(gpi_agent, env, W_corner, rep_eval)
            self.queue = []
            for wc in W_corner:
                priority = self.ols_priority(wc) if algo == "ols" else self.gpi_ls_priority(wc, gpi_expanded_set)
                if self.epsilon is None or priority >= self.epsilon:
                    # OLS does not try the same weight vector twice
                    if not (algo == "ols" and any(np.allclose(wc, wv) for wv in self.visited_weights)):
                        self.queue.append((priority, wc))
            if len(self.queue) > 0:
                self.queue.sort(key=lambda t: t[0], reverse=True)  # stable, descending
                if self.queue[0][0] == 0.0:  # every priority is 0: shuffle so that the same weights are not repeated
                    random.shuffle(self.queue)
        if self.verbose:
            print("CCS:", self.ccs, "CCS size:", len(self.ccs))
        if len(self.queue) == 0:
            if self.verbose:
                print("There are no corner weights in the queue. Returning None.")
            self.ols_ended = True
            return None
        next_w = self.queue.pop(0)[1]
        if self.verbose:
            print("Next weight:", next_w)
        return next_w

    @staticmethod
    def _gpi_expanded_set(gpi_agent, env, W_corner: List[np.ndarray], rep_eval: int) -> List[np.ndarray]:
        """Discounted vector return of the GPI agent at every corner weight: one lockstep round for all corners (float64 weights and
        accumulators, as the serial routine has for float64 weights), or the serial routine per corner without ``eval_batch``."""
        if hasattr(gpi_agent, "eval_batch"):
            return [r[3] for r in policy_evaluation_mo_batched(gpi_agent, env, W_corner, rep=rep_eval, weight_dtype=np.float64)]
        return [policy_evaluation_mo(gpi_agent, env, wc, rep=rep_eval)[3] for wc in W_corner]

    def get_weight_support(self) -> List[np.ndarray]:
        """The weight vectors of the CCS (a copy)."""
        return deepcopy(self.weight_support)

    def get_corner_weights(self, top_k: Optional[int] = None) -> List[np.ndarray]:
        """The queued corner weights in priority order (copies), the first ``top_k`` of them if given."""
        weights = [w.copy() for (_, w) in self.queue]
        return weights if top_k is None else weights[:top_k]

    def ended(self) -> bool:
        """True once ``next_weight`` found no corner weight to return (call it after ``next_weight``)."""
        return self.ols_ended

    def add_solution(self, value: np.ndarray, w: np.ndarray) -> List[int]:
        """Add the value vector found for weight ``w``; returns the indices of the CCS vectors removed (``[len(ccs)]`` when ``value``
        itself is dominated and discarded)."""
        if self.verbose:
            print(f"Adding value={value} for weight={w} to CCS.")
        self.iteration += 1
        self.visited_weights.append(w)
        if self.is_dominated(value):
            if self.verbose:
                print(f"Value {value} is dominated. Discarding.")
            return [len(self.ccs)]
        removed_indx = self.remove_obsolete_values(value)
        self.ccs.append(value)
        self.weight_support.append(w)
        return removed_indx

    def ols_priority(self, w: np.ndarray) -> float:
        """OLS priority: optimistic bound minus the best CCS value at ``w``."""
        return self.max_value_lp(w) - self.max_scalarized_value(w)

    def gpi_ls_priority(self, w: np.ndarray, gpi_expanded_set: List[np.ndarray]) -> float:
        """GPI-LS priority: best scalarised value of the expanded set at ``w`` (first vector reaching the maximum, strict >) minus the
        best CCS value at ``w``."""
        best = gpi_expanded_set[0]
        for v in gpi_expanded_set[1:]:
            if v @ w > best @ w:
                best = v
        return np.dot(best, w) - self.max_scalarized_value(w)

    def max_scalarized_value(self, w: np.ndarray) -> Optional[float]:
        """max_{v in CCS} v . w (None for an empty CCS)."""
        if len(self.ccs) == 0:
            return None
        return np.max([np.dot(v, w) for v in self.ccs])

    def remove_obsolete_values(self, value: np.ndarray) -> List[int]:
        """Remove the CCS vectors that are no longer optimal at any visited weight once ``value`` is added; returns their indices."""
        removed_indx = []
        for i in reversed(range(len(self.ccs))):
            still_optimal = any(np.dot(self.ccs[i], w) == self.max_scalarized_value(w) and np.dot(value, w) < np.dot(self.ccs[i], w)
                                for w in self.visited_weights)
            if not still_optimal:
                if self.verbose:
                    print("removed value", self.ccs[i])
                removed_indx.append(i)
                self.ccs.pop(i)
                self.weight_support.pop(i)
        return removed_indx

    def max_value_lp(self, w_new: np.ndarray) -> float:
        """Upper bound of max v . w_new over value vectors consistent with the visited weights: max w_new . v s.t. W v <= V (v free),
        V_i the best CCS value at visited weight W_i.  +inf with an empty CCS or an unbounded LP."""
        from scipy.optimize import linprog

        if len(self.ccs) == 0:
            return float("inf")
        W = np.vstack(self.visited_weights).astype(np.float64)
        V = np.array([self.max_scalarized_value(weight) for weight in self.visited_weights], dtype=np.float64)
        res = linprog(-np.asarray(w_new, dtype=np.float64), A_ub=W, b_ub=V, bounds=[(None, None)] * self.num_objectives, method="highs")
        if res.status == 3:
            return float("inf")
        if res.status != 0:
            raise RuntimeError(f"max_value_lp: linprog failed ({res.message})")
        return float(-res.fun)

    def compute_corner_weights(self) -> List[np.ndarray]:
        """Corner weights of the current CCS (Roijers, thesis Definition 19, with <= as the reference notes): the weight part of every
        vertex of { V w <= u, w >= 0, sum w = 1 } for the CCS rounded to 4 decimals, enumerated on the device, in canonical order."""
        A = np.round(np.vstack(self.ccs).astype(np.float64), decimals=4)
        verts = ops.corner_weights(th.from_numpy(A).to("cuda"))
        return list(canonical_corners(verts[:, :-1].cpu().numpy()))

    def is_dominated(self, value: np.ndarray) -> bool:
        """True iff ``value`` is below the best CCS value at every visited weight."""
        if len(self.ccs) == 0:
            return False
        for w in self.visited_weights:
            if np.dot(value, w) >= self.max_scalarized_value(w):
                return False
        return True
