"""Adam with gradient clipping as two CUDA launches (morl_adam_clip_f32) instead of ~25 foreach / elementwise kernels.

``FusedClipAdam`` IS a ``torch.optim.Adam`` (same param groups, same ``state_dict`` layout: per-parameter ``step`` (float32
device scalar), ``exp_avg``, ``exp_avg_sq``), so checkpoints interchange with the reference's optimiser state
(reference multi_policy/envelope/envelope.py:183, 240-247).  ``step_fused(max_grad_norm)`` performs
``clip_grad_norm_(params, max_grad_norm)`` + ``step()`` (reference envelope.py:324-326) with the arithmetic of the reference's
non-capturable single-tensor Adam.  Parameter gradients must already be populated; under CUDA-graph replay they keep their storage,
in eager mode the single pointer table is refreshed in place when a gradient tensor moved (no per-step allocation, nothing retained)."""

from __future__ import annotations

from typing import Optional

import torch as th
from torch import optim

from .. import _lib, ops


class FusedClipAdam(optim.Adam):
    def __init__(self, params, lr: float = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8):
        super().__init__(params, lr=lr, betas=betas, eps=eps, capturable=True)
        self._tables = None
        self._cache = {}   # tables referenced by captured CUDA graphs (one per capture)
        self._eager = None  # the single overwritable table of the eager path
        # optional float64 device scalar: when set, step_fused reads the learning rate from it at run time instead of from param_groups,
        # so a captured graph follows a schedule written into it
        self.lr_device: Optional[th.Tensor] = None

    def load_state_dict(self, state_dict):
        """``optim.Adam.load_state_dict`` replaces the state tensors: the cached pointer tables (which hold their addresses) are dropped."""
        super().load_state_dict(state_dict)
        self._tables, self._cache, self._eager = None, {}, None

    def _ensure_state(self):
        for group in self.param_groups:
            for p in group["params"]:
                st = self.state[p]
                if len(st) == 0:
                    st["step"] = th.zeros((), dtype=th.float32, device=p.device)
                    st["exp_avg"] = th.zeros_like(p, memory_format=th.preserve_format)
                    st["exp_avg_sq"] = th.zeros_like(p, memory_format=th.preserve_format)

    def _build_tables(self, params):
        """Device-side pointer tables for one set of gradient buffers, written through PINNED staging + an async copy so that it is legal
        inside a CUDA-graph capture (the copy becomes a graph node that re-writes the same pointers on every replay).

        Lifetime rules (ADVICE r1: the per-pointer cache used to grow without bound in eager mode):
          * while a graph is being CAPTURED the table is cached per gradient-pointer tuple and keeps the gradient tensors alive, because
            the captured graph keeps referencing both;
          * in eager mode ONE table (pinned staging, device copy, workspace) is allocated once and overwritten in place whenever a gradient
            tensor moved (``zero_grad(set_to_none=True)`` callers); nothing is retained, so memory stays flat however long the run is."""
        dev = params[0].device
        grads = [p.grad for p in params]
        key = tuple(g.data_ptr() for g in grads)
        capturing = th.cuda.is_current_stream_capturing()
        if capturing and key in self._cache:
            self._tables = self._cache[key]
            return
        lists = {
            "p": [t.data_ptr() for t in params], "g": list(key), "m": [self.state[p]["exp_avg"].data_ptr() for p in params],
            "v": [self.state[p]["exp_avg_sq"].data_ptr() for p in params], "s": [self.state[p]["step"].data_ptr() for p in params],
            "n": [p.numel() for p in params],
        }
        rows = th.tensor([lists[k] for k in ("p", "g", "m", "v", "s", "n")], dtype=th.int64)
        eager = None if capturing else self._eager
        if eager is not None and eager["pinned"].shape == rows.shape and eager["table"].device == dev:
            eager["copied"].synchronize()  # the previous refresh of the staging buffer has been consumed
            pinned, table, ws = eager["pinned"], eager["table"], eager["ws"]
            pinned.copy_(rows)
        else:
            pinned = rows.pin_memory()
            table = th.empty_like(pinned, device=dev)
            ws = None
        table.copy_(pinned, non_blocking=True)
        t = {k: table[i] for i, k in enumerate(("p", "g", "m", "v", "s", "n"))}
        t["max"] = max(lists["n"])
        t["key"] = key
        nbytes = _lib.load().morl_adam_workspace_bytes(len(params), t["max"])
        if ws is None or ws.numel() * 4 < nbytes:
            ws = th.empty((nbytes + 3) // 4, dtype=th.float32, device=dev)
        t["ws"] = ws
        if capturing:
            t["keep"] = (params, grads, pinned, table)
            self._cache[key] = t
        else:
            ev = eager["copied"] if eager is not None else th.cuda.Event()
            ev.record()
            self._eager = {"pinned": pinned, "table": table, "ws": ws, "copied": ev}
        self._tables = t

    @th.no_grad()
    def step_fused(self, max_grad_norm: Optional[float] = None):
        assert len(self.param_groups) == 1, "FusedClipAdam.step_fused supports a single parameter group"
        group = self.param_groups[0]
        params = [p for p in group["params"] if p.grad is not None]
        if not params:
            return
        if any(not (p.is_cuda and p.dtype == th.float32 and p.is_contiguous() and p.grad.is_contiguous()) for p in params):
            raise _lib.MorlB200Error("FusedClipAdam: parameters and gradients must be contiguous float32 CUDA tensors")
        self._ensure_state()
        # (a table a captured graph will keep reading must be a cached, never-overwritten one -- not the eager scratch table)
        if (self._tables is None or self._tables["key"] != tuple(p.grad.data_ptr() for p in params)
                or (th.cuda.is_current_stream_capturing() and "keep" not in self._tables)):
            self._build_tables(params)
        t = self._tables
        b1, b2 = group["betas"]
        if self.lr_device is not None:
            if not (self.lr_device.is_cuda and self.lr_device.dtype == th.float64 and self.lr_device.numel() == 1):
                raise _lib.MorlB200Error("FusedClipAdam.lr_device must be a float64 CUDA tensor with one element")
            rc = _lib.load().morl_adam_clip_lr_f32(t["p"].data_ptr(), t["g"].data_ptr(), t["m"].data_ptr(), t["v"].data_ptr(), t["s"].data_ptr(),
                                                   t["n"].data_ptr(), len(params), t["max"],
                                                   float(max_grad_norm) if max_grad_norm is not None else 0.0, self.lr_device.data_ptr(),
                                                   float(b1), float(b2), float(group["eps"]), t["ws"].data_ptr(), th.cuda.current_stream().cuda_stream)
            _lib.check(rc, "morl_adam_clip_lr_f32")
            ops._count(2)
            return
        rc = _lib.load().morl_adam_clip_f32(t["p"].data_ptr(), t["g"].data_ptr(), t["m"].data_ptr(), t["v"].data_ptr(), t["s"].data_ptr(),
                                            t["n"].data_ptr(), len(params), t["max"], float(max_grad_norm) if max_grad_norm is not None else 0.0,
                                            float(group["lr"]), float(b1), float(b2), float(group["eps"]), t["ws"].data_ptr(),
                                            th.cuda.current_stream().cuda_stream)
        _lib.check(rc, "morl_adam_clip_f32")
        ops._count(2)
