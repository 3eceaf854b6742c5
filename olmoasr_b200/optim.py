"""Fused AdamW with global-norm clipping (the optimizer step right after the hot path:
scripts/training/train_timestamps.py:1508-1522, defaults :2110-2116).  Three kernel launches per step for the whole
model; state (`exp_avg`, `exp_avg_sq`, `step`) uses torch.optim.AdamW's names so `state_dict()` round-trips with the
reference's `optimizer_state_dict` checkpoints (train_timestamps.py:930-955).

Two storage forms:
  * `FusedAdamW(model.parameters())` -- any fp32 parameters; a device table of pointers drives the kernels.  After the
    step every parameter's autograd version is bumped, so the model's bf16 weight shadows are re-cast lazily.
  * `FusedAdamW(model.parameters(), slabs=model.use_slabs())` -- parameters, gradients and moments are contiguous slabs
    (olmoasr_b200/slab.py): no table, and the update kernel writes the bf16 shadows the GEMMs read.

The step counter lives on the device and only advances when an update is applied (a non-finite gradient norm skips the
step, as GradScaler + AdamW do); `state[p]["step"]` is refreshed from it when `state_dict()` is taken.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from ._lib import DTYPE_F16 as _DTYPE_F16, call, lib, ptr, stream


def _f32_scalar(t):
    """One fp32 element on the device (GradScaler's scale and found_inf are fp32; None passes through)."""
    if t is None or t.dtype == torch.float32:
        return t
    return t.float()


class FusedAdamW(torch.optim.Optimizer):
    # torch.amp.GradScaler.step hands a scaling-aware optimizer its loss scale and found-inf flag as the device tensors
    # `grad_scale` / `found_inf` instead of unscaling the gradients and reading the flag on the host
    _step_supports_amp_scaling = True

    def __init__(self, params, lr=1.5e-3, betas=(0.9, 0.98), eps=1e-6, weight_decay=0.1, max_grad_norm=1.0, slabs=None):
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay)
        super().__init__(params, defaults)
        if len(self.param_groups) != 1:
            raise ValueError("FusedAdamW: one param group (the reference uses one: train_timestamps.py:706-735)")
        self.max_grad_norm = max_grad_norm
        self.slabs = slabs
        self._built = False

    # ---- state ------------------------------------------------------------------------------------------
    def _params(self):
        return [p for p in self.param_groups[0]["params"] if p.requires_grad]

    def _build(self):
        ps = self._params()
        dev = ps[0].device
        self._dev_state = torch.zeros(8, device=dev, dtype=torch.float32)   # see oasr_optim_prepare
        self._norm_sq = torch.zeros(1, device=dev, dtype=torch.float32)
        self._found_inf = torch.zeros(1, device=dev, dtype=torch.float32)
        first = next((self.state[p] for p in ps if "step" in self.state[p]), None)
        if first is not None:   # resumed from a state_dict
            self._dev_state[0] = float(first["step"])
        sl = self.slabs
        if sl is not None:
            if {id(p) for p in ps} != set(sl.layout_order):
                raise ValueError("FusedAdamW(slabs=...): the optimizer must own exactly the slab's parameters")
            old = {id(p): self.state[p] for p in ps if "exp_avg" in self.state[p]}
            sl.M = torch.zeros_like(sl.P)
            sl.V = torch.zeros_like(sl.P)
            for p in ps:
                st = self.state[p]
                m, v = sl.span("M", p, p.numel()).view(p.shape), sl.span("V", p, p.numel()).view(p.shape)
                if id(p) in old:
                    m.copy_(old[id(p)]["exp_avg"]); v.copy_(old[id(p)]["exp_avg_sq"])
                st["exp_avg"], st["exp_avg_sq"] = m, v
                st.setdefault("step", torch.tensor(0.0))
        else:
            chunk = lib().oasr_optim_chunk_elems()
            recs = np.zeros((len(ps), 6), dtype=np.int64)
            chunks = []
            for i, p in enumerate(ps):
                if p.dtype != torch.float32 or not p.is_contiguous():
                    raise ValueError("FusedAdamW: fp32 contiguous parameters only")
                st = self.state[p]
                if "exp_avg" not in st:
                    st["step"] = torch.tensor(0.0)
                    st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                recs[i] = (p.data_ptr(), 0, st["exp_avg"].data_ptr(), st["exp_avg_sq"].data_ptr(), p.numel(), 0)
                chunks += [(i, c) for c in range(math.ceil(p.numel() / chunk))]
            # two pinned copies of the pointer table: the H2D copy of step N reads its buffer when it EXECUTES, possibly
            # after the host has already started writing step N+1's gradient pointers
            self._host = [torch.from_numpy(recs.copy()).pin_memory() for _ in range(2)]
            self._host_ev = [None, None]
            self._flip = 0
            self._dev_tab = torch.empty((len(ps), 6), dtype=torch.int64, device=dev)
            self._last_grad_ptrs = None
            self._chunks = torch.tensor(chunks, dtype=torch.int32, device=dev)
            self._n_chunks = len(chunks)
        self._built = True

    # ---- step -------------------------------------------------------------------------------------------
    @torch.no_grad()
    def step(self, closure=None, inv_scale: float = 1.0):
        """`inv_scale` multiplies every gradient before clipping: 1 / loss_scale (GradScaler.unscale_) and / or
        1 / world_size when the gradients were summed, not averaged, across ranks (olmoasr_b200.ddp).

        Under `scaler.step(opt)` GradScaler sets `self.grad_scale` (its scale S, or None when `scaler.unscale_(opt)` already
        ran) and `self.found_inf` (device tensors): the gradients are then also multiplied by 1 / S and the update is skipped,
        and not counted, when found_inf is set or the norm is not finite -- decided on the device, so the step never waits
        for the host."""
        if closure is not None:
            raise ValueError("FusedAdamW does not take a closure")
        if not self._built:
            self._build()
        group = self.param_groups[0]
        b1, b2 = group["betas"]
        s = stream()
        sl = self.slabs
        if sl is not None:
            call("oasr_grad_sqnorm_flat", ptr(sl.G), sl.numel, float(inv_scale), ptr(self._norm_sq), s)
        else:
            self._upload_grad_pointers()
            call("oasr_grad_sqnorm", ptr(self._dev_tab), ptr(self._chunks), self._n_chunks, float(inv_scale), ptr(self._norm_sq), s)
        # instance attributes set by GradScaler.step (found_inf also names a method of this class)
        grad_scale, found_inf = self.__dict__.get("grad_scale"), self.__dict__.get("found_inf")
        if grad_scale is None and found_inf is None:
            call("oasr_optim_prepare", ptr(self._norm_sq), ptr(self._found_inf), ptr(self._dev_state), float(inv_scale),
                 float(self.max_grad_norm or 0.0), b1, b2, s)
        else:
            call("oasr_optim_prepare_amp", ptr(self._norm_sq), ptr(self._found_inf), ptr(self._dev_state),
                 ptr(_f32_scalar(grad_scale)), ptr(_f32_scalar(found_inf)), float(inv_scale), float(self.max_grad_norm or 0.0),
                 b1, b2, s)
        if sl is not None and sl.S_dtype != torch.bfloat16:
            call("oasr_adamw_flat16", ptr(sl.P), ptr(sl.G), ptr(sl.M), ptr(sl.V), ptr(sl.S), sl.numel, ptr(self._dev_state),
                 float(group["lr"]), b1, b2, group["eps"], group["weight_decay"], _DTYPE_F16, s)
        elif sl is not None:
            call("oasr_adamw_flat", ptr(sl.P), ptr(sl.G), ptr(sl.M), ptr(sl.V), ptr(sl.S), sl.numel, ptr(self._dev_state),
                 float(group["lr"]), b1, b2, group["eps"], group["weight_decay"], s)
        else:
            call("oasr_adamw_step", ptr(self._dev_tab), ptr(self._chunks), self._n_chunks, ptr(self._dev_state),
                 float(group["lr"]), b1, b2, group["eps"], group["weight_decay"], s)
        # the kernels wrote through raw pointers: tell autograd (and every version-keyed cache, e.g. the bf16 weight
        # shadows of olmoasr_b200._core) that the parameters changed
        ps = self._params()
        torch.autograd.graph.increment_version(ps)
        if sl is not None:
            sl.mark_synced()    # S was refreshed by the update kernel itself
        return None

    def _upload_grad_pointers(self):
        ps = self._params()
        ptrs = []
        for p in ps:
            g = p.grad
            if g is None or g.dtype != torch.float32:
                raise ValueError("FusedAdamW: every parameter needs an fp32 grad")
            if not g.is_contiguous():
                g = p.grad = g.contiguous()
            ptrs.append(g.data_ptr())
        if ptrs == self._last_grad_ptrs:
            return                                   # stable gradient storage: nothing to upload
        k = self._flip
        self._flip ^= 1
        if self._host_ev[k] is not None:
            self._host_ev[k].synchronize()           # the copy that last read this pinned buffer has executed
        host = self._host[k]
        host[:, 1] = torch.tensor(ptrs, dtype=torch.int64)
        self._dev_tab.copy_(host, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._host_ev[k] = ev
        self._last_grad_ptrs = ptrs

    # ---- introspection ------------------------------------------------------------------------------------
    def zero_grad(self, set_to_none: bool = True):
        if self.slabs is not None:
            self.slabs.zero_grad()
        else:
            super().zero_grad(set_to_none=set_to_none)

    def grad_norm(self) -> torch.Tensor:
        """Global L2 norm of the last step's unscaled gradients (before clipping), on the device."""
        return self._dev_state[5]

    def found_inf(self) -> torch.Tensor:
        return self._found_inf

    def applied_steps(self) -> int:
        """Number of updates actually applied (synchronises)."""
        return int(self._dev_state[0].item()) if self._built else 0

    def state_dict(self):
        if self._built:
            step = torch.tensor(float(self.applied_steps()))
            for p in self._params():
                self.state[p]["step"] = step
        return super().state_dict()

    def load_state_dict(self, state_dict):
        super().load_state_dict(state_dict)
        self._built = False     # moments are re-homed (slab views / pointer table) on the next step
