"""Low-rank adapters (LoRA) on the projections of the fused blocks.

    add_lora(model, r, alpha, targets)   registers lora_A (r, in) / lora_B (out, r) on every targeted Linear and freezes
                                         every other parameter
    merge_lora(model)                    folds s B A into the fp32 weights and removes the adapters

An adapted Linear computes y = x W^T + b + s (x A^T) B^T with s = alpha / r.  The low-rank product never makes a pass of
its own over the activations: the projection GEMM accumulates it as extra k-blocks of its mainloop (oasr_gemm_lowrank16),
so the bias / GELU / residual epilogues apply to the sum unchanged, and with B = 0 (its initial value) the outputs are
bit-identical to the model without adapters.  The training backward gives dA = s (dy B)^T x and dB = s dy^T (x A^T)
from the wgrad GEMMs, and no gradient work at all for frozen parameters.  state_dict() holds the reference's keys plus
`<linear>.lora_A` / `.lora_B`; after merge_lora it holds exactly the reference's keys.
"""
from __future__ import annotations

import math
from typing import Iterable, List, Tuple

import torch
from torch import nn

from . import kernels as K
from ._core import Linear, OLMoASRBase

DEFAULT_TARGETS = ("encoder.attn.query", "encoder.attn.value", "decoder.attn.query", "decoder.attn.value")
_NAMES = ("attn.query", "attn.key", "attn.value", "attn.out", "cross_attn.query", "cross_attn.key", "cross_attn.value",
          "cross_attn.out", "mlp.0", "mlp.2")
MAX_RANK_PER_SITE = 192   # K2 limit of the GEMM's low-rank tail; a fused q / k / v or k / v site stacks its members' ranks


def _blocks(model: OLMoASRBase, stack: str):
    return list((model.encoder if stack == "encoder" else model.decoder).blocks)


def _linear(block: nn.Module, name: str) -> Linear:
    obj = block
    for part in name.split("."):
        obj = obj[int(part)] if part.isdigit() else getattr(obj, part)
    return obj


def _adapted(model: OLMoASRBase) -> List[Tuple[nn.Module, Linear]]:
    return [(b, m) for stack in ("encoder", "decoder") for b in _blocks(model, stack) for m in b.modules()
            if isinstance(m, Linear) and m.has_lora]


def _refresh_blocks(model: OLMoASRBase):
    for stack in ("encoder", "decoder"):
        for b in _blocks(model, stack):
            b._param_names = [n for n, _ in b.named_parameters()]
            b._lora_on = any(isinstance(m, Linear) and m.has_lora for m in b.modules())
            b._lora_cache = {}


def add_lora(model: OLMoASRBase, r: int, alpha: float, targets: Iterable[str] = DEFAULT_TARGETS) -> OLMoASRBase:
    """Register a rank-`r` adapter with scale alpha / r on every Linear named by `targets` and freeze every other
    parameter (re-enable any of them with requires_grad_(True); the fused training path honours it per parameter).

    A target is "<encoder|decoder>.<name>", name one of attn.{query,key,value,out}, cross_attn.{query,key,value,out}
    (decoder only), mlp.0 or mlp.2; it applies to every block of that stack.  lora_A is drawn like PEFT
    (kaiming_uniform_(a=sqrt(5))) and lora_B starts at zero.  Call it before use_slabs(), on an unwrapped model."""
    from torch.distributed.fsdp import FullyShardedDataParallel

    if not isinstance(model, OLMoASRBase):
        raise TypeError("add_lora takes an OLMoASR model (not a DDP / FSDP wrapper)")
    if any(isinstance(m, FullyShardedDataParallel) for m in model.modules()):
        raise ValueError("add_lora: adapters are not supported under FSDP")
    if any(p.dtype != torch.float32 for p in model.parameters()):
        raise ValueError("add_lora: the model's parameters must be fp32 masters (the 16-bit compute types are chosen per "
                         "call, e.g. by torch.autocast)")
    if getattr(model, "_slabs", None) is not None:
        raise ValueError("add_lora must be called before use_slabs(): the slabs are laid out once")
    if _adapted(model):
        raise ValueError("add_lora: the model already has adapters (merge_lora() them first)")
    r = int(r)
    if r < 8 or r % 8 or r > MAX_RANK_PER_SITE:
        raise ValueError(f"add_lora: r must be a multiple of 8 in [8, {MAX_RANK_PER_SITE}] (16-byte rows of the GEMM's "
                         f"tail, whose rank is at most {MAX_RANK_PER_SITE}), got {r}")
    targets = list(targets)
    if not targets:
        raise ValueError("add_lora: no targets")
    chosen = []
    for t in targets:
        stack, _, name = t.partition(".")
        if stack not in ("encoder", "decoder") or name not in _NAMES:
            raise ValueError(f"add_lora: bad target {t!r}; expected <encoder|decoder>.<{'|'.join(_NAMES)}>")
        if stack == "encoder" and name.startswith("cross_attn."):
            raise ValueError(f"add_lora: the encoder has no cross-attention ({t!r})")
        if (stack, name) not in chosen:
            chosen.append((stack, name))
    for stack in ("encoder", "decoder"):
        for group in (("attn.query", "attn.key", "attn.value"), ("cross_attn.key", "cross_attn.value")):
            if r * sum((stack, n) in chosen for n in group) > MAX_RANK_PER_SITE:
                raise ValueError(f"add_lora: {stack} {'/'.join(group)} share one GEMM whose tail takes a total rank of at "
                                 f"most {MAX_RANK_PER_SITE}; r = {r} on all of them is too large")
    model._lora_frozen_before = {n for n, p in model.named_parameters() if not p.requires_grad}   # merge_lora restores it
    for p in model.parameters():
        p.requires_grad_(False)
    for stack, name in chosen:
        for b in _blocks(model, stack):
            lin = _linear(b, name)
            w = lin.weight
            lin.lora_A = nn.Parameter(torch.empty((r, lin.in_features), device=w.device, dtype=torch.float32))
            nn.init.kaiming_uniform_(lin.lora_A, a=math.sqrt(5))
            lin.lora_B = nn.Parameter(torch.zeros((lin.out_features, r), device=w.device, dtype=torch.float32))
            lin.lora_scale = float(alpha) / r
    _refresh_blocks(model)
    return model


@torch.no_grad()
def merge_lora(model: OLMoASRBase) -> OLMoASRBase:
    """Fold s B A into every adapted Linear's fp32 weight (W <- W + s B A on the device) and remove the adapters.  The
    model then has exactly the reference's parameters (state_dict keys and shapes), with the requires_grad flags they
    had before add_lora."""
    if getattr(model, "_slabs", None) is not None:
        raise ValueError("merge_lora: the model's parameters live in slabs; merge an unslabbed copy (load its state_dict)")
    for _, lin in _adapted(model):
        merged = K.lora_merge(lin.weight.detach().contiguous(), lin.lora_B.detach().contiguous(),
                              lin.lora_A.detach().contiguous(), lin.lora_scale)
        lin.weight.copy_(merged)
        del lin.lora_A
        del lin.lora_B
        lin.lora_scale = 0.0
        lin.__dict__.pop("_lora_shadow", None)
    frozen = model.__dict__.pop("_lora_frozen_before", set())
    for n, p in model.named_parameters():
        p.requires_grad_(n not in frozen)
    _refresh_blocks(model)
    return model


def effective_weight(lin: Linear) -> torch.Tensor:
    """fp32 W + s B A of an adapted Linear (its weight itself without an adapter), computed on the device."""
    if not lin.has_lora:
        return lin.weight.detach()
    return K.lora_merge(lin.weight.detach().contiguous(), lin.lora_B.detach().contiguous(), lin.lora_A.detach().contiguous(),
                        lin.lora_scale)
