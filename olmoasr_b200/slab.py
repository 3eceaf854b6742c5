"""Parameter slabs: the HBM layout of everything the optimizer step touches.

The reference keeps ~950 separately allocated fp32 parameters, lets autograd allocate ~950 gradients per step, lets DDP copy
them into 25 MB buckets (scripts/training/train_timestamps.py:2329-2330) and re-casts every weight to bf16 on every
forward (olmoasr/model.py:97-101).  Here the model's state lives in five contiguous slabs with ONE shared element
layout:

    P  fp32 master weights      (every nn.Parameter is a view into it; state_dict names / shapes are unchanged)
    G  fp32 gradients           (p.grad is a view; wgrad GEMM epilogues accumulate straight into it)
    M, V  fp32 AdamW moments    (optimizer state views, torch.optim.AdamW's names)
    S  16-bit shadow of P       (what the wgmma GEMMs read; rewritten by the AdamW kernel from registers).  It holds the
                                type the model last computed in: bf16, or fp16 under torch.autocast(float16)

so that the optimizer is three launches over flat memory, zero_grad is one memset, the bf16 weights cost no extra
pass, and a data-parallel gradient sum is a handful of large contiguous NCCL all-reduces (`SlabGradSync` in ddp.py)
issued in the order the backward completes them -- the layout order IS the backward order.

Elements are laid out by a `layout` (list of parameters and integer zero-gaps).  A model may ask for specific
adjacency (e.g. [Wq; Wk; Wv] contiguous so that the fused QKV weight is a plain view, or [bq; 0; bv] with a zero gap for
the bias-less key projection); gaps stay zero for ever (zero gradient, zero moments, decay of zero).
"""
from __future__ import annotations

from typing import Callable, Dict, Iterable, List, Optional, Sequence, Tuple, Union

import torch
from torch import Tensor, nn

ALIGN = 64  # elements: 256 B for fp32, 128 B for the bf16 shadow (TMA needs 16 B, vector loads 16 B)

LayoutItem = Union[nn.Parameter, int]


def default_layout(model: nn.Module) -> List[LayoutItem]:
    """Reverse registration order ~ the order in which a backward pass completes the gradients."""
    return list(reversed([p for p in model.parameters() if p.requires_grad]))


class ParamSlabs:
    def __init__(self, model: nn.Module, layout: Optional[Sequence[LayoutItem]] = None, *, shadows: bool = True,
                 extra_sync: Optional[Callable[[], None]] = None):
        items = list(layout) if layout is not None else default_layout(model)
        params = [it for it in items if not isinstance(it, int)]
        want = [p for p in model.parameters() if p.requires_grad]
        if {id(p) for p in params} != {id(p) for p in want} or len(params) != len(want):
            raise ValueError("slab layout must contain every trainable parameter exactly once")
        dev = params[0].device
        for p in params:
            if p.dtype != torch.float32 or p.device != dev:
                raise ValueError("ParamSlabs: fp32 parameters on one device only")
        self.model = model
        self.device = dev
        self.params: List[nn.Parameter] = params
        self.offset: Dict[int, int] = {}
        off = 0
        for it in items:
            if isinstance(it, int):
                off += it
                continue
            self.offset[id(it)] = off
            off += it.numel()
            off = (off + ALIGN - 1) // ALIGN * ALIGN
        self.numel = off
        self.P = torch.zeros(off, device=dev, dtype=torch.float32)
        self.G = torch.zeros(off, device=dev, dtype=torch.float32)
        self.S = torch.zeros(off, device=dev, dtype=torch.bfloat16) if shadows else None
        self.S_dtype = torch.bfloat16   # what S holds; S itself stays a bf16 tensor and is read as S_dtype (same size)
        self.M: Optional[Tensor] = None     # allocated by the optimizer (FusedAdamW) on first use
        self.V: Optional[Tensor] = None
        with torch.no_grad():
            for p in params:
                o, n = self.offset[id(p)], p.numel()
                self.P[o:o + n].copy_(p.detach().reshape(-1))
                p.data = self.P[o:o + n].view(p.shape)           # the Parameter object (and its name) stays; storage moves
                p.grad = self.G[o:o + n].view(p.shape)
        self.direct_grads = False   # True: the model's backward kernels accumulate into G themselves (no autograd hand-over)
        self._extra_sync = extra_sync
        self._synced_sig = None
        self.layout_order = [id(p) for p in params]

    # ---- views ------------------------------------------------------------------------------------------
    def span(self, kind: str, first: nn.Parameter, numel: int) -> Tensor:
        """1-D view of `numel` elements starting at `first`'s slot in slab `kind` ("P", "G", "S", "M", "V")."""
        slab = getattr(self, kind)
        o = self.offset[id(first)]
        if o + numel > self.numel:
            raise ValueError("span runs past the slab")
        return slab[o:o + numel]

    def adjacent(self, *ps: nn.Parameter) -> bool:
        """True when the parameters occupy consecutive elements (no alignment padding in between)."""
        return all(self.offset[id(b)] == self.offset[id(a)] + a.numel() for a, b in zip(ps, ps[1:]))

    def shadow(self, p: nn.Parameter) -> Tensor:
        return self.span("S", p, p.numel()).view(p.shape)

    def grad(self, p: nn.Parameter) -> Tensor:
        return self.span("G", p, p.numel()).view(p.shape)

    def range_of(self, ps: Iterable[nn.Parameter]) -> Tuple[int, int]:
        """[start, end) element range covering the given parameters (they should be contiguous in the layout)."""
        offs = [(self.offset[id(p)], p.numel()) for p in ps]
        start = min(o for o, _ in offs)
        end = max(o + n for o, n in offs)
        return start, (end + ALIGN - 1) // ALIGN * ALIGN

    # ---- gradients ---------------------------------------------------------------------------------------
    def zero_grad(self):
        """One memset for the whole model; re-attaches p.grad views (zero_grad(set_to_none=True) elsewhere drops them)."""
        self.G.zero_()
        for p in self.params:
            g = p.grad
            o = self.offset[id(p)]
            if g is None or g.data_ptr() != self.G.data_ptr() + 4 * o:
                p.grad = self.G[o:o + p.numel()].view(p.shape)

    # ---- 16-bit shadows ----------------------------------------------------------------------------------
    def _signature(self):
        return tuple(p._version for p in self.params)

    def shadow_slab(self) -> Optional[Tensor]:
        """S read as the type it holds."""
        return None if self.S is None else (self.S if self.S_dtype == torch.bfloat16 else self.S.view(self.S_dtype))

    def sync_shadows(self):
        """S <- S_dtype(P) in one flat cast (+ the model's non-elementwise shadows).  Needed after anything other than the
        fused optimizer changed the masters (initialisation, load_state_dict, a foreign optimizer)."""
        if self.S is not None:
            from . import kernels as K
            if self.S_dtype == torch.bfloat16:
                K.cast_bf16(self.P, self.S)
            else:
                K.convert(self.P, self.shadow_slab())
        if self._extra_sync is not None:
            self._extra_sync()
        self._synced_sig = self._signature()

    def ensure_synced(self, dtype: torch.dtype = torch.bfloat16):
        """Make S current, in `dtype` (the type of the forward about to run): a change of type re-casts it, e.g. an fp16
        training step followed by a bf16 evaluation."""
        if self.S is not None and dtype != self.S_dtype:
            self.S_dtype = dtype
            self._synced_sig = None
        if self._synced_sig != self._signature():
            self.sync_shadows()

    def mark_synced(self):
        """Called by the fused optimizer after a step whose kernel refreshed S itself."""
        if self._extra_sync is not None:
            self._extra_sync()
        self._synced_sig = self._signature()

    def invalidate(self):
        """Masters were changed behind autograd's back (e.g. a broadcast into p.data): force a re-cast."""
        self._synced_sig = None
