"""Block-wise gradient all-reduce: a leaner stand-in for DistributedDataParallel on this path (opt-in).

The reference wraps the model in `DDP(model, device_ids=[rank])` (scripts/training/train_timestamps.py:2329-2330): 25 MB
buckets, one flatten-copy and one divide kernel per parameter (946 + 948 launches per step at medium) and 87 all-reduce launches wherever a bucket happens to fill.  Here the
gradients stay where the backward kernels wrote them: when the last parameter of a ResidualAttentionBlock has its
gradient, the block's tensors are summed across ranks by ONE coalesced NCCL call (ncclGroupStart / ncclAllReduce per
tensor / ncclGroupEnd -- no flattening), and the 1 / world_size average is folded into the fused optimizer's
`inv_scale` (the clip threshold then applies to the averaged gradient norm, exactly like clip_grad_norm_ after DDP).

    reducer = BlockwiseGradReducer(model)          # after torch.distributed.init_process_group
    loss.backward()
    opt.step(inv_scale=reducer.finish())           # waits for the collectives; returns 1 / world_size

Same collective order on every rank (the autograd graph is the same), same result as DDP up to fp32 summation order.

`SlabGradSync` (below) is the preferred form and what bench.py uses: gradients already live in ONE flat fp32 slab in
backward-completion order (olmoasr_b200/slab.py), so the sum across ranks is a handful of large contiguous all-reduces
-- NCCL's bandwidth regime over NVLink 5 / NVSwitch instead of 87 latency-protocol bucket launches -- issued as soon as
the backward has finished a slab range, with no flatten copies and no per-parameter divides.
"""
from __future__ import annotations

from typing import Iterable, List, Optional, Sequence

import torch
import torch.distributed as dist
from torch import nn


def default_buckets(model: nn.Module) -> List[List[nn.Parameter]]:
    """One bucket per module that owns a `_param_names` list (the fused ResidualAttentionBlocks), one for the rest."""
    seen, buckets = set(), []
    for m in model.modules():
        if hasattr(m, "_param_names") and hasattr(m, "attn"):
            ps = [p for p in m.parameters() if p.requires_grad and id(p) not in seen]
            if ps:
                buckets.append(ps)
                seen.update(id(p) for p in ps)
    rest = [p for p in model.parameters() if p.requires_grad and id(p) not in seen]
    if rest:
        buckets.append(rest)
    return buckets


class BlockwiseGradReducer:
    def __init__(self, model: nn.Module, process_group=None, buckets: Optional[Sequence[Iterable[nn.Parameter]]] = None,
                 coalesce: bool = True):
        if not dist.is_initialized():
            raise RuntimeError("BlockwiseGradReducer needs an initialised process group")
        self.group = process_group
        # torch.distributed._coalescing_manager is a private API: without it every tensor gets its own async all-reduce
        self.coalesce = coalesce and hasattr(dist, "_coalescing_manager")
        self.world = dist.get_world_size(process_group)
        self.buckets = [list(b) for b in (buckets if buckets is not None else default_buckets(model))]
        self._left = [len(b) for b in self.buckets]
        self._launched = [False] * len(self.buckets)
        self._works = []
        self._hooks = []
        for i, b in enumerate(self.buckets):
            for p in b:
                self._hooks.append(p.register_post_accumulate_grad_hook(self._make_hook(i)))
        # every rank must start from the same weights, as DDP's constructor guarantees
        with torch.no_grad():
            for p in model.parameters():
                dist.broadcast(p.data, src=dist.get_global_rank(process_group, 0) if process_group is not None else 0,
                               group=process_group)
            for b in model.buffers():
                dist.broadcast(b.data, src=dist.get_global_rank(process_group, 0) if process_group is not None else 0,
                               group=process_group)

    def _make_hook(self, i: int):
        def hook(_param):
            self._left[i] -= 1
            if self._left[i] == 0:
                self._launch(i)
        return hook

    def _launch(self, i: int):
        grads = [p.grad for p in self.buckets[i] if p.grad is not None]
        self._launched[i] = True
        if not grads or self.world == 1:
            return
        if self.coalesce:
            with dist._coalescing_manager(group=self.group, async_ops=True) as cm:
                for g in grads:
                    dist.all_reduce(g, op=dist.ReduceOp.SUM, group=self.group)
            self._works.append(cm)
        else:
            self._works.extend(dist.all_reduce(g, op=dist.ReduceOp.SUM, group=self.group, async_op=True) for g in grads)

    def finish(self) -> float:
        """Launch whatever did not complete through the hooks (parameters without a gradient this step), wait for every
        collective in the order it was issued, re-arm, and return the factor that turns the sums into averages."""
        for i in range(len(self.buckets)):
            if not self._launched[i]:
                self._launch(i)
        for w in self._works:
            w.wait()
        self._works.clear()
        self._left = [len(b) for b in self.buckets]
        self._launched = [False] * len(self.buckets)
        return 1.0 / self.world

    def remove(self):
        for h in self._hooks:
            h.remove()
        self._hooks.clear()


class SlabGradSync:
    """Data-parallel gradient sum over a model in slab mode (`model.use_slabs()`): replaces
    `DDP(model, device_ids=[rank])` of scripts/training/train_timestamps.py:2329-2330.

        slabs = model.use_slabs()
        sync = SlabGradSync(model, slabs)              # broadcasts rank 0's weights, like DDP's constructor
        opt = FusedAdamW(model.parameters(), slabs=slabs)
        loss = model(mel, tokens, mask, targets=y); opt.zero_grad(); loss.backward()
        opt.step(inv_scale=sync.finish())              # SUM across ranks, 1 / world folded into the fused optimizer

    The slab is cut into segments of >= `bucket_bytes` at module boundaries (`model.grad_units()`); a segment's all-reduce
    is launched from the backward pass the moment its last producer (a fused block, the embedding, the conv stem) has
    enqueued its kernels, on NCCL's own stream, so it overlaps the rest of the backward.  The last `tail_bytes` of the slab
    (the gradients the backward finishes last) are cut finer, into `tail_bucket_bytes` pieces: whatever is still in flight
    when the backward ends is exposed, so the final collectives must be short (measured at 8 GPUs: the 256 MB tail segment
    cost ~8 ms of a 212 ms step).  Semantics are DDP's: every
    rank ends with the same SUM, the caller's optimizer divides by world (per-rank mean loss, gradient averaged over
    ranks -- train_timestamps.py:1444-1450 + DDP).  Models without `grad_units()` get one all-reduce in finish()."""

    def __init__(self, model: nn.Module, slabs, process_group=None, bucket_bytes: int = 256 << 20, broadcast: bool = True,
                 tail_bytes: int = 256 << 20, tail_bucket_bytes: int = 32 << 20):
        if not dist.is_initialized():
            raise RuntimeError("SlabGradSync needs an initialised process group")
        self.group = process_group
        self.world = dist.get_world_size(process_group)
        self.slabs = slabs
        self.enabled = True
        slabs.direct_grads = True
        units = model.grad_units() if hasattr(model, "grad_units") else [(list(slabs.params), None)]
        order = {pid: i for i, pid in enumerate(slabs.layout_order)}
        nxt = 0
        for ps, _ in units:     # every unit must be a contiguous run of the slab layout, units in layout order
            idx = sorted(order[id(p)] for p in ps)
            if idx != list(range(nxt, nxt + len(ps))):
                raise ValueError("grad_units() must partition the slab layout into consecutive runs, in layout order")
            nxt += len(ps)
        if nxt != len(order):
            raise ValueError("grad_units() must cover every slab parameter")
        self.segments: List[tuple] = []          # (start, end) element ranges of slabs.G, in backward order
        self._triggers: List[Optional[nn.Module]] = []
        start, cur = 0, []
        for k, (ps, mod) in enumerate(units):
            cur += ps
            last = k == len(units) - 1
            end = slabs.numel if last else slabs.range_of(cur)[1]
            want = tail_bucket_bytes if (slabs.numel - start) * 4 <= tail_bytes else bucket_bytes
            if last or (mod is not None and (end - start) * 4 >= want):
                self.segments.append((start, end))
                self._triggers.append(mod)
                start, cur = end, []
        self._launched = [False] * len(self.segments)
        self._works = []
        for i, mod in enumerate(self._triggers):
            if mod is not None:
                mod._bwd_done_cb = self._make_cb(i)
        if broadcast and self.world > 1:
            src = dist.get_global_rank(process_group, 0) if process_group is not None else 0
            with torch.no_grad():
                dist.broadcast(slabs.P, src=src, group=process_group)     # one flat broadcast of every parameter
                for b in model.buffers():
                    dist.broadcast(b.data, src=src, group=process_group)
            slabs.invalidate()

    def _make_cb(self, i: int):
        def cb():
            # everything before segment i in backward order is final as well (a trigger-less unit rides with the next one)
            for j in range(i + 1):
                if not self._launched[j]:
                    self._launch(j)
        return cb

    def _launch(self, i: int):
        self._launched[i] = True
        if not self.enabled or self.world == 1:
            return
        a, b = self.segments[i]
        self._works.append(dist.all_reduce(self.slabs.G[a:b], op=dist.ReduceOp.SUM, group=self.group, async_op=True))

    def finish(self) -> float:
        """Launch what the backward did not trigger, wait (stream-wise) for every collective, re-arm; returns 1 / world."""
        for i in range(len(self.segments)):
            if not self._launched[i]:
                self._launch(i)
        for w in self._works:
            w.wait()
        self._works.clear()
        self._launched = [False] * len(self.segments)
        return 1.0 / self.world

    class _NoSync:
        def __init__(self, outer):
            self.outer = outer

        def __enter__(self):
            self.outer.enabled = False

        def __exit__(self, *exc):
            self.outer.enabled = True
            self.outer._launched = [False] * len(self.outer.segments)

    def no_sync(self):
        """Gradient accumulation: backward passes inside this context only accumulate into the slab (the kernels always
        accumulate); the pass outside it triggers the all-reduces of the accumulated sum."""
        return SlabGradSync._NoSync(self)

    def remove(self):
        for mod in self._triggers:
            if mod is not None:
                mod._bwd_done_cb = None
