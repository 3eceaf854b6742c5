"""Shared implementation behind olmoasr_b200.model (training model) and olmoasr_b200.inf_model (inference model).

The module tree, parameter names / shapes and initialisation follow the reference exactly
(olmoasr/model.py:14-968, olmoasr/inf_model.py) so that `state_dict()`s are interchangeable and DDP / FSDP /
AdamW / checkpoint code written for the reference keeps working.  Every tensor operation is a call into
liboasr_b200.so; computation is 16-bit with fp32 master weights and fp32 statistics, i.e. the numerics of the
reference under `torch.autocast("cuda", dtype)` (scripts/training/train_timestamps.py:1414) with its rounding points
reproduced (Linear outputs, GELU, residual adds, LayerNorm casts, 16-bit logits).  dtype is fp16 when the call is made
under `torch.autocast("cuda", torch.float16)` (the reference trainer's default precision, :2128) and bf16 otherwise;
each top-level call resolves it once (`compute_dtype`) and the tensors carry it through every kernel.

Training fast path: one autograd.Function per ResidualAttentionBlock (+ stem, embedding and loss head) whose
backward is a hand-sequenced list of kernels -- dgrad / wgrad GEMMs read the saved activations MN-major through
the wgmma shared-memory descriptors, so nothing is transposed in HBM.
"""
from __future__ import annotations

import contextlib
import math
import os
from typing import Dict, Iterable, Optional

import numpy as np
import torch
from torch import Tensor, nn

from . import kernels as K
from .config.model_dims import ModelDimensions

PAD_ID_EN = 51864  # padding token / padding_idx of the English-only vocabulary (model.py:665-667)


# =====================================================================================================
# small helpers
# =====================================================================================================
def _sm_count() -> int:
    from ._lib import lib
    return lib().oasr_device_sm_count()


def _pick_block_n(M: int, N: int) -> int:
    """Tile width (256, 128 or 64) for the persistent GEMM (csrc/gemm_sm90.cu): the one that loads the fewest operand
    rows per SM, i.e. waves of the persistent grid times the 128 + BN rows of A and B one k-block of a tile reads.  Wave
    quantisation and the padding of N to a whole tile both count; ties go to the wider tile."""
    sms = _sm_count()
    tiles_m = math.ceil(M / 128)
    return min((256, 128, 64), key=lambda bn: math.ceil(tiles_m * math.ceil(N / bn) / sms) * (128 + bn))


def _pick_split_k(tiles: int, kblocks: int) -> int:
    sms = _sm_count()
    best, best_cost = 1, None
    for s in range(1, 9):
        if s > kblocks:
            break
        cost = math.ceil(tiles * s / sms) * (1.0 / s + 0.03)
        if best_cost is None or cost < best_cost - 1e-9:
            best, best_cost = s, cost
    return best


_bf16_pinned = 0   # > 0 inside bf16_compute()


def compute_dtype() -> torch.dtype:
    """The 16-bit type of a top-level call: fp16 under torch.autocast("cuda", torch.float16), bf16 otherwise (also under
    bf16 autocast, with no autocast at all, and inside `bf16_compute()`)."""
    if _bf16_pinned == 0 and torch.is_autocast_enabled("cuda") and torch.get_autocast_dtype("cuda") == torch.float16:
        return torch.float16
    return torch.bfloat16


@contextlib.contextmanager
def bf16_compute():
    """Run the model in bf16 whatever the autocast state: decode() and transcribe() keep their bf16 encoder and hook
    path when they are called inside an fp16 autocast region or inside `fp8_autocast()`."""
    global _bf16_pinned
    _bf16_pinned += 1
    try:
        yield
    finally:
        _bf16_pinned -= 1


_fp8_on = False   # set inside fp8_autocast(enabled=True)


@contextlib.contextmanager
def fp8_autocast(enabled: bool = True):
    """Run the forward and dgrad GEMMs of every block projection in FP8 (olmoasr_b200/fp8.py), or, with enabled=False,
    in bf16 inside an outer FP8 region.  Nests like torch.autocast: the state of the enclosing region comes back on exit."""
    global _fp8_on
    prev, _fp8_on = _fp8_on, bool(enabled)
    try:
        yield
    finally:
        _fp8_on = prev


def fp8_enabled() -> bool:
    """Whether a fused block's forward starting now runs its projections in FP8 (never inside `bf16_compute()`)."""
    return _fp8_on and _bf16_pinned == 0


def fp8_checkpoint_context_fn():
    """`context_fn` for torch.utils.checkpoint(..., use_reentrant=False): the recompute runs in the FP8 state of the
    forward, wherever the backward runs (torch restores autocast's state for a recompute, but not this one)."""
    return contextlib.nullcontext(), fp8_autocast(fp8_enabled())


def _f16_kw(dtype: torch.dtype) -> dict:
    """`dtype=` for the kernels whose inputs are all fp32; bf16 calls keep the argument lists they always had."""
    return {} if dtype == torch.bfloat16 else {"dtype": dtype}


def _cast16(src: Tensor, dtype: torch.dtype, *dst: Tensor) -> Tensor:
    """fp32 master -> 16-bit weight shadow, into `dst` when given (the bf16 cast keeps its own entry point)."""
    if dtype == torch.bfloat16:
        return K.cast_bf16(src, *dst)
    return K.convert(src, *dst, dtype=dtype)


def linear_fwd(x: Tensor, w_bf16: Tensor, bias: Optional[Tensor], *, epi=K.EPI_BF16, aux=None, out=None):
    """y = epi(x W^T + b): x (M, K) bf16, w (N, K) bf16 shadow of the fp32 master, bias (N,) f32."""
    M, Kd = x.shape
    N = w_bf16.shape[0]
    return K.gemm(x, w_bf16, M, N, Kd, bias=bias, aux=aux, epi=epi, out=out, block_n=_pick_block_n(M, N))


def linear_dgrad(dy: Tensor, w_bf16: Tensor, *, epi=K.EPI_BF16, aux=None, out=None):
    """dx = dy W: dy (M, N) bf16, w (N, K) bf16 read MN-major."""
    M, N = dy.shape
    Kd = w_bf16.shape[1]
    return K.gemm(dy, w_bf16, M, Kd, N, b_mn=True, epi=epi, aux=aux, out=out, block_n=_pick_block_n(M, Kd))


def _pick_block_n_fp8(M: int, N: int) -> int:
    """Tile width (128 or 64) of the FP8 GEMM, by `_pick_block_n`'s cost: its temporary accumulator (promotion every
    128 k) doubles the accumulator registers, which leaves no room for 256-wide tiles."""
    sms = _sm_count()
    tiles_m = math.ceil(M / 128)
    return min((128, 64), key=lambda bn: math.ceil(tiles_m * math.ceil(N / bn) / sms) * (128 + bn))


def linear_fwd_fp8(x8, w8, bias: Optional[Tensor], *, epi=K.EPI_BF16, aux=None, out=None):
    """y = epi(x W^T + b) in FP8: x8 = (q, s) the e4m3 rows of x (M, K), w8 = (q, s) the e4m3 rows of W (N, K)."""
    (xq, xs), (wq, ws) = x8, w8
    M, Kd = xq.shape
    N = wq.shape[0]
    return K.gemm_fp8(xq, xs, wq, ws, M, N, Kd, bias=bias, aux=aux, epi=epi, out=out, block_n=_pick_block_n_fp8(M, N))


def linear_dgrad_fp8(dy8, wt8, *, epi=K.EPI_BF16, aux=None, out=None):
    """dx = epi(dy W) in FP8: dy8 = (q, s) the e5m2 rows of dy (M, N), wt8 = (q, s) the e4m3 rows of W^T (K, N)."""
    (dq, ds), (wq, ws) = dy8, wt8
    M, N = dq.shape
    Kd = wq.shape[0]
    return K.gemm_fp8(dq, ds, wq, ws, M, Kd, N, epi=epi, aux=aux, out=out, block_n=_pick_block_n_fp8(M, Kd))


def fp8_inputs(xa: Optional[Tensor]) -> dict:
    """The per-forward FP8 operands shared by the layers of a stack: the e4m3 rows of the encoder output, which feeds
    every decoder layer's cross K/V projection (None for the encoder)."""
    return {"xa": None if xa is None else K.quantize_fp8_rows(_as16_2d(xa, torch.bfloat16), K.FP8_E4M3)}


# weight operands of a block's projections: forward (W, e4m3 rows) and dgrad (W^T, e4m3 rows = per input feature)
_FP8_WEIGHTS = ("wqkv", "wo", "wcq", "wckv", "wco", "w1", "w2")


def linear_wgrad(dy: Tensor, x: Tensor, n_valid: Optional[int] = None, side=None, out: Optional[Tensor] = None):
    """dW (N, K) f32 = dy^T x.  Both operands are read MN-major straight from their (M, *) row-major storage
    (A = dy^T is "stored (K=M, M=N)", B = x is "stored (K=M, N=K)"); split-K (partial products added up in split
    order) when the output has too few tiles to fill the GPU.  With `out` (a gradient-slab view, olmoasr_b200/slab.py) the product is ACCUMULATED
    into it by the epilogue: no allocation, no zero fill, no hand-over through autograd."""
    M = dy.shape[0]
    N = dy.shape[1] if n_valid is None else n_valid
    Kd = x.shape[1]
    bn = 256 if Kd >= 256 else (128 if Kd > 64 else 64)
    tiles = math.ceil(N / 128) * math.ceil(Kd / bn)
    split = _pick_split_k(tiles, math.ceil(M / 64))
    dyv = dy if n_valid is None else dy[:, :n_valid]
    accumulate = out is not None
    if out is None:
        alloc = torch.empty if split == 1 else torch.zeros     # allocated (and zeroed) on the caller's stream
        out = alloc((N, Kd), device=x.device, dtype=torch.float32)

    def launch():
        return K.gemm(dyv, x, N, Kd, M, a_mn=True, b_mn=True, out=out,
                      epi=K.EPI_F32 if (split == 1 and not accumulate) else K.EPI_F32_ATOMIC_ADD, split_k=split, block_n=bn)

    return side.run(launch) if side is not None else launch()


class _LoraOps:
    """16-bit operands of the low-rank adapters of one projection site: a Linear, or the fused members of `_FUSED`
    (member i owns output rows [i*d, (i+1)*d)).  The adapters of the members that have one are stacked along the rank,
    R = sum of their ranks (member m's slice of the rank is cols[m] = (offset, r)):
        a  (R, in) = [A_m]          as (R, in) = [s_m A_m]
        bz (N, R)  = B_m in (rows of m, cols[m]), zero elsewhere; bzs the same with s_m B_m
    so that u = x as^T is s (x A^T) for every member and y += u bz^T adds each member's term to its own rows only."""

    def __init__(self, linears, dtype):
        d = linears[0].out_features
        self.cols = {}
        R = 0
        for i, lin in enumerate(linears):
            if lin.has_lora:
                self.cols[i] = (R, lin.lora_A.shape[0])
                R += lin.lora_A.shape[0]
        self.R = R
        dev = linears[0].weight.device
        n_in = linears[0].in_features
        self.a = torch.empty((R, n_in), device=dev, dtype=dtype)
        self.a_s = torch.empty((R, n_in), device=dev, dtype=dtype)
        self.bz = torch.zeros((len(linears) * d, R), device=dev, dtype=dtype)
        self.bz_s = torch.zeros((len(linears) * d, R), device=dev, dtype=dtype)
        for i, (off, r) in self.cols.items():
            lin = linears[i]
            A, B = lin.lora_A.detach().contiguous(), lin.lora_B.detach().contiguous()
            K.cast_scaled16(A, 1.0, self.a[off:off + r])
            K.cast_scaled16(A, lin.lora_scale, self.a_s[off:off + r])
            K.cast_scaled16(B, 1.0, self.bz[i * d:(i + 1) * d, off:off + r])
            K.cast_scaled16(B, lin.lora_scale, self.bz_s[i * d:(i + 1) * d, off:off + r])

    @staticmethod
    def of(linears, cache: "_ShadowCache", dtype):
        """The site's operands (rebuilt when an adapter changed), or None when no member has an adapter."""
        ps = [p for lin in linears if lin.has_lora for p in (lin.lora_A, lin.lora_B)]
        if not ps:
            return None
        return cache.get(ps, lambda: _LoraOps(linears, dtype), dtype)


def lora_fwd(x: Tensor, w: Tensor, bias: Optional[Tensor], ops: Optional[_LoraOps], *, epi=K.EPI_BF16, aux=None, out=None,
             u: Optional[Tensor] = None):
    """(epi(x W^T + b + u bz^T), u) with u = x as^T (M, R) the adapters' low-rank activations (kept for the backward),
    or (linear_fwd(...), None) without adapters.  `u` may be given preallocated (side-stream launches)."""
    if ops is None:
        return linear_fwd(x, w, bias, epi=epi, aux=aux, out=out), None
    M, Kd = x.shape
    N = w.shape[0]
    u = linear_fwd(x, ops.a_s, None, out=u)
    y = K.gemm_lowrank(x, w, u, ops.bz, M, N, Kd, ops.R, bias=bias, aux=aux, epi=epi, out=out, block_n=_pick_block_n(M, N))
    return y, u


def lora_v(dy: Tensor, ops: Optional[_LoraOps]) -> Optional[Tensor]:
    """v = dy bz_s (M, R) = s (dy B) per member: the dgrad tail's A2 and the A-gradient's left operand."""
    return None if ops is None else linear_dgrad(dy, ops.bz_s)


def lora_dgrad(dy: Tensor, w: Tensor, ops: Optional[_LoraOps], v: Optional[Tensor], *, epi=K.EPI_BF16, aux=None, out=None):
    """dx = epi(dy W + v a): the dgrad of a projection with adapters (plain `linear_dgrad` without)."""
    if ops is None:
        return linear_dgrad(dy, w, epi=epi, aux=aux, out=out)
    M, N = dy.shape
    Kd = w.shape[1]
    return K.gemm_lowrank(dy, w, v, ops.a, M, Kd, N, ops.R, b_mn=True, epi=epi, aux=aux, out=out, block_n=_pick_block_n(M, Kd))


# Projections of a block whose weight gradients one GEMM computes, stacked in this order (d rows each), and whose bias
# gradients one column sum covers.  The key projections have no bias (model.py:259): their rows of the fused [bq; 0; bv]
# bias are a gap of the slab that no gradient may ever be written to.
_FUSED = {"attn.qkv": ("attn.query", "attn.key", "attn.value"), "cross_attn.kv": ("cross_attn.key", "cross_attn.value")}


class _GradDest:
    """Where the parameter gradients of one backward go, decided once from `owner`, the module that holds them.

    Direct mode (`use_slabs()` with `direct_grads`): every kernel ACCUMULATES into its parameter's slice of the gradient
    slab, autograd is handed None, and `done()` fires the owner's `_bwd_done_cb` (olmoasr_b200.ddp.SlabGradSync).
    Hand-over mode (no slabs, or `direct_grads=False` for torch DDP; FSDP's parameter views): fresh tensors are returned
    to autograd, so wrappers that hook gradient accumulation and foreign optimizers keep working.  With `pool_size`, its
    zeroed vectors are slices of one zero fill (each fill is a separate ~4 us launch; ~700 of them per step otherwise).
    Weight and bias gradients are launched through `side` when given."""

    def __init__(self, owner, device=None, side: Optional["_Side"] = None, pool_size: int = 0):
        direct = owner is not None and owner._direct is not None and owner._slabs.direct_grads
        self.owner, self.device, self.side = owner, device, side
        self.slab: Optional[Dict[str, Tensor]] = owner._direct if direct else None
        self.pool = torch.zeros(pool_size, device=device, dtype=torch.float32) if (pool_size and not direct) else None
        self.used = 0
        self.grads: Dict[str, Tensor] = {}
        # names of the owner's parameters that take a gradient: a frozen one gets no kernel launch at all
        self.trainable = None if owner is None else {n for n, p in owner.named_parameters() if p.requires_grad}

    def wants(self, key: str) -> bool:
        """Whether parameter `key` (or, for a fused name of `_FUSED`, any of its members) takes a gradient."""
        have = self.slab if self.slab is not None else self.trainable   # direct mode: the slab holds what trains
        if have is None or key in have:
            return True
        name, kind = key.rsplit(".", 1)
        return any(m + "." + kind in have for m in _FUSED.get(name, ()))

    def out(self, key: str) -> Optional[Tensor]:
        """The slab view a kernel accumulates `key`'s gradient into, or None: the kernel allocates the gradient."""
        return None if self.slab is None else self.slab[key]

    def keep(self, key: str, g: Tensor) -> Tensor:
        self.grads[key] = g
        return g

    def _zeros(self, shape) -> Tensor:
        """The next slice of the pool, 64-element aligned so that every view stays 256-byte aligned, else its own fill."""
        if self.pool is None or self.used + (shape + 63) // 64 * 64 > self.pool.numel():
            return torch.zeros(shape, device=self.device, dtype=torch.float32)
        v = self.pool[self.used:self.used + shape]
        self.used += (shape + 63) // 64 * 64
        return v

    def vec(self, key: str, shape) -> Optional[Tensor]:
        """Zero-initialised accumulation target of `key`'s gradient (LayerNorm, embedding and bias vectors); None when
        `key` takes no gradient (kernels that accept a null target then skip that reduction)."""
        if not self.wants(key):
            return None
        return self.slab[key] if self.slab is not None else self.keep(key, self._zeros(shape))

    def _launch(self, fn):
        return self.side.run(fn) if self.side is not None else fn()

    def weight(self, key: str, dy: Tensor, x: Tensor, n_valid: Optional[int] = None) -> Tensor:
        return self.keep(key, linear_wgrad(dy, x, n_valid, side=self.side, out=self.out(key)))

    def bias(self, key: str, dy: Tensor):
        """Column sums of dy (M, n) bf16 into the bias gradient `key`."""
        db = self.vec(key, dy.shape[1])
        if db is not None:
            self._launch(lambda: K.colsum_(dy, db, dy.shape[1]))

    def linear(self, name: str, dy: Tensor, x: Tensor, lora: Optional[tuple] = None):
        """Weight and bias gradients of the Linear `name`, or of the projections `_FUSED[name]`, from the output
        gradient dy and the input x; with `lora` = (ops, u, v) also the gradients of the site's adapters.  Only the
        parameters that take a gradient get one."""
        members = _FUSED.get(name)
        if lora is not None:
            self._lora(members or (name,), dy, x, *lora)
        d = dy.shape[1] // len(members or (name,))
        if members is not None and not all(self.wants(m + ".weight") for m in members):
            for i, m in enumerate(members):     # a partly trainable fused weight: one GEMM per trainable member
                if self.wants(m + ".weight"):
                    self.weight(m + ".weight", dy[:, i * d:(i + 1) * d], x)
        elif self.wants(name + ".weight"):
            self.weight(name + ".weight", dy, x)
        if members is None:
            if self.wants(name + ".bias"):
                self.bias(name + ".bias", dy)
            return
        if self.slab is not None:      # one column sum per member that has a bias, so no gap of the slab is written
            for i, m in enumerate(members):
                if m + ".bias" in self.slab:
                    self.bias(m + ".bias", dy[:, i * d:(i + 1) * d])
            return
        if self.wants(name + ".bias"):
            self.bias(name + ".bias", dy)  # one column sum over the whole fused width; every member takes its rows
        for i, m in enumerate(members):
            for kind in (".weight", ".bias"):
                if name + kind in self.grads:
                    self.grads[m + kind] = self.grads[name + kind][i * d:(i + 1) * d]

    def _lora(self, members, dy: Tensor, x: Tensor, ops: _LoraOps, u: Tensor, v: Tensor):
        """dA = v^T x and dB = dy^T u per member, on its slices of v / u (rank columns) and dy (output rows)."""
        d = dy.shape[1] // len(members)
        for i, (off, r) in ops.cols.items():
            m = members[i]
            if self.wants(m + ".lora_A"):
                self.weight(m + ".lora_A", v[:, off:off + r], x)
            if self.wants(m + ".lora_B"):
                self.weight(m + ".lora_B", dy[:, i * d:(i + 1) * d], u[:, off:off + r])

    def grads_for(self, names: Iterable[str]) -> tuple:
        """What autograd receives for these parameters: all None in direct mode, where the slab already holds them."""
        if self.slab is not None:
            return tuple(None for _ in names)
        return tuple(self.grads.get(n) for n in names)

    def done(self):
        """Direct mode: tell the owner's gradient synchronisation hook that its slab range is final."""
        if self.slab is not None and self.owner._bwd_done_cb is not None:
            self.owner._bwd_done_cb()


# ----------------------------------------------------------------------------------------------------
# Weight / bias gradients of a block are leaves of the backward graph: nothing downstream in the same backward reads
# them.  They are enqueued on a second CUDA stream so that their CTAs fill the SMs that the dgrad / attention /
# LayerNorm chain on the main stream leaves idle: the partial last wave of tiles of each persistent wgmma GEMM
# (csrc/gemm_sm90.cu), and the gaps between launches.  Every block joins the side stream before its backward returns,
# so gradients are complete in main-stream order (DDP hooks, optimizer).
SIDE_STREAM = os.environ.get("OASR_SIDE_STREAM", "1") != "0"
_side_streams: Dict[int, "torch.cuda.Stream"] = {}


class _Side:
    def __init__(self, device):
        self.on = SIDE_STREAM and device.type == "cuda"
        if self.on:
            idx = device.index if device.index is not None else torch.cuda.current_device()
            if idx not in _side_streams:
                _side_streams[idx] = torch.cuda.Stream(device=idx)
            self.side = _side_streams[idx]
            self.main = torch.cuda.current_stream(idx)

    def run(self, fn):
        """fn() on the side stream, after everything enqueued on the main stream so far.  fn must only LAUNCH: every
        tensor it touches is allocated by the caller on the main stream (whose pool the caching allocator then keeps
        ordered with the main stream; the side stream's accesses sit between wait_stream and join), so no
        record_stream bookkeeping -- and no cross-pool churn -- is needed."""
        if not self.on:
            return fn()
        self.side.wait_stream(self.main)
        with torch.cuda.stream(self.side):
            return fn()

    def join(self):
        if self.on:
            self.main.wait_stream(self.side)


STRICT_MASK = os.environ.get("OASR_STRICT_MASK", "0") == "1"
_mask_err: Dict[int, tuple] = {}   # device index -> (device flag, pinned host flag, event of the last flag copy)


def check_deferred_errors(device=None, wait: bool = False):
    """Raise if an earlier padding_mask failed validation.  The check itself never stalls the stream: the kernel that
    derives the key counts also verifies the mask and raises a flag that is copied to pinned memory asynchronously; it is
    looked at on the NEXT call (or here, with wait=True / OASR_STRICT_MASK=1: immediately, at the cost of a sync)."""
    idx = torch.cuda.current_device() if device is None else (device.index if device.index is not None else torch.cuda.current_device())
    st = _mask_err.get(idx)
    if st is None or st[2] is None:
        return
    flag, host, ev = st
    if wait:
        ev.synchronize()
    if ev.query() and int(host[0]) != 0:
        host[0] = 0
        flag.zero_()
        raise ValueError("padding_mask is not of the form [0]*len + [-inf]*(n_ctx-len) on every row (the only structure "
                         "scripts/training/train_timestamps.py:314-315 produces); this implementation derives a per-sample "
                         "key count from it and supports no other additive mask")


def kv_len_from_padding_mask(padding_mask: Tensor) -> Tensor:
    """The reference passes a dense additive mask (B, 448, 448) whose columns >= len(text_input) are -inf for every
    row (scripts/training/train_timestamps.py:314-315).  The kernels take that as a per-sample key count, derived -- and
    the structure verified -- on the device.  A 1-D integer tensor is taken as the key counts themselves (what a data
    loader that never builds the 25.7 MB mask would pass)."""
    if padding_mask.dim() == 1 and not padding_mask.is_floating_point():
        return padding_mask if padding_mask.dtype == torch.int32 else padding_mask.to(torch.int32)
    cached = getattr(padding_mask, "_oasr_kv_len", None)   # computed once per decoder call, not once per block
    if cached is not None and cached[0] == padding_mask._version:
        return cached[1]
    if padding_mask.dim() != 3 or padding_mask.shape[1] != padding_mask.shape[2] or \
            padding_mask.dtype not in (torch.float32, torch.bfloat16, torch.float16):
        raise ValueError(f"padding_mask must be (B, n_ctx, n_ctx) float32, got {tuple(padding_mask.shape)} {padding_mask.dtype}")
    if not padding_mask.is_cuda:
        from ._lib import OasrError
        raise OasrError("padding_mask must be a CUDA tensor (the key counts are derived on the device; no CPU fallback)")
    dev = padding_mask.device
    idx = dev.index if dev.index is not None else torch.cuda.current_device()
    check_deferred_errors(dev)
    if idx not in _mask_err:
        _mask_err[idx] = (torch.zeros(1, device=dev, dtype=torch.int32), torch.zeros(1, dtype=torch.int32).pin_memory(), None)
    flag, host, _ = _mask_err[idx]
    mask32 = padding_mask.contiguous()
    if mask32.dtype != torch.float32:     # FSDP MixedPrecision casts the root module's floating-point inputs to bf16 (0 / -inf survive)
        mask32 = K.convert(mask32, dtype=torch.float32)
    kv = K.mask_to_kvlen(mask32, flag)
    host.copy_(flag, non_blocking=True)
    ev = torch.cuda.Event()
    ev.record()
    _mask_err[idx] = (flag, host, ev)
    if STRICT_MASK:
        check_deferred_errors(dev, wait=True)
    try:
        padding_mask._oasr_kv_len = (padding_mask._version, kv)   # rides on this tensor object; in-place edits invalidate
    except (AttributeError, RuntimeError):
        pass
    return kv


class PackedBatch:
    """The decoder rows of a batch whose sample b holds its first lens[b] tokens, stacked in (b, t) order: N rows
    instead of B*S.  One int32 device buffer, filled by one pinned non-blocking copy, carries what the kernels read:
        cu     (B+1,)        sample b owns packed rows [cu[b], cu[b+1])
        tiles  (n_tiles, 2)  (b, j) for every 128-row tile j of sample b that holds a row: the attention grids
        rows   (N,)          dense index b*S + t of each packed row: the embedding gather, the target gather
    Every decoder layer reads the same buffer in forward and backward."""

    TILE = 128   # query / key rows per attention tile (csrc/attention_*_sm90.cu)

    def __init__(self, lens, S: int, device):
        self.lens = [int(n) for n in lens]
        self.B, self.S = len(self.lens), int(S)
        cu = np.zeros(self.B + 1, dtype=np.int32)
        cu[1:] = np.cumsum(self.lens)
        self.N = int(cu[-1])
        tiles = [(b, j) for b, n in enumerate(self.lens) for j in range((n + self.TILE - 1) // self.TILE)]
        self.n_tiles = len(tiles)
        rows = np.concatenate([b * self.S + np.arange(n, dtype=np.int32) for b, n in enumerate(self.lens)])
        host = torch.from_numpy(np.concatenate([cu, np.asarray(tiles, dtype=np.int32).reshape(-1), rows]))
        device = torch.device(device)
        if device.type == "cuda":
            buf = torch.empty(host.shape, device=device, dtype=torch.int32)
            buf.copy_(host.pin_memory(), non_blocking=True)
        else:
            buf = host
        n_cu, n_t = self.B + 1, 2 * self.n_tiles
        self.cu, self.tiles, self.rows = buf[:n_cu], buf[n_cu:n_cu + n_t].view(-1, 2), buf[n_cu + n_t:]


def packed_text_lens(text_lens, tokens: Tensor, targets: Optional[Tensor], padding_mask: Optional[Tensor]) -> list:
    """Validate the `text_lens=` argument of the loss calls and return it as a list of ints.  It is host data by design:
    reading a CUDA tensor would put a device-to-host sync into every step."""
    if targets is None:
        raise ValueError("text_lens packs the loss route only: pass targets= as well (the logits route is dense)")
    if padding_mask is not None:
        raise ValueError("pass either text_lens or padding_mask, not both: text_lens already defines the key counts")
    if isinstance(text_lens, Tensor):
        if text_lens.is_cuda:
            raise ValueError("text_lens must be host data (a CPU tensor or a sequence of ints): reading a CUDA tensor "
                             "would synchronise with the device on every step")
        if text_lens.is_floating_point() or text_lens.is_complex() or text_lens.dtype == torch.bool or text_lens.dim() != 1:
            raise ValueError(f"text_lens must be a 1-D integer tensor, got {text_lens.dtype} {tuple(text_lens.shape)}")
        lens = [int(n) for n in text_lens.tolist()]
    else:
        try:
            lens = list(text_lens)
        except TypeError:
            raise ValueError("text_lens must be a CPU integer tensor or a sequence of ints") from None
        if not all(isinstance(n, (int, np.integer)) and not isinstance(n, bool) for n in lens):
            raise ValueError("text_lens must be a CPU integer tensor or a sequence of ints")
        lens = [int(n) for n in lens]
    B, S = tokens.shape
    if tuple(targets.shape) != (B, S):
        raise ValueError(f"targets {tuple(targets.shape)} must have the shape of tokens {(B, S)} with text_lens")
    if len(lens) != B:
        raise ValueError(f"text_lens has {len(lens)} entries for a batch of {B}")
    bad = [n for n in lens if not 1 <= n <= S]
    if bad:
        raise ValueError(f"text_lens entries must lie in [1, {S}], got {bad[0]}")
    return lens


class _ShadowCache:
    """16-bit copies of fp32 master weights (+ fused biases), rebuilt only when a master or the wanted type changed."""

    def __init__(self):
        self.key = None
        self.val = None

    def get(self, params: Iterable[Tensor], build, dtype: torch.dtype = torch.bfloat16):
        key = (dtype,) + tuple((p.data_ptr(), p._version, p.device) for p in params)
        if key != self.key:
            with torch.no_grad():
                self.val = build()
            self.key = key
        return self.val


# =====================================================================================================
# leaf modules (parameters live here, names identical to the reference)
# =====================================================================================================
class LayerNorm(nn.LayerNorm):
    """olmoasr/model.py:14-39."""

    def forward(self, x: Tensor) -> Tensor:
        shp = x.shape
        y = K.layernorm_fwd(_as16_2d(x, compute_dtype()), _f32(self.weight), _f32(self.bias), self.eps, want_stats=False)
        return y.view(shp)


class Linear(nn.Linear):
    """olmoasr/model.py:42-101: kaiming-normal weight, bf16 compute with the fp32 master cast on the fly."""

    def __init__(self, in_features: int, out_features: int, bias: bool = True, device=None, dtype=None):
        super().__init__(in_features, out_features, bias=bias, device=device, dtype=dtype)
        nn.init.kaiming_normal_(self.weight, mode="fan_in", nonlinearity="relu")
        self._shadow = _ShadowCache()

    _slab_view: Optional[Tensor] = None   # set by OLMoASRBase.use_slabs(): a view into the shadow slab
    lora_scale = 0.0                      # s = alpha / r of the adapter that olmoasr_b200.lora.add_lora registers

    @property
    def has_lora(self) -> bool:
        """True when a low-rank adapter (lora_A (r, in), lora_B (out, r)) is registered on this Linear."""
        return "lora_A" in self._parameters

    def weight_bf16(self) -> Tensor:
        return self.weight16(torch.bfloat16)

    def weight16(self, dtype: torch.dtype) -> Tensor:
        if self._slab_view is not None:
            return _slab16(self._slab_view, dtype)
        if self.weight.dtype == dtype:      # FSDP param_dtype: the unsharded view IS the operand (never cached)
            return self.weight.detach()
        if not _is_master(self.weight):
            return K.convert(self.weight.detach().contiguous(), dtype=dtype)
        return self._shadow.get((self.weight,), lambda: _cast16(self.weight.detach().contiguous(), dtype), dtype)

    def forward(self, x: Tensor) -> Tensor:  # inference / hook path (no autograd through the kernels)
        shp = x.shape
        dt = compute_dtype()
        ops = _LoraOps.of((self,), self.__dict__.setdefault("_lora_shadow", _ShadowCache()), dt) if self.has_lora else None
        y, _ = lora_fwd(_as16_2d(x, dt), self.weight16(dt), None if self.bias is None else _f32(self.bias), ops)
        return y.view(*shp[:-1], self.out_features)


class Conv1d(nn.Conv1d):
    """olmoasr/model.py:104-195 (parameters only; the stem kernels are driven by AudioEncoder)."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, bias=True,
                 padding_mode="zeros", device=None, dtype=None):
        super().__init__(in_channels, out_channels, kernel_size, stride=stride, padding=padding, dilation=dilation,
                         groups=groups, bias=bias, padding_mode=padding_mode, device=device, dtype=dtype)
        nn.init.kaiming_normal_(self.weight, mode="fan_in", nonlinearity="relu")
        self._shadow = _ShadowCache()

    def weight_bf16(self) -> Tensor:
        return self.weight16(torch.bfloat16)

    def weight16(self, dtype: torch.dtype) -> Tensor:  # (C_out, 3*C_in) with column = k*C_in + c
        if not _is_master(self.weight):
            return K.cast_conv_weight(_f32(self.weight).contiguous(), **_f16_kw(dtype))
        return self._shadow.get((self.weight,), lambda: K.cast_conv_weight(self.weight.detach().contiguous(), **_f16_kw(dtype)),
                                dtype)


def sinusoids(length, channels, max_timescale=10000):
    """olmoasr/model.py:199-230."""
    assert channels % 2 == 0
    log_timescale_increment = np.log(max_timescale) / (channels // 2 - 1)
    inv_timescales = torch.exp(-log_timescale_increment * torch.arange(channels // 2))
    scaled_time = torch.arange(length)[:, np.newaxis] * inv_timescales[np.newaxis, :]
    return torch.cat([torch.sin(scaled_time), torch.cos(scaled_time)], dim=1)


def _as16_2d(x: Tensor, dtype: torch.dtype) -> Tensor:
    if x.dtype != dtype:
        x = x.to(dtype)
    return x.reshape(-1, x.shape[-1]).contiguous()


def _as_bf16_2d(x: Tensor) -> Tensor:
    return _as16_2d(x, torch.bfloat16)


def _slab16(view: Tensor, dtype: torch.dtype) -> Tensor:
    """A view of the shadow slab S as `dtype`: S holds the type the model last computed in (ParamSlabs.ensure_synced),
    and bf16 and fp16 have the same size, so either is a reinterpretation of the same bytes."""
    return view if view.dtype == dtype else view.view(dtype)


def _f32(p: Tensor) -> Tensor:
    """fp32 view of a vector parameter / buffer.  Parameters are fp32 masters except under FSDP MixedPrecision(param_dtype=
    bf16) (scripts/training/train_fsdp_timestamps.py:2588-2615), where the unsharded views are bf16: converted per call."""
    p = p.detach()
    if p.dtype == torch.float32:
        return p
    return K.convert(p.contiguous(), dtype=torch.float32)


def _is_master(p: Tensor) -> bool:
    return p.dtype == torch.float32


def _attr_by_path(mod: nn.Module, path: str) -> Tensor:
    obj = mod
    for part in path.split("."):
        obj = getattr(obj, part)
    return obj


class MultiHeadAttention(nn.Module):
    """olmoasr/model.py:233-442.  `double_init` reproduces the training model's second kaiming draw (model.py:258-264)
    so that seeds give the reference's weights; the inference model draws once (inf_model.py:131-138)."""

    def __init__(self, n_state: int, n_head: int, double_init: bool = True):
        super().__init__()
        self.n_head = n_head
        self.query = Linear(n_state, n_state)
        if double_init:
            nn.init.kaiming_normal_(self.query.weight, mode="fan_in", nonlinearity="relu")
        self.key = Linear(n_state, n_state, bias=False)
        if double_init:
            nn.init.kaiming_normal_(self.key.weight, mode="fan_in", nonlinearity="relu")
        self.value = Linear(n_state, n_state)
        if double_init:
            nn.init.kaiming_normal_(self.value.weight, mode="fan_in", nonlinearity="relu")
        self.out = Linear(n_state, n_state)
        if double_init:
            nn.init.kaiming_normal_(self.out.weight, mode="fan_in", nonlinearity="relu")
        self._fused = _ShadowCache()

    # ---- fused 16-bit shadows -----------------------------------------------------------------------
    _slab_fused = None   # set by OLMoASRBase.use_slabs(): ([Wq;Wk;Wv] view of the shadow slab, [bq;0;bv] view of the masters)

    def fused_qkv(self, dtype: torch.dtype = torch.bfloat16):
        """([Wq;Wk;Wv] (3d, d) in `dtype`, [bq;0;bv] (3d,) f32) -- key has no bias (model.py:259)."""
        if self._slab_fused is not None:
            w, b = self._slab_fused
            return _slab16(w, dtype), b
        ps = (self.query.weight, self.key.weight, self.value.weight, self.query.bias, self.value.bias)

        def build():
            d = self.query.weight.shape[0]
            w = torch.empty((3 * d, d), device=ps[0].device, dtype=dtype)
            b = torch.zeros(3 * d, device=ps[0].device, dtype=torch.float32)
            for i, p in enumerate(ps[:3]):
                if _is_master(p):
                    _cast16(p.detach().contiguous(), dtype, w[i * d:(i + 1) * d])
                elif p.dtype == dtype:
                    w[i * d:(i + 1) * d].copy_(p.detach())     # bf16 unsharded FSDP view: a device-to-device copy
                else:
                    K.convert(p.detach().contiguous(), w[i * d:(i + 1) * d])
            for p, sl in ((ps[3], slice(0, d)), (ps[4], slice(2 * d, 3 * d))):
                if _is_master(p):
                    b[sl].copy_(p.detach())
                else:
                    K.convert(p.detach().contiguous(), b[sl])
            return w, b

        if not _is_master(ps[0]):
            with torch.no_grad():
                return build()                                  # transient FSDP views: nothing to key a cache on
        return self._fused.get(ps, build, dtype)

    def fused_kv(self, dtype: torch.dtype = torch.bfloat16):
        w, b = self.fused_qkv(dtype)
        d = self.query.weight.shape[0]
        return w[d:], b[d:]

    # ---- generic (hook-compatible) path: used for decoding with a kv cache --------------------------------
    def forward(self, x: Tensor, xa: Optional[Tensor] = None, mask: Optional[Tensor] = None,
                kv_cache: Optional[dict] = None, verbose: bool = False):
        B, Tq, d = x.shape
        q = self.query(x)
        if kv_cache is None or xa is None or self.key not in kv_cache:
            k = self.key(x if xa is None else xa)      # forward hooks (install_kv_cache_hooks) may swap these for the cache
            v = self.value(x if xa is None else xa)
        else:
            k = kv_cache[self.key]
            v = kv_cache[self.value]
        Tkv = k.shape[1]
        causal = mask is not None and xa is None and Tq == Tkv and Tq > 1
        kv_len = None
        if mask is not None and mask.dim() == 3:
            kv_len = kv_len_from_padding_mask(mask)
        o, _ = K.attention_fwd(q.reshape(B * Tq, d), k.reshape(B * Tkv, d), v.reshape(B * Tkv, d), B, self.n_head, Tq, Tkv,
                               causal=causal, kv_len=kv_len, want_lse=False)
        return self.out(o.view(B, Tq, d)), None


# =====================================================================================================
# fused training blocks
# =====================================================================================================
def _self_attn_fwd(q, k, v, B, H, T, causal, kv_len, pk):
    if pk is not None:
        return K.attention_fwd_varlen(q, k, v, pk, H)
    return K.attention_fwd(q, k, v, B, H, T, T, causal=causal, kv_len=kv_len)


def _cross_attn_fwd(q, k, v, B, H, T, Ta, pk):
    if pk is not None:
        return K.attention_fwd_varlen(q, k, v, pk, H, Tkv=Ta)
    return K.attention_fwd(q, k, v, B, H, T, Ta)


class _BlockFn(torch.autograd.Function):
    """ResidualAttentionBlock.forward (model.py:485-528) for a (B*T, d) bf16 or fp16 residual stream (x's type is the
    block's compute type), or for the (N, d) rows of a packed decoder batch `pk` (PackedBatch; then B, T are its batch
    size and dense length, the self-attention is causal over each sample's own rows and kv_len is None).

    inputs: x, xa (or None), kv_len (or None), then the block's parameters in `ResidualAttentionBlock._param_list`
    order.  Saves every GEMM input it needs for wgrad; recomputes nothing.

    f8: None, or (inside `fp8_autocast()`) `fp8_inputs(xa)`: every projection's forward then runs as an e4m3 x e4m3 GEMM
    over per-row quantised operands, and the backward (wherever it runs) its dgrad as e5m2 x e4m3; the wgrads keep
    reading the saved bf16 activations."""

    @staticmethod
    def forward(ctx, blk, B, T, Ta, causal, kv_len, xa_state, pk, f8, x, xa, *params):
        ctx.xa_state = xa_state
        H = blk.attn.n_head
        d = x.shape[1]
        sh = blk._shadows(x.dtype)
        lo = blk._lora_ops(x.dtype)   # site -> _LoraOps of its adapters, or None
        w8 = None
        if f8 is not None:
            if x.dtype != torch.bfloat16:
                raise ValueError("fp8_autocast() computes in bf16: it cannot be combined with torch.autocast(\"cuda\", "
                                 "torch.float16)")
            if blk._lora_on:
                raise ValueError("fp8_autocast() does not support LoRA adapters: train them in bf16, or merge_lora() first")
            w8 = blk._fp8_weights(sh)
        us = {}                       # site -> low-rank activations u, saved for the backward

        def proj(w, b, site, x_in, x8=None, **kw):
            """(y, u) of one projection site: bf16 (with its adapters), or FP8 over the e4m3 rows of x_in."""
            if w8 is None:
                return lora_fwd(x_in, sh[w], sh[b], lo.get(site), **kw)
            if x8 is None:
                x8 = K.quantize_fp8_rows(x_in, K.FP8_E4M3)
            kw.pop("u", None)    # (no adapters under FP8)
            return linear_fwd_fp8(x8, w8[w][0], sh[b], **kw), None

        side = _Side(x.device)
        kvc = None
        if xa is not None:   # the cross-attention K/V projection only needs the encoder output: side stream, joined below
            kvc = torch.empty((xa.shape[0], 2 * d), device=x.device, dtype=x.dtype)
            ops = lo.get("cross_attn.kv")
            u = None if ops is None else torch.empty((xa.shape[0], ops.R), device=x.device, dtype=x.dtype)
            xa8 = None if f8 is None else f8["xa"]   # quantised on the main stream before the first layer
            side.run(lambda: proj("wckv", "bckv", "cross_attn.kv", xa, xa8, out=kvc, u=u))
            us["cross_attn.kv"] = u
        ln1, mean1, rstd1 = K.layernorm_fwd(x, sh["ln1w"], sh["ln1b"])
        qkv, us["attn.qkv"] = proj("wqkv", "bqkv", "attn.qkv", ln1)
        ao, lse = _self_attn_fwd(qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:], B, H, T, causal, kv_len, pk)
        x1, us["attn.out"] = proj("wo", "bo", "attn.out", ao, epi=K.EPI_BF16_RESIDUAL, aux=x)
        saved = [x, mean1, rstd1, ln1, qkv, ao, lse, x1]
        if xa is not None:
            lnc, meanc, rstdc = K.layernorm_fwd(x1, sh["lncw"], sh["lncb"])
            qc, us["cross_attn.query"] = proj("wcq", "bcq", "cross_attn.query", lnc)
            side.join()
            co, lsec = _cross_attn_fwd(qc, kvc[:, :d], kvc[:, d:], B, H, T, Ta, pk)
            x2, us["cross_attn.out"] = proj("wco", "bco", "cross_attn.out", co, epi=K.EPI_BF16_RESIDUAL, aux=x1)
            saved += [xa, meanc, rstdc, lnc, qc, kvc, co, lsec, x2]
        else:
            x2 = x1
        ln2, mean2, rstd2 = K.layernorm_fwd(x2, sh["ln2w"], sh["ln2b"])
        (h, g), us["mlp.0"] = proj("w1", "b1", "mlp.0", ln2, epi=K.EPI_BF16_GELU)
        x3, us["mlp.2"] = proj("w2", "b2", "mlp.2", g, epi=K.EPI_BF16_RESIDUAL, aux=x2)
        saved += [mean2, rstd2, ln2, h, g]
        if kv_len is not None:
            saved.append(kv_len)
        sites = [k for k, u in us.items() if u is not None]
        saved += [us[k] for k in sites]
        ctx.save_for_backward(*saved)
        ctx.blk, ctx.dims, ctx.sh, ctx.pk = blk, (B, T, Ta, H, d, causal, xa is not None, kv_len is not None), sh, pk
        ctx.lora = lo, sites
        # the FP8 weight copies, for the dgrads; FSDP's unsharded views are gone by the backward, which rebuilds them
        # from the re-gathered parameters, so only the mode is kept then
        ctx.fp8 = w8 is not None
        ctx.w8 = w8 if _is_master(blk.attn.query.weight) else None
        return x3

    @staticmethod
    def backward(ctx, dx3):
        blk, sh = ctx.blk, ctx.sh
        sv = list(ctx.saved_tensors)
        w8 = ctx.w8     # the FP8 weight copies when the forward ran under fp8_autocast()
        if not _is_master(blk.attn.query.weight):
            sh = blk._shadows(sv[0].dtype)   # FSDP frees and re-gathers the unsharded parameters between forward and backward
            if ctx.fp8:
                w8 = blk._fp8_weights(sh)
        B, T, Ta, H, d, causal, cross, has_len = ctx.dims
        pk = ctx.pk
        lo, sites = ctx.lora
        us = dict(zip(sites, sv[len(sv) - len(sites):]))
        del sv[len(sv) - len(sites):]
        kv_len = sv.pop() if has_len else None
        x, mean1, rstd1, ln1, qkv, ao, lse, x1 = sv[:8]
        if cross:
            xa, meanc, rstdc, lnc, qc, kvc, co, lsec, x2 = sv[8:17]
            mean2, rstd2, ln2, h, g = sv[17:22]
        else:
            x2 = x1
            mean2, rstd2, ln2, h, g = sv[8:13]
        dx3 = dx3.contiguous()
        side = _Side(x.device)
        # hand-over mode takes all bias / LayerNorm gradient vectors (<= 26 d) from one zero fill
        grads = _GradDest(blk, x.device, side, pool_size=32 * d + 4096)

        # Operands allocated here on the main stream and read by side-stream launches (the adapters' v) must outlive
        # side.join(): dropped earlier, the allocator could hand their memory to a main-stream tensor while the side
        # stream still reads it.
        live = []

        def site(name, dy, x_in):
            """The site's weight / bias / adapter gradients; returns (ops, v) for its dgrad."""
            ops = lo.get(name)
            v = lora_v(dy, ops)
            live.append(v)
            grads.linear(name, dy, x_in, None if ops is None else (ops, us[name], v))
            return ops, v

        def dgrad(w, dy, ops, v, dy8=None, **kw):
            """dx of the projection with weight sh[w]: bf16 (with its adapters), or FP8 over the e5m2 rows of dy."""
            if w8 is None:
                return lora_dgrad(dy, sh[w], ops, v, **kw)
            return linear_dgrad_fp8(K.quantize_fp8_rows(dy, K.FP8_E5M2) if dy8 is None else dy8, w8[w][1], **kw)

        # ---- MLP: x3 = x2 + fc2(gelu(fc1(ln(x2))))
        ops, v = site("mlp.2", dx3, g)
        dh = dgrad("w2", dx3, ops, v, epi=K.EPI_BF16_GELU_BWD, aux=h)
        ops, v = site("mlp.0", dh, ln2)
        dln2 = dgrad("w1", dh, ops, v)
        dx2 = K.layernorm_bwd(dln2, x2, sh["ln2w"], mean2, rstd2, grads.vec("mlp_ln.weight", d), grads.vec("mlp_ln.bias", d),
                              dresidual=dx3)
        dxa = None
        if cross:
            # ---- cross attention: x2 = x1 + out(attn(q(ln(x1)), kv(xa)))
            ops, v = site("cross_attn.out", dx2, co)
            dco = dgrad("wco", dx2, ops, v)
            dqc = torch.empty_like(qc)
            dkvc = torch.empty_like(kvc)
            if pk is not None:
                K.attention_bwd_varlen(qc, kvc[:, :d], kvc[:, d:], co, dco, lsec, pk, H, Tkv=Ta, dq=dqc, dk=dkvc[:, :d],
                                       dv=dkvc[:, d:])
            else:
                K.attention_bwd(qc, kvc[:, :d], kvc[:, d:], co, dco, lsec, B, H, T, Ta, dq=dqc, dk=dkvc[:, :d], dv=dkvc[:, d:])
            ops_q, v_q = site("cross_attn.query", dqc, lnc)
            ops, v = site("cross_attn.kv", dkvc, xa)         # [dWk; dWv] in one GEMM
            # d(loss)/d(xa): every decoder layer contributes one (B*1500, d) term.  Instead of 24 separate tensors that
            # autograd adds pairwise (23 elementwise kernels over 98 MB each at medium), the layers accumulate into ONE buffer
            # through the GEMM's residual epilogue (bf16(buf + bf16(acc)), the rounding autograd's bf16 adds would apply);
            # the layer whose backward runs last hands the sum to autograd.
            # No dxa at all when the encoder output takes no gradient (a frozen encoder).
            st = ctx.xa_state
            # FP8: dkvc is quantised here, on the main stream, and kept alive until the side stream is joined
            dk8 = None if (w8 is None or not ctx.needs_input_grad[10]) else K.quantize_fp8_rows(dkvc, K.FP8_E5M2)
            live.append(dk8)
            if not ctx.needs_input_grad[10]:
                pass
            elif st is None:
                dxa = torch.empty_like(xa)
                side.run(lambda: dgrad("wckv", dkvc, ops, v, dk8, out=dxa))
            else:
                first = st["buf"] is None
                if first:
                    st["buf"] = torch.empty_like(xa)
                buf = st["buf"]
                if first:
                    side.run(lambda: dgrad("wckv", dkvc, ops, v, dk8, out=buf))
                else:
                    side.run(lambda: dgrad("wckv", dkvc, ops, v, dk8, epi=K.EPI_BF16_RESIDUAL, aux=buf, out=buf))
                st["left"] -= 1
                dxa = buf if st["left"] == 0 else None
            dlnc = dgrad("wcq", dqc, ops_q, v_q)
            dx1 = K.layernorm_bwd(dlnc, x1, sh["lncw"], meanc, rstdc, grads.vec("cross_attn_ln.weight", d),
                                  grads.vec("cross_attn_ln.bias", d), dresidual=dx2)
        else:
            dx1 = dx2
        # ---- self attention: x1 = x + out(attn(qkv(ln(x))))
        ops, v = site("attn.out", dx1, ao)
        dao = dgrad("wo", dx1, ops, v)
        dqkv = torch.empty_like(qkv)
        if pk is not None:
            K.attention_bwd_varlen(qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:], ao, dao, lse, pk, H,
                                   dq=dqkv[:, :d], dk=dqkv[:, d:2 * d], dv=dqkv[:, 2 * d:])
        else:
            K.attention_bwd(qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:], ao, dao, lse, B, H, T, T, causal=causal, kv_len=kv_len,
                            dq=dqkv[:, :d], dk=dqkv[:, d:2 * d], dv=dqkv[:, 2 * d:])
        ops, v = site("attn.qkv", dqkv, ln1)                 # [dWq; dWk; dWv] in one GEMM
        dx = None
        dw_ln1, db_ln1 = grads.vec("attn_ln.weight", d), grads.vec("attn_ln.bias", d)
        if ctx.needs_input_grad[9] or dw_ln1 is not None or db_ln1 is not None:   # else nothing below the qkv site trains
            dln1 = dgrad("wqkv", dqkv, ops, v)
            dx = K.layernorm_bwd(dln1, x, sh["ln1w"], mean1, rstd1, dw_ln1, db_ln1, dresidual=dx1)
        side.join()
        del live
        grads.done()
        if not ctx.needs_input_grad[9]:
            dx = None
        return (None, None, None, None, None, None, None, None, None, dx, dxa, *grads.grads_for(blk._param_names))


class ResidualAttentionBlock(nn.Module):
    """olmoasr/model.py:445-528 (the FSDP wrap / activation-checkpoint unit of train_fsdp_timestamps.py:2665-2719)."""

    def __init__(self, n_state: int, n_head: int, cross_attention: bool = False, double_init: bool = True):
        super().__init__()
        self.attn = MultiHeadAttention(n_state, n_head, double_init)
        self.attn_ln = LayerNorm(n_state)
        self.cross_attn = MultiHeadAttention(n_state, n_head, double_init) if cross_attention else None
        self.cross_attn_ln = LayerNorm(n_state) if cross_attention else None
        n_mlp = n_state * 4
        self.mlp = nn.Sequential(Linear(n_state, n_mlp), nn.GELU(), Linear(n_mlp, n_state))
        self.mlp_ln = LayerNorm(n_state)
        self._param_names = [n for n, _ in self.named_parameters()]
        self._shadow = _ShadowCache()
        # slab mode (OLMoASRBase.use_slabs): precomputed operand views, gradient-slab targets, completion callback
        self._slabs = None
        self._slab_sh: Optional[Dict[str, Tensor]] = None
        self._slab_sh16: Optional[Dict[str, Tensor]] = None
        self._direct: Optional[Dict[str, Tensor]] = None
        self._bwd_done_cb = None
        self._lora_on = False                             # set by olmoasr_b200.lora.add_lora / merge_lora
        self._lora_cache: Dict[str, _ShadowCache] = {}   # site -> cached adapter operands
        self._fp8_cache = _ShadowCache()                  # FP8 weight copies (fp8_autocast())

    def _build_shadows(self, dtype: torch.dtype = torch.bfloat16) -> Dict[str, Tensor]:
        """Every operand the fused block kernels read that derives from a parameter: 16-bit weights of type `dtype` (fused
        where the GEMMs are fused) and fp32 vectors (biases, LayerNorm affine)."""
        a, c = self.attn, self.cross_attn
        sh: Dict[str, Tensor] = {}
        sh["wqkv"], sh["bqkv"] = a.fused_qkv(dtype)
        sh["wo"], sh["bo"] = a.out.weight16(dtype), _f32(a.out.bias)
        sh["ln1w"], sh["ln1b"] = _f32(self.attn_ln.weight), _f32(self.attn_ln.bias)
        if c is not None:
            sh["wcq"], sh["bcq"] = c.query.weight16(dtype), _f32(c.query.bias)
            sh["wckv"], sh["bckv"] = c.fused_kv(dtype)
            sh["wco"], sh["bco"] = c.out.weight16(dtype), _f32(c.out.bias)
            sh["lncw"], sh["lncb"] = _f32(self.cross_attn_ln.weight), _f32(self.cross_attn_ln.bias)
        sh["w1"], sh["b1"] = self.mlp[0].weight16(dtype), _f32(self.mlp[0].bias)
        sh["w2"], sh["b2"] = self.mlp[2].weight16(dtype), _f32(self.mlp[2].bias)
        sh["ln2w"], sh["ln2b"] = _f32(self.mlp_ln.weight), _f32(self.mlp_ln.bias)
        return sh

    def _shadows(self, dtype: torch.dtype = torch.bfloat16) -> Dict[str, Tensor]:
        if self._slab_sh is not None:
            if dtype == torch.bfloat16:
                return self._slab_sh
            if self._slab_sh16 is None:     # the same slab bytes, read as fp16 (see _slab16)
                self._slab_sh16 = {k: _slab16(v, torch.float16) if v.dtype == torch.bfloat16 else v for k, v in self._slab_sh.items()}
            return self._slab_sh16
        if not _is_master(self.attn.query.weight):
            with torch.no_grad():
                return self._build_shadows(dtype)   # FSDP mixed precision: parameters are transient views, never cached
        base = [p for n, p in self.named_parameters() if ".lora_" not in n]   # adapter updates leave the base shadows alone
        return self._shadow.get(base, lambda: self._build_shadows(dtype), dtype)

    def _build_fp8_weights(self, sh: Dict[str, Tensor]) -> Dict[str, tuple]:
        """Weight key of `_FP8_WEIGHTS` -> ((W8, s), (W^T8, s)): the e4m3 rows of the 16-bit operand W (N, K), for the
        forward, and of W^T (K, N), i.e. one scale per input feature, for the dgrad."""
        return {k: (K.quantize_fp8_rows(sh[k], K.FP8_E4M3), K.quantize_fp8_rows(sh[k], K.FP8_E4M3, transpose=True))
                for k in _FP8_WEIGHTS if k in sh}

    def _fp8_weights(self, sh: Dict[str, Tensor]) -> Dict[str, tuple]:
        """The FP8 weight copies of the 16-bit operands `sh`: rebuilt when a parameter changed (once per optimizer
        step), or on every call under FSDP, whose unsharded views are transient like the 16-bit operands."""
        if not _is_master(self.attn.query.weight):
            with torch.no_grad():
                return self._build_fp8_weights(sh)
        base = [p for n, p in self.named_parameters() if ".lora_" not in n]
        return self._fp8_cache.get(base, lambda: self._build_fp8_weights(sh), torch.float8_e4m3fn)

    def _lora_sites(self):
        """Projection site of the fused block -> its Linears (in `_FUSED` member order)."""
        a, c = self.attn, self.cross_attn
        sites = {"attn.qkv": (a.query, a.key, a.value), "attn.out": (a.out,)}
        if c is not None:
            sites.update({"cross_attn.query": (c.query,), "cross_attn.kv": (c.key, c.value), "cross_attn.out": (c.out,)})
        sites.update({"mlp.0": (self.mlp[0],), "mlp.2": (self.mlp[2],)})
        return sites

    def _lora_ops(self, dtype: torch.dtype) -> Dict[str, _LoraOps]:
        """Site -> `_LoraOps` for every site with an adapter (empty without adapters)."""
        if not self._lora_on:
            return {}
        out = {}
        for name, lins in self._lora_sites().items():
            ops = _LoraOps.of(lins, self._lora_cache.setdefault(name, _ShadowCache()), dtype)
            if ops is not None:
                out[name] = ops
        return out

    def forward(self, x: Tensor, xa: Optional[Tensor] = None, mask: Optional[Tensor] = None,
                kv_cache: Optional[dict] = None, verbose: bool = False, _xa_state: Optional[dict] = None,
                _packed: Optional[PackedBatch] = None, _fp8: Optional[dict] = None):
        if kv_cache is not None:
            return self._forward_cached(x, xa, mask, kv_cache)
        # inside fp8_autocast(): the FP8 operands the layers share, unless the decoder quantised them for all layers
        f8 = (_fp8 if _fp8 is not None else fp8_inputs(xa)) if fp8_enabled() else None
        if _packed is not None:      # x: the (N, d) rows of a packed decoder batch (TextDecoder.hidden)
            params = [_attr_by_path(self, n) for n in self._param_names]
            xa2 = _as16_2d(xa, x.dtype)
            return _BlockFn.apply(self, _packed.B, _packed.S, xa.shape[1], True, None, _xa_state, _packed, f8, x, xa2, *params)
        B, T, d = x.shape
        causal, kv_len = False, None
        if mask is not None:
            causal = True
            if mask.dim() == 3:
                kv_len = kv_len_from_padding_mask(mask)
        Ta = xa.shape[1] if xa is not None else 0
        dt = x.dtype if x.dtype in K.ACT16 else torch.bfloat16
        xa2 = _as16_2d(xa, dt) if xa is not None else None
        # attribute walk, not get_parameter(): under FSDP the attributes are plain tensor views of the flat parameter
        params = [_attr_by_path(self, n) for n in self._param_names]
        y = _BlockFn.apply(self, B, T, Ta, causal, kv_len, _xa_state, None, f8, _as16_2d(x, dt), xa2, *params)
        return y.view(B, T, d)

    def _forward_cached(self, x, xa, mask, kv_cache):
        """Decode path: unfused modules so that the forward hooks on key / value fire (model.py:925-964)."""
        B, T, d = x.shape
        dt = compute_dtype()     # the type the Linear / LayerNorm modules below compute in
        x = x + self.attn(self.attn_ln(x), mask=mask, kv_cache=kv_cache)[0]
        if self.cross_attn is not None:
            x = x + self.cross_attn(self.cross_attn_ln(x), xa, kv_cache=kv_cache)[0]
        h, g = linear_fwd(_as16_2d(self.mlp_ln(x), dt), self.mlp[0].weight16(dt), _f32(self.mlp[0].bias), epi=K.EPI_BF16_GELU)
        y = linear_fwd(g, self.mlp[2].weight16(dt), _f32(self.mlp[2].bias), epi=K.EPI_BF16_RESIDUAL, aux=_as16_2d(x, dt))
        return y.view(B, T, d)


# =====================================================================================================
# encoder
# =====================================================================================================
class _StemFn(torch.autograd.Function):
    """conv1 -> GELU -> conv2 (stride 2) -> GELU -> transpose -> + sinusoids (model.py:592-602) as
    im2col + wgmma GEMM with fused bias/GELU epilogues, time-major throughout."""

    @staticmethod
    def forward(ctx, enc, mel, w1, b1, w2, b2, dtype=torch.bfloat16):
        B, C, T = mel.shape
        d = w1.shape[0]
        T2 = (T + 2 - 3) // 2 + 1
        mel = mel.contiguous()
        if mel.dtype != torch.float32:        # FSDP MixedPrecision hands the root module a bf16 mel, as it does to the reference
            mel = K.convert(mel, dtype=torch.float32)
        A1 = K.im2col_conv1(mel, 3 * C, **_f16_kw(dtype))
        pre1, h1 = linear_fwd(A1, enc.conv1.weight16(dtype), _f32(b1), epi=K.EPI_BF16_GELU)
        A2 = K.im2col_conv2(h1, B, T, d)
        pre2, h2 = linear_fwd(A2, enc.conv2.weight16(dtype), _f32(b2), epi=K.EPI_BF16_GELU)
        x0 = K.add_pos(h2, _f32(enc.positional_embedding), T2)
        ctx.save_for_backward(A1, pre1, A2, pre2)
        ctx.enc, ctx.dims = enc, (B, C, T, T2, d)
        return x0

    @staticmethod
    def backward(ctx, dx0):
        A1, pre1, A2, pre2 = ctx.saved_tensors
        enc = ctx.enc
        B, C, T, T2, d = ctx.dims
        grads = _GradDest(enc, dx0.device)
        dpre2 = K.gelu_bwd(dx0.contiguous(), pre2)
        if grads.wants("conv2.weight"):
            grads.keep("conv2.weight", K.unpermute_conv_wgrad(linear_wgrad(dpre2, A2), d, d, out=grads.out("conv2.weight")))
        grads.bias("conv2.bias", dpre2)
        if grads.wants("conv1.weight") or grads.wants("conv1.bias"):
            dA2 = linear_dgrad(dpre2, enc.conv2.weight16(pre2.dtype))
            dpre1 = K.col2im_conv2_gelu_bwd(dA2, pre1, B, T, T2, d)
            if grads.wants("conv1.weight"):
                grads.keep("conv1.weight", K.unpermute_conv_wgrad(linear_wgrad(dpre1, A1), d, C, out=grads.out("conv1.weight")))
            grads.bias("conv1.bias", dpre1)
        grads.done()     # last gradients of the whole backward pass
        return (None, None, *grads.grads_for(("conv1.weight", "conv1.bias", "conv2.weight", "conv2.bias")), None)


class AudioEncoder(nn.Module):
    """olmoasr/model.py:531-623."""

    def __init__(self, n_mels: int, n_ctx: int, n_state: int, n_head: int, n_layer: int, double_init: bool = True):
        super().__init__()
        self.conv1 = Conv1d(n_mels, n_state, kernel_size=3, padding=1)
        self.conv2 = Conv1d(n_state, n_state, kernel_size=3, stride=2, padding=1)
        self.register_buffer("positional_embedding", sinusoids(n_ctx, n_state))
        self.blocks: Iterable[ResidualAttentionBlock] = nn.ModuleList(
            [ResidualAttentionBlock(n_state, n_head, double_init=double_init) for _ in range(n_layer)])
        self.ln_post = LayerNorm(n_state)
        self._slabs = None
        self._direct: Optional[Dict[str, Tensor]] = None
        self._bwd_done_cb = None

    def forward(self, x: Tensor, verbose: bool = False):
        dt = compute_dtype()
        if self._slabs is not None:
            self._slabs.ensure_synced(dt)
        B = x.shape[0]
        n_ctx, d = self.positional_embedding.shape
        assert x.dim() == 3 and (x.shape[2] + 2 - 3) // 2 + 1 == n_ctx and x.shape[1] == self.conv1.in_channels, \
            "incorrect audio shape"
        x0 = _StemFn.apply(self, x, self.conv1.weight, self.conv1.bias, self.conv2.weight, self.conv2.bias, dt)
        h = x0.view(B, n_ctx, d)
        for block in self.blocks:
            h = block(h)
        return _LayerNormFn.apply(h.reshape(B * n_ctx, d), self.ln_post.weight, self.ln_post.bias, self.ln_post.eps,
                                  self, "ln_post").view(B, n_ctx, d)


class _LayerNormFn(torch.autograd.Function):
    """Final LayerNorm of the encoder / decoder, whose parameters are `owner`'s `key + ".weight"` / `key + ".bias"`."""

    @staticmethod
    def forward(ctx, x, w, b, eps, owner, key):
        y, mean, rstd = K.layernorm_fwd(x, _f32(w), _f32(b), eps)
        ctx.save_for_backward(x, w, mean, rstd)
        ctx.owner, ctx.key = owner, key
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, mean, rstd = ctx.saved_tensors
        w = _f32(w)
        grads, names = _GradDest(ctx.owner, w.device), (ctx.key + ".weight", ctx.key + ".bias")
        dw, db = grads.vec(names[0], w.shape), grads.vec(names[1], w.shape)
        dx = K.layernorm_bwd(dy.contiguous(), x, w, mean, rstd, dw, db)
        return (dx, *grads.grads_for(names), None, None, None)


# =====================================================================================================
# decoder
# =====================================================================================================
class _EmbedFn(torch.autograd.Function):
    """(token_embedding(ids) + positional_embedding[offset:offset+S]).to(dtype)  (model.py:728-732); with a PackedBatch
    `pk` only its N rows, (N, d)."""

    @staticmethod
    def forward(ctx, ids, emb, pos, offset, padding_idx, dec=None, dtype=torch.bfloat16, pk=None):
        if pk is not None:
            out = K.embed_fwd_packed(ids.contiguous(), _f32(emb), _f32(pos), pk, dtype)
        else:
            out = K.embed_fwd(ids.contiguous(), _f32(emb), _f32(pos), offset, **_f16_kw(dtype))
        ctx.save_for_backward(ids)
        ctx.meta = (emb.shape, pos.shape, offset, padding_idx)
        ctx.dec, ctx.pk = dec, pk
        return out

    @staticmethod
    def backward(ctx, dx):
        (ids,) = ctx.saved_tensors
        eshape, pshape, offset, padding_idx = ctx.meta
        pad = -1 if padding_idx is None else padding_idx
        grads, names = _GradDest(ctx.dec, dx.device), ("token_embedding.weight", "positional_embedding")
        # in direct mode a scatter-add straight into the slab, where the tied logits wgrad has already accumulated
        demb, dpos = grads.vec(names[0], eshape), grads.vec(names[1], pshape)
        if demb is None and dpos is None:
            grads.done()
            return (None, None, None, None, None, None, None, None)
        if ctx.pk is not None:        # a null target (frozen) skips its sums
            K.embed_bwd_packed(ids.contiguous(), dx.contiguous(), demb, dpos, ctx.pk, pad)
        elif dpos is None:
            K.embed_bwd(ids.contiguous(), dx.contiguous(), demb, None, pad)
        else:
            K.embed_bwd(ids.contiguous(), dx.contiguous(), demb, dpos[offset:], pad)
        grads.done()     # decoder gradients (incl. the tied embedding) are final
        return (None, *grads.grads_for(names), None, None, None, None, None)


def _logits_ld(V: int) -> int:
    return (V + 255) // 256 * 256  # 51865 -> 51968: no ragged tile in the logits GEMM, 16-byte aligned rows


class _LogitsFn(torch.autograd.Function):
    """(x @ token_embedding.weight.to(x.dtype).T).float()  (model.py:768-770) for callers that want logits."""

    @staticmethod
    def forward(ctx, x, emb, emb_bf16, dec=None):
        M, d = x.shape
        V = emb.shape[0]
        buf = torch.empty((M, _logits_ld(V)), device=x.device, dtype=x.dtype)
        K.gemm(x, emb_bf16, M, V, d, out=buf, block_n=256)
        ctx.save_for_backward(x, emb_bf16)
        ctx.dec = dec
        return K.logits_to_f32(buf, V)

    @staticmethod
    def backward(ctx, dlogits):
        x, emb_bf16 = ctx.saved_tensors
        M, d = x.shape
        V = emb_bf16.shape[0]
        buf = torch.empty((M, _logits_ld(V)), device=x.device, dtype=x.dtype)
        buf[:, :V].copy_(dlogits)  # `.float()` backward: the gradient enters the matmul in the logits' 16-bit type
        dx = K.gemm(buf[:, :V], emb_bf16, M, d, V, b_mn=True, block_n=_pick_block_n(M, d))
        grads = _GradDest(ctx.dec)
        if grads.wants("token_embedding.weight"):
            grads.weight("token_embedding.weight", buf, x, n_valid=V)
        return (dx, *grads.grads_for(("token_embedding.weight",)), None, None)


class _LossHeadFn(torch.autograd.Function):
    """Fused tail of the training step: tied logits GEMM (16-bit, never widened to fp32) + token cross-entropy
    (model.py:768-770 followed by train_timestamps.py:1444-1448).  The backward turns the logits buffer into
    d(logits) in place and feeds it to the dgrad / wgrad GEMMs."""

    @staticmethod
    def forward(ctx, x, emb, emb_bf16, targets, ignore_index, dec=None):
        ctx.dec = dec
        M, d = x.shape
        V = emb.shape[0]
        buf = torch.empty((M, _logits_ld(V)), device=x.device, dtype=x.dtype)
        K.gemm(x, emb_bf16, M, V, d, out=buf, block_n=256)
        t = targets.reshape(-1).contiguous()
        lse, lsc = K.ce_fwd(buf, t, V, ignore_index)
        ctx.save_for_backward(x, emb_bf16, buf, t, lse, lsc)
        ctx.meta = (V, ignore_index)
        ctx.consumed = [False]
        return K.ce_finalize(lsc)

    @staticmethod
    def backward(ctx, dloss):
        x, emb_bf16, buf, t, lse, lsc = ctx.saved_tensors
        V, ignore_index = ctx.meta
        M, d = x.shape
        if ctx.consumed[0]:
            raise RuntimeError("the fused loss head keeps d(logits) in the logits buffer: backward through it twice "
                               "(retain_graph) is not supported")
        ctx.consumed[0] = True
        K.ce_bwd_(buf, t, lse, lsc, dloss.reshape(1).float().contiguous(), V, ignore_index)
        dx = K.gemm(buf[:, :V], emb_bf16, M, d, V, b_mn=True, block_n=_pick_block_n(M, d))
        grads = _GradDest(ctx.dec)
        if grads.wants("token_embedding.weight"):
            grads.weight("token_embedding.weight", buf, x, n_valid=V)
        return (dx, *grads.grads_for(("token_embedding.weight",)), None, None, None, None)


class TextDecoder(nn.Module):
    """olmoasr/model.py:626-775 (train_vocab_pad=True: n_vocab+1 rows with padding_idx) and
    olmoasr/inf_model.py:284-362 (train_vocab_pad=False)."""

    def __init__(self, n_vocab: int, n_ctx: int, n_state: int, n_head: int, n_layer: int, train_vocab_pad: bool = True):
        super().__init__()
        if train_vocab_pad:
            self.token_embedding = nn.Embedding(n_vocab + 1, n_state, padding_idx=51864 if n_vocab == 51864 else 51865)
        else:
            self.token_embedding = nn.Embedding(n_vocab, n_state)
        nn.init.kaiming_normal_(self.token_embedding.weight, mode="fan_in", nonlinearity="relu")
        self.positional_embedding = nn.Parameter(torch.empty(n_ctx, n_state))
        if train_vocab_pad:
            nn.init.kaiming_normal_(self.positional_embedding, mode="fan_in", nonlinearity="relu")
        self.blocks: Iterable[ResidualAttentionBlock] = nn.ModuleList(
            [ResidualAttentionBlock(n_state, n_head, cross_attention=True, double_init=train_vocab_pad) for _ in range(n_layer)])
        self.ln = LayerNorm(n_state)
        mask = torch.empty(n_ctx, n_ctx).fill_(-np.inf).triu_(1)
        self.register_buffer("mask", mask, persistent=False)
        self._emb_shadow = _ShadowCache()
        self._slabs = None
        self._direct: Optional[Dict[str, Tensor]] = None
        self._bwd_done_cb = None
        self._emb_slab_view: Optional[Tensor] = None

    def embedding_bf16(self) -> Tensor:
        return self.embedding16(torch.bfloat16)

    def embedding16(self, dtype: torch.dtype) -> Tensor:
        if self._emb_slab_view is not None:
            return _slab16(self._emb_slab_view, dtype)
        w = self.token_embedding.weight
        if w.dtype == dtype:
            return w.detach()
        if not _is_master(w):
            return K.convert(w.detach().contiguous(), dtype=dtype)
        return self._emb_shadow.get((w,), lambda: _cast16(w.detach().contiguous(), dtype), dtype)

    def hidden(self, x: Tensor, xa: Tensor, kv_cache: Optional[dict] = None, padding_mask: Optional[Tensor] = None,
               dtype: Optional[torch.dtype] = None, packed: Optional[PackedBatch] = None) -> Tensor:
        """Everything up to and including the final LayerNorm: (B, S) ids -> (B*S, d) in `dtype` (default: compute_dtype()),
        or -> (N, d) for the rows of a PackedBatch."""
        dt = compute_dtype() if dtype is None else dtype
        if self._slabs is not None:
            self._slabs.ensure_synced(dt)
        offset = next(iter(kv_cache.values())).shape[1] if kv_cache else 0
        B, S = x.shape
        d = self.positional_embedding.shape[1]
        # shared accumulator of the layers' gradients w.r.t. the encoder output (see _BlockFn.backward); one per forward pass
        xa_state = {"buf": None, "left": len(self.blocks)} if (kv_cache is None and torch.is_grad_enabled() and xa.requires_grad) else None
        # fp8_autocast(): the encoder output feeds every layer's cross K/V projection; quantise it once, here on the main
        # stream, so that each layer's side-stream GEMM is ordered after it
        kw = {} if xa_state is None else {"_xa_state": xa_state}
        if kv_cache is None and fp8_enabled() and dt == torch.bfloat16:
            kw["_fp8"] = fp8_inputs(xa)
        if packed is not None:
            h = _EmbedFn.apply(x, self.token_embedding.weight, self.positional_embedding, 0, self.token_embedding.padding_idx,
                               self, dt, packed)
            for block in self.blocks:
                h = block(h, xa, _packed=packed, **kw)
            return _LayerNormFn.apply(h, self.ln.weight, self.ln.bias, self.ln.eps, self, "ln")
        h = _EmbedFn.apply(x, self.token_embedding.weight, self.positional_embedding, offset,
                           self.token_embedding.padding_idx, self, dt).view(B, S, d)
        mask = padding_mask if padding_mask is not None else self.mask[:S, :S]
        for block in self.blocks:
            h = block(h, xa, mask=mask, kv_cache=kv_cache, **kw)
        return _LayerNormFn.apply(h.reshape(B * S, d), self.ln.weight, self.ln.bias, self.ln.eps, self, "ln")

    def forward(self, x: Tensor, xa: Tensor, kv_cache: Optional[dict] = None, padding_mask: Optional[Tensor] = None,
                verbose: bool = False):
        B, S = x.shape
        dt = compute_dtype()
        h = self.hidden(x, xa, kv_cache, padding_mask, dt)
        logits = _LogitsFn.apply(h, self.token_embedding.weight, self.embedding16(dt), self)
        return logits.view(B, S, -1)

    def loss(self, x: Tensor, xa: Tensor, targets: Tensor, padding_mask: Optional[Tensor] = None, ignore_index: int = PAD_ID_EN,
             text_lens=None):
        """Mean token cross-entropy.  With `text_lens` (host-side lengths, one per sample) the decoder runs on each
        sample's first text_lens[b] rows only; targets at t >= text_lens[b] count as ignored.  That is the loss of the
        dense call with the reference's padding mask for those lengths (train_timestamps.py:314-315)."""
        dt = compute_dtype()
        if text_lens is None:
            h = self.hidden(x, xa, None, padding_mask, dt)
            return _LossHeadFn.apply(h, self.token_embedding.weight, self.embedding16(dt), targets, ignore_index, self)
        lens = packed_text_lens(text_lens, x, targets, padding_mask)
        pk = PackedBatch(lens, x.shape[1], x.device)
        h = self.hidden(x, xa, None, None, dt, packed=pk)
        t = targets.reshape(-1).index_select(0, pk.rows)
        return _LossHeadFn.apply(h, self.token_embedding.weight, self.embedding16(dt), t, ignore_index, self)


# =====================================================================================================
# top-level model
# =====================================================================================================
class OLMoASRBase(nn.Module):
    """olmoasr/model.py:778-968 / olmoasr/inf_model.py:365-457."""

    _train_vocab_pad = True

    def __init__(self, dims: ModelDimensions):
        super().__init__()
        self.dims = dims
        tv = self._train_vocab_pad
        self.encoder = AudioEncoder(dims.n_mels, dims.n_audio_ctx, dims.n_audio_state, dims.n_audio_head,
                                    dims.n_audio_layer, double_init=tv)
        self.decoder = TextDecoder(dims.n_vocab, dims.n_text_ctx, dims.n_text_state, dims.n_text_head,
                                   dims.n_text_layer, train_vocab_pad=tv)

    # ---- slab mode ------------------------------------------------------------------------------------------
    def use_slabs(self, direct_grads: bool = True):
        """Move parameters, gradients and bf16 weight shadows into contiguous slabs (olmoasr_b200/slab.py) laid out in
        backward-completion order, and hand every fused block precomputed views: the fused [Wq;Wk;Wv] / [Wk;Wv] weights
        and [bq;0;bv] biases ARE slab ranges, weight gradients are accumulated in place by the wgrad GEMM epilogues.
        Call after `.to(device)`; `state_dict()` names, shapes and values are unchanged.  Returns the ParamSlabs
        (pass it to FusedAdamW(slabs=...) and, for data parallelism, to olmoasr_b200.ddp.SlabGradSync).

        direct_grads=False keeps the hand-over of gradients through autograd (needed under torch DDP / FSDP hooks)."""
        from .slab import ParamSlabs

        if getattr(self, "_slabs", None) is not None:
            self._slabs.direct_grads = direct_grads
            return self._slabs
        d_enc = self.dims.n_audio_state
        if d_enc % 64 or self.dims.n_text_state % 64:
            raise ValueError("use_slabs: model widths must be multiples of 64")

        def lora(*lins):   # adapters sit with their site, so a block's parameters stay one run of the layout
            return [p for lin in lins if lin.has_lora for p in (lin.lora_A, lin.lora_B)]

        def mha_items(a: "MultiHeadAttention"):
            d = a.query.weight.shape[0]
            return ([a.out.weight, a.out.bias] + lora(a.out) + [a.query.weight, a.key.weight, a.value.weight, a.query.bias,
                    d, a.value.bias] + lora(a.query, a.key, a.value))

        def block_items(b: "ResidualAttentionBlock"):
            it = [b.mlp_ln.weight, b.mlp_ln.bias, b.mlp[2].weight, b.mlp[2].bias] + lora(b.mlp[2])
            it += [b.mlp[0].weight, b.mlp[0].bias] + lora(b.mlp[0])
            if b.cross_attn is not None:
                it += [b.cross_attn_ln.weight, b.cross_attn_ln.bias] + mha_items(b.cross_attn)
            it += [b.attn_ln.weight, b.attn_ln.bias] + mha_items(b.attn)
            return it

        enc, dec = self.encoder, self.decoder
        layout = [dec.ln.weight, dec.ln.bias]
        for b in reversed(list(dec.blocks)):
            layout += block_items(b)
        layout += [dec.token_embedding.weight, dec.positional_embedding, enc.ln_post.weight, enc.ln_post.bias]
        for b in reversed(list(enc.blocks)):
            layout += block_items(b)
        layout += [enc.conv2.weight, enc.conv2.bias, enc.conv1.weight, enc.conv1.bias]
        # Only what trains is laid out.  The zero gap of a [bq; 0; bv] bias stays when both biases train.
        keep = []
        for i, it in enumerate(layout):
            if isinstance(it, int):
                if layout[i - 1].requires_grad and layout[i + 1].requires_grad:
                    keep.append(it)
            elif it.requires_grad:
                keep.append(it)
        if not any(not isinstance(it, int) for it in keep):
            raise ValueError("use_slabs: the model has no trainable parameter")
        sl = ParamSlabs(self, keep)
        sl.direct_grads = direct_grads

        def install_mha(a: "MultiHeadAttention"):
            d = a.query.weight.shape[0]
            group = (a.query.weight, a.key.weight, a.value.weight, a.query.bias, a.value.bias)
            if all(p.requires_grad for p in group):   # the fused [Wq;Wk;Wv] / [bq;0;bv] operands ARE slab ranges
                assert sl.adjacent(a.query.weight, a.key.weight, a.value.weight)
                assert sl.offset[id(a.value.bias)] == sl.offset[id(a.query.bias)] + 2 * d
                a._slab_fused = (sl.span("S", a.query.weight, 3 * d * d).view(3 * d, d), sl.span("P", a.query.bias, 3 * d))
            # else the fused shadow is built from the members' masters (slab views for those that train) and cached
            # on their versions, which the fused optimizer bumps
            for lin in (a.query, a.key, a.value, a.out):
                if lin.weight.requires_grad:
                    lin._slab_view = sl.shadow(lin.weight)

        def grad_views(mod: nn.Module) -> Dict[str, Tensor]:   # the gradients its own backward writes, by name
            return {n: sl.grad(p) for n, p in mod.named_parameters() if not n.startswith("blocks.") and p.requires_grad}

        for b in list(enc.blocks) + list(dec.blocks):
            install_mha(b.attn)
            if b.cross_attn is not None:
                install_mha(b.cross_attn)
            for lin in (b.mlp[0], b.mlp[2]):
                if lin.weight.requires_grad:
                    lin._slab_view = sl.shadow(lin.weight)
            direct = grad_views(b)
            for name, members in _FUSED.items():     # a fused weight gradient is the slab span of its adjacent members
                if all(m + ".weight" in direct for m in members):
                    w = _attr_by_path(b, members[0]).weight
                    direct[name + ".weight"] = sl.span("G", w, len(members) * w.numel()).view(len(members) * w.shape[0], -1)
            # A block whose base parameters all train reads slab views throughout (16-bit weights from S, fp32 vectors
            # from P).  Otherwise its frozen weights keep their cached shadows, and its operand dictionary is cached on
            # the parameters' versions like outside slab mode (_shadows).
            full = all(p.requires_grad for n, p in b.named_parameters() if ".lora_" not in n)
            b._slabs, b._slab_sh, b._slab_sh16, b._direct = sl, (b._build_shadows() if full else None), None, direct
        enc._slabs, dec._slabs = sl, sl
        enc._direct, dec._direct = grad_views(enc), grad_views(dec)
        if dec.token_embedding.weight.requires_grad:
            dec._emb_slab_view = sl.shadow(dec.token_embedding.weight)
        self._slabs = sl
        if sl.device.type == "cuda":
            sl.sync_shadows()
        return sl

    def grad_units(self):
        """[(parameters, module whose `_bwd_done_cb` fires when their gradients are final | None)] in the order the
        backward pass completes them (= slab layout order); consumed by olmoasr_b200.ddp.SlabGradSync."""
        enc, dec = self.encoder, self.decoder
        units = [([dec.ln.weight, dec.ln.bias], None)]
        units += [(list(b.parameters()), b) for b in reversed(list(dec.blocks))]
        units.append(([dec.token_embedding.weight, dec.positional_embedding], dec))
        units.append(([enc.ln_post.weight, enc.ln_post.bias], None))
        units += [(list(b.parameters()), b) for b in reversed(list(enc.blocks))]
        units.append(([enc.conv2.weight, enc.conv2.bias, enc.conv1.weight, enc.conv1.bias], enc))
        # the trainable parameters only (what the slabs hold); a unit with none left drops out
        units = [([p for p in ps if p.requires_grad], mod) for ps, mod in units]
        return [(ps, mod) for ps, mod in units if ps]

    def embed_audio(self, mel: Tensor):
        return self.encoder(mel)

    def logits(self, tokens: Tensor, audio_features: Tensor, padding_mask: Tensor = None):
        return self.decoder(tokens, audio_features, padding_mask=padding_mask)

    def forward(self, mel: Tensor, tokens: Tensor, padding_mask: Tensor = None, verbose: bool = False, *,
                targets: Optional[Tensor] = None, ignore_index: int = PAD_ID_EN, text_lens=None) -> Tensor:
        """Reference signature (model.py:856-887) -> fp32 logits.  With the keyword-only `targets` the call returns
        the token cross-entropy instead (fused head); going through forward() keeps DDP / FSDP wrappers in the loop.
        `text_lens` (with `targets`, instead of `padding_mask`): see `loss`."""
        if text_lens is not None:
            packed_text_lens(text_lens, tokens, targets, padding_mask)    # reject a bad call before the encoder runs
        if targets is not None:
            return self.decoder.loss(tokens, self.encoder(mel), targets, padding_mask, ignore_index, text_lens)
        return self.decoder(tokens, self.encoder(mel), padding_mask=padding_mask)

    def loss(self, mel: Tensor, tokens: Tensor, targets: Tensor, padding_mask: Tensor = None, ignore_index: int = PAD_ID_EN,
             text_lens=None):
        """Fused equivalent of `F.cross_entropy(model(mel, tokens, padding_mask).view(-1, V), targets.view(-1),
        ignore_index=51864)` (train_timestamps.py:1440-1448) that never materialises fp32 logits.

        text_lens: host-side lengths (a CPU integer tensor or a sequence of ints, 1 <= text_lens[b] <= tokens.shape[1]),
        e.g. the `len(text_input)` a loader computes per sample, in place of `padding_mask`.  The decoder then runs on
        each transcript's own rows only, packed back to back, and returns the loss of the dense call with the reference's
        padding mask for those lengths, targets at t >= text_lens[b] counting as ignored."""
        if text_lens is not None:
            packed_text_lens(text_lens, tokens, targets, padding_mask)
        return self.decoder.loss(tokens, self.encoder(mel), targets, padding_mask, ignore_index, text_lens)

    @property
    def device(self):
        return next(self.parameters()).device

    @property
    def is_multilingual(self):
        return self.dims.n_vocab >= 51865

    @property
    def num_languages(self):
        return self.dims.n_vocab - 51765 - int(self.is_multilingual)

    # ---- word-timestamp alignment heads -------------------------------------------------------------------------
    # A plain attribute, not a buffer: state_dict(), buffers(), the slab layout and FSDP see exactly the parameters and
    # buffers of the reference.  Default as upstream Whisper: every head of the upper half of the decoder layers.
    _alignment_mask: Optional[Tensor] = None

    @property
    def alignment_heads(self) -> Tensor:
        """Sparse bool (n_text_layer, n_text_head) tensor of the cross-attention heads word timestamps align with;
        `.indices()` lists them in ascending (layer, head) order."""
        if self._alignment_mask is None:
            mask = torch.zeros(self.dims.n_text_layer, self.dims.n_text_head, dtype=torch.bool)
            mask[self.dims.n_text_layer // 2:] = True
            self._alignment_mask = mask
        return self._alignment_mask.to_sparse()

    def set_alignment_heads(self, dump):
        """Select the alignment heads: upstream's base85-encoded gzip dump of the bool mask (bytes or str), or a bool
        array / tensor of shape (n_text_layer, n_text_head)."""
        shape = (self.dims.n_text_layer, self.dims.n_text_head)
        if isinstance(dump, (bytes, str)):
            import base64
            import gzip
            array = np.frombuffer(gzip.decompress(base64.b85decode(dump)), dtype=bool).copy()
            if array.size != shape[0] * shape[1]:
                raise ValueError(f"alignment-head dump has {array.size} entries, the model has {shape[0]} x {shape[1]} heads")
            mask = torch.from_numpy(array).reshape(shape)
        else:
            mask = torch.as_tensor(dump)
            if mask.is_sparse:
                mask = mask.to_dense()
            if mask.dtype != torch.bool or tuple(mask.shape) != shape:
                raise ValueError(f"alignment heads must be a bool {shape} mask, got {mask.dtype} {tuple(mask.shape)}")
            mask = mask.detach().cpu().clone()
        if not bool(mask.any()):
            raise ValueError("at least one alignment head is needed")
        self._alignment_mask = mask

    def install_kv_cache_hooks(self, cache: Optional[dict] = None):
        """The reference's kv-cache protocol (model.py:925-964 / inf_model.py:422-453), kept for third-party loops
        (whisper.decoding.PyTorchInference) and for this package's sampling / timestamp-rule paths: forward hooks on every
        decoder key / value Linear, a dict keyed by module identity, cross-attention outputs (longer than n_text_ctx) stored
        once.  Unlike the reference there is no torch.cat per step: each self-attention projection owns one pre-allocated
        (B, n_text_ctx, d) buffer, new rows are written behind the cached ones and the dict entry is a growing VIEW of it.
        (The greedy fast path does not come through here at all: olmoasr_b200/decode_engine.py.)"""
        store = _KVCacheStore(self.dims.n_text_ctx, dict(cache) if cache is not None else {})
        hooks = []
        for blk in self.decoder.blocks:
            for att in (blk.attn, blk.cross_attn):
                if att is not None:
                    hooks.append(att.key.register_forward_hook(store.on_projection))
                    hooks.append(att.value.register_forward_hook(store.on_projection))
        return store.cache, hooks

    def decode_engine(self, dtype: torch.dtype = torch.float16, max_batch: int = 64, *, fp8: bool = False):
        """The device-resident greedy decoder for this model (one per activation dtype, batch and weight storage, built on
        first use); `fp8=True` is the engine with e4m3 block weights and cross K / V (DecodingOptions.fp8)."""
        from .decode_engine import DecodeEngine

        engines = self.__dict__.setdefault("_engines", {})
        key = (dtype, max_batch, bool(fp8))
        if key not in engines:
            engines[key] = DecodeEngine(self, dtype, max_batch, fp8=bool(fp8))
        return engines[key]


class _KVCacheStore:
    """Backing storage of `install_kv_cache_hooks`: module -> (buffer, rows in use)."""

    def __init__(self, n_text_ctx: int, cache: dict):
        self.n_text_ctx = n_text_ctx
        self.cache = cache
        self.buffers: Dict[nn.Module, Tensor] = {}

    def on_projection(self, module, _inputs, output: Tensor):
        rows = output.shape[1]
        if rows > self.n_text_ctx:                     # cross-attention keys / values of the 1500 audio frames: computed once
            self.cache[module] = output
            return output
        buf = self.buffers.get(module)
        used = self.cache[module].shape[1] if (buf is not None and module in self.cache) else 0
        if buf is None or buf.shape[0] != output.shape[0] or buf.dtype != output.dtype or used + rows > buf.shape[1]:
            buf = torch.empty((output.shape[0], max(self.n_text_ctx, rows), output.shape[2]), device=output.device, dtype=output.dtype)
            self.buffers[module] = buf
            used = 0
        buf[:, used:used + rows] = output.detach()
        self.cache[module] = buf[:, :used + rows]
        return self.cache[module]
