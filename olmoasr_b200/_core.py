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
    path when they are called inside an fp16 autocast region."""
    global _bf16_pinned
    _bf16_pinned += 1
    try:
        yield
    finally:
        _bf16_pinned -= 1


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

    def vec(self, key: str, shape) -> Tensor:
        """Zero-initialised accumulation target of `key`'s gradient (LayerNorm, embedding and bias vectors)."""
        return self.slab[key] if self.slab is not None else self.keep(key, self._zeros(shape))

    def _launch(self, fn):
        return self.side.run(fn) if self.side is not None else fn()

    def weight(self, key: str, dy: Tensor, x: Tensor, n_valid: Optional[int] = None) -> Tensor:
        return self.keep(key, linear_wgrad(dy, x, n_valid, side=self.side, out=self.out(key)))

    def bias(self, key: str, dy: Tensor):
        """Column sums of dy (M, n) bf16 into the bias gradient `key`."""
        db = self.vec(key, dy.shape[1])
        self._launch(lambda: K.colsum_(dy, db, dy.shape[1]))

    def linear(self, name: str, dy: Tensor, x: Tensor):
        """Weight and bias gradients of the Linear `name`, or of the projections `_FUSED[name]`, from the output
        gradient dy and the input x."""
        dw = self.weight(name + ".weight", dy, x)
        members = _FUSED.get(name)
        if members is None:
            return self.bias(name + ".bias", dy)
        d = dw.shape[0] // len(members)
        if self.slab is not None:      # one column sum per member that has a bias, so no gap of the slab is written
            for i, m in enumerate(members):
                if m + ".bias" in self.slab:
                    self.bias(m + ".bias", dy[:, i * d:(i + 1) * d])
            return
        self.bias(name + ".bias", dy)  # one column sum over the whole fused width; every member takes its rows
        for i, m in enumerate(members):
            for kind in (".weight", ".bias"):
                self.grads[m + kind] = self.grads[name + kind][i * d:(i + 1) * d]

    def grads_for(self, names: Iterable[str]) -> tuple:
        """What autograd receives for these parameters: all None in direct mode, where the slab already holds them."""
        if self.slab is not None:
            return tuple(None for _ in names)
        return tuple(self.grads[n] for n in names)

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
        y = linear_fwd(_as16_2d(x, dt), self.weight16(dt), None if self.bias is None else _f32(self.bias))
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
class _BlockFn(torch.autograd.Function):
    """ResidualAttentionBlock.forward (model.py:485-528) for a (B*T, d) bf16 or fp16 residual stream (x's type is the
    block's compute type).

    inputs: x, xa (or None), kv_len (or None), then the block's parameters in `ResidualAttentionBlock._param_list`
    order.  Saves every GEMM input it needs for wgrad; recomputes nothing."""

    @staticmethod
    def forward(ctx, blk, B, T, Ta, causal, kv_len, xa_state, x, xa, *params):
        ctx.xa_state = xa_state
        H = blk.attn.n_head
        d = x.shape[1]
        sh = blk._shadows(x.dtype)
        side = _Side(x.device)
        kvc = None
        if xa is not None:   # the cross-attention K/V projection only needs the encoder output: side stream, joined below
            kvc = torch.empty((xa.shape[0], 2 * d), device=x.device, dtype=x.dtype)
            side.run(lambda: linear_fwd(xa, sh["wckv"], sh["bckv"], out=kvc))
        ln1, mean1, rstd1 = K.layernorm_fwd(x, sh["ln1w"], sh["ln1b"])
        qkv = linear_fwd(ln1, sh["wqkv"], sh["bqkv"])
        ao, lse = K.attention_fwd(qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:], B, H, T, T, causal=causal, kv_len=kv_len)
        x1 = linear_fwd(ao, sh["wo"], sh["bo"], epi=K.EPI_BF16_RESIDUAL, aux=x)
        saved = [x, mean1, rstd1, ln1, qkv, ao, lse, x1]
        if xa is not None:
            lnc, meanc, rstdc = K.layernorm_fwd(x1, sh["lncw"], sh["lncb"])
            qc = linear_fwd(lnc, sh["wcq"], sh["bcq"])
            side.join()
            co, lsec = K.attention_fwd(qc, kvc[:, :d], kvc[:, d:], B, H, T, Ta)
            x2 = linear_fwd(co, sh["wco"], sh["bco"], epi=K.EPI_BF16_RESIDUAL, aux=x1)
            saved += [xa, meanc, rstdc, lnc, qc, kvc, co, lsec, x2]
        else:
            x2 = x1
        ln2, mean2, rstd2 = K.layernorm_fwd(x2, sh["ln2w"], sh["ln2b"])
        h, g = linear_fwd(ln2, sh["w1"], sh["b1"], epi=K.EPI_BF16_GELU)
        x3 = linear_fwd(g, sh["w2"], sh["b2"], epi=K.EPI_BF16_RESIDUAL, aux=x2)
        saved += [mean2, rstd2, ln2, h, g]
        if kv_len is not None:
            saved.append(kv_len)
        ctx.save_for_backward(*saved)
        ctx.blk, ctx.dims, ctx.sh = blk, (B, T, Ta, H, d, causal, xa is not None, kv_len is not None), sh
        return x3

    @staticmethod
    def backward(ctx, dx3):
        blk, sh = ctx.blk, ctx.sh
        sv = list(ctx.saved_tensors)
        if not _is_master(blk.attn.query.weight):
            sh = blk._shadows(sv[0].dtype)   # FSDP frees and re-gathers the unsharded parameters between forward and backward
        B, T, Ta, H, d, causal, cross, has_len = ctx.dims
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
        # ---- MLP: x3 = x2 + fc2(gelu(fc1(ln(x2))))
        grads.linear("mlp.2", dx3, g)
        dh = linear_dgrad(dx3, sh["w2"], epi=K.EPI_BF16_GELU_BWD, aux=h)
        grads.linear("mlp.0", dh, ln2)
        dln2 = linear_dgrad(dh, sh["w1"])
        dx2 = K.layernorm_bwd(dln2, x2, sh["ln2w"], mean2, rstd2, grads.vec("mlp_ln.weight", d), grads.vec("mlp_ln.bias", d),
                              dresidual=dx3)
        dxa = None
        if cross:
            # ---- cross attention: x2 = x1 + out(attn(q(ln(x1)), kv(xa)))
            grads.linear("cross_attn.out", dx2, co)
            dco = linear_dgrad(dx2, sh["wco"])
            dqc = torch.empty_like(qc)
            dkvc = torch.empty_like(kvc)
            K.attention_bwd(qc, kvc[:, :d], kvc[:, d:], co, dco, lsec, B, H, T, Ta, dq=dqc, dk=dkvc[:, :d], dv=dkvc[:, d:])
            grads.linear("cross_attn.query", dqc, lnc)
            grads.linear("cross_attn.kv", dkvc, xa)         # [dWk; dWv] in one GEMM
            # d(loss)/d(xa): every decoder layer contributes one (B*1500, d) term.  Instead of 24 separate tensors that
            # autograd adds pairwise (23 elementwise kernels over 98 MB each at medium), the layers accumulate into ONE buffer
            # through the GEMM's residual epilogue (bf16(buf + bf16(acc)), the rounding autograd's bf16 adds would apply);
            # the layer whose backward runs last hands the sum to autograd.
            st = ctx.xa_state
            if st is None:
                dxa = torch.empty_like(xa)
                side.run(lambda: linear_dgrad(dkvc, sh["wckv"], out=dxa))
            else:
                first = st["buf"] is None
                if first:
                    st["buf"] = torch.empty_like(xa)
                buf = st["buf"]
                if first:
                    side.run(lambda: linear_dgrad(dkvc, sh["wckv"], out=buf))
                else:
                    side.run(lambda: linear_dgrad(dkvc, sh["wckv"], epi=K.EPI_BF16_RESIDUAL, aux=buf, out=buf))
                st["left"] -= 1
                dxa = buf if st["left"] == 0 else None
            dlnc = linear_dgrad(dqc, sh["wcq"])
            dx1 = K.layernorm_bwd(dlnc, x1, sh["lncw"], meanc, rstdc, grads.vec("cross_attn_ln.weight", d),
                                  grads.vec("cross_attn_ln.bias", d), dresidual=dx2)
        else:
            dx1 = dx2
        # ---- self attention: x1 = x + out(attn(qkv(ln(x))))
        grads.linear("attn.out", dx1, ao)
        dao = linear_dgrad(dx1, sh["wo"])
        dqkv = torch.empty_like(qkv)
        K.attention_bwd(qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:], ao, dao, lse, B, H, T, T, causal=causal, kv_len=kv_len,
                        dq=dqkv[:, :d], dk=dqkv[:, d:2 * d], dv=dqkv[:, 2 * d:])
        grads.linear("attn.qkv", dqkv, ln1)                 # [dWq; dWk; dWv] in one GEMM
        dln1 = linear_dgrad(dqkv, sh["wqkv"])
        dx = K.layernorm_bwd(dln1, x, sh["ln1w"], mean1, rstd1, grads.vec("attn_ln.weight", d), grads.vec("attn_ln.bias", d),
                             dresidual=dx1)
        side.join()
        grads.done()
        return (None, None, None, None, None, None, None, dx, dxa, *grads.grads_for(blk._param_names))


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
        return self._shadow.get([p for _, p in self.named_parameters()], lambda: self._build_shadows(dtype), dtype)

    def forward(self, x: Tensor, xa: Optional[Tensor] = None, mask: Optional[Tensor] = None,
                kv_cache: Optional[dict] = None, verbose: bool = False, _xa_state: Optional[dict] = None):
        if kv_cache is not None:
            return self._forward_cached(x, xa, mask, kv_cache)
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
        y = _BlockFn.apply(self, B, T, Ta, causal, kv_len, _xa_state, _as16_2d(x, dt), xa2, *params)
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
        grads.keep("conv2.weight", K.unpermute_conv_wgrad(linear_wgrad(dpre2, A2), d, d, out=grads.out("conv2.weight")))
        grads.bias("conv2.bias", dpre2)
        dA2 = linear_dgrad(dpre2, enc.conv2.weight16(pre2.dtype))
        dpre1 = K.col2im_conv2_gelu_bwd(dA2, pre1, B, T, T2, d)
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
    """(token_embedding(ids) + positional_embedding[offset:offset+S]).to(dtype)  (model.py:728-732)."""

    @staticmethod
    def forward(ctx, ids, emb, pos, offset, padding_idx, dec=None, dtype=torch.bfloat16):
        out = K.embed_fwd(ids.contiguous(), _f32(emb), _f32(pos), offset, **_f16_kw(dtype))
        ctx.save_for_backward(ids)
        ctx.meta = (emb.shape, pos.shape, offset, padding_idx)
        ctx.dec = dec
        return out

    @staticmethod
    def backward(ctx, dx):
        (ids,) = ctx.saved_tensors
        eshape, pshape, offset, padding_idx = ctx.meta
        pad = -1 if padding_idx is None else padding_idx
        grads, names = _GradDest(ctx.dec, dx.device), ("token_embedding.weight", "positional_embedding")
        # in direct mode a scatter-add straight into the slab, where the tied logits wgrad has already accumulated
        demb, dpos = grads.vec(names[0], eshape), grads.vec(names[1], pshape)
        K.embed_bwd(ids.contiguous(), dx.contiguous(), demb, dpos[offset:], pad)
        grads.done()     # decoder gradients (incl. the tied embedding) are final
        return (None, *grads.grads_for(names), None, None, None, None)


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
               dtype: Optional[torch.dtype] = None) -> Tensor:
        """Everything up to and including the final LayerNorm: (B, S) ids -> (B*S, d) in `dtype` (default: compute_dtype())."""
        dt = compute_dtype() if dtype is None else dtype
        if self._slabs is not None:
            self._slabs.ensure_synced(dt)
        offset = next(iter(kv_cache.values())).shape[1] if kv_cache else 0
        B, S = x.shape
        d = self.positional_embedding.shape[1]
        h = _EmbedFn.apply(x, self.token_embedding.weight, self.positional_embedding, offset,
                           self.token_embedding.padding_idx, self, dt).view(B, S, d)
        mask = padding_mask if padding_mask is not None else self.mask[:S, :S]
        # shared accumulator of the layers' gradients w.r.t. the encoder output (see _BlockFn.backward); one per forward pass
        xa_state = {"buf": None, "left": len(self.blocks)} if (kv_cache is None and torch.is_grad_enabled() and xa.requires_grad) else None
        for block in self.blocks:
            h = block(h, xa, mask=mask, kv_cache=kv_cache, _xa_state=xa_state) if xa_state is not None else \
                block(h, xa, mask=mask, kv_cache=kv_cache)
        return _LayerNormFn.apply(h.reshape(B * S, d), self.ln.weight, self.ln.bias, self.ln.eps, self, "ln")

    def forward(self, x: Tensor, xa: Tensor, kv_cache: Optional[dict] = None, padding_mask: Optional[Tensor] = None,
                verbose: bool = False):
        B, S = x.shape
        dt = compute_dtype()
        h = self.hidden(x, xa, kv_cache, padding_mask, dt)
        logits = _LogitsFn.apply(h, self.token_embedding.weight, self.embedding16(dt), self)
        return logits.view(B, S, -1)

    def loss(self, x: Tensor, xa: Tensor, targets: Tensor, padding_mask: Optional[Tensor] = None, ignore_index: int = PAD_ID_EN):
        dt = compute_dtype()
        h = self.hidden(x, xa, None, padding_mask, dt)
        return _LossHeadFn.apply(h, self.token_embedding.weight, self.embedding16(dt), targets, ignore_index, self)


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

        def mha_items(a: "MultiHeadAttention"):
            d = a.query.weight.shape[0]
            return [a.out.weight, a.out.bias, a.query.weight, a.key.weight, a.value.weight, a.query.bias, d, a.value.bias]

        def block_items(b: "ResidualAttentionBlock"):
            it = [b.mlp_ln.weight, b.mlp_ln.bias, b.mlp[2].weight, b.mlp[2].bias, b.mlp[0].weight, b.mlp[0].bias]
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
        sl = ParamSlabs(self, layout)
        sl.direct_grads = direct_grads

        def install_mha(a: "MultiHeadAttention"):
            d = a.query.weight.shape[0]
            assert sl.adjacent(a.query.weight, a.key.weight, a.value.weight)
            assert sl.offset[id(a.value.bias)] == sl.offset[id(a.query.bias)] + 2 * d
            a._slab_fused = (sl.span("S", a.query.weight, 3 * d * d).view(3 * d, d), sl.span("P", a.query.bias, 3 * d))
            for lin in (a.query, a.key, a.value, a.out):
                lin._slab_view = sl.shadow(lin.weight)

        def grad_views(mod: nn.Module) -> Dict[str, Tensor]:   # the gradients its own backward writes, by name
            return {n: sl.grad(p) for n, p in mod.named_parameters() if not n.startswith("blocks.")}

        for b in list(enc.blocks) + list(dec.blocks):
            install_mha(b.attn)
            if b.cross_attn is not None:
                install_mha(b.cross_attn)
            for lin in (b.mlp[0], b.mlp[2]):
                lin._slab_view = sl.shadow(lin.weight)
            direct = grad_views(b)
            for name, members in _FUSED.items():     # a fused weight gradient is the slab span of its adjacent members
                if members[0] + ".weight" in direct:
                    w = _attr_by_path(b, members[0]).weight
                    direct[name + ".weight"] = sl.span("G", w, len(members) * w.numel()).view(len(members) * w.shape[0], -1)
            sh = b._build_shadows()      # slab views throughout: 16-bit weights from S, fp32 vectors from P
            b._slabs, b._slab_sh, b._slab_sh16, b._direct = sl, sh, None, direct
        enc._slabs, dec._slabs = sl, sl
        enc._direct, dec._direct = grad_views(enc), grad_views(dec)
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
        return units

    def embed_audio(self, mel: Tensor):
        return self.encoder(mel)

    def logits(self, tokens: Tensor, audio_features: Tensor, padding_mask: Tensor = None):
        return self.decoder(tokens, audio_features, padding_mask=padding_mask)

    def forward(self, mel: Tensor, tokens: Tensor, padding_mask: Tensor = None, verbose: bool = False, *,
                targets: Optional[Tensor] = None, ignore_index: int = PAD_ID_EN) -> Tensor:
        """Reference signature (model.py:856-887) -> fp32 logits.  With the keyword-only `targets` the call returns
        the token cross-entropy instead (fused head); going through forward() keeps DDP / FSDP wrappers in the loop."""
        if targets is not None:
            return self.decoder.loss(tokens, self.encoder(mel), targets, padding_mask, ignore_index)
        return self.decoder(tokens, self.encoder(mel), padding_mask=padding_mask)

    def loss(self, mel: Tensor, tokens: Tensor, targets: Tensor, padding_mask: Tensor = None, ignore_index: int = PAD_ID_EN):
        """Fused equivalent of `F.cross_entropy(model(mel, tokens, padding_mask).view(-1, V), targets.view(-1),
        ignore_index=51864)` (train_timestamps.py:1440-1448) that never materialises fp32 logits."""
        return self.decoder.loss(tokens, self.encoder(mel), targets, padding_mask, ignore_index)

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

    def decode_engine(self, dtype: torch.dtype = torch.float16, max_batch: int = 64):
        """The device-resident greedy decoder for this model (one per activation dtype, built on first use)."""
        from .decode_engine import DecodeEngine

        engines = self.__dict__.setdefault("_engines", {})
        key = (dtype, max_batch)
        if key not in engines:
            engines[key] = DecodeEngine(self, dtype, max_batch)
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
