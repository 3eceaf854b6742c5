"""Shared implementation behind olmoasr_b200.model (training model) and olmoasr_b200.inf_model (inference model).

The module tree, parameter names / shapes and initialisation follow the reference exactly
(olmoasr/model.py:14-968, olmoasr/inf_model.py) so that `state_dict()`s are interchangeable and DDP / FSDP /
AdamW / checkpoint code written for the reference keeps working.  Every tensor operation is a call into
liboasr_b200.so; computation is bf16 with fp32 master weights and fp32 statistics, i.e. the numerics of the
reference under `torch.autocast("cuda", torch.bfloat16)` (scripts/training/train_timestamps.py:1414) with
its rounding points reproduced (Linear outputs, GELU, residual adds, LayerNorm casts, bf16 logits).

Training fast path: one autograd.Function per ResidualAttentionBlock (+ stem, embedding and loss head) whose
backward is a hand-sequenced list of kernels -- dgrad / wgrad GEMMs read the saved activations through
MN-major UMMA descriptors, so nothing is transposed in HBM.
"""
from __future__ import annotations

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
    """Tile width for the persistent GEMM: 128 (the widest sm_90a tile, csrc/gemm_sm90.cu) unless N fits a 64-wide tile."""
    return 64 if N <= 64 else 128


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


class _ZeroPool:
    """One zero-fill per backward instead of one per small gradient vector (each fill is a separate ~4 us launch;
    ~700 of them per step otherwise).  Slices are 64-element aligned so every view stays 256-byte aligned."""

    def __init__(self, n_total: int, device):
        self.buf = torch.zeros(n_total, device=device, dtype=torch.float32)
        self.off = 0

    def take(self, n: int) -> Tensor:
        m = (n + 63) // 64 * 64
        if self.off + m > self.buf.numel():  # defensive: never hand out overlapping storage
            return torch.zeros(n, device=self.buf.device, dtype=torch.float32)
        v = self.buf[self.off:self.off + n]
        self.off += m
        return v


def bias_grad(dy: Tensor, n: Optional[int] = None, pool: Optional[_ZeroPool] = None, side=None, out: Optional[Tensor] = None) -> Tensor:
    """Column sums of dy (M, >= n) bf16, accumulated into `out` (a gradient-slab view) or a fresh zeroed vector."""
    n = dy.shape[1] if n is None else n
    db = out if out is not None else (pool.take(n) if pool is not None else torch.zeros(n, device=dy.device, dtype=torch.float32))
    if side is not None:
        return side.run(lambda: K.colsum_(dy, db, n))
    return K.colsum_(dy, db, n)


# ----------------------------------------------------------------------------------------------------
# Weight / bias gradients of a block are leaves of the backward graph: nothing downstream in the same backward reads
# them.  They are enqueued on a second CUDA stream so that their CTAs fill the tail waves (and launch gaps) of the
# dgrad / attention / LayerNorm chain on the main stream -- e.g. the decoder's 14336 x 1024 x 1024 GEMMs are 3.03
# waves of 256 x 256 tiles on 74 SM pairs, i.e. a quarter of their time runs on 2 pairs.  Every block joins the side
# stream before its backward returns, so gradients are complete in main-stream order (DDP hooks, optimizer).
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
    """bf16 copies of fp32 master weights (+ fused biases), rebuilt only when a master changed."""

    def __init__(self):
        self.key = None
        self.val = None

    def get(self, params: Iterable[Tensor], build):
        key = tuple((p.data_ptr(), p._version, p.device) for p in params)
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
        y = K.layernorm_fwd(_as_bf16_2d(x), _f32(self.weight), _f32(self.bias), self.eps, want_stats=False)
        return y.view(shp)


class Linear(nn.Linear):
    """olmoasr/model.py:42-101: kaiming-normal weight, bf16 compute with the fp32 master cast on the fly."""

    def __init__(self, in_features: int, out_features: int, bias: bool = True, device=None, dtype=None):
        super().__init__(in_features, out_features, bias=bias, device=device, dtype=dtype)
        nn.init.kaiming_normal_(self.weight, mode="fan_in", nonlinearity="relu")
        self._shadow = _ShadowCache()

    _slab_view: Optional[Tensor] = None   # set by OLMoASRBase.use_slabs(): a view into the bf16 shadow slab

    def weight_bf16(self) -> Tensor:
        if self._slab_view is not None:
            return self._slab_view
        if self.weight.dtype == torch.bfloat16:      # FSDP bf16 param_dtype: the unsharded view IS the operand (never cached)
            return self.weight.detach()
        return self._shadow.get((self.weight,), lambda: K.cast_bf16(self.weight.detach().contiguous()))

    def forward(self, x: Tensor) -> Tensor:  # inference / hook path (no autograd through the kernels)
        shp = x.shape
        y = linear_fwd(_as_bf16_2d(x), self.weight_bf16(), None if self.bias is None else _f32(self.bias))
        return y.view(*shp[:-1], self.out_features)


class Conv1d(nn.Conv1d):
    """olmoasr/model.py:104-195 (parameters only; the stem kernels are driven by AudioEncoder)."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, bias=True,
                 padding_mode="zeros", device=None, dtype=None):
        super().__init__(in_channels, out_channels, kernel_size, stride=stride, padding=padding, dilation=dilation,
                         groups=groups, bias=bias, padding_mode=padding_mode, device=device, dtype=dtype)
        nn.init.kaiming_normal_(self.weight, mode="fan_in", nonlinearity="relu")
        self._shadow = _ShadowCache()

    def weight_bf16(self) -> Tensor:  # (C_out, 3*C_in) with column = k*C_in + c
        if not _is_master(self.weight):
            return K.cast_conv_weight(_f32(self.weight).contiguous())
        return self._shadow.get((self.weight,), lambda: K.cast_conv_weight(self.weight.detach().contiguous()))


def sinusoids(length, channels, max_timescale=10000):
    """olmoasr/model.py:199-230."""
    assert channels % 2 == 0
    log_timescale_increment = np.log(max_timescale) / (channels // 2 - 1)
    inv_timescales = torch.exp(-log_timescale_increment * torch.arange(channels // 2))
    scaled_time = torch.arange(length)[:, np.newaxis] * inv_timescales[np.newaxis, :]
    return torch.cat([torch.sin(scaled_time), torch.cos(scaled_time)], dim=1)


def _as_bf16_2d(x: Tensor) -> Tensor:
    if x.dtype != torch.bfloat16:
        x = x.to(torch.bfloat16)
    return x.reshape(-1, x.shape[-1]).contiguous()


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

    # ---- fused bf16 shadows -------------------------------------------------------------------------
    _slab_fused = None   # set by OLMoASRBase.use_slabs(): ([Wq;Wk;Wv] view of the shadow slab, [bq;0;bv] view of the masters)

    def fused_qkv(self):
        """([Wq;Wk;Wv] (3d, d) bf16, [bq;0;bv] (3d,) f32) -- key has no bias (model.py:259)."""
        if self._slab_fused is not None:
            return self._slab_fused
        ps = (self.query.weight, self.key.weight, self.value.weight, self.query.bias, self.value.bias)

        def build():
            d = self.query.weight.shape[0]
            w = torch.empty((3 * d, d), device=ps[0].device, dtype=torch.bfloat16)
            b = torch.zeros(3 * d, device=ps[0].device, dtype=torch.float32)
            for i, p in enumerate(ps[:3]):
                if _is_master(p):
                    K.cast_bf16(p.detach().contiguous(), w[i * d:(i + 1) * d])
                else:
                    w[i * d:(i + 1) * d].copy_(p.detach())     # bf16 unsharded FSDP view: a device-to-device copy
            for p, sl in ((ps[3], slice(0, d)), (ps[4], slice(2 * d, 3 * d))):
                if _is_master(p):
                    b[sl].copy_(p.detach())
                else:
                    K.convert(p.detach().contiguous(), b[sl])
            return w, b

        if not _is_master(ps[0]):
            with torch.no_grad():
                return build()                                  # transient FSDP views: nothing to key a cache on
        return self._fused.get(ps, build)

    def fused_kv(self):
        w, b = self.fused_qkv()
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
    """ResidualAttentionBlock.forward (model.py:485-528) for a (B*T, d) bf16 residual stream.

    inputs: x, xa (or None), kv_len (or None), then the block's parameters in `ResidualAttentionBlock._param_list`
    order.  Saves every GEMM input it needs for wgrad; recomputes nothing."""

    @staticmethod
    def forward(ctx, blk, B, T, Ta, causal, kv_len, xa_state, x, xa, *params):
        ctx.xa_state = xa_state
        H = blk.attn.n_head
        d = x.shape[1]
        sh = blk._shadows()
        side = _Side(x.device)
        kvc = None
        if xa is not None:   # the cross-attention K/V projection only needs the encoder output: side stream, joined below
            kvc = torch.empty((xa.shape[0], 2 * d), device=x.device, dtype=torch.bfloat16)
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
        if not _is_master(blk.attn.query.weight):
            sh = blk._shadows()      # FSDP frees and re-gathers the unsharded parameters between forward and backward
        B, T, Ta, H, d, causal, cross, has_len = ctx.dims
        sv = list(ctx.saved_tensors)
        kv_len = sv.pop() if has_len else None
        x, mean1, rstd1, ln1, qkv, ao, lse, x1 = sv[:8]
        if cross:
            xa, meanc, rstdc, lnc, qc, kvc, co, lsec, x2 = sv[8:17]
            mean2, rstd2, ln2, h, g = sv[17:22]
        else:
            x2 = x1
            mean2, rstd2, ln2, h, g = sv[8:13]
        dx3 = dx3.contiguous()
        dev = x.device
        # Where the parameter gradients go.  Slab mode (OLMoASRBase.use_slabs + direct_grads): every kernel ACCUMULATES into
        # its parameter's slice of the flat gradient slab and autograd is handed None.  Otherwise: fresh tensors returned
        # to autograd (DistributedDataParallel / any foreign optimizer keep working).
        D = blk._direct if (blk._direct is not None and blk._slabs.direct_grads) else None
        grads: Dict[str, Tensor] = {}
        pool = None if D is not None else _ZeroPool(32 * d + 4096, dev)   # all bias / LayerNorm gradient vectors (<= 26 d)
        side = _Side(dev)

        def wg(key, dy, xin):
            return linear_wgrad(dy, xin, side=side, out=None if D is None else D[key])

        def bg(key, dy, n=None):
            return bias_grad(dy, n, pool=pool, side=side, out=None if D is None else D[key])

        def vec(key):
            return D[key] if D is not None else pool.take(d)

        # ---- MLP: x3 = x2 + fc2(gelu(fc1(ln(x2))))
        grads["mlp.2.weight"] = wg("mlp.2.weight", dx3, g)
        grads["mlp.2.bias"] = bg("mlp.2.bias", dx3)
        dh = linear_dgrad(dx3, sh["w2"], epi=K.EPI_BF16_GELU_BWD, aux=h)
        grads["mlp.0.weight"] = wg("mlp.0.weight", dh, ln2)
        grads["mlp.0.bias"] = bg("mlp.0.bias", dh)
        dln2 = linear_dgrad(dh, sh["w1"])
        grads["mlp_ln.weight"], grads["mlp_ln.bias"] = vec("mlp_ln.weight"), vec("mlp_ln.bias")
        dx2 = K.layernorm_bwd(dln2, x2, sh["ln2w"], mean2, rstd2, grads["mlp_ln.weight"], grads["mlp_ln.bias"],
                              dresidual=dx3)
        dxa = None
        if cross:
            # ---- cross attention: x2 = x1 + out(attn(q(ln(x1)), kv(xa)))
            grads["cross_attn.out.weight"] = wg("cross_attn.out.weight", dx2, co)
            grads["cross_attn.out.bias"] = bg("cross_attn.out.bias", dx2)
            dco = linear_dgrad(dx2, sh["wco"])
            dqc = torch.empty_like(qc)
            dkvc = torch.empty_like(kvc)
            K.attention_bwd(qc, kvc[:, :d], kvc[:, d:], co, dco, lsec, B, H, T, Ta, dq=dqc, dk=dkvc[:, :d], dv=dkvc[:, d:])
            grads["cross_attn.query.weight"] = wg("cross_attn.query.weight", dqc, lnc)
            grads["cross_attn.query.bias"] = bg("cross_attn.query.bias", dqc)
            dwkv = wg("cross_attn.kv.weight", dkvc, xa)     # [dWk; dWv] in one GEMM
            if D is None:
                grads["cross_attn.key.weight"], grads["cross_attn.value.weight"] = dwkv[:d], dwkv[d:]
                grads["cross_attn.value.bias"] = bias_grad(dkvc, pool=pool, side=side)[d:]
            else:
                bias_grad(dkvc[:, d:], d, side=side, out=D["cross_attn.value.bias"])
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
            grads["cross_attn_ln.weight"], grads["cross_attn_ln.bias"] = vec("cross_attn_ln.weight"), vec("cross_attn_ln.bias")
            dx1 = K.layernorm_bwd(dlnc, x1, sh["lncw"], meanc, rstdc, grads["cross_attn_ln.weight"],
                                  grads["cross_attn_ln.bias"], dresidual=dx2)
        else:
            dx1 = dx2
        # ---- self attention: x1 = x + out(attn(qkv(ln(x))))
        grads["attn.out.weight"] = wg("attn.out.weight", dx1, ao)
        grads["attn.out.bias"] = bg("attn.out.bias", dx1)
        dao = linear_dgrad(dx1, sh["wo"])
        dqkv = torch.empty_like(qkv)
        K.attention_bwd(qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:], ao, dao, lse, B, H, T, T, causal=causal, kv_len=kv_len,
                        dq=dqkv[:, :d], dk=dqkv[:, d:2 * d], dv=dqkv[:, 2 * d:])
        dw = wg("attn.qkv.weight", dqkv, ln1)               # [dWq; dWk; dWv] in one GEMM
        if D is None:
            grads["attn.query.weight"], grads["attn.key.weight"], grads["attn.value.weight"] = dw[:d], dw[d:2 * d], dw[2 * d:]
            db = bias_grad(dqkv, pool=pool, side=side)
            grads["attn.query.bias"], grads["attn.value.bias"] = db[:d], db[2 * d:]
        else:   # the key projection has no bias (model.py:259): its slot in the fused [bq; 0; bv] vector must stay zero
            bias_grad(dqkv[:, :d], d, side=side, out=D["attn.query.bias"])
            bias_grad(dqkv[:, 2 * d:], d, side=side, out=D["attn.value.bias"])
        dln1 = linear_dgrad(dqkv, sh["wqkv"])
        grads["attn_ln.weight"], grads["attn_ln.bias"] = vec("attn_ln.weight"), vec("attn_ln.bias")
        dx = K.layernorm_bwd(dln1, x, sh["ln1w"], mean1, rstd1, grads["attn_ln.weight"], grads["attn_ln.bias"],
                             dresidual=dx1)
        side.join()
        if D is not None:
            if blk._bwd_done_cb is not None:
                blk._bwd_done_cb()      # gradient synchronisation hook: this block's slab range is final
            return (None, None, None, None, None, None, None, dx, dxa, *([None] * len(blk._param_names)))
        return (None, None, None, None, None, None, None, dx, dxa, *[grads[n] for n in blk._param_names])


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
        self._direct: Optional[Dict[str, Tensor]] = None
        self._bwd_done_cb = None

    def _build_shadows(self) -> Dict[str, Tensor]:
        """Every operand the fused block kernels read that derives from a parameter: bf16 weights (fused where the GEMMs are
        fused) and fp32 vectors (biases, LayerNorm affine)."""
        a, c = self.attn, self.cross_attn
        sh: Dict[str, Tensor] = {}
        sh["wqkv"], sh["bqkv"] = a.fused_qkv()
        sh["wo"], sh["bo"] = a.out.weight_bf16(), _f32(a.out.bias)
        sh["ln1w"], sh["ln1b"] = _f32(self.attn_ln.weight), _f32(self.attn_ln.bias)
        if c is not None:
            sh["wcq"], sh["bcq"] = c.query.weight_bf16(), _f32(c.query.bias)
            sh["wckv"], sh["bckv"] = c.fused_kv()
            sh["wco"], sh["bco"] = c.out.weight_bf16(), _f32(c.out.bias)
            sh["lncw"], sh["lncb"] = _f32(self.cross_attn_ln.weight), _f32(self.cross_attn_ln.bias)
        sh["w1"], sh["b1"] = self.mlp[0].weight_bf16(), _f32(self.mlp[0].bias)
        sh["w2"], sh["b2"] = self.mlp[2].weight_bf16(), _f32(self.mlp[2].bias)
        sh["ln2w"], sh["ln2b"] = _f32(self.mlp_ln.weight), _f32(self.mlp_ln.bias)
        return sh

    def _shadows(self) -> Dict[str, Tensor]:
        if self._slab_sh is not None:
            return self._slab_sh
        if not _is_master(self.attn.query.weight):
            with torch.no_grad():
                return self._build_shadows()        # FSDP mixed precision: parameters are transient views, never cached
        return self._shadow.get([p for _, p in self.named_parameters()], self._build_shadows)

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
        xa2 = _as_bf16_2d(xa) if xa is not None else None
        # attribute walk, not get_parameter(): under FSDP the attributes are plain tensor views of the flat parameter
        params = [_attr_by_path(self, n) for n in self._param_names]
        y = _BlockFn.apply(self, B, T, Ta, causal, kv_len, _xa_state, _as_bf16_2d(x), xa2, *params)
        return y.view(B, T, d)

    def _forward_cached(self, x, xa, mask, kv_cache):
        """Decode path: unfused modules so that the forward hooks on key / value fire (model.py:925-964)."""
        B, T, d = x.shape
        x = x + self.attn(self.attn_ln(x), mask=mask, kv_cache=kv_cache)[0]
        if self.cross_attn is not None:
            x = x + self.cross_attn(self.cross_attn_ln(x), xa, kv_cache=kv_cache)[0]
        h, g = linear_fwd(_as_bf16_2d(self.mlp_ln(x)), self.mlp[0].weight_bf16(), _f32(self.mlp[0].bias), epi=K.EPI_BF16_GELU)
        y = linear_fwd(g, self.mlp[2].weight_bf16(), _f32(self.mlp[2].bias), epi=K.EPI_BF16_RESIDUAL, aux=_as_bf16_2d(x))
        return y.view(B, T, d)


# =====================================================================================================
# encoder
# =====================================================================================================
class _StemFn(torch.autograd.Function):
    """conv1 -> GELU -> conv2 (stride 2) -> GELU -> transpose -> + sinusoids (model.py:592-602) as
    im2col + wgmma GEMM with fused bias/GELU epilogues, time-major throughout."""

    @staticmethod
    def forward(ctx, enc, mel, w1, b1, w2, b2):
        B, C, T = mel.shape
        d = w1.shape[0]
        T2 = (T + 2 - 3) // 2 + 1
        mel = mel.contiguous()
        if mel.dtype != torch.float32:        # FSDP MixedPrecision hands the root module a bf16 mel, as it does to the reference
            mel = K.convert(mel, dtype=torch.float32)
        A1 = K.im2col_conv1(mel, 3 * C)
        pre1, h1 = linear_fwd(A1, enc.conv1.weight_bf16(), _f32(b1), epi=K.EPI_BF16_GELU)
        A2 = K.im2col_conv2(h1, B, T, d)
        pre2, h2 = linear_fwd(A2, enc.conv2.weight_bf16(), _f32(b2), epi=K.EPI_BF16_GELU)
        x0 = K.add_pos(h2, _f32(enc.positional_embedding), T2)
        ctx.save_for_backward(A1, pre1, A2, pre2)
        ctx.enc, ctx.dims = enc, (B, C, T, T2, d)
        return x0

    @staticmethod
    def backward(ctx, dx0):
        A1, pre1, A2, pre2 = ctx.saved_tensors
        enc = ctx.enc
        B, C, T, T2, d = ctx.dims
        D = enc._direct if (enc._direct is not None and enc._slabs.direct_grads) else None
        dpre2 = K.gelu_bwd(dx0.contiguous(), pre2)
        dw2 = K.unpermute_conv_wgrad(linear_wgrad(dpre2, A2), d, d, out=None if D is None else D["conv2.weight"])
        db2 = bias_grad(dpre2, out=None if D is None else D["conv2.bias"])
        dA2 = linear_dgrad(dpre2, enc.conv2.weight_bf16())
        dpre1 = K.col2im_conv2_gelu_bwd(dA2, pre1, B, T, T2, d)
        dw1 = K.unpermute_conv_wgrad(linear_wgrad(dpre1, A1), d, C, out=None if D is None else D["conv1.weight"])
        db1 = bias_grad(dpre1, out=None if D is None else D["conv1.bias"])
        if D is not None:
            if enc._bwd_done_cb is not None:
                enc._bwd_done_cb()     # last gradients of the whole backward pass
            return None, None, None, None, None, None
        return None, None, dw1, db1, dw2, db2


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
        if self._slabs is not None:
            self._slabs.ensure_synced()
        B = x.shape[0]
        n_ctx, d = self.positional_embedding.shape
        assert x.dim() == 3 and (x.shape[2] + 2 - 3) // 2 + 1 == n_ctx and x.shape[1] == self.conv1.in_channels, \
            "incorrect audio shape"
        x0 = _StemFn.apply(self, x, self.conv1.weight, self.conv1.bias, self.conv2.weight, self.conv2.bias)
        h = x0.view(B, n_ctx, d)
        for block in self.blocks:
            h = block(h)
        return _LayerNormFn.apply(h.reshape(B * n_ctx, d), self.ln_post.weight, self.ln_post.bias, self.ln_post.eps,
                                  self, "ln_post").view(B, n_ctx, d)


class _LayerNormFn(torch.autograd.Function):
    """Final LayerNorm of the encoder / decoder.  `owner._direct[key + ".weight" / ".bias"]` are the gradient-slab targets
    in slab mode."""

    @staticmethod
    def forward(ctx, x, w, b, eps, owner=None, key=None):
        y, mean, rstd = K.layernorm_fwd(x, _f32(w), _f32(b), eps)
        ctx.save_for_backward(x, w, mean, rstd)
        ctx.owner, ctx.key = owner, key
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, mean, rstd = ctx.saved_tensors
        w = _f32(w)
        owner = ctx.owner
        D = owner._direct if (owner is not None and owner._direct is not None and owner._slabs.direct_grads) else None
        if D is not None:
            dx = K.layernorm_bwd(dy.contiguous(), x, w, mean, rstd, D[ctx.key + ".weight"], D[ctx.key + ".bias"])
            return dx, None, None, None, None, None
        dw = torch.zeros(w.shape, device=w.device, dtype=torch.float32)
        db = torch.zeros(w.shape, device=w.device, dtype=torch.float32)
        dx = K.layernorm_bwd(dy.contiguous(), x, w, mean, rstd, dw, db)
        return dx, dw, db, None, None, None


# =====================================================================================================
# decoder
# =====================================================================================================
class _EmbedFn(torch.autograd.Function):
    """(token_embedding(ids) + positional_embedding[offset:offset+S]).to(bf16)  (model.py:728-732)."""

    @staticmethod
    def forward(ctx, ids, emb, pos, offset, padding_idx, dec=None):
        out = K.embed_fwd(ids.contiguous(), _f32(emb), _f32(pos), offset)
        ctx.save_for_backward(ids)
        ctx.meta = (emb.shape, pos.shape, offset, padding_idx)
        ctx.dec = dec
        return out

    @staticmethod
    def backward(ctx, dx):
        (ids,) = ctx.saved_tensors
        eshape, pshape, offset, padding_idx = ctx.meta
        dec = ctx.dec
        pad = -1 if padding_idx is None else padding_idx
        D = dec._direct if (dec is not None and dec._direct is not None and dec._slabs.direct_grads) else None
        if D is not None:   # scatter-add straight into the slab (the tied logits wgrad already accumulated there)
            K.embed_bwd(ids.contiguous(), dx.contiguous(), D["token_embedding.weight"], D["positional_embedding"][offset:], pad)
            if dec._bwd_done_cb is not None:
                dec._bwd_done_cb()     # decoder gradients (incl. the tied embedding) are final
            return None, None, None, None, None, None
        demb = torch.zeros(eshape, device=dx.device, dtype=torch.float32)
        dpos = torch.zeros(pshape, device=dx.device, dtype=torch.float32)
        K.embed_bwd(ids.contiguous(), dx.contiguous(), demb, dpos[offset:], pad)
        return None, demb, dpos, None, None, None


def _direct_of(mod):
    """Gradient-slab targets of a module when the model runs in slab mode with direct gradients, else None."""
    if mod is not None and mod._direct is not None and mod._slabs.direct_grads:
        return mod._direct
    return None


def _logits_ld(V: int) -> int:
    return (V + 255) // 256 * 256  # 51865 -> 51968: no ragged tile in the logits GEMM, 16-byte aligned rows


class _LogitsFn(torch.autograd.Function):
    """(x @ token_embedding.weight.to(x.dtype).T).float()  (model.py:768-770) for callers that want logits."""

    @staticmethod
    def forward(ctx, x, emb, emb_bf16, dec=None):
        M, d = x.shape
        V = emb.shape[0]
        buf = torch.empty((M, _logits_ld(V)), device=x.device, dtype=torch.bfloat16)
        K.gemm(x, emb_bf16, M, V, d, out=buf, block_n=256)
        ctx.save_for_backward(x, emb_bf16)
        ctx.dec = dec
        return K.logits_to_f32(buf, V)

    @staticmethod
    def backward(ctx, dlogits):
        x, emb_bf16 = ctx.saved_tensors
        M, d = x.shape
        V = emb_bf16.shape[0]
        buf = torch.empty((M, _logits_ld(V)), device=x.device, dtype=torch.bfloat16)
        buf[:, :V].copy_(dlogits)  # `.float()` backward: the gradient enters the matmul as bf16
        dx = K.gemm(buf[:, :V], emb_bf16, M, d, V, b_mn=True, block_n=_pick_block_n(M, d))
        D = _direct_of(ctx.dec)
        demb = linear_wgrad(buf, x, n_valid=V, out=None if D is None else D["token_embedding.weight"])
        return dx, (None if D is not None else demb), None, None


class _LossHeadFn(torch.autograd.Function):
    """Fused tail of the training step: tied logits GEMM (bf16, never widened to fp32) + token cross-entropy
    (model.py:768-770 followed by train_timestamps.py:1444-1448).  The backward turns the logits buffer into
    d(logits) in place and feeds it to the dgrad / wgrad GEMMs."""

    @staticmethod
    def forward(ctx, x, emb, emb_bf16, targets, ignore_index, dec=None):
        ctx.dec = dec
        M, d = x.shape
        V = emb.shape[0]
        buf = torch.empty((M, _logits_ld(V)), device=x.device, dtype=torch.bfloat16)
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
        D = _direct_of(ctx.dec)
        demb = linear_wgrad(buf, x, n_valid=V, out=None if D is None else D["token_embedding.weight"])
        return dx, (None if D is not None else demb), None, None, None, None


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
        if self._emb_slab_view is not None:
            return self._emb_slab_view
        w = self.token_embedding.weight
        if w.dtype == torch.bfloat16:
            return w.detach()
        return self._emb_shadow.get((w,), lambda: K.cast_bf16(w.detach().contiguous()))

    def hidden(self, x: Tensor, xa: Tensor, kv_cache: Optional[dict] = None, padding_mask: Optional[Tensor] = None) -> Tensor:
        """Everything up to and including the final LayerNorm: (B, S) ids -> (B*S, d) bf16."""
        if self._slabs is not None:
            self._slabs.ensure_synced()
        offset = next(iter(kv_cache.values())).shape[1] if kv_cache else 0
        B, S = x.shape
        d = self.positional_embedding.shape[1]
        h = _EmbedFn.apply(x, self.token_embedding.weight, self.positional_embedding, offset,
                           self.token_embedding.padding_idx, self).view(B, S, d)
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
        h = self.hidden(x, xa, kv_cache, padding_mask)
        logits = _LogitsFn.apply(h, self.token_embedding.weight, self.embedding_bf16(), self)
        return logits.view(B, S, -1)

    def loss(self, x: Tensor, xa: Tensor, targets: Tensor, padding_mask: Optional[Tensor] = None, ignore_index: int = PAD_ID_EN):
        h = self.hidden(x, xa, None, padding_mask)
        return _LossHeadFn.apply(h, self.token_embedding.weight, self.embedding_bf16(), targets, ignore_index, self)


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

        def install_mha(a: "MultiHeadAttention", direct: Dict[str, Tensor], prefix: str, cross: bool):
            d = a.query.weight.shape[0]
            assert sl.adjacent(a.query.weight, a.key.weight, a.value.weight)
            assert sl.offset[id(a.value.bias)] == sl.offset[id(a.query.bias)] + 2 * d
            a._slab_fused = (sl.span("S", a.query.weight, 3 * d * d).view(3 * d, d), sl.span("P", a.query.bias, 3 * d))
            for lin in (a.query, a.key, a.value, a.out):
                lin._slab_view = sl.shadow(lin.weight)
            direct[prefix + ".out.weight"], direct[prefix + ".out.bias"] = sl.grad(a.out.weight), sl.grad(a.out.bias)
            direct[prefix + ".query.bias"], direct[prefix + ".value.bias"] = sl.grad(a.query.bias), sl.grad(a.value.bias)
            if cross:
                direct[prefix + ".query.weight"] = sl.grad(a.query.weight)
                direct[prefix + ".kv.weight"] = sl.span("G", a.key.weight, 2 * d * d).view(2 * d, d)
            else:
                direct[prefix + ".qkv.weight"] = sl.span("G", a.query.weight, 3 * d * d).view(3 * d, d)

        for b in list(enc.blocks) + list(dec.blocks):
            direct: Dict[str, Tensor] = {}
            install_mha(b.attn, direct, "attn", cross=False)
            if b.cross_attn is not None:
                install_mha(b.cross_attn, direct, "cross_attn", cross=True)
            for name, lin in (("mlp.0", b.mlp[0]), ("mlp.2", b.mlp[2])):
                lin._slab_view = sl.shadow(lin.weight)
                direct[name + ".weight"], direct[name + ".bias"] = sl.grad(lin.weight), sl.grad(lin.bias)
            for name, ln in (("attn_ln", b.attn_ln), ("cross_attn_ln", b.cross_attn_ln), ("mlp_ln", b.mlp_ln)):
                if ln is not None:
                    direct[name + ".weight"], direct[name + ".bias"] = sl.grad(ln.weight), sl.grad(ln.bias)
            sh = b._build_shadows()      # slab views throughout: bf16 weights from S, fp32 vectors from P
            b._slabs, b._slab_sh, b._direct = sl, sh, direct
        enc._slabs, dec._slabs = sl, sl
        enc._direct = {"conv1.weight": sl.grad(enc.conv1.weight), "conv1.bias": sl.grad(enc.conv1.bias),
                       "conv2.weight": sl.grad(enc.conv2.weight), "conv2.bias": sl.grad(enc.conv2.bias),
                       "ln_post.weight": sl.grad(enc.ln_post.weight), "ln_post.bias": sl.grad(enc.ln_post.bias)}
        dec._direct = {"token_embedding.weight": sl.grad(dec.token_embedding.weight),
                       "positional_embedding": sl.grad(dec.positional_embedding),
                       "ln.weight": sl.grad(dec.ln.weight), "ln.bias": sl.grad(dec.ln.bias)}
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
