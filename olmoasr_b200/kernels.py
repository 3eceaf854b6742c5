"""Thin tensor-level wrappers over the C ABI (one Python function per entry point).

Shapes / dtypes are validated here so that a bad call fails with a Python exception before any
kernel is launched; the kernels themselves never allocate.

Activations are bf16 or fp16 (the model under torch.autocast(dtype=torch.float16)); each wrapper takes the type from
its 16-bit tensor arguments, or from `dtype` where every input is fp32.  bf16 calls go to the bf16 entry points, fp16
calls to their `16` twins (include/oasr_b200.h).
"""
from __future__ import annotations

import torch

from . import _lib
from ._lib import call, ptr, stream

K_MAJOR, MN_MAJOR = 0, 1
EPI_BF16, EPI_BF16_GELU, EPI_BF16_RESIDUAL, EPI_BF16_GELU_BWD, EPI_F32, EPI_F32_ATOMIC_ADD = range(6)


# When set to a list, every GEMM launch is bracketed by CUDA events on the launching stream and
# (flops, start, end, shape-key) is appended: bench.py derives the tensor-pipe roofline figure of the dominant kernel from it.
GEMM_PROFILE = None


def set_gemm_sm_budget(n_sms: int) -> int:
    """SMs the persistent GEMM may occupy (0 = all); returns the previous setting.  Under DDP the NCCL all-reduce
    CTAs need SMs of their own: a persistent grid that no longer fits runs its displaced CTAs as a second wave."""
    return _lib.lib().oasr_gemm_set_sm_budget(int(n_sms))


def _req(cond, msg):
    if not cond:
        raise ValueError(msg)


ACT16 = (torch.bfloat16, torch.float16)
_TWIN16 = {"oasr_gemm_bf16": "oasr_gemm16", "oasr_colsum_bf16": "oasr_colsum16", "oasr_logits_to_f32": "oasr_logits_to_f32_16",
           "oasr_im2col_conv1": "oasr_im2col_conv1_16"}


def _call16(name, dtype, *args):
    """Entry point `name` for bf16; for fp16 its twin, which takes the dtype code before the stream."""
    if dtype == torch.bfloat16:
        return call(name, *args)
    _req(dtype == torch.float16, f"{name}: 16-bit activations must be bf16 or fp16, got {dtype}")
    call(_TWIN16.get(name, name + "16"), *args[:-1], _lib.DTYPE_F16, args[-1])


def gemm(a, b, M, N, K, *, a_mn=False, b_mn=False, out=None, out2=None, bias=None, aux=None,
         epi=EPI_BF16, split_k=1, block_n=0):
    """D[M,N] = epi(sum_k A[m,k] B[n,k]) on wgmma.  `a` is (M,K) (or (K,M) when a_mn), `b` is (N,K)
    (or (K,N) when b_mn); both bf16 or both fp16, with unit inner stride.  See include/oasr_b200.h."""
    dt = a.dtype
    _req(dt in ACT16 and b.dtype == dt, "gemm: operands must be both bf16 or both fp16")
    _req(a.is_cuda and b.is_cuda, "gemm: operands must be CUDA tensors")
    _req(a.dim() == 2 and b.dim() == 2 and a.stride(1) == 1 and b.stride(1) == 1, "gemm: 2-D, unit inner stride")
    _req(tuple(a.shape) == ((K, M) if a_mn else (M, K)), f"gemm: A shape {tuple(a.shape)} vs M={M} K={K} a_mn={a_mn}")
    _req(tuple(b.shape) == ((K, N) if b_mn else (N, K)), f"gemm: B shape {tuple(b.shape)} vs N={N} K={K} b_mn={b_mn}")
    f32_out = epi in (EPI_F32, EPI_F32_ATOMIC_ADD)
    if out is None:
        _req(epi != EPI_F32_ATOMIC_ADD, "gemm: atomic-add epilogue needs a pre-initialised `out`")
        out = torch.empty((M, N), device=a.device, dtype=torch.float32 if f32_out else dt)
    _req(out.dtype == (torch.float32 if f32_out else dt), "gemm: out dtype")
    _req(out.dim() == 2 and out.shape[0] == M and out.shape[1] >= N and out.stride(1) == 1, "gemm: out shape")
    if epi == EPI_BF16_GELU and out2 is None:
        out2 = torch.empty_like(out)
    if aux is not None:
        _req(aux.dtype == dt and aux.stride(1) == 1 and aux.shape[0] == M, "gemm: aux")
    if bias is not None:
        _req(bias.dtype == torch.float32 and bias.numel() >= N and bias.is_contiguous(), "gemm: bias must be f32")
    prof = GEMM_PROFILE
    if prof is not None:
        e0 = torch.cuda.Event(enable_timing=True)
        e1 = torch.cuda.Event(enable_timing=True)
        e0.record()
    _call16("oasr_gemm_bf16", dt, ptr(a), a.stride(0), int(a_mn), ptr(b), b.stride(0), int(b_mn),
         ptr(out), out.stride(0), ptr(out2), ptr(bias), ptr(aux), aux.stride(0) if aux is not None else 0,
         M, N, K, epi, split_k, block_n, stream())
    if prof is not None:
        e1.record()
        prof.append((2.0 * M * N * K, e0, e1, (M, N, K, int(a_mn), int(b_mn), epi, split_k, block_n)))
    if epi == EPI_BF16_GELU:
        return out, out2
    return out


# ----------------------------------------------------------------------------------------------------
def _bf16_2d(t, name, dtype=torch.bfloat16):
    _req(t.is_cuda and t.dtype == dtype and t.dim() == 2 and t.stride(1) == 1,
         f"{name}: 2-D {str(dtype).removeprefix('torch.')} CUDA tensor, unit inner stride")


def layernorm_fwd(x, weight, bias, eps=1e-5, want_stats=True):
    """x (rows, d) bf16 / fp16 contiguous -> y of x's type [, mean, rstd f32].  model.py:25-39."""
    _req(x.dtype in ACT16, "layernorm: x must be bf16 or fp16")
    _bf16_2d(x, "layernorm x", x.dtype)
    _req(x.is_contiguous() and weight.dtype == torch.float32 and bias.dtype == torch.float32, "layernorm: contiguous x, f32 params")
    rows, d = x.shape
    y = torch.empty_like(x)
    mean = rstd = None
    if want_stats:
        mean = torch.empty(rows, device=x.device, dtype=torch.float32)
        rstd = torch.empty(rows, device=x.device, dtype=torch.float32)
    _call16("oasr_layernorm_fwd", x.dtype, ptr(x), ptr(weight), ptr(bias), ptr(y), ptr(mean), ptr(rstd), rows, d, eps, stream())
    return (y, mean, rstd) if want_stats else y


def layernorm_bwd(dy, x, weight, mean, rstd, dweight, dbias, dresidual=None):
    """Returns dx = T(dresidual + T(dx_ln)) (T = x's 16-bit type); accumulates into dweight / dbias (f32)."""
    _req(x.dtype in ACT16, "layernorm_bwd: x must be bf16 or fp16")
    _bf16_2d(dy, "layernorm dy", x.dtype); _bf16_2d(x, "layernorm x", x.dtype)
    _req(dy.is_contiguous() and x.is_contiguous() and (dresidual is None or dresidual.is_contiguous()), "layernorm_bwd: contiguous")
    rows, d = x.shape
    dx = torch.empty_like(x)
    _call16("oasr_layernorm_bwd", x.dtype, ptr(dy), ptr(x), ptr(weight), ptr(mean), ptr(rstd), ptr(dresidual), ptr(dx), ptr(dweight),
         ptr(dbias), rows, d, stream())
    return dx


def attention_fwd(q, k, v, B, H, Tq, Tkv, causal=False, kv_len=None, scale=None, want_lse=True, out=None):
    """q (B*Tq, >=H*64) bf16 / fp16 view, k/v (B*Tkv, ...) views (column slices of fused projections are fine)."""
    _req(q.dtype in ACT16, "attention: q must be bf16 or fp16")
    for t, n in ((q, "q"), (k, "k"), (v, "v")):
        _bf16_2d(t, n, q.dtype)
    _req(q.shape[0] == B * Tq and k.shape[0] == B * Tkv and v.shape[0] == B * Tkv, "attention: row counts")
    _req(q.shape[1] == H * 64 and k.shape[1] == H * 64 and v.shape[1] == H * 64, "attention: width must be H*64")
    if scale is None:
        scale = 64 ** -0.5
    if out is None:
        out = torch.empty((B * Tq, H * 64), device=q.device, dtype=q.dtype)
    lse = torch.empty((B, H, Tq), device=q.device, dtype=torch.float32) if want_lse else None
    if kv_len is not None:
        _req(kv_len.dtype == torch.int32 and kv_len.numel() == B, "attention: kv_len must be int32 (B,)")
    _call16("oasr_attention_fwd", q.dtype, ptr(q), q.stride(0), ptr(k), k.stride(0), ptr(v), v.stride(0), ptr(out), out.stride(0),
         ptr(lse), B, H, Tq, Tkv, 64, int(causal), ptr(kv_len), float(scale), stream())
    return out, lse


def attention_bwd(q, k, v, o, dout, lse, B, H, Tq, Tkv, causal=False, kv_len=None, scale=None, dq=None, dk=None, dv=None):
    dt = q.dtype
    _req(dt in ACT16, "attention_bwd: q must be bf16 or fp16")
    for t, n in ((q, "q"), (k, "k"), (v, "v"), (o, "o"), (dout, "dout")):
        _bf16_2d(t, n, dt)
    if scale is None:
        scale = 64 ** -0.5
    dev = q.device
    if dq is None:
        dq = torch.empty((B * Tq, H * 64), device=dev, dtype=dt)
    if dk is None:
        dk = torch.empty((B * Tkv, H * 64), device=dev, dtype=dt)
    if dv is None:
        dv = torch.empty((B * Tkv, H * 64), device=dev, dtype=dt)
    delta = torch.empty((B, H, Tq), device=dev, dtype=torch.float32)
    _call16("oasr_attention_bwd", dt, ptr(q), q.stride(0), ptr(k), k.stride(0), ptr(v), v.stride(0), ptr(o), o.stride(0),
         ptr(dout), dout.stride(0), ptr(lse), ptr(delta), ptr(dq), dq.stride(0), ptr(dk), dk.stride(0),
         ptr(dv), dv.stride(0), B, H, Tq, Tkv, 64, int(causal), ptr(kv_len), float(scale), stream())
    return dq, dk, dv


def ce_fwd(logits, targets, V, ignore_index):
    """logits (rows, ld) bf16 / fp16; returns (lse (rows,), lsc (4,)): lsc = [loss sum, target count, bad-target count, -];
    `ce_finalize(lsc)` turns it into the mean loss."""
    _req(logits.dtype in ACT16, "ce: logits must be bf16 or fp16")
    _bf16_2d(logits, "ce logits", logits.dtype)
    rows = logits.shape[0]
    _req(targets.dtype == torch.int64 and targets.numel() == rows and targets.is_contiguous(), "ce: targets int64 (rows,)")
    lse = torch.empty(rows, device=logits.device, dtype=torch.float32)
    lsc = torch.zeros(4, device=logits.device, dtype=torch.float32)
    _call16("oasr_ce_fwd", logits.dtype, ptr(logits), ptr(targets), ptr(lse), ptr(lsc), rows, V, logits.stride(0), ignore_index, stream())
    return lse, lsc


def ce_finalize(lsc):
    """0-d mean loss = lsc[0] / lsc[1] (no torch arithmetic on the way to the loss)."""
    loss = torch.empty((), device=lsc.device, dtype=torch.float32)
    call("oasr_ce_finalize", ptr(lsc), ptr(loss), stream())
    return loss


def ce_bwd_(logits, targets, lse, lsc, grad_out, V, ignore_index):
    """In place: logits <- d(loss)/d(logits) in the logits' 16-bit type."""
    _req(grad_out.dtype == torch.float32 and grad_out.numel() == 1, "ce_bwd: grad_out must be one f32")
    _call16("oasr_ce_bwd", logits.dtype, ptr(logits), ptr(targets), ptr(lse), ptr(lsc), ptr(grad_out), logits.shape[0], V, logits.stride(0),
         ignore_index, stream())
    return logits


def logits_to_f32(logits, V):
    out = torch.empty((logits.shape[0], V), device=logits.device, dtype=torch.float32)
    _call16("oasr_logits_to_f32", logits.dtype, ptr(logits), ptr(out), logits.shape[0], V, logits.stride(0), stream())
    return out


def embed_fwd(ids, emb, pos, pos_offset=0, dtype=torch.bfloat16):
    _req(ids.dtype == torch.int64 and ids.dim() == 2 and ids.is_contiguous(), "embed: ids int64 (B,S)")
    B, S = ids.shape
    d = emb.shape[1]
    out = torch.empty((B * S, d), device=emb.device, dtype=dtype)
    _call16("oasr_embed_fwd", dtype, ptr(ids), ptr(emb), ptr(pos), ptr(out), B, S, d, pos_offset, emb.shape[0], stream())
    return out


def embed_bwd(ids, dx, demb, dpos, padding_idx):
    B, S = ids.shape
    _call16("oasr_embed_bwd", dx.dtype, ptr(ids), ptr(dx), ptr(demb), ptr(dpos), B, S, dx.shape[1], padding_idx, demb.shape[0], stream())


def cast_bf16(src, dst=None):
    _req(src.dtype == torch.float32 and src.is_contiguous(), "cast: f32 contiguous")
    if dst is None:
        dst = torch.empty(src.shape, device=src.device, dtype=torch.bfloat16)
    call("oasr_cast_f32_to_bf16", ptr(src), ptr(dst), src.numel(), stream())
    return dst


def cast_conv_weight(w, dst=None, dtype=torch.bfloat16):
    c_out, c_in, k = w.shape
    _req(k == 3 and w.is_contiguous() and w.dtype == torch.float32, "conv weight (C_out, C_in, 3) f32")
    if dst is None:
        dst = torch.empty((c_out, 3 * c_in), device=w.device, dtype=dtype)
    _call16("oasr_cast_conv_weight", dst.dtype, ptr(w), ptr(dst), c_out, c_in, stream())
    return dst


def unpermute_conv_wgrad(g, c_out, c_in, out=None):
    """(C_out, 3, C_in) f32 -> (C_out, C_in, 3) f32; with `out` (a gradient-slab view) the result is ADDED into it."""
    accumulate = out is not None
    if out is None:
        out = torch.empty((c_out, c_in, 3), device=g.device, dtype=torch.float32)
    call("oasr_unpermute_conv_wgrad", ptr(g), ptr(out), c_out, c_in, int(accumulate), stream())
    return out


def mask_to_kvlen(mask, err_flag):
    """(B, S, S) f32 additive padding mask -> (B,) int32 key counts; err_flag (1,) int32 is OR-ed with 1 on a malformed mask."""
    _req(mask.is_cuda and mask.dtype == torch.float32 and mask.dim() == 3 and mask.is_contiguous(), "mask: (B,S,S) f32 CUDA")
    kv = torch.empty(mask.shape[0], device=mask.device, dtype=torch.int32)
    call("oasr_mask_to_kvlen", ptr(mask), ptr(kv), ptr(err_flag), mask.shape[0], mask.shape[1], stream())
    return kv


def im2col_conv1(mel, kpad, dtype=torch.bfloat16):
    B, C, T = mel.shape
    _req(mel.dtype == torch.float32 and mel.is_contiguous(), "mel f32 contiguous")
    A = torch.empty((B * T, kpad), device=mel.device, dtype=dtype)
    _call16("oasr_im2col_conv1", dtype, ptr(mel), ptr(A), B, C, T, kpad, stream())
    return A


def im2col_conv2(h, B, T_in, d):
    T_out = (T_in + 2 - 3) // 2 + 1
    A = torch.empty((B * T_out, 3 * d), device=h.device, dtype=h.dtype)   # a copy: one kernel serves both 16-bit types
    call("oasr_im2col_conv2", ptr(h), ptr(A), B, T_in, T_out, d, stream())
    return A


def col2im_conv2_gelu_bwd(dA, pre1, B, T_in, T_out, d):
    out = torch.empty((B * T_in, d), device=dA.device, dtype=dA.dtype)
    _call16("oasr_col2im_conv2_gelu_bwd", dA.dtype, ptr(dA), ptr(pre1), ptr(out), B, T_in, T_out, d, stream())
    return out


def add_pos(x, pos, T):
    out = torch.empty_like(x)
    _call16("oasr_add_pos", x.dtype, ptr(x), ptr(pos), ptr(out), x.shape[0], T, x.shape[1], stream())
    return out


def gelu_bwd(dy, pre):
    out = torch.empty_like(dy)
    _call16("oasr_gelu_bwd", dy.dtype, ptr(dy), ptr(pre), ptr(out), dy.numel(), stream())
    return out


def colsum_(dy, db, N=None):
    """db (f32) += column sums of dy (M, N) bf16 / fp16."""
    M = dy.shape[0]
    N = dy.shape[1] if N is None else N
    _call16("oasr_colsum_bf16", dy.dtype, ptr(dy), ptr(db), M, N, dy.stride(0), stream())
    return db


_DTYPE_CODE = {torch.bfloat16: _lib.DTYPE_BF16, torch.float16: _lib.DTYPE_F16, torch.float32: _lib.DTYPE_F32}


def convert(src, dst=None, dtype=None):
    """Elementwise dtype conversion between contiguous tensors (f32 / bf16 / f16), round-to-nearest-even."""
    _req(src.is_cuda and src.is_contiguous(), "convert: contiguous CUDA tensor")
    if dst is None:
        dst = torch.empty(src.shape, device=src.device, dtype=dtype)
    _req(dst.is_contiguous() and dst.numel() == src.numel(), "convert: dst must be contiguous with the same number of elements")
    call("oasr_convert", ptr(src), _DTYPE_CODE[src.dtype], ptr(dst), _DTYPE_CODE[dst.dtype], src.numel(), stream())
    return dst


def align_cost(heads, n_frames, medfilt_width=7, out=None):
    """DTW input of one window (include/oasr_b200.h oasr_align_cost): `heads` lists (q, k) per alignment head in
    ascending (layer, head) order, q (n_tok, 64) and k (>= n_frames, 64) column slices (unit inner stride) of the
    cross-attention query rows and cross keys, all bf16 or all fp16.  Returns cost (n_tok - 2, n_frames) fp32."""
    _req(len(heads) >= 1, "align_cost: need at least one head")
    q0, k0 = heads[0]
    dt, dev, n_tok = q0.dtype, q0.device, q0.shape[0]
    for q, k in heads:
        _req(q.is_cuda and k.is_cuda and q.dtype == dt and k.dtype == dt and dt in ACT16,
             "align_cost: q and k must be CUDA tensors of one 16-bit type")
        _req(q.dim() == 2 and k.dim() == 2 and q.shape == (n_tok, 64) and k.shape[1] == 64 and k.shape[0] >= n_frames,
             "align_cost: q (n_tok, 64) and k (>= n_frames, 64) per head")
        _req(q.stride(1) == 1 and k.stride(1) == 1, "align_cost: unit inner stride")
    table = torch.tensor([[q.data_ptr(), k.data_ptr(), q.stride(0), k.stride(0)] for q, k in heads],
                         dtype=torch.int64).to(dev, non_blocking=True)
    stats = torch.empty((len(heads), n_tok, 2), device=dev, dtype=torch.float32)
    if out is None:
        out = torch.empty((max(n_tok - 2, 0), n_frames), device=dev, dtype=torch.float32)
    _req(out.dtype == torch.float32 and out.stride(1) == 1 and out.shape == (n_tok - 2, n_frames),
         "align_cost: out (n_tok - 2, n_frames) fp32")
    call("oasr_align_cost", ptr(table), len(heads), 64, n_tok, n_frames, medfilt_width, ptr(stats), ptr(out), out.stride(0),
         _DTYPE_CODE[dt], stream())
    return out


def dtw(x):
    """Dynamic time warping of x (rows, cols) fp32 with whisper's tie order (oasr_dtw).  Returns (path, length) on the
    device: path (2, rows + cols) int32 whose first `length` columns are (text index, time index) in path order."""
    _req(x.is_cuda and x.dtype == torch.float32 and x.dim() == 2 and x.stride(1) == 1, "dtw: 2-D fp32 CUDA matrix, unit inner stride")
    rows, cols = x.shape
    _req(rows >= 1 and cols >= 1, "dtw: empty matrix")
    trace = torch.empty((rows + 1) * (cols + 1), device=x.device, dtype=torch.uint8)
    path = torch.empty((2, rows + cols), device=x.device, dtype=torch.int32)
    length = torch.empty(1, device=x.device, dtype=torch.int32)
    call("oasr_dtw", ptr(x), x.stride(0), rows, cols, ptr(trace), ptr(path[0]), ptr(path[1]), ptr(length), stream())
    return path, length
