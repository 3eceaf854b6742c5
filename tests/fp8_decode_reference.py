"""fp64 statements of the fp8 decode step (`DecodingOptions(fp8=True)`; include/oasr_b200.h, "FP8 decoding") (TEST
INFRASTRUCTURE).  Plain torch on whichever device the inputs live; no import of olmoasr_b200.

    quantise     per row: amax = max |x|, inv = 448 / amax, Q = e4m3(x * inv), s = amax / 448 (fp32 arithmetic; a zero
                 row has inv = s = 1) -- oasr_quantize_fp8_rows, i.e. `(x.float() * inv).to(torch.float8_e4m3fn)`
    cross K / V  the (rows, 2d) projection quantised as rows of 64: one scale per (key, head, K|V), laid out (rows, 2H)
                 with the H key heads first
    linear       y = epi( round_T( s_n sum_k x~_k Q_nk + round_T(b_n) ) ): the 16-bit statement of decode_reference
                 with the weight W_nk = s_n Q_nk, exact in fp64 (a 24-bit scale times a 4-bit code)
    attention    score_j = round_T( sK_j hd^-1/4 sum_c q~_c QK_jc ), p_j = round_T(softmax_j), out_c = sum_j p_j sV_j QV_jc

The kernels' fp32 arithmetic meets these statements under decode_reference's rules: the skinny GEMM's sum has one
rounding stage more (the product with s_n), which `linear` adds to the allowance; the attention's scale products are
single fp32 roundings, far inside check_attention's tolerance.
"""
from __future__ import annotations

import torch

from tests import decode_reference as dr

E4M3_MAX = 448.0
F8 = torch.float8_e4m3fn


def quantize_rows(x: torch.Tensor):
    """(codes (R, C) float8_e4m3fn, scales (R,) fp32) of a 2-D x, per row as oasr_quantize_fp8_rows."""
    xf = x.float()
    amax = xf.abs().amax(dim=1)
    zero = amax == 0
    one = torch.ones_like(amax)
    inv = torch.where(zero, one, torch.full_like(amax, E4M3_MAX) / amax)
    scale = torch.where(zero, one, amax / torch.full_like(amax, E4M3_MAX))
    return (xf * inv[:, None]).to(F8), scale


def quantize_kv(kv: torch.Tensor, n_head: int):
    """Cross K / V (rows, 2d) -> (codes (rows, 2d), scales (rows, 2 n_head)): rows of 64 = one (key, head, K|V)."""
    rows, width = kv.shape
    q, s = quantize_rows(kv.reshape(rows * 2 * n_head, width // (2 * n_head)))
    return q.reshape(rows, width), s.reshape(rows, 2 * n_head)


def dequantize(q: torch.Tensor, s: torch.Tensor, group: int = 0) -> torch.Tensor:
    """s Q in fp64 (exact): a scale per row of q, or with `group` one per `group` consecutive elements of a row."""
    qd = q.double() if q.dtype == F8 else q.view(F8).double()
    if not group:
        return qd * s.double()[:, None]
    return (qd.reshape(*qd.shape[:-1], -1, group) * s.double()[..., None]).reshape(qd.shape)


def linear(x, q, s, bias, dtype, *, work=torch.float64, **kw):
    """decode_reference.linear with W = s Q (N, K): the statement in fp64 (`work`), or the fp32 yardstick."""
    W = dequantize(q, s)
    return dr.linear(x, W if work == torch.float64 else W.float(), bias, dtype, work=work,
                     stages=dr.acc_stages(q.shape[1]) + 1, **kw)


def attention(q, kq, ks, vq, vs, dtype):
    """Single-query attention of n rows over e4m3 K / V: q (n, d) in T; kq / vq (n, keys, d) codes; ks / vs (n, keys, H)
    fp32 scales -> the unrounded output (n, d) in fp64 (the fp32 partials of the kernels, added up)."""
    n, keys, d = kq.shape
    H = d // dr.HD
    qs = (q.float() * dr.SCALE).to(dtype).double().view(n, H, dr.HD)
    kc = kq.view(F8).double().reshape(n, keys, H, dr.HD) if kq.dtype != F8 else kq.double().reshape(n, keys, H, dr.HD)
    vc = vq.view(F8).double().reshape(n, keys, H, dr.HD) if vq.dtype != F8 else vq.double().reshape(n, keys, H, dr.HD)
    sk = ks.double().permute(0, 2, 1) * dr.SCALE                                   # (n, H, keys)
    score = dr.rnd(torch.einsum("nhc,njhc->nhj", qs, kc) * sk, dtype)
    p = dr.rnd(torch.softmax(score, dim=-1), dtype) * vs.double().permute(0, 2, 1)
    return torch.einsum("nhj,njhc->nhc", p, vc).reshape(n, d)
