"""fp64 reference of the training step's memory-bound kernels and the fused AdamW, and the bounds their tests use
(TEST INFRASTRUCTURE).

Plain torch, on whichever device the inputs live; no import of olmoasr_b200.  Each function states one kernel launch
at the rounding points its source writes down, in the activation type T (bf16 or fp16).  The rule machinery (check16 /
check32, errors16 / errors32, ALPHA, F32_ALPHA) is tests/training_reference.py's.

Exact copies (no arithmetic; compared bit for bit):
    im2col_conv1          csrc/elementwise.cu: A[b,t][k C + c] = T(mel[b,c,t+k-1]), zero outside [0, T), Kpad columns zero
    im2col_conv2          A[b,t] = [h[b,2t-1], h[b,2t], h[b,2t+1]], rows outside [0, T_in) zero
    cast_conv_weight      (C_out, C_in, 3) fp32 -> (C_out, 3, C_in) in T
    unpermute_conv_wgrad  (C_out, 3, C_in) -> (C_out, C_in, 3) fp32, fresh or out + g (one fp32 add)

Rounded once to T (check16):
    col2im_conv2_gelu_bwd dpre1[b,r] = T(T(sum_{2t+k-1=r} dA[b,t,k]) gelu'(pre1[b,r])): at most two taps, k = 0 before k = 2
    gelu_bwd              T(dy gelu'(pre))
    add_pos               T(x + pos[row mod T])
    embed_fwd             T(emb[id] + pos[s + offset]); an id outside [0, V) reads row 0
  gelu' is the Abramowitz-Stegun erf of common.cuh (erf_fast, __expf); its distance from the erf gelu' is below
  training_reference.GELU_APPROX and the fp32 evaluation of cdf + x pdf adds a few 2^-24 (absolute): GELU_GRAD_TOL.
  The inner T(sum) may flip where the fp32 two-tap sum lies within 2^-24 of a rounding boundary: one inner ulp times
  |gelu'| there.  add_pos and embed_fwd add in fp32 and round to T, which can double-round: rule 1's one ulp covers
  it, and the kernel equals the fp32 restatement (work=torch.float32) bit for bit.

fp32 sums (check32, every element within its stage bound):
    embed_bwd   dE[id] += sum of the rows carrying id (skipping padding_idx and ids outside [0, V)), dP[s] += sum_b.
                work=torch.float32 restates the kernel's documented order: acc from zero over the matching rows in
                ascending row order, then out = out_in + acc; dP the same over b.  Plain fp32 adds (no product to
                contract), so the kernel must equal it bit for bit; the packed kernel equals the dense kernel run on
                the same rows with zeros in the padded rows.  Bound: (rows summed + 1) 2^-24 (sum |x| + |out_in|).
    colsum      db += sum_m dy[m, n].  Stages on the longest path from a term to the result (colsum_stages): the
                lane's ceil(rows_per_block / 8) adds (8 row lanes; the 16-byte path sums a pair of rows, r and r + 8,
                before accumulating it, so it takes half as many), 8 for the shared-memory sum of the 8 lanes,
                row_blocks for add_partials and 1 for the add to db.  row_blocks = min(ceil(M / 64), 6 SMs /
                ceil(N / 256) + 1) is a tuning choice, so the geometry is not restated bit for bit; instead two runs
                must give the same bits.  Bound: stages 2^-24 (sum |dy| + |db_in|).

The optimizer (csrc/optimizer.cu), its hyperparameters taken as the fp32 values the kernels receive (f32):
    grad_sqnorm   sqnorm = sum over every tensor (or the flat slab) of (g inv_scale)^2.  Stages (sqnorm_stages): 3
                  for the term (g k, its square, the 4-term group), CHUNK / 256 for a thread's loop (scalar path), 5
                  shuffles, 8 warps, ceil(parts / 1024) + 10 for add_partials' strided sums and tree, 1 for the add.
                  All terms are positive: |error| <= stages 2^-24 sqnorm.
    optim_prepare ||g|| = sqrt(sqnorm), coef = inv_scale min(1, max_norm / (||g|| + 1e-6)); the amp form divides
                  sqnorm by S^2, so ||g|| = sqrt(sqnorm) / S and coef gains 1 / S.  A set found_inf or a non-finite
                  norm skips the step: st[4] = 1, no counter advance, and grad_norm() = ||g|| on every path.
                  bc1 = 1 - b1^t, bc2s = sqrt(1 - b2^t) with powf in fp32: POW_ULPS ulps of b^t, which 1 - b^t
                  amplifies by b^t / (1 - b^t) at small t -- their own relative term, checked at t = 1, 2 and large t.
    adamw         gi = g coef, m' = b1 m + (1 - b1) gi, v' = b2 v + (1 - b2) gi^2,
                  p' = p (1 - lr wd) - (lr / bc1) m' / (sqrt(v') / bc2s + eps), shadow = T(p') bit for bit from the
                  kernel's own p'.  nvcc contracts to FMA here, so the fp32 result is not matched bit for bit; the
                  allowance counts fp32 operations times 2^-24 of the magnitudes they combine (adamw's docstring),
                  plus the prepare's relative errors carried through coef, bc1 and bc2s.

With OASR_ATTN_REPORT set to a file name, every check appends one JSON line to it (attention_reference's log);
tools/step_error_table.py runs tests/test_step_parity_gpu.py that way and prints the table below.

Measured on an H100 SXM (80 GB HBM3, 700 W power limit, 132 SMs) over tests/test_step_parity_gpu.py: the largest value
over the cases of each group of rule 1 (worst error over its bound; <= 1 passes), rule 2 (unexplained differing
elements over ALPHA x the yardstick's + SLACK; <= 1 passes), the fp32 outputs' element bound (<= 1 passes) with their
row-L2 ratio to the yardstick (<= F32_ALPHA passes), and the optimizer state's (norm, coef, bc1, bc2s) error over its
bound (<= 1 passes).

    group                               dtype  rule 1  rule 2  fp32 bound  other
    stem glue, 2 x 3000, every width    bf16   1.000   0
                                        fp16   0.999   0
    stem glue, T = 37                   bf16   0.998   0
                                        fp16   0.998   0
    stem glue, fp16 overflow            fp16   0.999   0
    stem, B = 32 (col2im, conv1 bias)   bf16   1.000   0       0.00044     bias rows 1.62
                                        fp16   0.999   0
    embedding forward, dense / offset   both   0       0                   bits of the fp32 restatement
    embedding backward (all forms)                             0.675       bits of the kernel-order restatement
    column sums, every step form                               0.0077      rows 1.98
    column sums, scalar path                                   0.0037      rows 1.44
    AdamW flat, tiny, t = 1 .. 10^6                            0.592       rows 1.01, state 0.036
    AdamW flat, 5 x 10^7                                       0.560       rows 1.00, state 0.020
    AdamW flat, amp and skips                                  0.506       rows 0.98, state 0.018
    AdamW pointer table                                        0.543       rows 1.27, state 0.012

Rule 1 sits at 1 because an element one ulp off is 1 / (1 + allowance / ulp) of its bound.  Rule 2 found no
unexplained difference anywhere: every element that differs from the fp64 rounding lies within GELU_GRAD_TOL or fp32
noise of a rounding boundary, and add_pos / embed_fwd differ from it nowhere.  The column-sum bound is structural and
loose (the kernel's worst element used 0.8% of it); the embedding and AdamW allowances are used to 0.68 and 0.59, the
optimizer state's to 0.04 (a bound the powf term dominates at small t).  tests/test_step_parity_gpu.py runs in 34 s on that H100 (58
cases), and fails against builds with col2im's k = 0 and k = 2 taps swapped, col2im without the inner T(), the
embedding backward summing each 128-row batch's matches in reverse order, a column sum that drops one row per lane,
AdamW without the bias-correction square root, or shadows cast from the old master.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import numpy as np
import torch
import torch.nn.functional as F

from tests.attention_reference import _report
from tests.decode_reference import rnd, ulp
from tests.training_reference import GELU_APPROX, N_SMS, gelu_grad

U = 2.0 ** -24
GELU_GRAD_TOL = GELU_APPROX + 2.0 ** -21   # |kernel gelu' - erf gelu'|: A&S (2.1e-7) plus the fp32 evaluation
CHUNK = 16384                              # elements per optimizer block (oasr_optim_chunk_elems)
POW_ULPS = 4                               # CUDA powf's maximum error, in ulps (CUDA C Programming Guide)


def f32(x: float) -> float:
    """The fp32 value a kernel receives for the Python float x."""
    return float(np.float32(x))


def _band(v, n, dtype):
    """v within n of a T rounding boundary."""
    return rnd(v - n, dtype) != rnd(v + n, dtype)


# ---------------------------------------------------------------------------------------------------- exact copies
def im2col_conv1(mel, kpad: int, dtype):
    B, C, T = mel.shape
    cols = F.pad(mel, (1, 1)).unfold(2, 3, 1)                         # (B, C, T, 3): mel[b, c, t + k - 1]
    out = torch.zeros(B * T, kpad, dtype=dtype, device=mel.device)
    out[:, :3 * C] = cols.permute(0, 2, 3, 1).reshape(B * T, 3 * C).to(dtype)
    return out


def conv2_out_len(T_in: int) -> int:
    return (T_in + 2 - 3) // 2 + 1


def im2col_conv2(h, B: int, T_in: int, d: int):
    T_out = conv2_out_len(T_in)
    hp = torch.zeros(B, T_in + 2, d, dtype=h.dtype, device=h.device)
    hp[:, 1:T_in + 1] = h.view(B, T_in, d)
    return torch.stack([hp[:, k:k + 2 * T_out:2] for k in range(3)], dim=2).reshape(B * T_out, 3 * d)


def cast_conv_weight(w, dtype):
    c_out, c_in, _ = w.shape
    return w.permute(0, 2, 1).reshape(c_out, 3 * c_in).to(dtype)


def unpermute_conv_wgrad(g, c_out: int, c_in: int, out=None):
    v = g.view(c_out, 3, c_in).permute(0, 2, 1)
    return v.clone() if out is None else out + v


# ---------------------------------------------------------------------------------------------------- rounded to T
def _gelu_grad_out(h, pre, dtype, work, inner_band=None) -> Dict[str, torch.Tensor]:
    """T(h gelu'(pre)) and, in fp64, rule 1's allowance and rule 2's explained differences."""
    gp = gelu_grad(pre.to(work))
    po = h * gp
    r = {"out": rnd(po, dtype)}
    if work == torch.float64:
        n = GELU_GRAD_TOL * h.abs() + 2.0 ** -21 * po.abs()
        r["extra"], r["expl"] = n, _band(po, n, dtype)
        if inner_band is not None:              # the inner T(sum) one ulp off
            r["extra"] = r["extra"] + torch.where(inner_band, gp.abs() * ulp(h.abs() * (1 + 2.0 ** -7), dtype), torch.zeros_like(n))
            r["expl"] = r["expl"] | inner_band
    return r


def col2im_conv2_gelu_bwd(dA, pre1, B: int, T_in: int, T_out: int, d: int, dtype, work=torch.float64):
    cols = dA.to(work).view(B, T_out, 3, d)
    g = torch.zeros(B, T_in + 2, d, dtype=work, device=dA.device)     # row r at index r + 1
    for k in range(3):                                                 # k = 0 before k = 2, as the kernel adds them
        g[:, k:k + 2 * T_out:2] += cols[:, :, k]
    g = g[:, 1:T_in + 1].reshape(B * T_in, d)
    h = rnd(g, dtype)
    inner = _band(g, U * g.abs(), dtype) if work == torch.float64 else None
    return _gelu_grad_out(h, pre1, dtype, work, inner)


def gelu_bwd(dy, pre, dtype, work=torch.float64):
    return _gelu_grad_out(dy.to(work), pre, dtype, work)


def _add_rounded(po, dtype, work):
    r = {"out": rnd(po, dtype)}
    if work == torch.float64:
        n = U * po.abs()                        # the kernel's fp32 add
        r["extra"], r["expl"] = n, _band(po, n, dtype)
    return r


def add_pos(x, pos, T: int, dtype, work=torch.float64):
    rows = torch.arange(x.shape[0], device=x.device) % T
    return _add_rounded(x.to(work) + pos.to(work)[rows], dtype, work)


def embed_fwd(ids, emb, pos, offset: int, dtype, work=torch.float64, rows=None):
    """ids (B, S); rows: the dense rows b S + t to produce (a packed batch), all of them when None."""
    B, S = ids.shape
    dense = torch.arange(B * S, device=ids.device) if rows is None else rows.long()
    flat = ids.reshape(-1)[dense]
    flat = torch.where((flat < 0) | (flat >= emb.shape[0]), torch.zeros_like(flat), flat)
    return _add_rounded(emb.to(work)[flat] + pos.to(work)[dense % S + offset], dtype, work)


# ---------------------------------------------------------------------------------------------------- fp32 sums
def embed_bwd(ids, dx, demb0, dpos0, padding_idx: int, work=torch.float64) -> Dict[str, Optional[torch.Tensor]]:
    """Dense backward: ids (B, S), dx (B S, d) in T, demb0 (V, d) / dpos0 (S, d) fp32 or None (frozen).  Returns "demb"
    / "dpos" in `work` and, in fp64, "allow_demb" / "allow_dpos".  work=torch.float32 is the kernel's order."""
    B, S = ids.shape
    V = None if demb0 is None else demb0.shape[0]
    x = dx.to(work)
    r: Dict[str, Optional[torch.Tensor]] = {"demb": None, "dpos": None}
    if dpos0 is not None:
        xs = x.view(B, S, -1)
        acc = torch.zeros_like(xs[0])
        for b in range(B):                                   # v = 0; v += dx[b S + s] for b ascending
            acc = acc + xs[b]
        r["dpos"] = dpos0.to(work) + acc
        if work == torch.float64:
            r["allow_dpos"] = (B + 1) * U * (xs.abs().sum(0) + dpos0.double().abs())
    if demb0 is not None:
        flat = ids.reshape(-1)
        valid = (flat != padding_idx) & (flat >= 0) & (flat < V)
        rows = torch.nonzero(valid)[:, 0]
        rid = flat[rows]
        acc = torch.zeros(V, x.shape[1], dtype=work, device=x.device)
        if work == torch.float64:
            acc.index_add_(0, rid, x[rows])
            cnt = torch.zeros(V, dtype=work, device=x.device).index_add_(0, rid, torch.ones_like(rid, dtype=work))
            mag = torch.zeros_like(acc).index_add_(0, rid, x[rows].abs())
            r["allow_demb"] = (cnt[:, None] + 1) * U * (mag + demb0.double().abs())
        else:
            order = torch.argsort(rid, stable=True)           # rows of one id stay in ascending row order
            rs, ids_s = rows[order], rid[order]
            first = torch.ones_like(ids_s, dtype=torch.bool)
            first[1:] = ids_s[1:] != ids_s[:-1]
            start = torch.cummax(torch.where(first, torch.arange(len(ids_s), device=x.device), torch.zeros_like(ids_s)), 0)[0]
            rank = torch.arange(len(ids_s), device=x.device) - start
            for k in range(int(rank.max()) + 1 if len(rank) else 0):   # the k-th row of every id: distinct targets
                sel = rank == k
                acc[ids_s[sel]] = acc[ids_s[sel]] + x[rs[sel]]
        r["demb"] = demb0.to(work) + acc
    return r


def embed_bwd_packed(ids, dx, demb0, dpos0, padding_idx: int, rows, work=torch.float64):
    """The packed backward: dx (N, d) holds dense rows `rows` of ids (B, S).  The same sums as the dense backward with
    zeros in the padded rows."""
    B, S = ids.shape
    dense = torch.zeros(B * S, dx.shape[1], dtype=dx.dtype, device=dx.device)
    dense[rows.long()] = dx
    return embed_bwd(ids, dense, demb0, dpos0, padding_idx, work)


def colsum_stages(M: int, N: int, n_sms: int = N_SMS) -> int:
    """Serial fp32 stages of oasr_colsum16 from a term to the result (module docstring)."""
    col_tiles = -(-N // 256)
    row_blocks = max(1, min(-(-M // 64), n_sms * 6 // col_tiles + 1))
    rpb = -(-M // row_blocks)
    row_blocks = -(-M // rpb)
    return -(-rpb // 8) + 8 + row_blocks + 1


def colsum(dy, db0, work=torch.float64, n_sms: int = N_SMS) -> Dict[str, torch.Tensor]:
    """db0 + column sums of dy (M, N) in T; in fp64 also "allow"."""
    x = dy.to(work)
    r = {"out": db0.to(work) + x.sum(0)}
    if work == torch.float64:
        r["allow"] = colsum_stages(*dy.shape, n_sms=n_sms) * U * (x.abs().sum(0) + db0.double().abs())
    return r


# ---------------------------------------------------------------------------------------------------- optimizer
def sqnorm_stages(n_parts: int) -> int:
    return 3 + CHUNK // 256 + 5 + 8 + -(-n_parts // 1024) + 10 + 1


def n_parts(numels) -> int:
    """Blocks of the norm pass: one per CHUNK of every tensor (a flat slab is one tensor)."""
    return sum(-(-n // CHUNK) for n in numels)


def grad_sqnorm(grads, inv_scale: float, work=torch.float64) -> Dict[str, float]:
    k = f32(inv_scale)
    s = sum(float(((g.to(work) * k) ** 2).sum()) for g in grads)
    r = {"sqnorm": s}
    if work == torch.float64:
        r["allow"] = sqnorm_stages(n_parts([g.numel() for g in grads])) * U * s
    return r


def _pow_rel(b: float, t: float) -> float:
    """Relative error of 1 - powf(b, t) in fp32: POW_ULPS ulps of b^t (at most 2^-23 b^t each), amplified by the
    subtraction, plus its rounding."""
    bt = b ** t
    return POW_ULPS * 2.0 ** -23 * bt / (1.0 - bt) + U


def prepare(sqnorm: float, inv_scale: float, max_norm: float, beta1: float, beta2: float, step: float,
            loss_scale: Optional[float] = None, found_inf: bool = False, sqnorm_allow: float = 0.0) -> Dict[str, float]:
    """optim_prepare(_amp) from the step counter `step` before the call.  Returns the device state's values -- "step",
    "coef", "bc1", "bc2s", "skip", "norm" -- and their relative allowances "*_rel"."""
    nsq, k = sqnorm, f32(inv_scale)
    amp = loss_scale is not None
    if amp:
        nsq, k = nsq / loss_scale ** 2, k / loss_scale
    norm = math.sqrt(nsq) if math.isfinite(nsq) else nsq
    r = {"norm": norm, "norm_rel": 0.5 * sqnorm_allow / max(sqnorm, 1e-300) + (5 if amp else 2) * U}
    if found_inf or not math.isfinite(nsq):
        r.update(step=step, skip=1.0)
        return r
    coef = k * (min(1.0, f32(max_norm) / (norm + f32(1e-6))) if max_norm > 0 else 1.0)
    t = step + 1.0
    b1, b2 = f32(beta1), f32(beta2)
    r.update(step=t, skip=0.0, coef=coef, coef_rel=r["norm_rel"] + (6 if amp else 4) * U,
             bc1=1.0 - b1 ** t, bc1_rel=_pow_rel(b1, t), bc2s=math.sqrt(1.0 - b2 ** t), bc2s_rel=0.5 * _pow_rel(b2, t) + U)
    return r


def adamw(p, g, m, v, st: Dict[str, float], lr: float, beta1: float, beta2: float, eps: float, wd: float,
          work=torch.float64) -> Dict[str, torch.Tensor]:
    """One AdamW update from prepare()'s state `st` (for the yardstick, fp32 values of the same).  Returns "p", "m",
    "v" in `work` and, in fp64, "allow_p" / "allow_m" / "allow_v":
        m'  4 operations (g coef, (1 - b1) gi, b1 m, the add) on |b1 m| + |(1 - b1) gi|, and coef's error on gi;
        v'  6 (gi enters squared, (1 - b2) gi, times gi, b2 v, the add) on |b2 v| + (1 - b2) gi^2, coef's twice;
        p'  the denominator's error (half v''s relative error, sqrt, the divide, bc2s's own, eps's add), the quotient's
            and lr / bc1's roundings and bc1's own on the update, 3 on |p (1 - lr wd)| and 1 on |p'|."""
    b1, b2, lr, eps, wd = (f32(x) for x in (beta1, beta2, lr, eps, wd))
    pw, gw, mw, vw = (t.to(work) for t in (p, g, m, v))
    gi = gw * st["coef"]
    m1 = b1 * mw + (1.0 - b1) * gi
    v1 = b2 * vw + (1.0 - b2) * gi * gi
    s = torch.sqrt(v1) / st["bc2s"]
    den = s + eps
    step_size = lr / st["bc1"]
    upd = step_size * (m1 / den)
    pd = pw * (1.0 - lr * wd)
    p1 = pd - upd
    r = {"p": p1, "m": m1, "v": v1}
    if work == torch.float64:
        cr = st["coef_rel"]
        A, Bm = (b1 * mw).abs(), ((1.0 - b1) * gi).abs()
        am = 4 * U * (A + Bm) + cr * Bm
        C, D = b2 * vw, (1.0 - b2) * gi * gi
        av = 6 * U * (C + D) + 2 * cr * D
        es = s * (0.5 * av / v1.clamp_min(1e-300) + 2 * U + st["bc2s_rel"])
        eden = es + U * den
        eq = (m1.abs() * eden / den + am) / den + U * (m1 / den).abs()
        eu = upd.abs() * (U + st["bc1_rel"]) + step_size * eq + U * upd.abs()
        r.update(allow_m=am, allow_v=av, allow_p=eu + 3 * U * pd.abs() + U * p1.abs())
    return r


def check_scalar(got: float, want: float, rel: float, name: str = "") -> float:
    """|got - want| <= rel |want| for one value of the optimizer's device state; returns the ratio to the bound."""
    if not math.isfinite(want):
        assert (math.isnan(want) and math.isnan(got)) or got == want, f"{name}: {got!r} vs {want!r}"
        return 0.0
    ratio = abs(got - want) / max(rel * abs(want), 1e-300) if got != want else 0.0
    _report(kind="scalar", name=name, worst=ratio)
    assert ratio <= 1.0, f"{name}: {got!r} vs {want!r} ({ratio:.3g} x its bound {rel:.3g})"
    return ratio
