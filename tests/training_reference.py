"""fp64 reference of the training step's GEMM, LayerNorm and cross-entropy kernels and the tolerance rule their tests
use (TEST INFRASTRUCTURE).

Plain torch, on whichever device the inputs live; no import of olmoasr_b200.  Each function states one kernel launch
at the rounding points its source writes down, in the activation type T (bf16 or fp16):

    gemm            csrc/gemm_sm90.cu, acc = sum_k A[m,k] B[n,k] over the logical (M, K) / (N, K) operands:
                    BF16       h = T(acc + T(bias))
                    GELU       (h, T(gelu_erf(h)))
                    RESIDUAL   T(aux + h)
                    GELU_BWD   T(h gelu_erf'(aux))          (production passes no bias: h = T(acc))
                    F32        acc + bias                   (the fp32 bias, unrounded)
                    F32_ATOMIC_ADD  out0 + acc; split-K: out0 + (p0 + p1 + ...), the partials over the kernel's k-block
                               ranges added in split order (no bias: the kernel rejects one)
    layernorm_fwd   csrc/layernorm.cu: two-pass statistics of each row, y = T((x - mean) rstd w + b)
    layernorm_bwd   dx_ln = rstd (dy w - mean(dy w) - xhat mean(dy w xhat)), dx = T(dres + T(dx_ln)) with a residual
                    gradient, T(dx_ln) without; dw = sum_rows dy xhat, db = sum_rows dy (fp32 outputs)
    ce_fwd          csrc/cross_entropy.cu: lse = logsumexp(logits[:, :V]) per counted row (0 for the others), loss =
                    sum over counted rows of (lse - x[y]) / count; a row counts when y != ignore_index and 0 <= y < V,
                    a target outside [0, V) that is not ignore_index is counted as bad
    ce_bwd          d = T(g (exp(x - lse) - [c == y])), g = grad_out / count; ignored and bad rows get d = 0

`work=torch.float64` is the statement: every value between two rounding points is exact (to fp64).
`work=torch.float32` is the rounding-point yardstick: the same computation in fp32 (TF32 off), rounded to T at the
same points.  Its distance from fp64 is what fp32 arithmetic between T roundings costs.

The rule for an output rounded once to T (`check16`, decode_reference.check_linear's two parts):

 1. Every element lies within one T ulp of the fp64 rounded value plus an allowance for the kernel's fp32 error.
    GEMM: every k16 wgmma adds one 16-product sum into the fp32 accumulator registers, so a product passes through at
    most ceil(K / 16) accumulations, plus one for the alignment inside the 16-product sum and one for the bias add;
    split-K adds the partials in order (one stage per split) and the result to out0 (one more).  Each stage errs by at
    most 2^-23 of the sum of |terms| beneath it whatever its rounding mode (the tensor-core adder aligns and
    truncates), so

        |acc_kernel - acc| <= E = (ceil(K / 16) + 2 [+ splits + 1]) 2^-23 (sum_k |A B| + |bias| [+ |out0|]).

    At K = 51865 that is 3244 x 2^-23 where the textbook (K - 1) 2^-24 is 25932 x 2^-23.  (Each stage's 2^-23 is
    an upper bound of one truncation; the measured worst element used 0.33 of E at that K.)  An inner rounding (the
    GELU, RESIDUAL and GELU_BWD input h) may flip too: one more inner ulp, times max |gelu'| = 1.13 for GELU and
    |gelu'(aux)| for GELU_BWD.
    GELU and GELU' are not erf: the epilogue evaluates the Abramowitz-Stegun erf (common.cuh gelu_core2) with
    rcp.approx / ex2.approx.  Its distance from erf-GELU and erf-GELU', evaluated in fp64, is below GELU_APPROX
    (absolute; tests/test_training_reference_host.py checks it on a dense grid), and the fp32 evaluation adds a few
    2^-24 of |h|; both are in the allowance.
    LayerNorm forward: the fp32 statistics move z by at most 2^-20 ((|x - mean| + |mean|) rstd |w| + |b|)
    (decode_reference's LAYERNORM allowance).  Backward: the row sums of dy w and dy w xhat pass through d / 32 + 5
    fp32 stages (8-wide vectors per lane, then 5 shuffles) and xhat carries the fp32 mean's error, q = mean|x| rstd
    units of 2^-24 per stage, so E = (d / 32 + 10) 2^-24 rstd (|dy w| + mean|dy w| + (|xhat| + q) mean(|dy w| (|xhat| + q))).
    Cross-entropy backward: the kernel's lse is within LSE_TOL (1 + max|x|) of the row's (the lse rule below), and
    __expf of the fp32 difference x - lse errs by 2^-22 (3 + 1.5 |x - lse|) relative, so
    E = |g| p (LSE_TOL (1 + max|x|) + 2^-22 (3 + 1.5 |x - lse|)) + 2^-21 |pre|.
 2. Elements that differ at all from the fp64 rounded value, leaving out those whose difference an approximation the
    kernel is allowed explains (the pre-rounding value within fp32 noise, GELU_APPROX, or the lse allowance of a
    rounding boundary): at most ALPHA x the yardstick's count plus SLACK(n) = 4 + n / 4096.  A tanh GELU (4.7e-4 from
    erf), an unrounded bias or a variance over d - 1 stays far below one ulp and still moves a few percent of the
    roundings, which this part sees.

fp32 outputs (`check32`: the F32 / F32_ATOMIC_ADD GEMMs, LayerNorm dw / db): every element within its stage bound E of
the fp64 value (for the LayerNorm column sums, over rows / (8 blocks) + 8 + blocks serial stages with blocks = min(rows
/ 8, 2 x SMs)), and the relative L2 error of every row (a GEMM output row, or the whole dw / db vector) within
F32_ALPHA x the yardstick's, both for the worst and the mean row.

lse (`check_lse`): the kernel's within LSE_TOL (1 + max|x|) of the fp64 logsumexp, per row, the attention kernels'
form; the mean loss within the mean of those plus the fp32 sum's (rows / 1024 + 12) 2^-24 of mean |lse - x_y|.

With OASR_ATTN_REPORT set to a file name, every check appends one JSON line to it (attention_reference's log);
tools/training_error_table.py runs tests/test_training_parity_gpu.py that way and prints the table below.

Measured on an H100 SXM (80 GB HBM3, 700 W power limit) over tests/test_training_parity_gpu.py: the largest value
over the cases of each group of rule 1 (worst error over its bound; <= 1 passes), of rule 2 (unexplained differing
elements over ALPHA x the yardstick's + SLACK; <= 1 passes), and of the fp32 outputs' row ratios to the yardstick
(<= F32_ALPHA passes) and lse errors in LSE_TOL units (<= 1 passes).

    group                      dtype  rule 1  rule 2  count ratio  other
    forward forms              bf16   0.998   0.46    13.8
                               fp16   0.989   0.39     8.0
    conv stem                  bf16   0.999   0.52    11.3
                               fp16   0.994   0.28     5.5
    dgrad forms                bf16   0.998   0.30     8.9
                               fp16   0.984   0.26     5.6
    edges (tails, 3 SMs)       bf16   0.999   0.08     1.5
                               fp16   0.998   0.08     2.0
    MN-major, padded strides   bf16   0.999   0.08     1.0    f32 rows 1.24 / 1.19, bound 0.13
                               fp16   0.998   0.07     1.5
    GELU inputs in [-8, 8]     bf16   0.607   0
                               fp16   0.774   0
    fp16 overflow              fp16   0.483   0
    wgrad forms (fp32)                                       f32 rows 19.0 / 20.5, bound 0.030
    tied logits                bf16   0.999   0.48    72.1   f32 rows 6.77 / 7.34, bound 0.020 (the dgrad's
                               fp16   0.990   0.21    32     count ratio, under LOGITS_ALPHA = 150 of its test)
    cross-entropy backward     bf16   0.998   0       0      lse 0.11, loss 0.011
                               fp16   1.000   0       0
    LayerNorm                  bf16   1.000   0.04     2.0   f32 (dw, db) 3.17 / 3.17, bound 0.005
                               fp16   0.999   0.05     1.7

Rule 1 sits just under 1 because an element one ulp off is 1 / (1 + allowance / ulp) of its bound.  The tensor-core
accumulation flips up to 14 x as many T roundings as cuBLAS's fp32 sum at K = 4d (fc2, bf16, d = 1024 -- decode_reference
saw "several times" at its smaller K), so ALPHA = 20; that leaves every deliberately wrong GEMM of
tests/test_training_reference_host.py failing by 6 or more.  At K = 51865 (the logits dgrad) the ratio reaches 72 and its
test states its own bound.  The wgmma wgrad's fp32 row error is up to 20.5 x cuBLAS's (3.6e-6 against 1.5e-7 .. 7.7e-7
relative over 3000 rows) while every element stays within 3% of its stage bound: F32_ALPHA = 32.  lse errors reach 0.11
LSE_TOL.  The fp16 GELU flips the rule admits through GELU_APPROX were measured with the rest: no fp16 GELU case came
near rule 2's limit (conv stem 0.28, forward forms 0.39).
tests/test_training_parity_gpu.py runs in 20 s on that H100 (199 cases), and fails against builds with a tanh GELU in
the GEMM epilogue, the bias slice not rounded to T, the K tail dropped (kblocks_total = K / BK), the LayerNorm variance
over d - 1, or the cross-entropy backward's scalar tail loop without its one-hot.
"""
from __future__ import annotations

from typing import Dict, List, NamedTuple, Sequence

import torch

from tests.attention_reference import _report
from tests.decode_reference import _exact_fp32, gelu, layer_norm, rnd, slack, ulp

EPI_BF16, EPI_GELU, EPI_RESIDUAL, EPI_GELU_BWD, EPI_F32, EPI_F32_ATOMIC_ADD = range(6)
BK = 64                    # the GEMM's k-block: split-K splits whole k-blocks
ALPHA = 20.0
F32_ALPHA = 32.0
LSE_TOL = 2.0 ** -20
GELU_APPROX = 2.5e-7       # |A&S GELU - erf GELU| and |A&S GELU' - erf GELU'| in fp64 (host-checked: 2.1e-7)
GELU_SLOPE = 1.13          # max |gelu'(x)| = 1.1289 (at x = 0.7518)
N_SMS = 132                # the H100 SXM's SMs: the LayerNorm backward runs at most 2 blocks per SM


def gelu_grad(x):
    """Exact (erf) GELU': Phi(x) + x phi(x)."""
    return 0.5 * (1.0 + torch.erf(x * 0.7071067811865476)) + x * torch.exp(-0.5 * x * x) * 0.3989422804014327


def _as_poly(x):
    """(erf(|x| / sqrt 2), exp(-x^2 / 2)) by the Abramowitz-Stegun 7.1.26 form of gelu_core2, in x's type."""
    t = 1.0 / (1.0 + 0.23164189 * x.abs())
    p = ((((1.061405429 * t - 1.453152027) * t + 1.421413741) * t - 0.284496736) * t + 0.254829592)
    e = torch.exp(-0.5 * x * x)
    return 1.0 - p * t * e, e


def gelu_as(x):
    """The GEMM epilogue's GELU (gelu_erf2) evaluated in x's type: hx + |hx| erf(|x| / sqrt 2)."""
    ea, _ = _as_poly(x)
    hx = 0.5 * x
    return hx + hx.abs() * ea


def gelu_grad_as(x):
    """The GEMM epilogue's GELU' (gelu_erf_grad2) evaluated in x's type."""
    ea, e = _as_poly(x)
    return 0.5 + 0.5 * torch.sign(x) * ea + x * 0.3989422804014327 * e


def split_ranges(K: int, split_k: int):
    """The k ranges of gemm()'s splits: whole k-blocks of BK, ceil(kblocks / split_k) per split, the last one short."""
    kb = -(-K // BK)
    split_k = max(1, min(split_k, kb))
    per = -(-kb // split_k)
    return [(s * per * BK, min((s + 1) * per * BK, K)) for s in range(-(-kb // per))]


def gemm_stages(K: int, splits: int = 1, accumulate: bool = False) -> int:
    """Rounding stages of the wgmma accumulation of K products, the bias add, the split-K sum and the add to out0."""
    return -(-K // 16) + 2 + (splits if splits > 1 else 0) + (1 if accumulate else 0)


# ---------------------------------------------------------------------------------------------------------- statements
def gemm(A, B, epi, dtype, bias=None, aux=None, out0=None, split_k: int = 1, work=torch.float64) -> Dict[str, torch.Tensor]:
    """One GEMM launch: A (M, K) and B (N, K) in T (logical operands: transpose MN-major storage first), bias (N,) fp32,
    aux (M, N) in T, out0 (M, N) fp32 (F32_ATOMIC_ADD).  Returns in `work` "out" (and "out2", GELU's second output)
    and, in fp64, "extra" / "extra2" (the allowance beyond one ulp) and "expl" / "expl2" (rule 2's explained
    differences) for the 16-bit outputs, "allow" for the fp32 ones."""
    with _exact_fp32():
        a, b = A.to(work), B.to(work)
        K = a.shape[1]
        ranges = split_ranges(K, split_k) if epi == EPI_F32_ATOMIC_ADD else [(0, K)]
        acc = None
        for k0, k1 in ranges:       # the partials, added in split order
            part = a[:, k0:k1] @ b[:, k0:k1].t()
            acc = part if acc is None else acc + part
        exact = work == torch.float64
        mag = (a.abs() @ b.abs().t()) if exact else None
        if epi in (EPI_F32, EPI_F32_ATOMIC_ADD):
            if epi == EPI_F32:
                out = acc if bias is None else acc + bias.to(work)
                side = 0.0 if bias is None else bias.to(work).abs()
            else:
                out = out0.to(work) + acc
                side = out0.to(work).abs()
            r = {"out": out}
            if exact:
                st = gemm_stages(K, len(ranges), epi == EPI_F32_ATOMIC_ADD)
                r["allow"] = st * 2.0 ** -23 * (mag + side) + 2.0 ** -24 * out.abs()
            return r
        rb = torch.zeros(b.shape[0], dtype=work, device=b.device) if bias is None else rnd(bias.to(work), dtype)
        pre = acc + rb
        h = rnd(pre, dtype)
        if epi == EPI_GELU:
            r = {"out": h, "out2": rnd(gelu(h), dtype)}
        elif epi == EPI_RESIDUAL:
            po = aux.to(work) + h
            r = {"out": rnd(po, dtype)}
        elif epi == EPI_GELU_BWD:
            gp = gelu_grad(aux.to(work))
            po = h * gp
            r = {"out": rnd(po, dtype)}
        else:
            r = {"out": h}
        if not exact:
            return r
        E = gemm_stages(K) * 2.0 ** -23 * (mag + rb.abs())
        noise = lambda v: 2.0 ** -21 * v.abs()               # noqa: E731  fp32 rounding of the epilogue's arithmetic
        band = lambda v, n: rnd(v - n, dtype) != rnd(v + n, dtype)   # noqa: E731  v within n of a rounding boundary
        h_flip = ulp(h.abs() * (1 + 2.0 ** -7), dtype)      # the kernel's h one ulp off the reference's
        if epi == EPI_GELU:
            r["extra"], r["expl"] = E, band(pre, noise(pre))
            gv = gelu(h)
            n2 = GELU_APPROX + noise(gv) + noise(h)
            r["extra2"], r["expl2"] = GELU_SLOPE * (h_flip + E) + n2, band(gv, n2)
        elif epi == EPI_RESIDUAL:
            r["extra"], r["expl"] = h_flip + E, band(po, noise(po))
        elif epi == EPI_GELU_BWD:
            n = GELU_APPROX * h.abs() + noise(po)
            r["extra"], r["expl"] = gp.abs() * (h_flip + E) + n, band(po, n)
        else:
            r["extra"], r["expl"] = E, band(pre, noise(pre))
        return r


def _row_stats(x, work):
    xf = x.to(work)
    mean = xf.mean(dim=-1, keepdim=True)
    c = xf - mean
    return xf, mean, c, (c * c).mean(dim=-1, keepdim=True)


def layernorm_fwd(x, w, b, eps, dtype, work=torch.float64) -> Dict[str, torch.Tensor]:
    """LayerNorm forward of x (rows, d) in T with fp32 w, b: "out" (T-rounded, in `work`), "mean", "rstd" (rows,) and,
    in fp64, "extra" / "expl"."""
    y, z, mean, rstd = layer_norm(x, w, b, eps, dtype, work)
    r = {"out": y, "mean": mean[:, 0], "rstd": rstd[:, 0]}
    if work == torch.float64:
        n = 2.0 ** -20 * (((x.double() - mean).abs() + mean.abs()) * rstd * w.double().abs() + b.double().abs())
        r["extra"], r["expl"] = n, rnd(z - n, dtype) != rnd(z + n, dtype)
    return r


def ln_sum_stages(rows: int, n_sms: int = N_SMS) -> int:
    """Serial fp32 stages of the LayerNorm backward's column sums: a lane's rows, the 8-warp fold, the block partials."""
    blocks = min(-(-rows // 8), 2 * n_sms)
    return -(-rows // (8 * blocks)) + 8 + blocks


def layernorm_bwd(dy, x, w, eps, dtype, dres=None, work=torch.float64) -> Dict[str, torch.Tensor]:
    """LayerNorm backward: dy, x (rows, d) in T, w fp32, dres (rows, d) in T or None.  Returns "out" (dx, T-rounded, in
    `work`), "dw", "db" (d,) and, in fp64, "extra" / "expl" for dx and "allow_dw" / "allow_db"."""
    d = x.shape[1]
    xf, mean, c, var = _row_stats(x, work)
    rstd = torch.rsqrt(var + eps)
    xhat = c * rstd
    g = dy.to(work)
    gw = g * w.to(work)
    m1 = gw.mean(dim=-1, keepdim=True)
    m2 = (gw * xhat).mean(dim=-1, keepdim=True)
    dxln = rstd * (gw - m1 - xhat * m2)
    if dres is None:
        po = dxln
    else:
        inner = rnd(dxln, dtype)
        po = dres.to(work) + inner
    r = {"out": rnd(po, dtype), "dw": (g * xhat).sum(dim=0), "db": g.sum(dim=0)}
    if work == torch.float64:
        u = 2.0 ** -24
        q = xf.abs().mean(dim=-1, keepdim=True) * rstd            # the fp32 mean's error in units of xhat
        xa = xhat.abs() + q
        E = (d / 32 + 10) * u * rstd * (gw.abs() + gw.abs().mean(dim=-1, keepdim=True) + xa * (gw.abs() * xa).mean(dim=-1, keepdim=True))
        n = 2.0 ** -21 * po.abs()
        r["extra"] = E + n if dres is None else ulp(inner.abs() * (1 + 2.0 ** -7), dtype) + E + n
        r["expl"] = rnd(po - n, dtype) != rnd(po + n, dtype)
        st = ln_sum_stages(x.shape[0])
        r["allow_dw"] = st * u * (g.abs() * xhat.abs()).sum(dim=0) + (d / 32 + 10) * u * (g.abs() * xa).sum(dim=0)
        r["allow_db"] = st * u * g.abs().sum(dim=0)
    return r


def counted_rows(targets, V: int, ignore_index: int):
    """Rows the loss counts: target != ignore_index and inside [0, V)."""
    return (targets != ignore_index) & (targets >= 0) & (targets < V)


def ce_fwd(logits, targets, V: int, ignore_index: int, work=torch.float64, slab: int = 2048) -> Dict[str, torch.Tensor]:
    """Cross-entropy forward of logits (rows, >= V) in T; only columns [0, V) are read.  Returns "lse" (rows,; 0 for
    rows not counted), "xmax" (max |finite logit| per row), "loss_sum", "count", "bad" and "loss", in `work`.  Row
    slabs keep the fp64 copy of the logits small."""
    rows = logits.shape[0]
    lse = torch.zeros(rows, dtype=work, device=logits.device)
    xmax = torch.zeros(rows, dtype=torch.float64, device=logits.device)
    xy = torch.zeros(rows, dtype=work, device=logits.device)
    cnt = counted_rows(targets, V, ignore_index)
    for r0 in range(0, rows, slab):
        x = logits[r0:r0 + slab, :V].to(work)
        lse[r0:r0 + slab] = torch.logsumexp(x, dim=-1)
        xmax[r0:r0 + slab] = torch.where(torch.isfinite(x), x.abs(), torch.zeros_like(x)).amax(dim=-1).double()
        xy[r0:r0 + slab] = x.gather(1, targets[r0:r0 + slab].clamp(0, V - 1)[:, None])[:, 0]
    lse = torch.where(cnt, lse, torch.zeros_like(lse))
    loss_sum = (lse - xy)[cnt].sum()
    count = cnt.sum().to(work)
    bad = (~cnt & (targets != ignore_index)).sum()
    return {"lse": lse, "xmax": xmax, "xy": xy, "loss_sum": loss_sum, "count": count, "bad": bad, "loss": loss_sum / count,
            "counted": cnt}


def ce_bwd(logits, targets, V: int, ignore_index: int, grad_out: float, count, dtype, lse=None, xmax=None,
           work=torch.float64) -> Dict[str, torch.Tensor]:
    """d(loss)/d(logits[:, :V]) of a row slab, rounded to T, in `work`: g (exp(x - lse) - onehot) with g = grad_out /
    count for counted rows, 0 for the others.  lse / xmax: the slab's from ce_fwd (computed here when None).  In fp64
    also "extra" / "expl"."""
    x = logits[:, :V].to(work)
    if lse is None:
        lse = torch.logsumexp(x, dim=-1)
    cnt = counted_rows(targets, V, ignore_index)
    g = torch.tensor(grad_out, dtype=work, device=x.device) / torch.as_tensor(count, dtype=work, device=x.device)
    gr = torch.where(cnt, g, torch.zeros_like(g))[:, None]
    dx = x - lse.to(work)[:, None]
    p = torch.exp(dx)
    onehot = torch.zeros_like(x)
    onehot.scatter_(1, targets.clamp(0, V - 1)[:, None], 1.0)
    pre = gr * (p - onehot)
    r = {"out": rnd(pre, dtype)}
    if work == torch.float64:
        if xmax is None:
            xmax = torch.where(torch.isfinite(x), x.abs(), torch.zeros_like(x)).amax(dim=-1)
        delta = LSE_TOL * (1.0 + xmax.double())[:, None]
        gp = gr.abs() * p
        e_exp = torch.where(p > 0, 2.0 ** -22 * (3.0 + 1.5 * dx.abs()), torch.zeros_like(p))
        n = gp * delta + 2.0 ** -21 * pre.abs()
        r["extra"] = gp * (delta + e_exp) + 2.0 ** -21 * pre.abs()
        r["expl"] = rnd(pre - n, dtype) != rnd(pre + n, dtype)
    return r


# ---------------------------------------------------------------------------------------------------------- the rule
class Errors16(NamedTuple):
    worst: float        # largest |got - ref| in units of the element's bound (rule 1: <= 1)
    n_diff: int         # elements that differ from the fp64 rounded value, not explained
    emu_diff: int       # the same for the yardstick
    numel: int


def errors16(got, ref, emu, dtype, key: str = "out") -> Errors16:
    """Rule 1 and 2 counts of one T output against ref / emu from a statement in fp64 / fp32.  Elements the reference
    makes non-finite (fp16 overflow to +-inf) must be the same value in the kernel's output; NaN nowhere else."""
    sfx = key[3:]                           # "" or "2"
    g, r, e = got.double(), ref[key], emu[key].double()
    spec = ~torch.isfinite(r)
    gs = ~torch.isfinite(g)
    assert torch.equal(gs, spec), f"non-finite elements differ: {int((gs != spec).sum())} of {g.numel()}"
    assert bool(((g[spec] == r[spec]) | (torch.isnan(g[spec]) & torch.isnan(r[spec]))).all()), "a different infinity"
    fin = ~spec
    g, r, e = g[fin], r[fin], e[fin]
    extra, expl = ref["extra" + sfx][fin], ref["expl" + sfx][fin]
    tol = ulp(torch.maximum(g.abs(), r.abs()), dtype) + extra
    diff = (g - r).abs()
    worst = float((diff / tol).max()) if diff.numel() else 0.0
    n_diff, emu_diff = int(((g != r) & ~expl).sum()), int(((e != r) & ~expl).sum())
    return Errors16(worst, n_diff, emu_diff, int(fin.sum()))


def merge16(parts: Sequence[Errors16]) -> Errors16:
    """Errors of one output computed in slabs."""
    return Errors16(max(p.worst for p in parts), sum(p.n_diff for p in parts), sum(p.emu_diff for p in parts),
                    sum(p.numel for p in parts))


def fail_ratio16(r: Errors16) -> float:
    """How far the rule is from accepting r (<= 1: accepted)."""
    return max(r.worst, r.n_diff / (ALPHA * r.emu_diff + slack(r.numel)))


def check16(r, dtype, name: str = "", alpha: float = ALPHA) -> Errors16:
    """Assert the rule for a T output: r an Errors16 or the slabs' list of them (alpha: rule 2's ALPHA)."""
    if not isinstance(r, Errors16):
        r = merge16(r)
    _report(kind="t16", name=name, dtype=str(dtype).removeprefix("torch."), alpha=alpha, **r._asdict())
    assert r.worst <= 1.0, f"{name}: an element is {r.worst:.3g} x its bound off the fp64 value ({r})"
    assert r.n_diff <= alpha * r.emu_diff + slack(r.numel), f"{name}: {r.n_diff} of {r.numel} elements differ ({r})"
    return r


class Errors32(NamedTuple):
    worst: float        # largest |got - ref| over its bound
    row_worst: float    # the kernel's largest / mean row relative L2 error
    row_mean: float
    emu_worst: float    # the same for the yardstick
    emu_mean: float


def errors32(got, ref, emu, allow) -> Errors32:
    """An fp32 output (rows, n) or (n,) against the fp64 value ref with per-element bound allow, and the yardstick."""
    g, r, e = (t.double().reshape(-1, t.shape[-1]) for t in (got, ref, emu))
    a = allow.double().reshape(r.shape)
    assert bool(torch.isfinite(g).all()), "a non-finite fp32 result"
    worst = float(((g - r).abs() / a.clamp_min(1e-300)).max())
    norm = r.norm(dim=1).clamp_min(1e-300)
    eg, ee = (g - r).norm(dim=1) / norm, (e - r).norm(dim=1) / norm
    return Errors32(worst, float(eg.max()), float(eg.mean()), float(ee.max()), float(ee.mean()))


def merge32(parts: Sequence[Errors32], rows: Sequence[int]) -> Errors32:
    n = sum(rows)
    return Errors32(max(p.worst for p in parts), max(p.row_worst for p in parts), sum(p.row_mean * k for p, k in zip(parts, rows)) / n,
                    max(p.emu_worst for p in parts), sum(p.emu_mean * k for p, k in zip(parts, rows)) / n)


def fail_ratio32(r: Errors32) -> float:
    return max(r.worst, r.row_worst / (F32_ALPHA * max(r.emu_worst, 1e-300)), r.row_mean / (F32_ALPHA * max(r.emu_mean, 1e-300)))


def check32(r: Errors32, name: str = "") -> Errors32:
    """Assert the fp32-output rule: every element within its bound, the worst and mean row L2 within F32_ALPHA x the
    yardstick's."""
    _report(kind="f32", name=name, **r._asdict(), worst_ratio=r.row_worst / max(r.emu_worst, 1e-300),
            mean_ratio=r.row_mean / max(r.emu_mean, 1e-300))
    assert r.worst <= 1.0, f"{name}: an element is {r.worst:.3g} x its bound off the fp64 value ({r})"
    assert r.row_worst <= F32_ALPHA * r.emu_worst and r.row_mean <= F32_ALPHA * r.emu_mean, f"{name}: {r}"
    return r


def lse_error(got, ref) -> float:
    """Worst |lse_kernel - lse| / (1 + max|x|) over the counted rows, in LSE_TOL units; rows not counted must be 0."""
    cnt = ref["counted"]
    g = got.double()
    assert bool((g[~cnt] == 0).all()), "lse of a row that does not count is not 0"
    if not bool(cnt.any()):
        return 0.0
    return float(((g - ref["lse"].double()).abs() / (1.0 + ref["xmax"]))[cnt].max()) / LSE_TOL


def loss_bound(ref) -> float:
    """Allowance of the mean loss: the mean lse bound plus the fp32 loss sum's (rows / 1024 + 12) 2^-24 stages."""
    cnt = ref["counted"]
    n = max(int(cnt.sum()), 1)
    rows = cnt.numel()
    lse_part = float((LSE_TOL * (1.0 + ref["xmax"]))[cnt].sum()) / n
    sum_part = (rows / 1024 + 12) * 2.0 ** -24 * float((ref["lse"] - ref["xy"]).double().abs()[cnt].sum()) / n
    return lse_part + sum_part + 2.0 ** -23 * abs(float(ref["loss"]))


def check_lse(got_lse, got_loss, ref, name: str = "ce") -> float:
    """Assert the lse rule for every counted row and the loss bound; returns the worst lse error in LSE_TOL units."""
    worst = lse_error(got_lse, ref)
    loss_err = abs(float(got_loss) - float(ref["loss"])) / loss_bound(ref)
    _report(kind="lse", name=name, lse_tol_units=worst, loss_units=loss_err)
    assert worst <= 1.0, f"{name}: lse error {worst:.3g} x LSE_TOL"
    assert loss_err <= 1.0, f"{name}: loss {float(got_loss)!r} vs {float(ref['loss'])!r} ({loss_err:.3g} x its bound)"
    return worst


def rows_in_slabs(n: int, slab: int) -> List[slice]:
    return [slice(r0, min(r0 + slab, n)) for r0 in range(0, n, slab)]


def gemm_in_slabs(got, A, B, epi, dtype, slab: int = 1024, keys=("out",), **kw) -> Dict[str, Errors16]:
    """errors16 of a 16-bit GEMM output computed one row slab of A at a time (the fp64 product of a tied-logits
    launch is 5.9 GB whole).  got: the output (M, >= N), or for GELU the pair (h, g)."""
    N = B.shape[0]
    outs = got if isinstance(got, tuple) else (got,)
    parts: Dict[str, list] = {k: [] for k in keys}
    for s in rows_in_slabs(A.shape[0], slab):
        kws = {k: (v[s] if k == "aux" and v is not None else v) for k, v in kw.items()}
        ref = gemm(A[s], B, epi, dtype, **kws)
        emu = gemm(A[s], B, epi, dtype, work=torch.float32, **kws)
        for k, o in zip(keys, outs):
            parts[k].append(errors16(o[s, :N], ref, emu, dtype, key=k))
        del ref, emu
    return {k: merge16(v) for k, v in parts.items()}
