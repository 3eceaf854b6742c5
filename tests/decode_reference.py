"""fp64 reference of the device decoder's step (csrc/decode.cu) and the tolerance rule its tests use (TEST INFRASTRUCTURE).

Plain torch, on whichever device the inputs live; no import of olmoasr_b200.  Each function states one launch of the
step at the rounding points of decode.cu's header, in the activation type T (bf16 or fp16):

    dec_embed    T(emb[tok] + pos[p]), the add in fp32 (the embeddings are fp32 parameters); tokens outside
                 [0, V) read row 0
    dec_linear   x-mode   PLAIN: x;  LAYERNORM: round_T((x - mean) rstd g + b) with two-pass statistics of the row;
                          PARTIAL_SUM: round_T(sum of the fp32 partials, added in split order)
                 epilogue STORE / QKV_SCATTER: round_T(acc + round_T(bias));  GELU: round_T(gelu_erf(that));
                          RESIDUAL: round_T(res + that);  LOGITS_F32: float(round_T(acc))
    decode attention  round_T(q s) . round_T(k s) rounded to T, softmax, P rounded to T, P V unrounded (s = 64^-1/4)

`linear(..., work=torch.float64)` is the statement: every value between two rounding points is exact (to fp64).
`linear(..., work=torch.float32)` is the rounding-point yardstick: the same computation in fp32, rounded to T at the
same points.  Its distance from fp64 is what fp32 arithmetic between T roundings costs.  `step()` composes the
statements into one decoder step.

The rule for an output rounded once to T (`check_linear`):

 1. Every element lies within one T ulp of the fp64 rounded value, plus an allowance for the kernel's fp32 error.
    The kernel forms acc = sum_k x_k w_k with m16n8k16 MMAs: each of the 8 warps accumulates K/8 products in K/128
    MMAs, the 8 warp sums are added in order, then the bias.  That is at most K/128 + 10 rounding stages on any path
    from a product to the result, and each stage errs by at most 2^-23 of the sum of |terms| beneath it, whatever
    its rounding mode (the tensor-core adder aligns and truncates).  So

        |acc_kernel - acc| <= E = (K/128 + 10) 2^-23 (sum_k |x_k w_k| + |bias|).

    At K = 5120 that is 50 x 2^-23, where the textbook (K - 1) 2^-24 sum |x w| is 2560 x 2^-23 -- wider than a bf16
    ulp of most outputs, so it would accept anything.  E matters only where the terms cancel.  An inner rounding
    (GELU's and RESIDUAL's input) may flip too: one more inner ulp, times max |gelu'| = 1.13 for GELU.
    In LAYERNORM mode the fp32 statistics may flip the T rounding of a normalised input x_k that lies within
    d_k = 2^-20 ((|x_k - mean| + |mean|) rstd |g_k| + |b_k|) of a rounding boundary; each such x_k adds
    ulp_T(x_k) |w_k| to the allowance.
 2. Elements that differ at all from the fp64 rounded value, leaving out those whose difference the inputs' own
    rounding explains (the inner value within the LayerNorm / partial-sum allowance of a rounding boundary, or the
    outer value within fp32 noise of one): at most ALPHA x the yardstick's count plus SLACK(n) = 4 + n / 4096.
    This is the part that sees subtle errors: a tanh GELU, an unrounded bias or a statistics error far below one
    ulp still moves a few percent of the roundings.  Counting every difference does not work: when the fp32
    statistics flip one normalised input of a row, about 2 / sqrt(K) of that row's outputs flip with it (4810
    logits of 64 rows at d = 512 in bf16, against the yardstick's 360 -- its flips fall in other rows), and the
    tensor-core accumulation flips several times more roundings than cuBLAS's fp32 sum does.

The composed step (`check_rows`) is compared per row (one sequence's logits, one K or V row of one layer) by relative
L2 error against the fp64 step, with the yardstick's error as the scale, like attention_reference.check:

    max row error (kernel)  <= STEP_ALPHA x max row error (yardstick)
    mean row error (kernel) <= STEP_ALPHA x mean row error (yardstick)

With OASR_ATTN_REPORT set to a file name, check_linear(), check_rows() and check_attention() append one JSON line per call to it
(attention_reference's log); tools/decode_error_table.py runs tests/test_decode_parity_gpu.py that way and prints the
table below.

Measured on an H100 SXM (80 GB HBM3, 700 W power limit) over tests/test_decode_parity_gpu.py:
the largest value over the cases of each group of rule 1 (worst error over its bound; <= 1 passes) and of rule 2
(unexplained differing elements over ALPHA x the yardstick's + SLACK; <= 1 passes), and for the composed step the
largest max-row / mean-row ratios to the yardstick (<= STEP_ALPHA passes).

    group                 dtype  rule 1   rule 2   other
    dec_linear forms      bf16   0.999    0.50
                          fp16   0.989    0.56
    LayerNorm regimes     bf16   0.997    0.24
                          fp16   0.992    0.26
    fp16 overflow         fp16   0.990    0.00
    QKV scatter           bf16   0.994    0.15
                          fp16   0.974    0.10
    step, by launch       bf16   0.999    0.44     attention launches 0.61 u
                          fp16   0.992    0.71     attention launches 2.34 u
    prepare (bf16 GEMM)   bf16   0.995    0.63
    composed step         bf16                     1.05 / 1.22
                          fp16                     1.07 / 1.01

Rule 1 sits just under 1 because an element one ulp off is 1 / (1 + allowance / ulp) of its bound.  The tightest
rule-2 case was fc2 of a one-row step at d = 1024 in fp16: 3 unexplained differences where the yardstick had none
(SLACK admits 4); the largest ratio to a non-zero yardstick count was 20 against 7 (fc2, 33 rows).  The composed
step tracks the yardstick to within 22%; STEP_ALPHA = 2.  The decode-attention launches' worst row, 2.34 u, is an
fp16 row whose sum cancels; ATTN_TOL = 4.
Every deliberately wrong dec_linear of tests/test_decode_reference_host.py fails by a factor of 68 or more, and
test_decode_parity_gpu fails against builds whose GELU is the tanh form or whose LayerNorm divides the variance by
K - 1.
"""
from __future__ import annotations

import contextlib
from typing import Dict, NamedTuple, Optional

import torch

from tests.attention_reference import _report

X_PLAIN, X_LAYERNORM, X_PARTIAL_SUM = 0, 1, 2
EPI_STORE, EPI_GELU, EPI_RESIDUAL, EPI_LOGITS_F32, EPI_QKV_SCATTER = 0, 1, 2, 3, 4
HD = 64
SCALE = HD ** -0.25
U = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
ALPHA = 3.0
STEP_ALPHA = 2.0
ATTN_TOL = 4.0             # decode-attention launches: row error in units of u
GELU_SLOPE = 1.13          # max |gelu'(x)| = 1.1289 (at x = 0.7518)


def slack(n: int) -> float:
    return 4 + n / 4096


def rnd(x: torch.Tensor, dtype) -> torch.Tensor:
    """x rounded to the 16-bit type, kept in x's type."""
    return x.to(dtype).to(x.dtype)


def ulp(x, dtype):
    """Spacing of the 16-bit type at |x| (at 0: the smallest subnormal)."""
    e = torch.frexp(x.abs().double())[1] - 1
    e = torch.where(x == 0, torch.full_like(e, -1000), e)   # frexp(0) has exponent 0; the clamp below takes over
    return torch.exp2((e - (7 if dtype == torch.bfloat16 else 10)).clamp_min(-24 if dtype == torch.float16 else -133).double())


def acc_stages(K: int) -> int:
    """Rounding stages of dec_linear's fp32 sum of K products and the bias (see the module docstring)."""
    return K // 128 + 10


@contextlib.contextmanager
def _exact_fp32():
    """fp32 matmuls in fp32 (no TF32) while the yardstick runs."""
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev


# ---------------------------------------------------------------------------------------------------------- statements
def embed(emb, pos_emb, tokens, pos: int, dtype) -> torch.Tensor:
    """dec_embed: T(emb[tokens[:, pos]] + pos_emb[pos]) with an fp32 add; a token outside [0, V) reads row 0."""
    tok = tokens[:, pos].long()
    tok = torch.where((tok < 0) | (tok >= emb.shape[0]), torch.zeros_like(tok), tok)
    return (emb[tok].float() + pos_emb[pos].float()).to(dtype)


def layer_norm(x, gamma, beta, eps, dtype, work=torch.float64):
    """(round_T(z), z, mean, rstd): z = (x - mean) rstd g + b with two-pass statistics of each row in `work`."""
    xf = x.to(work)
    mean = xf.mean(dim=-1, keepdim=True)
    c = xf - mean
    rstd = torch.rsqrt((c * c).mean(dim=-1, keepdim=True) + eps)
    z = c * rstd * gamma.to(work) + beta.to(work)
    return rnd(z, dtype), z, mean, rstd


def gelu(x):
    """Exact (erf) GELU."""
    return 0.5 * x * (1.0 + torch.erf(x * 0.7071067811865476))


def linear(x, W, bias, dtype, *, x_mode=X_PLAIN, ln=None, epi=EPI_STORE, res=None, work=torch.float64,
           stages: Optional[int] = None) -> Dict[str, torch.Tensor]:
    """dec_linear of M rows: x (M, K) in T, or (S, M, K) fp32 partials for PARTIAL_SUM; W (N, K) in T; bias (N,) fp32 or
    None; ln = (gamma, beta, eps); res (M, N) in T.  Returns in `work`: "out" (for QKV_SCATTER the [q | k | v] row),
    "inner" (round_T(acc + round_T(bias)), the GELU / RESIDUAL input), "x" (the rounded input row) and, in fp64,
    "allow": the kernel's fp32 allowance E (plus the LayerNorm flips) per output element.  stages: the rounding stages
    of the kernel's sum (default dec_linear's, acc_stages(K))."""
    with _exact_fp32():
        Wt = W.to(work)
        z = None
        if x_mode == X_PARTIAL_SUM:
            s = x[0].to(work)
            for p in x[1:]:
                s = s + p.to(work)
            xin = rnd(s, dtype)
        elif x_mode == X_LAYERNORM:
            xin, z, mean, rstd = layer_norm(x, ln[0], ln[1], ln[2], dtype, work)
        else:
            xin = x.to(work)
        acc = xin @ Wt.t()
        rb = torch.zeros(W.shape[0], dtype=work, device=W.device) if bias is None or epi == EPI_LOGITS_F32 else rnd(bias.to(work), dtype)
        pre = acc + rb
        inner = rnd(pre, dtype)
        if epi == EPI_GELU:
            pre_out = gelu(inner)
        elif epi == EPI_RESIDUAL:
            pre_out = res.to(work) + inner
        else:
            pre_out = pre
        out = rnd(pre_out, dtype)
        r = {"out": out, "inner": inner, "pre": pre, "pre_out": pre_out, "x": xin}
        if work == torch.float64:
            Wa = Wt.abs().t()
            flip = None
            if z is not None:           # normalised inputs whose rounding the fp32 statistics can flip
                g, b = ln[0].double(), ln[1].double()
                d = 2.0 ** -20 * (((x.double() - mean).abs() + mean.abs()) * rstd * g.abs() + b.abs())
                flip = rnd(z - d, dtype) != rnd(z + d, dtype)
            elif x_mode == X_PARTIAL_SUM:   # summed inputs whose rounding the fp32 sum of the partials can flip
                d = (len(x) + 1) * 2.0 ** -24 * sum(p.double().abs() for p in x)
                flip = rnd(s - d, dtype) != rnd(s + d, dtype)
            in_allow = torch.zeros_like(acc) if flip is None else (flip * ulp(xin, dtype)) @ Wa
            r["in_allow"] = in_allow
            r["allow"] = (stages or acc_stages(W.shape[1])) * 2.0 ** -23 * (xin.abs() @ Wa + rb.abs()) + in_allow
        return r


def dec_scores_ref(q, kc, dtype, scale):
    """Per (n, h, key): round_T(sum_c round_T(q_c s) round_T(k_c s)) in fp64, and sum_c |q_c s k_c s| (the scale of the
    kernel's fp32 summation error).  q (n, H, 64), kc (n, keys, H, 64)."""
    qs = (q.float() * scale).to(dtype).double()
    ks = (kc.float() * scale).to(dtype).double()
    return rnd(torch.einsum("nhc,njhc->nhj", qs, ks), dtype), torch.einsum("nhc,njhc->nhj", qs.abs(), ks.abs())


def dec_out_ref(scores, vc, dtype):
    """softmax of the rounded scores (n, H, keys), P rounded to T, then sum_j p_j v_j in fp64 -> (n, H, 64)."""
    p = rnd(torch.softmax(scores.double(), dim=-1), dtype)
    return torch.einsum("nhj,njhc->nhc", p, vc.double())


def attention(q, kc, vc, dtype, work=torch.float64):
    """Decode attention of n single queries: q (n, d) in T, kc / vc (n, keys, d) in T -> the unrounded output (n, d) in
    `work` (the fp32 partial sums of the kernels, added up)."""
    n, keys, d = kc.shape
    H = d // HD
    qh, kh, vh = q.view(n, H, HD), kc.reshape(n, keys, H, HD), vc.reshape(n, keys, H, HD)
    if work == torch.float64:
        s = dec_scores_ref(qh, kh, dtype, SCALE)[0]
        return dec_out_ref(s, vh, dtype).reshape(n, d)
    with _exact_fp32():
        qs = (qh.float() * SCALE).to(dtype).float()
        ks = (kh.float() * SCALE).to(dtype).float()
        s = rnd(torch.einsum("nhc,njhc->nhj", qs, ks), dtype)
        p = rnd(torch.softmax(s, dim=-1), dtype)
        return torch.einsum("nhj,njhc->nhc", p, vh.float()).reshape(n, d)


def step(w, x0, self_k, self_v, cross_kv, pos: int, dtype, kv_group: int = 1, work=torch.float64):
    """One decoder step of n rows from the embedded input x0 (n, d) in T.  w: the engine's weights (refresh_weights
    layout: per layer wqkv, bqkv, wo, bo, wcq, bcq, wco, bco, w1, b1, w2, b2, ln1, lnc, ln2; emb_t; ln).  self_k / self_v:
    (L, n, >= pos, d) caches holding positions [0, pos); cross_kv: (L, n_clips, T_audio, 2d) with row r reading clip
    r // kv_group.  Returns {"logits": (n, V), "k": [L x (n, d)], "v": [L x (n, d)]} in `work`."""
    n, d = x0.shape
    x = x0
    ks, vs = [], []
    for l, lw in enumerate(w["layers"]):
        qkv = linear(x, lw["wqkv"], lw["bqkv"], dtype, x_mode=X_LAYERNORM, ln=lw["ln1"], work=work)["out"]
        q, k, v = (qkv[:, i * d:(i + 1) * d].to(dtype) for i in range(3))
        ks.append(qkv[:, d:2 * d])
        vs.append(qkv[:, 2 * d:])
        kc = torch.cat([self_k[l][:n, :pos], k[:, None]], dim=1)
        vc = torch.cat([self_v[l][:n, :pos], v[:, None]], dim=1)
        a = attention(q, kc, vc, dtype, work)
        x = linear(a[None], lw["wo"], lw["bo"], dtype, x_mode=X_PARTIAL_SUM, epi=EPI_RESIDUAL, res=x, work=work)["out"].to(dtype)
        cq = linear(x, lw["wcq"], lw["bcq"], dtype, x_mode=X_LAYERNORM, ln=lw["lnc"], work=work)["out"].to(dtype)
        ckv = cross_kv[l].repeat_interleave(kv_group, dim=0)[:n]
        a = attention(cq, ckv[..., :d], ckv[..., d:], dtype, work)
        x = linear(a[None], lw["wco"], lw["bco"], dtype, x_mode=X_PARTIAL_SUM, epi=EPI_RESIDUAL, res=x, work=work)["out"].to(dtype)
        h = linear(x, lw["w1"], lw["b1"], dtype, x_mode=X_LAYERNORM, ln=lw["ln2"], epi=EPI_GELU, work=work)["out"].to(dtype)
        x = linear(h, lw["w2"], lw["b2"], dtype, epi=EPI_RESIDUAL, res=x, work=work)["out"].to(dtype)
    logits = linear(x, w["emb_t"], None, dtype, x_mode=X_LAYERNORM, ln=w["ln"], epi=EPI_LOGITS_F32, work=work)["out"]
    return {"logits": logits, "k": ks, "v": vs}


# ---------------------------------------------------------------------------------------------------------- the rule
class LinearErrors(NamedTuple):
    worst: float        # largest |got - ref| in units of the element's bound (rule 1: <= 1)
    n_diff: int         # elements that differ from the fp64 rounded value where the input flips do not explain it
    emu_diff: int       # the same for the yardstick
    numel: int
    diff_ratio: float   # n_diff / max(emu_diff, 1)


def linear_errors(got, ref, emu, dtype, epi) -> LinearErrors:
    g, r, e = got.double(), ref["out"], emu["out"].double()
    inf = torch.isinf(r)
    assert torch.equal(torch.isinf(g), inf) and bool((g[inf] == r[inf]).all()), "overflow to +-inf differs from the reference"
    assert not torch.isnan(g).any(), "NaN in the result"
    fin = ~inf
    g, r, e = g[fin], r[fin], e[fin]
    allow = ref["allow"][fin]
    inner = ref["inner"][fin].abs()
    tol = ulp(torch.maximum(g.abs(), r.abs()), dtype)
    if epi == EPI_GELU:
        tol = tol + GELU_SLOPE * (ulp(inner * (1 + 2.0 ** -7), dtype) + allow) + 2.0 ** -21 * r.abs()
    elif epi == EPI_RESIDUAL:
        tol = tol + ulp(inner * (1 + 2.0 ** -7), dtype) + allow
    else:
        tol = tol + allow
    diff = (g - r).abs()
    worst = float((diff / tol).max()) if diff.numel() else 0.0
    # differences the inputs' own rounding flips explain: the element's inner value within in_allow of a rounding
    # boundary, or its outer value within fp32 noise of one
    ia, pre, po = ref["in_allow"][fin], ref["pre"][fin], ref["pre_out"][fin]
    explained = (rnd(pre - ia, dtype) != rnd(pre + ia, dtype)) | (rnd(po - 2.0 ** -21 * po.abs(), dtype) != rnd(po + 2.0 ** -21 * po.abs(), dtype))
    n_diff, emu_diff = int(((g != r) & ~explained).sum()), int(((e != r) & ~explained).sum())
    return LinearErrors(worst, n_diff, emu_diff, int(fin.sum()), n_diff / max(emu_diff, 1))


def check_linear(got, ref, emu, dtype, epi, name: str = "") -> LinearErrors:
    """Assert the rule of the module docstring for one dec_linear output (M, N): ref / emu from linear() in fp64 / fp32.
    Elements the reference rounds to +-inf (fp16 overflow) must be the same infinity."""
    r = linear_errors(got, ref, emu, dtype, epi)
    _report(kind="linear", name=name, dtype=str(dtype).removeprefix("torch."), **r._asdict())
    assert r.worst <= 1.0, f"{name}: an element is {r.worst:.3g} x its bound off the fp64 value ({r})"
    assert r.n_diff <= ALPHA * r.emu_diff + slack(r.numel), f"{name}: {r.n_diff} of {r.numel} elements differ (yardstick {r.emu_diff})"
    return r


class RowErrors(NamedTuple):
    worst: float
    mean: float
    emu_worst: float
    emu_mean: float
    worst_ratio: float
    mean_ratio: float


def row_errors(got, ref, emu) -> RowErrors:
    """Relative L2 error per row (the first dimension) of got and of the yardstick against the fp64 reference."""
    ref = ref.double().reshape(ref.shape[0], -1)
    g, e = got.double().reshape(ref.shape), emu.double().reshape(ref.shape)
    norm = ref.norm(dim=1).clamp_min(1e-300)
    eg, ee = (g - ref).norm(dim=1) / norm, (e - ref).norm(dim=1) / norm
    w, m, ew, em = float(eg.max()), float(eg.mean()), float(ee.max()), float(ee.mean())
    return RowErrors(w, m, ew, em, w / max(ew, 1e-300), m / max(em, 1e-300))


def check_rows(got, ref, emu, dtype, name: str = "") -> RowErrors:
    """The composed step's rule: per-row relative L2 of the kernel within STEP_ALPHA x the yardstick's."""
    r = row_errors(got, ref, emu)
    _report(kind="step", name=name, dtype=str(dtype).removeprefix("torch."), **r._asdict())
    assert r.worst <= STEP_ALPHA * r.emu_worst and r.mean <= STEP_ALPHA * r.emu_mean, f"{name}: {r}"
    return r


def check_attention(got, ref, dtype, name: str = "") -> float:
    """A decode-attention launch inside the step (its arithmetic is pinned in test_attention_parity_gpu): the output of
    every (sequence, head) within relative L2 ATTN_TOL x u of the fp64 statement.  Scores and probabilities that round
    the other way move it by a fraction of u, more where the row's sum cancels; a wrong key range, cache or clip moves
    it by a large fraction."""
    n = ref.shape[0]
    g, r = got.double().reshape(n, -1, HD), ref.double().reshape(n, -1, HD)
    err = float(((g - r).norm(dim=-1) / r.norm(dim=-1).clamp_min(1e-300)).max())
    _report(kind="attention", name=name, dtype=str(dtype).removeprefix("torch."), worst_u=err / U[dtype])
    assert err <= ATTN_TOL * U[dtype], f"{name}: worst (sequence, head) error {err / U[dtype]:.3g} u"
    return err
