"""The step reference against plain fp64 torch, and the power of its bounds (no GPU needed).

tests/step_reference.py is what the conv-stem glue, the embedding, the bias column sums and the fused AdamW are held
to, so it is checked on its own: its statements against F.conv1d / F.gelu / F.embedding autograd, dy.sum(0) and
torch.nn.utils.clip_grad_norm_ + torch.optim.AdamW on fp64 parameters, and its rules against deliberately wrong
kernels -- each a plausible bug, emulated in fp32 -- which they must reject in both 16-bit types while they accept the
fp32 yardstick itself.  Each variant's test asserts the smallest failure ratio stated in its table (the rule's value
over its limit, or for bit-for-bit rules the number of differing elements; run with -s to see every ratio).
"""
import math

import pytest
import torch
import torch.nn.functional as F

from tests import step_reference as sr
from tests import training_reference as tr
from tests.decode_reference import rnd

DTYPES = [torch.bfloat16, torch.float16]
DT_ID = {torch.bfloat16: "bf16", torch.float16: "fp16"}
HYPER = dict(lr=1.5e-3, beta1=0.9, beta2=0.98, eps=1e-6, wd=0.1)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# ---------------------------------------------------------------------------------------------------- statements
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_stem_statements_match_fp64_conv_and_gelu_autograd(dtype):
    """im2col_conv1 / cast_conv_weight as conv1, im2col_conv2 as conv2 (k3, s2, p1) at an odd T, col2im + GELU' as the
    gradient through conv2's input and conv1's GELU, gelu_bwd as F.gelu's backward."""
    g = _gen(0)
    B, C, T, d = 2, 5, 37, 16
    T2 = sr.conv2_out_len(T)
    mel = torch.randn(B, C, T, generator=g)
    w1, w2 = torch.randn(d, C, 3, generator=g), torch.randn(d, d, 3, generator=g) / 7
    A1 = sr.im2col_conv1(mel, 3 * C + 8, dtype)
    assert not A1[:, 3 * C:].any()
    want = F.conv1d(mel.to(dtype).double(), w1.to(dtype).double(), padding=1)          # (B, d, T)
    got = A1[:, :3 * C].double() @ sr.cast_conv_weight(w1, dtype).double().t()
    assert float((got - want.permute(0, 2, 1).reshape(B * T, d)).abs().max()) < 1e-12
    pre1 = (torch.randn(B * T, d, generator=g) * 2).to(dtype)
    x = pre1.double().requires_grad_(True)
    h = F.gelu(x)
    h.retain_grad()
    y = F.conv1d(h.view(B, T, d).permute(0, 2, 1), w2.double(), stride=2, padding=1)  # (B, d, T2)
    A2 = sr.im2col_conv2(h.detach().to(dtype), B, T, d)
    got = A2.double() @ sr.cast_conv_weight(w2, torch.float64).t()
    want = F.conv1d(h.detach().to(dtype).double().view(B, T, d).permute(0, 2, 1), w2.double(), stride=2, padding=1)
    assert float((got - want.permute(0, 2, 1).reshape(B * T2, d)).abs().max()) < 1e-12
    dy = torch.randn(B, d, T2, generator=g, dtype=torch.float64)
    y.backward(dy)
    # dA = the im2col matrix's gradient; with T = fp64 the statement is col2im(dA) gelu'(pre1) unrounded
    dA = dy.permute(0, 2, 1).reshape(B * T2, d) @ sr.cast_conv_weight(w2, torch.float64)
    got = sr.col2im_conv2_gelu_bwd(dA, pre1, B, T, T2, d, torch.float64)["out"]
    assert float((got - x.grad).abs().max()) < 1e-12
    assert float((x.grad - h.grad * tr.gelu_grad(x.detach())).abs().max()) < 1e-12     # gelu' is F.gelu's derivative
    # in T: the inner rounding of the tap sum, then the rounded product (gelu'(0) = 1/2, so at pre1 = 0 the unrounded
    # statement is half the tap sum)
    dA16 = dA.to(dtype)
    taps = 2 * sr.col2im_conv2_gelu_bwd(dA16, torch.zeros_like(pre1), B, T, T2, d, torch.float64)["out"]
    xa = pre1.double().requires_grad_(True)
    F.gelu(xa).backward(rnd(taps, dtype))
    assert torch.equal(sr.col2im_conv2_gelu_bwd(dA16, pre1, B, T, T2, d, dtype)["out"], rnd(xa.grad, dtype))
    # the last odd frame's k = 2 tap has no source row (2 t + 1 = T for t = T2 - 1): only its k = 0 tap reaches row T - 2
    assert T % 2 == 1 and 2 * (T2 - 1) + 2 - 1 == T
    dyb = torch.randn(B * T, d, generator=g).to(dtype)
    xb = pre1.double().requires_grad_(True)
    F.gelu(xb).backward(dyb.double())
    assert torch.equal(sr.gelu_bwd(dyb, pre1, dtype)["out"], rnd(xb.grad, dtype))


def test_conv_weight_permutations_round_trip():
    g = _gen(1)
    w = torch.randn(6, 5, 3, generator=g)
    perm = sr.cast_conv_weight(w, torch.float32)
    assert torch.equal(sr.unpermute_conv_wgrad(perm, 6, 5), w)
    out = torch.randn(6, 5, 3, generator=g)
    assert torch.equal(sr.unpermute_conv_wgrad(perm, 6, 5, out=out), out + w)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_embedding_statements_match_fp64_autograd(dtype):
    g = _gen(2)
    B, S, d, V, pad, off = 3, 11, 8, 40, 39, 4
    ids = torch.randint(0, V, (B, S), generator=g)
    ids[0, 3:6] = pad
    ids[:, 7] = 5                                                    # one id in several rows of every sample
    E, P = torch.randn(V, d, generator=g), torch.randn(S + off + 2, d, generator=g)
    Er, Pr = E.double().requires_grad_(True), P.double().requires_grad_(True)
    y = F.embedding(ids, Er, padding_idx=pad) + Pr[off:off + S]
    assert torch.equal(sr.embed_fwd(ids, E, P, off, dtype)["out"], rnd(y.detach().reshape(B * S, d), dtype))
    dx = torch.randn(B * S, d, generator=g).to(dtype)
    y.reshape(B * S, d).backward(dx.double())
    r = sr.embed_bwd(ids, dx, torch.zeros(V, d), torch.zeros(S, d), pad)
    assert float((r["demb"] - Er.grad).abs().max()) < 1e-12 and not r["demb"][pad].any()
    assert float((r["dpos"] - Pr.grad[off:off + S]).abs().max()) < 1e-12
    # the kernel-order restatement is an fp32 sum of the same rows
    r32 = sr.embed_bwd(ids, dx, torch.zeros(V, d), torch.zeros(S, d), pad, work=torch.float32)
    assert float(((r32["demb"] - r["demb"]).abs() - r["allow_demb"]).max()) <= 0
    assert float(((r32["dpos"] - r["dpos"]).abs() - r["allow_dpos"]).max()) <= 0
    # ids outside [0, V): the forward reads row 0, the backward skips them
    bad = ids.clone()
    bad[1, 2], bad[2, 0] = V, -3
    f = sr.embed_fwd(bad, E, P, 0, dtype)["out"].view(B, S, d)
    assert torch.equal(f[1, 2], rnd(E[0].double() + P[2].double(), dtype))
    r2 = sr.embed_bwd(bad, dx, torch.zeros(V, d), None, pad)
    keep = (bad >= 0) & (bad < V) & (bad != pad)
    want = torch.zeros(V, d, dtype=torch.float64).index_add_(0, bad[keep], dx.double().view(B, S, d)[keep])
    assert float((r2["demb"] - want).abs().max()) < 1e-12 and r2["dpos"] is None
    # packed: the dense sums with zeros in the padded rows
    lens = [S, 4, 0]
    rows = torch.cat([b * S + torch.arange(n) for b, n in enumerate(lens)])
    dxp = dx[rows]
    rp = sr.embed_bwd_packed(ids, dxp, torch.zeros(V, d), torch.zeros(S, d), pad, rows, work=torch.float32)
    dense = torch.zeros_like(dx)
    dense[rows] = dxp
    rd = sr.embed_bwd(ids, dense, torch.zeros(V, d), torch.zeros(S, d), pad, work=torch.float32)
    assert torch.equal(rp["demb"], rd["demb"]) and torch.equal(rp["dpos"], rd["dpos"])


def test_colsum_statement_and_stages():
    g = _gen(3)
    dy = torch.randn(300, 24, generator=g).to(torch.bfloat16)
    db0 = torch.randn(24, generator=g)
    r = sr.colsum(dy, db0)
    assert float((r["out"] - (db0.double() + dy.double().sum(0))).abs().max()) < 1e-12
    # the stem's conv1 bias at B = 32 (96000 rows, d = 1024 -> 4 column tiles): 199 row blocks of 483 rows
    assert sr.colsum_stages(96000, 1024, 132) == 61 + 8 + 199 + 1
    assert sr.colsum_stages(100, 384, 132) == 7 + 8 + 2 + 1


def _torch_adamw_steps(params, grads_per_step, max_norm, steps_before=0, **hp):
    """torch's clip_grad_norm_ + AdamW in fp64: the parameters after every step and the returned norms."""
    ps = [p.clone().requires_grad_(True) for p in params]
    opt = torch.optim.AdamW(ps, lr=hp["lr"], betas=(hp["beta1"], hp["beta2"]), eps=hp["eps"], weight_decay=hp["wd"])
    out = []
    for grads in grads_per_step:
        for p, gr in zip(ps, grads):
            p.grad = gr.clone()
        norm = float(torch.nn.utils.clip_grad_norm_(ps, max_norm))
        opt.step()
        out.append(([p.detach().clone() for p in ps], norm))
    return out


def test_optimizer_statement_matches_fp64_clip_and_adamw():
    """Five steps of the statement (prepare + adamw per tensor) against clip_grad_norm_ + AdamW on fp64 parameters,
    clipped and unclipped, with hyperparameters that are fp32 numbers (so f32() changes nothing)."""
    hp = dict(lr=2.0 ** -9, beta1=0.875, beta2=1 - 2.0 ** -6, eps=2.0 ** -20, wd=0.125)
    g = _gen(4)
    shapes = [(33, 7), (5,), (1000,)]
    params = [torch.randn(*s, generator=g, dtype=torch.float64) for s in shapes]
    grads = [[torch.randn(*s, generator=g, dtype=torch.float64) * (3.0 if k % 2 else 0.01) for s in shapes] for k in range(5)]
    want = _torch_adamw_steps(params, grads, 1.0, **hp)
    ps = [p.clone() for p in params]
    ms = [torch.zeros_like(p) for p in params]
    vs = [torch.zeros_like(p) for p in params]
    step = 0.0
    for k, (wp, wnorm) in enumerate(want):
        sq = sr.grad_sqnorm(grads[k], 1.0)["sqnorm"]
        st = sr.prepare(sq, 1.0, 1.0, hp["beta1"], hp["beta2"], step)
        assert abs(st["norm"] - wnorm) <= 1e-14 * wnorm
        assert (st["coef"] < 1.0) == (k % 2 == 1)                     # the large-gradient steps clip
        step = st["step"]
        for i in range(len(ps)):
            r = sr.adamw(ps[i], grads[k][i], ms[i], vs[i], st, **hp)
            ps[i], ms[i], vs[i] = r["p"], r["m"], r["v"]
            assert float((ps[i] - wp[i]).abs().max()) <= 1e-14, (k, i)
    # the amp form: gradients scaled by S, found_inf from outside
    S = 1024.0
    sq = sr.grad_sqnorm([gr * S for gr in grads[0]], 1.0)["sqnorm"]
    st = sr.prepare(sq, 1.0, 1.0, hp["beta1"], hp["beta2"], 0.0, loss_scale=S)
    assert abs(st["norm"] - want[0][1]) <= 1e-14 * want[0][1] and abs(st["coef"] * S - 1.0) < 1e-15
    skip = sr.prepare(sq, 1.0, 1.0, hp["beta1"], hp["beta2"], 7.0, loss_scale=S, found_inf=True)
    assert skip["skip"] == 1.0 and skip["step"] == 7.0 and abs(skip["norm"] - want[0][1]) <= 1e-14 * want[0][1]
    inf = sr.prepare(float("inf"), 1.0, 1.0, hp["beta1"], hp["beta2"], 7.0)
    assert inf["skip"] == 1.0 and inf["step"] == 7.0 and inf["norm"] == float("inf")


def test_bias_correction_allowance_covers_fp32_powf():
    """The bias corrections' relative allowance holds for numpy's fp32 pow at t = 1, 2, 300 and 10^6, and the
    amplification by b^t / (1 - b^t) is what makes t = 1 the widest."""
    import numpy as np
    for b in (0.9, 0.98):
        bf = np.float32(b)
        for t in (1.0, 2.0, 300.0, 1e6):
            got = float(np.float32(1.0) - np.power(bf, np.float32(t)))
            want = 1.0 - float(bf) ** t
            assert abs(got - want) <= sr._pow_rel(float(bf), t) * want, (b, t)
    assert sr._pow_rel(sr.f32(0.98), 1) > 100 * sr._pow_rel(sr.f32(0.98), 300)


# ---------------------------------------------------------------------------------------------------- the rule's power
def _stem_case(dtype, seed=5, B=2, T=301, d=64):
    g = _gen(seed)
    T2 = sr.conv2_out_len(T)
    dA = torch.randn(B * T2, 3 * d, generator=g).to(dtype)
    pre1 = (torch.randn(B * T, d, generator=g) * 1.5).to(dtype)
    return dA, pre1, B, T, T2, d


def _tanh_gelu_grad(x):
    x = x.float().clone().requires_grad_(True)
    F.gelu(x, approximate="tanh").backward(torch.ones_like(x))
    return x.grad


def _wrong_col2im(wrong, dA, pre1, B, T, T2, d, dtype):
    cols = dA.float().view(B, T2, 3, d)
    if wrong == "col2im taps k = 0 and k = 2 swapped":
        cols = cols[:, :, [2, 1, 0]]
    gs = torch.zeros(B, T + 2, d)
    for k in range(3):
        gs[:, k:k + 2 * T2:2] += cols[:, :, k]
    gs = gs[:, 1:T + 1].reshape(B * T, d)
    gp = tr.gelu_grad(pre1.float())
    if wrong == "col2im without the inner T()":
        return rnd(gs * gp, dtype)
    if wrong == "tanh GELU'":
        gp = _tanh_gelu_grad(pre1)
    return rnd(rnd(gs, dtype) * gp, dtype)


# variant: the smallest failure ratio its test asserts (measured smallest over both types in the comment)
T16_WRONG = {"col2im taps k = 0 and k = 2 swapped": 500,     # 1.1e3 (bf16)
             "col2im without the inner T()": 50,               # 114 (fp16)
             "tanh GELU'": 300,                                # 740 (bf16)
             "positional row off by one": 1000}                # 3.8e3 (bf16)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("wrong", list(T16_WRONG))
def test_rule_rejects_wrong_rounded_kernels(wrong, dtype):
    if wrong == "positional row off by one":
        g = _gen(6)
        T, d = 1500, 64
        x = torch.randn(2 * T, d, generator=g).to(dtype)
        pos = torch.randn(T, d, generator=g)
        ref, emu = sr.add_pos(x, pos, T, dtype), sr.add_pos(x, pos, T, dtype, work=torch.float32)
        got = rnd(x.float() + pos[(torch.arange(2 * T) + 1) % T], dtype)
    else:
        case = _stem_case(dtype)
        ref = sr.col2im_conv2_gelu_bwd(*case, dtype)
        emu = sr.col2im_conv2_gelu_bwd(*case, dtype, work=torch.float32)
        got = _wrong_col2im(wrong, *case, dtype)
    tr.check16(tr.errors16(emu["out"], ref, emu, dtype), dtype, name="yardstick")
    ratio = tr.fail_ratio16(tr.errors16(got, ref, emu, dtype))
    print(f"{wrong} {DT_ID[dtype]}: fails by {ratio:.3g}")
    assert ratio > T16_WRONG[wrong], f"{wrong}: fails by only {ratio:.3g}"


def _emb_case(dtype):
    g = _gen(7)
    B, S, d, V, pad = 4, 448, 64, 300, 299
    ids = torch.randint(0, V, (B, S), generator=g)
    ids.view(-1)[130::7] = 17                                        # a hot id past the first 128-row batch
    # magnitudes over 2^-10 .. 2^10: fp32 sums of a few 16-bit values are exact, so only a wide range makes them round
    dx = (torch.randn(B * S, d, generator=g) * torch.exp2(torch.randint(-10, 11, (B * S, d), generator=g).float())).to(dtype)
    demb0 = torch.randn(V, d, generator=g)                           # the tied logits' wgrad already accumulated
    return ids, dx, demb0, pad


# variant: (output, smallest failure ratio); "bit" rules count the elements that differ from the kernel-order
# restatement (the rule allows none), the others are check32's ratio against fp64
SUM_WRONG = {"an embedding sum with one row twice": ("check32", 1e6),            # 2.0e6
             "out += x per row instead of out + acc": ("bit", 1000),            # 3.5e3 of 19200 elements (bf16)
             "embedding rows in reverse order": ("bit", 500),                   # 1.3e3 (bf16)
             "a colsum that drops one row per lane": ("check32", 5e4)}          # 1.7e5 (fp16)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("wrong", list(SUM_WRONG))
def test_rule_rejects_wrong_sums(wrong, dtype):
    kind, limit = SUM_WRONG[wrong]
    if "colsum" in wrong:
        g = _gen(8)
        M, N = 3000, 384
        dy = torch.randn(M, N, generator=g).to(dtype)
        db0 = torch.randn(N, generator=g)
        ref, emu = sr.colsum(dy, db0), sr.colsum(dy, db0, work=torch.float32)
        tr.check32(tr.errors32(emu["out"], ref["out"], emu["out"], ref["allow"]), name="yardstick")
        blocks = max(1, min(-(-M // 64), 132 * 6 // 2 + 1))
        rpb = -(-M // blocks)
        keep = torch.ones(M, dtype=torch.bool)
        for r0 in range(0, M, rpb):                                  # each of the 8 lanes loses its last row
            r1 = min(M, r0 + rpb)
            for lane in range(8):
                rows = list(range(r0 + lane, r1, 8))
                if rows:
                    keep[rows[-1]] = False
        got = db0 + dy[keep].float().sum(0)
        ratio = tr.fail_ratio32(tr.errors32(got, ref["out"], emu["out"], ref["allow"]))
    else:
        ids, dx, demb0, pad = _emb_case(dtype)
        ref = sr.embed_bwd(ids, dx, demb0, None, pad)
        emu = sr.embed_bwd(ids, dx, demb0, None, pad, work=torch.float32)
        tr.check32(tr.errors32(emu["demb"], ref["demb"], emu["demb"], ref["allow_demb"]), name="yardstick")
        flat = ids.reshape(-1)
        x = dx.float()
        if wrong == "an embedding sum with one row twice":
            twice = torch.cat([x, x[140:141]])
            got = sr.embed_bwd(torch.cat([flat, flat[140:141]])[None], twice.to(dtype), demb0, None, pad, work=torch.float32)["demb"]
            ratio = tr.fail_ratio32(tr.errors32(got, ref["demb"], emu["demb"], ref["allow_demb"]))
        else:
            if wrong == "embedding rows in reverse order":
                got = sr.embed_bwd(flat.flip(0)[None], dx.flip(0), demb0, None, pad, work=torch.float32)["demb"]
            else:
                got = demb0.clone()
                for r in range(flat.numel()):
                    if flat[r] != pad:
                        got[flat[r]] += x[r]
            ratio = float((got != emu["demb"]).sum())
            assert tr.fail_ratio32(tr.errors32(got, ref["demb"], emu["demb"], ref["allow_demb"])) <= 1.0   # only bit-exactness sees it
    print(f"{wrong} {DT_ID[dtype]}: fails by {ratio:.3g}")
    assert ratio > limit, f"{wrong}: fails by only {ratio:.3g}"


def _opt_case(seed=9, n=4096):
    g = _gen(seed)
    p = 0.02 * torch.randn(n, generator=g)                           # a weight at the model's init scale
    grad = 1e-4 * torch.randn(n, generator=g)                        # ||g|| = 6.4e-3: the clip's 1e-6 is 1.6e-4 of it
    m = 1e-4 * torch.randn(n, generator=g)
    v = (1e-4 * torch.randn(n, generator=g)) ** 2
    return p, grad, m, v


def _wrong_adamw(wrong, p, grad, m, v, max_norm, step, dtype):
    """The fp32 kernel with one deliberate error: (p', m', v', shadow)."""
    lr, b1, b2, eps, wd = (sr.f32(HYPER[k]) for k in ("lr", "beta1", "beta2", "eps", "wd"))
    norm = float(grad.double().norm())
    den = norm if wrong == "the clip without +1e-6" else norm + sr.f32(1e-6)
    coef = min(1.0, max_norm / den)
    t = step + 1
    bc1 = 1 - b1 ** t
    bc2 = 1 - b2 ** t if wrong == "1-b2^t in place of its square root" else math.sqrt(1 - b2 ** t)
    gi = grad * coef
    m1 = b1 * m + (1 - b1) * gi
    v1 = b2 * v + (1 - b2) * gi * gi
    if wrong == "AdamW with eps inside the sqrt":
        den = torch.sqrt(v1 / bc2 ** 2 + eps)
    else:
        den = torch.sqrt(v1) / bc2 + eps
    upd = (lr / bc1) * (m1 / den)
    p1 = (p - upd) * (1 - lr * wd) if wrong == "weight decay after the Adam step" else p * (1 - lr * wd) - upd
    shadow = (p if wrong == "shadows cast from the old master" else p1).to(dtype)
    return p1, m1, v1, shadow


# variant: the smallest failure ratio its test asserts (check32's ratio on p', m', v'; for the shadow the number of
# elements that are not T(p'))
OPT_WRONG = {"AdamW with eps inside the sqrt": 5e5,                 # 1.1e6
             "1-b2^t in place of its square root": 500,             # 1.2e3 (at t = 300)
             "weight decay after the Adam step": 80,                # 167
             "the clip without +1e-6": 20,                          # 48
             "shadows cast from the old master": 2000}              # 4.0e3 of 4096 (bf16)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("wrong", list(OPT_WRONG))
def test_rule_rejects_wrong_adamw(wrong, dtype):
    p, grad, m, v = _opt_case()
    max_norm, step = 2e-3, 299.0
    sq = sr.grad_sqnorm([grad], 1.0)
    st = sr.prepare(sq["sqnorm"], 1.0, max_norm, HYPER["beta1"], HYPER["beta2"], step, sqnorm_allow=sq["allow"])
    ref = sr.adamw(p, grad, m, v, st, **HYPER)
    st32 = {k: sr.f32(x) for k, x in st.items()}
    emu = sr.adamw(p, grad, m, v, st32, **HYPER, work=torch.float32)
    for k in ("p", "m", "v"):
        tr.check32(tr.errors32(emu[k], ref[k], emu[k], ref["allow_" + k]), name=f"yardstick {k}")
    p1, m1, v1, shadow = _wrong_adamw(wrong, p, grad, m, v, max_norm, step, dtype)
    if wrong == "shadows cast from the old master":
        ratio = float((shadow != p1.to(dtype)).sum())
    else:
        ratio = max(tr.fail_ratio32(tr.errors32(got, ref[k], emu[k], ref["allow_" + k])) for got, k in ((p1, "p"), (m1, "m"), (v1, "v")))
    print(f"{wrong} {DT_ID[dtype]}: fails by {ratio:.3g}")
    assert ratio > OPT_WRONG[wrong], f"{wrong}: fails by only {ratio:.3g}"
