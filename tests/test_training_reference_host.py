"""The training reference against plain fp64 torch, and the power of its tolerance rule (no GPU needed).

tests/training_reference.py is what the training GEMM, LayerNorm and cross-entropy kernels are held to, so it is
checked on its own: its statements against F.linear, F.gelu, F.layer_norm and F.cross_entropy (and their autograd) in
fp64, the GEMM epilogue's GELU against erf-GELU, and its rule against deliberately wrong kernels -- each a plausible
bug, emulated in fp32 -- which it must reject in both 16-bit types while it accepts the yardstick itself.  Each
variant's test asserts the smallest failure ratio stated in GEMM_WRONG, LN_WRONG or CE_WRONG (the rule's value over
its limit; run with -s to see every ratio).
"""
import pytest
import torch
import torch.nn.functional as F

from tests import training_reference as tr
from tests.decode_reference import rnd

DTYPES = [torch.bfloat16, torch.float16]
DT_ID = {torch.bfloat16: "bf16", torch.float16: "fp16"}
V, LD, IGNORE = 51865, 51968, 51863


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# ---------------------------------------------------------------------------------------------------- statements
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_gemm_statement_matches_fp64_linear_and_gelu_autograd(dtype):
    g = _gen(0)
    M, N, K = 40, 200, 3 * 64 + 25
    A = torch.randn(M, K, generator=g).to(dtype)
    B = (torch.randn(N, K, generator=g) / K ** 0.5).to(dtype)
    bias = torch.randn(N, generator=g)
    aux = torch.randn(M, N, generator=g).to(dtype)
    h = rnd(F.linear(A.double(), B.double(), bias.to(dtype).double()), dtype)
    assert torch.equal(tr.gemm(A, B, tr.EPI_BF16, dtype, bias=bias)["out"], h)
    r = tr.gemm(A, B, tr.EPI_GELU, dtype, bias=bias)
    assert torch.equal(r["out"], h) and torch.equal(r["out2"], rnd(F.gelu(h), dtype))
    assert torch.equal(tr.gemm(A, B, tr.EPI_RESIDUAL, dtype, bias=bias, aux=aux)["out"], rnd(aux.double() + h, dtype))
    x = aux.double().requires_grad_(True)
    acc = rnd(A.double() @ B.double().t(), dtype)
    F.gelu(x).backward(acc)
    assert torch.equal(tr.gemm(A, B, tr.EPI_GELU_BWD, dtype, aux=aux)["out"], rnd(x.grad, dtype))
    f32 = tr.gemm(A, B, tr.EPI_F32, dtype, bias=bias)["out"]
    assert float((f32 - F.linear(A.double(), B.double(), bias.double())).abs().max()) < 1e-12
    out0 = torch.randn(M, N, generator=g)
    for split in (1, 2, 3):
        got = tr.gemm(A, B, tr.EPI_F32_ATOMIC_ADD, dtype, out0=out0, split_k=split)["out"]
        assert float((got - (out0.double() + A.double() @ B.double().t())).abs().max()) < 1e-12
    # split ranges: whole k-blocks, the last split short, never an empty split
    assert tr.split_ranges(K, 3) == [(0, 128), (128, 217)]
    assert tr.split_ranges(51865, 7) == [(s * 116 * 64, min((s + 1) * 116 * 64, 51865)) for s in range(7)]
    assert tr.split_ranges(100, 8) == [(0, 64), (64, 100)]


def test_layernorm_statement_matches_fp64_autograd():
    g = _gen(1)
    rows, d = 33, 384
    dt = torch.float16
    x = (torch.randn(rows, d, generator=g) * 3 + 20).to(dt)
    w, b = torch.randn(d, generator=g), torch.randn(d, generator=g)
    dy, dres = torch.randn(rows, d, generator=g).to(dt), torch.randn(rows, d, generator=g).to(dt)
    xr = x.double().requires_grad_(True)
    wr, br = w.double().requires_grad_(True), b.double().requires_grad_(True)
    y = F.layer_norm(xr, (d,), wr, br, 1e-5)
    f = tr.layernorm_fwd(x, w, b, 1e-5, dt)
    assert torch.equal(f["out"], rnd(y.detach(), dt))
    y.backward(dy.double())
    r = tr.layernorm_bwd(dy, x, w, 1e-5, dt)
    assert torch.equal(r["out"], rnd(xr.grad, dt))
    assert float((r["dw"] - wr.grad).abs().max()) < 1e-9 and float((r["db"] - br.grad).abs().max()) < 1e-9
    r = tr.layernorm_bwd(dy, x, w, 1e-5, dt, dres=dres)
    assert torch.equal(r["out"], rnd(dres.double() + rnd(xr.grad, dt), dt))


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_cross_entropy_statement_matches_fp64_autograd(dtype):
    g = _gen(2)
    rows = 12
    logits = torch.full((rows, LD), float("nan")).to(dtype)          # padding columns: never read
    logits[:, :V] = (torch.randn(rows, V, generator=g) * 3).to(dtype)
    y = torch.randint(0, V, (rows,), generator=g)
    y[2], y[5], y[7] = IGNORE, V - 1, 0
    ref = tr.ce_fwd(logits, y, V, IGNORE)
    x = logits[:, :V].double().requires_grad_(True)
    loss = F.cross_entropy(x, y, ignore_index=IGNORE)
    assert abs(float(ref["loss"]) - float(loss.detach())) < 1e-12 and int(ref["count"]) == rows - 1 and int(ref["bad"]) == 0
    (loss * 1024.0).backward()
    d = tr.ce_bwd(logits, y, V, IGNORE, 1024.0, ref["count"], dtype, lse=ref["lse"])["out"]
    want = rnd(x.grad, dtype)
    assert float(((d - want).abs() / tr.ulp(want, dtype)).max()) <= 1.0     # a tie may round either way
    assert bool((d[2] == 0).all())
    y2 = y.clone()
    y2[3], y2[4] = V, -2                 # out of range: not counted, counted as bad, zero gradient
    r2 = tr.ce_fwd(logits, y2, V, IGNORE)
    assert int(r2["count"]) == rows - 3 and int(r2["bad"]) == 2 and float(r2["lse"][3]) == 0.0
    assert bool((tr.ce_bwd(logits, y2, V, IGNORE, 1.0, r2["count"], dtype)["out"][3:5] == 0).all())


def test_gelu_approx_bounds_the_epilogue_gelu():
    x = torch.linspace(-10, 10, 2_000_001, dtype=torch.float64)
    e_gelu = float((tr.gelu_as(x) - tr.gelu(x)).abs().max())
    e_grad = float((tr.gelu_grad_as(x) - tr.gelu_grad(x)).abs().max())
    print(f"A&S GELU error {e_gelu:.3g}, GELU' error {e_grad:.3g} (GELU_APPROX {tr.GELU_APPROX:.3g})")
    assert e_gelu <= tr.GELU_APPROX and e_grad <= tr.GELU_APPROX
    assert e_gelu > 0.5 * tr.GELU_APPROX            # the constant is tight, not a guess
    tanh = float((F.gelu(x, approximate="tanh") - tr.gelu(x)).abs().max())
    assert tanh > 1000 * tr.GELU_APPROX             # a tanh GELU stays 3 orders outside the band


# ---------------------------------------------------------------------------------------------------- the rule's power
def _acc32(A, B):
    return A.float() @ B.float().t()


def _gemm_case(wrong, dtype, d=768, M=64, seed=0):
    g = _gen(seed)
    N, K, epi, split = {"tanh GELU": (4 * d, d, tr.EPI_GELU, 1),
                        "bias not rounded": (3 * d, d, tr.EPI_BF16, 1),
                        "bias rounded twice": (3 * d, d, tr.EPI_BF16, 1),
                        "GELU' of the unrounded acc": (4 * d, d, tr.EPI_GELU_BWD, 1),
                        "residual added before the inner rounding": (d, 4 * d, tr.EPI_RESIDUAL, 1),
                        "bias added per split": (d, 4 * d, tr.EPI_F32, 3),
                        "last k-block dropped": (d, V, tr.EPI_BF16, 1),
                        "an 8-column group of the last box left at zero": (d, d, tr.EPI_BF16, 1)}[wrong]
    if K == V:
        M = 16
    A = torch.randn(M, K, generator=g).to(dtype)
    B = (torch.randn(N, K, generator=g) / K ** 0.5).to(dtype)
    bias = None if epi == tr.EPI_GELU_BWD else 0.5 * torch.randn(N, generator=g)
    aux = (2 * torch.randn(M, N, generator=g)).to(dtype)
    return A, B, bias, aux, epi, split


def _wrong_gemm(wrong, A, B, bias, aux, dtype, split):
    """An fp32 GEMM launch with one deliberate error: (key of the output that shows it, the output)."""
    acc = _acc32(A, B)
    rb = None if bias is None else rnd(bias.float(), dtype)
    if wrong == "tanh GELU":
        return "out2", rnd(F.gelu(rnd(acc + rb, dtype), approximate="tanh"), dtype)
    if wrong == "bias not rounded":
        return "out", rnd(acc + bias.float(), dtype)
    if wrong == "bias rounded twice":
        return "out", rnd(rnd(acc, dtype) + rb, dtype)
    if wrong == "GELU' of the unrounded acc":
        return "out", rnd(acc * tr.gelu_grad(aux.float()), dtype)
    if wrong == "residual added before the inner rounding":
        return "out", rnd(aux.float() + acc + rb, dtype)
    if wrong == "bias added per split":
        out = None
        for k0, k1 in tr.split_ranges(A.shape[1], split):
            p = A[:, k0:k1].float() @ B[:, k0:k1].float().t() + bias.float()
            out = p if out is None else out + p
        return "out", out
    if wrong == "last k-block dropped":
        k1 = (A.shape[1] - 1) // tr.BK * tr.BK
        return "out", rnd(A[:, :k1].float() @ B[:, :k1].float().t() + rb, dtype)
    out = rnd(acc + rb, dtype)
    n0 = (B.shape[0] - 1) // 64 * 64
    out[:, n0 + 8:n0 + 16] = 0
    return "out", out


# variant: the smallest failure ratio its test asserts (measured smallest over both types in the comment)
GEMM_WRONG = {"tanh GELU": 7,                                         # 14.3 (fp16)
              "bias not rounded": 3,                                  # 6.55 (fp16)
              "bias rounded twice": 4,                                # 9.58 (fp16)
              "GELU' of the unrounded acc": 3,                        # 6.3 (fp16)
              "residual added before the inner rounding": 9,          # 19.9 (fp16)
              "bias added per split": 4e4,                            # 9.0e4 (fp16)
              "last k-block dropped": 12,                             # 26 (fp16, K = 51865: 25 of its columns)
              "an 8-column group of the last box left at zero": 100}  # 247 (bf16)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("wrong", list(GEMM_WRONG))
def test_rule_rejects_wrong_gemm(wrong, dtype):
    A, B, bias, aux, epi, split = _gemm_case(wrong, dtype)
    kw = dict(bias=bias, aux=aux)
    ref = tr.gemm(A, B, epi, dtype, **kw)
    emu = tr.gemm(A, B, epi, dtype, work=torch.float32, **kw)
    key, got = _wrong_gemm(wrong, A, B, bias, aux, dtype, split)
    if epi == tr.EPI_F32:
        tr.check32(tr.errors32(emu["out"], ref["out"], emu["out"], ref["allow"]), name="yardstick")
        ratio = tr.fail_ratio32(tr.errors32(got, ref["out"], emu["out"], ref["allow"]))
    else:
        for k in ("out", "out2") if epi == tr.EPI_GELU else ("out",):
            tr.check16(tr.errors16(emu[k], ref, emu, dtype, key=k), dtype, name="yardstick")
        r = tr.errors16(got, ref, emu, dtype, key=key)
        ratio = tr.fail_ratio16(r)
    print(f"{wrong} {DT_ID[dtype]}: fails by {ratio:.3g}")
    assert ratio > GEMM_WRONG[wrong], f"{wrong}: fails by only {ratio:.3g}"


LN_WRONG = {"variance over d - 1": 150,             # 314 (bf16, d = 1280)
            "eps outside the sqrt": 400,            # 877 (bf16, d = 384)
            "dx without the inner rounding": 35}    # 77 (fp16, d = 384)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("d", [384, 1280])
@pytest.mark.parametrize("wrong", list(LN_WRONG))
def test_rule_rejects_wrong_layernorm(wrong, d, dtype):
    g = _gen(d)
    rows = 64
    x = (torch.randn(rows, d, generator=g) * 0.05).to(dtype)     # a small variance: eps matters
    w, b = 1 + 0.2 * torch.randn(d, generator=g), 0.2 * torch.randn(d, generator=g)
    eps = 1e-5
    if wrong == "dx without the inner rounding":
        dy, dres = torch.randn(rows, d, generator=g).to(dtype), torch.randn(rows, d, generator=g).to(dtype)
        ref = tr.layernorm_bwd(dy, x, w, eps, dtype, dres=dres)
        emu = tr.layernorm_bwd(dy, x, w, eps, dtype, dres=dres, work=torch.float32)
        xf = x.float()
        mean = xf.mean(-1, keepdim=True)
        rstd = torch.rsqrt((xf - mean).square().mean(-1, keepdim=True) + eps)
        xhat = (xf - mean) * rstd
        gw = dy.float() * w
        dxln = rstd * (gw - gw.mean(-1, keepdim=True) - xhat * (gw * xhat).mean(-1, keepdim=True))
        got = rnd(dres.float() + dxln, dtype)
    else:
        ref = tr.layernorm_fwd(x, w, b, eps, dtype)
        emu = tr.layernorm_fwd(x, w, b, eps, dtype, work=torch.float32)
        xf = x.float()
        mean = xf.mean(-1, keepdim=True)
        c = xf - mean
        if wrong == "variance over d - 1":
            rstd = torch.rsqrt(c.square().sum(-1, keepdim=True) / (d - 1) + eps)
        else:
            rstd = 1 / (c.square().mean(-1, keepdim=True).sqrt() + eps)
        got = rnd(c * rstd * w + b, dtype)
    tr.check16(tr.errors16(emu["out"], ref, emu, dtype), dtype, name="yardstick")
    ratio = tr.fail_ratio16(tr.errors16(got, ref, emu, dtype))
    print(f"{wrong} {DT_ID[dtype]} d={d}: fails by {ratio:.3g}")
    assert ratio > LN_WRONG[wrong], f"{wrong}: fails by only {ratio:.3g}"


CE_WRONG = {"lse without the tail column": 1e4,     # 2.8e4
            "ignored rows counted": 1e4,            # 3.8e4
            "no one-hot at the tail column": 130,   # 273 (bf16)
            "g over rows, not count": 1e3}          # 3.7e3


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("wrong", list(CE_WRONG))
def test_rule_rejects_wrong_cross_entropy(wrong, dtype):
    g = _gen(5)
    rows = 16
    logits = (torch.randn(rows, V, generator=g) * 2).to(dtype)
    y = torch.randint(0, V, (rows,), generator=g)
    y[3], y[9] = IGNORE, V - 1
    logits[9, V - 1] = 12.0          # the tail target holds much of its row's mass
    grad_out = 1024.0
    ref = tr.ce_fwd(logits, y, V, IGNORE)
    emu = tr.ce_fwd(logits, y, V, IGNORE, work=torch.float32)
    dref = tr.ce_bwd(logits, y, V, IGNORE, grad_out, ref["count"], dtype, lse=ref["lse"], xmax=ref["xmax"])
    demu = tr.ce_bwd(logits, y, V, IGNORE, grad_out, emu["count"], dtype, lse=emu["lse"], work=torch.float32)
    tr.check_lse(emu["lse"].float(), emu["loss"], ref, name="yardstick")
    tr.check16(tr.errors16(demu["out"], dref, demu, dtype), dtype, name="yardstick")
    x = logits.float()
    cnt = tr.counted_rows(y, V, IGNORE)
    lse, count = emu["lse"], emu["count"]
    if wrong == "lse without the tail column":
        lse = torch.where(cnt, torch.logsumexp(x[:, :V - 1], dim=-1), torch.zeros_like(lse))
    if wrong == "ignored rows counted":
        count = torch.tensor(float(rows))
    loss = (lse - x.gather(1, y.clamp(0, V - 1)[:, None])[:, 0])[cnt].sum() / count
    gsc = grad_out / (rows if wrong == "g over rows, not count" else count)
    p = torch.exp(x - lse[:, None])
    onehot = torch.zeros_like(x)
    onehot.scatter_(1, y.clamp(0, V - 1)[:, None], 1.0)
    if wrong == "no one-hot at the tail column":
        onehot[:, V - 1] = 0
    d = torch.where(cnt[:, None], rnd(gsc * (p - onehot), dtype), torch.zeros_like(p))
    lse_ratio = max(tr.lse_error(lse, ref), abs(float(loss) - float(ref["loss"])) / tr.loss_bound(ref))
    ratio = max(lse_ratio, tr.fail_ratio16(tr.errors16(d, dref, demu, dtype)))
    print(f"{wrong} {DT_ID[dtype]}: fails by {ratio:.3g}")
    assert ratio > CE_WRONG[wrong], f"{wrong}: fails by only {ratio:.3g}"
