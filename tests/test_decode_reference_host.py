"""The decode-step reference against plain fp64 torch, and the power of its tolerance rule (no GPU needed).

tests/decode_reference.py is what the decoder-step kernels are held to, so it is checked on its own: its statements
against F.layer_norm, F.gelu, matmul and softmax in fp64, and its rule against deliberately wrong dec_linear variants
-- each a plausible kernel bug, emulated in fp32 at production widths -- which it must reject while it accepts the
yardstick itself.

Each variant's failure ratio (rule 1: worst error over its bound; rule 2: unexplained differing elements over
ALPHA x the yardstick's + SLACK; the larger of the two) over d = 384 .. 1280, the smallest / largest (run with -s to
see every case):

    variant                                  type   smallest / largest
    tanh GELU                                bf16     68.3 /  201
                                             fp16      121 /  190
    bias not rounded                         bf16      282 /  405
                                             fp16      119 /  230
    residual rounded once                    bf16      120 /  294
                                             fp16     75.7 /  211
    LayerNorm variance over K-1              bf16      256 /  761
                                             fp16      190 /  359
    LayerNorm statistics over K-32 columns   bf16     1110 / 1480
                                             fp16      946 / 1870
    last 32 k columns dropped                bf16      503 / 1190
                                             fp16      536 / 1900
    logits not rounded                       bf16     2100 / 3250
                                             fp16     2150 / 3180
    partial sums rounded per split           bf16      175 /  367   (8 partials; with one it is the correct result)
                                             fp16      109 /  209

Every variant is detectable in both types at every width.
"""
import pytest
import torch
import torch.nn.functional as F

from tests import decode_reference as dr

DTYPES = [torch.bfloat16, torch.float16]
DT_ID = {torch.bfloat16: "bf16", torch.float16: "fp16"}
WIDTHS = [384, 512, 768, 1024, 1280]
V = 51864


# ---------------------------------------------------------------------------------------------------- statements
def test_layer_norm_gelu_and_linear_match_fp64_torch():
    g = torch.Generator().manual_seed(0)
    M, K, N = 5, 768, 300
    x = (torch.randn(M, K, generator=g, dtype=torch.float64) * 3 + 50).to(torch.bfloat16)
    gam = torch.randn(K, generator=g)
    bet = torch.randn(K, generator=g)
    W = torch.randn(N, K, generator=g).to(torch.bfloat16)
    b = torch.randn(N, generator=g)
    res = torch.randn(M, N, generator=g).to(torch.bfloat16)
    dt = torch.bfloat16
    _, z, _, _ = dr.layer_norm(x, gam, bet, 1e-5, dt)
    want = F.layer_norm(x.double(), (K,), gam.double(), bet.double(), 1e-5)
    assert float((z - want).abs().max()) < 1e-12
    t = torch.linspace(-8, 8, 1001, dtype=torch.float64)
    assert float((dr.gelu(t) - F.gelu(t)).abs().max()) < 1e-12
    xn = want.to(dt).double()
    rb = b.to(dt).double()
    inner = (xn @ W.double().t() + rb).to(dt).double()
    for epi, out in ((dr.EPI_STORE, inner), (dr.EPI_GELU, F.gelu(inner).to(dt).double()),
                     (dr.EPI_RESIDUAL, (res.double() + inner).to(dt).double())):
        got = dr.linear(x, W, b, dt, x_mode=dr.X_LAYERNORM, ln=(gam, bet, 1e-5), epi=epi, res=res)["out"]
        assert float((got - out).abs().max()) < 1e-12, epi
    parts = torch.randn(3, M, K, generator=g)
    got = dr.linear(parts, W, b, dt, x_mode=dr.X_PARTIAL_SUM)["out"]
    want = ((parts.double().sum(0)).to(dt).double() @ W.double().t() + rb).to(dt).double()
    # the statement adds the partials in split order; a different order may flip a rounding of the input row only
    assert float((got - want).abs().max() / want.abs().max()) < 1e-2
    lg = dr.linear(x, W, None, dt, epi=dr.EPI_LOGITS_F32)["out"]
    assert torch.equal(lg, (x.double() @ W.double().t()).to(dt).double())


def test_attention_and_embedding_match_fp64_torch():
    g = torch.Generator().manual_seed(1)
    n, keys, d = 3, 37, 256
    dt = torch.float16
    q = torch.randn(n, d, generator=g).to(dt)
    kc = torch.randn(n, keys, d, generator=g).to(dt)
    vc = torch.randn(n, keys, d, generator=g).to(dt)
    got = dr.attention(q, kc, vc, dt)
    H = d // 64
    qs = (q.float() * dr.SCALE).to(dt).double().view(n, H, 64)
    ks = (kc.float() * dr.SCALE).to(dt).double().view(n, keys, H, 64)
    s = torch.einsum("nhc,njhc->nhj", qs, ks).to(dt).double()
    p = torch.softmax(s, dim=-1).to(dt).double()
    want = torch.einsum("nhj,njhc->nhc", p, vc.double().view(n, keys, H, 64)).reshape(n, d)
    assert float((got - want).abs().max()) < 1e-12
    emb, pos = torch.randn(100, 64, generator=g), torch.randn(448, 64, generator=g)
    tokens = torch.tensor([[5, 7, 99], [1, 100, -1]], dtype=torch.int32)
    x = dr.embed(emb, pos, tokens, 1, torch.bfloat16)
    assert torch.equal(x[0], (emb[7] + pos[1]).to(torch.bfloat16))
    assert torch.equal(x[1], (emb[0] + pos[1]).to(torch.bfloat16))        # out of range: row 0


# ---------------------------------------------------------------------------------------------------- the rule's power
WRONG = ["tanh GELU", "bias not rounded", "residual rounded once", "LayerNorm variance over K-1",
         "LayerNorm statistics over K-32 columns", "last 32 k columns dropped", "logits not rounded",
         "partial sums rounded per split"]


def _wrong_linear(wrong, x, W, bias, dt, x_mode, ln, epi, res):
    """An fp32 dec_linear with one deliberate error."""
    K = W.shape[1]
    if x_mode == dr.X_PARTIAL_SUM:
        xin = dr.rnd(sum(dr.rnd(p, dt) for p in x), dt)           # "partial sums rounded per split"
    elif x_mode == dr.X_LAYERNORM:
        xf = x.float()
        cols = K - 32 if wrong == "LayerNorm statistics over K-32 columns" else K
        mean = xf[:, :cols].mean(dim=-1, keepdim=True)
        div = K - 1 if wrong == "LayerNorm variance over K-1" else cols
        var = (xf[:, :cols] - mean).square().sum(dim=-1, keepdim=True) / div
        xin = dr.rnd((xf - mean) * torch.rsqrt(var + ln[2]) * ln[0] + ln[1], dt)
    else:
        xin = x.float()
    Wf = W.float()
    if wrong == "last 32 k columns dropped":
        acc = xin[:, :K - 32] @ Wf[:, :K - 32].t()
    else:
        acc = xin @ Wf.t()
    if epi == dr.EPI_LOGITS_F32:
        return acc if wrong == "logits not rounded" else dr.rnd(acc, dt)
    b = bias.float() if wrong == "bias not rounded" else dr.rnd(bias.float(), dt)
    if wrong == "residual rounded once":
        return dr.rnd(res.float() + acc + b, dt)
    y = dr.rnd(acc + b, dt)
    if epi == dr.EPI_GELU:
        return dr.rnd(F.gelu(y, approximate="tanh") if wrong == "tanh GELU" else F.gelu(y), dt)
    if epi == dr.EPI_RESIDUAL:
        return dr.rnd(res.float() + y, dt)
    return y


def _case(wrong, d, dt, M=8, seed=0):
    """Inputs of the launch the variant lives in, at width d (ln = the engine's LayerNorm affine parameters)."""
    g = torch.Generator().manual_seed(seed + d)
    ln = (1 + 0.2 * torch.randn(d, generator=g), 0.2 * torch.randn(d, generator=g), 1e-5)
    shapes = {"tanh GELU": (4 * d, d, dr.X_LAYERNORM, dr.EPI_GELU),
              "bias not rounded": (3 * d, d, dr.X_LAYERNORM, dr.EPI_STORE),
              "residual rounded once": (d, 4 * d, dr.X_PLAIN, dr.EPI_RESIDUAL),
              "LayerNorm variance over K-1": (4 * d, d, dr.X_LAYERNORM, dr.EPI_GELU),
              "LayerNorm statistics over K-32 columns": (3 * d, d, dr.X_LAYERNORM, dr.EPI_STORE),
              "last 32 k columns dropped": (d, 4 * d, dr.X_PLAIN, dr.EPI_RESIDUAL),
              "logits not rounded": (V, d, dr.X_LAYERNORM, dr.EPI_LOGITS_F32),
              "partial sums rounded per split": (d, d, dr.X_PARTIAL_SUM, dr.EPI_RESIDUAL)}
    N, K, x_mode, epi = shapes[wrong]
    if x_mode == dr.X_PARTIAL_SUM:
        x = torch.randn(8, M, K, generator=g) / 8 ** 0.5
    else:
        x = torch.randn(M, K, generator=g).to(dt)
    W = (torch.randn(N, K, generator=g) / K ** 0.5).to(dt)
    bias = 0.5 * torch.randn(N, generator=g)
    res = torch.randn(M, N, generator=g).to(dt)
    return x, W, bias, x_mode, ln, epi, res


def _fail_ratio(r: dr.LinearErrors) -> float:
    return max(r.worst, r.n_diff / (dr.ALPHA * r.emu_diff + dr.slack(r.numel)))


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("d", WIDTHS)
@pytest.mark.parametrize("wrong", WRONG)
def test_rule_rejects_wrong_linear(wrong, d, dtype):
    x, W, bias, x_mode, ln, epi, res = _case(wrong, d, dtype, M=4 if wrong == "logits not rounded" else 8)
    kw = dict(x_mode=x_mode, ln=ln, epi=epi, res=res)
    ref = dr.linear(x, W, bias, dtype, **kw)
    emu = dr.linear(x, W, bias, dtype, work=torch.float32, **kw)
    dr.check_linear(emu["out"], ref, emu, dtype, epi, name="yardstick")      # the rule accepts fp32 arithmetic
    got = _wrong_linear(wrong, x, W, bias, dtype, x_mode, ln, epi, res)
    r = dr.linear_errors(got, ref, emu, dtype, epi)
    ratio = _fail_ratio(r)
    print(f"{wrong} {DT_ID[dtype]} d={d}: fails by {ratio:.3g} ({r})")
    assert ratio > 1.0, f"{wrong}: not rejected ({r})"
    with pytest.raises(AssertionError):
        dr.check_linear(got, ref, emu, dtype, epi, name=wrong)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_one_partial_rounded_per_split_is_the_correct_result(dtype):
    """With one partial, rounding it per split is the same rounding: that variant is undetectable there by definition,
    which is why the GPU tests run PARTIAL_SUM with 8 partials too."""
    g = torch.Generator().manual_seed(3)
    parts = torch.randn(1, 4, 384, generator=g)
    W = (torch.randn(384, 384, generator=g) / 384 ** 0.5).to(dtype)
    b = torch.randn(384, generator=g)
    ref = dr.linear(parts, W, b, dtype, x_mode=dr.X_PARTIAL_SUM)
    got = _wrong_linear("partial sums rounded per split", parts, W, b, dtype, dr.X_PARTIAL_SUM, None, dr.EPI_STORE, None)
    assert torch.equal(got.double(), dr.linear(parts, W, b, dtype, x_mode=dr.X_PARTIAL_SUM, work=torch.float32)["out"].double())
    assert ref["out"].shape == got.shape


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_step_rule_rejects_a_wrong_row(dtype):
    g = torch.Generator().manual_seed(4)
    ref = torch.randn(6, 1000, generator=g, dtype=torch.float64)
    emu = ref + 1e-3 * torch.randn(6, 1000, generator=g, dtype=torch.float64) * dr.U[dtype]
    dr.check_rows(emu, ref, emu, dtype)
    bad = emu.clone()
    bad[3] += 0.05 * dr.U[dtype] * ref[3]
    with pytest.raises(AssertionError):
        dr.check_rows(bad, ref, emu, dtype)
