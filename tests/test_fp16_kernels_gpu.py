"""fp16 instantiations of the training kernels against fp32 torch rounded to fp16 at the same points.

Tolerances are in fp16 units: a result that is rounded once to fp16 may differ from the reference by one rounding
(2^-11 relative) plus the fp32 summation-order noise of the reference.  Two checks show the kernels really run in fp16:
operands with 10-bit mantissas give exact products (bf16 keeps 7 bits), and an output above 65504 is +inf.
"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

H16 = torch.float16
EPS = 2.0 ** -11          # fp16 unit roundoff


def _rel(a, b):
    return float((a.detach().float() - b.detach().float()).norm() / (b.detach().float().norm() + 1e-30))


def _h(x):
    return x.to(H16).float()


@pytest.fixture(scope="module")
def K():
    from olmoasr_b200 import kernels
    return kernels


def _gelu(x):
    return F.gelu(x)


@pytest.mark.parametrize("bn", [64, 128, 256])
@pytest.mark.parametrize("layout", ["fwd", "dgrad"])
@pytest.mark.parametrize("epi", ["plain", "gelu", "residual", "gelu_bwd", "f32"])
def test_gemm_epilogues(K, bn, layout, epi):
    torch.manual_seed(1)
    M, N, Kd = 300, 520, 384
    a = torch.randn(M, Kd, device="cuda").to(H16)
    w = (torch.randn(N, Kd, device="cuda") / math.sqrt(Kd)).to(H16)
    bias = torch.randn(N, device="cuda")
    aux = torch.randn(M, N, device="cuda").to(H16)
    acc = a.float() @ w.float().T
    kw = dict(block_n=bn)
    if layout == "dgrad":           # B stored (K, N): MN-major read
        b_op, kw["b_mn"] = w.T.contiguous(), True
    else:
        b_op = w
    if epi == "plain":
        got = K.gemm(a, b_op, M, N, Kd, bias=bias, **kw)
        ref = _h(acc + _h(bias))
    elif epi == "gelu":
        got, g = K.gemm(a, b_op, M, N, Kd, bias=bias, epi=K.EPI_BF16_GELU, **kw) if layout == "fwd" else (None, None)
        if got is None:
            pytest.skip("GELU epilogue is a forward-only kernel")
        ref = _h(acc + _h(bias))
        assert _rel(g, _h(_gelu(ref))) < 4 * EPS
    elif epi == "residual":
        got = K.gemm(a, b_op, M, N, Kd, bias=bias, aux=aux, epi=K.EPI_BF16_RESIDUAL, **kw)
        ref = _h(aux.float() + _h(acc + _h(bias)))
    elif epi == "gelu_bwd":
        got = K.gemm(a, b_op, M, N, Kd, aux=aux, epi=K.EPI_BF16_GELU_BWD, **kw)
        x = aux.float()
        cdf = 0.5 * (1 + torch.erf(x / math.sqrt(2)))
        ref = _h(_h(acc) * (cdf + x * torch.exp(-0.5 * x * x) / math.sqrt(2 * math.pi)))
    else:
        got = K.gemm(a, b_op, M, N, Kd, bias=bias, epi=K.EPI_F32, **kw)
        ref = acc + bias
    assert got.dtype == (torch.float32 if epi == "f32" else H16)
    tol = 1e-5 if epi == "f32" else 4 * EPS
    assert _rel(got, ref) < tol, (epi, layout, bn, _rel(got, ref))


@pytest.mark.parametrize("split", [1, 3])
@pytest.mark.parametrize("bn", [64, 128, 256])
def test_gemm_wgrad_split_k(K, split, bn):
    torch.manual_seed(2)
    M, N, Kd = 1000, 192, 320
    dy = torch.randn(M, N, device="cuda").to(H16)
    x = torch.randn(M, Kd, device="cuda").to(H16)
    ref = dy.float().T @ x.float()
    out = torch.zeros(N, Kd, device="cuda")
    K.gemm(dy, x, N, Kd, M, a_mn=True, b_mn=True, out=out, epi=K.EPI_F32_ATOMIC_ADD, split_k=split, block_n=bn)
    assert _rel(out, ref) < 1e-5
    if split == 1:      # the plain fp32 epilogue of a fresh weight gradient (split-K always accumulates)
        out = K.gemm(dy, x, N, Kd, M, a_mn=True, b_mn=True, epi=K.EPI_F32, block_n=bn)
        assert _rel(out, ref) < 1e-5


def test_gemm_operands_are_fp16_exact_products(K):
    """1 + 2^-9 is an fp16 number but not a bf16 one: its square 1 + 2^-8 + 2^-18 summed 64 times is exact in fp32."""
    v = 1.0 + 2.0 ** -9
    a = torch.full((128, 64), v, device="cuda", dtype=H16)
    b = torch.full((64, 64), v, device="cuda", dtype=H16)
    out = K.gemm(a, b, 128, 64, 64, epi=K.EPI_F32)
    assert torch.all(out == 64 * v * v)
    assert 64 * v * v != 64 * float(torch.tensor(v).bfloat16()) ** 2


def test_gemm_overflow_is_inf(K):
    a = torch.full((128, 64), 256.0, device="cuda", dtype=H16)
    b = torch.full((64, 64), 256.0, device="cuda", dtype=H16)
    out = K.gemm(a, b, 128, 64, 64)                          # 64 * 65536 > 65504
    assert torch.all(torch.isposinf(out.float()))
    neg = K.gemm(a, -b, 128, 64, 64)
    assert torch.all(torch.isneginf(neg.float()))


def _attn_ref(q, k, v, B, H, Tq, Tkv, causal, kv_len):
    qh = q.float().view(B, Tq, H, 64).transpose(1, 2)
    kh = k.float().view(B, Tkv, H, 64).transpose(1, 2)
    vh = v.float().view(B, Tkv, H, 64).transpose(1, 2)
    mask = torch.zeros(B, 1, Tq, Tkv, device=q.device)
    if causal:
        mask = mask + torch.full((Tq, Tkv), float("-inf"), device=q.device).triu(1)
    if kv_len is not None:
        cols = torch.arange(Tkv, device=q.device)
        mask = mask.masked_fill(cols[None, None, None, :] >= kv_len.view(B, 1, 1, 1), float("-inf"))
    return qh, kh, vh, mask


@pytest.mark.parametrize("use", ["encoder", "decoder", "cross"])
def test_attention_fwd_bwd(K, use):
    torch.manual_seed(3)
    B, H = 2, 4
    Tq, Tkv = {"encoder": (300, 300), "decoder": (200, 200), "cross": (200, 300)}[use]
    causal = use == "decoder"
    kv_len = torch.tensor([150, 200], device="cuda", dtype=torch.int32) if use == "decoder" else None
    q, k, v, do = (torch.randn(B * t, H * 64, device="cuda").to(H16) for t in (Tq, Tkv, Tkv, Tq))
    o, lse = K.attention_fwd(q, k, v, B, H, Tq, Tkv, causal=causal, kv_len=kv_len)
    assert o.dtype == H16
    qh, kh, vh, mask = _attn_ref(q, k, v, B, H, Tq, Tkv, causal, kv_len)
    qh, kh, vh = (t.clone().requires_grad_() for t in (qh, kh, vh))
    ref = F.scaled_dot_product_attention(qh, kh, vh, attn_mask=mask)
    assert _rel(o, ref.transpose(1, 2).reshape(B * Tq, H * 64)) < 8 * EPS
    ref.backward(do.float().view(B, Tq, H, 64).transpose(1, 2))
    dq, dk, dv = K.attention_bwd(q, k, v, o, do, lse, B, H, Tq, Tkv, causal=causal, kv_len=kv_len)
    for got, r in ((dq, qh.grad), (dk, kh.grad), (dv, vh.grad)):
        assert got.dtype == H16
        assert _rel(got, r.transpose(1, 2).reshape(got.shape)) < 16 * EPS


def test_cross_entropy_and_logits(K):
    torch.manual_seed(5)
    rows, V, ld = 100, 51865, 51968
    buf = torch.zeros(rows, ld, device="cuda", dtype=H16)
    buf[:, :V] = (3 * torch.randn(rows, V, device="cuda")).to(H16)
    t = torch.randint(0, V, (rows,), device="cuda")
    t[::7] = 51864
    logits = buf[:, :V].float().requires_grad_()
    assert torch.equal(K.logits_to_f32(buf, V), logits.detach())
    ref = F.cross_entropy(logits, t, ignore_index=51864)
    lse, lsc = K.ce_fwd(buf, t, V, 51864)
    loss = K.ce_finalize(lsc)
    assert abs(loss.item() - ref.item()) <= 1e-5 * abs(ref.item())
    ref.backward()
    K.ce_bwd_(buf, t, lse, lsc, torch.full((1,), 1024.0, device="cuda"), V, 51864)   # a loss scale rides on grad_out
    assert buf.dtype == H16 and _rel(buf[:, :V], _h(1024.0 * logits.grad)) < 2 * EPS
