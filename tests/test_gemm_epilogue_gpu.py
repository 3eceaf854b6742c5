"""16-bit GEMM epilogues, which load the bias and aux of up to 128 columns before any of their stores: every tile width
must give the same bits, and the fp32 torch product with the epilogue's rounding points.  The cases are the ones the
chunking touches: N ending inside a chunk and inside an 8-column group, the in-place residual (aux is the output),
GELU's two outputs, both operand majors of B and both 16-bit types."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def K():
    from olmoasr_b200 import kernels
    return kernels


def _rel_l2(got, want):
    return float((got.float() - want.float()).norm() / want.float().norm())


def _tuple(x):
    return x if isinstance(x, tuple) else (x,)


# b_mn -> 16-bit epilogues compiled for it with a K-major A (csrc/gemm_sm90.cu, dispatch)
PAIRS16 = {0: (0, 1, 2, 3), 1: (0, 2, 3)}
CASES16 = [(b_mn, epi) for b_mn, epis in PAIRS16.items() for epi in epis]
# M tail.  N = 520 ends 8 columns into the last tile at every width, so the last chunk is mostly past N.  N = 300 ends
# inside an 8-column group and gives rows that are not 16-byte aligned: the scalar loads and stores (K-major B only, an
# MN-major operand needs a 16-byte aligned row stride).
M = 1000
NS = (520, 300)
KS = (64, 1096)


def _operands(K, N, Kd, b_mn, epi, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = torch.randn(M, Kd, device="cuda", generator=g).to(dtype)
    B = (torch.randn(N, Kd, device="cuda", generator=g) / math.sqrt(Kd)).to(dtype)
    bias = torch.randn(N, device="cuda", generator=g)
    aux = torch.randn(M, N, device="cuda", generator=g).to(dtype) if epi in (K.EPI_BF16_RESIDUAL, K.EPI_BF16_GELU_BWD) else None
    b = B.t().contiguous() if b_mn else B
    return A, B, b, bias, aux


def _want(K, A, B, bias, aux, epi, dtype):
    """fp32 torch product with the epilogue's rounding points; GELU: its first output (the pre-activation)."""
    h = (A.float() @ B.float().t() + bias.to(dtype).float()).to(dtype).float()
    if epi == K.EPI_BF16_RESIDUAL:
        return aux.float() + h
    if epi == K.EPI_BF16_GELU_BWD:
        x = aux.float().requires_grad_(True)
        torch.nn.functional.gelu(x).backward(h)
        return x.grad
    return h


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("N,Kd", [(n, k) for n in NS for k in KS])
@pytest.mark.parametrize("b_mn,epi", CASES16)
def test_epilogue_same_bits_at_every_width(K, b_mn, epi, N, Kd, dtype):
    if b_mn and N % 8:
        pytest.skip("MN-major operands need a 16-byte aligned row stride")
    A, B, b, bias, aux = _operands(K, N, Kd, b_mn, epi, dtype, seed=Kd + N + 7 * epi + 31 * b_mn)
    outs = {bn: _tuple(K.gemm(A, b, M, N, Kd, b_mn=bool(b_mn), bias=bias, aux=aux, epi=epi, block_n=bn))
            for bn in (256, 128, 64)}
    for bn in (128, 64):
        assert len(outs[bn]) == len(outs[256])
        for x, y in zip(outs[256], outs[bn]):
            assert torch.equal(x, y), f"block_n={bn} differs from block_n=256"
    base = outs[256]
    assert _rel_l2(base[0], _want(K, A, B, bias, aux, epi, dtype)) < 4e-3
    if epi == K.EPI_BF16_GELU:
        g = torch.nn.functional.gelu(base[0].float()).to(dtype)
        assert _rel_l2(base[1], g) < 4e-3


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("b_mn", [0, 1])
def test_epilogue_in_place_residual(K, b_mn, dtype):
    """aux is the output itself, as linear_dgrad uses it: each element must be read before it is overwritten."""
    N, Kd = 520, 1096
    A, B, b, bias, aux = _operands(K, N, Kd, b_mn, K.EPI_BF16_RESIDUAL, dtype, seed=5 + b_mn)
    outs = {}
    for bn in (256, 128, 64):
        out = aux.clone()
        K.gemm(A, b, M, N, Kd, b_mn=bool(b_mn), bias=bias, aux=out, out=out, epi=K.EPI_BF16_RESIDUAL, block_n=bn)
        outs[bn] = out
    for bn, out in outs.items():
        assert torch.equal(out, outs[256]), bn
    assert _rel_l2(outs[256], _want(K, A, B, bias, aux, K.EPI_BF16_RESIDUAL, dtype)) < 4e-3
