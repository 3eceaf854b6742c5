"""128 x 256 GEMM tiles against the narrower widths: per-element arithmetic does not depend on the tile, so every
instantiated (operand majors, epilogue) pair must give the same bits at block_n = 256, 128 and 64, under any SM budget."""
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


# (a_mn, b_mn) -> epilogues compiled for it (csrc/gemm_sm90.cu, dispatch)
PAIRS = {(0, 0): (0, 1, 2, 3, 4), (0, 1): (0, 2, 3, 4), (1, 1): (4, 5)}
CASES = [(a_mn, b_mn, epi) for (a_mn, b_mn), epis in PAIRS.items() for epi in epis]
# M, N and K tails; 776 rows = 7 row tiles (odd); N = 40 fits one 64-wide tile
SHAPES = [(1000, 1865, 240), (776, 1864, 240), (776, 40, 136)]


def _operands(K, M, N, Kd, a_mn, b_mn, epi, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = torch.randn(M, Kd, device="cuda", generator=g).bfloat16()
    B = (torch.randn(N, Kd, device="cuda", generator=g) / math.sqrt(Kd)).bfloat16()
    bias = torch.randn(N, device="cuda", generator=g) if epi != K.EPI_F32_ATOMIC_ADD else None
    aux = torch.randn(M, N, device="cuda", generator=g).bfloat16() if epi in (K.EPI_BF16_RESIDUAL, K.EPI_BF16_GELU_BWD) else None
    a = A.t().contiguous() if a_mn else A
    b = B.t().contiguous() if b_mn else B
    return A, B, a, b, bias, aux


def _run(K, a, b, M, N, Kd, a_mn, b_mn, epi, bias, aux, bn, split_k=1):
    out = torch.full((M, N), 0.5, device="cuda") if epi == K.EPI_F32_ATOMIC_ADD else None
    r = K.gemm(a, b, M, N, Kd, a_mn=bool(a_mn), b_mn=bool(b_mn), out=out, bias=bias, aux=aux, epi=epi,
               split_k=split_k, block_n=bn)
    return r if out is None else out


@pytest.mark.parametrize("M,N,Kd", SHAPES)
@pytest.mark.parametrize("a_mn,b_mn,epi", CASES)
def test_gemm_widths_bit_identical(K, M, N, Kd, a_mn, b_mn, epi):
    if (a_mn and M % 8) or (b_mn and N % 8):
        pytest.skip("MN-major operands need a 16-byte aligned row stride")
    A, B, a, b, bias, aux = _operands(K, M, N, Kd, a_mn, b_mn, epi, seed=M + N + Kd)
    outs = {bn: _run(K, a, b, M, N, Kd, a_mn, b_mn, epi, bias, aux, bn) for bn in (256, 128, 64)}
    for bn in (128, 64):
        for x, y in zip(outs[256] if isinstance(outs[256], tuple) else (outs[256],),
                        outs[bn] if isinstance(outs[bn], tuple) else (outs[bn],)):
            assert torch.equal(x, y), f"block_n=256 differs from block_n={bn}"
    # and the common result is the right one
    ref = A.float() @ B.float().t()
    if epi == K.EPI_F32_ATOMIC_ADD:
        assert _rel_l2(outs[256] - 0.5, ref) < 1e-5
    elif epi == K.EPI_F32:
        assert _rel_l2(outs[256], ref + bias) < 1e-5
    else:
        h = (ref + bias.bfloat16().float()).bfloat16().float()
        got = outs[256][0] if epi == K.EPI_BF16_GELU else outs[256]
        if epi == K.EPI_BF16_RESIDUAL:
            want = aux.float() + h
        elif epi == K.EPI_BF16_GELU_BWD:
            x = aux.float().requires_grad_(True)
            torch.nn.functional.gelu(x).backward(h)
            want = x.grad
        else:
            want = h
        assert _rel_l2(got, want) < 4e-3


@pytest.mark.parametrize("a_mn,b_mn,epi", [(0, 0, 1), (0, 1, 3), (1, 1, 4)])
def test_gemm_wide_same_bits_under_any_budget(K, a_mn, b_mn, epi):
    M, N, Kd = 6144, 3072, 512      # 48 x 12 = 576 tiles of 128 x 256
    A, B, a, b, bias, aux = _operands(K, M, N, Kd, a_mn, b_mn, epi, seed=21)
    base = _run(K, a, b, M, N, Kd, a_mn, b_mn, epi, bias, aux, 256)
    prev = K.set_gemm_sm_budget(21)
    try:
        b21 = _run(K, a, b, M, N, Kd, a_mn, b_mn, epi, bias, aux, 256)
        K.set_gemm_sm_budget(131)
        b131 = _run(K, a, b, M, N, Kd, a_mn, b_mn, epi, bias, aux, 256)
    finally:
        K.set_gemm_sm_budget(prev)
    for got in (b21, b131):
        for x, y in zip(base if isinstance(base, tuple) else (base,), got if isinstance(got, tuple) else (got,)):
            assert torch.equal(x, y)


def test_gemm_wide_split_k(K):
    torch.manual_seed(13)
    M, N, Kd = 12000, 1024, 1000            # dW = dy^T x: reduction over 12000 rows, 8 x 4 output tiles of 128 x 256
    dy = (torch.randn(M, N, device="cuda") * 0.05).bfloat16()
    x = torch.randn(M, Kd, device="cuda").bfloat16()
    ref = dy.float().t() @ x.float()
    for split in (1, 4, 7):
        out = torch.full((N, Kd), 1.0, device="cuda")
        K.gemm(dy, x, N, Kd, M, a_mn=True, b_mn=True, out=out, epi=K.EPI_F32_ATOMIC_ADD, split_k=split, block_n=256)
        assert _rel_l2(out - 1.0, ref) < 2e-4, split
