"""16-bit GEMM epilogues staged through shared memory.  Results leave through TMA stores, and aux arrives through TMA
loads, where TMA can address the tensor (16-byte aligned base and row stride); otherwise the same staged epilogue moves
them with plain bounded copies.  Both ways must give the same bits, in either direction, as must an output that is a
column slice of a wider buffer, and nothing outside the M x N output may change.  A small SM budget makes every CTA
walk many tiles, so the epilogue buffers and their barriers turn over many times."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def K():
    from olmoasr_b200 import kernels
    return kernels


@pytest.fixture
def few_sms(K):
    prev = K.set_gemm_sm_budget(3)
    yield
    K.set_gemm_sm_budget(prev)


# b_mn -> 16-bit epilogues compiled for it with a K-major A (csrc/gemm_sm90.cu, dispatch)
CASES16 = [(0, 0), (0, 1), (0, 2), (0, 3), (1, 0), (1, 2), (1, 3)]
# The last 128-row tile has 104 rows: its second warpgroup's boxes hold 40.  N = 520 / 1000 end 8 / 40 columns into
# the last 64-column box.  K = 1096 ends inside a k-block.
M, KD = 1000, 1096
NS = (520, 1000)
SENTINEL = 7.0


def _rel_l2(got, want):
    return float((got.float() - want.float()).norm() / want.float().norm())


def _operands(K, N, b_mn, epi, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    A = torch.randn(M, KD, device="cuda", generator=g).to(dtype)
    B = (torch.randn(N, KD, device="cuda", generator=g) / math.sqrt(KD)).to(dtype)
    bias = torch.randn(N, device="cuda", generator=g)
    aux = torch.randn(M, N, device="cuda", generator=g).to(dtype) if epi in (K.EPI_BF16_RESIDUAL, K.EPI_BF16_GELU_BWD) else None
    return A, B, (B.t().contiguous() if b_mn else B), bias, aux


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


def _slice(N, dtype, ld, off, fill=SENTINEL):
    """(M, N) view at column `off` of an (M, ld) buffer filled with `fill`"""
    return torch.full((M, ld), fill, device="cuda", dtype=dtype)[:, off:off + N]


def _gemm(K, A, b, N, b_mn, epi, bias, aux, dtype, ld, off, bn):
    """the product into (M, N) view(s) at column `off` of (M, ld) buffers (two for GELU)"""
    out = _slice(N, dtype, ld, off)
    out2 = _slice(N, dtype, ld, off) if epi == K.EPI_BF16_GELU else None
    r = K.gemm(A, b, M, N, KD, b_mn=bool(b_mn), out=out, out2=out2, bias=bias, aux=aux, epi=epi, block_n=bn)
    return r if isinstance(r, tuple) else (r,)


def _untouched(view, N, off):
    base = view.as_strided((M, view.stride(0)), (view.stride(0), 1), view.storage_offset() - off)
    outside = torch.cat([base[:, :off], base[:, off + N:]], dim=1)
    return bool((outside.float() == SENTINEL).all())


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("N", NS)
@pytest.mark.parametrize("b_mn,epi", CASES16)
def test_tma_and_plain_copies_same_bits(K, few_sms, b_mn, epi, N, dtype):
    A, B, b, bias, aux = _operands(K, N, b_mn, epi, dtype, seed=N + 7 * epi + 31 * b_mn)
    for bn in (256, 128, 64):
        ref = _gemm(K, A, b, N, b_mn, epi, bias, aux, dtype, N, 0, bn)   # contiguous: TMA both ways
        if bn == 256:
            assert _rel_l2(ref[0], _want(K, A, B, bias, aux, epi, dtype)) < 4e-3
            if epi == K.EPI_BF16_GELU:
                assert _rel_l2(ref[1], torch.nn.functional.gelu(ref[0].float()).to(dtype)) < 4e-3
        # output: a column slice of a wider buffer (TMA, ldc > N, 32-byte offset); a row stride of N + 3 (plain stores)
        variants = [(N + 56, 16, aux), (N + 3, 0, aux)]
        if aux is not None:   # aux read with plain loads (row stride N + 5), output stored by TMA
            aux_odd = _slice(N, dtype, N + 5, 0)
            aux_odd.copy_(aux)
            variants.append((N, 0, aux_odd))
        for ld, off, a in variants:
            got = _gemm(K, A, b, N, b_mn, epi, bias, a, dtype, ld, off, bn)
            for x, y in zip(got, ref):
                assert torch.equal(x, y), f"block_n={bn} ld={ld} off={off} aux ld={a.stride(0) if a is not None else None}"
                assert _untouched(x, N, off), f"block_n={bn} ld={ld} off={off}: wrote outside the output"


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("b_mn", [0, 1])
@pytest.mark.parametrize("ld", [1000, 1003], ids=["tma", "plain"])
def test_in_place_residual(K, few_sms, b_mn, ld, dtype):
    """aux is the output itself, as linear_dgrad uses it: each tile's aux must be in shared memory before its stores."""
    N = 1000
    A, B, b, bias, aux = _operands(K, N, b_mn, K.EPI_BF16_RESIDUAL, dtype, seed=11 + b_mn)
    want = _gemm(K, A, b, N, b_mn, K.EPI_BF16_RESIDUAL, bias, aux, dtype, N, 0, 256)[0]
    for bn in (256, 128, 64):
        out = _slice(N, dtype, ld, 0)
        out.copy_(aux)
        K.gemm(A, b, M, N, KD, b_mn=bool(b_mn), bias=bias, aux=out, out=out, epi=K.EPI_BF16_RESIDUAL, block_n=bn)
        assert torch.equal(out, want), bn
        assert _untouched(out, N, 0)
