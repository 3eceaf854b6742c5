"""The training step's GEMM launches, fused loss head and LayerNorm against the fp64 statements of
tests/training_reference.py, at every launch form the step makes, in bf16 and fp16, at the widths of
config/model_dims.py (d = 384 .. 1280, MLP 4d), and at the edges where tiled kernels go wrong: M, N and K tails, MN-major
operands with padded row strides, a small SM budget, both aux / output paths (TMA and plain copies), GELU inputs across
[-8, 8], fp16 overflow, peaked / ignored / tail-target cross-entropy rows and LayerNorm statistics near eps.
"""
import math

import pytest
import torch

from tests import decode_reference as dr
from tests import training_reference as tr

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]
DT_ID = {torch.bfloat16: "bf16", torch.float16: "fp16"}
WIDTHS = [384, 512, 768, 1024, 1280]
V, LD, IGNORE = 51865, 51968, 51863
SENTINEL = 7.0
# Rule 2 of the logits dgrad (K = 51865): the wgmma accumulation passes a product through 3242 truncating fp32 stages
# where cuBLAS's fp32 yardstick sums far more accurately, so the kernel flips up to 72 x as many T roundings (bf16,
# d = 1280; 39 at d = 384, 23 in fp16; measured on an H100 SXM) while rule 1 holds every element within one ulp plus
# its stage bound (worst 0.33 of it).
LOGITS_ALPHA = 150.0
# The composed loss head per row against the fp64 composition: the worst row within HEAD_ALPHA x the yardstick's
# (measured 4.6, d(embedding) at d = 768 in bf16) and the mean row within HEAD_MEAN_ALPHA x (measured 44: the
# flipped roundings of the logits dgrad above reach every dx row, where the yardstick's rows are nearly exact).
HEAD_ALPHA, HEAD_MEAN_ALPHA = 8.0, 100.0


@pytest.fixture(scope="module")
def K():
    from olmoasr_b200 import kernels
    return kernels


@pytest.fixture(scope="module")
def core():
    from olmoasr_b200 import _core
    return _core


def _dev_gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _rand(shape, g, scale=1.0, dtype=torch.float32):
    return (torch.randn(shape, device="cuda", generator=g) * scale).to(dtype)


def _keys(epi):
    return ("out", "out2") if epi == tr.EPI_GELU else ("out",)


def _check_16(got, A, B, epi, dtype, name, alpha=tr.ALPHA, **kw):
    """got: the kernel's output (or (h, g) for GELU) for the logical operands A (M, K), B (N, K)."""
    errs = tr.gemm_in_slabs(got, A, B, epi, dtype, keys=_keys(epi), **kw)
    for k, r in errs.items():
        tr.check16(r, dtype, name=f"{name} {k}", alpha=alpha)


def _check_32(got, A, B, epi, dtype, name, slab=4096, **kw):
    parts, rows = [], []
    for s in tr.rows_in_slabs(A.shape[0], slab):
        kws = {k: (v[s] if k == "out0" else v) for k, v in kw.items()}
        ref = tr.gemm(A[s], B, epi, dtype, **kws)
        emu = tr.gemm(A[s], B, epi, dtype, work=torch.float32, **kws)
        parts.append(tr.errors32(got[s], ref["out"], emu["out"], ref["allow"]))
        rows.append(s.stop - s.start)
        del ref, emu
    tr.check32(tr.merge32(parts, rows), name=name)


# ================================================================================================ GEMM: forward
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("d", WIDTHS)
def test_gemm_forward_forms(core, K, d, dtype):
    """qkv (zero key-bias rows), attention out / cross out RESIDUAL, fc1 GELU, fc2 RESIDUAL (K = 4d) at M = 2 x 1500."""
    g = _dev_gen(d)
    M = 3000
    x = _rand((M, d), g, 1.0, dtype)
    wqkv = _rand((3 * d, d), g, d ** -0.5, dtype)
    bqkv = _rand(3 * d, g, 0.5)
    bqkv[d:2 * d] = 0                       # the key projection has no bias
    _check_16(core.linear_fwd(x, wqkv, bqkv), x, wqkv, tr.EPI_BF16, dtype, f"qkv d={d}", bias=bqkv)
    wo, bo = _rand((d, d), g, d ** -0.5, dtype), _rand(d, g, 0.5)
    res = _rand((M, d), g, 2.0, dtype)
    got = core.linear_fwd(x, wo, bo, epi=K.EPI_BF16_RESIDUAL, aux=res)
    _check_16(got, x, wo, tr.EPI_RESIDUAL, dtype, f"out d={d}", bias=bo, aux=res)
    w1, b1 = _rand((4 * d, d), g, d ** -0.5, dtype), _rand(4 * d, g, 0.5)
    h, gl = core.linear_fwd(x, w1, b1, epi=K.EPI_BF16_GELU)
    _check_16((h, gl), x, w1, tr.EPI_GELU, dtype, f"fc1 d={d}", bias=b1)
    w2, b2 = _rand((d, 4 * d), g, (4 * d) ** -0.5, dtype), _rand(d, g, 0.5)
    got = core.linear_fwd(gl, w2, b2, epi=K.EPI_BF16_RESIDUAL, aux=res)
    _check_16(got, gl, w2, tr.EPI_RESIDUAL, dtype, f"fc2 d={d}", bias=b2, aux=res)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("d", WIDTHS)
def test_gemm_conv_stem_forms(core, K, d, dtype):
    """conv1 (K = 3 x 80 mels = 240, M = B x 3000) and conv2 (K = 3d, M = B x 1500) with the GELU epilogue, B = 2."""
    g = _dev_gen(100 + d)
    A1 = _rand((6000, 240), g, 1.0, dtype)
    w1, b1 = _rand((d, 240), g, 240 ** -0.5, dtype), _rand(d, g, 0.5)
    _check_16(core.linear_fwd(A1, w1, b1, epi=K.EPI_BF16_GELU), A1, w1, tr.EPI_GELU, dtype, f"conv1 d={d}", bias=b1)
    A2 = _rand((3000, 3 * d), g, 1.0, dtype)
    w2, b2 = _rand((d, 3 * d), g, (3 * d) ** -0.5, dtype), _rand(d, g, 0.5)
    _check_16(core.linear_fwd(A2, w2, b2, epi=K.EPI_BF16_GELU), A2, w2, tr.EPI_GELU, dtype, f"conv2 d={d}", bias=b2)


# ================================================================================================ GEMM: backward
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("d", WIDTHS)
def test_gemm_dgrad_forms(core, K, d, dtype):
    """dx = dy W (W read MN-major): plain, GELU_BWD into fc1's output (N = 4d), RESIDUAL in place (aux is out)."""
    g = _dev_gen(200 + d)
    M = 3000
    dy = _rand((M, d), g, 1.0, dtype)
    w = _rand((d, d), g, d ** -0.5, dtype)
    _check_16(core.linear_dgrad(dy, w), dy, w.t(), tr.EPI_BF16, dtype, f"dgrad d={d}")
    w2 = _rand((d, 4 * d), g, d ** -0.5, dtype)
    h = _rand((M, 4 * d), g, 2.0, dtype)
    got = core.linear_dgrad(dy, w2, epi=K.EPI_BF16_GELU_BWD, aux=h)
    _check_16(got, dy, w2.t(), tr.EPI_GELU_BWD, dtype, f"gelu_bwd d={d}", aux=h)
    dkv = _rand((M, 2 * d), g, 1.0, dtype)
    wkv = _rand((2 * d, d), g, d ** -0.5, dtype)
    buf = _rand((M, d), g, 2.0, dtype)
    before = buf.clone()
    core.linear_dgrad(dkv, wkv, epi=K.EPI_BF16_RESIDUAL, aux=buf, out=buf)
    _check_16(buf, dkv, wkv.t(), tr.EPI_RESIDUAL, dtype, f"cross kv dgrad in place d={d}", aux=before)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("d", WIDTHS)
def test_gemm_wgrad_forms(core, K, d, dtype):
    """dW = dy^T x (both MN-major), fc1's shape (N = 4d, K = d, M = 3000 rows): F32 fresh, then ATOMIC_ADD into a
    non-zero slab at _pick_split_k's split and at splits whose last split is short."""
    g = _dev_gen(300 + d)
    M = 3000
    dy = _rand((M, 4 * d), g, 0.1, dtype)
    x = _rand((M, d), g, 1.0, dtype)
    bn = 256 if d >= 256 else 128
    fresh = K.gemm(dy, x, 4 * d, d, M, a_mn=True, b_mn=True, epi=K.EPI_F32, block_n=bn)
    _check_32(fresh, dy.t(), x.t(), tr.EPI_F32, dtype, f"wgrad fresh d={d}")
    pick = core._pick_split_k(math.ceil(4 * d / 128) * math.ceil(d / bn), math.ceil(M / 64))
    for split in sorted({pick, 3, 7}):          # 47 k-blocks: 3 x 16 leaves 15, 7 x 7 leaves 5
        out0 = _rand((4 * d, d), g, 0.5)
        out = out0.clone()
        K.gemm(dy, x, 4 * d, d, M, a_mn=True, b_mn=True, out=out, epi=K.EPI_F32_ATOMIC_ADD, split_k=split, block_n=bn)
        _check_32(out, dy.t(), x.t(), tr.EPI_F32_ATOMIC_ADD, dtype, f"wgrad split {split} d={d}", out0=out0, split_k=split)


def test_gemm_rejects_a_bias_with_the_accumulating_epilogue(K):
    """C += acc takes no bias: under split-K every split's partial would add it once."""
    from olmoasr_b200 import _lib
    from olmoasr_b200._lib import OasrError, ptr, stream
    g = _dev_gen(5)
    dy = _rand((512, 256), g, 1.0, torch.bfloat16)
    x = _rand((512, 128), g, 1.0, torch.bfloat16)
    bias = torch.ones(256, device="cuda")
    out = torch.zeros(256, 128, device="cuda")
    with pytest.raises(ValueError):
        K.gemm(dy, x, 256, 128, 512, a_mn=True, b_mn=True, out=out, bias=bias, epi=K.EPI_F32_ATOMIC_ADD, split_k=3)
    for split in (1, 3):     # the C entry point refuses it too
        with pytest.raises(OasrError):
            _lib.call("oasr_gemm_bf16", ptr(dy), dy.stride(0), 1, ptr(x), x.stride(0), 1, ptr(out), out.stride(0), None,
                      ptr(bias), None, 0, 256, 128, 512, K.EPI_F32_ATOMIC_ADD, split, 0, stream())
    torch.cuda.synchronize()
    assert not out.any()


# ================================================================================================ GEMM: tied logits
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("d", WIDTHS)
def test_gemm_tied_logits_forms(core, K, d, dtype):
    """B x 448 rows (B = 7: M % 128 = 64): logits into ld 51968, dgrad at K = 51865 reading buf[:, :V] with NaN in the
    padding columns, and the tied embedding's wgrad (N = 51865 output rows, A MN-major with inner extent 51865)."""
    g = _dev_gen(400 + d)
    M = 7 * 448
    x = _rand((M, d), g, 1.0, dtype)
    E = _rand((V, d), g, d ** -0.5, dtype)
    buf = torch.full((M, LD), SENTINEL, device="cuda", dtype=dtype)
    K.gemm(x, E, M, V, d, out=buf, block_n=256)
    assert bool((buf[:, V:] == SENTINEL).all()), "the logits GEMM wrote a padding column"
    _check_16(buf, x, E, tr.EPI_BF16, dtype, f"logits d={d}")
    dl = torch.full((M, LD), float("nan"), device="cuda", dtype=dtype)
    dl[:, :V] = _rand((M, V), g, 0.05, dtype)
    dx = K.gemm(dl[:, :V], E, M, d, V, b_mn=True, block_n=core._pick_block_n(M, d))
    _check_16(dx, dl[:, :V], E.t(), tr.EPI_BF16, dtype, f"logits dgrad d={d}", alpha=LOGITS_ALPHA)
    dE = core.linear_wgrad(dl, x, n_valid=V)
    _check_32(dE, dl[:, :V].t(), x.t(), tr.EPI_F32, dtype, f"embedding wgrad d={d}", slab=8192)


# ================================================================================================ GEMM: edges
EDGES = [(129, 264, 72), (136, 320, 89), (192, 321, 72), (193, 409, 89), (255, 409, 72)]   # M%128, N%256, K%64 tails


def _strided(rows, cols, ld, g, scale, dtype, fill=None):
    """A (rows, cols) view of a (rows + 2, ld) buffer (extra rows and columns hold `fill`, random when None)."""
    base = _rand((rows + 2, ld), g, scale, dtype) if fill is None else torch.full((rows + 2, ld), fill, device="cuda", dtype=dtype)
    return base, base[:rows, :cols]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("path", ["tma", "plain"])
@pytest.mark.parametrize("epi", [tr.EPI_BF16, tr.EPI_GELU, tr.EPI_RESIDUAL, tr.EPI_GELU_BWD], ids=["bf16", "gelu", "residual", "gelu_bwd"])
@pytest.mark.parametrize("M,N,Kd", EDGES)
def test_gemm_edges(K, M, N, Kd, epi, path, dtype):
    """Tails of M, N and K (A and B with padded row strides) on 3 SMs, so every CTA walks many tiles; the outputs and aux
    moved by TMA (16-byte aligned row strides) or by plain copies (odd row strides).  Columns and rows outside M x N
    keep their sentinel: with N % 8 != 0 the box holding column N - 1 must not go out as whole 16-byte TMA chunks."""
    g = _dev_gen(M * N + Kd)
    _, A = _strided(M, Kd, (Kd + 7) // 8 * 8 + 8, g, 1.0, dtype)
    _, B = _strided(N, Kd, (Kd + 7) // 8 * 8 + 8, g, Kd ** -0.5, dtype)
    bias = None if epi == tr.EPI_GELU_BWD else _rand(N, g, 0.5)
    ld = (N + 7) // 8 * 8 + 8 if path == "tma" else N + 1
    aux = None
    if epi in (tr.EPI_RESIDUAL, tr.EPI_GELU_BWD):
        _, aux = _strided(M, N, ld, g, 2.0, dtype)
    obuf, out = _strided(M, N, ld, g, 0, dtype, fill=SENTINEL)
    o2buf, out2 = _strided(M, N, ld, g, 0, dtype, fill=SENTINEL)
    prev = K.set_gemm_sm_budget(3)
    try:
        K.gemm(A, B, M, N, Kd, out=out, out2=out2 if epi == tr.EPI_GELU else None, bias=bias, aux=aux, epi=epi)
    finally:
        K.set_gemm_sm_budget(prev)
    for buf in (obuf, o2buf) if epi == tr.EPI_GELU else (obuf,):
        out_mn = torch.ones_like(buf, dtype=torch.bool)
        out_mn[:M, :N] = False
        assert bool((buf[out_mn] == SENTINEL).all()), "wrote outside M x N"
    got = (out, out2) if epi == tr.EPI_GELU else out
    _check_16(got, A, B, epi, dtype, f"edge {M}x{N}x{Kd} {path}", bias=bias, aux=aux)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("M,N,Kd", EDGES)
def test_gemm_mn_major_with_padded_strides(K, M, N, Kd, dtype):
    """MN-major operands whose inner extent is not a multiple of 8, legal by a padded row stride: dgrad (B MN-major,
    inner extent N) and wgrad (A and B MN-major, inner extents M and N)."""
    g = _dev_gen(7 * M + N)
    # dgrad: out (M, N) = A (M, Kd) . Bs, Bs stored (Kd, N) with row stride N padded to 8
    _, A = _strided(M, Kd, (Kd + 7) // 8 * 8, g, 1.0, dtype)
    _, Bs = _strided(Kd, N, (N + 7) // 8 * 8 + 8, g, Kd ** -0.5, dtype)
    out = K.gemm(A, Bs, M, N, Kd, b_mn=True)
    _check_16(out, A, Bs.t(), tr.EPI_BF16, dtype, f"b_mn {M}x{N}x{Kd}")
    # wgrad: out (M, N) fp32 = As^T Bs over Kd rows, As stored (Kd, M), Bs (Kd, N), both with padded strides
    _, As = _strided(Kd, M, (M + 7) // 8 * 8 + 8, g, 1.0, dtype)
    out0 = _rand((M, N), g, 0.5)
    out = out0.clone()
    K.gemm(As, Bs, M, N, Kd, a_mn=True, b_mn=True, out=out, epi=K.EPI_F32_ATOMIC_ADD, split_k=2)
    _check_32(out, As.t(), Bs.t(), tr.EPI_F32_ATOMIC_ADD, dtype, f"a_mn b_mn {M}x{N}x{Kd}", out0=out0, split_k=2)


def _one_hot_operands(vals, M, dtype):
    """A (M, 64) with one 1 per row and B (N, 64) = vals (N, 64): acc[m, n] = vals[n, m % 64] exactly."""
    A = torch.zeros(M, 64, device="cuda", dtype=dtype)
    A[torch.arange(M), torch.arange(M) % 64] = 1
    return A, vals.to(dtype)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_gemm_gelu_inputs_across_the_range(K, dtype):
    """GELU and GELU' at h and aux spanning [-8, 8] in T, exact zeros included (the epilogue's A&S erf)."""
    M, N = 640, 512
    grid = torch.linspace(-8, 8, N * 64 - 1, device="cuda")
    vals = torch.cat([grid, torch.zeros(1, device="cuda")]).to(dtype).float().view(N, 64)
    A, B = _one_hot_operands(vals, M, dtype)
    h, gl = K.gemm(A, B, M, N, 64, epi=K.EPI_BF16_GELU)
    _check_16((h, gl), A, B, tr.EPI_GELU, dtype, "gelu range")
    aux = torch.cat([torch.linspace(-8, 8, M * N - 1, device="cuda"), torch.zeros(1, device="cuda")])
    aux = aux[torch.randperm(M * N, device="cuda", generator=_dev_gen(8))].view(M, N).to(dtype)
    got = K.gemm(A, B, M, N, 64, aux=aux, epi=K.EPI_BF16_GELU_BWD)
    _check_16(got, A, B, tr.EPI_GELU_BWD, dtype, "gelu_bwd range", aux=aux)


def test_gemm_fp16_overflow_matches_the_reference_infinities(K):
    """fp16 overflow to +-inf in the bias add, the residual add and GELU_BWD's product."""
    dtype = torch.float16
    M, N = 256, 128
    g = _dev_gen(9)
    vals = torch.where(torch.rand(N, 64, device="cuda", generator=g) < 0.3,
                       torch.sign(torch.randn(N, 64, device="cuda", generator=g)) * 60000.0,
                       torch.randn(N, 64, device="cuda", generator=g))
    A, B = _one_hot_operands(vals, M, dtype)
    bias = torch.where(torch.arange(N, device="cuda") % 2 == 0, 10000.0, -3.0)
    got = K.gemm(A, B, M, N, 64, bias=bias)
    assert bool(torch.isinf(got).any())
    _check_16(got, A, B, tr.EPI_BF16, dtype, "fp16 overflow bias", bias=bias)
    aux = torch.where(torch.rand(M, N, device="cuda", generator=g) < 0.5, 30000.0, 1.0).to(dtype)
    got = K.gemm(A, B, M, N, 64, aux=aux, epi=K.EPI_BF16_RESIDUAL)
    assert bool(torch.isinf(got).any())
    _check_16(got, A, B, tr.EPI_RESIDUAL, dtype, "fp16 overflow residual", aux=aux)
    aux = (1.5 + torch.rand(M, N, device="cuda", generator=g)).to(dtype)     # gelu' in (1.06, 1.13): 60000 overflows
    got = K.gemm(A, B, M, N, 64, aux=aux, epi=K.EPI_BF16_GELU_BWD)
    assert bool(torch.isinf(got).any())
    _check_16(got, A, B, tr.EPI_GELU_BWD, dtype, "fp16 overflow gelu_bwd", aux=aux)


# ================================================================================================ cross-entropy
def _ce_rows(rows, dtype, g):
    """Production-sized logits (rows, LD) with NaN padding and targets exercising every kernel path."""
    logits = torch.full((rows, LD), float("nan"), device="cuda", dtype=dtype)
    logits[:, :V] = _rand((rows, V), g, 2.0, dtype)
    y = torch.randint(0, V, (rows,), device="cuda", generator=g)
    logits[0, :V] = 0.0                                   # all equal
    logits[1, 12345] = 30.0                               # peaked
    y[1] = 12345
    for i, t in enumerate((0, 7, 8, V - 2, V - 1)):       # group edges and the scalar tail (V = 8 x 6483 + 1)
        y[2 + i] = t
    logits[6, V - 1] = 30.0                               # a peaked tail column
    y[7:40:3] = IGNORE
    y[8], y[9] = V, -1                                    # out of range
    logits[10:20, 2048:2056] = float("-inf")              # an all -inf group after finite ones (thread 0's second)
    logits[20, 0:8] = float("-inf")                       # ... and as a thread's first group
    logits[21, :V:3] = float("-inf")
    return logits, y


@pytest.mark.parametrize("dtype,grad_out", [(torch.bfloat16, 1.0), (torch.float16, 1024.0), (torch.float16, 65536.0)],
                         ids=["bf16", "fp16-1024", "fp16-65536"])
def test_cross_entropy_production_rows(K, dtype, grad_out):
    """14336 rows x 51865 (each thread of the loss sum adds 14 rows): lse, count, bad count and loss, then d(logits) in
    place; the NaN padding columns are neither read nor written, ignored and out-of-range rows get zero gradients."""
    g = _dev_gen(11)
    rows = 14336
    logits, y = _ce_rows(rows, dtype, g)
    keep = logits.clone()
    lse, lsc = K.ce_fwd(logits, y, V, IGNORE)
    loss = K.ce_finalize(lsc)
    ref = tr.ce_fwd(logits, y, V, IGNORE)
    assert float(lsc[1]) == float(ref["count"]) and float(lsc[2]) == float(ref["bad"]) == 2.0
    assert bool(torch.isfinite(lse).all()), "a non-finite lse"
    tr.check_lse(lse, loss, ref, name=f"ce {DT_ID[dtype]}")
    K.ce_bwd_(logits, y, lse, lsc, torch.tensor([grad_out], device="cuda"), V, IGNORE)
    assert bool(torch.isnan(logits[:, V:]).all()), "ce_bwd wrote a padding column"
    cnt = tr.counted_rows(y, V, IGNORE)
    assert not logits[~cnt, :V].any(), "an ignored row has a gradient"
    emu = tr.ce_fwd(keep, y, V, IGNORE, work=torch.float32)
    parts = []
    for s in tr.rows_in_slabs(rows, 2048):
        dref = tr.ce_bwd(keep[s], y[s], V, IGNORE, grad_out, ref["count"], dtype, lse=ref["lse"][s], xmax=ref["xmax"][s])
        demu = tr.ce_bwd(keep[s], y[s], V, IGNORE, grad_out, emu["count"], dtype, lse=emu["lse"][s], work=torch.float32)
        parts.append(tr.errors16(logits[s, :V], dref, demu, dtype))
        del dref, demu
    tr.check16(parts, dtype, name=f"ce_bwd {DT_ID[dtype]} x{grad_out:g}")


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_cross_entropy_inf_logits(K, dtype):
    """-inf logits (fp16 logits overflow) give the finite loss F.cross_entropy gives; a +inf logit gives NaN in both."""
    g = _dev_gen(12)
    logits = _rand((4, LD), g, 2.0, dtype)
    logits[0, 2048:2056] = float("-inf")
    logits[1, 8:16] = float("-inf")
    logits[1, 40000:40008] = float("-inf")
    y = torch.tensor([3, 5, 6, 7], device="cuda")
    lse, lsc = K.ce_fwd(logits, y, V, IGNORE)
    want = torch.nn.functional.cross_entropy(logits[:3, :V].double(), y[:3], reduction="none")
    assert bool(torch.isfinite(lse[:3]).all()) and bool(torch.isfinite(want).all())
    ref = tr.ce_fwd(logits[:3], y[:3], V, IGNORE)
    assert float(tr.lse_error(lse[:3], ref)) <= 1.0
    logits[3, 100] = float("inf")
    lse, lsc = K.ce_fwd(logits, y, V, IGNORE)
    loss = K.ce_finalize(lsc)
    want = torch.nn.functional.cross_entropy(logits[:, :V].double(), y)
    assert math.isnan(float(want)) and math.isnan(float(loss)) and math.isnan(float(lse[3]))


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("d", WIDTHS)
def test_loss_head_composition(core, d, dtype):
    """_LossHeadFn (logits GEMM -> CE -> d(logits) in place -> dgrad and embedding wgrad) against the fp64 composition
    of the statements, per row of dx and of d(embedding), and the loss."""
    g = _dev_gen(500 + d)
    M = 4 * 448
    x = _rand((M, d), g, 1.0, dtype).requires_grad_(True)
    emb = _rand((V, d), g, d ** -0.5).requires_grad_(True)
    emb16 = emb.detach().to(dtype)
    y = torch.randint(0, V, (M,), device="cuda", generator=g)
    y[::7] = IGNORE
    loss = core._LossHeadFn.apply(x, emb, emb16, y, IGNORE)
    loss.backward()
    xd = x.detach()
    out = {}
    for work in (torch.float64, torch.float32):
        logits = tr.gemm(xd, emb16, tr.EPI_BF16, dtype, work=work)["out"].to(dtype)
        f = tr.ce_fwd(logits, y, V, IGNORE, work=work)
        dl = tr.ce_bwd(logits, y, V, IGNORE, 1.0, f["count"], dtype, lse=f["lse"], xmax=f.get("xmax"), work=work)["out"].to(dtype)
        with dr._exact_fp32():
            out[work] = (f["loss"], tr.rnd(dl.to(work) @ emb16.to(work), dtype), dl.to(work).t() @ xd.to(work))
        del logits, dl
    (l64, dx64, de64), (l32, dx32, de32) = out[torch.float64], out[torch.float32]
    assert abs(float(loss) - float(l64)) <= 4 * abs(float(l32) - float(l64)) + 2.0 ** -20 * (1 + abs(float(l64)))
    for got, r64, r32, what in ((x.grad, dx64, dx32, "dx"), (emb.grad, de64, de32, "demb")):
        r = dr.row_errors(got, r64, r32)
        dr._report(kind="step", name=f"loss head {what} d={d}", dtype=str(dtype).removeprefix("torch."), **r._asdict())
        assert r.worst <= HEAD_ALPHA * r.emu_worst and r.mean <= HEAD_MEAN_ALPHA * r.emu_mean, f"loss head {what} d={d}: {r}"


# ================================================================================================ LayerNorm
REGIMES = {"normal": (1.0, 0.0), "mean >> std": (4.0, 200.0), "variance near eps": (3e-3, 0.0), "zero gamma": (1.0, 0.5)}
ROWS = {"normal": 48000, "mean >> std": 777, "variance near eps": 3000, "zero gamma": 1500}


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("regime", list(REGIMES))
@pytest.mark.parametrize("d", WIDTHS)
def test_layernorm(K, d, regime, dtype):
    """Forward (y, mean, rstd) and backward with and without a residual gradient (dx, dw, db).  Rows: 48000 (the
    encoder's B x 1500 at B = 32: the backward at its 2 x SM block cap), 1500 (B = 1: 1500 % 8 = 4, the last block has
    idle warps, below the cap), 777 (an odd count) and 3000."""
    g = _dev_gen(600 + d)
    rows = ROWS[regime]
    std, mean = REGIMES[regime]
    x = (torch.randn(rows, d, device="cuda", generator=g) * std + mean).to(dtype)
    w, b = 1 + 0.3 * torch.randn(d, device="cuda", generator=g), 0.3 * torch.randn(d, device="cuda", generator=g)
    if regime == "zero gamma":
        w[::5] = 0
    y, mu, rs = K.layernorm_fwd(x, w, b)
    ref = tr.layernorm_fwd(x, w, b, 1e-5, dtype)
    emu = tr.layernorm_fwd(x, w, b, 1e-5, dtype, work=torch.float32)
    tr.check16(tr.errors16(y, ref, emu, dtype), dtype, name=f"ln fwd {regime} d={d}")
    assert float(((mu.double() - ref["mean"]).abs() / (x.double().abs().mean(-1) * 2.0 ** -18)).max()) <= 1.0
    assert float(((rs.double() / ref["rstd"] - 1).abs()).max()) <= 2.0 ** -16
    dy = _rand((rows, d), g, 1.0, dtype)
    for dres in (None, _rand((rows, d), g, 1.0, dtype)):
        dw = torch.zeros(d, device="cuda")
        db = torch.zeros(d, device="cuda")
        dx = K.layernorm_bwd(dy, x, w, mu, rs, dw, db, dresidual=dres)
        tag = "with" if dres is not None else "without"
        rb = tr.layernorm_bwd(dy, x, w, 1e-5, dtype, dres=dres)
        eb = tr.layernorm_bwd(dy, x, w, 1e-5, dtype, dres=dres, work=torch.float32)
        tr.check16(tr.errors16(dx, rb, eb, dtype), dtype, name=f"ln bwd dx {tag} dres {regime} d={d}")
        tr.check32(tr.errors32(dw, rb["dw"], eb["dw"], rb["allow_dw"]), name=f"ln dw {regime} d={d}")
        tr.check32(tr.errors32(db, rb["db"], eb["db"], rb["allow_db"]), name=f"ln db {regime} d={d}")
        del rb, eb
