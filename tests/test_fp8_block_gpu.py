"""The FP8 route of the fused training blocks against an fp64 emulation that quantises at the same points.

The emulation states what `_BlockFn` computes under `fp8_autocast()`.  Every projection's forward is
Q4(x) Q4(W)^T + T(b) over the dequantised operands in fp64.  Q4 / Q5 are the per-row e4m3 / e5m2 recipe of
tests/test_fp8_gpu.py, and W is the fused bf16 operand: [Wq; Wk; Wv] and [Wck; Wcv].  The dgrad is
Q5(T(dy)) Q4(W^T)^T, whose weight scales are per input feature of the fused weight.  The wgrad is T(dy)^T x over the
bf16 activations.  LayerNorm, attention, GELU and the residual adds are fp64, rounded to bf16 (T) where the kernels
round.  Outputs, dx, the encoder-output gradient dxa (two decoder layers sharing one quantised xa and accumulating dxa
in place) and every parameter gradient are compared by relative L2.  Checked: an encoder block, and a decoder pair
dense (causal) and packed.

The emulation runs free: its bf16 roundings are not bit for bit the kernels' (attention, LayerNorm and epilogue
internals), and an input one bf16 ulp off flips the fp8 rounding of that element (1/8 to 1/4 of its value), so the two
FP8 computations drift apart by fp8 quantisation noise.  The bf16 route (no context) against the same emulation is the
yardstick.  It differs by the full recipe error, which is what the model-level FP8-vs-bf16 bounds of
tests/test_fp8_gpu.py allow.  The FP8 kernels must be clearly closer to the emulation than that.

The second test settles the routing exactly.  It records every FP8 GEMM of a block's forward and backward.  Its weight
operand must be bit for bit the e4m3 rows of one projection's fused 16-bit weight (forward, e4m3 activations) or of its
transpose (dgrad, e5m2 gradients).  Every forward activation operand must be the quantised input the block saved
(LayerNorm outputs, attention outputs, the GELU output, the encoder output).  Each output must meet the fp64 bound of
tests/test_fp8_gpu.py over its dequantised operands.
"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
FMAX = {0: 448.0, 1: 57344.0}
FP8 = {0: torch.float8_e4m3fn, 1: torch.float8_e5m2}
D, H = 512, 8


def q_rows(x, fmt):
    """Dequantised per-row fp8 of the bf16 values x (the recipe, IEEE fp32 divisions), in fp64."""
    xf = x.float()
    amax = xf.abs().amax(1)
    zero = amax == 0
    fmax = torch.full_like(amax, FMAX[fmt])
    inv = torch.where(zero, torch.ones_like(amax), fmax / amax)
    s = torch.where(zero, torch.ones_like(amax), amax / fmax)
    return (xf * inv[:, None]).to(FP8[fmt]).double() * s.double()[:, None]


class R(torch.autograd.Function):
    """Round to bf16 (a kernel's 16-bit output); the gradient arrives in bf16 as well."""

    @staticmethod
    def forward(ctx, x):
        return x.to(BF).double()

    @staticmethod
    def backward(ctx, g):
        return g.to(BF).double()


class Lin8(torch.autograd.Function):
    """acc = Q4(x) Q4(T(W))^T + T(b); dx = Q5(T(dy)) Q4(T(W)^T)^T; dW = T(dy)^T x; db = sum T(dy)."""

    @staticmethod
    def forward(ctx, x, w, b):
        w16 = w.to(BF)
        ctx.save_for_backward(x, w16)
        ctx.has_b = b is not None
        acc = q_rows(x.to(BF), 0) @ q_rows(w16, 0).t()
        return acc if b is None else acc + b.float().to(BF).double()

    @staticmethod
    def backward(ctx, g):
        x, w16 = ctx.saved_tensors
        g16 = g.to(BF)
        dx = q_rows(g16, 1) @ q_rows(w16.t().contiguous(), 0).t()
        g16 = g16.double()
        return dx, g16.t() @ x, (g16.sum(0) if ctx.has_b else None)


def _ln(x, w, b):
    mean = x.mean(-1, keepdim=True)
    var = ((x - mean) ** 2).mean(-1, keepdim=True)
    return R.apply((x - mean) / torch.sqrt(var + 1e-5) * w + b)


def _attn(q, k, v, causal):
    T, Tk = q.shape[0], k.shape[0]
    qh, kh, vh = (t.reshape(t.shape[0], H, 64).transpose(0, 1) for t in (q, k, v))
    s = qh @ kh.transpose(-1, -2) / 8.0
    if causal:
        s = s + torch.full((T, Tk), -math.inf, dtype=s.dtype, device=s.device).triu(1)
    return R.apply((torch.softmax(s, -1) @ vh).transpose(0, 1).reshape(T, -1))


def emu_block(p, x, xa, lens, causal, cross):
    """x (N, d): the rows of the samples of `lens` stacked; xa (B, Ta, d) or None.  p: fp64 leaves by parameter name."""
    zero = torch.zeros(D, dtype=torch.float64, device=x.device)
    rows = torch.split(torch.arange(x.shape[0], device=x.device), lens)
    ln1 = _ln(x, p["attn_ln.weight"], p["attn_ln.bias"])
    wqkv = torch.cat([p["attn.query.weight"], p["attn.key.weight"], p["attn.value.weight"]])
    qkv = R.apply(Lin8.apply(ln1, wqkv, torch.cat([p["attn.query.bias"], zero, p["attn.value.bias"]])))
    ao = torch.cat([_attn(qkv[r, :D], qkv[r, D:2 * D], qkv[r, 2 * D:], causal) for r in rows])
    x1 = R.apply(x + R.apply(Lin8.apply(ao, p["attn.out.weight"], p["attn.out.bias"])))
    x2 = x1
    if cross:
        lnc = _ln(x1, p["cross_attn_ln.weight"], p["cross_attn_ln.bias"])
        qc = R.apply(Lin8.apply(lnc, p["cross_attn.query.weight"], p["cross_attn.query.bias"]))
        wkv = torch.cat([p["cross_attn.key.weight"], p["cross_attn.value.weight"]])
        kvc = R.apply(Lin8.apply(xa.reshape(-1, D), wkv, torch.cat([zero, p["cross_attn.value.bias"]])))
        kvc = kvc.view(xa.shape[0], xa.shape[1], 2 * D)
        co = torch.cat([_attn(qc[r], kvc[b, :, :D], kvc[b, :, D:], False) for b, r in enumerate(rows)])
        x2 = R.apply(x1 + R.apply(Lin8.apply(co, p["cross_attn.out.weight"], p["cross_attn.out.bias"])))
    ln2 = _ln(x2, p["mlp_ln.weight"], p["mlp_ln.bias"])
    h = R.apply(Lin8.apply(ln2, p["mlp.0.weight"], p["mlp.0.bias"]))
    g = R.apply(F.gelu(h))
    return R.apply(x2 + R.apply(Lin8.apply(g, p["mlp.2.weight"], p["mlp.2.bias"])))


def _rel(a, b):
    return float((a.double() - b.double()).norm() / b.double().norm())


# FP8 kernel against the FP8 emulation, relative L2 per output, the worst over forward output, dx, dxa and every
# parameter gradient, measured on one H100 80GB HBM3 (700 W): encoder 0.090, decoder dense 0.171, packed 0.180 (LayerNorm
# affine and bias gradients, sums of many small terms); the bf16 route against the same emulation: 0.152, 0.249, 0.258.
FP8_REL = 0.25
FP8_VS_BF16 = 0.9     # summed over all outputs, the FP8 kernels' distance to the emulation against the bf16 route's


def _setup(case):
    from olmoasr_b200 import _core

    torch.manual_seed(0)
    cross = case != "encoder"
    n_blocks = 2 if cross else 1
    blocks = [_core.ResidualAttentionBlock(D, H, cross_attention=cross).cuda() for _ in range(n_blocks)]
    with torch.no_grad():      # LayerNorm affine and biases away from their initial 1 / 0
        for blk in blocks:
            for n, prm in blk.named_parameters():
                if n.endswith("bias") or "_ln." in n:
                    prm.add_(0.1 * torch.randn_like(prm))
    g = torch.Generator(device="cuda").manual_seed(1)
    if case == "encoder":
        B, T, lens, causal = 2, 1500, [1500, 1500], False
    elif case == "decoder_dense":
        B, T, lens, causal = 2, 192, [192, 192], True
    else:
        B, T, lens, causal = 3, 192, [150, 37, 129], True
    N = sum(lens)
    x0 = torch.randn((N, D), device="cuda", generator=g).to(BF)
    xa0 = torch.randn((B, 1500, D), device="cuda", generator=g).to(BF) if cross else None
    dy = torch.randn((N, D), device="cuda", generator=g).to(BF)
    return blocks, cross, n_blocks, B, T, lens, causal, N, x0, xa0, dy


def _run(case, blocks, cross, n_blocks, B, T, lens, causal, N, x0, xa0, dy, fp8, keep=None):
    """One forward + backward of the blocks; keep: a list that receives the block nodes' saved tensors."""
    from olmoasr_b200 import _core
    from olmoasr_b200.fp8 import fp8_autocast

    for blk in blocks:
        blk.zero_grad(set_to_none=True)
    x = x0.clone().requires_grad_(True)
    xa = xa0.clone().requires_grad_(True) if cross else None
    with fp8_autocast(fp8):
        st = {"buf": None, "left": n_blocks} if cross else None
        if case == "encoder":
            h = x.view(B, T, D)
            for blk in blocks:
                h = blk(h)
            y = h.reshape(N, D)
        elif case == "decoder_dense":
            f8 = _core.fp8_inputs(xa) if fp8 else None
            mask = torch.full((T, T), -math.inf, device="cuda").triu_(1)
            h = x.view(B, T, D)
            for blk in blocks:
                h = blk(h, xa, mask=mask, _xa_state=st, _fp8=f8)
            y = h.reshape(N, D)
        else:
            f8 = _core.fp8_inputs(xa) if fp8 else None
            pk = _core.PackedBatch(lens, T, "cuda")
            h = x
            for blk in blocks:
                h = blk(h, xa, _xa_state=st, _packed=pk, _fp8=f8)
            y = h
        if keep is not None:
            node, seen = y.grad_fn, []
            while node is not None and len(seen) < n_blocks:   # _BlockFn nodes, last block first
                if type(node).__name__ == "_BlockFnBackward":
                    seen.append([t.detach().clone() for t in node.saved_tensors])
                nxt = [f for f, _ in node.next_functions if f is not None]
                node = nxt[0] if nxt else None
            keep.extend(reversed(seen))
        y.backward(dy)
    torch.cuda.synchronize()
    out = {"y": y.detach(), "dx": x.grad}
    if cross:
        out["dxa"] = xa.grad
    for i, blk in enumerate(blocks):
        for n, prm in blk.named_parameters():
            out[f"{i}.{n}"] = prm.grad
    return out


@pytest.mark.parametrize("case", ["encoder", "decoder_dense", "decoder_packed"])
def test_fp8_blocks_against_the_fp64_emulation(case):
    blocks, cross, n_blocks, B, T, lens, causal, N, x0, xa0, dy = st = _setup(case)
    got8, got16 = _run(case, *st, fp8=True), _run(case, *st, fp8=False)

    ps = [{n: prm.detach().double().requires_grad_(True) for n, prm in blk.named_parameters()} for blk in blocks]
    x = x0.double().requires_grad_(True)
    xa = xa0.double().requires_grad_(True) if cross else None
    h = x
    for p in ps:
        h = emu_block(p, h, xa, lens, causal, cross)
    h.backward(dy.double())
    want = {"y": h.detach(), "dx": x.grad}
    if cross:
        want["dxa"] = xa.grad
    for i, p in enumerate(ps):
        for n, leaf in p.items():
            want[f"{i}.{n}"] = leaf.grad

    rows = sorted(((_rel(got8[k], want[k]), _rel(got16[k], want[k]), k) for k in want), reverse=True)
    print(f"\n{case}: worst FP8-kernel vs FP8-emulation (and bf16-kernel vs FP8-emulation) relative L2:")
    for r8, r16, k in rows[:6]:
        print(f"  {k:40s} {r8:.3e} ({r16:.3e})")
    assert all(bool(torch.isfinite(v).all()) for v in got8.values())
    assert rows[0][0] <= FP8_REL, rows[0]
    assert sum(r[0] for r in rows) <= FP8_VS_BF16 * sum(r[1] for r in rows)


@pytest.mark.parametrize("case", ["encoder", "decoder_dense", "decoder_packed"])
def test_fp8_block_sites_read_the_right_operands(case, monkeypatch):
    from olmoasr_b200 import kernels as K
    from tests.test_fp8_gpu import _check_fp8

    blocks, cross, n_blocks, B, T, lens, causal, N, x0, xa0, dy = st = _setup(case)
    calls = []
    real = K.gemm_fp8

    def rec(a, a_scale, b, b_scale, M, N_, K_, **kw):
        aux = kw.get("aux")
        before = None if aux is None else aux.clone()     # the in-place RESIDUAL overwrites its aux
        out = real(a, a_scale, b, b_scale, M, N_, K_, **kw)
        calls.append(((a.clone(), a_scale.clone()), (b.clone(), b_scale.clone()), kw.get("epi", K.EPI_BF16),
                      kw.get("bias"), before, tuple(t.clone() for t in out) if isinstance(out, tuple) else out.clone()))
        return out

    monkeypatch.setattr(K, "gemm_fp8", rec)
    saved = []
    _run(case, *st, fp8=True, keep=saved)

    def bits(q8):
        return q8[0].view(torch.uint8), q8[1]

    weights = {}          # (block, site) -> (W8 bits, W^T8 bits)
    for i, blk in enumerate(blocks):
        sh = blk._shadows(BF)
        for k in ("wqkv", "wo", "wcq", "wckv", "wco", "w1", "w2"):
            if k in sh:
                weights[(i, k)] = (bits(K.quantize_fp8_rows(sh[k], 0)), bits(K.quantize_fp8_rows(sh[k], 0, transpose=True)))
    # the quantised forward inputs each site must read, from what each block saved: x, mean1, rstd1, ln1, qkv, ao, lse,
    # x1, [xa, meanc, rstdc, lnc, qc, kvc, co, lsec, x2], mean2, rstd2, ln2, h, g
    inputs = {}
    for i, sv in enumerate(saved):
        ins = {"wqkv": sv[3], "wo": sv[5]}
        if cross:
            ins.update({"wckv": sv[8], "wcq": sv[11], "wco": sv[14]})
        ins.update({"w1": sv[-3], "w2": sv[-1]})
        inputs.update({(i, k): bits(K.quantize_fp8_rows(v, 0)) for k, v in ins.items()})

    def same(u, v):
        return u[0].shape == v[0].shape and torch.equal(u[0], v[0]) and torch.equal(u[1], v[1])

    seen = []
    for a8, b8, epi, bias, aux, out in calls:
        hit = [(key, form) for key, ws in weights.items() for form in (0, 1) if same(bits(b8), ws[form])]
        assert len(hit) == 1, f"a weight operand that is no projection's W8 / W^T8 ({len(hit)} matches)"
        key, form = hit[0]
        fwd = form == 0
        assert a8[0].dtype == (torch.float8_e4m3fn if fwd else torch.float8_e5m2), (key, a8[0].dtype)
        if fwd:
            assert same(bits(a8), inputs[key]), f"{key}: the forward reads another activation than the one saved"
        seen.append((key, "fwd" if fwd else "dgrad"))
        kw = {"bias": bias} if bias is not None else {}
        if aux is not None:
            kw["aux"] = aux
        _check_fp8(out, a8, b8, epi, f"{key} {'fwd' if fwd else 'dgrad'}", **kw)
    want = sorted((key, f) for key in weights for f in ("fwd", "dgrad"))
    assert sorted(seen) == want, (sorted(seen), want)
