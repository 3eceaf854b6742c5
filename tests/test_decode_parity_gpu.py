"""The device decoder's step (csrc/decode.cu as decode_engine.py wires it) against the fp64 statements of
tests/decode_reference.py, in bf16 and fp16.

  * dec_linear alone: every (x-mode, epilogue) pair the engine issues, at the qkv / out / fc1 / fc2 / logits shapes of
    d = 384 .. 1280 and at 1 .. 64 rows -- both direct forms (<= 16 and 17 .. 32 rows) and the staged form (33 .. 64,
    with K-chunked staging for fc2 and several column groups per CTA for the logits); outputs written into
    sentinel-filled buffers; LayerNorm regimes where one-pass statistics or a missing eps fail; fp16 overflow;
    the QKV scatter at device positions 0, 1 and 447; a row's bits at every row count and row position;
  * dec_embed and oasr_convert: bit-exact;
  * the real step launch by launch: each launch checked from a snapshot of what it read, against the statement built
    from the model's own parameters, so the wiring (LayerNorm, bias, partial-sum layout, cache position, clip of a
    beam) is checked with the arithmetic;
  * the composed step at full depth against the fp64 step; graph replay and programmatic dependent launch bit-exact;
  * prepare(): the cross K / V projection's documented rounding.

prepare() computes cross K / V with the bf16 GEMM and, for an fp16 decoder, converts that bf16 result to fp16 exactly
(decode_engine.py documents this).  Against an fp16-rounded fp64 projection that leaves bf16's resolution: measured on
an H100 SXM (80 GB HBM3, 700 W power limit) at d = 768, 88% of the elements differ and the worst row's relative L2
error is 1.9e-3, about 4 fp16 unit roundoffs (test_prepare_rounding prints it).
"""
import os
import subprocess
import sys
import types

import pytest
import torch

from tests import decode_reference as dr

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DTYPES = [torch.bfloat16, torch.float16]
DT_ID = {torch.bfloat16: "bf16", torch.float16: "fp16"}
WIDTHS = [384, 512, 768, 1024, 1280]
ROWS = [1, 16, 17, 31, 32, 33, 63, 64]
V = 51864
CTX = 448
SENTINEL = -1032.0          # exact in bf16 and fp16


def _code(dtype):
    from olmoasr_b200._lib import DTYPE_BF16, DTYPE_F16

    return DTYPE_F16 if dtype == torch.float16 else DTYPE_BF16


def _linear_fn(dtype, pos):
    """DecodeEngine._linear without a model: the engine's own argument packing."""
    from olmoasr_b200.decode_engine import DecodeEngine

    sh = types.SimpleNamespace(dt=_code(dtype), n_ctx=CTX, pos=pos)
    return lambda *a, **k: DecodeEngine._linear(sh, *a, **k)


def _shapes(d):
    """name -> (N, K, x_mode, epi, n_partials): the launches of one decoder layer and the logits head."""
    return {"qkv": (3 * d, d, dr.X_LAYERNORM, dr.EPI_QKV_SCATTER, 0),
            "self_out": (d, d, dr.X_PARTIAL_SUM, dr.EPI_RESIDUAL, 1),
            "cross_q": (d, d, dr.X_LAYERNORM, dr.EPI_STORE, 0),
            "cross_out": (d, d, dr.X_PARTIAL_SUM, dr.EPI_RESIDUAL, 8),
            "fc1": (4 * d, d, dr.X_LAYERNORM, dr.EPI_GELU, 0),
            "fc2": (d, 4 * d, dr.X_PLAIN, dr.EPI_RESIDUAL, 0),
            "logits": (V, d, dr.X_LAYERNORM, dr.EPI_LOGITS_F32, 0)}


def _operands(N, K, x_mode, n_partials, dtype, seed, rows=64, x_regime=None):
    g = torch.Generator(device="cuda").manual_seed(seed)
    rn = lambda *s: torch.randn(*s, device="cuda", generator=g)   # noqa: E731
    if x_mode == dr.X_PARTIAL_SUM:
        x = rn(n_partials, rows, K) / n_partials ** 0.5
    else:
        x = rn(rows, K)
        if x_regime is not None:
            x = x_regime(x, g)
        x = x.to(dtype)
    W = (rn(N, K) / K ** 0.5).to(dtype)
    bias = 0.5 * rn(N)
    ln = (1 + 0.2 * rn(K), 0.2 * rn(K), 1e-5)
    res = rn(rows, N).to(dtype)
    return x, W, bias, ln, res


def _run_linear(dtype, M, N, K, x_mode, epi, n_partials, x, W, bias, ln, res, pos_value=0):
    """One oasr_dec_linear call of M rows into sentinel-filled buffers: returns the (M, N) result (for QKV_SCATTER
    [q | k row at pos | v row at pos]) after checking that nothing outside it was written."""
    d = N // 3
    pos = torch.tensor([pos_value], device="cuda", dtype=torch.int32)
    lin = _linear_fn(dtype, pos)
    odt = torch.float32 if epi == dr.EPI_LOGITS_F32 else dtype
    width = d if epi == dr.EPI_QKV_SCATTER else N
    buf = torch.full((M + 1, width + 16), SENTINEL, device="cuda", dtype=odt)
    out = buf[:M, :width]
    xin = x[:, :M] if x_mode == dr.X_PARTIAL_SUM else x[:M]
    kw = dict(x_mode=x_mode, ln=ln if x_mode == dr.X_LAYERNORM else None, epi=epi, n_partials=n_partials)
    if epi == dr.EPI_RESIDUAL:                 # in place, as the engine calls it
        out.copy_(res[:M])
        kw["res"] = out
    caches = None
    if epi == dr.EPI_QKV_SCATTER:
        caches = [torch.full((M + 1, CTX, d), SENTINEL, device="cuda", dtype=dtype) for _ in range(2)]
        kw["kv"] = caches
    lin(M, xin.contiguous() if x_mode != dr.X_PARTIAL_SUM else xin, W, None if epi == dr.EPI_LOGITS_F32 else bias, out, **kw)
    torch.cuda.synchronize()
    inside = torch.zeros_like(buf, dtype=torch.bool)
    inside[:M, :width] = True
    assert bool((buf[~inside] == SENTINEL).all()), "written outside the output"
    got = out.clone()
    if caches is not None:
        rows = [c[:M, pos_value].clone() for c in caches]
        for c in caches:
            c[:M, pos_value] = SENTINEL
            assert bool((c == SENTINEL).all()), "cache written outside rows [row, pos]"
        got = torch.cat([got] + rows, dim=1)
    return got


def _ref(dtype, M, x_mode, epi, x, W, bias, ln, res):
    xin = x[:, :M] if x_mode == dr.X_PARTIAL_SUM else x[:M]
    kw = dict(x_mode=x_mode, ln=ln, epi=epi, res=res[:M])
    b = None if epi == dr.EPI_LOGITS_F32 else bias
    return dr.linear(xin, W, b, dtype, **kw), dr.linear(xin, W, b, dtype, work=torch.float32, **kw)


# ---------------------------------------------------------------------------------------------------- dec_linear
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("d", WIDTHS)
def test_dec_linear_every_form_and_mode(d, dtype):
    """Every launch shape of a decoder layer and the logits head, at row counts on both sides of each form's edge."""
    for s, (name, (N, K, x_mode, epi, n_partials)) in enumerate(_shapes(d).items()):
        ops = _operands(N, K, x_mode, n_partials, dtype, seed=1000 * d + s)
        for i, M in enumerate(ROWS):
            pos_value = (0, 1, CTX - 1)[i % 3]
            got = _run_linear(dtype, M, N, K, x_mode, epi, n_partials, *ops, pos_value=pos_value)
            ref, emu = _ref(dtype, M, x_mode, epi, *ops)
            dr.check_linear(got, ref, emu, dtype, epi, name=f"{name} d={d} M={M}")


def _mean_gg_std(x, g):
    return 50.0 + x


def _near_constant(x, g):          # variance ~ 1e-5: comparable to eps
    return 1.0 + 2.0 ** -7 * torch.sign(x)


REGIMES = {"mean_gg_std": _mean_gg_std, "near_constant": _near_constant}


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("regime", ["mean_gg_std", "near_constant", "gamma_zeros"])
def test_dec_linear_layer_norm_regimes(regime, dtype):
    """Rows of mean 50 and std 1 (one-pass statistics lose the variance), rows whose variance is about eps, and
    gamma with zeros; at a direct and the staged form, at the smallest and the widest LayerNorm."""
    for d in (384, 1280):
        for name in ("qkv", "fc1", "logits"):
            N, K, x_mode, epi, n_partials = _shapes(d)[name]
            x, W, bias, ln, res = _operands(N, K, x_mode, n_partials, dtype, seed=d, x_regime=REGIMES.get(regime))
            if regime == "gamma_zeros":
                ln = (ln[0] * (torch.arange(K, device="cuda") % 5 != 0), ln[1], ln[2])
            for M in (1, 17, 64):
                got = _run_linear(dtype, M, N, K, x_mode, epi, n_partials, x, W, bias, ln, res, pos_value=3)
                ref, emu = _ref(dtype, M, x_mode, epi, x, W, bias, ln, res)
                dr.check_linear(got, ref, emu, dtype, epi, name=f"{regime} {name} d={d} M={M}")


@pytest.mark.parametrize("M", [1, 17, 64])
def test_dec_linear_fp16_residual_overflow(M):
    """fp16 residual sums beyond 65504 give +-inf, like the reference's fp16 add."""
    dtype, d = torch.float16, 768
    N, K = d, 4 * d
    x, W, bias, ln, res = _operands(N, K, dr.X_PLAIN, 0, dtype, seed=5)
    W = (W.float() * 600).to(dtype)                         # outputs ~ N(0, 600^2): res + y crosses 65504 for some
    res = (torch.sign(res.float()) * 65000).to(dtype)
    got = _run_linear(dtype, M, N, K, dr.X_PLAIN, dr.EPI_RESIDUAL, 0, x, W, bias, ln, res)
    ref, emu = _ref(dtype, M, dr.X_PLAIN, dr.EPI_RESIDUAL, x, W, bias, ln, res)
    assert bool(torch.isinf(ref["out"]).any()) and bool(torch.isfinite(ref["out"]).any())
    dr.check_linear(got, ref, emu, dtype, dr.EPI_RESIDUAL, name=f"overflow M={M}")


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("pos_value", [0, 1, CTX - 1])
def test_qkv_scatter_positions(pos_value, dtype):
    """The K / V rows land at [row, pos] of the first M rows of each cache and nowhere else (checked inside
    _run_linear), and match the statement."""
    d = 512
    N, K, x_mode, epi, n_partials = _shapes(d)["qkv"]
    ops = _operands(N, K, x_mode, n_partials, dtype, seed=7)
    for M in (1, 17, 33, 64):
        got = _run_linear(dtype, M, N, K, x_mode, epi, n_partials, *ops, pos_value=pos_value)
        ref, emu = _ref(dtype, M, x_mode, epi, *ops)
        dr.check_linear(got, ref, emu, dtype, epi, name=f"qkv pos={pos_value} M={M}")


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("d", [384, 1280])
def test_a_rows_bits_do_not_depend_on_the_row_form(d, dtype):
    """One row's outputs have the same bits at every row count and at every row position (first, middle, last): the
    three forms sum k in the same order, which transcribe_batch()'s equal-bits promise rests on."""
    for s, (name, (N, K, x_mode, epi, n_partials)) in enumerate(_shapes(d).items()):
        x, W, bias, ln, res = _operands(N, K, x_mode, n_partials, dtype, seed=77 + s)
        want = None
        for M in ROWS:
            for p in sorted({0, M // 2, M - 1}):
                perm = torch.arange(64, device="cuda")
                perm[0], perm[p] = p, 0                 # row 0 of the operands sits at position p
                xp = x[:, perm] if x_mode == dr.X_PARTIAL_SUM else x[perm]
                got = _run_linear(dtype, M, N, K, x_mode, epi, n_partials, xp, W, bias, ln, res[perm], pos_value=2)[p]
                if want is None:
                    want = got
                assert torch.equal(got, want), f"{name}: row bits at M={M}, position {p}"


# ---------------------------------------------------------------------------------------------------- embed, convert
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_dec_embed_is_bit_exact(dtype):
    from olmoasr_b200._lib import call, ptr, stream

    n, d = 7, 768
    g = torch.Generator(device="cuda").manual_seed(3)
    emb = torch.randn(V, d, device="cuda", generator=g) * 0.3
    pos_emb = torch.randn(CTX, d, device="cuda", generator=g)
    tokens = torch.randint(0, V, (n, CTX + 2), device="cuda", generator=g, dtype=torch.int32)
    tokens[1] = V                  # out of range: row 0
    tokens[2] = -1
    tokens[3] = V - 1
    for p in (0, 5, CTX - 1):
        pos = torch.tensor([p], device="cuda", dtype=torch.int32)
        x = torch.full((n + 1, d), SENTINEL, device="cuda", dtype=dtype)
        call("oasr_dec_embed", ptr(tokens), tokens.stride(0), ptr(pos), ptr(emb), ptr(pos_emb), ptr(x), n, d, V,
             _code(dtype), stream())
        torch.cuda.synchronize()
        assert torch.equal(x[:n], dr.embed(emb, pos_emb, tokens, p, dtype)), p
        assert bool((x[n] == SENTINEL).all())


def _special_values(src, n, seed):
    """n values of type src: random bit patterns (NaN, inf, subnormals, overflow), normal values and exact ties."""
    g = torch.Generator().manual_seed(seed)
    if src == torch.float32:
        bits = torch.randint(-2 ** 31, 2 ** 31, (n,), generator=g, dtype=torch.int64).to(torch.int32)
        v = bits.view(torch.float32).clone()
        k = n // 4
        v[:k] = torch.randn(k, generator=g) * 1000
        # exact ties of bf16 (low 16 bits 0x8000) and of fp16 (low 13 bits 0x1000) over the fp16 range (exponents -24 .. 15)
        t = (torch.randint(0, 2, (k,), generator=g) << 31) | (torch.randint(103, 143, (k,), generator=g) << 23) | \
            torch.randint(0, 2 ** 23, (k,), generator=g)
        half = k // 2
        t[:half] = (t[:half] & ~0xFFFF) | 0x8000
        t[half:] = (t[half:] & ~0x1FFF) | 0x1000
        t = t - ((t >> 31) & 1) * 2 ** 32
        v[k:2 * k] = t.to(torch.int32).view(torch.float32)
    else:
        bits = torch.randint(-2 ** 15, 2 ** 15, (n,), generator=g, dtype=torch.int32).to(torch.int16)
        v = bits.view(src).clone()
        k = n // 4
        v[:k] = (torch.randn(k, generator=g) * 100).to(src)
    specials = torch.tensor([0.0, -0.0, float("inf"), -float("inf"), float("nan"), 65504.0, 65520.0, -65536.0, 1e5,
                             2.0 ** -24, 2.0 ** -25, 3 * 2.0 ** -26, 2.0 ** -14, 2.0 ** -126, 2.0 ** -133, 1e-40])
    m = min(n, specials.numel())
    v[:m] = specials[:m].to(src)
    return v


@pytest.mark.parametrize("n", [1, 257, 2 ** 20 + 3])
@pytest.mark.parametrize("pair", [("f32", "f16"), ("f32", "bf16"), ("bf16", "f16"), ("f16", "bf16"), ("bf16", "f32"),
                                  ("f16", "f32")], ids="-".join)
def test_convert_is_bit_exact(pair, n):
    """oasr_convert (refresh_weights' cast of every decoder weight) against torch .to(): the same bits, NaN for NaN."""
    from olmoasr_b200 import kernels as K

    T = {"f32": torch.float32, "bf16": torch.bfloat16, "f16": torch.float16}
    src, dst = T[pair[0]], T[pair[1]]
    x = _special_values(src, n, seed=n).cuda()
    got = K.convert(x, dtype=dst)
    torch.cuda.synchronize()
    want = x.to(dst)
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(got), nan)
    ib = torch.int32 if dst == torch.float32 else torch.int16
    assert torch.equal(got[~nan].view(ib), want[~nan].view(ib))


def test_convert_rejects_an_unsupported_pair():
    from olmoasr_b200 import kernels as K
    from olmoasr_b200._lib import OasrError

    x = torch.ones(16, device="cuda")
    with pytest.raises(OasrError, match="unsupported"):
        K.convert(x, dtype=torch.float32)
    with pytest.raises(OasrError, match="unsupported"):
        K.convert(x.to(torch.bfloat16), dtype=torch.bfloat16)


# ---------------------------------------------------------------------------------------------------- the real step
def _engine(d, L, dtype, seed=0):
    """A DecodeEngine over a seeded text decoder of width d and L layers (n_vocab 51864, 448 positions), its LayerNorm
    affine parameters, biases and positional embedding randomised so that every one of them matters."""
    from olmoasr_b200._core import TextDecoder
    from olmoasr_b200.config.model_dims import ModelDimensions
    from olmoasr_b200.decode_engine import DecodeEngine

    torch.manual_seed(seed)
    dec = TextDecoder(V, CTX, d, d // 64, L, train_vocab_pad=False)
    with torch.no_grad():
        dec.positional_embedding.normal_(0, 0.1)
        for name, p in dec.named_parameters():
            if name.endswith("ln.weight") or name.endswith("_ln.weight"):
                p.copy_(1 + 0.2 * torch.randn_like(p))
            elif name.endswith(".bias"):
                p.copy_(0.2 * torch.randn_like(p))
    dims = ModelDimensions(n_mels=80, n_audio_ctx=1500, n_audio_state=d, n_audio_head=d // 64, n_audio_layer=1,
                           n_vocab=V, n_text_ctx=CTX, n_text_state=d, n_text_head=d // 64, n_text_layer=L)
    model = types.SimpleNamespace(decoder=dec.cuda(), dims=dims)
    return DecodeEngine(model, dtype, 64)


def _start(eng, n, kv_group, prefix, seed):
    """prepare() over random features of n / kv_group clips, then a teacher-forced prefix of `prefix` positions:
    the step that follows runs at position `prefix`."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    clips = n // kv_group
    xa = torch.randn(clips, 1500, eng.d, device="cuda", generator=g).to(torch.bfloat16)
    eng.prepare(xa)
    tok = torch.randint(0, 50000, (n, prefix + 1), generator=torch.Generator().manual_seed(seed), dtype=torch.int32)
    eng.reset(n, tok, sample_begin=prefix + 5)
    eng._group = kv_group
    for _ in range(prefix):
        eng._enqueue_step(n)
    torch.cuda.synchronize()
    assert int(eng.pos.item()) == prefix
    return tok


def _layer_params(blk, dtype):
    """The statement's operands of one decoder layer, taken from the model (not from the engine's cast buffers)."""
    a, c = blk.attn, blk.cross_attn
    W = lambda m: m.weight.detach().to(dtype)   # noqa: E731
    b = lambda m: m.bias.detach().float()       # noqa: E731
    ln = lambda m: (m.weight.detach().float(), m.bias.detach().float(), m.eps)   # noqa: E731
    d = a.query.weight.shape[0]
    return dict(wqkv=torch.cat([W(a.query), W(a.key), W(a.value)]),
                bqkv=torch.cat([b(a.query), torch.zeros(d, device=a.query.weight.device), b(a.value)]),
                wo=W(a.out), bo=b(a.out), wcq=W(c.query), bcq=b(c.query), wco=W(c.out), bco=b(c.out),
                w1=W(blk.mlp[0]), b1=b(blk.mlp[0]), w2=W(blk.mlp[2]), b2=b(blk.mlp[2]),
                ln1=ln(blk.attn_ln), lnc=ln(blk.cross_attn_ln), ln2=ln(blk.mlp_ln))


def _model_weights(eng):
    dec, T = eng.model.decoder, eng.dtype
    return dict(layers=[_layer_params(blk, T) for blk in dec.blocks], emb_t=dec.token_embedding.weight.detach().to(T),
                ln=(dec.ln.weight.detach().float(), dec.ln.bias.detach().float(), dec.ln.eps))


class _LaunchChecker:
    """Wraps an engine's _linear and _attention for one step: before each launch it synchronises and snapshots what
    the launch reads; after it, what the launch wrote; then it checks the launch against the statement of the launch
    the step should issue at that point, with the operands taken from the model and the inputs from the previous
    launches' snapshots."""

    def __init__(self, eng, n, kv_group, tokens):
        from olmoasr_b200.decode_engine import DecodeEngine

        self.eng, self.n, self.kv_group, self.dtype = eng, n, kv_group, eng.dtype
        self.w = _model_weights(eng)
        self.pos = int(eng.pos.item())
        self.tokens = tokens
        self.plan = []
        for l, lw in enumerate(self.w["layers"]):
            self.plan += [("qkv", l, lw), ("self", l, None), ("self_out", l, lw), ("cross_q", l, lw), ("cross", l, None),
                          ("cross_out", l, lw), ("fc1", l, lw), ("fc2", l, lw)]
        self.plan.append(("logits", None, self.w))
        self.x = self.h = self.q = self.part = None
        self.checked = []
        self._lin, self._att = DecodeEngine._linear, DecodeEngine._attention
        eng._linear, eng._attention = self.linear, self.attention

    def close(self):
        del self.eng._linear, self.eng._attention

    def _name(self, what, l):
        return f"{what} layer {l} n={self.n}" if l is not None else f"{what} n={self.n}"

    def attention(self, n, k, v, seq_stride, row_stride, part, splits, n_keys=None, kv_group=1):
        what, l, _ = self.plan.pop(0)
        assert what in ("self", "cross"), f"expected {what}, got an attention launch"
        eng, T, d = self.eng, self.dtype, self.eng.d
        torch.cuda.synchronize()
        q = eng.q[:n].clone()
        assert torch.equal(q, self.q), "attention: q is not the last projection's output"
        self._att(eng, n, k, v, seq_stride, row_stride, part, splits, n_keys, kv_group)
        torch.cuda.synchronize()
        if what == "self":
            kc, vc = eng.self_k[l][:n, :self.pos + 1], eng.self_v[l][:n, :self.pos + 1]
        else:
            clips = -(-n // self.kv_group)
            ckv = eng.cross_kv[l][:clips * eng.n_audio_ctx].view(clips, eng.n_audio_ctx, 2 * d)
            ckv = ckv.repeat_interleave(self.kv_group, dim=0)[:n]
            kc, vc = ckv[..., :d], ckv[..., d:]
        self.part = part.clone()
        got = self.part[0].clone()
        for s in range(1, splits):             # the consumer adds the fp32 partials in split order
            got += self.part[s]
        dr.check_attention(got, dr.attention(q, kc, vc, T), T, name=self._name(what, l))
        self.checked.append(what)

    def linear(self, n, x, W, bias, out, *, x_mode=0, ln=None, epi=0, res=None, n_partials=0, kv=None, K_=None):
        what, l, lw = self.plan.pop(0)
        eng, T, d = self.eng, self.dtype, self.eng.d
        torch.cuda.synchronize()
        if self.x is None:                     # the first launch reads dec_embed's output
            self.x = eng.x[:n].clone()
            emb, pos_emb = eng.model.decoder.token_embedding.weight.detach(), eng.model.decoder.positional_embedding.detach()
            assert torch.equal(self.x, dr.embed(emb, pos_emb, self.tokens.cuda(), self.pos, T)), "dec_embed"
        caches = [c.clone() for c in kv] if kv is not None else None
        if x_mode == dr.X_PARTIAL_SUM:          # the partials the previous attention launch wrote, all of them
            assert n_partials == self.part.shape[0] and torch.equal(x, self.part), f"{what}: not the attention's partials"
        self._lin(eng, n, x, W, bias, out, x_mode=x_mode, ln=ln, epi=epi, res=res, n_partials=n_partials, kv=kv, K_=K_)
        torch.cuda.synchronize()
        key = {"qkv": ("wqkv", "bqkv", "ln1"), "self_out": ("wo", "bo", None), "cross_q": ("wcq", "bcq", "lnc"),
               "cross_out": ("wco", "bco", None), "fc1": ("w1", "b1", "ln2"), "fc2": ("w2", "b2", None),
               "logits": ("emb_t", None, "ln")}[what]
        Wm, bm, lnm = lw[key[0]], (lw[key[1]] if key[1] else None), (lw[key[2]] if key[2] else None)
        mode, ep = {"qkv": (dr.X_LAYERNORM, dr.EPI_QKV_SCATTER), "self_out": (dr.X_PARTIAL_SUM, dr.EPI_RESIDUAL),
                    "cross_q": (dr.X_LAYERNORM, dr.EPI_STORE), "cross_out": (dr.X_PARTIAL_SUM, dr.EPI_RESIDUAL),
                    "fc1": (dr.X_LAYERNORM, dr.EPI_GELU), "fc2": (dr.X_PLAIN, dr.EPI_RESIDUAL),
                    "logits": (dr.X_LAYERNORM, dr.EPI_LOGITS_F32)}[what]
        assert (x_mode, epi) == (mode, ep), f"{what}: launched as x-mode {x_mode}, epilogue {epi}"
        src = {dr.X_PARTIAL_SUM: self.part, dr.X_PLAIN: self.h}.get(mode, self.x)
        kw = dict(x_mode=mode, ln=lnm, epi=ep, res=self.x)
        ref = dr.linear(src, Wm, bm, T, **kw)
        emu = dr.linear(src, Wm, bm, T, work=torch.float32, **kw)
        if ep == dr.EPI_QKV_SCATTER:
            q = eng.q[:n].clone()
            rows = [c[:n, self.pos].clone() for c in kv]
            for before, after in zip(caches, kv):
                after = after.clone()
                after[:n, self.pos] = before[:n, self.pos]
                assert torch.equal(after, before), f"{what}: cache changed outside rows [row, pos]"
            got = torch.cat([q] + rows, dim=1)
            self.q = q
        elif ep == dr.EPI_LOGITS_F32:
            got = eng.logits[:n].clone()
        else:
            dst = {"self_out": eng.x, "cross_out": eng.x, "fc2": eng.x, "cross_q": eng.q, "fc1": eng.h}[what]
            got = dst[:n].clone()
            if what == "cross_q":
                self.q = got
            elif what == "fc1":
                self.h = got
            else:
                self.x = got
        dr.check_linear(got, ref, emu, T, ep, name=self._name(what, l))
        self.checked.append(what)


def _launch_by_launch(eng, n, kv_group, seed):
    tok = _start(eng, n, kv_group, prefix=3, seed=seed)
    chk = _LaunchChecker(eng, n, kv_group, tok)
    try:
        eng._enqueue_step(n)
        torch.cuda.synchronize()
    finally:
        chk.close()
    assert not chk.plan, f"launches not issued: {chk.plan}"
    assert len(chk.checked) == 8 * eng.L + 1


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("d", WIDTHS)
def test_step_launch_by_launch(d, dtype):
    """Every launch of a 2-layer step, at 1 .. 64 rows, and with five beams per clip at 10 and 20 rows."""
    eng = _engine(d, 2, dtype, seed=d)
    for n in (1, 5, 17, 33, 64):
        _launch_by_launch(eng, n, 1, seed=n)
    for n in (10, 20):
        _launch_by_launch(eng, n, 5, seed=n)


_LIVE = ("pos", "tokens", "sum_logprobs", "no_speech", "n_unfinished", "done", "sample_counters")


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("n", [5, 64])
@pytest.mark.parametrize("variant", ["small", "medium"])
def test_composed_step(variant, n, dtype):
    """One step at full depth from a teacher-forced state: the logits of every row and the K / V rows appended at pos
    against the fp64 step; the replayed graph's logits equal the eager step's bit for bit."""
    d, L = {"small": (768, 12), "medium": (1024, 24)}[variant]
    eng = _engine(d, L, dtype, seed=L)
    tok = _start(eng, n, 1, prefix=4, seed=11)
    pos = int(eng.pos.item())
    live = {k: getattr(eng, k).clone() for k in _LIVE}
    self_k = eng.self_k[:, :n, :pos].clone()
    self_v = eng.self_v[:, :n, :pos].clone()
    cross = eng.cross_kv[:, :n * 1500].view(L, n, 1500, 2 * d)
    eng._enqueue_step(n)
    torch.cuda.synchronize()
    logits = eng.logits[:n].clone()
    k_new, v_new = eng.self_k[:, :n, pos].clone(), eng.self_v[:, :n, pos].clone()

    w = _model_weights(eng)
    dec = eng.model.decoder
    x0 = dr.embed(dec.token_embedding.weight.detach(), dec.positional_embedding.detach(), tok.cuda(), pos, dtype)
    ref = dr.step(w, x0, self_k, self_v, cross, pos, dtype)
    emu = dr.step(w, x0, self_k, self_v, cross, pos, dtype, work=torch.float32)
    name = f"{variant} n={n}"
    dr.check_rows(logits, ref["logits"], emu["logits"], dtype, name=name + " logits")
    for key, got in (("k", k_new), ("v", v_new)):
        dr.check_rows(got.reshape(L * n, d), torch.cat(ref[key]), torch.cat(emu[key]), dtype, name=f"{name} {key}")

    for k, t in live.items():
        getattr(eng, k).copy_(t)
    eng.replay(n)
    torch.cuda.synchronize()
    assert torch.equal(eng.logits[:n], logits), "graph replay differs from the eager step"


_PDL_SCRIPT = """
import sys, torch
sys.path.insert(0, {root!r})
from tests.test_decode_parity_gpu import _engine, _start
eng = _engine(512, 4, torch.float16, seed=4)
_start(eng, 9, 1, prefix=0, seed=3)
for _ in range(6):
    eng.replay(9)
torch.cuda.synchronize()
torch.save(eng.logits[:9].cpu(), {out!r})
"""


def test_programmatic_dependent_launch_keeps_the_bits(tmp_path):
    """OASR_DEC_PDL=1 (read once per process) lets each step kernel start under its predecessor's tail: the replayed
    graph's logits equal the default launch's bit for bit."""
    outs = []
    for flag in ("0", "1"):
        out = str(tmp_path / f"logits_pdl{flag}.pt")
        env = dict(os.environ, OASR_DEC_PDL=flag)
        subprocess.run([sys.executable, "-c", _PDL_SCRIPT.format(root=ROOT, out=out)], cwd=ROOT, env=env, check=True,
                       timeout=600)
        outs.append(torch.load(out))
    assert torch.equal(outs[0], outs[1])


def test_prepare_rounding():
    """prepare(): cross K / V is round_bf16(xa W^T + round_bf16(b)) from the bf16 GEMM (held to the dec_linear rule with
    the GEMM's K/16 accumulation stages), and an fp16 decoder's cross K / V is exactly that bf16 result converted."""
    d, L, n = 768, 2, 3
    eng16 = _engine(d, L, torch.bfloat16, seed=5)
    g = torch.Generator(device="cuda").manual_seed(9)
    xa = torch.randn(n, 1500, d, device="cuda", generator=g).to(torch.bfloat16)
    eng16.prepare(xa)
    engh = _engine(d, L, torch.float16, seed=5)
    engh.prepare(xa)
    torch.cuda.synchronize()
    rows = n * 1500
    for l, blk in enumerate(eng16.model.decoder.blocks):
        c = blk.cross_attn
        W = torch.cat([c.key.weight, c.value.weight]).detach().to(torch.bfloat16)
        b = torch.cat([torch.zeros(d, device="cuda"), c.value.bias.detach().float()])
        got = eng16.cross_kv[l][:rows]
        ref = dr.linear(xa.view(rows, d), W, b, torch.bfloat16, stages=d // 16 + 2)
        emu = dr.linear(xa.view(rows, d), W, b, torch.bfloat16, work=torch.float32)
        dr.check_linear(got, ref, emu, torch.bfloat16, dr.EPI_STORE, name=f"prepare layer {l}")
        assert torch.equal(engh.cross_kv[l][:rows], got.to(torch.float16)), "fp16 cross K / V is not the converted bf16 result"
        # the documented gap: the distance of the fp16 decoder's cross K / V from an fp16-rounded projection
        f16 = dr.linear(xa.view(rows, d), W, b, torch.float16)["out"]
        h = engh.cross_kv[l][:rows].double()
        differ = float((h != f16).double().mean())
        rel = float(((h - f16).norm(dim=1) / f16.norm(dim=1)).max())
        dr._report(kind="prepare", name=f"layer {l}", share_differing=differ, worst_row_rel=rel)
        print(f"prepare layer {l}: fp16 cross K/V vs an fp16-rounded projection: {differ:.3f} of elements differ, "
              f"worst row relative L2 {rel:.3g}")
