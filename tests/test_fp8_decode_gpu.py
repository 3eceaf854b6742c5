"""fp8 decoding (`DecodingOptions(fp8=True)`) on the device: e4m3 block weights and cross K / V in the decoder step.

  * quantisation: the engine's e4m3 weights, cross K / V and scales are bit-exact against torch's
    `(x.float() * inv).to(torch.float8_e4m3fn)`, and the cross K / V buffer takes half the 16-bit bytes plus its scales;
  * oasr_dec_linear_fp8w at every (x-mode, epilogue) pair of a decoder layer, rows 1 .. 64 (both direct forms and the
    staged one), d = 384 .. 1280, fp16 and bf16, into sentinel-filled outputs, against the fp64 statement of
    tests/fp8_decode_reference.py under decode_reference's rule (the tolerances of the 16-bit parity tests, with one
    more rounding stage for the scale); a row's bits at every row count and position;
  * oasr_dec_attention_fp8kv, fused and split, with beams sharing a clip's K / V, against the fp64 statement;
  * the composed step and greedy decoding on the margin-sharpened models of tests/test_decode_engine_gpu.py: the logits'
    distance from the fp64 unquantised step, argmax agreement where the 16-bit margin exceeds the measured error;
  * determinism, graph replay == eager, transcribe_batch() == transcribe() under fp8, every decode route, and the
    same launches per step as the 16-bit engine.

No checkpoint or speech data exists here, so no word error rate can be stated: what is measured is the logit error and
the token agreement on seeded weights.
"""
import math

import pytest
import torch

from tests import decode_reference as dr
from tests import fp8_decode_reference as fr
from tests import test_decode_parity_gpu as tdp
from tests.test_decode_engine_gpu import SHARPEN, _build

pytestmark = pytest.mark.gpu

DTYPES, DT_ID, WIDTHS, ROWS = tdp.DTYPES, tdp.DT_ID, tdp.WIDTHS, tdp.ROWS
LAYER_SHAPES = ("qkv", "self_out", "cross_q", "cross_out", "fc1", "fc2")   # the launches fp8 quantises (not the logits head)
SOT, NO_TIMESTAMPS = 50257, 50362
# RMS relative error of rounding to a 3-bit mantissa: at most ulp / sqrt(12) of the smallest value of a binade, 2^-3 / sqrt(12)
RHO = 2.0 ** -3 / math.sqrt(12)


def _u8(t):
    return t.contiguous().view(torch.uint8)


def _pair(d, L, dtype, seed):
    """A 16-bit and an fp8 engine over one seeded decoder (tests/test_decode_parity_gpu.py's model)."""
    from olmoasr_b200.decode_engine import DecodeEngine

    eng16 = tdp._engine(d, L, dtype, seed=seed)
    return eng16, DecodeEngine(eng16.model, dtype, 64, fp8=True)


# ---------------------------------------------------------------------------------------------------- quantisation
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_quantised_weights_and_cross_kv_are_bit_exact(dtype):
    from olmoasr_b200._core import _as_bf16_2d, linear_fwd
    from olmoasr_b200.decode_engine import FP8_WEIGHTS

    d, L, n = 768, 2, 3
    eng16, eng8 = _pair(d, L, dtype, seed=5)
    xa = torch.randn(n, 1500, d, device="cuda", generator=torch.Generator(device="cuda").manual_seed(9)).to(torch.bfloat16)
    eng16.prepare(xa)
    eng8.prepare(xa)
    torch.cuda.synchronize()
    rows, H = n * 1500, eng8.H
    for l, blk in enumerate(eng8.model.decoder.blocks):
        lw8, lw16 = eng8._w["layers"][l], eng16._w["layers"][l]
        for name in FP8_WEIGHTS:
            q, s = fr.quantize_rows(lw16[name])
            assert lw8[name].dtype == torch.float8_e4m3fn and lw8[name].shape == lw16[name].shape
            assert torch.equal(_u8(lw8[name]), _u8(q)), f"layer {l} {name} codes"
            assert torch.equal(lw8[name + "_s"], s), f"layer {l} {name} scales"
        wkv, bkv = blk.cross_attn.fused_kv()
        q, s = fr.quantize_kv(linear_fwd(_as_bf16_2d(xa), wkv, bkv), H)
        assert torch.equal(eng8.cross_kv[l][:rows], _u8(q)), f"layer {l} cross K / V codes"
        assert torch.equal(eng8.cross_scale[l][:rows], s), f"layer {l} cross K / V scales"
    assert eng8.cross_kv.dtype == torch.uint8 and 2 * eng8.cross_kv.nbytes == eng16.cross_kv.nbytes
    assert eng8.cross_scale.shape == (L, 64 * 1500, 2 * H) and eng8.cross_scale.dtype == torch.float32


# ---------------------------------------------------------------------------------------------------- dec_linear_fp8w
def _run_fp8(monkeypatch, dtype, M, N, K, x_mode, epi, n_partials, x, q, s, bias, ln, res, pos_value=0):
    """tests/test_decode_parity_gpu.py's sentinel-checked launch, through oasr_dec_linear_fp8w."""
    orig = tdp._linear_fn
    monkeypatch.setattr(tdp, "_linear_fn", lambda dt, pos: (lambda *a, **k: orig(dt, pos)(*a, w_scale=s, **k)))
    try:
        return tdp._run_linear(dtype, M, N, K, x_mode, epi, n_partials, x, q, bias, ln, res, pos_value=pos_value)
    finally:
        monkeypatch.setattr(tdp, "_linear_fn", orig)


def _ref8(dtype, M, x_mode, epi, x, q, s, bias, ln, res):
    xin = x[:, :M] if x_mode == dr.X_PARTIAL_SUM else x[:M]
    kw = dict(x_mode=x_mode, ln=ln, epi=epi, res=res[:M])
    return fr.linear(xin, q, s, bias, dtype, **kw), fr.linear(xin, q, s, bias, dtype, work=torch.float32, **kw)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("d", WIDTHS)
def test_dec_linear_fp8w_every_form_and_mode(d, dtype, monkeypatch):
    shapes = tdp._shapes(d)
    for si, name in enumerate(LAYER_SHAPES):
        N, K, x_mode, epi, n_partials = shapes[name]
        x, W, bias, ln, res = tdp._operands(N, K, x_mode, n_partials, dtype, seed=2000 * d + si)
        q, s = fr.quantize_rows(W)
        for i, M in enumerate(ROWS):
            got = _run_fp8(monkeypatch, dtype, M, N, K, x_mode, epi, n_partials, x, q, s, bias, ln, res,
                           pos_value=(0, 1, tdp.CTX - 1)[i % 3])
            ref, emu = _ref8(dtype, M, x_mode, epi, x, q, s, bias, ln, res)
            dr.check_linear(got, ref, emu, dtype, epi, name=f"fp8 {name} d={d} M={M}")


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("d", [384, 1280])
def test_fp8w_rows_bits_do_not_depend_on_the_row_form(d, dtype, monkeypatch):
    shapes = tdp._shapes(d)
    for si, name in enumerate(LAYER_SHAPES):
        N, K, x_mode, epi, n_partials = shapes[name]
        x, W, bias, ln, res = tdp._operands(N, K, x_mode, n_partials, dtype, seed=88 + si)
        q, s = fr.quantize_rows(W)
        want = None
        for M in ROWS:
            for p in sorted({0, M // 2, M - 1}):
                perm = torch.arange(64, device="cuda")
                perm[0], perm[p] = p, 0
                xp = x[:, perm] if x_mode == dr.X_PARTIAL_SUM else x[perm]
                got = _run_fp8(monkeypatch, dtype, M, N, K, x_mode, epi, n_partials, xp, q, s, bias, ln, res[perm], 2)[p]
                if want is None:
                    want = got
                assert torch.equal(got, want), f"{name}: row bits at M={M}, position {p}"


# ---------------------------------------------------------------------------------------------------- dec_attention_fp8kv
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("n,kv_group", [(7, 1), (10, 5), (64, 1)])
@pytest.mark.parametrize("splits", [1, 3, 8])
def test_dec_attention_fp8kv(splits, n, kv_group, dtype):
    import types

    from olmoasr_b200._lib import DTYPE_BF16, DTYPE_F16
    from olmoasr_b200.decode_engine import DecodeEngine

    d, keys = 768, 1500
    H = d // 64
    clips = -(-n // kv_group)
    g = torch.Generator(device="cuda").manual_seed(31 * n + splits)
    q = torch.randn(64, d, device="cuda", generator=g).to(dtype)
    kv = torch.randn(clips * keys, 2 * d, device="cuda", generator=g) * (1 + torch.arange(2 * d, device="cuda") % 7)
    codes, scales = fr.quantize_kv(kv.to(torch.bfloat16), H)
    codes = _u8(codes)
    sh = types.SimpleNamespace(q=q, scores=torch.zeros(64, H, 1536, device="cuda"), d=d, H=H, pos=None,
                               dt=DTYPE_F16 if dtype == torch.float16 else DTYPE_BF16)
    part = torch.full((splits, n, d), float("nan"), device="cuda")
    DecodeEngine._attention(sh, n, codes, codes[:, d:], keys * 2 * d, 2 * d, part, splits, n_keys=keys, kv_group=kv_group,
                            kv_scales=(scales, scales[:, H:], keys * 2 * H, 2 * H))
    torch.cuda.synchronize()
    got = part[0].clone()
    for s in range(1, splits):
        got += part[s]
    rep = lambda t: t.view(clips, keys, -1).repeat_interleave(kv_group, dim=0)[:n]   # noqa: E731
    cq, cs = rep(codes), rep(scales)
    ref = fr.attention(q[:n], cq[..., :d], cs[..., :H], cq[..., d:], cs[..., H:], dtype)
    dr.check_attention(got, ref, dtype, name=f"fp8 attention n={n} group={kv_group} splits={splits}")


# ---------------------------------------------------------------------------------------------------- the model
@pytest.fixture(scope="module", params=["tiny", "small"])
def sharpened(request):
    m, _, dims, _, xa = _build(request.param, *SHARPEN[request.param])
    return request.param, m, dims, xa


def _teacher_forced_logits(eng, xa, toks):
    """Logits after every replay of a fully teacher-forced prefix: (P - 1, n, V)."""
    n, P = toks.shape
    eng.prepare(xa)
    eng.reset(n, toks, sample_begin=P)
    out = []
    for _ in range(P - 1):
        eng.replay(n)
        out.append(eng.logits[:n].clone())
    return torch.stack(out)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_composed_step_against_the_unquantised_fp64_step(sharpened, dtype):
    """One fp8 step at full depth from a teacher-forced state against the fp64 step with the unquantised 16-bit weights
    and cross K / V (both from the same self-attention cache).

    Bound: rounding to e4m3 leaves each stored element a relative error of RMS at most RHO = 2^-3 / sqrt(12) = 0.036
    (uniform over half an ulp, measured at the smallest mantissa of a binade).  A product sum_k x_k w_k (1 + e_k) with
    independent e_k errs by RHO times ||x w||, which for the unstructured seeded weights is the output's own size.  A
    layer stores 8 such tensors (six projections, cross K and V); if every one of the 8 L contributions reached the
    logits at full size and independently, the logits would err by RHO sqrt(8 L): 0.20 for tiny (L = 4), 0.35 for small
    (L = 12).  Every branch is smaller than the residual stream it joins, so the measured error is well below that; the
    bound is the full-size statement, the printed number the measurement."""
    name, m, dims, xa = sharpened
    L, d, n = dims.n_text_layer, dims.n_text_state, xa.shape[0]
    eng8, eng16 = m.decode_engine(dtype, fp8=True), m.decode_engine(dtype)
    toks = torch.randint(0, 50000, (n, 6), generator=torch.Generator().manual_seed(4), dtype=torch.int32)
    toks[:, 0] = SOT
    eng16.prepare(xa)
    eng8.prepare(xa)
    eng8.reset(n, toks, sample_begin=20)
    for _ in range(4):
        eng8.replay(n)
    pos = int(eng8.pos.item())
    self_k, self_v = eng8.self_k[:, :n, :pos].clone(), eng8.self_v[:, :n, :pos].clone()
    live = {k: getattr(eng8, k).clone() for k in tdp._LIVE}
    eng8._enqueue_step(n)
    torch.cuda.synchronize()
    logits = eng8.logits[:n].clone()
    dec = eng16.model.decoder
    x0 = dr.embed(dec.token_embedding.weight.detach(), dec.positional_embedding.detach(), toks.cuda(), pos, dtype)
    cross = eng16.cross_kv[:, :n * 1500].view(L, n, 1500, 2 * d)
    ref = dr.step(tdp._model_weights(eng16), x0, self_k, self_v, cross, pos, dtype)["logits"]
    rel = (logits.double() - ref).norm(dim=1) / ref.norm(dim=1)
    bound = RHO * math.sqrt(8 * L)
    print(f"{name} {DT_ID[dtype]}: fp8 step logits vs the fp64 unquantised step, relative L2 per row "
          f"max {float(rel.max()):.4f} mean {float(rel.mean()):.4f} (bound {bound:.3f})")
    assert float(rel.max()) <= bound

    for k, t in live.items():                          # graph replay == the eager step, bit for bit
        getattr(eng8, k).copy_(t)
    eng8.replay(n)
    torch.cuda.synchronize()
    assert torch.equal(eng8.logits[:n], logits), "graph replay differs from the eager step"
    eng16.reset(n, toks, sample_begin=20)
    eng16.replay(n)
    assert eng8.launches_per_step == eng16.launches_per_step > 0


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_argmax_agrees_where_the_margin_exceeds_the_error(sharpened, dtype):
    """The 16-bit engine's greedy tokens teacher-forced into both engines: wherever the 16-bit top-1 / top-2 margin
    exceeds twice the largest logit difference measured over the whole run, the fp8 argmax is the same token."""
    name, m, _, xa = sharpened
    eng8, eng16 = m.decode_engine(dtype, fp8=True), m.decode_engine(dtype)
    toks, _, _, _ = eng16.greedy(xa, [SOT, NO_TIMESTAMPS], 40)
    l16 = _teacher_forced_logits(eng16, xa, toks)
    l8 = _teacher_forced_logits(eng8, xa, toks)
    err = float((l8 - l16).abs().max())
    rel = float(((l8 - l16).norm(dim=-1) / l16.norm(dim=-1)).max())
    top2 = l16.topk(2, dim=-1).values
    decided = (top2[..., 0] - top2[..., 1]) > 2 * err
    same = l8.argmax(-1) == l16.argmax(-1)
    g8, _, _, _ = eng8.greedy(xa, [SOT, NO_TIMESTAMPS], 40)
    width = min(g8.shape[1], toks.shape[1])
    tok_agree = float((g8[:, :width] == toks[:, :width]).double().mean())
    print(f"{name} {DT_ID[dtype]}: logits max |diff| {err:.4g}, worst row relative L2 {rel:.4f}; argmax agrees at "
          f"{int(same.sum())}/{same.numel()} positions, {int(decided.sum())} decided by the margin rule; free-running "
          f"greedy tokens equal at {tok_agree:.3f} of positions")
    assert bool(same[decided].all())


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_two_runs_are_bit_identical(sharpened, dtype):
    _, m, _, xa = sharpened
    eng8 = m.decode_engine(dtype, fp8=True)
    a = eng8.greedy(xa, [SOT, NO_TIMESTAMPS], 24)
    b = eng8.greedy(xa, [SOT, NO_TIMESTAMPS], 24)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2])


def test_every_decode_route_runs_in_fp8(sharpened):
    """Greedy, timestamp rules, best_of sampling and beam search through decode(fp8=True) on the fp8 engine."""
    from olmoasr_b200.decoding import DecodingOptions, decode

    _, m, _, xa = sharpened
    for kw in (dict(without_timestamps=True), dict(), dict(temperature=0.5, best_of=3), dict(beam_size=3),
               dict(beam_size=2, fp16=False)):
        torch.manual_seed(0)
        res = decode(m, xa, DecodingOptions(fp8=True, sample_len=24, **kw))
        assert len(res) == xa.shape[0] and all(math.isfinite(r.avg_logprob) for r in res), kw
        assert all(isinstance(t, int) for r in res for t in r.tokens), kw
    assert (torch.float16, 64, True) in m._engines and (torch.bfloat16, 64, True) in m._engines


def test_transcribe_batch_equals_transcribe_in_fp8():
    """Under splits_of, a window decoded inside transcribe_batch() has the bits it has alone in transcribe()."""
    from olmoasr_b200 import synthetic
    from olmoasr_b200.transcribe import transcribe, transcribe_batch
    from tests.test_timing_gpu import SpaceTokenizer
    from tests.test_transcribe_batch_gpu import _compare

    m, _, _, _, _ = _build("tiny", *SHARPEN["tiny"], n_clips=1)
    audios = [synthetic.waveforms(1, rank=r, n_samples=int(s * 16000))[0] for r, s in enumerate((0.5, 71.0, 12.0))]
    tok = SpaceTokenizer()
    for kw in (dict(), dict(without_timestamps=False, beam_size=3, best_of=3)):
        want = [transcribe(m, a, temperature=0.0, sample_len=64, tokenizer=tok, fp8=True, **kw) for a in audios]
        got = transcribe_batch(m, audios, temperature=0.0, sample_len=64, tokenizer=tok, fp8=True, **kw)
        for g, w in zip(got, want):
            _compare(g, w)
    assert (torch.float16, 64, True) in m._engines
