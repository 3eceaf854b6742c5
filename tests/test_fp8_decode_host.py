"""fp8 decoding without a GPU: the option's plumbing (engine cache key, NotImplementedError routes, transcribe()'s
per-temperature options), the fp8 `step_bytes` arithmetic, and the fp64 statements of tests/fp8_decode_reference.py
against torch's own float8_e4m3fn dequantisation, including the (key, head, K|V) scale layout of cross K / V."""
import math
import types

import pytest
import torch

from olmoasr_b200 import decoding as D
from tests import decode_reference as dr
from tests import fp8_decode_reference as fr


# ---------------------------------------------------------------------------------------------------- plumbing
class _Eng:
    def __init__(self, dtype, max_batch, fp8):
        self.key, self.max_batch = (dtype, max_batch, fp8), max_batch


def test_decode_engine_cache_key_separates_fp8(monkeypatch):
    """decode_engine(dtype) is still the one 16-bit engine; fp8=True is a separate engine, cached per key."""
    import olmoasr_b200.decode_engine as de
    from olmoasr_b200._core import OLMoASRBase

    monkeypatch.setattr(de, "DecodeEngine", lambda model, dtype, max_batch, fp8=False: _Eng(dtype, max_batch, fp8))
    m = types.SimpleNamespace()
    get = lambda *a, **k: OLMoASRBase.decode_engine(m, *a, **k)   # noqa: E731
    e16 = get(torch.float16)
    assert e16.key == (torch.float16, 64, False)
    assert get(torch.float16) is e16 and get(torch.float16, 64, fp8=False) is e16
    e8 = get(torch.float16, fp8=True)
    assert e8 is not e16 and e8.key == (torch.float16, 64, True) and get(torch.float16, fp8=True) is e8
    assert get(torch.bfloat16, fp8=True).key == (torch.bfloat16, 64, True)


def test_options_field_and_transcribe_keeps_it():
    from olmoasr_b200.transcribe import _options_at

    assert D.DecodingOptions().fp8 is False
    assert [f.name for f in D.DecodingOptions.__dataclass_fields__.values()][-2:] == ["fp16", "fp8"]
    for t in (0.0, 0.4):
        assert _options_at(dict(fp8=True, beam_size=5, best_of=5), t).fp8 is True
        assert _options_at(dict(beam_size=5, best_of=5), t).fp8 is False


class _Model:
    is_multilingual = False

    def __init__(self, engine=True):
        self.dims = types.SimpleNamespace(n_text_ctx=448, n_audio_ctx=1500, n_audio_state=8, n_vocab=51864)
        self.asked = []
        if engine:
            self.decode_engine = self._decode_engine

    def _decode_engine(self, dtype, max_batch=64, *, fp8=False):
        self.asked.append((dtype, fp8))
        return types.SimpleNamespace(max_batch=64, splits_of=lambda rows: __import__("contextlib").nullcontext())

    def encoder(self, mel):
        return torch.zeros(mel.shape[0], 1500, 8)

    def install_kv_cache_hooks(self):
        raise AssertionError("the hook loop must not run with fp8=True")


def test_fp8_without_the_device_decoder_raises(monkeypatch):
    with pytest.raises(NotImplementedError, match="fp8"):
        D.DecodingTask(_Model(engine=False), D.DecodingOptions(fp8=True))
    monkeypatch.setattr(D, "USE_ENGINE", False)          # OASR_DECODE_ENGINE=0
    with pytest.raises(NotImplementedError, match="fp8"):
        D.DecodingTask(_Model(), D.DecodingOptions(fp8=True))
    D.DecodingTask(_Model(), D.DecodingOptions())        # the 16-bit hook loop is still a route


def test_fp8_best_of_above_the_engine_batch_raises():
    m = _Model()
    with pytest.raises(NotImplementedError, match="fp8"):
        D.decode(m, torch.zeros(1, 80, 3000), D.DecodingOptions(fp8=True, temperature=0.5, best_of=65))
    assert m.asked == [(torch.float16, True)]


def test_every_engine_site_asks_for_the_fp8_engine():
    """_window_splits, the greedy / sampling route and beam search all select the engine by (dtype, fp8)."""
    m = _Model()
    task = D.DecodingTask(m, D.DecodingOptions(fp8=True, fp16=False, beam_size=2))
    with task._window_splits((0, [0])):
        pass
    with pytest.raises(Exception):                       # the stub engine has no beam_search: the route is what counts
        task._run_beam_on_device(torch.zeros(1, 1500, 8), None)
    assert m.asked == [(torch.bfloat16, True)] * 2


# ---------------------------------------------------------------------------------------------------- step_bytes
@pytest.mark.parametrize("variant,d,L,H", [("small", 768, 12, 12), ("medium", 1024, 24, 16)])
def test_step_bytes(variant, d, L, H):
    from olmoasr_b200.decode_engine import DecodeEngine

    V, A, t = 51864, 1500, 114
    eng = types.SimpleNamespace(d=d, L=L, H=H, V=V, n_audio_ctx=A)
    for fp8 in (False, True):
        eng.fp8 = fp8
        got = [DecodeEngine.step_bytes(eng, n, t) for n in (1, 64)]
        wb, kvb = (1, 1) if fp8 else (2, 2)
        weights = L * 14 * d * d * wb + (L * 4 * 11 * d if fp8 else 0) + V * d * 2
        cross = L * A * 2 * d * kvb + (L * A * 2 * H * 4 if fp8 else 0)
        per_seq = cross + L * 2 * t * d * 2 + V * 4
        assert got == [weights + n * per_seq for n in (1, 64)]
    eng.fp8 = False
    b16 = DecodeEngine.step_bytes(eng, 64, t)
    eng.fp8 = True
    b8 = DecodeEngine.step_bytes(eng, 64, t)
    assert 1.7 < b16 / b8 < 1.8                          # the block weights and cross K / V dominate at 64 sequences


# ---------------------------------------------------------------------------------------------------- the statements
def test_quantize_rows_matches_torch_and_round_trips():
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(40, 96, generator=g) * torch.logspace(-3, 3, 40)[:, None]).to(torch.bfloat16)
    x[3] = 0
    q, s = fr.quantize_rows(x)
    inv = 448.0 / x.float().abs().amax(1).clamp_min(1e-30)
    inv[3] = 1.0
    assert torch.equal(q.view(torch.uint8), (x.float() * inv[:, None]).to(torch.float8_e4m3fn).view(torch.uint8))
    assert s[3] == 1 and bool((q.float().abs().amax(1)[torch.arange(40) != 3] == 448).all())
    rel = (fr.dequantize(q, s) - x.double()).abs() / x.double().abs().amax(1, keepdim=True).clamp_min(1e-300)
    assert float(rel.max()) <= 2.0 ** -4        # half an e4m3 ulp at the row maximum's exponent


def test_cross_kv_scale_layout():
    """Scale (row, g) belongs to elements [64 g, 64 g + 64) of the row: g < H a key head, g >= H a value head."""
    H, rows = 3, 5
    d = 64 * H
    g = torch.Generator().manual_seed(1)
    kv = torch.randn(rows, 2 * d, generator=g) * torch.arange(1, 2 * H + 1).repeat_interleave(64)
    q, s = fr.quantize_kv(kv.to(torch.bfloat16), H)
    assert q.shape == (rows, 2 * d) and s.shape == (rows, 2 * H)
    for r in range(rows):
        for grp in range(2 * H):
            seg = kv[r, 64 * grp:64 * grp + 64].to(torch.bfloat16).float()
            assert s[r, grp] == seg.abs().max() / 448.0
            assert torch.equal(q[r, 64 * grp:64 * grp + 64].view(torch.uint8),
                               (seg * (448.0 / seg.abs().max())).to(torch.float8_e4m3fn).view(torch.uint8))
    deq = fr.dequantize(q, s, group=64)
    assert torch.equal(deq[:, :64], q[:, :64].double() * s[:, :1].double())
    assert torch.equal(deq[:, d:d + 64], q[:, d:d + 64].double() * s[:, H:H + 1].double())


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("epi", [dr.EPI_STORE, dr.EPI_GELU, dr.EPI_RESIDUAL])
def test_linear_statement_is_the_dequantised_linear(epi, dtype):
    """s_n sum_k x Q_nk is the 16-bit statement on torch's dequantised weight; the fp32 yardstick stays within it."""
    g = torch.Generator().manual_seed(epi)
    M, N, K = 5, 48, 256
    x = torch.randn(M, K, generator=g).to(dtype)
    q, s = fr.quantize_rows((torch.randn(N, K, generator=g) / 16).to(dtype))
    bias, res = 0.3 * torch.randn(N, generator=g), torch.randn(M, N, generator=g).to(dtype)
    ref = fr.linear(x, q, s, bias, dtype, epi=epi, res=res)
    W = q.to(torch.float64) * s.double()[:, None]
    acc = x.double() @ W.t() + dr.rnd(bias.double(), dtype)
    inner = dr.rnd(acc, dtype)
    want = {dr.EPI_STORE: inner, dr.EPI_GELU: dr.gelu(inner), dr.EPI_RESIDUAL: res.double() + inner}[epi]
    assert torch.equal(ref["out"], dr.rnd(want, dtype))
    emu = fr.linear(x, q, s, bias, dtype, epi=epi, res=res, work=torch.float32)
    dr.check_linear(emu["out"], ref, emu, dtype, epi, name="yardstick")


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_attention_statement_is_the_dequantised_attention(dtype):
    """Per (key, head) scales outside the sums equal attention over torch's dequantised K / V at the same rounding
    points, and a K scale moved to the wrong head changes the result."""
    g = torch.Generator().manual_seed(2)
    n, keys, H = 3, 40, 2
    d = 64 * H
    q = torch.randn(n, d, generator=g).to(dtype)
    kv = torch.randn(n * keys, 2 * d, generator=g) * (1 + torch.arange(2 * H).repeat_interleave(64))
    codes, s = fr.quantize_kv(kv.to(torch.bfloat16), H)
    codes, s = codes.view(n, keys, 2 * d), s.view(n, keys, 2 * H)
    got = fr.attention(q, codes[..., :d], s[..., :H], codes[..., d:], s[..., H:], dtype)
    kd = codes[..., :d].double().reshape(n, keys, H, 64) * s[..., :H, None].double()
    vd = codes[..., d:].double().reshape(n, keys, H, 64) * s[..., H:, None].double()
    qs = (q.float() * dr.SCALE).to(dtype).double().view(n, H, 64)
    score = dr.rnd(torch.einsum("nhc,njhc->nhj", qs, kd * dr.SCALE), dtype)
    want = torch.einsum("nhj,njhc->nhc", dr.rnd(torch.softmax(score, -1), dtype), vd).reshape(n, d)
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-12)
    swapped = fr.attention(q, codes[..., :d], s[..., :H].flip(-1), codes[..., d:], s[..., H:], dtype)
    assert not torch.allclose(swapped, want, rtol=1e-3)
    assert math.isfinite(float(got.abs().max()))
