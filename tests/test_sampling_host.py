"""Temperature sampling and greedy decoding with timestamp rules, on the CPU.

A numpy restatement of the device sampler (csrc/decode.cu dec_sample_kernel with SAMPLING): Philox4x32-10 keyed on the
row's 64-bit key and counted with (vocabulary id / 4, position), Gumbel-max over the filtered row at temperature T.  It is
checked here against softmax(x / T) by a chi-square test, and it is the reference the GPU tests compare the kernel's ids
with (tests/test_sampling_gpu.py).  Then the routing of DecodingTask.run to the device decoder, against a stub model with
a recording `decode_engine`.
"""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch
from scipy import stats

from olmoasr_b200 import decoding as D

V = 51864
EOT, SOT, NO_TIMESTAMPS, TB = D.EOT, D.SOT, D.NO_TIMESTAMPS, D.TIMESTAMP_BEGIN
_M32, _M64 = (1 << 32) - 1, (1 << 64) - 1


# ---- the restatement ---------------------------------------------------------------------------------------------------
def splitmix64(x: int) -> int:
    x = (x + 0x9E3779B97F4A7C15) & _M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & _M64
    return x ^ (x >> 31)


def row_key(seed: int, clip: int, sample: int) -> int:
    return splitmix64(splitmix64(splitmix64(seed & _M64) ^ clip) ^ sample)


def philox4x32_10(c0, c1, k0, k1):
    """Philox4x32-10 on broadcastable uint arrays (counter words 2, 3 are zero); returns (..., 4) uint64 words < 2^32."""
    c0, c1 = np.asarray(c0, np.uint64), np.asarray(c1, np.uint64)
    k0, k1 = np.asarray(k0, np.uint64), np.asarray(k1, np.uint64)
    c0, c1, k0, k1 = np.broadcast_arrays(c0, c1, k0, k1)
    c2, c3 = np.zeros_like(c0), np.zeros_like(c0)
    m32 = np.uint64(_M32)
    for r in range(10):
        if r:
            k0, k1 = (k0 + np.uint64(0x9E3779B9)) & m32, (k1 + np.uint64(0xBB67AE85)) & m32
        p0, p1 = np.uint64(0xD2511F53) * c0, np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & m32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & m32
    return np.stack([c0, c1, c2, c3], axis=-1)


def gumbel(keys, pos, ids):
    """g[d, i] for row key keys[d] at position pos (scalar or (D,)) and vocabulary id ids[i], in fp32 as the kernel."""
    keys = np.asarray([k & _M64 for k in keys], dtype=np.uint64)[:, None]
    ids = np.asarray(ids, dtype=np.int64)[None, :]
    pos = np.asarray(pos, dtype=np.uint64).reshape(-1, 1)
    words = philox4x32_10(ids >> 2, pos, keys & np.uint64(_M32), keys >> np.uint64(32))
    bits = np.take_along_axis(words, np.broadcast_to(ids & 3, words.shape[:-1])[..., None].astype(np.int64), -1)[..., 0]
    u = ((bits >> np.uint64(9)).astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -23)
    return -np.log(-np.log(u))


def sample_ids(filtered, keys, pos, temperature):
    """Gumbel-max over the allowed ids (finite entries of `filtered`, (D, V) or (V,)), lowest id on ties.  Returns (ids,
    margins): the margin between the best and second-best perturbed value says how far rounding is from flipping a draw."""
    x = np.atleast_2d(np.asarray(filtered, dtype=np.float32))
    if x.shape[0] == 1 and len(keys) > 1:
        x = np.repeat(x, len(keys), axis=0)
    ids, margins = [], []
    for d in range(x.shape[0]):
        live = np.nonzero(np.isfinite(x[d]))[0]
        y = x[d, live] / np.float32(temperature) + gumbel([keys[d]], np.atleast_1d(pos)[d % np.size(pos)], live)[0]
        order = np.argsort(-y, kind="stable")
        ids.append(int(live[order[0]]))
        margins.append(float(y[order[0]] - y[order[1]]) if len(live) > 1 else math.inf)
    return np.array(ids), np.array(margins)


def filter_row(logits, tokens, sample_begin, suppress, timestamps, mi, suppress_blank=True):
    """The filtered logits of DecodingTask._main_loop (the hook loop's own rules, the mass rule included): -inf = banned."""
    lg = logits.clone().float()
    if suppress_blank and tokens.shape[1] == sample_begin:
        lg[:, [D.BLANK, EOT]] = -math.inf
    lg[:, list(suppress)] = -math.inf
    if timestamps:
        D._TimestampRules(sample_begin, mi).apply(lg, tokens)
    return lg


# ---- the restatement samples softmax(x / T) ----------------------------------------------------------------------------
LIVE = [11, 300, 301, 302, 7000, 7003, 40000, 51000]


@pytest.mark.parametrize("temperature", [0.5, 1.0])
def test_keyed_gumbel_max_samples_softmax_over_t(temperature):
    x = np.full(V, -np.inf, dtype=np.float32)
    x[LIVE] = np.array([1.0, 0.2, -0.5, 0.7, 1.3, -1.0, 0.0, 0.4], dtype=np.float32)
    n = 4000
    keys = [row_key(1234, c, j) for c in range(n // 5) for j in range(5)]
    pos = np.arange(n) % 37 + 3
    ids, _ = sample_ids(x, keys, pos, temperature)
    assert set(ids.tolist()) <= set(LIVE)
    p = torch.softmax(torch.from_numpy(x[LIVE].astype(np.float64)) / temperature, 0).numpy()
    counts = np.array([(ids == v).sum() for v in LIVE])
    chi = stats.chisquare(counts, p * n)
    assert chi.pvalue > 1e-3, (counts, p * n, chi)


def test_draws_are_a_function_of_key_position_and_id_only():
    x = np.random.default_rng(0).standard_normal(V).astype(np.float32) * 3
    keys = [row_key(9, c, 0) for c in range(6)]
    a, _ = sample_ids(x, keys, 5, 1.0)
    b, _ = sample_ids(x, keys[::-1], 5, 1.0)
    assert a.tolist() == b[::-1].tolist()                   # the row's slot does not matter
    c, _ = sample_ids(x, keys, 6, 1.0)
    assert a.tolist() != c.tolist()                         # the position does
    assert row_key(9, 0, 0) != row_key(9, 0, 1) != row_key(9, 1, 0) != row_key(10, 0, 0)


def test_the_mass_rule_leaves_only_timestamps():
    from olmoasr_b200.decode_engine import sample_row_key

    assert all(sample_row_key(s, c, j) == row_key(s, c, j) for s in (0, 1, 2 ** 61 + 5) for c in (0, 12) for j in (0, 4))
    logits = torch.full((1, V), -30.0)
    logits[0, 500] = 5.0                                     # best text token
    ts_ids = [TB + 3, TB + 4, TB + 5, TB + 9, TB + 10, TB + 20, TB + 21, TB + 40]
    logits[0, ts_ids] = 4.5                                  # lse = 4.5 + log 8 > 5: text is banned
    tokens = torch.tensor([[SOT, TB + 2, 400]])              # a closed segment start and text: timestamps >= TB + 3
    f = filter_row(logits, tokens, 1, D.suppress_token_ids(D.DecodingOptions()), True, 50)
    assert torch.isinf(f[0, :TB]).all()
    n = 3000
    keys = [row_key(77, c, 0) for c in range(n)]
    ids, _ = sample_ids(f[0].numpy(), keys, 3, 1.0)
    counts = np.array([(ids == v).sum() for v in ts_ids])
    assert counts.sum() == n
    assert stats.chisquare(counts, np.full(8, n / 8)).pvalue > 1e-3


# ---- routing ---------------------------------------------------------------------------------------------------------
class _RecordingEngine:
    max_batch = 64

    def __init__(self):
        self.calls = []

    def greedy(self, feats, init, sample_len, suppress, suppress_blank, sot_index, **kw):
        self.calls.append(("greedy", feats.shape[0], kw))
        n = feats.shape[0]
        toks = torch.tensor([list(init) + [TB, 600, TB + 4, EOT]] * n)
        return toks, torch.full((n,), -1.0), torch.full((n,), 0.1), 5

    def sample(self, feats, init, sample_len, temperature, best_of, seed, clip_offset, suppress, suppress_blank, sot_index, **kw):
        self.calls.append(("sample", feats.shape[0], dict(kw, temperature=temperature, best_of=best_of, seed=seed,
                                                        clip_offset=clip_offset)))
        cands = []
        for c in range(feats.shape[0]):     # sample j of every clip: j + 1 tokens, each at log-prob log 0.5
            clip = clip_offset + c
            cands.append([(list(init) + [500 + clip] * (j + 1) + [EOT], (j + 2) * math.log(0.5)) for j in range(best_of)])
        return cands, torch.full((feats.shape[0],), 0.2), 7


class _StubModel:
    is_multilingual = False

    def __init__(self):
        self.dims = SimpleNamespace(n_text_ctx=448, n_audio_ctx=1500, n_audio_state=8, n_vocab=V)
        self.eng = _RecordingEngine()
        self.hooks = 0

    def encoder(self, mel):
        return torch.zeros(mel.shape[0], 1500, 8)

    def decode_engine(self, dtype):
        return self.eng

    def install_kv_cache_hooks(self):
        self.hooks += 1
        raise RuntimeError("hook loop")


def test_greedy_with_timestamps_goes_to_the_engine():
    m = _StubModel()
    res = D.decode(m, torch.zeros(3, 80, 3000), D.DecodingOptions())
    assert m.eng.calls == [("greedy", 3, dict(timestamps=True, max_initial_timestamp_index=50))]
    assert [r.tokens for r in res] == [[TB, 600, TB + 4]] * 3
    D.decode(m, torch.zeros(2, 80, 3000), D.DecodingOptions(without_timestamps=True))
    assert m.eng.calls[-1] == ("greedy", 2, dict(timestamps=False, max_initial_timestamp_index=None))
    assert m.hooks == 0


def test_best_of_chunks_clips_and_ranks():
    m = _StubModel()
    torch.manual_seed(3)
    res = D.decode(m, torch.zeros(13, 80, 3000), D.DecodingOptions(best_of=5, temperature=0.4))
    calls = m.eng.calls
    assert [(c[0], c[1], c[2]["clip_offset"]) for c in calls] == [("sample", 12, 0), ("sample", 1, 12)]
    assert all(c[2]["best_of"] == 5 and c[2]["temperature"] == 0.4 and c[2]["timestamps"] is True
               and c[2]["max_initial_timestamp_index"] == 50 for c in calls)
    assert calls[0][2]["seed"] == calls[1][2]["seed"]            # one seed per decode() call
    # ranked by sum_logprob / length: sample j scores (j + 2) log 0.5 / (j + 1), the longest sample wins
    for k, r in enumerate(res):
        assert r.tokens == [500 + k] * 5 and r.temperature == 0.4 and r.no_speech_prob == pytest.approx(0.2)
        assert math.isclose(r.avg_logprob, 6 * math.log(0.5) / 6, rel_tol=1e-6)
    m2 = _StubModel()
    res = D.decode(m2, torch.zeros(2, 80, 3000), D.DecodingOptions(best_of=5, temperature=0.4, length_penalty=0.0))
    assert [r.tokens for r in res] == [[500], [501]]             # no length normalisation: the shortest sample wins
    assert m.hooks == 0 and m2.hooks == 0


def test_the_seed_follows_torch_manual_seed():
    seeds = []
    for s in (5, 5, 6):
        m = _StubModel()
        torch.manual_seed(s)
        D.decode(m, torch.zeros(1, 80, 3000), D.DecodingOptions(temperature=0.6))
        assert m.eng.calls[0][2]["best_of"] == 1
        seeds.append(m.eng.calls[0][2]["seed"])
    assert seeds[0] == seeds[1] != seeds[2]


def test_hook_loop_keeps_best_of_above_the_engine_batch_and_the_engine_switch(monkeypatch):
    m = _StubModel()
    with pytest.raises(RuntimeError, match="hook loop"):
        D.decode(m, torch.zeros(1, 80, 3000), D.DecodingOptions(best_of=65, temperature=0.4))
    assert m.hooks == 1 and m.eng.calls == []
    monkeypatch.setattr(D, "USE_ENGINE", False)
    for opts in (D.DecodingOptions(), D.DecodingOptions(best_of=5, temperature=0.4), D.DecodingOptions(without_timestamps=True)):
        with pytest.raises(RuntimeError, match="hook loop"):
            D.decode(m, torch.zeros(1, 80, 3000), opts)
    assert m.hooks == 4 and m.eng.calls == []
