"""Beam search and best-of-n on the CPU: the reference restatement (tests/beam_reference.py) on a scripted decoder against
hand-derived outcomes, the option checks of DecodingTask, and best-of grouping / ranking on the hook loop.  The device
kernels are covered by tests/test_beam_search_gpu.py against the same reference."""
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from olmoasr_b200 import decoding as D
from tests import beam_reference as R

V = 51864
EOT = R.EOT
INIT = [R.SOT, R.NO_TIMESTAMPS]


class ScriptedLM:
    """step_fn for R.beam_search: the next-token log-probs are a function of the sampled prefix.  `table` maps a prefix
    tuple to {token: probability}; the rest of the mass is spread evenly over 1000 filler ids (1000 .. 1999)."""

    def __init__(self, table, default=None):
        self.table, self.default = table, default or {EOT: 0.9}
        self.rows = None

    def dist(self, prefix):
        p = dict(self.table.get(tuple(prefix), self.default))
        rest = max(1e-6, 1.0 - sum(p.values()))
        logits = torch.full((V,), -1e4)
        logits[1000:2000] = math.log(rest / 1000)
        for t, q in p.items():
            logits[t] = math.log(q)
        return logits

    def __call__(self, inp, sources):
        if sources is None:
            self.rows = [list(r) for r in inp.tolist()]
        else:
            self.rows = [self.rows[s] + [int(t)] for s, t in zip(sources, inp[:, -1].tolist())]
        out = torch.stack([self.dist(r[len(INIT):]) for r in self.rows])
        return out[:, None, :].repeat(1, inp.shape[1], 1)


def _run(table, beam, sample_len=6, **kw):
    return R.beam_search(ScriptedLM(table, kw.pop("default", None)), 1, INIT, sample_len, beam, **kw)


def test_beam_escapes_the_greedy_trap():
    # greedy takes 100 (0.5) and then only weak continuations; beam 2 keeps 200 (0.4), whose continuation is certain
    table = {(): {100: 0.5, 200: 0.4}, (100,): {101: 0.3, 102: 0.3}, (200,): {201: 0.95},
             (100, 101): {EOT: 0.99}, (100, 102): {EOT: 0.99}, (200, 201): {EOT: 0.99}}
    res = _run(table, 2)
    assert res.tokens == [[200, 201]]
    greedy = _run(table, 1)
    assert greedy.tokens == [[100, 101]]


def test_first_step_uses_one_row_of_candidates():
    # every beam holds the same prefix at the first step: the three kept beams are three different tokens
    table = {(): {100: 0.5, 200: 0.3, 300: 0.15}}
    res = _run(table, 3, sample_len=1)
    assert sorted(res.steps[0][:, -1].tolist()) == [100, 200, 300]


def test_eot_below_the_cut_is_not_recorded():
    # ranking 100, 200 (kept: beam 2 full) then eot: the walk stops before eot, so nothing is finished at step 0
    table = {(): {100: 0.5, 200: 0.3, EOT: 0.1}}
    st = R.BeamState(2, 2)
    lm = ScriptedLM(table)
    toks = torch.tensor([INIT, INIT])
    lp = torch.log_softmax(lm(toks, None)[:, -1], -1)
    R.beam_update(st, toks, lp, torch.zeros(2))
    assert st.finished == [{}]
    # with eot ranked second it is recorded, and the walk goes on to keep two beams
    table = {(): {100: 0.5, EOT: 0.3, 200: 0.1}}
    st = R.BeamState(2, 2)
    lp = torch.log_softmax(ScriptedLM(table)(toks, None)[:, -1], -1)
    out, src, done = R.beam_update(st, toks, lp, torch.zeros(2))
    assert list(st.finished[0].keys()) == [tuple(INIT + [EOT])] and out[:, -1].tolist() == [100, 200] and not done


def test_patience_two_collects_ten_candidates():
    res = _run({}, 5, sample_len=40, patience=2.0, default={EOT: 0.5, 7: 0.3, 8: 0.15})
    assert len(res.candidates[0]) == 10
    assert all(seq[-1] == EOT for seq, _ in res.candidates[0])
    res1 = _run({}, 5, sample_len=40, default={EOT: 0.5, 7: 0.3, 8: 0.15})
    assert len(res1.candidates[0]) == 5


def test_length_penalty_changes_the_choice():
    tokens = [[[1], [1, 2, 3, 4]]]
    sums = [[-1.0, -2.0]]
    assert R.rank(tokens, sums, None) == [1]            # -1/1 < -2/4
    assert R.rank(tokens, sums, 1.0) == [0]             # -1/1 > -2/1.5
    ranker = D.MaximumLikelihoodRanker(None)
    assert ranker.rank(tokens, sums) == [1] and D.MaximumLikelihoodRanker(1.0).rank(tokens, sums) == [0]
    for alpha in (None, 0.0, 0.6, 1.0):
        t = [[[5] * n for n in (1, 3, 6, 9)]]
        s = [[-0.5, -1.4, -2.2, -3.9]]
        assert D.MaximumLikelihoodRanker(alpha).rank(t, s) == R.rank(t, s, alpha)


def test_finalize_fills_with_live_beams():
    # nothing finishes within sample_len: finalize appends the live beams, best first, each closed by eot
    table = {(): {100: 0.6, 200: 0.3}, (100,): {101: 0.9}, (200,): {201: 0.9}}
    res = _run(table, 2, sample_len=2, default={300: 0.9})
    cands = res.candidates[0]
    assert [c[0][len(INIT):] for c in cands] == [[100, 101, EOT], [200, 201, EOT]]
    assert cands[0][1] > cands[1][1]
    assert res.tokens == [[100, 101]]


def test_option_checks():
    m = SimpleNamespace(is_multilingual=False, dims=SimpleNamespace(n_text_ctx=32, n_audio_ctx=4))
    bad = [dict(beam_size=5, best_of=5), dict(best_of=5), dict(patience=2.0), dict(beam_size=5, length_penalty=1.5),
           dict(beam_size=5, length_penalty=-0.1)]
    for kw in bad:
        with pytest.raises(ValueError):
            D.DecodingTask(m, D.DecodingOptions(**kw))
    # beam search without a device decoder is not available
    with pytest.raises(NotImplementedError):
        D.DecodingTask(m, D.DecodingOptions(beam_size=5, temperature=0.5))
    # best_of at a sampling temperature is accepted on the hook loop
    D.DecodingTask(m, D.DecodingOptions(best_of=5, temperature=0.4))


class _SamplingStub:
    """decoder() gives row r of the repeated batch a certain text determined by its row index, so best-of ranking is
    observable: within every clip, sample j emits j + 1 copies of token 500 + clip (each at log-prob log 0.5)."""

    is_multilingual = False

    def __init__(self, n_audio, best_of):
        self.dims = SimpleNamespace(n_text_ctx=32, n_audio_ctx=4, n_audio_state=8, n_vocab=V)
        self.n_audio, self.G = n_audio, best_of
        self.step, self.batches = 0, []

    def encoder(self, mel):
        return torch.arange(mel.shape[0], dtype=torch.float32)[:, None, None].repeat(1, 4, 8)

    def install_kv_cache_hooks(self):
        return {}, []

    def decoder(self, inp, xa, kv_cache=None):
        B, T = inp.shape
        self.batches.append(xa[:, 0, 0].tolist())
        logits = torch.full((B, T, V), -1e9)
        for r in range(B):
            clip, j = divmod(r, self.G)
            tok = 500 + clip if self.step < j + 1 else EOT
            logits[r, -1, tok] = 0.0
            logits[r, -1, 50300] = 0.0          # a second token at the same probability: log-prob log 0.5 each
        self.step += 1
        return logits


def test_best_of_groups_rows_and_ranks(monkeypatch):
    n_audio, G = 2, 3
    m = _SamplingStub(n_audio, G)
    # "sampling" that always picks the scripted token (the lowest id among the two equally likely)
    monkeypatch.setattr(torch.distributions, "Categorical", lambda logits: SimpleNamespace(sample=lambda: logits.argmax(-1)))
    res = D.DecodingTask(m, D.DecodingOptions(best_of=G, temperature=0.5, without_timestamps=True)).run(torch.zeros(n_audio, 80, 3000))
    # rows are clip-major: every clip's features repeated best_of times
    assert m.batches[0] == [0.0, 0.0, 0.0, 1.0, 1.0, 1.0]
    # sum_logprob of sample j = (j + 2) log 0.5 (its tokens and the eot) over length j + 1: the longest sample wins
    for k, r in enumerate(res):
        assert r.tokens == [500 + k] * G
        assert math.isclose(r.avg_logprob, (G + 1) * math.log(0.5) / (G + 1), rel_tol=1e-5)
        assert r.temperature == 0.5
    # with a strong length penalty toward short outputs the shortest sample wins
    m = _SamplingStub(n_audio, G)
    res = D.DecodingTask(m, D.DecodingOptions(best_of=G, temperature=0.5, length_penalty=0.0,
                                              without_timestamps=True)).run(torch.zeros(n_audio, 80, 3000))
    assert [r.tokens for r in res] == [[500], [501]]
