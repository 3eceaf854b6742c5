"""Temperature sampling and greedy decoding with timestamp rules on the device decoder (csrc/decode.cu dec_sample_kernel
through oasr_dec_sample_rules, DecodeEngine.greedy(timestamps=True) / DecodeEngine.sample, decode(), transcribe()).

The kernel is compared with the hook loop's own filters on crafted fp32 logits (temperature 0: exact ids; temperature > 0:
exact ids against the numpy restatement of tests/test_sampling_host.py for the same keys) and, by a chi-square test,
with softmax(filtered / T).  Whole decodes are compared with a reference loop over oracle/model.py on the GPU in the same
dtype, up to the first step whose margin is within rounding noise (the rule of tests/test_beam_search_gpu.py).
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from scipy import stats

from tests import test_sampling_host as H
from tests.test_decode_engine_gpu import SHARPEN, _build

pytestmark = pytest.mark.gpu

EOT, SOT, NO_SPEECH, TB = H.EOT, H.SOT, 50361, H.TB
SURE = {torch.float16: 8e-3, torch.bfloat16: 4e-2}     # margins, relative to max |logit|, that rounding cannot flip


def _suppress():
    from olmoasr_b200 import decoding as D

    return D.suppress_token_ids(D.DecodingOptions())


def _signed(keys):
    return torch.tensor([k - (1 << 64) if k >> 63 else k for k in keys], dtype=torch.int64)


def _step(eng, logits, n, timestamps, mi, temperature=None, keys=None):
    """One rule-aware sampling step over rows [0, n) on the given fp32 logits."""
    eng.logits[:n] = logits.cuda()
    eng._rules_cfg = (int(timestamps), -1 if mi is None else mi, int(temperature is not None))
    if temperature is not None:
        eng.temperature.fill_(temperature)
        eng.row_keys[:n] = _signed(keys).cuda()
    eng._enqueue_sample_rules(n)
    torch.cuda.synchronize()


HIST = [[TB + 10, 500, 600, 700],          # text after a closed segment: timestamps >= 11 only
        [TB + 10, 500, 600, TB + 20],      # open timestamp: no text below eot, timestamps >= 20
        [TB + 10, 500, TB + 20, TB + 21],  # closed pair: text must follow
        [500, 600, 700, 800],              # no timestamp yet
        [TB + 10, TB + 12, 500, TB + 30],  # open after a pair
        [TB + 3, 500, 600, 700],
        [500, 600, 700, TB + 1490],        # near the end of the range
        [TB + 10, 500, 600, 700]]


def _crafted():
    rows = torch.tensor([[SOT] + h for h in HIST])
    g = torch.Generator().manual_seed(5)
    logits = torch.randn(len(HIST), 51864, generator=g) * 3
    logits[[0, 5, 6], TB:] += 6.0               # mass rule on
    logits[7, TB:] += 1.0                       # close to it
    logits[1, EOT] = 25.0                       # eot at the top
    return rows, logits


def _engine():
    m, sd, dims, OM, xa = _build("tiny", n_clips=1)
    eng = m.decode_engine(torch.float16)
    eng.refresh_weights()
    return eng


def test_greedy_kernel_matches_the_hook_loop_filters():
    eng = _engine()
    sup = _suppress()
    n, mi = 12, 50
    ref = torch.tensor([[SOT]] * n)
    eng.reset(n, ref, sample_begin=1, suppress=sup, suppress_blank=True, sot_index=0)
    sums = torch.zeros(n)
    g = torch.Generator().manual_seed(21)
    for step in range(9):
        logits = torch.randn(n, eng.V, generator=g) * 3
        if step >= 1:
            logits[1::3, TB:] += 6.0                        # timestamp mass beats every text token on these rows
        if step >= 3:
            logits[::4, EOT] = logits[::4].max(-1).values + 1.0
        if step == 8:                                       # every row can end here
            logits[:] = -5.0
            logits[:, EOT] = 30.0
        f = H.filter_row(logits, ref, 1, sup, True, mi)
        lp = F.log_softmax(f, -1)
        nxt = f.argmax(-1)
        ended = ref[:, -1] == EOT
        sums += torch.where(ended, torch.zeros(n), lp[torch.arange(n), nxt])
        nxt[ended] = EOT
        ref = torch.cat([ref, nxt[:, None]], 1)
        _step(eng, logits, n, True, mi)
        assert eng.tokens[:n, : ref.shape[1]].cpu().long().tolist() == ref.tolist(), step
        assert torch.allclose(eng.sum_logprobs[:n].cpu(), sums, rtol=0, atol=1e-5 * (step + 1) * (1 + float(sums.abs().max()) / 10))
        if step == 0:
            want = torch.softmax(logits, -1)[:, NO_SPEECH]
            assert torch.allclose(eng.no_speech[:n].cpu(), want, rtol=1e-5, atol=1e-12)
        assert int(eng.done.item()) == int(bool((nxt == EOT).all())) and int(eng.pos.item()) == step + 1
    assert int(eng.done.item()) == 1
    assert int(eng.sample_counters.abs().sum()) == 0
    # crafted histories: every branch of ApplyTimestampRules
    rows, logits = _crafted()
    n = rows.shape[0]
    eng.reset(n, rows, sample_begin=1, suppress=sup, suppress_blank=True, sot_index=0)
    eng.pos.fill_(rows.shape[1] - 1)
    _step(eng, logits, n, True, mi)
    f = H.filter_row(logits, rows, 1, sup, True, mi)
    nxt = f.argmax(-1)
    assert eng.tokens[:n, rows.shape[1]].cpu().long().tolist() == nxt.tolist()
    assert torch.allclose(eng.sum_logprobs[:n].cpu(), F.log_softmax(f, -1)[torch.arange(n), nxt], rtol=0, atol=1e-5)
    assert all(int(t) >= TB for t in nxt[[0, 5, 6]])


@pytest.mark.parametrize("temperature", [0.2, 0.6, 1.0])
def test_sampling_kernel_matches_the_restatement(temperature):
    eng = _engine()
    sup = _suppress()
    cases = []
    g = torch.Generator().manual_seed(8)
    rand = torch.randn(16, eng.V, generator=g) * 3
    rand[1::3, TB:] += 6.0
    cases.append((torch.tensor([[SOT]] * 16), rand, True))                  # first step: timestamps only
    cases.append((torch.tensor([[SOT, 50362]] * 16), rand.clone(), False))  # no timestamp rules
    cases.append(_crafted() + (True,))
    decided = total = 0
    for case, (rows, logits, ts) in enumerate(cases):
        n = rows.shape[0]
        eng.reset(n, rows, sample_begin=1 if ts else 2, suppress=sup, suppress_blank=True, sot_index=0)
        pos = rows.shape[1] - 1
        eng.pos.fill_(pos)
        keys = [H.row_key(31 + case, r, 0) for r in range(n)]
        _step(eng, logits, n, ts, 50, temperature, keys)
        f = H.filter_row(logits, rows, 1 if ts else 2, sup, ts, 50)
        got = eng.tokens[:n, pos + 1].cpu().long()
        assert torch.isfinite(f[torch.arange(n), got]).all(), "a banned id was drawn"
        want, margin = H.sample_ids(f.numpy(), keys, pos, temperature)
        sure = margin > 1e-4
        assert (got.numpy()[sure] == want[sure]).all(), (got.tolist(), want.tolist(), margin)
        decided += int(sure.sum()); total += n
        lp = F.log_softmax(f, -1)[torch.arange(n), got]                     # log-probs at temperature 1
        assert torch.allclose(eng.sum_logprobs[:n].cpu(), lp, rtol=0, atol=1e-5)
    assert decided >= 0.9 * total


def test_sampling_kernel_draws_follow_softmax():
    eng = _engine()
    n, T, rounds = 64, 0.7, 50
    x = torch.full((eng.V,), -3.0)
    x[H.LIVE] = torch.tensor([1.0, 0.2, -0.5, 0.7, 1.3, -1.0, 0.0, 0.4])
    rows = torch.tensor([[SOT, 50362]] * n)
    ids, keys_all = [], []
    for r in range(rounds):
        eng.reset(n, rows, sample_begin=2, suppress=(), suppress_blank=False, sot_index=0)
        eng.suppress.fill_(1)
        eng.suppress[H.LIVE] = 0                       # eight live ids
        eng.pos.fill_(1)
        keys = [H.row_key(99, r, j) for j in range(n)]
        _step(eng, x.repeat(n, 1), n, False, None, T, keys)
        ids += eng.tokens[:n, 2].cpu().tolist()
        keys_all += keys
    ids = np.array(ids)
    assert set(ids.tolist()) <= set(H.LIVE)
    counts = np.array([(ids == v).sum() for v in H.LIVE])
    p = torch.softmax(x[H.LIVE].double() / T, 0).numpy()
    assert stats.chisquare(counts, p * len(ids)).pvalue > 1e-3, (counts, p * len(ids))
    f = torch.full((eng.V,), -math.inf)
    f[H.LIVE] = x[H.LIVE]
    want, margin = H.sample_ids(f.numpy(), keys_all, 1, T)
    sure = margin > 1e-4
    assert (ids[sure] == want[sure]).all() and sure.mean() > 0.95


def _index_mask(logits, tokens, sb, sup, mi):
    """Ids banned by the index rules alone (the text region lifted so that the mass rule cannot fire)."""
    lifted = logits.clone()
    lifted[:, :TB] = 1e4
    banned = torch.isinf(H.filter_row(lifted, tokens, sb, sup, True, mi))
    return banned


def _ref_greedy_ts(OM, sd, dims, xa, dtype, n_steps, suppress, mi, train_model=False):
    """DecodingTask._main_loop at temperature 0 with ApplyTimestampRules over oracle/model.py, stock torch on the GPU.
    Returns tokens, per-step relative margins (top-1 / top-2 after every filter, and |lse(ts) - max(text)| before the
    mass rule, over unfinished rows), sum_logprobs and no-speech probabilities."""
    n = xa.shape[0]
    tokens = torch.tensor([[SOT]] * n)
    cache, rel, sums, nsp = {}, [], torch.zeros(n), None
    with torch.no_grad():
        for i in range(n_steps):
            inp = tokens if i == 0 else tokens[:, -1:]
            logits = OM.decoder_forward(sd, dims, inp.cuda(), xa.to(dtype), None, train_model=train_model, cache=cache)
            if i == 0:
                nsp = logits[:, 0].float().softmax(-1)[:, NO_SPEECH].cpu()
            logits = logits[:, -1].float().cpu()
            f = H.filter_row(logits, tokens, 1, suppress, True, mi)
            pre = logits.masked_fill(_index_mask(logits, tokens, 1, suppress, mi), -math.inf)
            live = tokens[:, -1] != EOT
            top2 = f.topk(2, dim=-1).values
            mass = (pre[:, TB:].logsumexp(-1) - pre[:, :TB].max(-1).values).abs().nan_to_num(math.inf)
            m = torch.minimum(top2[:, 0] - top2[:, 1], mass) / logits.abs().max(-1).values
            rel.append(float(m[live].min()) if bool(live.any()) else math.inf)
            nxt = f.argmax(-1)
            sums += torch.where(live, F.log_softmax(f, -1)[torch.arange(n), nxt], torch.zeros(n))
            nxt[~live] = EOT
            tokens = torch.cat([tokens, nxt[:, None]], 1)
            if bool((nxt == EOT).all()):
                break
    return tokens, rel, sums, nsp


@pytest.mark.parametrize("variant", ["tiny", "small"])
@pytest.mark.parametrize("fp16", [True, False])
def test_greedy_with_timestamps_matches_the_reference_loop(variant, fp16):
    from olmoasr_b200.decoding import DecodingOptions, DecodingTask, decode

    dtype = torch.float16 if fp16 else torch.bfloat16
    m, sd, dims, OM, xa = _build(variant, emb_scale=SHARPEN[variant][0], pos_scale=SHARPEN[variant][1])
    n_steps = 24
    opts = DecodingOptions(without_timestamps=False, sample_len=n_steps, fp16=fp16)
    task = DecodingTask(m, opts)
    mi = task.ts_rules.max_initial_timestamp_index
    want, rel, sums, nsp = _ref_greedy_ts(OM, sd, dims, xa, dtype, n_steps, task.suppress, mi)
    res = decode(m, xa, opts)
    n_cmp = next((i for i, r in enumerate(rel) if r < SURE[dtype]), len(rel))
    print(f"{variant} fp16={fp16}: min relative margin {min(rel):.4f}, decided steps {n_cmp}/{len(rel)}; tokens {res[0].tokens[:8]}")
    for k in range(xa.shape[0]):
        seq = want[k, 1:].tolist()
        seq = seq[: seq.index(EOT)] if EOT in seq else seq
        assert res[k].tokens[:n_cmp] == seq[:n_cmp], k
        if n_cmp == len(rel):
            assert res[k].tokens == seq
            lp_ref = float(sums[k]) / (len(seq) + 1)
            assert abs(res[k].avg_logprob - lp_ref) <= 2e-2 * abs(lp_ref) + 1e-3
        assert abs(res[k].no_speech_prob - float(nsp[k])) <= 0.05 * float(nsp[k]) + 1e-6
        assert not res[k].tokens or res[k].tokens[0] >= TB
    eng = m.decode_engine(dtype)
    cross = 1 if eng.cross_splits(xa.shape[0]) == 1 else 2
    assert eng.launches_per_step == (6 + 1 + cross) * dims.n_text_layer + 1 + 1 + 2


def _check_timestamps(seq):
    """ApplyTimestampRules invariants of a sampled sequence (initial tokens removed, cut at eot)."""
    if not seq:
        return
    assert seq[0] >= TB, "the first token is a timestamp"
    ts = [t for t in seq if t >= TB]
    assert ts == sorted(ts), "timestamps never decrease"
    for i in range(len(seq) - 2):
        assert not (seq[i] >= TB and seq[i + 1] >= TB and seq[i + 2] >= TB), "no three timestamps in a row"
    for i in range(1, len(seq) - 1):
        if seq[i] >= TB and seq[i - 1] < TB:
            assert seq[i + 1] >= TB, "a segment's closing timestamp is followed by a timestamp or eot"


@pytest.mark.parametrize("timestamps", [False, True])
def test_best_of_sampling_is_reproducible_and_batch_independent(timestamps):
    from olmoasr_b200.decoding import DecodingOptions, decode

    m, sd, dims, OM, xa = _build("tiny", emb_scale=3.0, pos_scale=0.5, n_clips=3)
    opts = DecodingOptions(best_of=5, temperature=0.6, without_timestamps=not timestamps, sample_len=24)
    runs = []
    for s in (11, 11, 12):
        torch.manual_seed(s)
        runs.append([(r.tokens, r.avg_logprob) for r in decode(m, xa, opts)])
    assert runs[0] == runs[1], "same torch seed, same bits"
    assert runs[0] != runs[2], "another seed, other draws"
    # a clip's candidates do not depend on where it sits: alone (clip 12 of a decode() call of 13, which runs in a call
    # of its own) or inside a batch of 12 clips (cross-attention K/V shared by the group, split differently)
    eng = m.decode_engine(torch.float16)
    init = [SOT] if timestamps else [SOT, 50362]
    kw = dict(suppress=_suppress(), timestamps=timestamps, max_initial_timestamp_index=50 if timestamps else None)
    one, _, _ = eng.sample(xa[:1], init, 24, 0.6, 5, 1234, 12, **kw)
    feats = xa[[1, 2, 0, 1, 2, 0, 1, 2, 0, 1, 2, 0]]
    many, _, _ = eng.sample(feats, init, 24, 0.6, 5, 1234, 1, **kw)
    assert [t for t, _ in many[11]] == [t for t, _ in one[0]]
    assert [t for t, _ in many[2]] != [t for t, _ in one[0]]        # the same clip under another key draws otherwise
    for cands in many + one:
        assert len(cands) == 5
        for row, _ in cands:
            seq = row[len(init):]
            seq = seq[: seq.index(EOT)]
            if timestamps:
                _check_timestamps(seq)


def test_transcribe_runs_device_resident(monkeypatch):
    import olmoasr_b200.transcribe as T
    from olmoasr_b200 import synthetic

    m, sd, dims, OM, xa = _build("tiny", emb_scale=3.0, pos_scale=0.5, n_clips=1)

    def no_hooks():
        raise AssertionError("a window took the hook loop")

    monkeypatch.setattr(m, "install_kv_cache_hooks", no_hooks)
    seconds = 75.0
    audio = synthetic.waveforms(1, n_samples=int(seconds * 16000))[0]
    seen = []
    real = T.decode

    def spy(model, segment, options, **kw):
        seen.append(options)
        return real(model, segment, options, **kw)

    monkeypatch.setattr(T, "decode", spy)
    for kw in (dict(), dict(without_timestamps=False, beam_size=5, best_of=5)):
        seen.clear()
        torch.manual_seed(0)
        out = T.transcribe(m, audio, sample_len=96, **kw)
        assert seen, "decode was never called"
        prev = 0.0
        for seg in out["segments"]:
            assert prev - 1e-6 <= seg["start"] <= seg["end"] and seg["start"] <= seconds
            prev = seg["start"]
            toks = seg["tokens"]
            if toks:
                assert toks[0] >= TB, "a segment starts with a timestamp"
                ts = [t for t in toks if t >= TB]
                assert ts == sorted(ts), "timestamps never decrease inside a segment"
                assert not any(toks[i] >= TB and toks[i + 1] >= TB and toks[i + 2] >= TB for i in range(len(toks) - 2))
        print(f"transcribe {kw}: {len(out['segments'])} segments, {len(seen)} decode calls, "
              f"temperatures {sorted(set(o.temperature for o in seen))}")
