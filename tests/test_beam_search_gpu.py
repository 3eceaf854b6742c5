"""Beam search on the device decoder (csrc/decode.cu dec_beam_*, DecodeEngine.beam_search, decode(beam_size=...)) against
the CPU restatement of whisper/decoding.py in tests/beam_reference.py and the package's own _TimestampRules.

The candidate / select kernels are compared with the reference `update` on the same fp32 logits (exact ids, scores
within 1e-5).  Whole decodes are compared with the reference run over oracle/model.py on the GPU in the same activation
dtype, up to the first step at which the reference's own selection gap falls into rounding noise.
"""
import ctypes
import math

import pytest
import torch
import torch.nn.functional as F

from tests import beam_reference as R
from tests.test_decode_engine_gpu import SHARPEN, _build

pytestmark = pytest.mark.gpu

EOT, SOT, NO_TIMESTAMPS, TB = R.EOT, R.SOT, R.NO_TIMESTAMPS, R.TIMESTAMP_BEGIN


def _suppress():
    from olmoasr_b200 import decoding as D

    return D.suppress_token_ids(D.DecodingOptions())


def _device_step(eng, logits):
    from olmoasr_b200._lib import call, stream

    n = logits.shape[0]
    eng.logits[:n] = logits.cuda()
    a = eng.beam_args()
    call("oasr_dec_beam_candidates", ctypes.byref(a), stream())
    call("oasr_dec_beam_select", ctypes.byref(a), stream())
    torch.cuda.synchronize()


def _ref_filter(logits, tokens, sample_begin, suppress, timestamps, mi):
    from olmoasr_b200 import decoding as D

    lg = logits.clone()
    if tokens.shape[1] == sample_begin:
        lg[:, [R.BLANK, EOT]] = -math.inf
    lg[:, list(suppress)] = -math.inf
    if timestamps:
        D._TimestampRules(sample_begin, mi).apply(lg, tokens)
    return F.log_softmax(lg, dim=-1)


def _compare(eng, st, ref_tokens, ref_sum, sources, C, beam, first, steps=1):
    n = C * beam
    T = ref_tokens.shape[1]
    got = eng.tokens[:n, :T].cpu().long()
    assert torch.equal(got, ref_tokens), (got[:, -3:], ref_tokens[:, -3:])
    # log-prob sums: the fp32 normalisers differ in the last places, and a sum collects one such difference per step
    assert torch.allclose(eng.sum_logprobs[:n].cpu(), ref_sum, rtol=0, atol=1e-5 * steps * (1 + float(ref_sum.abs().max()) / 10))
    if not first:   # at the first step upstream's dict keeps the last beam as the source; every beam is the same there
        assert eng.src_rows[:n].cpu().tolist() == sources
    cnt, lens, fin, scores = (t.cpu() for t in eng.finished_lists(C, st.max_candidates))
    for c in range(C):
        want = list(st.finished[c].items())
        assert int(cnt[c]) == len(want)
        for i, (seq, sc) in enumerate(want):
            assert fin[c, i, : int(lens[c, i])].tolist() == list(seq)
            assert abs(float(scores[c, i]) - sc) <= 1e-5 * steps * (1 + abs(sc) / 10)


@pytest.mark.parametrize("timestamps", [False, True])
@pytest.mark.parametrize("beam", [1, 2, 5, 8])
def test_candidate_and_select_kernels_match_update(beam, timestamps):
    m, sd, dims, OM, xa = _build("tiny", n_clips=1)
    eng = m.decode_engine(torch.float16)
    eng.refresh_weights()
    C = 3
    n = C * beam
    init = [SOT] if timestamps else [SOT, NO_TIMESTAMPS]
    sb = len(init)
    sup = _suppress()
    ref_tokens = torch.tensor([init]).repeat(n, 1)
    eng.reset(n, ref_tokens, suppress=sup, suppress_blank=True, sot_index=0)
    eng.reset_beam(C, beam, beam, timestamps, 50)
    eng.pos.fill_(sb - 1)
    st = R.BeamState(beam, beam)
    ref_sum = torch.zeros(n)
    g = torch.Generator().manual_seed(100 + beam)
    for step in range(8):
        logits = torch.randn(n, eng.V, generator=g) * 3
        if step == 0:                           # every beam of a clip holds the same prefix: the same logits
            logits = logits[::beam].repeat_interleave(beam, dim=0)
        if step >= 2:
            logits[::2, EOT] = logits[::2].max(-1).values + torch.rand(n, generator=g)[::2]   # some rows want to end
        if timestamps and step >= 1:
            logits[1::3, TB:] += 6.0            # timestamp mass beats every text token on these rows
        lp = _ref_filter(logits, ref_tokens, sb, sup, timestamps, 50)
        first = ref_tokens.shape[1] == sb
        ref_tokens, sources, completed = R.beam_update(st, ref_tokens, lp, ref_sum)
        _device_step(eng, logits)
        _compare(eng, st, ref_tokens, ref_sum, sources, C, beam, first, step + 1)
        assert int(eng.done.item()) == int(completed) and int(eng.pos.item()) == sb + step
        if completed:
            break


def test_device_timestamp_filter_on_crafted_histories():
    """Every branch of ApplyTimestampRules: open / closed timestamp pairs, monotonic timestamps, no timestamps yet, and
    the timestamp-mass rule (on and off), each in one beam of an 8-beam clip."""
    m, sd, dims, OM, xa = _build("tiny", n_clips=1)
    eng = m.decode_engine(torch.float16)
    eng.refresh_weights()
    beam, sb, mi = 8, 1, 50
    hist = [[TB + 10, 500, 600, 700],          # text after a closed segment: timestamps >= 11 only
            [TB + 10, 500, 600, TB + 20],      # open timestamp: no text below eot, timestamps >= 20
            [TB + 10, 500, TB + 20, TB + 21],  # closed pair: text must follow
            [500, 600, 700, 800],              # no timestamp yet
            [TB + 10, TB + 12, 500, TB + 30],  # open after a pair
            [TB + 3, 500, 600, 700],
            [500, 600, 700, TB + 1490],        # near the end of the range
            [TB + 10, 500, 600, 700]]
    rows = torch.tensor([[SOT] + h for h in hist])
    sup = _suppress()
    eng.reset(beam, rows, sample_begin=sb, suppress=sup, suppress_blank=True, sot_index=0)
    eng.reset_beam(1, beam, 16, True, mi)
    eng.pos.fill_(rows.shape[1] - 1)
    g = torch.Generator().manual_seed(5)
    sums = -torch.rand(beam, generator=g) * 4
    eng.sum_logprobs[:beam] = sums.cuda()
    logits = torch.randn(beam, eng.V, generator=g) * 3
    logits[[0, 5, 6], TB:] += 6.0               # mass rule on
    logits[7, TB:] += 1.0                       # close to it
    logits[1, EOT] = 25.0                       # an eot candidate at the top
    st = R.BeamState(beam, 16)
    ref_sum = sums.clone()
    lp = _ref_filter(logits, rows, sb, sup, True, mi)
    ref_tokens, sources, completed = R.beam_update(st, rows, lp, ref_sum)
    _device_step(eng, logits)
    _compare(eng, st, ref_tokens, ref_sum, sources, 1, beam, False)
    # the same rows against torch's topk of the filtered log-probs: every kept (row, token) is in its row's top beam + 1
    top = lp.topk(beam + 1, dim=-1).indices
    for k in range(beam):
        src = sources[k]
        assert int(ref_tokens[k, -1]) in top[src].tolist()


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_kv_reorder_matches_index_select(dtype):
    m, sd, dims, OM, xa = _build("tiny", n_clips=1)
    eng = m.decode_engine(dtype)
    eng.refresh_weights()
    C, beam, P = 2, 4, 17
    n = C * beam
    eng.self_k.copy_(torch.randn_like(eng.self_k, dtype=torch.float32).to(dtype))
    eng.self_v.copy_(torch.randn_like(eng.self_v, dtype=torch.float32).to(dtype))
    k0, v0 = eng.self_k.clone(), eng.self_v.clone()
    src = [1, 0, 3, 2,              # clip 0: two swaps (cycles)
           4, 4, 6, 7]              # clip 1: a fork (rows 4, 5 from 4) and identity rows
    eng.src_rows[:n] = torch.tensor(src, dtype=torch.int32, device="cuda")
    eng.pos.fill_(P)
    eng.reorder_kv(C, beam)
    torch.cuda.synchronize()
    idx = torch.tensor(src, device="cuda")
    for got, ref in ((eng.self_k, k0), (eng.self_v, v0)):
        want = ref.clone()
        want[:, :n, :P] = ref[:, :n, :P].index_select(1, idx)
        assert torch.equal(got, want)


@pytest.mark.parametrize("splits", [1, 4])
def test_grouped_cross_attention_is_bit_identical_to_replicated(splits):
    from olmoasr_b200._lib import DecAttnArgs, call, ptr, stream

    m, sd, dims, OM, xa = _build("tiny", n_clips=1)
    eng = m.decode_engine(torch.float16)
    eng.refresh_weights()
    C, beam, d, T = 3, 5, eng.d, eng.n_audio_ctx
    n = C * beam
    kv = (torch.randn(C, T, 2 * d, device="cuda") * 0.5).half()
    rep = kv.repeat_interleave(beam, dim=0).contiguous()
    eng.q[:n] = torch.randn(n, d, device="cuda").half()
    outs = []
    for buf, group in ((kv, beam), (rep, 1)):
        part = torch.zeros(splits, n, d, device="cuda")
        a = DecAttnArgs()
        a.q, a.ldq = ptr(eng.q), eng.q.stride(0)
        a.k, a.v, a.kv_seq_stride, a.kv_row_stride = ptr(buf), ptr(buf[:, :, d:]), T * 2 * d, 2 * d
        a.scores, a.scores_ld = ptr(eng.scores), eng.scores.stride(1)
        a.out_partial, a.ld_out = ptr(part), d
        a.pos_ptr, a.n_keys = None, T
        a.n_seq, a.n_head, a.n_splits, a.scale, a.dtype = n, eng.H, splits, 64 ** -0.25, eng.dt
        if group == 1:
            call("oasr_dec_attention", ctypes.byref(a), stream())
        else:
            call("oasr_dec_attention_grouped", ctypes.byref(a), group, stream())
        outs.append(part)
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1])


TOL = {torch.float16: 4e-3, torch.bfloat16: 3e-2}      # relative L2 of a logits row (as tests/test_decode_engine_gpu.py)
SURE = {torch.float16: 8e-3, torch.bfloat16: 4e-2}     # margins, relative to max |logit|, that rounding cannot flip

CONFIGS = [("tiny", True, False, None, None), ("tiny", False, False, None, None), ("tiny", True, True, None, None),
           ("tiny", False, True, None, None), ("small", True, False, None, None), ("small", False, True, None, None),
           ("tiny", True, True, 2.0, 0.6), ("small", True, False, 2.0, 0.6)]


@pytest.mark.parametrize("variant,fp16,timestamps,patience,length_penalty", CONFIGS)
def test_beam_decode_matches_the_reference(variant, fp16, timestamps, patience, length_penalty):
    """Two comparisons.  Step by step: after every graph replay the engine's logits equal the oracle decoder's on the
    engine's own beams (its cache rearranged by index_select), and the engine's new beams, sums and finished lists equal
    the reference update applied to those logits.  End to end: `decode()` against the reference beam decode in the same
    dtype, ids equal up to the first step whose selection gap (or timestamp-mass margin) is within rounding noise."""
    from olmoasr_b200.decoding import DecodingOptions, DecodingTask, decode

    dtype = torch.float16 if fp16 else torch.bfloat16
    m, sd, dims, OM, xa = _build(variant, emb_scale=SHARPEN[variant][0], pos_scale=SHARPEN[variant][1])
    beam, sample_len = 5, 24
    opts = DecodingOptions(beam_size=beam, without_timestamps=not timestamps, sample_len=sample_len, fp16=fp16,
                           patience=patience, length_penalty=length_penalty)
    task = DecodingTask(m, opts)
    mi = task.ts_rules.max_initial_timestamp_index if timestamps else None
    init, sup = list(task.initial_tokens), task.suppress
    C, sb = xa.shape[0], len(init)
    n, max_cand = C * beam, round(beam * (patience or 1.0))
    # ---- step by step
    eng = m.decode_engine(dtype)
    eng.prepare(xa)
    eng.reset(n, torch.tensor([init]).repeat(n, 1), None, sup, True, 0)
    eng.reset_beam(C, beam, max_cand, timestamps, mi)
    g = eng._graph(n)
    for _ in range(sb - 1):
        g.replay()
    st, tokens, sums = R.BeamState(beam, max_cand), torch.tensor([init]).repeat(n, 1), torch.zeros(n)
    cache, xa_rep, worst = {}, xa.to(dtype).repeat_interleave(beam, dim=0), 0.0
    for step in range(sample_len):
        g.replay()
        got = eng.logits[:n].float().cpu()
        with torch.no_grad():
            inp = tokens if step == 0 else tokens[:, -1:]
            want = OM.decoder_forward(sd, dims, inp.cuda(), xa_rep, None, train_model=False, cache=cache)[:, -1].float().cpu()
        worst = max(worst, float(((got - want).norm(dim=-1) / want.norm(dim=-1)).max()))
        lp = _ref_filter(got, tokens, sb, sup, timestamps, mi)
        tokens, sources, completed = R.beam_update(st, tokens, lp, sums)
        _compare(eng, st, tokens, sums, sources, C, beam, step == 0, step + 1)
        idx = torch.tensor(sources, device="cuda")
        for key in list(cache):
            if ".cross_attn." not in key:
                cache[key] = cache[key].index_select(0, idx)
        if completed:
            assert int(eng.done.item()) == 1
            break
    assert worst <= TOL[dtype], worst
    # ---- end to end
    ref = R.beam_decode(sd, dims, xa, beam, init, sample_len, dtype=dtype, patience=patience, length_penalty=length_penalty,
                        suppress=sup, timestamps=timestamps, max_initial_timestamp_index=mi)
    rel = [min(min(gp), mm) / sc for gp, mm, sc in zip(ref.gaps, ref.mass_margins, ref.logit_scale)]
    n_cmp = next((i for i, r in enumerate(rel) if r < SURE[dtype]), len(rel))
    res = decode(m, xa, opts)
    print(f"{variant} fp16={fp16} ts={timestamps} patience={patience} lp={length_penalty}: {step + 1} steps equal to the "
          f"reference update, worst logits rel-L2 {worst:.1e}; end to end min relative gap {min(rel):.4f}, "
          f"decided steps {n_cmp}/{len(rel)}; tokens {res[0].tokens[:8]}")
    if n_cmp == len(rel):
        for c in range(C):
            assert res[c].tokens == ref.tokens[c]
            assert abs(res[c].avg_logprob - ref.avg_logprobs[c]) <= 2e-2 * abs(ref.avg_logprobs[c]) + 1e-3
    for c in range(C):
        want = [tuple(r) for r in ref.steps[n_cmp - 1][c * beam:(c + 1) * beam].tolist()] if n_cmp else []
        if want and n_cmp < len(rel):   # the decided prefix: the selected sequence extends one of the decided beams
            assert any(tuple(init + res[c].tokens)[: len(w)] == w for w in want) or len(res[c].tokens) < n_cmp
        assert abs(res[c].no_speech_prob - ref.no_speech_probs[c]) <= 0.05 * ref.no_speech_probs[c] + 1e-6
        if timestamps and res[c].tokens:
            assert res[c].tokens[0] >= TB


def test_batch_independence_and_run_to_run_bits():
    m, sd, dims, OM, xa = _build("tiny", emb_scale=3.0, pos_scale=0.5, n_clips=3)
    eng = m.decode_engine(torch.float16)
    sup = _suppress()
    init = [SOT]
    feats = xa[[0, 1, 2, 1, 0, 2, 2, 1, 0, 1, 2, 0]]
    one, _, _ = eng.beam_search(xa[:1], init, 24, 5, suppress=sup, timestamps=True, max_initial_timestamp_index=50)
    many, _, _ = eng.beam_search(feats, init, 24, 5, suppress=sup, timestamps=True, max_initial_timestamp_index=50)
    again, _, _ = eng.beam_search(feats, init, 24, 5, suppress=sup, timestamps=True, max_initial_timestamp_index=50)
    assert many == again                                               # ids and scores: the same bits on every run
    for c in (0, 4, 8, 11):
        # alone, the clip's cross-attention splits its key range; in a batch of 12 it does not, so the fp32 partial sums
        # are grouped differently and the scores agree to rounding only: the ids are compared
        assert [t for t, _ in many[c]] == [t for t, _ in one[0]], c
    assert all(many[c] == many[0] for c in (4, 8, 11))                 # one clip, one result, wherever it sits in the batch


def test_transcribe_long_form_with_eval_options(monkeypatch):
    import olmoasr_b200.transcribe as T
    from olmoasr_b200 import synthetic

    m, sd, dims, OM, xa = _build("tiny", emb_scale=3.0, pos_scale=0.5, n_clips=1)
    seconds = 75.0
    audio = synthetic.waveforms(1, n_samples=int(seconds * 16000))[0]
    seen = []
    real = T.decode

    def spy(model, segment, options, **kw):
        seen.append(options)
        return real(model, segment, options, **kw)

    monkeypatch.setattr(T, "decode", spy)
    out = T.transcribe(m, audio, without_timestamps=False, beam_size=5, best_of=5, sample_len=96)
    assert seen, "decode was never called"
    for o in seen:
        if o.temperature == 0:
            assert o.beam_size == 5 and o.best_of is None
        else:
            assert o.beam_size is None and o.patience is None and o.best_of == 5
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
    print(f"transcribe: {len(out['segments'])} segments, {len(seen)} decode calls, "
          f"temperatures {sorted(set(o.temperature for o in seen))}")
