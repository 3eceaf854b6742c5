"""The device decoder's token selection (csrc/decode.cu dec_sample_kernel<TS, SAMPLING>, dec_beam_cand_kernel,
dec_beam_select_kernel) against the fp64 statements of tests/selection_reference.py, through the engine's own argument
blocks, at both vocabulary widths: 51864 (inference layout) and 51865 (training layout, the pad row included).

Rows come from two sources.  Harvested: the fp32 logits the tiny engine writes in fp16 and bf16 while it decodes, with
the ties 16-bit values bring.  Planted: 16-bit-quantised random rows with exact ties placed inside one float4, across
threads, warps and every slice boundary, at eot against text, with more tied ids than beam + 1, and rows where only eot
is allowed; plus the row whose single allowed timestamp equals the text maximum (lse_ts == max_text exactly).  Every
form is also run twice (same bits) and with a row copied into slots 0..3 (same bits in every slot), with sentinels in
the rows and clips past the launched ones.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

from tests import selection_reference as S
from tests import test_sampling_host as H
from tests.test_decode_engine_gpu import SHARPEN, _build

pytestmark = pytest.mark.gpu

EOT, SOT, TB, NS = S.EOT, H.SOT, S.TB, S.NO_SPEECH
WIDTHS = [51864, 51865]
RATIOS = {}


def _sup():
    from olmoasr_b200 import decoding as D

    return D.suppress_token_ids(D.DecodingOptions())


@pytest.fixture(scope="module")
def engines():
    """V -> (tiny engine in fp16): the inference-layout model and a training-layout model (n_vocab + 1 rows)."""
    import olmoasr_b200 as ob
    from olmoasr_b200.model import OLMoASR

    inf = _build("tiny", n_clips=1)[0]
    torch.manual_seed(0)
    train = OLMoASR(ob.VARIANT_TO_DIMS["tiny"]).cuda()
    out = {}
    for m in (inf, train):
        eng = m.decode_engine(torch.float16)
        eng.refresh_weights()
        out[eng.V] = eng
    assert sorted(out) == WIDTHS
    yield out
    print("\nselection error / bound, worst per form: " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(RATIOS.items())))


def _note(form, r):
    RATIOS[form] = max(RATIOS.get(form, 0.0), r)


# ---- launches -------------------------------------------------------------------------------------------------------------
def _plain_sample(eng, n):
    """The oasr_dec_sample call of DecodeEngine._enqueue_step (greedy without timestamp rules)."""
    from olmoasr_b200._lib import DecSampleArgs, call, ptr, stream

    s = DecSampleArgs()
    s.logits, s.ld_logits = ptr(eng.logits), eng.logits.stride(0)
    s.tokens, s.ld_tokens, s.pos_ptr = ptr(eng.tokens), eng.tokens.stride(0), ptr(eng.pos)
    s.suppress, s.sum_logprobs, s.no_speech_prob = ptr(eng.suppress), ptr(eng.sum_logprobs), ptr(eng.no_speech)
    s.n_unfinished, s.done_flag = ptr(eng.n_unfinished), ptr(eng.done)
    s.scratch, s.counters, s.n_slices = ptr(eng.sample_scratch), ptr(eng.sample_counters), eng.sample_slices
    s.n_seq, s.n_vocab = n, eng.V
    s.sample_begin, s.sot_index, s.suppress_blank, s.blank, s.eot, s.no_speech = eng._sample_cfg
    call("oasr_dec_sample", ctypes.byref(s), stream())


def _beam_step(eng):
    from olmoasr_b200._lib import call, stream

    a = eng.beam_args()
    call("oasr_dec_beam_candidates", ctypes.byref(a), stream())
    call("oasr_dec_beam_select", ctypes.byref(a), stream())


GUARD = 4
GUARDED = {"rows": 0, "clips": 0}     # launches whose guard cells existed (a launch of all 64 rows has none)


def _sentinels(eng, n):
    if n + GUARD > eng.max_batch:
        return None
    eng.tokens[n:n + GUARD] = -7
    eng.sum_logprobs[n:n + GUARD] = -1234.5
    eng.no_speech[n:n + GUARD] = 7.5
    return [t[n:n + GUARD].clone() for t in (eng.tokens, eng.sum_logprobs, eng.no_speech)]


def _check_sentinels(eng, n, saved):
    if saved is None:
        return
    for t, s in zip((eng.tokens, eng.sum_logprobs, eng.no_speech), saved):
        assert torch.equal(t[n:n + GUARD], s), "a row past the launched ones was written"
    GUARDED["rows"] += 1


# ---- greedy and sampling ----------------------------------------------------------------------------------------------------
FORMS = ["plain", "ts", "sample", "sample_ts"]


def _sample_launch(eng, form, x, prefix, sb, sums, T=0.6, keys=None, mi=50, suppress=None):
    n, pos = x.shape[0], prefix.shape[1] - 1
    eng.reset(n, prefix, sample_begin=sb, suppress=_sup() if suppress is None else suppress, suppress_blank=True, sot_index=0)
    eng.pos.fill_(pos)
    eng.sum_logprobs[:n] = sums.cuda()
    eng.logits[:n] = x.cuda()
    saved = _sentinels(eng, n)
    if form == "plain":
        _plain_sample(eng, n)
    else:
        ts, sampling = form.endswith("ts"), form.startswith("sample")
        eng._rules_cfg = (int(ts), mi, int(sampling))
        if sampling:
            eng.temperature.fill_(T)
            eng.row_keys[:n] = torch.tensor([k - (1 << 64) if k >> 63 else k for k in keys], dtype=torch.int64).cuda()
        eng._enqueue_sample_rules(n)
    torch.cuda.synchronize()
    _check_sentinels(eng, n, saved)
    assert int(eng.sample_counters.abs().sum()) == 0, "slice counters not re-armed"
    return (eng.tokens[:n, pos + 1].cpu().long(), eng.sum_logprobs[:n].cpu().clone(), eng.no_speech[:n].cpu().clone(),
            int(eng.pos.item()), int(eng.done.item()))


def _check_sample(eng, form, x, prefix, sb, sums, T=0.6, keys=None, mi=50, suppress=None):
    ts, sampling = form.endswith("ts"), form.startswith("sample")
    sup = _sup() if suppress is None else suppress
    out = _sample_launch(eng, form, x, prefix, sb, sums, T, keys, mi, suppress)
    again = _sample_launch(eng, form, x, prefix, sb, sums, T, keys, mi, suppress)
    assert all(torch.equal(a, b) if torch.is_tensor(a) else a == b for a, b in zip(out, again)), "two runs differ"
    nxt, got_sum, nsp, pos_after, done = out
    pos = prefix.shape[1] - 1
    banned = S.banned_by_index(x, prefix, sb, sup, ts, mi if ts else None)
    r = S.check_sample_step(x.numpy(), banned, timestamps=ts, prev=prefix[:, -1], sum_in=sums.numpy(), got_next=nxt.numpy(),
                            got_sum=got_sum.numpy(), temperature=T if sampling else 0.0, keys=keys, pos=pos)
    _note(f"{form} V={eng.V}", r)
    if pos == 0:
        _note(f"no_speech V={eng.V}", S.check_no_speech(x.numpy(), nsp.numpy()))
    assert pos_after == pos + 1 and done == int(bool((nxt == EOT).all()))
    return nxt


def _q16(x, dtype):
    return x.to(dtype).float()


def _planted(n, V, seed, dtype):
    """Rows with exact ties at the top placed at the launch geometry's seams (one kind per row, cycling)."""
    g = torch.Generator().manual_seed(seed)
    x = _q16(torch.randn(n, V, generator=g) * 3, dtype)
    per = S.slice_len(V)
    seams = [(101, 103), (99, 100), (127, 128), (EOT, 100), (EOT, TB + 5)] + [(per * s - 1, per * s) for s in range(1, 16)]
    seams.append(tuple(range(1000, 1000 + 13 * 3244, 3244)))          # 13 tied ids, one per slice
    for r in range(n):
        ids = seams[(seed + r) % len(seams)]
        x[r, list(ids)] = float(x[r].max()) + 1.0
    return x


def _prefix(n, pos, seed):
    """Token rows up to `pos`: SOT, then a segment (timestamp, text ..., timestamp, timestamp, text ...)."""
    g = torch.Generator().manual_seed(seed)
    p = torch.randint(0, 50000, (n, pos + 1), generator=g)
    p[:, 0] = SOT
    if pos >= 1:
        p[:, 1] = TB + 2
    if pos >= 6:
        p[:, 4], p[:, 5] = TB + 9, TB + 9
    return p


POSITIONS = {"first": 0, "mid": 200, "last": 447}


@pytest.mark.parametrize("V", WIDTHS)
@pytest.mark.parametrize("form", FORMS)
def test_sample_forms_on_planted_rows(engines, V, form):
    eng = engines[V]
    guarded = GUARDED["rows"]
    for k, (n, where, T) in enumerate(((1, "first", 0.2), (5, "mid", 0.6), (37, "last", 1.0), (64, "mid", 0.4))):
        pos = POSITIONS[where]
        ts = form.endswith("ts")
        if where == "first" and not ts:
            prefix, sb = torch.tensor([[SOT, 50362]] * n)[:, :1], 1
        else:
            prefix, sb = _prefix(n, pos, k), 1
        for dtype in (torch.bfloat16, torch.float16):
            x = _planted(n, V, 3 * k + (dtype == torch.float16), dtype)
            sums = -torch.rand(n, generator=torch.Generator().manual_seed(k)) * 10
            if n > 4:
                prefix = prefix.clone()
                prefix[3, -1] = EOT                                        # a finished row: eot, frozen sum
            keys = [H.row_key(17, k, r) for r in range(n)]
            _check_sample(eng, form, x, prefix, sb, sums, T, keys)
    assert GUARDED["rows"] - guarded == 12, "the launches below 61 rows check their guard rows"


@pytest.mark.parametrize("V", WIDTHS)
@pytest.mark.parametrize("form", FORMS)
def test_sample_forms_give_the_same_bits_in_every_slot(engines, V, form):
    eng = engines[V]
    x = _planted(1, V, 5, torch.bfloat16).repeat(4, 1)
    prefix = _prefix(1, 200, 1).repeat(4, 1)
    keys = [H.row_key(3, 0, 0)] * 4
    nxt, sums, _, _, _ = _sample_launch(eng, form, x, prefix, 1, torch.full((4,), -2.5), 0.6, keys)
    assert nxt.tolist() == [nxt[0].item()] * 4
    assert sums.view(torch.int32).tolist() == [sums.view(torch.int32)[0].item()] * 4, \
        f"log-prob sums differ by slot: {sums.tolist()}"


@pytest.mark.parametrize("V", WIDTHS)
def test_single_timestamp_equal_to_the_text_maximum_keeps_text(engines, V):
    """lse_ts == max_text exactly: the strict ">" keeps text, and the tie goes to the lower id (eot)."""
    eng = engines[V]
    for form in ("ts", "sample_ts"):
        x = torch.full((2, V), -20.0)
        x[:, EOT] = 7.0
        x[:, V - 1] = 7.0                                  # the last id: at V = 51865 the pad row, a timestamp here
        prefix = torch.tensor([[SOT, TB + 3, 400, V - 1]] * 2)
        nxt = _check_sample(eng, form, x, prefix, 1, torch.zeros(2), 1.0, [H.row_key(1, 0, 0), H.row_key(1, 0, 1)])
        if form == "ts":
            assert nxt.tolist() == [EOT, EOT]


@pytest.mark.parametrize("V", WIDTHS)
def test_only_eot_allowed(engines, V):
    eng = engines[V]
    sup = [v for v in range(V) if v != EOT]
    x = _planted(3, V, 9, torch.float16)
    for form in FORMS:
        nxt = _check_sample(eng, form, x, _prefix(3, 20, 2), 1, torch.zeros(3), 0.6,
                            [H.row_key(2, 0, r) for r in range(3)], suppress=sup)
        assert nxt.tolist() == [EOT] * 3


# ---- beam search -------------------------------------------------------------------------------------------------------------
def _beam_launch(eng, x, prefix, sb, sums, C, beam, max_cand, ts, fin_count=None, done=0, suppress=None):
    n, pos = x.shape[0], prefix.shape[1] - 1
    eng.reset(n, prefix, sample_begin=sb, suppress=_sup() if suppress is None else suppress, suppress_blank=True, sot_index=0)
    eng.reset_beam(C, beam, max_cand, ts, 50)
    eng.pos.fill_(pos)
    eng.done.fill_(done)
    eng.sum_logprobs[:n] = sums.cuda()
    if fin_count is not None:
        eng.fin_count[:C] = torch.tensor(fin_count, dtype=torch.int32).cuda()
    clip_guard = C + 2 <= eng.max_batch
    eng.fin_count[C:C + 2] = 5
    eng.fin_scores.view(-1)[C * max_cand:] = -99.0
    eng.logits[:n] = x.cuda()
    saved = _sentinels(eng, n)
    before = [t.clone() for t in (eng.tokens, eng.sum_logprobs, eng.fin_tokens, eng.fin_scores, eng.fin_len, eng.fin_count)]
    _beam_step(eng)
    torch.cuda.synchronize()
    _check_sentinels(eng, n, saved)
    if clip_guard:
        assert bool((eng.fin_count[C:C + 2] == 5).all()), "a clip past the launched ones was written"
        assert bool((eng.fin_scores.view(-1)[C * max_cand:] == -99.0).all()), "a clip past the launched ones was written"
        GUARDED["clips"] += 1
    cnt, lens, fin, scores = (t.cpu().clone() for t in eng.finished_lists(C, max_cand))
    return (eng.tokens[:n, :pos + 2].cpu().clone(), eng.sum_logprobs[:n].cpu().clone(), eng.src_rows[:n].cpu().clone(),
            cnt, lens, fin, scores, before, eng.no_speech[:n].cpu().clone())


def _check_beam(eng, x, prefix, sb, sums, C, beam, max_cand, ts, fin_count=None, suppress=None):
    n, pos = x.shape[0], prefix.shape[1] - 1
    first = pos == sb - 1
    fc = fin_count or [0] * C
    out = _beam_launch(eng, x, prefix, sb, sums, C, beam, max_cand, ts, fc, suppress=suppress)
    again = _beam_launch(eng, x, prefix, sb, sums, C, beam, max_cand, ts, fc, suppress=suppress)
    assert all(torch.equal(a, b) for a, b in zip(out[:7] + out[8:], again[:7] + again[8:])), "two runs differ"
    toks, got_sums, src, cnt, lens, fin, scores, _, nsp = out
    if pos == 0:                                         # the select kernel's own no-speech probability (sot_index 0)
        _note(f"beam no_speech V={eng.V}", S.check_no_speech(x.numpy(), nsp.numpy()))
    banned = S.banned_by_index(x, prefix, sb, _sup() if suppress is None else suppress, ts, 50 if ts else None)
    decided = 0
    for c in range(C):
        rows = slice(c * beam, (c + 1) * beam)
        new = [(float(scores[c, i]), fin[c, i, : int(lens[c, i])].tolist()) for i in range(fc[c], int(cnt[c]))]
        res = S.check_beam_step(x[rows].numpy(), banned[rows], timestamps=ts, sums=sums[rows].numpy(),
                                prefix=prefix[rows].tolist(), pos=pos, beam=beam, max_cand=max_cand, fin_count=fc[c],
                                first=first, got_tokens=toks[rows].tolist(), got_sums=got_sums[rows].numpy(),
                                got_src=(src[rows] - c * beam).tolist(), got_fin=new)
        decided += res["decided"]
        _note(f"beam V={eng.V}", res["ratio"])
    return decided


def _beam_rows(C, beam, V, seed, dtype, first):
    x = _planted(C * beam, V, seed, dtype)
    sums = (-torch.rand(C * beam, generator=torch.Generator().manual_seed(seed)) * 6).float()
    if first:
        for c in range(C):
            x[c * beam:(c + 1) * beam] = x[c * beam]
            sums[c * beam:(c + 1) * beam] = 0.0
    elif beam >= 2:                                      # clip 0: beams 0 and 1 twins (one row, one sum): exact cross-beam ties
        x[1] = x[0]
        sums[1] = sums[0]
    x[2::3, EOT] = x[2::3].max(-1).values + 0.25          # rows that want to end (eot tied with text on some)
    return x, sums


@pytest.mark.parametrize("V", WIDTHS)
@pytest.mark.parametrize("beam", [1, 2, 5, 8])
def test_beam_forms_on_planted_rows(engines, V, beam):
    eng = engines[V]
    decided = total = 0
    guarded = dict(GUARDED)
    clips = max(1, 64 // beam)
    for k, (C, where, ts, patience) in enumerate(((1, "first", True, 1), (3, "mid", True, 2), (clips, "last", False, 1),
                                                  (2, "mid", False, 4))):
        max_cand = min(32, beam * patience)
        pos = POSITIONS[where]
        prefix = _prefix(C * beam, pos, k) if where != "first" else torch.tensor([[SOT]] * (C * beam))
        for dtype in (torch.bfloat16, torch.float16):
            x, sums = _beam_rows(C, beam, V, 7 * k + beam, dtype, where == "first")
            fc = [max_cand - 1 if c % 2 else 0 for c in range(C)] if where != "first" else None
            decided += _check_beam(eng, x, prefix, 1, sums, C, beam, max_cand, ts, fc)
            total += C
    assert decided >= 0.9 * total, (decided, total)
    assert GUARDED["rows"] > guarded["rows"] and GUARDED["clips"] > guarded["clips"], "no launch checked its guard cells"


@pytest.mark.parametrize("V", WIDTHS)
@pytest.mark.parametrize("beam", [1, 2, 5, 8])
def test_beam_rows_with_fewer_allowed_ids_than_candidates(engines, V, beam):
    """An open segment at the last timestamp (at V = 51865 the pad id) with the special ids suppressed leaves eot and
    one timestamp; a second clip allows eot alone.  The top beam + 1 then continues with banned ids at -inf, lowest
    first (text ids 0, 1, ... when the mass rule bans text), and -inf scores of different beams tie exactly.  The
    timestamp equal to eot's logit makes lse_ts == max_text exactly: the strict ">" keeps text in the select kernel."""
    eng = engines[V]
    C = 3
    n = C * beam
    sup = list(_sup()) + list(range(EOT + 1, TB))
    x = torch.full((n, V), -20.0)
    x[:, EOT] = 7.0
    vals = [7.0, 8.0, 6.0]                               # per clip: equal (no ban), above (text banned), below
    for c in range(C):
        x[c * beam:(c + 1) * beam, V - 1] = vals[c]
    prefix = torch.tensor([[SOT, TB + 3, 400 + j, V - 1] for j in range(n)])
    sums = -torch.arange(n, dtype=torch.float32) * 0.3
    banned = S.banned_by_index(x, prefix, 1, sup, True, 50)
    assert (~banned).sum(-1).tolist() == [2] * n
    assert _check_beam(eng, x, prefix, 1, sums, C, beam, beam, True, suppress=sup) == C
    # equal: text stays, every eot finishes; above: text (eot with it) banned, nothing finishes; below: eot finishes
    assert eng.fin_count[:C].cpu().tolist() == [beam, 0, beam]
    # eot alone: every eot finishes, the kept beams are -inf continuations of beam 0 (ties in (beam, rank) order)
    sup_eot = sup + [V - 1]
    fc = [0] * C
    assert _check_beam(eng, x, prefix, 1, sums, C, beam, 2 * beam, True, fc, suppress=sup_eot) == C
    assert (eng.src_rows[:n].cpu() % beam == 0).all()
    assert eng.fin_count[:C].cpu().tolist() == [beam] * C


@pytest.mark.parametrize("V", WIDTHS)
def test_beam_done_state_is_frozen(engines, V):
    eng = engines[V]
    C, beam = 2, 5
    x, sums = _beam_rows(C, beam, V, 3, torch.bfloat16, False)
    prefix = _prefix(C * beam, 30, 4)
    toks, got_sums, src, cnt, lens, fin, scores, before, _ = _beam_launch(eng, x, prefix, 1, sums, C, beam, 5, True, [5, 5], done=1)
    assert torch.equal(eng.tokens.cpu(), before[0].cpu()) and torch.equal(eng.sum_logprobs.cpu(), before[1].cpu())
    for t, b in zip((eng.fin_tokens, eng.fin_scores, eng.fin_len, eng.fin_count), before[2:]):
        assert torch.equal(t, b)
    assert src.tolist() == list(range(C * beam)) and int(eng.pos.item()) == 31 and int(eng.done.item()) == 1


@pytest.mark.parametrize("V", WIDTHS)
def test_beam_gives_the_same_bits_in_every_clip_slot(engines, V):
    eng = engines[V]
    beam, C = 2, 4
    x1, s1 = _beam_rows(1, beam, V, 11, torch.float16, False)
    x, sums = x1.repeat(C, 1), s1.repeat(C)
    prefix = _prefix(beam, 50, 5).repeat(C, 1)
    toks, got_sums, src, *_ = _beam_launch(eng, x, prefix, 1, sums, C, beam, beam, True)
    for c in range(1, C):
        assert torch.equal(toks[c * beam:(c + 1) * beam], toks[:beam])
        assert torch.equal(got_sums[c * beam:(c + 1) * beam].view(torch.int32), got_sums[:beam].view(torch.int32))
        assert (src[c * beam:(c + 1) * beam] - c * beam).tolist() == src[:beam].tolist()


# ---- harvested rows --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("variant,layout,dtype", [("tiny", "inference", torch.float16), ("tiny", "inference", torch.bfloat16),
                                                  ("small", "inference", torch.float16), ("small", "inference", torch.bfloat16),
                                                  ("tiny", "training", torch.float16), ("tiny", "training", torch.bfloat16)])
def test_harvested_rows(variant, layout, dtype):
    """Real logits rows: every replay of the engine's step is checked against the statement on the rows it wrote."""
    if layout == "training":
        m, sd, dims, OM, xa = _train_layout_model()
    else:
        m, sd, dims, OM, xa = _build(variant, emb_scale=SHARPEN[variant][0], pos_scale=SHARPEN[variant][1], n_clips=3)
    eng = m.decode_engine(dtype)
    sup = _sup()
    ties2 = tiesk = beam_decided = beam_total = 0
    for form in ("plain", "ts", "sample", "sample_ts", "beam"):
        C = xa.shape[0]
        beam = 5 if form == "beam" else 1
        n = C * beam
        ts = form in ("ts", "sample_ts", "beam")
        init = [SOT] if ts else [SOT, 50362]
        eng.prepare(xa)
        eng.reset(n, torch.tensor([init]).repeat(n, 1), None, sup, True, 0)
        keys = [H.row_key(4, c, 0) for c in range(n)]
        if form == "beam":
            eng.reset_beam(C, beam, beam, True, 50)
        else:
            eng._rules_cfg = None if form == "plain" else (int(ts), 50, int(form.startswith("sample")))
            if form.startswith("sample"):
                eng.temperature.fill_(0.6)
                eng.row_keys[:n] = torch.tensor([k - (1 << 64) if k >> 63 else k for k in keys], dtype=torch.int64).cuda()
        g = eng._graph(n)
        for _ in range(len(init) - 1):
            g.replay()
        for step in range(10):
            pos = int(eng.pos.item())
            prefix = eng.tokens[:n, :pos + 1].cpu().long()
            sums = eng.sum_logprobs[:n].cpu().clone()
            fc = eng.fin_count[:C].cpu().tolist()
            if form == "beam" and int(eng.done.item()):
                break
            g.replay()
            torch.cuda.synchronize()
            x = eng.logits[:n].cpu().clone()
            banned = S.banned_by_index(x, prefix, len(init), sup, ts, 50 if ts else None)
            for r in range(n):
                f = np.sort(S.filtered(x[r].numpy(), banned[r], False))[::-1]
                ties2 += int(f[0] == f[1])
                tiesk += int(np.isfinite(f[:6]).all() and len(set(f[:6].tolist())) < 6)
            if form == "beam":
                cnt, lens, fin, scores = (t.cpu() for t in eng.finished_lists(C, beam))
                toks, got_sums, src = eng.tokens[:n, :pos + 2].cpu(), eng.sum_logprobs[:n].cpu(), eng.src_rows[:n].cpu()
                for c in range(C):
                    rows = slice(c * beam, (c + 1) * beam)
                    new = [(float(scores[c, i]), fin[c, i, : int(lens[c, i])].tolist()) for i in range(fc[c], int(cnt[c]))]
                    res = S.check_beam_step(x[rows].numpy(), banned[rows], timestamps=True, sums=sums[rows].numpy(),
                                            prefix=prefix[rows].tolist(), pos=pos, beam=beam, max_cand=beam,
                                            fin_count=fc[c], first=pos == 0, got_tokens=toks[rows].tolist(),
                                            got_sums=got_sums[rows].numpy(), got_src=(src[rows] - c * beam).tolist(),
                                            got_fin=new)
                    beam_decided += res["decided"]
                    beam_total += 1
                    _note(f"harvested beam {variant} {layout} {dtype}", res["ratio"])
            else:
                nxt = eng.tokens[:n, pos + 1].cpu()
                r = S.check_sample_step(x.numpy(), banned, timestamps=ts, prev=prefix[:, -1], sum_in=sums.numpy(),
                                        got_next=nxt.numpy(), got_sum=eng.sum_logprobs[:n].cpu().numpy(),
                                        temperature=0.6 if form.startswith("sample") else 0.0, keys=keys, pos=pos)
                _note(f"harvested {form} {variant} {layout} {dtype}", r)
    print(f"harvested {variant} {layout} {dtype}: {ties2} rows with an exact top-2 tie, {tiesk} with a tie among the top 6; "
          f"beam steps decided {beam_decided}/{beam_total}")
    assert beam_decided >= 0.5 * beam_total > 0


# ---- end to end on a training-layout model ------------------------------------------------------------------------------
def _train_layout_model():
    import olmoasr_b200 as ob
    from olmoasr_b200 import synthetic
    from olmoasr_b200.model import OLMoASR
    from oracle import logmel
    from oracle import model as OM

    dims = OM.variant_dims("tiny")
    sd = OM.init_state_dict(dims, 0, train=True)
    g = torch.Generator().manual_seed(7)
    sd["decoder.positional_embedding"] = torch.randn(448, dims.n_text_state, generator=g) * SHARPEN["tiny"][1]
    sd["decoder.token_embedding.weight"] = sd["decoder.token_embedding.weight"] * SHARPEN["tiny"][0]
    m = OLMoASR(ob.VARIANT_TO_DIMS["tiny"])
    m.load_state_dict(sd)
    m = m.cuda()
    assert m.decoder.token_embedding.weight.shape[0] == 51865
    mel = torch.from_numpy(logmel.log_mel_spectrogram(synthetic.waveforms(3).numpy())).cuda()
    with torch.no_grad():
        xa = m.encoder(mel)
    return m, {k: v.cuda() for k, v in sd.items()}, dims, OM, xa


def test_training_layout_greedy_with_timestamps_matches_the_hook_loop(monkeypatch):
    """decode() on the engine and on the hook loop (OASR_DECODE_ENGINE=0) of the same training-layout model, compared up
    to the first step whose margin in the training oracle's greedy loop is within rounding noise (the rule of
    tests/test_sampling_gpu.py)."""
    from olmoasr_b200 import decoding as D
    from tests.test_sampling_gpu import SURE, _ref_greedy_ts

    m, sd, dims, OM, xa = _train_layout_model()
    n_steps = 24
    opts = D.DecodingOptions(without_timestamps=False, sample_len=n_steps, fp16=True)
    task = D.DecodingTask(m, opts)
    _, rel, _, _ = _ref_greedy_ts(OM, sd, dims, xa, torch.float16, n_steps, task.suppress,
                                  task.ts_rules.max_initial_timestamp_index, train_model=True)
    n_cmp = next((i for i, r in enumerate(rel) if r < SURE[torch.float16]), len(rel))
    got = D.decode(m, xa, opts)
    monkeypatch.setattr(D, "USE_ENGINE", False)
    want = D.decode(m, xa, opts)
    print(f"training layout greedy+ts: min relative margin {min(rel):.4f}, decided steps {n_cmp}/{len(rel)}; "
          f"tokens {got[0].tokens[:8]}")
    assert n_cmp >= 4, "sharpening failed: the comparison would be decided by rounding noise from the start"
    for g, w in zip(got, want):
        assert g.tokens[:n_cmp] == w.tokens[:n_cmp]
        if n_cmp == len(rel):
            assert g.tokens == w.tokens
            assert abs(g.avg_logprob - w.avg_logprob) <= 2e-2 * abs(w.avg_logprob) + 1e-3
        assert abs(g.no_speech_prob - w.no_speech_prob) <= 0.05 * w.no_speech_prob + 1e-6
        assert not g.tokens or g.tokens[0] >= TB


def test_training_layout_beam_with_timestamps_matches_the_reference():
    from olmoasr_b200.decoding import DecodingOptions, DecodingTask, decode
    from tests import beam_reference as R

    m, sd, dims, OM, xa = _train_layout_model()
    beam = 5
    opts = DecodingOptions(beam_size=beam, without_timestamps=False, sample_len=24, fp16=True)
    task = DecodingTask(m, opts)
    mi = task.ts_rules.max_initial_timestamp_index
    res = decode(m, xa, opts)
    ref = R.beam_decode(sd, dims, xa, beam, list(task.initial_tokens), 24, dtype=torch.float16, suppress=task.suppress,
                        timestamps=True, max_initial_timestamp_index=mi, train_model=True)
    rel = [min(min(gp), mm) / sc for gp, mm, sc in zip(ref.gaps, ref.mass_margins, ref.logit_scale)]
    n_cmp = next((i for i, r in enumerate(rel) if r < 8e-3), len(rel))
    print(f"training layout beam+ts: decided steps {n_cmp}/{len(rel)}; tokens {res[0].tokens[:8]}")
    # this model's beams repeat one token, so their scores fall within rounding noise after the first step (measured:
    # 1 decided step of 24 on an H100); test_harvested_rows holds every step of its beams to the fp64 statement instead
    assert n_cmp >= 1, "sharpening failed: the comparison would be decided by rounding noise from the start"
    for c in range(xa.shape[0]):
        assert abs(res[c].no_speech_prob - ref.no_speech_probs[c]) <= 0.05 * ref.no_speech_probs[c] + 1e-6
        if n_cmp == len(rel):
            assert res[c].tokens == ref.tokens[c]
            assert abs(res[c].avg_logprob - ref.avg_logprobs[c]) <= 2e-2 * abs(ref.avg_logprobs[c]) + 1e-3
        want = [tuple(r) for r in ref.steps[n_cmp - 1][c * beam:(c + 1) * beam].tolist()] if n_cmp else []
        if want and n_cmp < len(rel):
            init = list(task.initial_tokens)
            assert any(tuple(init + res[c].tokens)[: len(w)] == w for w in want) or len(res[c].tokens) < n_cmp
        if res[c].tokens:
            assert res[c].tokens[0] >= TB


def test_training_layout_transcribe_runs_on_the_device(monkeypatch):
    from olmoasr_b200 import synthetic
    import olmoasr_b200.transcribe as T

    m = _train_layout_model()[0]

    def no_hooks():
        raise AssertionError("a window took the hook loop")

    monkeypatch.setattr(m, "install_kv_cache_hooks", no_hooks)
    torch.manual_seed(0)
    out = T.transcribe(m, synthetic.waveforms(1, n_samples=40 * 16000)[0], sample_len=48)
    assert out["segments"] is not None
    print(f"training layout transcribe: {len(out['segments'])} segments")
