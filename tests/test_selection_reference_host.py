"""tests/selection_reference.py on the CPU: its fp64 statements of greedy, sampling and beam-search selection agree with
the fp32 restatements the GPU suites use (test_sampling_host.filter_row / sample_ids, beam_reference.beam_update) on
continuous rows, and reject deliberately wrong selections at both vocabulary widths (51864: inference layout, 51865:
training layout with the pad row), each by a stated margin."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from olmoasr_b200 import decoding as D
from tests import beam_reference as BR
from tests import selection_reference as S
from tests import test_sampling_host as H

EOT, SOT, TB, NS = S.EOT, H.SOT, S.TB, S.NO_SPEECH
SUP = D.suppress_token_ids(D.DecodingOptions())
WIDTHS = [51864, 51865]


def _q16(x):
    return x.to(torch.bfloat16).float()


def _rows(n, V, seed, scale=3.0):
    return torch.randn(n, V, generator=torch.Generator().manual_seed(seed)) * scale


def test_depth_and_bounds_follow_the_launch_geometry():
    assert S.slice_len(51864) == 3244 and S.slice_len(51865) == 3244
    assert 15 * 3244 + 3204 == 51864 and 15 * 3244 + 3205 == 51865     # the last slice: 801 float4s, or 801 and a tail
    assert S.sum_depth(51864) == 16 + 5 + 8 + 16 + 1
    assert S.lse_bound(51864, 20.0, 19.0) < 3e-5


@pytest.mark.parametrize("V", WIDTHS)
def test_greedy_statement_agrees_with_the_fp32_restatement(V):
    n = 12
    x = _rows(n, V, 1)
    x[1::3, TB:] += 6.0                               # the mass rule bans text on these rows
    tokens = torch.tensor([[SOT, TB + 2, 400]] * n)
    banned = S.banned_by_index(x, tokens, 1, SUP, True, 50)
    f = H.filter_row(x, tokens, 1, SUP, True, 50)
    nxt = f.argmax(-1)
    lp = F.log_softmax(f, -1)[torch.arange(n), nxt]
    sums = -torch.rand(n, generator=torch.Generator().manual_seed(2)) * 5
    ratio = S.check_sample_step(x.numpy(), banned, timestamps=True, prev=tokens[:, -1], sum_in=sums.numpy(),
                                got_next=nxt.numpy(), got_sum=(sums + lp).numpy())
    assert ratio < 1
    assert all(int(t) >= TB for t in nxt[1::3])


@pytest.mark.parametrize("V", WIDTHS)
def test_sampling_statement_agrees_with_the_numpy_draw(V):
    n, T, pos = 10, 0.6, 2
    x = _rows(n, V, 3)
    tokens = torch.tensor([[SOT, TB + 2, 400]] * n)
    banned = S.banned_by_index(x, tokens, 1, SUP, True, 50)
    f = H.filter_row(x, tokens, 1, SUP, True, 50)
    keys = [H.row_key(5, c, 0) for c in range(n)]
    ids, _ = H.sample_ids(f.numpy(), keys, pos, T)
    lp = F.log_softmax(f, -1)[torch.arange(n), torch.from_numpy(ids)]
    assert S.check_sample_step(x.numpy(), banned, timestamps=True, prev=tokens[:, -1], sum_in=np.zeros(n), got_next=ids,
                               got_sum=lp.numpy(), temperature=T, keys=keys, pos=pos) < 1


def _beam_case(V, beam, seed, first=False, twins=False):
    x = _rows(beam, V, seed)
    if first:
        x[:] = x[0]
    prefix = torch.tensor([[SOT, TB + 2, 400 + j] for j in range(beam)])
    sums = (-torch.rand(beam, generator=torch.Generator().manual_seed(seed + 1)) * 3).float()
    if first:                                           # every beam holds the same prefix and sum
        prefix = torch.tensor([[SOT]] * beam)
        sums[:] = sums[0]
    x[::2, EOT] = x[::2].max(-1).values + 0.5          # some rows want to end
    if twins:                                           # beams 0 and 1: one row, one sum -> exact cross-beam ties
        x[1] = x[0]
        sums[1] = sums[0]                               # (the prefixes differ: upstream's dict would merge equal ones)
    return _q16(x), prefix, sums


def _run_beam_update(x, prefix, sums, beam, max_cand, sb):
    st = BR.BeamState(beam, max_cand)
    lp = F.log_softmax(H.filter_row(x, prefix, sb, SUP, True, 50), -1)
    s = sums.clone()
    toks, src, _ = BR.beam_update(st, prefix, lp, s)
    fin = [(sc, list(seq)) for seq, sc in st.finished[0].items()]
    return toks, s, src, fin


@pytest.mark.parametrize("V", WIDTHS)
@pytest.mark.parametrize("beam", [2, 5])
def test_beam_statement_agrees_with_beam_update(V, beam):
    for seed, first, twins in ((10, False, False), (11, True, False), (12, False, True)):
        x, prefix, sums = _beam_case(V, beam, seed, first, twins)
        sb = 1
        toks, s, src, fin = _run_beam_update(x, prefix, sums, beam, beam, sb)
        banned = S.banned_by_index(x, prefix, sb, SUP, True, 50)
        res = S.check_beam_step(x.numpy(), banned, timestamps=True, sums=sums.numpy(), prefix=prefix.tolist(),
                                pos=prefix.shape[1] - 1, beam=beam, max_cand=beam, fin_count=0, first=first,
                                got_tokens=toks.tolist(), got_sums=s.numpy(), got_src=src, got_fin=fin)
        assert res["decided"] and res["ratio"] < 1, (seed, res)


# ---- wrong selections are rejected -------------------------------------------------------------------------------------
@pytest.mark.parametrize("V", WIDTHS)
def test_rejects_ties_to_the_highest_id(V):
    x = _q16(_rows(1, V, 20))
    top = float(x.max()) + 1.0
    for a, b in ((1022, 1025), (127, 128), (3242, 3245), (40000, 50000)):   # threads, warps, slices, far apart
        y = x.clone()
        y[0, a] = y[0, b] = top
        tokens = torch.tensor([[SOT, TB + 2, 400]])
        banned = S.banned_by_index(y, tokens, 1, SUP, True, None)
        lse = torch.logsumexp(torch.from_numpy(S.filtered(y[0].numpy(), banned[0], False)), 0)
        kw = dict(timestamps=True, prev=[400], sum_in=[0.0], got_sum=[float(top - lse)])
        S.check_sample_step(y.numpy(), banned, got_next=[a], **kw)
        with pytest.raises(AssertionError, match="lowest-id argmax"):
            S.check_sample_step(y.numpy(), banned, got_next=[b], **kw)


@pytest.mark.parametrize("V", WIDTHS)
def test_rejects_the_mass_rule_with_greater_or_equal(V):
    """One allowed timestamp equal to the text maximum: lse_ts == max_text exactly, so text stays (strict >) and the
    tie between the text maximum and the timestamp goes to the lower id."""
    x = torch.full((1, V), -20.0)
    x[0, EOT] = 7.0
    x[0, V - 1] = 7.0                                        # at V = 51865 the pad id, a timestamp to the hook loop
    tokens = torch.tensor([[SOT, TB + 3, 400, V - 1]])       # an open segment: eot or the last timestamp
    banned = S.banned_by_index(x, tokens, 1, SUP, True, None)
    assert (~banned[0, TB:]).sum() == 1 and not banned[0, EOT] and banned[0, :EOT].all()
    gap, bound = S.mass_gap(x[0].numpy(), banned[0])
    assert gap == 0.0 and bound == 0.0
    assert S.mass_branches(x[0].numpy(), banned[0], True) == [False]
    f = S.filtered(x[0].numpy(), banned[0], False)
    lp = 7.0 - float(torch.logsumexp(torch.from_numpy(f), 0))
    S.check_sample_step(x.numpy(), banned, timestamps=True, prev=[V - 1], sum_in=[0.0], got_next=[EOT], got_sum=[lp])
    lp_ts = 0.0                                              # text banned: the timestamp is the whole distribution
    with pytest.raises(AssertionError):
        S.check_sample_step(x.numpy(), banned, timestamps=True, prev=[V - 1], sum_in=[0.0], got_next=[V - 1],
                            got_sum=[lp_ts])


@pytest.mark.parametrize("V", WIDTHS)
def test_rejects_a_cross_beam_tie_broken_by_the_later_candidate(V):
    beam = 5
    x, prefix, sums = _beam_case(V, beam, 30, twins=True)
    toks, s, src, fin = _run_beam_update(x, prefix, sums, beam, beam, 1)
    banned = S.banned_by_index(x, prefix, 1, SUP, True, 50)
    kw = dict(timestamps=True, sums=sums.numpy(), prefix=prefix.tolist(), pos=2, beam=beam, max_cand=beam, fin_count=0,
              first=False, got_fin=fin)
    S.check_beam_step(x.numpy(), banned, got_tokens=toks.tolist(), got_sums=s.numpy(), got_src=src, **kw)
    k = next(k for k in range(beam - 1) if src[k] == 0 and src[k + 1] == 1 and int(toks[k, -1]) == int(toks[k + 1, -1]))
    wrong = list(src)
    wrong[k], wrong[k + 1] = 1, 0                            # the twin of beam 1 first
    with pytest.raises(AssertionError, match="source"):
        S.check_beam_step(x.numpy(), banned, got_tokens=toks.tolist(), got_sums=s.numpy(), got_src=wrong, **kw)


@pytest.mark.parametrize("V", WIDTHS)
def test_rejects_no_speech_from_the_filtered_row(V):
    x = _q16(_rows(3, V, 40))
    x[:, NS] = x.max(-1).values - 2.0
    raw = torch.softmax(x.double(), -1)[:, NS]
    assert S.check_no_speech(x.numpy(), raw.numpy()) < 1
    f = x.clone()
    f[:, SUP] = -math.inf                                    # no_speech is a suppressed id: 0 after the filter
    wrong = torch.softmax(f.double(), -1)[:, NS]
    with pytest.raises(AssertionError, match="no_speech"):
        S.check_no_speech(x.numpy(), wrong.numpy())
    # the filtered normaliser alone (no_speech itself kept) is off by far more than the bound
    f[:, NS] = x[:, NS]
    near = torch.softmax(f.double(), -1)[:, NS]
    b = (S.sum_depth(V) * 6 * S.U + 5 * S.U + 3 * S.U) * raw
    assert float(((near - raw).abs() / b).min()) > 10


@pytest.mark.parametrize("V", WIDTHS)
def test_rejects_the_log_prob_at_temperature_t(V):
    n, T, pos = 6, 0.4, 3
    x = _q16(_rows(n, V, 50))
    tokens = torch.tensor([[SOT, TB + 2, 400, 401]] * n)
    banned = S.banned_by_index(x, tokens, 1, SUP, True, 50)
    f = H.filter_row(x, tokens, 1, SUP, True, 50)
    keys = [H.row_key(8, c, 1) for c in range(n)]
    ids, _ = H.sample_ids(f.numpy(), keys, pos, T)
    idx = torch.from_numpy(ids)
    kw = dict(timestamps=True, prev=tokens[:, -1], sum_in=np.zeros(n), got_next=ids, temperature=T, keys=keys, pos=pos)
    S.check_sample_step(x.numpy(), banned, got_sum=F.log_softmax(f, -1)[torch.arange(n), idx].numpy(), **kw)
    wrong = F.log_softmax(f / T, -1)[torch.arange(n), idx]
    right = F.log_softmax(f.double(), -1)[torch.arange(n), idx]
    assert float((wrong - right).abs().min()) > 1000 * S.lse_bound(V, 30.0, 29.0)
    with pytest.raises(AssertionError, match="bound"):
        S.check_sample_step(x.numpy(), banned, got_sum=wrong.numpy(), **kw)


@pytest.mark.parametrize("V", WIDTHS)
def test_beam_rows_with_fewer_allowed_ids_than_candidates_are_decided(V):
    """An open segment at the last timestamp with the special ids suppressed leaves eot and one timestamp: the top
    beam + 1 continues with banned ids at -inf (lowest ids first), and -inf scores of different beams tie exactly."""
    beam = 5
    for ts_val in (7.0, 8.0, 6.0, None):        # equal to eot (no ban, the strict ">"), above (text banned), below; eot only
        sup = list(SUP) + list(range(EOT + 1, TB)) + ([V - 1] if ts_val is None else [])
        x = torch.full((beam, V), -20.0)
        x[:, EOT] = 7.0
        x[:, V - 1] = 0.0 if ts_val is None else ts_val
        prefix = torch.tensor([[SOT, TB + 3, 400 + j, V - 1] for j in range(beam)])
        sums = -torch.arange(beam, dtype=torch.float32) * 0.3
        st = BR.BeamState(beam, beam)
        lp = F.log_softmax(H.filter_row(x, prefix, 1, sup, True, 50), -1)
        s = sums.clone()
        toks, src, _ = BR.beam_update(st, prefix, lp, s)
        fin = [(sc, list(seq)) for seq, sc in st.finished[0].items()]
        banned = S.banned_by_index(x, prefix, 1, sup, True, 50)
        assert (~banned).sum(-1).tolist() == [1 if ts_val is None else 2] * beam
        res = S.check_beam_step(x.numpy(), banned, timestamps=True, sums=sums.numpy(), prefix=prefix.tolist(), pos=3,
                                beam=beam, max_cand=beam, fin_count=0, first=False, got_tokens=toks.tolist(),
                                got_sums=s.numpy(), got_src=src, got_fin=fin)
        assert res["decided"], ts_val
        if ts_val is not None:
            continue
        assert all(math.isinf(float(v)) for v in s) and len(fin) == beam     # every eot finished, -inf beams kept
        wrong = list(src)
        assert src == [0] * beam                            # -inf ties in (beam, rank) order: beam 0's ranks first
        wrong[0] = 1                                        # the tie broken by the later beam
        with pytest.raises(AssertionError):
            S.check_beam_step(x.numpy(), banned, timestamps=True, sums=sums.numpy(), prefix=prefix.tolist(), pos=3,
                              beam=beam, max_cand=beam, fin_count=0, first=False, got_tokens=toks.tolist(),
                              got_sums=s.numpy(), got_src=wrong, got_fin=fin)
