"""fp64 statements of the device decoder's token selection and the bounds its tests use (TEST INFRASTRUCTURE).

csrc/decode.cu turns one fp32 logits row into one token in three kernel families: dec_sample_kernel<TS, SAMPLING>
(greedy, greedy with timestamp rules, temperature sampling, sampling with timestamp rules), dec_beam_cand_kernel and
dec_beam_select_kernel.  This module states one step of each in fp64 over the fp32 rows the kernels read, and checks a
kernel's outputs against the statement.  The index rules (SuppressTokens, SuppressBlank, ApplyTimestampRules) are the
hook loop's own, through tests/test_sampling_host.filter_row; only the "timestamp mass beats every text token" decision
is restated, in fp64, as gap = lse(allowed timestamps) - max(allowed text).

Exact parts (the inputs are fp32 values, so fp64 compares them without error):
    greedy        next = the lowest id among the maxima of the filtered row
    candidates    a beam row's top beam + 1 by (value desc, id asc); banned ids take part as -inf, so a row with fewer
                  allowed ids than beam + 1 continues with the lowest banned ids (with text banned by the mass rule: the
                  text ids 0, 1, 2, ... before any banned timestamp)
    ties          equal scores of one row are equal in every precision; candidates of bit-identical rows with
                  bit-identical sums are equal too.  Both are ordered by (beam, rank), Python's stable sort over
                  BeamSearchDecoder's insertion order
    first step    only beam 0's candidates exist (upstream's dict keyed by sequence collapses the identical beams)
    finished      eot candidates in walk order while the list has room: score, the source prefix + eot, length pos + 2
    frozen        a finished row (previous token eot) emits eot and keeps its sum; a beam step with done set changes
                  nothing but the position

Bounds (u = 2^-24; CUDA's expf is within 2 ulp = 4u relative, logf within 1 ulp; IEEE +, *, / within u).  Every
(max, sum exp) in the kernels is an online accumulation whose levels each compute s = s_a e_a + s_b e_b: 6u of
relative error per level.  The depth is counted from the code (sum_depth):
    per-thread chain  one level per id a thread visits: 4 ids per float4 group, ceil(slice / 1024) groups, where a
                      slice is ceil(V / 16) rounded up to a multiple of 4 (3244 ids at V = 51864 and 51865)
    butterfly         5 shuffle levels;  warps  8 (merged into an empty accumulator);  slices  16 (likewise)
    regions           1 for merging the text and timestamp statistics (greedy / sampling) or the log1p of their lse
so the sum carries at most depth 6u relative error, and lse = m + logf(s) at most depth 6u + 2u |log s| + u |lse|.
    mass rule     the kernel compares lse_ts (fp32) > max_text (exact): decided where |gap| > lse bound.  A timestamp
                  region with a single allowed id has s = 1 exactly and log 1 = 0, so its gap is exact: the strict ">"
                  at gap == 0 is pinned, in dec_sample_kernel and in dec_beam_select_kernel alike.  Undecided rows
                  may take either branch; the rest of the step must follow one.
    log-prob      greedy -logf(s): depth 6u + 2u |log s|; sampling (x - m) - logf(s) adds u |x - m| + u |lp|; beam
                  v - lse over the two regions' lse adds the log1p(exp) merge (4u + 4u) and u |lp|
    sums          + u |sum| for the fp32 add
    no_speech     expf(x - m_raw) / s_raw relative: depth 6u + u |x - m_raw| + 4u + u
    Gumbel draw   g = -logf(-logf(u)) from 23 Philox bits (exact u): |g32 - g| <= 3u + 2u |g|; y = x / T + g adds
                  u |x / T| + u |y|.  The draw is decided where every other id's fp64 y is below the best by more
                  than the sum of the two bounds.

    -inf ties     candidates at -inf (banned ids filling a row with fewer allowed ids than beam + 1) tie exactly across
                  rows too: they are ordered by (beam, rank) like any exact tie

tests/test_selection_parity_gpu.py prints the largest error-to-bound ratio of every form (log-prob sums, no-speech
probabilities); tools/selection_error_table.py runs it and prints that line.  A test fails where a ratio exceeds 1, so
the ratios say how much room the bounds leave.  They have not been measured yet: no table is kept here.
"""
from __future__ import annotations

import math
from typing import List, Optional, Sequence

import numpy as np
import torch

from tests import test_sampling_host as H

U = 2.0 ** -24
EOT, NO_SPEECH, TB = H.EOT, 50361, H.TB
SLICES = 16


def slice_len(V: int, S: int = SLICES) -> int:
    return ((V + S - 1) // S + 3) & ~3


def sum_depth(V: int, S: int = SLICES) -> int:
    """Levels of the longest online (max, sum exp) chain from one logit to a row's statistics (module docstring)."""
    return 4 * math.ceil(slice_len(V, S) / 1024) + 5 + 8 + S + 1


def lse_bound(V: int, lse: float, m: float) -> float:
    """|fp32 m + logf(s) - fp64 lse| for a region whose max is m (exact)."""
    return sum_depth(V) * 6 * U + 2 * U * abs(lse - m) + U * abs(lse)


def _lse(x: np.ndarray) -> float:
    m = float(x.max()) if x.size else -math.inf
    if m == -math.inf:
        return -math.inf
    return m + math.log(float(np.exp(x - m).sum()))


# ---- filters -------------------------------------------------------------------------------------------------------------
def banned_by_index(logits: torch.Tensor, tokens: torch.Tensor, sample_begin: int, suppress: Sequence[int], timestamps: bool,
                    mi: Optional[int], suppress_blank: bool = True) -> np.ndarray:
    """(n, V) bool: the ids the hook loop's index rules ban for `tokens` (the rows up to the current position).  The
    text region is lifted out of reach first so that the mass rule cannot fire; it is decided separately (mass_gap)."""
    lifted = logits.clone().float()
    if timestamps:
        lifted[:, :TB] = 1e4
    return torch.isinf(H.filter_row(lifted, tokens, sample_begin, suppress, timestamps, mi, suppress_blank)).numpy()


def mass_gap(x: np.ndarray, banned: np.ndarray):
    """(gap, bound) of one row: lse(allowed timestamps) - max(allowed text) in fp64, and how far the kernel's fp32 lse
    may sit from it (0 when a single timestamp is allowed: s = 1 and log 1 = 0 exactly)."""
    V = x.shape[0]
    xs = x[TB:][~banned[TB:]].astype(np.float64)
    xt = x[:TB][~banned[:TB]].astype(np.float64)
    lse_ts = _lse(xs)
    m_text = float(xt.max()) if xt.size else -math.inf
    if lse_ts == -math.inf or m_text == -math.inf:
        return lse_ts - m_text if lse_ts != m_text else -math.inf, 0.0
    bound = 0.0 if xs.size == 1 else lse_bound(V, lse_ts, float(xs.max()))
    return lse_ts - m_text, bound


def mass_branches(x, banned, timestamps: bool) -> List[bool]:
    """The values of "text banned by the mass rule" the kernel may take on this row."""
    if not timestamps:
        return [False]
    gap, bound = mass_gap(x, banned)
    if abs(gap) > bound or bound == 0.0:
        return [gap > 0]
    return [False, True]


def filtered(x: np.ndarray, banned: np.ndarray, ban_text: bool) -> np.ndarray:
    f = x.astype(np.float64).copy()
    f[banned] = -math.inf
    if ban_text:
        f[:TB] = -math.inf
    return f


def gumbel64(key: int, pos: int, V: int) -> np.ndarray:
    """The kernel's Gumbel noise of one row in fp64 from the same Philox bits (tests/test_sampling_host.philox4x32_10)."""
    k = np.uint64(key & ((1 << 64) - 1))
    ids = np.arange(V, dtype=np.int64)
    words = H.philox4x32_10(ids >> 2, np.uint64(pos), k & np.uint64(0xFFFFFFFF), k >> np.uint64(32))
    bits = words[ids, ids & 3]
    u = ((bits >> np.uint64(9)).astype(np.float64) + 0.5) * 2.0 ** -23
    return -np.log(-np.log(u))


# ---- greedy and sampling -------------------------------------------------------------------------------------------------
def check_sample_step(x, banned, *, timestamps: bool, prev, sum_in, got_next, got_sum, temperature: float = 0.0,
                      keys=None, pos: int = 0, eot: int = EOT) -> float:
    """One dec_sample step over rows x (n, V) fp32.  Raises AssertionError where the kernel's choice contradicts the
    statement; returns the largest log-prob-sum error over its bound."""
    x = np.asarray(x, dtype=np.float32)
    n, V = x.shape
    T = float(np.float32(temperature))
    worst = 0.0
    for r in range(n):
        s_in, g_sum, g_next = float(np.float32(sum_in[r])), float(got_sum[r]), int(got_next[r])
        if int(prev[r]) == eot:
            assert g_next == eot and g_sum == s_in, f"row {r}: a finished row must emit eot and keep its sum"
            continue
        fails = []
        for ban_text in mass_branches(x[r], banned[r], timestamps):
            f = filtered(x[r], banned[r], ban_text)
            live = np.isfinite(f)
            if T > 0:
                y = np.where(live, f / T + gumbel64(int(keys[r]), pos, V), -math.inf)
                best = int(np.argmax(y))
                g = np.where(live, y - f / T, 0.0)
                yb = U * np.abs(f / T) + 3 * U + 2 * U * np.abs(g) + U * np.abs(y)
                close = live & (y[best] - y <= yb[best] + yb)
                if not close[g_next]:
                    fails.append(f"ban_text={ban_text}: drew {g_next}, fp64 draw {best} (margin to it "
                                 f"{y[best] - y[g_next] if live[g_next] else math.inf:.3g} > bound)")
                    continue
            else:
                best = int(np.argmax(f))
                if g_next != best:
                    fails.append(f"ban_text={ban_text}: picked {g_next}, lowest-id argmax {best}")
                    continue
            m = float(f[live].max())
            lse = _lse(f[live])
            lp = float(f[g_next]) - lse
            b = sum_depth(V) * 6 * U + 2 * U * abs(lse - m)
            if T > 0:
                b += U * abs(float(f[g_next]) - m) + U * abs(lp)
            want = s_in + lp
            b += U * abs(want)
            err = abs(g_sum - want)
            if err > b:
                fails.append(f"ban_text={ban_text}: sum {g_sum!r}, fp64 {want!r}, error {err:.3g} > bound {b:.3g}")
                continue
            worst = max(worst, err / b)
            break
        else:
            raise AssertionError(f"row {r}: " + "; ".join(fails))
    return worst


def check_no_speech(x, got) -> float:
    """no_speech_prob = softmax(raw row)[NO_SPEECH] within its relative bound; returns the largest error over bound."""
    x = np.asarray(x, dtype=np.float32).astype(np.float64)
    V = x.shape[1]
    worst = 0.0
    for r in range(x.shape[0]):
        m = float(x[r].max())
        want = math.exp(float(x[r, NO_SPEECH]) - _lse(x[r]))
        b = (sum_depth(V) * 6 * U + U * abs(float(x[r, NO_SPEECH]) - m) + 5 * U) * want + 1e-45
        err = abs(float(got[r]) - want)
        assert err <= b, f"row {r}: no_speech {float(got[r])!r}, fp64 {want!r}, error {err:.3g} > bound {b:.3g}"
        worst = max(worst, err / b)
    return worst


# ---- beam search ---------------------------------------------------------------------------------------------------------
def row_candidates(f: np.ndarray, K: int):
    """Top K of a filtered row by (value desc, id asc), -inf entries included; returns (ids, values)."""
    idx = np.lexsort((np.arange(f.size), -f))[:K]
    return idx, f[idx]


def _beam_lp_bound(V, lse_t, m_t, lse_s, m_s, lse, lp):
    b = 0.0
    for l, m in ((lse_t, m_t), (lse_s, m_s)):
        if l != -math.inf:
            b += lse_bound(V, l, m)
    return b + 8 * U + U * abs(lse) + U * abs(lp)


def beam_statement(x, banned, *, timestamps: bool, sums, beam: int, first: bool, branches=None):
    """Per clip row j: candidates [(score64, bound, beam j, rank, token)] and the row signature (for exact ties)."""
    x = np.asarray(x, dtype=np.float32)
    n, V = x.shape
    K = beam + 1
    cands = []
    for j in range(n):
        if first and j > 0:
            break
        ban_text = branches[j] if branches is not None else mass_branches(x[j], banned[j], timestamps)[0]
        f = filtered(x[j], banned[j], ban_text)
        ft, fs = f[:TB], f[TB:]
        lt, ls = _lse(ft[np.isfinite(ft)]), _lse(fs[np.isfinite(fs)])
        lse = _lse(f[np.isfinite(f)])
        mt = float(ft.max()) if np.isfinite(ft).any() else -math.inf
        ms = float(fs.max()) if np.isfinite(fs).any() else -math.inf
        ids, vals = row_candidates(f, K)
        s_in = float(np.float32(sums[j]))
        sig = (x[j].tobytes(), banned[j].tobytes(), ban_text, np.float32(sums[j]).tobytes())
        for r, (tok, v) in enumerate(zip(ids.tolist(), vals.tolist())):
            lp = v - lse
            score = s_in + lp
            b = (_beam_lp_bound(V, lt, mt, ls, ms, lse, lp) + U * abs(score)) if math.isfinite(score) else 0.0
            cands.append((score, b, j, r, int(tok), sig))
    return cands


def _walk(cands, beam, max_cand, fin_count, eot):
    order = sorted(range(len(cands)), key=lambda i: (-cands[i][0], cands[i][2], cands[i][3]))
    kept, fin, walked, count = [], [], 0, fin_count
    for i in order:
        if len(kept) >= beam:
            break
        walked += 1
        c = cands[i]
        if c[4] == eot:
            if count < max_cand:
                fin.append(c)
                count += 1
        else:
            kept.append(c)
    return order, walked, kept, fin, count


def _decided(cands, order, walked) -> bool:
    """The fp32 scores keep the fp64 order over the walked candidates and the next one."""
    for a, b in zip(order[: walked], order[1: walked + 1]):
        ca, cb = cands[a], cands[b]
        if ca[2] == cb[2]:
            continue                                  # one row: rounding is monotone, ties go to the lower rank
        if ca[0] == cb[0] and (ca[5] == cb[5] or ca[0] == -math.inf):
            continue                                  # bit-identical rows and sums, or both -inf: an exact tie in every
                                                      # precision, ordered by (beam, rank)
        if not (ca[0] - cb[0] > ca[1] + cb[1]):
            return False
    return True


def check_beam_step(x, banned, *, timestamps: bool, sums, prefix, pos: int, beam: int, max_cand: int, fin_count: int,
                    first: bool, got_tokens, got_sums, got_src, got_fin, eot: int = EOT) -> dict:
    """One clip's dec_beam_cand + dec_beam_select step.  x, banned: the clip's beam rows; prefix: (beam, pos + 1) token
    rows before the step; got_tokens: (beam, pos + 2); got_src: clip-local source beams; got_fin: the entries the step
    appended to the finished list [(score, tokens)].  Returns {"decided": bool, "ratio": worst error over bound}."""
    x = np.asarray(x, dtype=np.float32)
    options = [[mass_branches(x[j], banned[j], timestamps) for j in range(x.shape[0])]]
    combos = [[]]
    for br in options[0]:
        combos = [c + [b] for c in combos for b in br]
    errors = []
    for combo in combos:
        cands = beam_statement(x, banned, timestamps=timestamps, sums=sums, beam=beam, first=first, branches=combo)
        order, walked, kept, fin, _ = _walk(cands, beam, max_cand, fin_count, eot)
        decided = len(combos) == 1 and _decided(cands, order, walked)
        try:
            ratio = 0.0
            if decided:
                for k, c in enumerate(kept):
                    src = 0 if first else c[2]
                    assert int(got_tokens[k][-1]) == c[4] and list(got_tokens[k][:-1]) == list(prefix[c[2]]), \
                        f"beam {k}: got token {int(got_tokens[k][-1])} from beam {int(got_src[k])}, want {c[4]} from {c[2]}"
                    if not first:
                        assert int(got_src[k]) == src, f"beam {k}: source {int(got_src[k])}, want {src}"
                    err = abs(float(got_sums[k]) - c[0]) if math.isfinite(c[0]) else (0.0 if got_sums[k] == c[0] else math.inf)
                    assert err <= c[1] or err == 0.0, f"beam {k}: score {float(got_sums[k])!r}, fp64 {c[0]!r}, bound {c[1]:.3g}"
                    ratio = max(ratio, err / c[1]) if c[1] > 0 else ratio
                assert len(got_fin) == len(fin), f"{len(got_fin)} finished, want {len(fin)}"
                for (gs, gt), c in zip(got_fin, fin):
                    assert list(gt) == list(prefix[c[2]]) + [eot] and len(gt) == pos + 2, "finished tokens"
                    err = 0.0 if float(gs) == c[0] else abs(float(gs) - c[0])
                    assert err <= c[1], f"finished score {float(gs)!r}, fp64 {c[0]!r}, bound {c[1]:.3g}"
                    ratio = max(ratio, err / c[1]) if c[1] > 0 else ratio
            else:                          # undecided order: every kept entry is a candidate with its score in bound
                by = {(0 if first else c[2], c[4]): c for c in cands}
                for k in range(len(got_tokens)):
                    c = by.get((int(got_src[k]) if not first else 0, int(got_tokens[k][-1])))
                    assert c is not None, f"beam {k}: ({int(got_src[k])}, {int(got_tokens[k][-1])}) is no candidate"
                    if math.isfinite(c[0]):
                        assert abs(float(got_sums[k]) - c[0]) <= c[1], f"beam {k}: score out of bound"
            return {"decided": decided, "ratio": ratio}
        except AssertionError as e:
            errors.append(f"branches {combo if len(combos) > 1 else 'decided'}: {e}")
    raise AssertionError("; ".join(errors))
