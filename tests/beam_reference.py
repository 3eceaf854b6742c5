"""CPU restatement of beam search in whisper/decoding.py (TEST INFRASTRUCTURE).

Written from the published algorithm -- BeamSearchDecoder.update / finalize, MaximumLikelihoodRanker,
DecodingTask._main_loop / run and ApplyTimestampRules -- in its own dict-keyed form, kept independent of olmoasr_b200
(no import of the package).  `beam_search` runs over any logits callback; `beam_decode` runs it over oracle/model.py's
decoder with the self-attention cache rearranged by `index_select`, as upstream's PyTorchInference.rearrange_kv_cache.

Besides the decode result it reports per step the *selection gap* of every clip: the score of the last kept beam minus the
score of the first candidate that was not walked (kept or finished).  Where that gap is within rounding noise, two correct
implementations may keep different beams.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import torch.nn.functional as F

EOT, SOT, NO_SPEECH, NO_TIMESTAMPS, TIMESTAMP_BEGIN = 50256, 50257, 50361, 50362, 50363
BLANK = 220


def apply_timestamp_rules(logits: torch.Tensor, tokens: torch.Tensor, sample_begin: int,
                          max_initial_timestamp_index: Optional[int]) -> None:
    """ApplyTimestampRules.apply, in place on (N, V) logits."""
    logits[:, NO_TIMESTAMPS] = -np.inf
    for k in range(tokens.shape[0]):
        sampled = tokens[k, sample_begin:]
        seq = sampled.tolist()
        last_was_timestamp = len(seq) >= 1 and seq[-1] >= TIMESTAMP_BEGIN
        penultimate_was_timestamp = len(seq) < 2 or seq[-2] >= TIMESTAMP_BEGIN
        if last_was_timestamp:
            if penultimate_was_timestamp:   # has to be non-timestamp
                logits[k, TIMESTAMP_BEGIN:] = -np.inf
            else:                           # cannot be normal text tokens
                logits[k, :EOT] = -np.inf
        timestamps = sampled[sampled.ge(TIMESTAMP_BEGIN)]
        if timestamps.numel() > 0:
            # timestamps shouldn't decrease; forbid timestamp tokens smaller than the last
            if last_was_timestamp and not penultimate_was_timestamp:
                timestamp_last = timestamps[-1]
            else:
                timestamp_last = timestamps[-1] + 1
            logits[k, TIMESTAMP_BEGIN:timestamp_last] = -np.inf
    if tokens.shape[1] == sample_begin:
        logits[:, :TIMESTAMP_BEGIN] = -np.inf
        if max_initial_timestamp_index is not None:
            logits[:, TIMESTAMP_BEGIN + max_initial_timestamp_index + 1:] = -np.inf
    # if sum of probability over timestamps is above any other token, sample timestamp
    logprobs = F.log_softmax(logits.float(), dim=-1)
    for k in range(tokens.shape[0]):
        timestamp_logprob = logprobs[k, TIMESTAMP_BEGIN:].logsumexp(dim=-1)
        max_text_token_logprob = logprobs[k, :TIMESTAMP_BEGIN].max()
        if timestamp_logprob > max_text_token_logprob:
            logits[k, :TIMESTAMP_BEGIN] = -np.inf


def topk_lowest_id(x: torch.Tensor, k: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """topk of a 1-D tensor with ties (including -inf) going to the lower index."""
    vals = x.double().numpy()
    idx = torch.from_numpy(np.lexsort((np.arange(vals.size), -vals))[:k].copy())
    return x[idx], idx


@dataclass
class BeamState:
    beam_size: int
    max_candidates: int
    finished: Optional[List[Dict[tuple, float]]] = None
    gaps: List[List[float]] = field(default_factory=list)   # per step, per clip


def beam_update(state: BeamState, tokens: torch.Tensor, logprobs: torch.Tensor,
                sum_logprobs: torch.Tensor) -> Tuple[torch.Tensor, List[int], bool]:
    """BeamSearchDecoder.update on (N, V) log-probs; updates sum_logprobs in place.  Returns (tokens, sources, completed)."""
    B = state.beam_size
    n_audio = tokens.shape[0] // B
    if state.finished is None:
        state.finished = [{} for _ in range(n_audio)]
    next_tokens, source_indices, finished_sequences, gaps = [], [], [], []
    for i in range(n_audio):
        scores, sources, finished = {}, {}, {}
        for j in range(B):
            idx = i * B + j
            prefix = tokens[idx].tolist()
            vals, ids = topk_lowest_id(logprobs[idx], B + 1)
            for logprob, token in zip(vals.tolist(), ids.tolist()):
                new_logprob = float(np.float32(sum_logprobs[idx].item()) + np.float32(logprob))   # fp32, as upstream
                sequence = tuple(prefix + [token])
                scores[sequence] = new_logprob
                sources[sequence] = idx
        order = sorted(scores, key=scores.get, reverse=True)
        saved = 0
        walked = 0
        for sequence in order:
            walked += 1
            if sequence[-1] == EOT:
                finished[sequence] = scores[sequence]
            else:
                sum_logprobs[len(next_tokens)] = scores[sequence]
                next_tokens.append(sequence)
                source_indices.append(sources[sequence])
                saved += 1
                if saved == B:
                    break
        last = scores[order[walked - 1]]
        gaps.append(last - scores[order[walked]] if walked < len(order) else float("inf"))
        finished_sequences.append(finished)
    state.gaps.append(gaps)
    for previously_finished, newly_finished in zip(state.finished, finished_sequences):
        for seq in sorted(newly_finished, key=newly_finished.get, reverse=True):
            if len(previously_finished) >= state.max_candidates:
                break
            previously_finished[seq] = newly_finished[seq]
    completed = all(len(s) >= state.max_candidates for s in state.finished)
    return torch.tensor(next_tokens, device=tokens.device), source_indices, completed


def beam_finalize(state: BeamState, preceding_tokens: torch.Tensor, sum_logprobs: torch.Tensor):
    """BeamSearchDecoder.finalize: (n_audio, beam, T) tokens, (n_audio, beam) sums -> candidate lists per clip."""
    sum_logprobs = sum_logprobs.cpu()
    for i, sequences in enumerate(state.finished):
        if len(sequences) < state.beam_size:
            for j in list(np.argsort(sum_logprobs[i]))[::-1]:
                sequence = preceding_tokens[i, j].tolist() + [EOT]
                sequences[tuple(sequence)] = sum_logprobs[i][j].item()
                if len(sequences) >= state.beam_size:
                    break
    tokens = [[list(seq) for seq in sequences.keys()] for sequences in state.finished]
    sums = [list(sequences.values()) for sequences in state.finished]
    return tokens, sums


def rank(tokens: List[List[List[int]]], sum_logprobs: List[List[float]], length_penalty: Optional[float]) -> List[int]:
    """MaximumLikelihoodRanker.rank."""
    out = []
    for toks, lps in zip(tokens, sum_logprobs):
        s = []
        for t, lp in zip(toks, lps):
            penalty = len(t) if length_penalty is None else ((5 + len(t)) / 6) ** length_penalty
            s.append(lp / penalty)
        out.append(int(np.argmax(s)))
    return out


@dataclass
class BeamResult:
    tokens: List[List[int]]           # selected sampled ids per clip (before eot)
    sum_logprobs: List[float]
    avg_logprobs: List[float]
    no_speech_probs: List[float]
    candidates: List[List[Tuple[List[int], float]]]
    gaps: List[List[float]]           # per step, per clip
    steps: List[torch.Tensor]         # beam token rows after every step
    logit_scale: List[float]          # per step, the largest |finite logit| (what rounding errors scale with)
    mass_margins: List[float]         # per step, min over rows of |lse(timestamp log-probs) - max(text log-probs)|


def beam_search(step_fn: Callable[[torch.Tensor, Optional[List[int]]], torch.Tensor], n_audio: int,
                initial_tokens: Sequence[int], sample_len: int, beam_size: int, n_ctx: int = 448,
                patience: Optional[float] = None, length_penalty: Optional[float] = None, suppress: Sequence[int] = (),
                suppress_blank: bool = True, sot_index: int = 0, timestamps: bool = False,
                max_initial_timestamp_index: Optional[int] = None, device="cpu") -> BeamResult:
    """DecodingTask.run with a BeamSearchDecoder.  step_fn(tokens_in, sources) returns (N, T_in, V) logits for the given
    input (whole prefix on the first call, then the newest token); `sources` (None on the first call) are the rows the
    previous update kept, for the callback to rearrange its cache with."""
    B = beam_size
    initial = list(initial_tokens)
    sample_begin = len(initial)
    state = BeamState(B, round(B * (patience or 1.0)))
    tokens = torch.tensor([initial], device=device).repeat(n_audio * B, 1)
    sum_logprobs = torch.zeros(n_audio * B)
    sup = torch.tensor(sorted(set(suppress)), device=device, dtype=torch.long) if suppress else None
    no_speech = None
    sources = None
    steps, scales, margins = [], [], []
    for i in range(sample_len):
        inp = tokens if tokens.shape[-1] <= sample_begin else tokens[:, -1:]
        logits = step_fn(inp, sources)
        if i == 0:
            no_speech = logits[:, sot_index].float().softmax(dim=-1)[:, NO_SPEECH].tolist()
        logits = logits[:, -1].float().clone()
        if suppress_blank and tokens.shape[1] == sample_begin:
            logits[:, [BLANK, EOT]] = -np.inf
        if sup is not None:
            logits[:, sup] = -np.inf
        fin = logits[torch.isfinite(logits)]
        scales.append(float(fin.abs().max()) if fin.numel() else 0.0)
        if timestamps:
            pre = F.log_softmax(logits, dim=-1)
            margins.append(float((pre[:, TIMESTAMP_BEGIN:].logsumexp(-1) - pre[:, :TIMESTAMP_BEGIN].max(-1).values).abs()
                                 .nan_to_num(float("inf")).min()))
            apply_timestamp_rules(logits, tokens, sample_begin, max_initial_timestamp_index)
        else:
            margins.append(float("inf"))
        logprobs = F.log_softmax(logits, dim=-1).cpu()
        tokens, sources, completed = beam_update(state, tokens.cpu(), logprobs, sum_logprobs)
        tokens = tokens.to(device)
        steps.append(tokens.clone())
        if completed or tokens.shape[-1] > n_ctx:
            break
    cands, sums = beam_finalize(state, tokens.cpu().reshape(n_audio, B, -1), sum_logprobs.cpu().reshape(n_audio, B))
    trimmed = []
    for s in cands:
        row = []
        for t in s:
            seq = t[sample_begin:]
            row.append(seq[: seq.index(EOT)] if EOT in seq else seq)
        trimmed.append(row)
    sel = rank(trimmed, sums, length_penalty)
    toks = [trimmed[k][i] for k, i in enumerate(sel)]
    lps = [sums[k][i] for k, i in enumerate(sel)]
    return BeamResult(toks, lps, [lp / (len(t) + 1) for t, lp in zip(toks, lps)], no_speech[::B],
                      [list(zip(c, s)) for c, s in zip(cands, sums)], state.gaps, steps, scales, margins)


def beam_decode(sd, dims, xa: torch.Tensor, beam_size: int, initial_tokens: Sequence[int], sample_len: int,
                dtype=torch.float32, train_model: bool = False, **kw) -> BeamResult:
    """beam_search over oracle/model.py's kv-cache decoder (inf_model.py, or model.py's with `train_model`), one copy of
    the audio features per beam as upstream; the self-attention cache is rearranged with index_select."""
    from oracle import model as OM

    n_audio = xa.shape[0]
    xa_rep = xa.to(dtype).repeat_interleave(beam_size, dim=0)
    cache: dict = {}

    def step(inp, sources):
        if sources is not None:
            idx = torch.tensor(sources, device=xa.device)
            for key in list(cache):
                if ".cross_attn." not in key:
                    cache[key] = cache[key].index_select(0, idx)
        return OM.decoder_forward(sd, dims, inp, xa_rep, None, train_model=train_model, cache=cache)

    return beam_search(step, n_audio, initial_tokens, sample_len, beam_size, n_ctx=dims.n_text_ctx, device=xa.device, **kw)
