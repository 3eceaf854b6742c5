"""CPU restatement of upstream `whisper/timing.py` (the version matching the reference's transcribe.py, with
`hallucination_silence_threshold`) and of the word-timestamp part of the reference's transcribe loop
(olmoasr/transcribe.py:410-485).

TEST INFRASTRUCTURE.  Pieces:
  * `decoder_forward_qk`: oracle/model.py's decoder forward with the raw cross-attention logits of every layer captured
    where upstream's hooks read them (`outs[-1]` of each `cross_attn`, i.e. (q hd^-1/4)(k hd^-1/4)^T cast to fp32);
  * `alignment_matrix`: steps 3-7 of find_alignment (softmax over frames, std_mean over tokens, median filter, head mean,
    rows [1:-1]) in torch, on whatever device the QKs live;
  * `dtw` (float32 cost table, whisper's tie order) and `median_filter`;
  * the host logic: word split, `merge_punctuations`, `add_word_timestamps` and the transcribe window step.
"""
from __future__ import annotations

import string
from typing import List, Optional

import numpy as np
import torch
import torch.nn.functional as F

from . import model as OM

EOT, SOT, NO_TIMESTAMPS = 50256, 50257, 50362
TOKENS_PER_SECOND = 50
FRAMES_PER_SECOND = 100


# ---- model side ----------------------------------------------------------------------------------------------------
def decoder_forward_qk(sd, dims, tokens, xa):
    """inf_model TextDecoder.forward without a cache (manual attention throughout) -> (fp32 logits, [cross QK per layer,
    (B, n_head, n_tok, n_audio_ctx) fp32])."""
    qks = []
    x = F.embedding(tokens, sd["decoder.token_embedding.weight"]) + sd["decoder.positional_embedding"][:tokens.shape[-1]]
    x = x.to(xa.dtype)
    mask = OM.causal_mask(x.shape[1]).to(x.device)
    for i in range(dims.n_text_layer):
        p = f"decoder.blocks.{i}"
        x = x + OM._attention(sd, p + ".attn", dims.n_text_head, OM._layer_norm(sd, p + ".attn_ln", x), mask=mask, sdpa=False)
        h = OM._layer_norm(sd, p + ".cross_attn_ln", x)
        q, k = OM._lin(sd, p + ".cross_attn.query", h), OM._lin(sd, p + ".cross_attn.key", xa)
        scale = (q.shape[-1] // dims.n_text_head) ** -0.25
        qh = OM._split_heads(q, dims.n_text_head) * scale
        kh = k.view(*k.shape[:2], dims.n_text_head, -1).permute(0, 2, 3, 1) * scale
        qks.append((qh @ kh).float())
        x = x + OM._attention(sd, p + ".cross_attn", dims.n_text_head, h, xa, sdpa=False)
        g = OM._lin(sd, p + ".mlp.0", OM._layer_norm(sd, p + ".mlp_ln", x))
        x = x + OM._lin(sd, p + ".mlp.2", F.gelu(g))
    x = OM._layer_norm(sd, "decoder.ln", x)
    return (x @ sd["decoder.token_embedding.weight"].to(x.dtype).t()).float(), qks


def default_alignment_heads(n_layer: int, n_head: int) -> List[tuple]:
    return [(l, h) for l in range(n_layer // 2, n_layer) for h in range(n_head)]


def median_filter(x: torch.Tensor, filter_width: int) -> torch.Tensor:
    """Median along the last dimension with reflect padding; the input itself when it is not longer than the pad."""
    pad_width = filter_width // 2
    if x.shape[-1] <= pad_width:
        return x
    ndim = x.ndim
    if ndim <= 2:
        x = x[None, None, :]
    x = F.pad(x, (pad_width, pad_width, 0, 0), mode="reflect")
    result = x.unfold(-1, filter_width, 1).sort()[0][..., pad_width]
    if ndim <= 2:
        result = result[0, 0]
    return result


def alignment_matrix(qks, heads, num_frames: int, medfilt_width: int = 7, qk_scale: float = 1.0) -> torch.Tensor:
    """Steps 3-7: qks[l] (n_head, n_tok, frames) -> matrix (n_tok - 2, num_frames // 2) fp32 (the DTW input is its
    negation)."""
    weights = torch.stack([qks[l][h] for l, h in heads])
    weights = weights[:, :, : num_frames // 2]
    weights = (weights * qk_scale).softmax(dim=-1)
    std, mean = torch.std_mean(weights, dim=-2, keepdim=True, unbiased=False)
    weights = (weights - mean) / std
    weights = median_filter(weights, medfilt_width)
    matrix = weights.mean(axis=0)
    return matrix[1:-1]


def dtw(x: np.ndarray):
    """Dynamic time warping over a float32 cost table, swept by anti-diagonals (every cell of a diagonal depends on the
    two before it only), with whisper's tie order.  Returns (text_indices, time_indices)."""
    x = np.asarray(x, dtype=np.float32)
    N, M = x.shape
    cost = np.full((N + 1, M + 1), np.inf, dtype=np.float32)
    trace = np.full((N + 1, M + 1), -1, dtype=np.int8)
    cost[0, 0] = 0
    for d in range(2, N + M + 1):
        i = np.arange(max(1, d - M), min(N, d - 1) + 1)
        j = d - i
        c0, c1, c2 = cost[i - 1, j - 1], cost[i - 1, j], cost[i, j - 1]
        t = np.where((c0 < c1) & (c0 < c2), 0, np.where((c1 < c0) & (c1 < c2), 1, 2)).astype(np.int8)
        c = np.where(t == 0, c0, np.where(t == 1, c1, c2))
        cost[i, j] = x[i - 1, j - 1] + c          # float32 + float32, rounded to float32
        trace[i, j] = t
    trace[0, :] = 2
    trace[:, 0] = 1
    i, j = N, M
    text, time = [], []
    while i > 0 or j > 0:
        text.append(i - 1)
        time.append(j - 1)
        t = trace[i, j]
        if t == 0:
            i, j = i - 1, j - 1
        elif t == 1:
            i -= 1
        elif t == 2:
            j -= 1
        else:
            raise ValueError("unexpected trace value")
    return np.array(text[::-1], dtype=np.int64), np.array(time[::-1], dtype=np.int64)


# ---- host logic ----------------------------------------------------------------------------------------------------
class Word:
    def __init__(self, word, tokens, start, end, probability):
        self.word, self.tokens, self.start, self.end, self.probability = word, tokens, start, end, probability


def split_to_word_tokens(decode, tokens: List[int]):
    """split_tokens_on_spaces over split_tokens_on_unicode; `decode` maps text ids to a string, ids >= EOT are words
    of their own with no text."""
    def dec(ids):
        return decode([t for t in ids if t < EOT])

    full = dec(tokens)
    subwords, sub_tokens, cur, offset = [], [], [], 0
    for tok in tokens:
        cur.append(tok)
        s = dec(cur)
        if "�" not in s or full[offset + s.index("�")] == "�":
            subwords.append(s)
            sub_tokens.append(cur)
            cur = []
            offset += len(s)
    words, word_tokens = [], []
    for s, toks in zip(subwords, sub_tokens):
        if toks[0] >= EOT or s.startswith(" ") or s.strip() in string.punctuation or not words:
            words.append(s)
            word_tokens.append(list(toks))
        else:
            words[-1] += s
            word_tokens[-1].extend(toks)
    return words, word_tokens


def words_from_path(decode, text_tokens, text_indices, time_indices, probs) -> List[Word]:
    words, word_tokens = split_to_word_tokens(decode, list(text_tokens) + [EOT])
    if len(word_tokens) <= 1:
        return []
    bounds = np.pad(np.cumsum([len(t) for t in word_tokens[:-1]]), (1, 0))
    jumps = np.pad(np.diff(text_indices), (1, 0), constant_values=1).astype(bool)
    jump_times = np.asarray(time_indices)[jumps] / TOKENS_PER_SECOND
    out = []
    for k in range(min(len(words), len(bounds) - 1)):
        a, b = bounds[k], bounds[k + 1]
        out.append(Word(words[k], word_tokens[k], jump_times[a], jump_times[b], np.mean(probs[a:b])))
    return out


def merge_punctuations(alignment: List[Word], prepended: str, appended: str):
    i, j = len(alignment) - 2, len(alignment) - 1
    while i >= 0:
        prev, foll = alignment[i], alignment[j]
        if prev.word.startswith(" ") and prev.word.strip() in prepended:
            foll.word, foll.tokens = prev.word + foll.word, prev.tokens + foll.tokens
            prev.word, prev.tokens = "", []
        else:
            j = i
        i -= 1
    i, j = 0, 1
    while j < len(alignment):
        prev, foll = alignment[i], alignment[j]
        if not prev.word.endswith(" ") and foll.word in appended:
            prev.word, prev.tokens = prev.word + foll.word, prev.tokens + foll.tokens
            foll.word, foll.tokens = "", []
        else:
            i = j
        j += 1


def add_word_timestamps(segments: List[dict], alignment: List[Word], last_speech_timestamp: float,
                        prepend: str = "\"'“¿([{-", append: str = "\"'.。,，!！?？:：”)]}、"):
    """upstream add_word_timestamps after find_alignment (whose result is `alignment`)."""
    if not segments:
        return
    per_segment = [[t for t in s["tokens"] if t < EOT] for s in segments]
    durations = np.array([w.end - w.start for w in alignment])
    durations = durations[durations.nonzero()]
    median = min(0.7, float(np.median(durations) if len(durations) > 0 else 0.0))
    max_d = median * 2
    if len(durations) > 0:
        for i in range(1, len(alignment)):
            if alignment[i].end - alignment[i].start > max_d:
                if alignment[i].word in ".。!！?？":
                    alignment[i].end = alignment[i].start + max_d
                elif alignment[i - 1].word in ".。!！?？":
                    alignment[i].start = alignment[i].end - max_d
    merge_punctuations(alignment, prepend, append)
    offset = segments[0]["seek"] * 160 / 16000
    wi = 0
    for seg, toks in zip(segments, per_segment):
        saved, words = 0, []
        while wi < len(alignment) and saved < len(toks):
            w = alignment[wi]
            if w.word:
                words.append(dict(word=w.word, start=round(offset + w.start, 2), end=round(offset + w.end, 2),
                                  probability=w.probability))
            saved += len(w.tokens)
            wi += 1
        if words:
            if words[0]["end"] - last_speech_timestamp > median * 4 and (
                    words[0]["end"] - words[0]["start"] > max_d
                    or (len(words) > 1 and words[1]["end"] - words[0]["start"] > max_d * 2)):
                if len(words) > 1 and words[1]["end"] - words[1]["start"] > max_d:
                    boundary = max(words[1]["end"] / 2, words[1]["end"] - max_d)
                    words[0]["end"] = words[1]["start"] = boundary
                words[0]["start"] = max(0, words[0]["end"] - max_d)
            if seg["start"] < words[0]["end"] and seg["start"] - 0.5 > words[0]["start"]:
                words[0]["start"] = max(0, min(words[0]["end"] - median, seg["start"]))
            else:
                seg["start"] = words[0]["start"]
            if seg["end"] > words[-1]["start"] and seg["end"] + 0.5 < words[-1]["end"]:
                words[-1]["end"] = max(words[-1]["start"] + median, seg["end"])
            else:
                seg["end"] = words[-1]["end"]
            last_speech_timestamp = seg["end"]
        seg["words"] = words


_PUNCT = "\"'“¿([{-\"'.。,，!！?？:：”)]}、"


def _anomaly(w) -> float:
    p, dur, score = w.get("probability", 0.0), w["end"] - w["start"], 0.0
    if p < 0.15:
        score += 1.0
    if dur < 0.133:
        score += (0.133 - dur) * 15
    if dur > 2.0:
        score += dur - 2.0
    return score


def _is_anomaly(seg) -> bool:
    if seg is None or not seg["words"]:
        return False
    ws = [w for w in seg["words"] if w["word"] not in _PUNCT][:8]
    score = sum(_anomaly(w) for w in ws)
    return score >= 3 or score + 0.01 >= len(ws)


def _next_with_words(segs):
    return next((s for s in segs if s["words"]), None)


def _end(segs) -> Optional[float]:
    return next((w["end"] for s in reversed(segs) for w in s["words"]), segs[-1]["end"] if segs else None)


def window_step(segs, seek, previous_seek, segment_size, single_ending, time_offset, window_end_time, segment_duration,
                content_frames, content_duration, last_speech, threshold):
    """The reference's transcribe.py:420-478 -> (skip window, seek, last_speech_timestamp); trims `segs` in place."""
    if not single_ending:
        e = _end(segs)
        if e is not None and e > time_offset:
            seek = round(e * FRAMES_PER_SECOND)
    if threshold is not None:
        if not single_ending:
            e = _end(segs)
            if e is not None and e > time_offset:
                seek = round(e * FRAMES_PER_SECOND) if window_end_time - e > threshold else previous_seek + segment_size
        first = _next_with_words(segs)
        if first is not None and _is_anomaly(first):
            gap = first["start"] - time_offset
            if gap > threshold:
                return True, previous_seek + round(gap * FRAMES_PER_SECOND), last_speech
        hal_last_end = last_speech
        for si, seg in enumerate(segs):
            if not seg["words"]:
                continue
            if _is_anomaly(seg):
                nxt = _next_with_words(segs[si + 1:])
                nxt_start = nxt["words"][0]["start"] if nxt is not None else time_offset + segment_duration
                before = seg["start"] - hal_last_end > threshold or seg["start"] < threshold or seg["start"] - time_offset < 2.0
                after = nxt_start - seg["end"] > threshold or _is_anomaly(nxt) or window_end_time - seg["end"] < 2.0
                if before and after:
                    seek = round(max(time_offset + 1, seg["start"]) * FRAMES_PER_SECOND)
                    if content_duration - seg["end"] < threshold:
                        seek = content_frames
                    del segs[si:]
                    break
            hal_last_end = seg["end"]
    e = _end(segs)
    if e is not None:
        last_speech = e
    return False, seek, last_speech
