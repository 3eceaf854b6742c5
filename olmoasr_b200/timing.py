"""Word-level timestamps (`transcribe(word_timestamps=True)`): upstream `whisper/timing.py` restated over this package's
kernels.  The reference exposes the option (olmoasr/transcribe.py:59,410-485) but its models never define
`alignment_heads`; here they default to upstream's choice (every head of the upper half of the decoder layers, see
`OLMoASRBase.alignment_heads` / `set_alignment_heads`).

Per window:
  1. one decoder forward over [SOT, NO_TIMESTAMPS, *text_tokens, EOT] through the kv-cache hook path, under
     torch.autocast("cuda", torch.float16) (upstream's fp16 default), with forward hooks on the alignment layers'
     cross-attention query projections; the cross keys are the cache entries;
  2. `oasr_align_cost` turns the heads' query rows and cross keys into the DTW input (QK, softmax over the window's
     frames, per-frame normalisation over tokens, median filter, head mean) without materialising per-head weights;
  3. `oasr_dtw` aligns tokens to frames on the device; token probabilities are softmax(logits[1:, :EOT]) on the device;
  4. one copy to the host (path + probabilities), then words, durations and punctuation as upstream.
"""
from __future__ import annotations

import itertools
import string
from dataclasses import dataclass
from typing import List, Optional, Tuple

import numpy as np
import torch

from . import kernels as K
from .audio import HOP_LENGTH, SAMPLE_RATE
from .decoding import EOT, NO_TIMESTAMPS, SOT

TOKENS_PER_SECOND = SAMPLE_RATE // (2 * HOP_LENGTH)   # 50: one audio-context position per 20 ms


@dataclass
class WordTiming:
    word: str
    tokens: List[int]
    start: float
    end: float
    probability: float


# ---- device part ---------------------------------------------------------------------------------------------------
def alignment_cost(model, text_tokens: List[int], mel: torch.Tensor, num_frames: int, medfilt_width: int = 7):
    """Steps 1-2 for one window: (cost (n_text + 1, num_frames // 2) fp32, text-token probabilities (n_text,) fp32),
    both on the device.  `mel` is a mel segment (n_mels, 3000) or encoded features (n_audio_ctx, n_audio_state)."""
    dims = model.dims
    n_frames = num_frames // 2
    if not 1 <= n_frames <= dims.n_audio_ctx:
        raise ValueError(f"num_frames must be in 2 .. {2 * dims.n_audio_ctx} (got {num_frames})")
    dev = model.device
    tokens = torch.tensor([SOT, NO_TIMESTAMPS, *text_tokens, EOT], device=dev)
    if tokens.numel() > dims.n_text_ctx:
        raise ValueError(f"{len(text_tokens)} text tokens do not fit the {dims.n_text_ctx}-token context")
    heads = model.alignment_heads.indices().T.tolist()      # ascending (layer, head)
    blocks = model.decoder.blocks
    queries = {}
    hooks = [blocks[l].cross_attn.query.register_forward_hook(lambda _m, _i, out, l=l: queries.__setitem__(l, out))
             for l in sorted({l for l, _ in heads})]
    cache, kv_hooks = model.install_kv_cache_hooks()
    try:
        with torch.no_grad(), torch.autocast("cuda", torch.float16):
            if tuple(mel.shape[-2:]) == (dims.n_audio_ctx, dims.n_audio_state):
                xa = mel.reshape(1, dims.n_audio_ctx, dims.n_audio_state)
            else:
                xa = model.encoder(mel.reshape(1, *mel.shape[-2:]))
            logits = model.decoder(tokens[None], xa, kv_cache=cache)[0]
            hd = dims.n_text_state // dims.n_text_head
            pairs = [(queries[l][0][:, h * hd:(h + 1) * hd], cache[blocks[l].cross_attn.key][0][:, h * hd:(h + 1) * hd])
                     for l, h in heads]
            cost = K.align_cost(pairs, n_frames, medfilt_width)
            n_text = len(text_tokens)
            probs = logits[1:n_text + 1, :EOT].float().softmax(dim=-1)
            text_probs = probs[torch.arange(n_text, device=dev), tokens[2:2 + n_text]]
    finally:
        for h in hooks + kv_hooks:
            h.remove()
    return cost, text_probs


def _device_alignment(model, text_tokens: List[int], mel: torch.Tensor, num_frames: int, medfilt_width: int = 7):
    """Steps 1-3 and the window's one device-to-host copy: (text_indices, time_indices, text-token probabilities)."""
    cost, probs = alignment_cost(model, text_tokens, mel, num_frames, medfilt_width)
    path, length = K.dtw(cost)
    host = torch.cat([length.float(), path.flatten().float(), probs]).cpu().numpy()
    n, width = int(host[0]), path.shape[1]
    text_indices = host[1:1 + n].astype(np.int64)
    time_indices = host[1 + width:1 + width + n].astype(np.int64)
    return text_indices, time_indices, host[1 + 2 * width:].astype(np.float64).tolist()


# ---- host part -----------------------------------------------------------------------------------------------------
def _decode_piece(tokenizer, ids: List[int]) -> str:
    # ids >= EOT are special: they make words of their own and carry no text
    return tokenizer.decode([t for t in ids if t < EOT])


def split_tokens_on_unicode(tokenizer, tokens: List[int]):
    decoded_full = _decode_piece(tokenizer, tokens)
    replacement_char = "\ufffd"
    words, word_tokens, current_tokens = [], [], []
    unicode_offset = 0
    for token in tokens:
        current_tokens.append(token)
        decoded = _decode_piece(tokenizer, current_tokens)
        if replacement_char not in decoded or \
                decoded_full[unicode_offset + decoded.index(replacement_char)] == replacement_char:
            words.append(decoded)
            word_tokens.append(current_tokens)
            current_tokens = []
            unicode_offset += len(decoded)
    return words, word_tokens


def split_tokens_on_spaces(tokenizer, tokens: List[int]):
    subwords, subword_tokens_list = split_tokens_on_unicode(tokenizer, tokens)
    words, word_tokens = [], []
    for subword, subword_tokens in zip(subwords, subword_tokens_list):
        special = subword_tokens[0] >= EOT
        with_space = subword.startswith(" ")
        punctuation = subword.strip() in string.punctuation
        if special or with_space or punctuation or len(words) == 0:
            words.append(subword)
            word_tokens.append(subword_tokens)
        else:
            words[-1] = words[-1] + subword
            word_tokens[-1].extend(subword_tokens)
    return words, word_tokens


def split_to_word_tokens(tokenizer, tokens: List[int]):
    if hasattr(tokenizer, "split_to_word_tokens"):
        return tokenizer.split_to_word_tokens(tokens)
    return split_tokens_on_spaces(tokenizer, tokens)     # English-only vocabulary: words end at spaces


def words_from_path(tokenizer, text_tokens: List[int], text_indices: np.ndarray, time_indices: np.ndarray,
                    text_token_probs: List[float]) -> List[WordTiming]:
    """Steps 4 onwards of upstream find_alignment: word boundaries from the DTW jumps."""
    words, word_tokens = split_to_word_tokens(tokenizer, text_tokens + [EOT])
    if len(word_tokens) <= 1:
        return []
    word_boundaries = np.pad(np.cumsum([len(t) for t in word_tokens[:-1]]), (1, 0))
    jumps = np.pad(np.diff(text_indices), (1, 0), constant_values=1).astype(bool)
    jump_times = time_indices[jumps] / TOKENS_PER_SECOND
    start_times = jump_times[word_boundaries[:-1]]
    end_times = jump_times[word_boundaries[1:]]
    word_probabilities = [np.mean(text_token_probs[i:j]) for i, j in zip(word_boundaries[:-1], word_boundaries[1:])]
    return [WordTiming(word, tokens, start, end, probability)
            for word, tokens, start, end, probability in zip(words, word_tokens, start_times, end_times, word_probabilities)]


def find_alignment(model, tokenizer, text_tokens: List[int], mel: torch.Tensor, num_frames: int, *,
                   medfilt_width: int = 7, qk_scale: float = 1.0) -> List[WordTiming]:
    """whisper.timing.find_alignment: word timings (seconds from the window start) of `text_tokens`."""
    if len(text_tokens) == 0:
        return []
    if qk_scale != 1.0:
        raise ValueError("only qk_scale=1.0 (upstream's value) is supported")
    text_indices, time_indices, probs = _device_alignment(model, list(text_tokens), mel, num_frames, medfilt_width)
    return words_from_path(tokenizer, list(text_tokens), text_indices, time_indices, probs)


def merge_punctuations(alignment: List[WordTiming], prepended: str, appended: str):
    # merge prepended punctuations
    i = len(alignment) - 2
    j = len(alignment) - 1
    while i >= 0:
        previous = alignment[i]
        following = alignment[j]
        if previous.word.startswith(" ") and previous.word.strip() in prepended:
            following.word = previous.word + following.word
            following.tokens = previous.tokens + following.tokens
            previous.word = ""
            previous.tokens = []
        else:
            j = i
        i -= 1
    # merge appended punctuations
    i = 0
    j = 1
    while j < len(alignment):
        previous = alignment[i]
        following = alignment[j]
        if not previous.word.endswith(" ") and following.word in appended:
            previous.word = previous.word + following.word
            previous.tokens = previous.tokens + following.tokens
            following.word = ""
            following.tokens = []
        else:
            i = j
        j += 1


def add_word_timestamps(*, segments: List[dict], model, tokenizer, mel: torch.Tensor, num_frames: int,
                        prepend_punctuations: str = "\"'“¿([{-", append_punctuations: str = "\"'.。,，!！?？:：”)]}、",
                        last_speech_timestamp: float, **kwargs):
    """whisper.timing.add_word_timestamps: sets segment["words"] and adjusts the segments' first / last word and
    start / end in place."""
    if len(segments) == 0:
        return
    text_tokens_per_segment = [[token for token in segment["tokens"] if token < EOT] for segment in segments]
    text_tokens = list(itertools.chain.from_iterable(text_tokens_per_segment))
    alignment = find_alignment(model, tokenizer, text_tokens, mel, num_frames, **kwargs)
    word_durations = np.array([t.end - t.start for t in alignment])
    word_durations = word_durations[word_durations.nonzero()]
    median_duration = np.median(word_durations) if len(word_durations) > 0 else 0.0
    median_duration = min(0.7, float(median_duration))
    max_duration = median_duration * 2

    # truncate long words at sentence boundaries
    if len(word_durations) > 0:
        sentence_end_marks = ".。!！?？"
        for i in range(1, len(alignment)):
            if alignment[i].end - alignment[i].start > max_duration:
                if alignment[i].word in sentence_end_marks:
                    alignment[i].end = alignment[i].start + max_duration
                elif alignment[i - 1].word in sentence_end_marks:
                    alignment[i].start = alignment[i].end - max_duration

    merge_punctuations(alignment, prepend_punctuations, append_punctuations)

    time_offset = segments[0]["seek"] * HOP_LENGTH / SAMPLE_RATE
    word_index = 0
    for segment, text_tokens in zip(segments, text_tokens_per_segment):
        saved_tokens = 0
        words = []
        while word_index < len(alignment) and saved_tokens < len(text_tokens):
            timing = alignment[word_index]
            if timing.word:
                words.append(dict(word=timing.word, start=round(time_offset + timing.start, 2),
                                  end=round(time_offset + timing.end, 2), probability=timing.probability))
            saved_tokens += len(timing.tokens)
            word_index += 1

        # truncate long words at segment boundaries
        if len(words) > 0:
            # the first and second word after a pause are at most twice the median word duration
            if words[0]["end"] - last_speech_timestamp > median_duration * 4 and (
                    words[0]["end"] - words[0]["start"] > max_duration
                    or (len(words) > 1 and words[1]["end"] - words[0]["start"] > max_duration * 2)):
                if len(words) > 1 and words[1]["end"] - words[1]["start"] > max_duration:
                    boundary = max(words[1]["end"] / 2, words[1]["end"] - max_duration)
                    words[0]["end"] = words[1]["start"] = boundary
                words[0]["start"] = max(0, words[0]["end"] - max_duration)

            # prefer the segment-level start timestamp if the first word is too long
            if segment["start"] < words[0]["end"] and segment["start"] - 0.5 > words[0]["start"]:
                words[0]["start"] = max(0, min(words[0]["end"] - median_duration, segment["start"]))
            else:
                segment["start"] = words[0]["start"]

            # prefer the segment-level end timestamp if the last word is too long
            if segment["end"] > words[-1]["start"] and segment["end"] + 0.5 < words[-1]["end"]:
                words[-1]["end"] = max(words[-1]["start"] + median_duration, segment["end"])
            else:
                segment["end"] = words[-1]["end"]

            last_speech_timestamp = segment["end"]

        segment["words"] = words


# ---- the transcribe() window step after add_word_timestamps (reference transcribe.py:420-478) ------------------------
FRAMES_PER_SECOND = SAMPLE_RATE // HOP_LENGTH   # 100 mel frames per second
PUNCTUATION = "\"'“¿([{-\"'.。,，!！?？:：”)]}、"


def word_anomaly_score(word: dict) -> float:
    probability = word.get("probability", 0.0)
    duration = word["end"] - word["start"]
    score = 0.0
    if probability < 0.15:
        score += 1.0
    if duration < 0.133:
        score += (0.133 - duration) * 15
    if duration > 2.0:
        score += duration - 2.0
    return score


def is_segment_anomaly(segment: Optional[dict]) -> bool:
    if segment is None or not segment["words"]:
        return False
    words = [w for w in segment["words"] if w["word"] not in PUNCTUATION]
    words = words[:8]
    score = sum(word_anomaly_score(w) for w in words)
    return score >= 3 or score + 0.01 >= len(words)


def next_words_segment(segments: List[dict]) -> Optional[dict]:
    return next((s for s in segments if s["words"]), None)


def get_end(segments: List[dict]) -> Optional[float]:
    return next((w["end"] for s in reversed(segments) for w in s["words"]), segments[-1]["end"] if segments else None)


def after_word_timestamps(current_segments: List[dict], *, seek: int, previous_seek: int, segment_size: int,
                          single_timestamp_ending: bool, time_offset: float, window_end_time: float,
                          segment_duration: float, content_frames: int, content_duration: float,
                          last_speech_timestamp: float,
                          hallucination_silence_threshold: Optional[float]) -> Tuple[bool, int, float]:
    """Seek to the last word, skip silence around likely hallucinations.  Trims `current_segments` in place and returns
    (skip the window's segments, new seek, new last_speech_timestamp)."""
    if not single_timestamp_ending:
        last_word_end = get_end(current_segments)
        if last_word_end is not None and last_word_end > time_offset:
            seek = round(last_word_end * FRAMES_PER_SECOND)

    if hallucination_silence_threshold is not None:
        threshold = hallucination_silence_threshold
        if not single_timestamp_ending:
            last_word_end = get_end(current_segments)
            if last_word_end is not None and last_word_end > time_offset:
                remaining_duration = window_end_time - last_word_end
                if remaining_duration > threshold:
                    seek = round(last_word_end * FRAMES_PER_SECOND)
                else:
                    seek = previous_seek + segment_size

        # if the first segment might be a hallucination, skip leading silence
        first_segment = next_words_segment(current_segments)
        if first_segment is not None and is_segment_anomaly(first_segment):
            gap = first_segment["start"] - time_offset
            if gap > threshold:
                seek = previous_seek + round(gap * FRAMES_PER_SECOND)
                return True, seek, last_speech_timestamp

        # skip silence before any possible hallucination surrounded by silence or more hallucinations
        hal_last_end = last_speech_timestamp
        for si in range(len(current_segments)):
            segment = current_segments[si]
            if not segment["words"]:
                continue
            if is_segment_anomaly(segment):
                next_segment = next_words_segment(current_segments[si + 1:])
                if next_segment is not None:
                    hal_next_start = next_segment["words"][0]["start"]
                else:
                    hal_next_start = time_offset + segment_duration
                silence_before = (segment["start"] - hal_last_end > threshold or segment["start"] < threshold
                                  or segment["start"] - time_offset < 2.0)
                silence_after = (hal_next_start - segment["end"] > threshold or is_segment_anomaly(next_segment)
                                 or window_end_time - segment["end"] < 2.0)
                if silence_before and silence_after:
                    seek = round(max(time_offset + 1, segment["start"]) * FRAMES_PER_SECOND)
                    if content_duration - segment["end"] < threshold:
                        seek = content_frames
                    current_segments[si:] = []
                    break
            hal_last_end = segment["end"]

    last_word_end = get_end(current_segments)
    if last_word_end is not None:
        last_speech_timestamp = last_word_end
    return False, seek, last_speech_timestamp
