"""Long-form sliding-window driver with the reference's signature and result schema (olmoasr/transcribe.py:47-65,
519-523; README.md:199-246): `transcribe(model, audio, **opts) -> {"text", "segments", "language"}`.

Caller of the hot path, kept so that `model.transcribe(...)` stays callable: GPU log-mel of the whole recording, a
30 s window loop, decode with temperature fallback (transcribe.py:193-233), timestamp-token driven seek advance
(:348-408).  As in the reference (transcribe.py:199-207), `beam_size` / `patience` apply at temperature 0 (beam search on
the device decoder) and `best_of` at the fallback temperatures (best-of-n sampling), so the long-form eval options
`without_timestamps=False, beam_size=5, best_of=5` (scripts/eval/eval.py:2077-2084) work as given.  Like the reference,
previous-text prompt conditioning is disabled (transcribe.py:297-302).

`word_timestamps=True` adds upstream's per-word `"words": [{"word", "start", "end", "probability"}]` to every segment
(transcribe.py:410-485; olmoasr_b200/timing.py): the model's `alignment_heads` (upstream's default, or
`set_alignment_heads`) are aligned on the device against the window's encoded features, the seek moves to the last
word's end, `hallucination_silence_threshold` skips silence around anomalous segments, and segments that are
instantaneous or carry no text are cleared.  It needs `tokenizer=` to split words.  With the default False none of this
runs and `hallucination_silence_threshold` is ignored, as upstream.

`transcribe_batch(model, audios, ...)` transcribes many recordings with the same options and result schema.  A
recording's windows depend on each other (each seek follows the previous window's tokens), so the batch comes from many
recordings: every round takes the current window of up to `batch_size` recordings, encodes them in one encoder call,
decodes them together at each fallback temperature (one device-decoder call per temperature for up to 64 rows) and, with
`word_timestamps=True`, aligns them with one call of each batched alignment kernel.  Both functions drive one per-recording
state machine (`_Recording`), so the segment, seek and word-timestamp rules exist once.

Text needs a tokenizer: pass `tokenizer=` (object with `.decode(list[int]) -> str`); without one, segments carry token
ids and empty text (the `gpt2.tiktoken` vocabulary cannot be fetched offline).
"""
from __future__ import annotations

import itertools
import zlib
from collections import deque
from dataclasses import dataclass, replace
from typing import List, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from .audio import HOP_LENGTH, N_FRAMES, N_SAMPLES, SAMPLE_RATE, log_mel_spectrogram, pad_or_trim
from .decode_engine import DecodeEngine, window_clip_id
from .decoding import EOT, TIMESTAMP_BEGIN, DecodingOptions, DecodingResult, decode, decode_windows
from .timing import (add_word_timestamps, after_word_timestamps, apply_word_timings, device_alignments,
                     segment_text_tokens, words_from_path)

Audio = Union[str, np.ndarray, torch.Tensor]
DEFAULT_TEMPERATURES = (0.0, 0.2, 0.4, 0.6, 0.8, 1.0)
PREPEND_PUNCTUATIONS = "\"'“¿([{-"
APPEND_PUNCTUATIONS = "\"'.。,，!！?？:：”)]}、"


def _compression_ratio(result: DecodingResult) -> float:
    data = result.text.encode("utf-8") if result.text else np.asarray(result.tokens, dtype=np.uint16).tobytes()
    return len(data) / max(1, len(zlib.compress(data)))


def _with_ratio(r: DecodingResult) -> DecodingResult:
    return replace(r, compression_ratio=_compression_ratio(r))


def _options_at(decode_options: dict, t: float) -> DecodingOptions:
    # beam search at t == 0, best-of-n sampling at t > 0 (transcribe.py:199-207)
    drop = ("beam_size", "patience") if t > 0 else ("best_of",)
    return DecodingOptions(**{k: v for k, v in decode_options.items() if k not in drop}, temperature=t)


@dataclass(frozen=True)
class _Rules:
    """The options of one transcribe() / transcribe_batch() call that the window step reads."""
    model: object
    tokenizer: object
    compression_ratio_threshold: Optional[float]
    logprob_threshold: Optional[float]
    no_speech_threshold: Optional[float]
    word_timestamps: bool
    prepend_punctuations: str
    append_punctuations: str
    hallucination_silence_threshold: Optional[float]

    def needs_fallback(self, result: DecodingResult) -> bool:
        """decode_with_fallback's test: decode the window again at the next temperature."""
        retry = False
        if self.compression_ratio_threshold is not None and result.compression_ratio > self.compression_ratio_threshold:
            retry = True
        if self.logprob_threshold is not None and result.avg_logprob < self.logprob_threshold:
            retry = True
        if self.no_speech_threshold is not None and result.no_speech_prob > self.no_speech_threshold and \
                self.logprob_threshold is not None and result.avg_logprob < self.logprob_threshold:
            retry = False  # silence
        return retry


class _Recording:
    """One recording's long-form state (log-mel, seek, segments, tokens) and the window step of the reference's loop
    (transcribe.py:348-485): `window()` cuts the current 30 s window, `split(result)` turns the window's decode result into
    segments and advances the seek, the caller adds word timings to them when asked, `commit(segments)` finishes the
    window (word-timestamp seek, hallucination skip, clearing, ids)."""

    def __init__(self, mel: torch.Tensor, rules: _Rules, index: int = 0):
        dims = rules.model.dims
        self.rules, self.index = rules, index
        self.mel = mel
        self.content_frames = mel.shape[-1] - N_FRAMES
        self.time_precision = 30.0 / dims.n_audio_ctx
        self.input_stride = N_FRAMES // dims.n_audio_ctx
        self.seek = 0
        self.last_speech_timestamp = 0.0
        self.segments: List[dict] = []
        self.tokens: List[int] = []

    @property
    def done(self) -> bool:
        return self.seek >= self.content_frames

    def window(self) -> torch.Tensor:
        """The current window (n_mels, 3000), zero-padded past the recording's end."""
        self.previous_seek = self.seek
        self.segment_size = min(N_FRAMES, self.content_frames - self.seek)
        return pad_or_trim(self.mel[:, self.seek: self.seek + self.segment_size], N_FRAMES).contiguous()

    def _new_segment(self, start: float, end: float, tokens: List[int], result: DecodingResult) -> dict:
        tokenizer = self.rules.tokenizer
        ids = [t for t in tokens if t < EOT]
        return {"id": 0, "seek": self.previous_seek, "start": start, "end": end,
                "text": tokenizer.decode(ids) if tokenizer else "", "tokens": tokens, "temperature": result.temperature,
                "avg_logprob": result.avg_logprob, "compression_ratio": result.compression_ratio,
                "no_speech_prob": result.no_speech_prob}

    def split(self, result: DecodingResult) -> Optional[List[dict]]:
        """The window's segments, cut at its timestamp tokens, with the seek advanced past them; None when the window is
        skipped as silence."""
        r = self.rules
        tokens = list(result.tokens)
        seek, segment_size = self.previous_seek, self.segment_size
        if r.no_speech_threshold is not None and result.no_speech_prob > r.no_speech_threshold and not (
                r.logprob_threshold is not None and result.avg_logprob > r.logprob_threshold):
            self.seek = seek + segment_size  # skip silent window
            return None
        time_offset = seek * HOP_LENGTH / SAMPLE_RATE
        current: List[dict] = []
        is_ts = [t >= TIMESTAMP_BEGIN for t in tokens]
        self.single_ending = single_ending = len(is_ts) >= 2 and (not is_ts[-2]) and is_ts[-1]
        consecutive = [i + 1 for i in range(len(tokens) - 1) if is_ts[i] and is_ts[i + 1]]
        if consecutive:
            slices = list(consecutive)
            if single_ending:
                slices.append(len(tokens))
            last = 0
            for cur in slices:
                sl = tokens[last:cur]
                start_pos, end_pos = sl[0] - TIMESTAMP_BEGIN, sl[-1] - TIMESTAMP_BEGIN
                current.append(self._new_segment(time_offset + start_pos * self.time_precision,
                                                 time_offset + end_pos * self.time_precision, sl, result))
                last = cur
            if single_ending:
                self.seek = seek + segment_size
            else:
                self.seek = seek + (tokens[last - 1] - TIMESTAMP_BEGIN) * self.input_stride
        else:
            duration = segment_size * HOP_LENGTH / SAMPLE_RATE
            ts = [t for t in tokens if t >= TIMESTAMP_BEGIN]
            if ts and ts[-1] != TIMESTAMP_BEGIN:
                duration = (ts[-1] - TIMESTAMP_BEGIN) * self.time_precision
            current.append(self._new_segment(time_offset, time_offset + duration, tokens, result))
            self.seek = seek + segment_size
        return current

    def commit(self, current: List[dict]):
        """Finish the window whose `split` gave `current` (with its words when word_timestamps)."""
        r = self.rules
        if r.word_timestamps:
            previous_seek, segment_size = self.previous_seek, self.segment_size
            skip, self.seek, self.last_speech_timestamp = after_word_timestamps(
                current, seek=self.seek, previous_seek=previous_seek, segment_size=segment_size,
                single_timestamp_ending=self.single_ending, time_offset=previous_seek * HOP_LENGTH / SAMPLE_RATE,
                window_end_time=(previous_seek + N_FRAMES) * HOP_LENGTH / SAMPLE_RATE,
                segment_duration=segment_size * HOP_LENGTH / SAMPLE_RATE, content_frames=self.content_frames,
                content_duration=self.content_frames * HOP_LENGTH / SAMPLE_RATE,
                last_speech_timestamp=self.last_speech_timestamp,
                hallucination_silence_threshold=r.hallucination_silence_threshold)
            if skip:
                return
            for seg in current:     # an instantaneous or text-free segment is cleared
                if seg["start"] == seg["end"] or seg["text"].strip() == "":
                    seg["text"], seg["tokens"], seg["words"] = "", [], []
        for i, seg in enumerate(current, start=len(self.segments)):
            seg["id"] = i
        self.segments.extend(current)
        self.tokens.extend(t for seg in current for t in seg["tokens"])

    def result(self, language: str) -> dict:
        tokenizer = self.rules.tokenizer
        text = tokenizer.decode([t for t in self.tokens if t < EOT]) if tokenizer else ""
        return dict(text=text, segments=self.segments, language=language)


def _temperatures(temperature) -> Tuple[float, ...]:
    return (temperature,) if isinstance(temperature, (int, float)) else tuple(temperature)


def _log_mel(model, audio: Audio) -> torch.Tensor:
    return log_mel_spectrogram(audio, model.dims.n_mels, padding=N_SAMPLES, device=model.device)


def transcribe(model, audio: Audio, *, verbose: Optional[bool] = None,
               temperature: Union[float, Tuple[float, ...]] = DEFAULT_TEMPERATURES,
               compression_ratio_threshold: Optional[float] = 2.4, logprob_threshold: Optional[float] = -1.0,
               no_speech_threshold: Optional[float] = 0.6, condition_on_previous_text: bool = True,
               initial_prompt: Optional[str] = None, carry_initial_prompt: bool = False, word_timestamps: bool = False,
               prepend_punctuations: str = PREPEND_PUNCTUATIONS, append_punctuations: str = APPEND_PUNCTUATIONS,
               clip_timestamps: Union[str, List[float]] = "0", hallucination_silence_threshold: Optional[float] = None,
               tokenizer=None, **decode_options):
    if word_timestamps and tokenizer is None:
        raise ValueError("word_timestamps=True needs tokenizer= to split the text into words")
    decode_options.pop("fp16", None)
    decode_options.setdefault("language", "en")
    rules = _Rules(model, tokenizer, compression_ratio_threshold, logprob_threshold, no_speech_threshold, word_timestamps,
                   prepend_punctuations, append_punctuations, hallucination_silence_threshold)
    rec = _Recording(_log_mel(model, audio), rules)
    temps = _temperatures(temperature)
    while not rec.done:
        segment = rec.window()
        result = None
        for t in temps:
            result = _with_ratio(decode(model, segment, _options_at(decode_options, t), tokenizer=tokenizer))
            if not rules.needs_fallback(result):
                break
        current = rec.split(result)
        if current is None:
            continue
        if word_timestamps:
            add_word_timestamps(segments=current, model=model, tokenizer=tokenizer, mel=result.audio_features,
                                num_frames=rec.segment_size, prepend_punctuations=prepend_punctuations,
                                append_punctuations=append_punctuations, last_speech_timestamp=rec.last_speech_timestamp)
        rec.commit(current)
    return rec.result(decode_options.get("language", "en"))


def _is_default_clip(clip_timestamps) -> bool:
    try:
        points = [float(x) for x in clip_timestamps.split(",")] if isinstance(clip_timestamps, str) else \
            [float(x) for x in clip_timestamps]
    except (TypeError, ValueError):
        return False
    return points == [0.0]


def _decode_round(model, features: torch.Tensor, recordings: Sequence[_Recording], temps, decode_options: dict,
                  rules: _Rules, seed: int) -> List[DecodingResult]:
    """decode_with_fallback for every window of a round: one decode of the windows that still need a result per
    temperature, on the round's encoded features; a window keeps its last result."""
    results: List[Optional[DecodingResult]] = [None] * len(recordings)
    todo = list(range(len(recordings)))
    for ti, t in enumerate(temps):
        ids = [window_clip_id(recordings[w].index, recordings[w].previous_seek, ti) for w in todo]
        feats = features if len(todo) == len(recordings) else features[todo]
        decoded = decode_windows(model, feats, _options_at(decode_options, t), rules.tokenizer, (seed, ids))
        retry = []
        for w, r in zip(todo, decoded):
            results[w] = _with_ratio(r)
            if rules.needs_fallback(results[w]):
                retry.append(w)
        todo = retry
        if not todo:
            break
    return results


def _round_word_timestamps(model, recordings: Sequence[_Recording], currents: Sequence[Optional[List[dict]]],
                           features: torch.Tensor, rules: _Rules):
    """add_word_timestamps for every window of a round: the windows with text are aligned together on the device."""
    texts = [list(itertools.chain.from_iterable(segment_text_tokens(cur))) if cur is not None else [] for cur in currents]
    aligned = [w for w, (cur, text) in enumerate(zip(currents, texts)) if cur is not None and text]
    paths = device_alignments(model, [(texts[w], features[w], recordings[w].segment_size) for w in aligned]) if aligned else []
    paths = dict(zip(aligned, paths))
    for w, (rec, cur) in enumerate(zip(recordings, currents)):
        if cur is None:
            continue
        alignment = words_from_path(rules.tokenizer, texts[w], *paths[w]) if w in paths else []
        apply_word_timings(cur, alignment, prepend_punctuations=rules.prepend_punctuations,
                           append_punctuations=rules.append_punctuations, last_speech_timestamp=rec.last_speech_timestamp)


def transcribe_batch(model, audios: Sequence[Audio], *, batch_size: Optional[int] = None, verbose: Optional[bool] = None,
                     temperature: Union[float, Tuple[float, ...]] = DEFAULT_TEMPERATURES,
                     compression_ratio_threshold: Optional[float] = 2.4, logprob_threshold: Optional[float] = -1.0,
                     no_speech_threshold: Optional[float] = 0.6, condition_on_previous_text: bool = True,
                     initial_prompt: Optional[str] = None, carry_initial_prompt: bool = False,
                     word_timestamps: bool = False, prepend_punctuations: str = PREPEND_PUNCTUATIONS,
                     append_punctuations: str = APPEND_PUNCTUATIONS, clip_timestamps: Union[str, List[float]] = "0",
                     hallucination_silence_threshold: Optional[float] = None, tokenizer=None,
                     **decode_options) -> List[dict]:
    """transcribe() of every recording in `audios` (paths, arrays or 1-D tensors of any lengths): one result dict per
    recording, in order, with transcribe()'s schema.  Up to `batch_size` recordings are active at a time (default: the
    clips of one device-decoder call at the largest group, 64 // max(beam_size, best_of)); a recording's log-mel is
    computed when it becomes active.  Each round encodes the active recordings' current windows in one encoder call and
    reuses those features at every fallback temperature and for the word alignment.

    Sampled windows draw with one seed per call (from torch's default generator) and a key per window made of the
    recording's index in `audios`, the window's seek frame and the temperature's index, so under torch.manual_seed a
    recording's result does not depend on `batch_size` or on the recordings that share its rounds.  That holds on the
    device decoder; the hook loop (OASR_DECODE_ENGINE=0) draws from torch's generator in call order and does not promise it.
    `clip_timestamps` other than "0" raises ValueError (not supported)."""
    if batch_size is not None and batch_size < 1:
        raise ValueError(f"batch_size must be >= 1 (got {batch_size})")
    if word_timestamps and tokenizer is None:
        raise ValueError("word_timestamps=True needs tokenizer= to split the text into words")
    if not _is_default_clip(clip_timestamps):
        raise ValueError(f"transcribe_batch does not support clip_timestamps (got {clip_timestamps!r})")
    audios = list(audios)
    if not audios:
        return []
    from ._core import bf16_compute

    decode_options.pop("fp16", None)
    decode_options.setdefault("language", "en")
    language = decode_options.get("language", "en")
    if batch_size is None:
        group = max(decode_options.get("beam_size") or 1, decode_options.get("best_of") or 1)
        batch_size = max(1, DecodeEngine.MAX_BATCH // group)
    rules = _Rules(model, tokenizer, compression_ratio_threshold, logprob_threshold, no_speech_threshold, word_timestamps,
                   prepend_punctuations, append_punctuations, hallucination_silence_threshold)
    temps = _temperatures(temperature)
    seed = int(torch.randint(2 ** 62, (1,)))
    results: List[Optional[dict]] = [None] * len(audios)
    queue = deque(range(len(audios)))
    active: List[_Recording] = []
    while queue or active:
        while queue and len(active) < batch_size:
            i = queue.popleft()
            rec = _Recording(_log_mel(model, audios[i]), rules, index=i)
            if rec.done:
                results[i] = rec.result(language)
            else:
                active.append(rec)
        if not active:
            continue
        windows = torch.stack([rec.window() for rec in active])
        with torch.no_grad(), bf16_compute():
            features = model.encoder(windows)
        decoded = _decode_round(model, features, active, temps, decode_options, rules, seed)
        currents = [rec.split(r) for rec, r in zip(active, decoded)]
        if word_timestamps:
            _round_word_timestamps(model, active, currents, features, rules)
        for rec, cur in zip(active, currents):
            if cur is not None:
                rec.commit(cur)
            if rec.done:
                results[rec.index] = rec.result(language)
        active = [rec for rec in active if not rec.done]
    return results
