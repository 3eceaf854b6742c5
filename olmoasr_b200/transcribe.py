"""Long-form sliding-window driver with the reference's signature and result schema (olmoasr/transcribe.py:47-65,
519-523; README.md:199-246): `transcribe(model, audio, **opts) -> {"text", "segments", "language"}`.

Caller of the hot path, kept so that `model.transcribe(...)` stays callable: GPU log-mel of the whole recording, a
30 s window loop, decode with temperature fallback (transcribe.py:193-233), timestamp-token driven seek advance
(:348-408).  As in the reference (transcribe.py:199-207), `beam_size` / `patience` apply at temperature 0 (beam search on
the device decoder) and `best_of` at the fallback temperatures (best-of-n sampling), so the long-form eval options
`without_timestamps=False, beam_size=5, best_of=5` (scripts/eval/eval.py:2077-2084) work as given.  Like the reference,
previous-text prompt conditioning is disabled (transcribe.py:297-302).  Not implemented (raises): word_timestamps (needs
alignment heads OLMoASR never sets, __init__.py:145).

Text needs a tokenizer: pass `tokenizer=` (object with `.decode(list[int]) -> str`); without one, segments carry token
ids and empty text (the `gpt2.tiktoken` vocabulary cannot be fetched offline).
"""
from __future__ import annotations

import zlib
from typing import List, Optional, Tuple, Union

import numpy as np
import torch

from .audio import HOP_LENGTH, N_FRAMES, N_SAMPLES, SAMPLE_RATE, log_mel_spectrogram, pad_or_trim
from .decoding import EOT, TIMESTAMP_BEGIN, DecodingOptions, DecodingResult, decode


def _compression_ratio(result: DecodingResult) -> float:
    data = result.text.encode("utf-8") if result.text else np.asarray(result.tokens, dtype=np.uint16).tobytes()
    return len(data) / max(1, len(zlib.compress(data)))


def transcribe(model, audio: Union[str, np.ndarray, torch.Tensor], *, verbose: Optional[bool] = None,
               temperature: Union[float, Tuple[float, ...]] = (0.0, 0.2, 0.4, 0.6, 0.8, 1.0),
               compression_ratio_threshold: Optional[float] = 2.4, logprob_threshold: Optional[float] = -1.0,
               no_speech_threshold: Optional[float] = 0.6, condition_on_previous_text: bool = True,
               initial_prompt: Optional[str] = None, carry_initial_prompt: bool = False, word_timestamps: bool = False,
               prepend_punctuations: str = "\"'“¿([{-", append_punctuations: str = "\"'.。,，!！?？:：”)]}、",
               clip_timestamps: Union[str, List[float]] = "0", hallucination_silence_threshold: Optional[float] = None,
               tokenizer=None, **decode_options):
    if word_timestamps:
        raise NotImplementedError("word_timestamps needs alignment heads, which OLMoASR checkpoints do not define")
    decode_options.pop("fp16", None)
    decode_options.setdefault("language", "en")
    mel = log_mel_spectrogram(audio, model.dims.n_mels, padding=N_SAMPLES, device=model.device)
    content_frames = mel.shape[-1] - N_FRAMES
    time_precision = 30.0 / model.dims.n_audio_ctx
    input_stride = N_FRAMES // model.dims.n_audio_ctx
    temps = (temperature,) if isinstance(temperature, (int, float)) else tuple(temperature)

    def decode_with_fallback(segment: torch.Tensor) -> DecodingResult:
        result = None
        for t in temps:
            # beam search at t == 0, best-of-n sampling at t > 0 (transcribe.py:199-207)
            drop = ("beam_size", "patience") if t > 0 else ("best_of",)
            kw = {k: v for k, v in decode_options.items() if k not in drop}
            result = decode(model, segment, DecodingOptions(**kw, temperature=t), tokenizer=tokenizer)
            result = _with_ratio(result)
            retry = False
            if compression_ratio_threshold is not None and result.compression_ratio > compression_ratio_threshold:
                retry = True
            if logprob_threshold is not None and result.avg_logprob < logprob_threshold:
                retry = True
            if no_speech_threshold is not None and result.no_speech_prob > no_speech_threshold and \
                    logprob_threshold is not None and result.avg_logprob < logprob_threshold:
                retry = False  # silence
            if not retry:
                break
        return result

    def _with_ratio(r: DecodingResult) -> DecodingResult:
        from dataclasses import replace
        return replace(r, compression_ratio=_compression_ratio(r))

    def new_segment(start: float, end: float, tokens: List[int], result: DecodingResult, seek: int):
        ids = [t for t in tokens if t < EOT]
        return {"id": 0, "seek": seek, "start": start, "end": end, "text": tokenizer.decode(ids) if tokenizer else "",
                "tokens": tokens, "temperature": result.temperature, "avg_logprob": result.avg_logprob,
                "compression_ratio": result.compression_ratio, "no_speech_prob": result.no_speech_prob}

    all_segments: List[dict] = []
    all_tokens: List[int] = []
    seek = 0
    while seek < content_frames:
        time_offset = seek * HOP_LENGTH / SAMPLE_RATE
        segment_size = min(N_FRAMES, content_frames - seek)
        segment_duration = segment_size * HOP_LENGTH / SAMPLE_RATE
        segment = pad_or_trim(mel[:, seek: seek + segment_size], N_FRAMES).contiguous()
        result = decode_with_fallback(segment)
        tokens = list(result.tokens)
        if no_speech_threshold is not None and result.no_speech_prob > no_speech_threshold and not (
                logprob_threshold is not None and result.avg_logprob > logprob_threshold):
            seek += segment_size  # skip silent window
            continue
        current: List[dict] = []
        is_ts = [t >= TIMESTAMP_BEGIN for t in tokens]
        single_ending = len(is_ts) >= 2 and (not is_ts[-2]) and is_ts[-1]
        consecutive = [i + 1 for i in range(len(tokens) - 1) if is_ts[i] and is_ts[i + 1]]
        if consecutive:
            slices = list(consecutive)
            if single_ending:
                slices.append(len(tokens))
            last = 0
            for cur in slices:
                sl = tokens[last:cur]
                start_pos, end_pos = sl[0] - TIMESTAMP_BEGIN, sl[-1] - TIMESTAMP_BEGIN
                current.append(new_segment(time_offset + start_pos * time_precision, time_offset + end_pos * time_precision, sl,
                                           result, seek))
                last = cur
            if single_ending:
                seek += segment_size
            else:
                seek += (tokens[last - 1] - TIMESTAMP_BEGIN) * input_stride
        else:
            duration = segment_duration
            ts = [t for t in tokens if t >= TIMESTAMP_BEGIN]
            if ts and ts[-1] != TIMESTAMP_BEGIN:
                duration = (ts[-1] - TIMESTAMP_BEGIN) * time_precision
            current.append(new_segment(time_offset, time_offset + duration, tokens, result, seek))
            seek += segment_size
        for i, seg in enumerate(current, start=len(all_segments)):
            seg["id"] = i
        all_segments.extend(current)
        all_tokens.extend(t for seg in current for t in seg["tokens"])
    text = tokenizer.decode([t for t in all_tokens if t < EOT]) if tokenizer else ""
    return dict(text=text, segments=all_segments, language=decode_options.get("language", "en"))
