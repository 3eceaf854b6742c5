"""Greedy / temperature / best-of / beam-search decoding with a kv cache -- the `model.decode(mel, DecodingOptions(...))`
entry point the reference binds to third-party `whisper.decoding.decode` (olmoasr/model.py:9-10,966-968; call sites
scripts/training/train_timestamps.py:1916-1919, scripts/eval/eval.py:1846-1847, olmoasr/transcribe.py:209-210).

openai-whisper is not vendored by the reference and is absent here, so this restates the published algorithm of
`whisper/decoding.py` for the path OLMoASR uses (English-only `gpt2` vocabulary, n_vocab 51864):
DecodingTask._verify_options / _main_loop, PyTorchInference (first call = whole prefix, later calls = last token, kv cache
through `model.install_kv_cache_hooks()`), GreedyDecoder, BeamSearchDecoder, MaximumLikelihoodRanker, SuppressBlank,
SuppressTokens, ApplyTimestampRules.

Routes: every configuration runs on the device decoder (olmoasr_b200/decode_engine.py) as replays of one CUDA graph per
step: greedy decoding with or without timestamp rules, temperature sampling (best_of samples per clip sharing the clip's
cross-attention K/V, ranked like upstream) and beam search.  The hook loop below remains for OASR_DECODE_ENGINE=0, models
without `decode_engine` and best_of above the engine's batch (64 rows).  Beam search and `fp8` need the device decoder:
without it, `beam_size` and `fp8=True` raise NotImplementedError.  Sampled ids follow softmax(logits / T) like upstream's
`Categorical(...).sample()` but from the engine's own keyed random stream (reproducible under `torch.manual_seed`).

Token ids are the contract: text<->id conversion needs the `gpt2.tiktoken` vocabulary, which is not available offline;
pass `tokenizer=` (an object with `.decode(list[int])`) to get text, otherwise `DecodingResult.text` is empty.
"""
from __future__ import annotations

from dataclasses import dataclass, field, replace
from typing import TYPE_CHECKING, Iterable, List, Optional, Tuple, Union

import numpy as np
import torch
import torch.nn.functional as F
from torch import Tensor

if TYPE_CHECKING:
    from ._core import OLMoASRBase

import contextlib
import os

# OASR_DECODE_ENGINE=0 forces the generic hook-based loop below for every configuration (A/B runs, debugging)
USE_ENGINE = os.environ.get("OASR_DECODE_ENGINE", "1") != "0"

# ---- English-only vocabulary constants (SURVEY.md section 8(c)) -------------------------------------------------
EOT, SOT = 50256, 50257
TRANSLATE, TRANSCRIBE, SOT_LM, SOT_PREV, NO_SPEECH, NO_TIMESTAMPS, TIMESTAMP_BEGIN = 50357, 50358, 50359, 50360, 50361, 50362, 50363
BLANK = 220  # encode(" ") in the gpt2 vocabulary
# tokenizer.non_speech_tokens for the gpt2 vocabulary (symbols / brackets / music notes); the same table ships as
# transformers.models.whisper.configuration_whisper.NON_SPEECH_TOKENS (entries below the special-token range)
NON_SPEECH_TOKENS = (
    1, 2, 7, 8, 9, 10, 14, 25, 26, 27, 28, 29, 31, 58, 59, 60, 61, 62, 63, 90, 91, 92, 93, 357, 366, 438, 532, 685, 705, 796,
    930, 1058, 1220, 1267, 1279, 1303, 1343, 1377, 1391, 1635, 1782, 1875, 2162, 2361, 2488, 3467, 4008, 4211, 4600, 4808,
    5299, 5855, 6329, 7203, 9609, 9959, 10563, 10786, 11420, 11709, 11907, 13163, 13697, 13700, 14808, 15306, 16410, 16791,
    17992, 19203, 19510, 20724, 22305, 22935, 27007, 30109, 30420, 33409, 34949, 40283, 40493, 40549, 47282, 49146)


@dataclass(frozen=True)
class DecodingOptions:
    task: str = "transcribe"
    language: Optional[str] = None
    temperature: float = 0.0
    sample_len: Optional[int] = None
    best_of: Optional[int] = None
    beam_size: Optional[int] = None
    patience: Optional[float] = None
    length_penalty: Optional[float] = None
    prompt: Optional[Union[str, List[int]]] = None
    prefix: Optional[Union[str, List[int]]] = None
    suppress_tokens: Optional[Union[str, Iterable[int]]] = "-1"
    suppress_blank: bool = True
    without_timestamps: bool = False
    max_initial_timestamp: Optional[float] = 1.0
    fp16: bool = True  # decoder-step activation dtype: fp16 (upstream default) or, when False, bf16 (there are no fp32 kernels)
    fp8: bool = False  # store the decoder's block projection weights and cross-attention K/V as e4m3 (device decoder only)


@dataclass(frozen=True)
class DecodingResult:
    audio_features: Tensor
    language: str
    language_probs: Optional[dict] = None
    tokens: List[int] = field(default_factory=list)
    text: str = ""
    avg_logprob: float = np.nan
    no_speech_prob: float = np.nan
    temperature: float = np.nan
    compression_ratio: float = np.nan


def suppress_token_ids(options: DecodingOptions) -> Tuple[int, ...]:
    """DecodingTask._get_suppress_tokens."""
    st = options.suppress_tokens
    if isinstance(st, str):
        st = [int(t) for t in st.split(",")]
    st = list(st) if st is not None else []
    if -1 in st:
        st = [t for t in st if t >= 0]
        st.extend(NON_SPEECH_TOKENS)
    elif len(st) == 0:
        st = []
    st.extend([TRANSCRIBE, TRANSLATE, SOT, SOT_PREV, SOT_LM])
    st.append(NO_SPEECH)
    return tuple(sorted(set(st)))


class _TimestampRules:
    """ApplyTimestampRules of whisper/decoding.py (used when without_timestamps=False)."""

    def __init__(self, sample_begin: int, max_initial_timestamp_index: Optional[int]):
        self.sample_begin = sample_begin
        self.max_initial_timestamp_index = max_initial_timestamp_index

    def apply(self, logits: Tensor, tokens: Tensor):
        logits[:, NO_TIMESTAMPS] = -np.inf
        for k in range(tokens.shape[0]):
            seq = tokens[k, self.sample_begin:].tolist()
            last_was_ts = len(seq) >= 1 and seq[-1] >= TIMESTAMP_BEGIN
            penult_was_ts = len(seq) < 2 or seq[-2] >= TIMESTAMP_BEGIN
            if last_was_ts:
                if penult_was_ts:
                    logits[k, TIMESTAMP_BEGIN:] = -np.inf
                else:
                    logits[k, :EOT] = -np.inf
            ts = [t for t in seq if t >= TIMESTAMP_BEGIN]
            if ts:
                last = ts[-1] if (last_was_ts and not penult_was_ts) else ts[-1] + 1
                logits[k, TIMESTAMP_BEGIN:last] = -np.inf
        if tokens.shape[1] == self.sample_begin:
            logits[:, :TIMESTAMP_BEGIN] = -np.inf
            if self.max_initial_timestamp_index is not None:
                logits[:, TIMESTAMP_BEGIN + self.max_initial_timestamp_index + 1:] = -np.inf
        logprobs = F.log_softmax(logits.float(), dim=-1)
        for k in range(tokens.shape[0]):
            ts_lp = logprobs[k, TIMESTAMP_BEGIN:].logsumexp(dim=-1)
            if ts_lp > logprobs[k, :TIMESTAMP_BEGIN].max():
                logits[k, :TIMESTAMP_BEGIN] = -np.inf


class MaximumLikelihoodRanker:
    """whisper/decoding.py MaximumLikelihoodRanker: per clip the candidate with the highest sum_logprob / penalty,
    penalty = length without a length_penalty, else the Google NMT ((5 + length) / 6) ** length_penalty."""

    def __init__(self, length_penalty: Optional[float]):
        self.length_penalty = length_penalty

    def rank(self, tokens: List[List[List[int]]], sum_logprobs: List[List[float]]) -> List[int]:
        def scores(logprobs, lengths):
            result = []
            for logprob, length in zip(logprobs, lengths):
                penalty = length if self.length_penalty is None else ((5 + length) / 6) ** self.length_penalty
                result.append(logprob / penalty)
            return result

        lengths = [[len(t) for t in s] for s in tokens]
        return [int(np.argmax(scores(p, l))) for p, l in zip(sum_logprobs, lengths)]


def verify_options(options: DecodingOptions):
    """DecodingTask._verify_options (the checks that apply to the English-only models)."""
    if options.beam_size is not None and options.best_of is not None:
        raise ValueError("beam_size and best_of can't be given together")
    if options.temperature == 0 and options.best_of is not None:
        raise ValueError("best_of with greedy sampling (T=0) is not compatible")
    if options.patience is not None and options.beam_size is None:
        raise ValueError("patience requires beam_size to be given")
    if options.length_penalty is not None and not 0 <= options.length_penalty <= 1:
        raise ValueError("length_penalty (alpha) should be a value between 0 and 1")


class DecodingTask:
    def __init__(self, model: "OLMoASRBase", options: DecodingOptions):
        verify_options(options)
        if options.beam_size is not None:
            if not (USE_ENGINE and hasattr(model, "decode_engine")):
                raise NotImplementedError("beam search runs on the device decoder only (model.decode_engine)")
            from .decode_engine import BEAM_MAX, MAX_CANDIDATES
            if not 1 <= options.beam_size <= BEAM_MAX:
                raise ValueError(f"beam_size must be in 1 .. {BEAM_MAX}")
            if not 1 <= round(options.beam_size * (options.patience or 1.0)) <= MAX_CANDIDATES:
                raise ValueError(f"round(beam_size * patience) must be in 1 .. {MAX_CANDIDATES}")
        if options.fp8 and not (USE_ENGINE and hasattr(model, "decode_engine")):
            raise NotImplementedError("fp8 decoding runs on the device decoder only (model.decode_engine)")
        if model.is_multilingual:
            raise NotImplementedError("only the English-only vocabulary of the OLMoASR checkpoints is supported")
        self.model, self.options = model, options
        self.n_group = options.beam_size or options.best_of or 1
        self.ranker = MaximumLikelihoodRanker(options.length_penalty)
        self.n_ctx = model.dims.n_text_ctx
        self.sample_len = options.sample_len or model.dims.n_text_ctx // 2
        sot_seq = [SOT] + ([NO_TIMESTAMPS] if options.without_timestamps else [])
        prefix = list(options.prefix) if isinstance(options.prefix, (list, tuple)) else []
        prompt = list(options.prompt) if isinstance(options.prompt, (list, tuple)) else []
        tokens = list(sot_seq)
        if prefix:
            tokens += prefix[-(self.n_ctx // 2 - self.sample_len):] if self.sample_len < self.n_ctx // 2 else prefix
        if prompt:
            tokens = [SOT_PREV] + prompt[-(self.n_ctx // 2 - 1):] + tokens
        self.initial_tokens = tuple(tokens)
        self.sample_begin = len(self.initial_tokens)
        self.sot_index = self.initial_tokens.index(SOT)
        self.suppress = suppress_token_ids(options) if options.suppress_tokens is not None else ()
        self.ts_rules = None
        if not options.without_timestamps:
            precision = 30.0 / model.dims.n_audio_ctx
            mi = round(options.max_initial_timestamp / precision) if options.max_initial_timestamp else None
            self.ts_rules = _TimestampRules(self.sample_begin, mi)

    @torch.no_grad()
    def run(self, mel: Tensor, tokenizer=None, sample_keys: Optional[Tuple[int, List[int]]] = None) -> List[DecodingResult]:
        """`sample_keys` = (seed, one clip id per clip) replaces the per-call seed and the clips' indices in the sampling
        keys of the device decoder, and its steps split the cross-attention as a one-clip call does (transcribe_batch():
        a window's draws and bits then do not depend on the other windows of its call).  The hook loop
        (OASR_DECODE_ENGINE=0) draws from torch's generator and makes no such promise."""
        from ._core import bf16_compute

        with bf16_compute(), self._window_splits(sample_keys):   # bf16 / the engine's type, also inside fp16 autocast
            return self._run(mel, tokenizer, sample_keys)

    def _window_splits(self, sample_keys):
        if sample_keys is None or not (USE_ENGINE and hasattr(self.model, "decode_engine")):
            return contextlib.nullcontext()
        return self._engine().splits_of(self.n_group)

    def _engine(self):
        """The device decoder these options select: activation dtype and weight / cross K/V storage.  The 16-bit engine
        is asked for as `decode_engine(dtype)`, the signature models without fp8 decoding implement."""
        dtype = torch.float16 if self.options.fp16 else torch.bfloat16
        return self.model.decode_engine(dtype, fp8=True) if self.options.fp8 else self.model.decode_engine(dtype)

    def _run(self, mel: Tensor, tokenizer=None, sample_keys=None) -> List[DecodingResult]:
        model, opt = self.model, self.options
        if mel.shape[-2:] == (model.dims.n_audio_ctx, model.dims.n_audio_state):
            audio_features = mel  # encoded features were passed in (DecodingTask._get_audio_features)
        else:
            audio_features = model.encoder(mel)
        n_audio = audio_features.shape[0]
        dev = audio_features.device
        if opt.beam_size is not None:
            return self._run_beam_on_device(audio_features, tokenizer)
        if USE_ENGINE and hasattr(model, "decode_engine"):
            eng = self._engine()
            if opt.temperature == 0:
                return self._run_on_device(audio_features, tokenizer, eng)
            if self.n_group <= eng.max_batch:
                return self._run_sampling_on_device(audio_features, tokenizer, eng, sample_keys)
        if opt.fp8:
            raise NotImplementedError(f"fp8 decoding runs on the device decoder only: best_of {self.n_group} needs the "
                                      "hook loop (more rows than the device decoder's batch)")
        G = self.n_group                           # best_of samples per clip (temperature > 0), rows clip-major
        xa = audio_features.repeat_interleave(G, dim=0) if G > 1 else audio_features
        n_rows = n_audio * G
        tokens = torch.tensor([self.initial_tokens], device=dev).repeat(n_rows, 1)
        sum_logprobs = torch.zeros(n_rows, device=dev)
        no_speech_probs = [np.nan] * n_rows
        suppress = torch.tensor(self.suppress, device=dev, dtype=torch.long) if self.suppress else None
        cache, hooks = model.install_kv_cache_hooks()
        try:
            for i in range(self.sample_len):
                inp = tokens if tokens.shape[-1] <= len(self.initial_tokens) else tokens[:, -1:]
                logits = model.decoder(inp, xa, kv_cache=cache)
                if i == 0:
                    probs_at_sot = logits[:, self.sot_index].float().softmax(dim=-1)
                    no_speech_probs = probs_at_sot[:, NO_SPEECH].tolist()
                logits = logits[:, -1]
                if opt.suppress_blank and tokens.shape[1] == self.sample_begin:
                    logits[:, [BLANK, EOT]] = -np.inf
                if suppress is not None:
                    logits[:, suppress] = -np.inf
                if self.ts_rules is not None:
                    self.ts_rules.apply(logits, tokens)
                # GreedyDecoder.update
                if opt.temperature == 0:
                    next_tokens = logits.argmax(dim=-1)
                else:
                    next_tokens = torch.distributions.Categorical(logits=logits / opt.temperature).sample()
                logprobs = F.log_softmax(logits.float(), dim=-1)
                current = logprobs[torch.arange(n_rows, device=dev), next_tokens]
                sum_logprobs += current * (tokens[:, -1] != EOT)
                next_tokens[tokens[:, -1] == EOT] = EOT
                tokens = torch.cat([tokens, next_tokens[:, None]], dim=-1)
                if bool((tokens[:, -1] == EOT).all()) or tokens.shape[-1] > self.n_ctx:
                    break
        finally:
            for h in hooks:
                h.remove()
        tokens = F.pad(tokens, (0, 1), value=EOT)  # GreedyDecoder.finalize
        if G == 1:
            return self._results(audio_features, tokens, sum_logprobs.tolist(), no_speech_probs, tokenizer)
        rows, lps = tokens.tolist(), sum_logprobs.tolist()
        candidates = [[(rows[k * G + j], lps[k * G + j]) for j in range(G)] for k in range(n_audio)]
        return self._ranked(audio_features, candidates, no_speech_probs[::G], tokenizer)

    def _run_beam_on_device(self, audio_features: Tensor, tokenizer):
        """Beam search (the long-form eval configuration, scripts/eval/eval.py:2077-2084) on the device decoder: one CUDA
        graph replay per step, candidates / ranking / kv reorder in kernels, up to 64 // beam_size clips per call."""
        opt = self.options
        eng = self._engine()
        per = eng.max_batch // opt.beam_size
        ts = self.ts_rules is not None
        mi = self.ts_rules.max_initial_timestamp_index if ts else None
        candidates, nsp = [], []
        for s in range(0, audio_features.shape[0], per):
            c, ns, _ = eng.beam_search(audio_features[s:s + per], self.initial_tokens, self.sample_len, opt.beam_size, opt.patience,
                                       self.suppress, opt.suppress_blank, self.sot_index, timestamps=ts,
                                       max_initial_timestamp_index=mi)
            candidates += c
            nsp += ns.tolist()
        return self._ranked(audio_features, candidates, nsp, tokenizer)

    def _ranked(self, audio_features, candidates, no_speech_probs, tokenizer) -> List[DecodingResult]:
        """DecodingTask.run after finalize: candidates[k] = [(full token row ending in eot, sum_logprob), ...]; each is cut
        to the sampled tokens before the first eot and the ranker picks one per clip."""
        opt = self.options
        tokens, sum_logprobs = [], []
        for cands in candidates:
            seqs = []
            for row, _ in cands:
                seq = row[self.sample_begin:]
                seqs.append(seq[: seq.index(EOT)] if EOT in seq else seq)
            tokens.append(seqs)
            sum_logprobs.append([lp for _, lp in cands])
        selected = self.ranker.rank(tokens, sum_logprobs)
        results = []
        for k, i in enumerate(selected):
            ids, lp = tokens[k][i], sum_logprobs[k][i]
            text = tokenizer.decode([t for t in ids if t < EOT]).strip() if tokenizer is not None else ""
            results.append(DecodingResult(audio_features=audio_features[k], language="en", tokens=ids, text=text,
                                          avg_logprob=lp / (len(ids) + 1), no_speech_prob=no_speech_probs[k],
                                          temperature=opt.temperature))
        return results

    def _run_sampling_on_device(self, audio_features: Tensor, tokenizer, eng, sample_keys=None):
        """Temperature sampling, best_of samples per clip (every fallback temperature of transcribe()), on the device
        decoder: up to max_batch // best_of clips per call, ranked like the hook loop.  One seed per decode() call from
        torch's default generator; each clip's draws depend on it and on the clip's index in this call only.  With
        `sample_keys` = (seed, clip ids) the given seed and each clip's own id key the draws instead."""
        opt, G = self.options, self.n_group
        per = eng.max_batch // G
        ts = self.ts_rules is not None
        mi = self.ts_rules.max_initial_timestamp_index if ts else None
        seed = int(torch.randint(2 ** 62, (1,))) if sample_keys is None else sample_keys[0]
        candidates, nsp = [], []
        for s in range(0, audio_features.shape[0], per):
            ids = {} if sample_keys is None else dict(clip_ids=list(sample_keys[1][s:s + per]))
            c, ns, _ = eng.sample(audio_features[s:s + per], self.initial_tokens, self.sample_len, opt.temperature, G, seed, s,
                                  self.suppress, opt.suppress_blank, self.sot_index, timestamps=ts, max_initial_timestamp_index=mi,
                                  **ids)
            candidates += c
            nsp += ns.tolist()
        return self._ranked(audio_features, candidates, nsp, tokenizer)

    def _run_on_device(self, audio_features: Tensor, tokenizer, eng):
        """Greedy decoding (the short-form eval configuration, scripts/eval/eval.py:1846-1847, and the temperature-0 step of
        transcribe() with timestamp rules): the whole loop runs as replays of one CUDA graph (olmoasr_b200/decode_engine.py),
        up to 64 clips per call."""
        from .decode_engine import DecodeEngine

        ts = self.ts_rules is not None
        mi = self.ts_rules.max_initial_timestamp_index if ts else None
        toks, lps, nsp = [], [], []
        for s in range(0, audio_features.shape[0], DecodeEngine.MAX_BATCH):
            t, lp, ns, _ = eng.greedy(audio_features[s:s + DecodeEngine.MAX_BATCH], self.initial_tokens, self.sample_len, self.suppress,
                                      self.options.suppress_blank, self.sot_index, timestamps=ts, max_initial_timestamp_index=mi)
            toks.append(t); lps += lp.tolist(); nsp += ns.tolist()
        width = max(t.shape[1] for t in toks)
        tokens = torch.cat([F.pad(t, (0, width - t.shape[1]), value=EOT) for t in toks], dim=0)
        tokens = F.pad(tokens, (0, 1), value=EOT)  # GreedyDecoder.finalize
        return self._results(audio_features, tokens, lps, nsp, tokenizer)

    def _results(self, audio_features, tokens, sum_logprobs, no_speech_probs, tokenizer) -> List[DecodingResult]:
        opt = self.options
        n_audio = audio_features.shape[0]
        results = []
        for k in range(n_audio):
            seq = tokens[k, self.sample_begin:]
            end = int((seq == EOT).nonzero()[0, 0])
            ids = seq[:end].tolist()
            text = tokenizer.decode([t for t in ids if t < EOT]).strip() if tokenizer is not None else ""
            results.append(DecodingResult(audio_features=audio_features[k], language="en", tokens=ids, text=text,
                                          avg_logprob=float(sum_logprobs[k]) / (len(ids) + 1),
                                          no_speech_prob=no_speech_probs[k], temperature=opt.temperature))
        return results


@torch.no_grad()
def decode(model: "OLMoASRBase", mel: Tensor, options: DecodingOptions = DecodingOptions(), tokenizer=None, **kwargs):
    """whisper.decoding.decode: mel (80, 3000) or (B, 80, 3000) -> DecodingResult or list of them."""
    single = mel.ndim == 2
    if single:
        mel = mel.unsqueeze(0)
    if kwargs:
        options = replace(options, **kwargs)
    result = DecodingTask(model, options).run(mel, tokenizer)
    return result[0] if single else result


@torch.no_grad()
def decode_windows(model: "OLMoASRBase", features: Tensor, options: DecodingOptions, tokenizer=None,
                   sample_keys: Optional[Tuple[int, List[int]]] = None) -> List[DecodingResult]:
    """decode() of (W, n_audio_ctx, n_audio_state) encoded features with per-window sampling keys (see
    `DecodingTask.run`): the route of transcribe_batch()."""
    return DecodingTask(model, options).run(features, tokenizer, sample_keys)


@torch.no_grad()
def detect_language(model: "OLMoASRBase", mel: Tensor, tokenizer=None):
    raise ValueError("This model doesn't have language tokens so it can't perform lang id")  # same error as upstream for *.en
