"""Device-resident greedy decoder (BASELINE.json config 5; SURVEY.md 8(f)-1): the kv-cache decode step of
olmoasr/inf_model.py:320-362 and the greedy loop of third-party whisper/decoding.py (DecodingTask._main_loop,
PyTorchInference.logits, SuppressBlank, SuppressTokens, GreedyDecoder.update) as ONE CUDA graph per batch size that is
replayed once per token.  Nothing of the step runs on the host: position, token ids, log-prob sums and the
all-sequences-finished flag live in device memory; the host only replays the graph and looks at the flag every few steps.

What the reference does per step and what replaces it:
  * re-casts every fp32 weight to fp16 (inf_model.py:56-60)            -> weights cast once into the activation dtype
  * builds the causal mask on the CPU and copies it over (:341-352)     -> single-query kernels need no mask
  * torch.cat of every self-attention K / V (hooks, :439-445)           -> pre-allocated (L, 2, N, 448, d) cache written
                                                                           in place by the fused QKV projection's epilogue
  * cross-attention K / V projected once, kept in the hook dict         -> projected once by the wgmma GEMM into a static
                                                                           (L, N*1500, 2d) buffer
  * 4 small matmul / softmax kernels per attention + separate LN, bias,
    GELU, residual kernels                                               -> 8-9 launches per layer (csrc/decode.cu), 100-112 per step (small)

`greedy(timestamps=True)` and `sample` (temperature sampling, best_of samples per clip) end the step graph in the
rule-aware sampling kernel instead: ApplyTimestampRules as index tests and a Gumbel-max draw keyed per row, with the
temperature and the keys read from device memory, so one graph per (rows, group size, timestamps) serves every
temperature and seed.  `beam_search` runs whisper/decoding.py's BeamSearchDecoder (with ApplyTimestampRules when asked)
the same way: the step graph ends in a candidate kernel, a per-clip ranking kernel that keeps the finished lists on the
device, and an in-place reorder of the self-attention cache.  The beams (or the best_of samples) of one clip share its
cross-attention K / V: one projection per clip.

The activation dtype is fp16 (upstream default `fp16=True`) or bf16; the decoder-step kernels reproduce the reference's
rounding points in that dtype.  The audio encoder and the cross K/V projection run on the bf16 wgmma kernels in both
cases (their bf16 outputs are converted to fp16 for an fp16 decoder).

`fp8=True` (DecodingOptions.fp8) halves the two large byte streams of the step.  The six block projections of every
layer are stored as e4m3 codes with one fp32 scale per output row, quantised in refresh_weights() from the 16-bit cast;
cross K / V is quantised in prepare() from the bf16 projection, with one scale per (key, head, K|V) group of 64.  Both
are decoded to the activation dtype in registers (include/oasr_b200.h states the arithmetic).  The tied logits head, the
self-attention cache and every activation stay 16-bit; the step issues the same launches as the 16-bit engine.
"""
from __future__ import annotations

import contextlib
import ctypes
import math
from typing import Dict, Optional, Sequence, Tuple

import torch
from torch import Tensor, nn

from . import _lib
from ._lib import (DTYPE_BF16, DTYPE_F16, DTYPE_F32, DecAttnArgs, DecBeamArgs, DecLinearArgs, DecSampleArgs, DecSampleRulesArgs,
                   call, ptr, stream)
from .kernels import FP8_E4M3, quantize_fp8_rows

X_PLAIN, X_LAYERNORM, X_PARTIAL_SUM = 0, 1, 2
EPI_STORE, EPI_GELU, EPI_RESIDUAL, EPI_LOGITS_F32, EPI_QKV_SCATTER = 0, 1, 2, 3, 4
_DT = {torch.float16: DTYPE_F16, torch.bfloat16: DTYPE_BF16, torch.float32: DTYPE_F32}
TIMESTAMP_BEGIN, NO_TIMESTAMPS = 50363, 50362
BEAM_MAX, MAX_CANDIDATES = 8, 32
BEAM_SCRATCH = 48      # floats per (row, slice) of the beam candidate and rule-aware sampling kernels
FP8_WEIGHTS = ("wqkv", "wo", "wcq", "wco", "w1", "w2")    # the per-layer projections an fp8 engine stores as e4m3


_M64 = (1 << 64) - 1


def _mix64(x: int) -> int:
    """splitmix64 (Steele, Lea, Flood: "Fast splittable pseudorandom number generators", OOPSLA 2014)."""
    x = (x + 0x9E3779B97F4A7C15) & _M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & _M64
    return x ^ (x >> 31)


def sample_row_key(seed: int, clip: int, sample: int) -> int:
    """The 64-bit Philox key of sample `sample` of clip `clip` (counted over the whole decode() call) under `seed`: a
    clip's draws do not depend on how the call is split into engine batches."""
    return _mix64(_mix64(_mix64(seed & _M64) ^ clip) ^ sample)


def window_clip_id(recording: int, seek: int, temperature_index: int) -> int:
    """The clip id of one transcribe_batch() window (passed to `DecodeEngine.sample` as `clip_ids`): the recording's
    index in the call, the window's seek frame and the temperature's index in the fallback tuple, mixed like
    `sample_row_key`, so a window's draws do not depend on which windows share its engine call."""
    return _mix64(_mix64(_mix64(recording & _M64) ^ (seek & _M64)) ^ (temperature_index & _M64))


def _convert(src: Tensor, dst: Tensor) -> Tensor:
    call("oasr_convert", ptr(src), _DT[src.dtype], ptr(dst), _DT[dst.dtype], src.numel(), stream())
    return dst


class DecodeEngine:
    MAX_BATCH = 64

    def __init__(self, model, dtype: torch.dtype = torch.float16, max_batch: int = 64, fp8: bool = False):
        if dtype not in (torch.float16, torch.bfloat16):
            raise ValueError("DecodeEngine: dtype must be torch.float16 or torch.bfloat16")
        if not 1 <= max_batch <= self.MAX_BATCH:
            raise ValueError(f"DecodeEngine: 1 <= max_batch <= {self.MAX_BATCH}")
        self.model = model
        self.dtype = dtype
        self.dt = _DT[dtype]
        dec = model.decoder
        self.dev = dec.token_embedding.weight.device
        if self.dev.type != "cuda":
            raise _lib.OasrError("DecodeEngine needs the model on a CUDA device (no CPU fallback)")
        dims = model.dims
        self.d, self.H, self.L = dims.n_text_state, dims.n_text_head, dims.n_text_layer
        self.n_ctx, self.n_audio_ctx = dims.n_text_ctx, dims.n_audio_ctx
        self.V = dec.token_embedding.weight.shape[0]
        if self.d != self.H * 64:
            raise ValueError("DecodeEngine: head dimension must be 64")
        self.max_batch = max_batch
        self.fp8 = bool(fp8)
        N, d, L = max_batch, self.d, self.L
        dev = self.dev
        z = lambda *shape, dt=dtype: torch.zeros(shape, device=dev, dtype=dt)
        # static state -- addresses are baked into the CUDA graphs
        self.self_k, self.self_v = z(L, N, self.n_ctx, d), z(L, N, self.n_ctx, d)
        if self.fp8:    # e4m3 codes; one fp32 scale per (key, head, K|V): K heads first, then V heads
            self.cross_kv = z(L, N * self.n_audio_ctx, 2 * d, dt=torch.uint8)
            self.cross_scale = z(L, N * self.n_audio_ctx, 2 * self.H, dt=torch.float32)
        else:
            self.cross_kv = z(L, N * self.n_audio_ctx, 2 * d)
            self.cross_scale = None
        self.x, self.q, self.h = z(N, d), z(N, d), z(N, 4 * d)
        self.scores = z(N, self.H, 1536, dt=torch.float32)
        self.max_splits = 8       # key-range splits of the cross-attention at small batches (each split's fp32 partial is re-read by the out projection)
        self.part_self = z(1, N, d, dt=torch.float32)
        self.part_cross = z(self.max_splits, N, d, dt=torch.float32)
        # rows padded to a multiple of 4 floats: the selection kernels read them with 16-byte loads, and a training-layout
        # model's vocabulary (n_vocab + 1 = 51865 with the pad row) is odd
        self.logits = z(N, (self.V + 3) & ~3, dt=torch.float32)[:, : self.V]
        self.tokens = torch.zeros((N, self.n_ctx + 2), device=dev, dtype=torch.int32)
        self.pos = torch.zeros(1, device=dev, dtype=torch.int32)
        self.sum_logprobs = z(N, dt=torch.float32)
        self.no_speech = z(N, dt=torch.float32)
        self.n_unfinished = torch.zeros(1, device=dev, dtype=torch.int32)
        self.done = torch.zeros(1, device=dev, dtype=torch.int32)
        self.suppress = torch.zeros(self.V, device=dev, dtype=torch.uint8)
        self.sample_slices = 16          # blocks per sequence in the sampling kernel
        self.sample_scratch = z(N, self.sample_slices, 8, dt=torch.float32)
        self.sample_counters = torch.zeros(N, device=dev, dtype=torch.int32)
        # beam search state (row = clip * beam + j): candidates per slice, source rows, finished lists per clip
        self.beam_scratch = z(N, self.sample_slices, BEAM_SCRATCH, dt=torch.float32)
        self.src_rows = torch.zeros(N, device=dev, dtype=torch.int32)
        self.fin_tokens = torch.zeros((N, MAX_CANDIDATES, self.n_ctx + 1), device=dev, dtype=torch.int32)
        self.fin_scores = z(N, MAX_CANDIDATES, dt=torch.float32)
        self.fin_len = torch.zeros((N, MAX_CANDIDATES), device=dev, dtype=torch.int32)
        self.fin_count = torch.zeros(N, device=dev, dtype=torch.int32)
        self.seq_len = torch.zeros(1, device=dev, dtype=torch.int32)
        # temperature sampling: read by the kernel at every replay (not baked into the graphs)
        self.temperature = z(1, dt=torch.float32)
        self.row_keys = torch.zeros(N, device=dev, dtype=torch.int64)
        self._rules_cfg = None     # (timestamps, max_initial_timestamp_index or -1, sampling) for the rule-aware sampler
        self._group = 1            # rows per clip that share one cross-attention K / V (beam size or best_of)
        self._beam_cfg = None      # (beam, clips, max_candidates, timestamps, max_initial_timestamp_index or -1) while beam searching
        self._w: Optional[dict] = None
        self._w_sig = None
        self._graphs: Dict[tuple, torch.cuda.CUDAGraph] = {}
        self._sample_cfg = None
        self.split_rows: Optional[int] = None   # see splits_of()
        self.launches_per_step = 0

    # ---- weights ----------------------------------------------------------------------------------------------
    def _params(self):
        return [p for p in self.model.decoder.parameters()]

    def refresh_weights(self):
        """(Re)cast the decoder weights into the activation dtype when a parameter changed (checkpoint load, training);
        an fp8 engine then quantises the block projections (FP8_WEIGHTS) per output row and keeps only the e4m3 codes
        and their scales (`<name>_s`)."""
        sig = tuple((p.data_ptr(), p._version) for p in self._params())
        if sig == self._w_sig:
            return
        from .lora import effective_weight
        dec, d, T = self.model.decoder, self.d, self.dtype

        def cast(*ps, dtype=T):
            # a Linear with an adapter contributes its effective weight W + s B A
            ps = [effective_weight(p) if isinstance(p, nn.Module) else p for p in ps]
            out = torch.empty((sum(p.shape[0] for p in ps), ps[0].shape[1]), device=self.dev, dtype=dtype)
            r = 0
            for p in ps:
                _convert(p.detach().contiguous(), out[r:r + p.shape[0]])
                r += p.shape[0]
            return out

        layers = []
        for blk in dec.blocks:
            a, c = blk.attn, blk.cross_attn
            zeros = torch.zeros(d, device=self.dev)
            layers.append(dict(
                wqkv=cast(a.query, a.key, a.value),
                bqkv=torch.cat([a.query.bias.detach().float(), zeros, a.value.bias.detach().float()]).contiguous(),
                wo=cast(a.out), bo=a.out.bias.detach().float().contiguous(),
                wcq=cast(c.query), bcq=c.query.bias.detach().float().contiguous(),
                wco=cast(c.out), bco=c.out.bias.detach().float().contiguous(),
                w1=cast(blk.mlp[0]), b1=blk.mlp[0].bias.detach().float().contiguous(),
                w2=cast(blk.mlp[2]), b2=blk.mlp[2].bias.detach().float().contiguous(),
                # the bf16 cross K / V weight prepare() runs on the encoder output, when an adapter changes it
                wckv=cast(c.key, c.value, dtype=torch.bfloat16) if (c.key.has_lora or c.value.has_lora) else None,
                ln1=(blk.attn_ln.weight.detach(), blk.attn_ln.bias.detach(), blk.attn_ln.eps),
                lnc=(blk.cross_attn_ln.weight.detach(), blk.cross_attn_ln.bias.detach(), blk.cross_attn_ln.eps),
                ln2=(blk.mlp_ln.weight.detach(), blk.mlp_ln.bias.detach(), blk.mlp_ln.eps)))
            if self.fp8:
                lw = layers[-1]
                for name in FP8_WEIGHTS:
                    lw[name], lw[name + "_s"] = quantize_fp8_rows(lw[name], FP8_E4M3)
        self._w = dict(layers=layers, emb_t=cast(dec.token_embedding.weight), emb=dec.token_embedding.weight.detach(),
                       pos=dec.positional_embedding.detach(), ln=(dec.ln.weight.detach(), dec.ln.bias.detach(), dec.ln.eps))
        self._w_sig = sig
        self._graphs.clear()        # weight buffers were re-allocated: graphs hold their addresses

    # ---- kernel wrappers ----------------------------------------------------------------------------------------
    def _linear(self, n, x, W, bias, out, *, x_mode=X_PLAIN, ln=None, epi=EPI_STORE, res=None, n_partials=0, kv=None, K_=None,
                w_scale=None):
        """One skinny Linear; `w_scale` (N,) fp32 means W holds e4m3 codes (oasr_dec_linear_fp8w)."""
        a = DecLinearArgs()
        a.x, a.x_mode, a.n_partials = ptr(x), x_mode, n_partials
        a.K = W.shape[1] if K_ is None else K_
        a.ldx = x.stride(-2) if x_mode != X_PARTIAL_SUM else a.K
        a.partial_stride = x.stride(0) if x_mode == X_PARTIAL_SUM else 0
        if ln is not None:
            a.ln_gamma, a.ln_beta, a.ln_eps = ptr(ln[0]), ptr(ln[1]), float(ln[2])
        a.epi, a.W, a.bias = epi, ptr(W), ptr(bias)
        a.out, a.ldo = ptr(out), out.stride(0)
        if res is not None:
            a.res, a.ldres = ptr(res), res.stride(0)
        if kv is not None:
            a.k_cache, a.v_cache, a.cache_len, a.pos_ptr = ptr(kv[0]), ptr(kv[1]), self.n_ctx, ptr(self.pos)
        a.M, a.N, a.dtype = n, W.shape[0], self.dt
        if w_scale is None:
            call("oasr_dec_linear", ctypes.byref(a), stream())
        else:
            call("oasr_dec_linear_fp8w", ctypes.byref(a), ptr(w_scale), stream())

    def _attention(self, n, k, v, seq_stride, row_stride, part, splits, n_keys=None, kv_group=1, kv_scales=None):
        """One decode attention; kv_scales = (k_scale, v_scale, seq stride, row stride) means k / v hold e4m3 codes with
        one scale per (key, head) (oasr_dec_attention_fp8kv)."""
        a = DecAttnArgs()
        a.q, a.ldq = ptr(self.q), self.q.stride(0)
        a.k, a.v, a.kv_seq_stride, a.kv_row_stride = ptr(k), ptr(v), seq_stride, row_stride
        a.scores, a.scores_ld = ptr(self.scores), self.scores.stride(1)
        a.out_partial, a.ld_out = ptr(part), self.d
        a.pos_ptr = None if n_keys is not None else ptr(self.pos)
        a.n_keys = n_keys or 0
        a.n_seq, a.n_head, a.n_splits, a.scale, a.dtype = n, self.H, splits, 64 ** -0.25, self.dt
        if kv_scales is not None:
            ks, vs, s_seq, s_row = kv_scales
            call("oasr_dec_attention_fp8kv", ctypes.byref(a), ptr(ks), ptr(vs), s_seq, s_row, kv_group, stream())
        elif kv_group == 1:
            call("oasr_dec_attention", ctypes.byref(a), stream())
        else:                           # sequence r reads cross K / V entry r // kv_group (the beams of one clip)
            call("oasr_dec_attention_grouped", ctypes.byref(a), kv_group, stream())
        if splits == 1:
            _lib.LAUNCH_COUNT -= 1      # an unsplit key range runs as ONE fused kernel (scores + softmax + P V), not two

    def cross_splits(self, n: int) -> int:
        """Key-range splits of the cross-attention so that n x H x splits CTAs cover the SMs about twice."""
        return max(1, min(self.max_splits, math.ceil(2 * _lib.lib().oasr_device_sm_count() / (n * self.H))))

    @contextlib.contextmanager
    def splits_of(self, rows: int):
        """Inside, every step splits the cross-attention key range as a step of `rows` rows would, whatever its row count.
        The fp32 partial sums of a sequence then group alike in calls of any size, so its logits have the same bits
        alone and inside a batch (transcribe_batch() windows equal transcribe()'s)."""
        prev, self.split_rows = self.split_rows, rows
        try:
            yield
        finally:
            self.split_rows = prev

    def _enqueue_step(self, n: int):
        """One decoder step for sequences [0, n): per layer 6 fused Linear launches, 1 self-attention launch and 1 (unsplit key
        range) or 2 (split) cross-attention launches; plus the embedding, the logits head and the 2 sampling launches."""
        w, d = self._w, self.d
        c0 = _lib.LAUNCH_COUNT
        call("oasr_dec_embed", ptr(self.tokens), self.tokens.stride(0), ptr(self.pos), ptr(w["emb"]), ptr(w["pos"]), ptr(self.x),
             n, d, self.V, self.dt, stream())
        sc = self.cross_splits(self.split_rows or n)
        seq_self, seq_cross = self.n_ctx * d, self.n_audio_ctx * 2 * d
        x, q, h = self.x[:n], self.q[:n], self.h[:n]
        # the attention kernels lay their fp32 partial outputs out as (splits, n, d): views with exactly that geometry
        part_self = self.part_self.view(-1)[: n * d].view(1, n, d)
        part_cross = self.part_cross.view(-1)[: sc * n * d].view(sc, n, d)
        kv_group = self._group
        # fp8: the scales ride along as keyword arguments (the 16-bit engine's calls are exactly what they were)
        ws = (lambda lw, name: {"w_scale": lw[name + "_s"]}) if self.fp8 else (lambda lw, name: {})
        for l, lw in enumerate(w["layers"]):
            self._linear(n, x, lw["wqkv"], lw["bqkv"], q, x_mode=X_LAYERNORM, ln=lw["ln1"], epi=EPI_QKV_SCATTER,
                         kv=(self.self_k[l], self.self_v[l]), **ws(lw, "wqkv"))
            self._attention(n, self.self_k[l], self.self_v[l], seq_self, d, part_self, 1)
            self._linear(n, part_self, lw["wo"], lw["bo"], x, x_mode=X_PARTIAL_SUM, n_partials=1, epi=EPI_RESIDUAL, res=x,
                         **ws(lw, "wo"))
            self._linear(n, x, lw["wcq"], lw["bcq"], q, x_mode=X_LAYERNORM, ln=lw["lnc"], **ws(lw, "wcq"))
            ckv = self.cross_kv[l]
            kvs = {}
            if self.fp8:
                cs = self.cross_scale[l]
                kvs = {"kv_scales": (cs, cs[:, self.H:], self.n_audio_ctx * cs.stride(0), cs.stride(0))}
            self._attention(n, ckv, ckv[:, d:], seq_cross, 2 * d, part_cross, sc, n_keys=self.n_audio_ctx, kv_group=kv_group,
                            **kvs)
            self._linear(n, part_cross, lw["wco"], lw["bco"], x, x_mode=X_PARTIAL_SUM, n_partials=sc, epi=EPI_RESIDUAL, res=x,
                         **ws(lw, "wco"))
            self._linear(n, x, lw["w1"], lw["b1"], h, x_mode=X_LAYERNORM, ln=lw["ln2"], epi=EPI_GELU, **ws(lw, "w1"))
            self._linear(n, h, lw["w2"], lw["b2"], x, epi=EPI_RESIDUAL, res=x, **ws(lw, "w2"))
        self._linear(n, x, w["emb_t"], None, self.logits, x_mode=X_LAYERNORM, ln=w["ln"], epi=EPI_LOGITS_F32)
        if self._beam_cfg is not None:
            self._enqueue_beam_select()
            self.launches_per_step = _lib.LAUNCH_COUNT - c0
            return
        if self._rules_cfg is not None:
            self._enqueue_sample_rules(n)
            self.launches_per_step = _lib.LAUNCH_COUNT - c0
            return
        s = DecSampleArgs()
        s.logits, s.ld_logits = ptr(self.logits), self.logits.stride(0)
        s.tokens, s.ld_tokens, s.pos_ptr = ptr(self.tokens), self.tokens.stride(0), ptr(self.pos)
        s.suppress, s.sum_logprobs, s.no_speech_prob = ptr(self.suppress), ptr(self.sum_logprobs), ptr(self.no_speech)
        s.n_unfinished, s.done_flag = ptr(self.n_unfinished), ptr(self.done)
        s.scratch, s.counters, s.n_slices = ptr(self.sample_scratch), ptr(self.sample_counters), self.sample_slices
        cfg = self._sample_cfg
        s.n_seq, s.n_vocab = n, self.V
        s.sample_begin, s.sot_index, s.suppress_blank, s.blank, s.eot, s.no_speech = cfg
        call("oasr_dec_sample", ctypes.byref(s), stream())
        self.launches_per_step = _lib.LAUNCH_COUNT - c0

    def _enqueue_sample_rules(self, n: int):
        """The rule-aware sampling step (timestamp rules and / or temperature sampling) + position advance: 2 launches."""
        ts, mi, sampling = self._rules_cfg
        s = DecSampleRulesArgs()
        s.logits, s.ld_logits = ptr(self.logits), self.logits.stride(0)
        s.tokens, s.ld_tokens, s.pos_ptr = ptr(self.tokens), self.tokens.stride(0), ptr(self.pos)
        s.suppress, s.sum_logprobs, s.no_speech_prob = ptr(self.suppress), ptr(self.sum_logprobs), ptr(self.no_speech)
        s.n_unfinished, s.done_flag = ptr(self.n_unfinished), ptr(self.done)
        s.scratch, s.counters, s.n_slices = ptr(self.beam_scratch), ptr(self.sample_counters), self.sample_slices
        if sampling:
            s.temperature, s.row_keys = ptr(self.temperature), ptr(self.row_keys)
        s.n_seq, s.n_vocab = n, self.V
        s.sample_begin, s.sot_index, s.suppress_blank, s.blank, s.eot, s.no_speech = self._sample_cfg
        s.timestamps, s.timestamp_begin, s.no_timestamps, s.max_initial_timestamp = ts, TIMESTAMP_BEGIN, NO_TIMESTAMPS, mi
        call("oasr_dec_sample_rules", ctypes.byref(s), stream())

    def _graph(self, n: int) -> torch.cuda.CUDAGraph:
        key = (n, self._sample_cfg, self._beam_cfg, self._rules_cfg, self._group, self.split_rows)
        g = self._graphs.get(key)
        if g is None:
            # one eager run first (kernel modules are loaded lazily on first launch, which must not happen under capture),
            # with the device-side decode state saved and restored around it; the capture itself does not execute
            live = (self.pos, self.tokens, self.sum_logprobs, self.no_speech, self.n_unfinished, self.done, self.sample_counters,
                    self.src_rows, self.fin_tokens, self.fin_scores, self.fin_len, self.fin_count, self.seq_len,
                    self.temperature, self.row_keys)
            state = [t.clone() for t in live]
            self._enqueue_step(n)
            torch.cuda.synchronize(self.dev)
            for t, saved in zip(live, state):
                t.copy_(saved)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._enqueue_step(n)
            self._graphs[key] = g
        return g

    # ---- public API ---------------------------------------------------------------------------------------------
    @torch.no_grad()
    def prepare(self, audio_features: Tensor):
        """Project the encoder output into every layer's cross-attention K / V once (inf_model.py:164-167: `kv_cache[self.key]`
        is filled on the first call and only read afterwards) with the wgmma GEMM.  An fp8 engine quantises the bf16
        projection as rows of 64 (one per key, head and K|V) into the e4m3 buffer and its scales, for either dtype."""
        from ._core import _as_bf16_2d, linear_fwd

        self.refresh_weights()
        if getattr(self.model, "_slabs", None) is not None:
            self.model._slabs.ensure_synced()    # the shadow slab in bf16 again after an fp16 training step
        n = audio_features.shape[0]
        if n > self.max_batch:
            raise ValueError(f"DecodeEngine: {n} sequences > max_batch {self.max_batch}")
        if tuple(audio_features.shape[1:]) != (self.n_audio_ctx, self.d):
            raise ValueError(f"audio_features must be (N, {self.n_audio_ctx}, {self.d})")
        xa = _as_bf16_2d(audio_features)
        rows = n * self.n_audio_ctx
        for l, blk in enumerate(self.model.decoder.blocks):
            wkv, bkv = blk.cross_attn.fused_kv()
            if self._w["layers"][l]["wckv"] is not None:
                wkv = self._w["layers"][l]["wckv"]
            if self.fp8:
                kv = linear_fwd(xa, wkv, bkv)
                call("oasr_quantize_fp8_rows", ptr(kv), 64, rows * 2 * self.H, 64, DTYPE_BF16, FP8_E4M3, 0,
                     ptr(self.cross_kv[l]), 64, ptr(self.cross_scale[l]), stream())
            elif self.dtype == torch.bfloat16:
                linear_fwd(xa, wkv, bkv, out=self.cross_kv[l][:rows])
            else:
                _convert(linear_fwd(xa, wkv, bkv), self.cross_kv[l][:rows])
        return n

    @torch.no_grad()
    def reset(self, n: int, tokens: Tensor, sample_begin: Optional[int] = None, suppress: Sequence[int] = (),
              suppress_blank: bool = True, sot_index: int = 0, blank: int = 220, eot: int = 50256, no_speech: int = 50361):
        """Start a decode of `n` sequences (after `prepare`): `tokens` (n, P) are the given tokens per sequence; positions
        before sample_begin - 1 (default P - 1) are teacher-forced, from there on every replay appends one sampled token."""
        P = tokens.shape[1]
        if tokens.shape[0] != n or not 1 <= P <= self.n_ctx:
            raise ValueError("reset: tokens must be (n, 1 .. n_text_ctx)")
        self.tokens.zero_()
        self.tokens[:n, :P] = tokens.to(device=self.dev, dtype=torch.int32)
        self.pos.zero_(); self.sum_logprobs.zero_(); self.no_speech.zero_(); self.n_unfinished.zero_(); self.done.zero_()
        self.sample_counters.zero_()
        sup = torch.zeros(self.V, dtype=torch.uint8)
        ids = [t for t in suppress if 0 <= t < self.V]
        if ids:
            sup[torch.tensor(ids, dtype=torch.long)] = 1
        self.suppress.copy_(sup)
        self._sample_cfg = (P if sample_begin is None else sample_begin, sot_index, int(bool(suppress_blank)), blank, eot, no_speech)
        self._beam_cfg = None
        self._rules_cfg = None
        self._group = 1

    def replay(self, n: int):
        """One decoder step for sequences [0, n): feeds the token at the device-side position, leaves the fp32 logits of that
        position in `self.logits[:n]`, appends the sampled token when past the teacher-forced prefix, advances the position."""
        self._graph(n).replay()

    @torch.no_grad()
    def greedy(self, audio_features: Tensor, initial_tokens: Sequence[int], sample_len: int, suppress: Sequence[int] = (),
               suppress_blank: bool = True, sot_index: int = 0, blank: int = 220, eot: int = 50256, no_speech: int = 50361,
               check_every: int = 8, timestamps: bool = False,
               max_initial_timestamp_index: Optional[int] = None) -> Tuple[Tensor, Tensor, Tensor, int]:
        """Returns (tokens (N, len) int64 on the host incl. the initial tokens, sum_logprobs (N,), no_speech_probs (N,),
        number of graph replays).  Semantics of DecodingTask._main_loop for temperature 0, with ApplyTimestampRules when
        `timestamps`."""
        n = self.prepare(audio_features)
        init = list(initial_tokens)
        n_init = len(init)
        if not 1 <= n_init < self.n_ctx:
            raise ValueError("initial_tokens: need 1 .. n_text_ctx-1 tokens")
        self.reset(n, torch.tensor([init], dtype=torch.int32).repeat(n, 1), None, suppress, suppress_blank, sot_index, blank, eot, no_speech)
        if timestamps:
            self._rules_cfg = (1, -1 if max_initial_timestamp_index is None else int(max_initial_timestamp_index), 0)
        return self._run(n, n_init, sample_len, check_every)

    def _run(self, n: int, n_init: int, sample_len: int, check_every: int) -> Tuple[Tensor, Tensor, Tensor, int]:
        """Replay the step graph of the configured decode until every row has ended (looked at every `check_every` sampled
        tokens) or the length limit; (tokens, sum_logprobs, no_speech_probs, replays) as `greedy` returns them."""
        g = self._graph(n)
        # positions 0 .. n_init-2 are teacher-forced; every replay from position n_init-1 on samples one token; the loop
        # of the reference also ends when the sequence would exceed n_text_ctx (whisper/decoding.py: tokens.shape[-1] > n_ctx)
        n_sampling = min(sample_len, self.n_ctx + 1 - n_init)
        total = (n_init - 1) + n_sampling
        replays = 0
        for i in range(total):
            g.replay()
            replays += 1
            sampled = replays - (n_init - 1)
            if sampled > 0 and sampled % check_every == 0 and i + 1 < total and int(self.done.item()) == 1:
                break
        length = n_init + max(0, replays - (n_init - 1))
        return (self.tokens[:n, :length].to(torch.int64).cpu(), self.sum_logprobs[:n].clone(), self.no_speech[:n].clone(), replays)

    @torch.no_grad()
    def sample(self, audio_features: Tensor, initial_tokens: Sequence[int], sample_len: int, temperature: float,
               best_of: int = 1, seed: int = 0, clip_offset: int = 0, suppress: Sequence[int] = (), suppress_blank: bool = True,
               sot_index: int = 0, timestamps: bool = False, max_initial_timestamp_index: Optional[int] = None,
               blank: int = 220, eot: int = 50256, no_speech: int = 50361, check_every: int = 8,
               clip_ids: Optional[Sequence[int]] = None):
        """Temperature sampling with `best_of` samples per clip (DecodingTask._main_loop with GreedyDecoder at temperature
        > 0, and ApplyTimestampRules when `timestamps`).  Row c * best_of + j draws with the key sample_row_key(seed,
        clip_offset + c, j), or sample_row_key(seed, clip_ids[c], j) when `clip_ids` (one per clip) are given.  Cross K/V is projected once per clip and shared by its samples.  Returns (candidates,
        no_speech_probs (n_clips,), number of graph replays): candidates[c] is the list of best_of (token ids incl. the
        initial tokens and the final eot, sum_logprob), as `beam_search` returns them."""
        G = int(best_of)
        C = audio_features.shape[0]
        if not temperature > 0:
            raise ValueError(f"sample: temperature must be > 0 (got {temperature}); use greedy() for temperature 0")
        if not 1 <= G <= self.max_batch or C * G > self.max_batch:
            raise ValueError(f"sample: at most {self.max_batch // max(G, 1)} clips per call at best_of {G} (got {C})")
        init = list(initial_tokens)
        n_init = len(init)
        if not 1 <= n_init < self.n_ctx:
            raise ValueError("initial_tokens: need 1 .. n_text_ctx-1 tokens")
        self.prepare(audio_features)
        n = C * G
        self.reset(n, torch.tensor([init], dtype=torch.int32).repeat(n, 1), None, suppress, suppress_blank, sot_index, blank, eot, no_speech)
        mi = -1 if max_initial_timestamp_index is None else int(max_initial_timestamp_index)
        self._rules_cfg = (int(bool(timestamps)), mi, 1)
        self._group = G
        if clip_ids is not None and len(clip_ids) != C:
            raise ValueError(f"sample: {len(clip_ids)} clip ids for {C} clips")
        ids = list(clip_ids) if clip_ids is not None else [clip_offset + c for c in range(C)]
        keys = [sample_row_key(seed, ids[c], j) for c in range(C) for j in range(G)]
        self.row_keys[:n] = torch.tensor([k - (1 << 64) if k >> 63 else k for k in keys], dtype=torch.int64)
        self.temperature.fill_(float(temperature))
        toks, lps, nsp, replays = self._run(n, n_init, sample_len, check_every)
        rows, lps = toks.tolist(), lps.tolist()
        candidates = [[(rows[c * G + j] + [eot], lps[c * G + j]) for j in range(G)] for c in range(C)]
        return candidates, nsp[::G], replays

    # ---- beam search ------------------------------------------------------------------------------------------------
    def reset_beam(self, n_clips: int, beam: int, max_candidates: int, timestamps: bool = False,
                   max_initial_timestamp_index: Optional[int] = None):
        """Switch the state left by `reset` (n_clips * beam rows) to beam search: empty finished lists, identity sources."""
        self.fin_count.zero_(); self.fin_len.zero_(); self.seq_len.zero_()
        self.src_rows.copy_(torch.arange(self.max_batch, device=self.dev, dtype=torch.int32))
        mi = -1 if max_initial_timestamp_index is None else int(max_initial_timestamp_index)
        self._beam_cfg = (beam, n_clips, max_candidates, int(bool(timestamps)), mi)
        self._group = beam

    def beam_args(self) -> DecBeamArgs:
        """Argument block of the beam candidate / select kernels for the current state."""
        beam, clips, max_cand, ts, mi = self._beam_cfg
        sample_begin, sot_index, suppress_blank, blank, eot, no_speech = self._sample_cfg
        a = DecBeamArgs()
        a.logits, a.ld_logits = ptr(self.logits), self.logits.stride(0)
        a.tokens, a.ld_tokens, a.pos_ptr = ptr(self.tokens), self.tokens.stride(0), ptr(self.pos)
        a.suppress, a.sum_logprobs, a.no_speech_prob = ptr(self.suppress), ptr(self.sum_logprobs), ptr(self.no_speech)
        a.n_unfinished, a.done_flag = ptr(self.n_unfinished), ptr(self.done)
        a.scratch, a.src_rows = ptr(self.beam_scratch), ptr(self.src_rows)
        a.fin_tokens, a.ld_fin = ptr(self.fin_tokens), self.fin_tokens.stride(1)
        a.fin_scores, a.fin_len, a.fin_count, a.seq_len = ptr(self.fin_scores), ptr(self.fin_len), ptr(self.fin_count), ptr(self.seq_len)
        a.n_clips, a.beam, a.max_candidates, a.n_vocab, a.n_slices, a.n_ctx = clips, beam, max_cand, self.V, self.sample_slices, self.n_ctx
        a.sample_begin, a.sot_index, a.suppress_blank, a.blank, a.eot, a.no_speech = sample_begin, sot_index, suppress_blank, blank, eot, no_speech
        a.timestamps, a.timestamp_begin, a.no_timestamps, a.max_initial_timestamp = ts, TIMESTAMP_BEGIN, NO_TIMESTAMPS, mi
        return a

    def finished_lists(self, n_clips: int, max_candidates: int):
        """(count (C,), lengths (C, M), token rows (C, M, n_ctx + 1), scores (C, M)) views of the device finished lists
        (the kernels lay them out clip-major with max_candidates entries per clip)."""
        C, M, ld = n_clips, max_candidates, self.fin_tokens.shape[-1]
        return (self.fin_count[:C], self.fin_len.view(-1)[: C * M].view(C, M),
                self.fin_tokens.view(-1, ld)[: C * M].view(C, M, ld), self.fin_scores.view(-1)[: C * M].view(C, M))

    def reorder_blocks(self, n_clips: int) -> int:
        """Position blocks of the kv reorder grid (x 2 L layers-and-K/V x clips): about two CTAs per SM."""
        return max(1, min(self.n_ctx, math.ceil(2 * _lib.lib().oasr_device_sm_count() / (2 * self.L * n_clips))))

    def reorder_kv(self, n_clips: int, beam: int):
        call("oasr_dec_beam_reorder", ptr(self.self_k), ptr(self.self_v), self.self_k.stride(0), self.self_k.stride(1), self.L,
             ptr(self.src_rows), ptr(self.pos), n_clips, beam, self.d, self.reorder_blocks(n_clips), self.dt, stream())

    def _enqueue_beam_select(self):
        """Candidates, ranking + finished lists + position advance, kv reorder: 1 + 2 + 1 launches."""
        a = self.beam_args()
        call("oasr_dec_beam_candidates", ctypes.byref(a), stream())
        call("oasr_dec_beam_select", ctypes.byref(a), stream())
        self.reorder_kv(a.n_clips, a.beam)

    @torch.no_grad()
    def beam_search(self, audio_features: Tensor, initial_tokens: Sequence[int], sample_len: int, beam_size: int,
                    patience: Optional[float] = None, suppress: Sequence[int] = (), suppress_blank: bool = True,
                    sot_index: int = 0, timestamps: bool = False, max_initial_timestamp_index: Optional[int] = None,
                    blank: int = 220, eot: int = 50256, no_speech: int = 50361, check_every: int = 8):
        """Beam search over the clips of `audio_features` (whisper/decoding.py BeamSearchDecoder, with ApplyTimestampRules
        when `timestamps`).  Cross K/V is projected once per clip and shared by its beams.  Returns (candidates,
        no_speech_probs (n_clips,), number of graph replays): candidates[c] is the list of (token ids incl. the initial
        tokens and the final eot, sum_logprob) of BeamSearchDecoder.finalize, in its order."""
        import numpy as np

        if not 1 <= beam_size <= BEAM_MAX:
            raise ValueError(f"beam_size must be in 1 .. {BEAM_MAX} (got {beam_size})")
        max_cand = round(beam_size * (patience or 1.0))
        if not 1 <= max_cand <= MAX_CANDIDATES:
            raise ValueError(f"round(beam_size * patience) must be in 1 .. {MAX_CANDIDATES} (got {max_cand})")
        C = audio_features.shape[0]
        if C * beam_size > self.max_batch:
            raise ValueError(f"beam search: at most {self.max_batch // beam_size} clips per call at beam {beam_size} (got {C})")
        init = list(initial_tokens)
        n_init = len(init)
        if not 1 <= n_init < self.n_ctx:
            raise ValueError("initial_tokens: need 1 .. n_text_ctx-1 tokens")
        self.prepare(audio_features)
        n = C * beam_size
        self.reset(n, torch.tensor([init], dtype=torch.int32).repeat(n, 1), None, suppress, suppress_blank, sot_index, blank, eot, no_speech)
        self.reset_beam(C, beam_size, max_cand, timestamps, max_initial_timestamp_index)
        g = self._graph(n)
        n_sampling = min(sample_len, self.n_ctx + 1 - n_init)
        total = (n_init - 1) + n_sampling
        replays = 0
        for i in range(total):
            g.replay()
            replays += 1
            sampled = replays - (n_init - 1)
            if sampled > 0 and sampled % check_every == 0 and i + 1 < total and int(self.done.item()) == 1:
                break
        # one copy to the host at the end; BeamSearchDecoder.finalize there
        seq_len = int(self.seq_len.item())
        toks = self.tokens[:n, :seq_len].cpu()
        lps = self.sum_logprobs[:n].cpu()
        cnt, lens, fin, scores = (t.cpu() for t in self.finished_lists(C, max_cand))
        nsp = self.no_speech[:n:beam_size].clone()
        candidates = []
        for c in range(C):
            seqs = [(fin[c, i, : int(lens[c, i])].tolist(), float(scores[c, i])) for i in range(int(cnt[c]))]
            if len(seqs) < beam_size:        # not enough finished: the live beams, best first, each closed by eot
                lp = lps[c * beam_size:(c + 1) * beam_size]
                for j in list(np.argsort(lp.numpy()))[::-1]:
                    seqs.append((toks[c * beam_size + j].tolist() + [eot], float(lp[j])))
                    if len(seqs) >= beam_size:
                        break
            candidates.append(seqs)
        return candidates, nsp, replays

    # ---- roofline bookkeeping --------------------------------------------------------------------------------------
    def step_bytes(self, n: int, t: int) -> int:
        """Algorithmic HBM bytes of one step at self-attention length t (SURVEY.md 8(d)): every decoder weight once (shared by
        the batch), per sequence the cross K/V of every layer, the self K/V read so far, and the fp32 logits row.  An
        fp8 engine reads one byte per block-projection weight plus a 4-byte scale per output row, and one byte per cross
        K/V element plus a 4-byte scale per (key, head, K|V); the logits head and the self K/V stay 16-bit."""
        e = 2
        d, L, H = self.d, self.L, self.H
        block = 3 * d * d + d * d + d * d + d * d + 8 * d * d    # qkv, out, cross q, cross out, fc1 + fc2
        rows = 3 * d + d + d + d + 4 * d + d                      # their output rows
        if self.fp8:
            weights = L * (block + 4 * rows) + self.V * d * e
            cross = L * self.n_audio_ctx * (2 * d + 4 * 2 * H)
        else:
            weights = L * block * e + self.V * d * e
            cross = L * 2 * self.n_audio_ctx * d * e
        self_kv = L * 2 * t * d * e
        return weights + n * (cross + self_kv + self.V * 4)
