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

The activation dtype is fp16 (upstream default `fp16=True`) or bf16; the decoder-step kernels reproduce the reference's
rounding points in that dtype.  The audio encoder and the cross K/V projection run on the bf16 wgmma kernels in both
cases (their bf16 outputs are converted to fp16 for an fp16 decoder).
"""
from __future__ import annotations

import ctypes
import math
from typing import Dict, Optional, Sequence, Tuple

import torch
from torch import Tensor

from . import _lib
from ._lib import DTYPE_BF16, DTYPE_F16, DTYPE_F32, DecAttnArgs, DecLinearArgs, DecSampleArgs, call, ptr, stream

X_PLAIN, X_LAYERNORM, X_PARTIAL_SUM = 0, 1, 2
EPI_STORE, EPI_GELU, EPI_RESIDUAL, EPI_LOGITS_F32, EPI_QKV_SCATTER = 0, 1, 2, 3, 4
_DT = {torch.float16: DTYPE_F16, torch.bfloat16: DTYPE_BF16, torch.float32: DTYPE_F32}


def _convert(src: Tensor, dst: Tensor) -> Tensor:
    call("oasr_convert", ptr(src), _DT[src.dtype], ptr(dst), _DT[dst.dtype], src.numel(), stream())
    return dst


class DecodeEngine:
    MAX_BATCH = 64

    def __init__(self, model, dtype: torch.dtype = torch.float16, max_batch: int = 64):
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
        N, d, L = max_batch, self.d, self.L
        dev = self.dev
        z = lambda *shape, dt=dtype: torch.zeros(shape, device=dev, dtype=dt)
        # static state -- addresses are baked into the CUDA graphs
        self.self_k, self.self_v = z(L, N, self.n_ctx, d), z(L, N, self.n_ctx, d)
        self.cross_kv = z(L, N * self.n_audio_ctx, 2 * d)
        self.x, self.q, self.h = z(N, d), z(N, d), z(N, 4 * d)
        self.scores = z(N, self.H, 1536, dt=torch.float32)
        self.max_splits = 8       # key-range splits of the cross-attention at small batches (each split's fp32 partial is re-read by the out projection)
        self.part_self = z(1, N, d, dt=torch.float32)
        self.part_cross = z(self.max_splits, N, d, dt=torch.float32)
        self.logits = z(N, self.V, dt=torch.float32)
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
        self._w: Optional[dict] = None
        self._w_sig = None
        self._graphs: Dict[tuple, torch.cuda.CUDAGraph] = {}
        self._sample_cfg = None
        self.launches_per_step = 0

    # ---- weights ----------------------------------------------------------------------------------------------
    def _params(self):
        return [p for p in self.model.decoder.parameters()]

    def refresh_weights(self):
        """(Re)cast the decoder weights into the activation dtype when a parameter changed (checkpoint load, training)."""
        sig = tuple((p.data_ptr(), p._version) for p in self._params())
        if sig == self._w_sig:
            return
        dec, d, T = self.model.decoder, self.d, self.dtype

        def cast(*ps):
            out = torch.empty((sum(p.shape[0] for p in ps), ps[0].shape[1]), device=self.dev, dtype=T)
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
                wqkv=cast(a.query.weight, a.key.weight, a.value.weight),
                bqkv=torch.cat([a.query.bias.detach().float(), zeros, a.value.bias.detach().float()]).contiguous(),
                wo=cast(a.out.weight), bo=a.out.bias.detach().float().contiguous(),
                wcq=cast(c.query.weight), bcq=c.query.bias.detach().float().contiguous(),
                wco=cast(c.out.weight), bco=c.out.bias.detach().float().contiguous(),
                w1=cast(blk.mlp[0].weight), b1=blk.mlp[0].bias.detach().float().contiguous(),
                w2=cast(blk.mlp[2].weight), b2=blk.mlp[2].bias.detach().float().contiguous(),
                ln1=(blk.attn_ln.weight.detach(), blk.attn_ln.bias.detach(), blk.attn_ln.eps),
                lnc=(blk.cross_attn_ln.weight.detach(), blk.cross_attn_ln.bias.detach(), blk.cross_attn_ln.eps),
                ln2=(blk.mlp_ln.weight.detach(), blk.mlp_ln.bias.detach(), blk.mlp_ln.eps)))
        self._w = dict(layers=layers, emb_t=cast(dec.token_embedding.weight), emb=dec.token_embedding.weight.detach(),
                       pos=dec.positional_embedding.detach(), ln=(dec.ln.weight.detach(), dec.ln.bias.detach(), dec.ln.eps))
        self._w_sig = sig
        self._graphs.clear()        # weight buffers were re-allocated: graphs hold their addresses

    # ---- kernel wrappers ----------------------------------------------------------------------------------------
    def _linear(self, n, x, W, bias, out, *, x_mode=X_PLAIN, ln=None, epi=EPI_STORE, res=None, n_partials=0, kv=None, K_=None):
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
        call("oasr_dec_linear", ctypes.byref(a), stream())

    def _attention(self, n, k, v, seq_stride, row_stride, part, splits, n_keys=None):
        a = DecAttnArgs()
        a.q, a.ldq = ptr(self.q), self.q.stride(0)
        a.k, a.v, a.kv_seq_stride, a.kv_row_stride = ptr(k), ptr(v), seq_stride, row_stride
        a.scores, a.scores_ld = ptr(self.scores), self.scores.stride(1)
        a.out_partial, a.ld_out = ptr(part), self.d
        a.pos_ptr = None if n_keys is not None else ptr(self.pos)
        a.n_keys = n_keys or 0
        a.n_seq, a.n_head, a.n_splits, a.scale, a.dtype = n, self.H, splits, 64 ** -0.25, self.dt
        call("oasr_dec_attention", ctypes.byref(a), stream())
        if splits == 1:
            _lib.LAUNCH_COUNT -= 1      # an unsplit key range runs as ONE fused kernel (scores + softmax + P V), not two

    def cross_splits(self, n: int) -> int:
        """Key-range splits of the cross-attention so that n x H x splits CTAs cover the SMs about twice."""
        return max(1, min(self.max_splits, math.ceil(2 * _lib.lib().oasr_device_sm_count() / (n * self.H))))

    def _enqueue_step(self, n: int):
        """One decoder step for sequences [0, n): per layer 6 fused Linear launches, 1 self-attention launch and 1 (unsplit key
        range) or 2 (split) cross-attention launches; plus the embedding, the logits head and the 2 sampling launches."""
        w, d = self._w, self.d
        c0 = _lib.LAUNCH_COUNT
        call("oasr_dec_embed", ptr(self.tokens), self.tokens.stride(0), ptr(self.pos), ptr(w["emb"]), ptr(w["pos"]), ptr(self.x),
             n, d, self.V, self.dt, stream())
        sc = self.cross_splits(n)
        seq_self, seq_cross = self.n_ctx * d, self.n_audio_ctx * 2 * d
        x, q, h = self.x[:n], self.q[:n], self.h[:n]
        # the attention kernels lay their fp32 partial outputs out as (splits, n, d): views with exactly that geometry
        part_self = self.part_self.view(-1)[: n * d].view(1, n, d)
        part_cross = self.part_cross.view(-1)[: sc * n * d].view(sc, n, d)
        for l, lw in enumerate(w["layers"]):
            self._linear(n, x, lw["wqkv"], lw["bqkv"], q, x_mode=X_LAYERNORM, ln=lw["ln1"], epi=EPI_QKV_SCATTER,
                         kv=(self.self_k[l], self.self_v[l]))
            self._attention(n, self.self_k[l], self.self_v[l], seq_self, d, part_self, 1)
            self._linear(n, part_self, lw["wo"], lw["bo"], x, x_mode=X_PARTIAL_SUM, n_partials=1, epi=EPI_RESIDUAL, res=x)
            self._linear(n, x, lw["wcq"], lw["bcq"], q, x_mode=X_LAYERNORM, ln=lw["lnc"])
            ckv = self.cross_kv[l]
            self._attention(n, ckv, ckv[:, d:], seq_cross, 2 * d, part_cross, sc, n_keys=self.n_audio_ctx)
            self._linear(n, part_cross, lw["wco"], lw["bco"], x, x_mode=X_PARTIAL_SUM, n_partials=sc, epi=EPI_RESIDUAL, res=x)
            self._linear(n, x, lw["w1"], lw["b1"], h, x_mode=X_LAYERNORM, ln=lw["ln2"], epi=EPI_GELU)
            self._linear(n, h, lw["w2"], lw["b2"], x, epi=EPI_RESIDUAL, res=x)
        self._linear(n, x, w["emb_t"], None, self.logits, x_mode=X_LAYERNORM, ln=w["ln"], epi=EPI_LOGITS_F32)
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

    def _graph(self, n: int) -> torch.cuda.CUDAGraph:
        key = (n, self._sample_cfg)
        g = self._graphs.get(key)
        if g is None:
            # one eager run first (kernel modules are loaded lazily on first launch, which must not happen under capture),
            # with the device-side decode state saved and restored around it; the capture itself does not execute
            live = (self.pos, self.tokens, self.sum_logprobs, self.no_speech, self.n_unfinished, self.done, self.sample_counters)
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
        is filled on the first call and only read afterwards) with the wgmma GEMM."""
        from ._core import _as_bf16_2d, linear_fwd

        self.refresh_weights()
        n = audio_features.shape[0]
        if n > self.max_batch:
            raise ValueError(f"DecodeEngine: {n} sequences > max_batch {self.max_batch}")
        if tuple(audio_features.shape[1:]) != (self.n_audio_ctx, self.d):
            raise ValueError(f"audio_features must be (N, {self.n_audio_ctx}, {self.d})")
        xa = _as_bf16_2d(audio_features)
        rows = n * self.n_audio_ctx
        for l, blk in enumerate(self.model.decoder.blocks):
            wkv, bkv = blk.cross_attn.fused_kv()
            if self.dtype == torch.bfloat16:
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

    def replay(self, n: int):
        """One decoder step for sequences [0, n): feeds the token at the device-side position, leaves the fp32 logits of that
        position in `self.logits[:n]`, appends the sampled token when past the teacher-forced prefix, advances the position."""
        self._graph(n).replay()

    @torch.no_grad()
    def greedy(self, audio_features: Tensor, initial_tokens: Sequence[int], sample_len: int, suppress: Sequence[int] = (),
               suppress_blank: bool = True, sot_index: int = 0, blank: int = 220, eot: int = 50256, no_speech: int = 50361,
               check_every: int = 8) -> Tuple[Tensor, Tensor, Tensor, int]:
        """Returns (tokens (N, len) int64 on the host incl. the initial tokens, sum_logprobs (N,), no_speech_probs (N,),
        number of graph replays).  Semantics of DecodingTask._main_loop for temperature 0 without timestamp rules."""
        n = self.prepare(audio_features)
        init = list(initial_tokens)
        n_init = len(init)
        if not 1 <= n_init < self.n_ctx:
            raise ValueError("initial_tokens: need 1 .. n_text_ctx-1 tokens")
        self.reset(n, torch.tensor([init], dtype=torch.int32).repeat(n, 1), None, suppress, suppress_blank, sot_index, blank, eot, no_speech)
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

    # ---- roofline bookkeeping --------------------------------------------------------------------------------------
    def step_bytes(self, n: int, t: int) -> int:
        """Algorithmic HBM bytes of one step at self-attention length t (SURVEY.md 8(d)): every decoder weight once (shared by
        the batch), per sequence the cross K/V of every layer, the self K/V read so far, and the fp32 logits row."""
        e = 2
        d, L = self.d, self.L
        weights = L * (3 * d * d + d * d + d * d + d * d + 8 * d * d) * e + self.V * d * e
        cross = L * 2 * self.n_audio_ctx * d * e
        self_kv = L * 2 * t * d * e
        return weights + n * (cross + self_kv + self.V * 4)
