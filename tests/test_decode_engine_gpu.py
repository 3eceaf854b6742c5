"""The device-resident greedy decoder (olmoasr_b200/decode_engine.py, csrc/decode.cu) against the reference's own PyTorch
path: oracle/model.py's restatement of olmoasr/inf_model.py (pinned bit-exact to the unmodified reference in
tests/test_oracle_pin.py) executed by stock torch ON THE GPU in the same activation dtype -- i.e. what `model.decode`
computes when the reference runs on this device (fp16 = upstream default, and bf16).

Both sides round at the same points; what differs is the order of fp32 accumulation inside matmuls and reductions, which
flips an occasional last-place rounding.  Hence: per-position logits within a few units of the dtype's resolution
(relative L2), argmax ids identical wherever the reference's own top-1 / top-2 margin exceeds that noise, and greedy
token ids identical on a margin-sharpened model (SURVEY.md 8(d)).  BASELINE.json config 5 names `small`: it is tested at
full size next to tiny.
"""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

EOT, SOT, NO_TIMESTAMPS = 50256, 50257, 50362
TOL = {torch.float16: 4e-3, torch.bfloat16: 3e-2}      # relative L2 of a logits row after 4 / 12 decoder layers
SURE = {torch.float16: 8e-3, torch.bfloat16: 4e-2}     # top-1 / top-2 margin (relative to max |logit|) that rounding cannot flip
SHARPEN = {"tiny": (3.0, 0.5), "small": (6.0, 0.1)}    # (embedding scale, positional scale): reference margins >= 0.1


def _build(variant, emb_scale=1.0, pos_scale=0.05, n_clips=3):
    import olmoasr_b200 as ob
    from olmoasr_b200 import synthetic
    from olmoasr_b200.inf_model import OLMoASR
    from oracle import logmel
    from oracle import model as OM

    dims = OM.variant_dims(variant)
    sd = OM.init_state_dict(dims, 0, train=False)
    g = torch.Generator().manual_seed(7)
    sd["decoder.positional_embedding"] = torch.randn(448, dims.n_text_state, generator=g) * pos_scale
    sd["decoder.token_embedding.weight"] = sd["decoder.token_embedding.weight"] * emb_scale
    m = OLMoASR(ob.VARIANT_TO_DIMS[variant])
    m.load_state_dict(sd)
    m = m.cuda()
    mel = torch.from_numpy(logmel.log_mel_spectrogram(synthetic.waveforms(n_clips).numpy())).cuda()
    with torch.no_grad():
        xa = m.encoder(mel)                                  # (n, 1500, d) bf16: both sides decode over the same features
    sd_gpu = {k: v.cuda() for k, v in sd.items()}
    return m, sd_gpu, dims, OM, xa


def _ref_full_prefix_logits(OM, sd, dims, tokens, xa, dtype):
    """inf_model.TextDecoder.forward on the whole prefix (causal mask, manual attention) in `dtype`, stock torch on the GPU."""
    with torch.no_grad():
        return OM.decoder_forward(sd, dims, tokens, xa.to(dtype), None, train_model=False)


@pytest.mark.parametrize("variant", ["tiny", "small"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_step_logits_match_the_reference_path(variant, dtype):
    """Teacher-forced 20-token prefixes (different per sequence): after every replay the engine's logits for that position
    equal the reference's full-prefix forward (the kv-cache == re-forward invariant of SURVEY.md section 4 included)."""
    m, sd, dims, OM, xa = _build(variant)
    n, P = xa.shape[0], 20
    g = torch.Generator().manual_seed(3)
    toks = torch.randint(0, 50256, (n, P), generator=g)
    toks[:, 0] = SOT
    ref = _ref_full_prefix_logits(OM, sd, dims, toks.cuda(), xa, dtype)            # (n, P, V) fp32
    eng = m.decode_engine(dtype)
    eng.prepare(xa)
    eng.reset(n, toks, sample_begin=P + 5)                                            # everything teacher-forced
    worst, agree, decided = 0.0, 0, 0
    for t in range(P):
        eng.replay(n)
        got = eng.logits[:n].clone()
        want = ref[:, t]
        rel = float((got - want).norm() / want.norm())
        worst = max(worst, rel)
        top2 = want.topk(2, dim=-1).values
        sure = (top2[:, 0] - top2[:, 1]) > SURE[dtype] * want.abs().max()          # a margin well above the dtype's resolution
        decided += int(sure.sum())
        agree += int((got.argmax(-1) == want.argmax(-1))[sure].sum())
    print(f"{variant} {dtype}: worst per-position rel-L2 {worst:.2e}; argmax agreement {agree}/{decided} decided positions")
    assert worst <= TOL[dtype]
    assert agree == decided and (decided > 0 or dtype == torch.bfloat16)
    assert int(eng.pos.item()) == P
    # the static cache holds exactly the K / V rows the reference's hooks would have concatenated
    with torch.no_grad():
        cache = {}
        OM.decoder_forward(sd, dims, toks.cuda(), xa.to(dtype), None, train_model=False, cache=cache)
    k_ref = cache["decoder.blocks.0.attn.key"]
    k_got = eng.self_k[0, :n, :P]
    assert float((k_got.float() - k_ref.float()).norm() / k_ref.float().norm()) <= TOL[dtype]
    ck_ref = cache[f"decoder.blocks.{dims.n_text_layer - 1}.cross_attn.value"]
    d = dims.n_text_state
    ck_got = eng.cross_kv[dims.n_text_layer - 1][: n * 1500].view(n, 1500, 2 * d)[:, :, d:]
    assert float((ck_got.float() - ck_ref.float()).norm() / ck_ref.float().norm()) <= 2e-2


def _ref_greedy(OM, sd, dims, xa, dtype, n_steps, suppress, suppress_blank=True):
    """whisper/decoding.py greedy loop (DecodingTask._main_loop for temperature 0, without_timestamps) over the reference's
    kv-cache decoder, stock torch on the GPU."""
    n = xa.shape[0]
    dev = xa.device
    tokens = torch.tensor([[SOT, NO_TIMESTAMPS]], device=dev).repeat(n, 1)
    cache, margins, sum_lp, nsp = {}, [], torch.zeros(n, device=dev), None
    sup = torch.tensor(sorted(suppress), device=dev)
    with torch.no_grad():
        for i in range(n_steps):
            inp = tokens if tokens.shape[1] <= 2 else tokens[:, -1:]
            logits = OM.decoder_forward(sd, dims, inp, xa.to(dtype), None, train_model=False, cache=cache)
            if i == 0:
                nsp = logits[:, 0].float().softmax(-1)[:, 50361]
            logits = logits[:, -1]
            if suppress_blank and tokens.shape[1] == 2:
                logits[:, [220, EOT]] = -math.inf
            logits[:, sup] = -math.inf
            top2 = logits.topk(2, dim=-1).values
            margins.append(float((top2[:, 0] - top2[:, 1]).min()))
            nxt = logits.argmax(-1)
            lp = F.log_softmax(logits.float(), dim=-1)[torch.arange(n, device=dev), nxt]
            sum_lp += lp * (tokens[:, -1] != EOT)
            nxt[tokens[:, -1] == EOT] = EOT
            tokens = torch.cat([tokens, nxt[:, None]], dim=-1)
            if bool((tokens[:, -1] == EOT).all()):
                break
    return tokens, margins, sum_lp, nsp


@pytest.mark.parametrize("variant", ["tiny", "small"])
@pytest.mark.parametrize("fp16", [True, False])
def test_greedy_token_ids_match_the_reference_loop(variant, fp16):
    """north_star: "bit-exact argmax token ids for greedy decode" -- through the public `decode()` API (which routes greedy,
    timestamp-free decoding to the engine), on a margin-sharpened model, in fp16 (upstream default) and bf16."""
    from olmoasr_b200.decoding import DecodingOptions, DecodingTask, decode

    dtype = torch.float16 if fp16 else torch.bfloat16
    m, sd, dims, OM, xa = _build(variant, emb_scale=SHARPEN[variant][0], pos_scale=SHARPEN[variant][1])
    n_steps = 24
    opts = DecodingOptions(language="en", without_timestamps=True, sample_len=n_steps, fp16=fp16)
    task = DecodingTask(m, opts)
    want, margins, sum_lp, nsp = _ref_greedy(OM, sd, dims, xa, dtype, n_steps, task.suppress)
    want32, _, sum_lp32, _ = _ref_greedy(OM, sd, dims, xa, torch.float32, n_steps, task.suppress)
    res = decode(m, xa, opts)                                        # encoded features are accepted like upstream
    got = [r.tokens for r in res]
    # token ids are compared up to the first step at which the REFERENCE's own top-1 / top-2 margin drops into rounding
    # noise (from there on two correct fp16 implementations may legitimately pick different tokens and diverge)
    noise = 0.05
    n_cmp = next((i for i, mg in enumerate(margins) if mg < noise), len(margins))
    print(f"{variant} fp16={fp16}: reference margins min {min(margins):.3f}, decided steps {n_cmp}/{len(margins)}; tokens {got[0][:8]}")
    assert n_cmp >= 4, "sharpening failed: the comparison would be decided by rounding noise from the start"
    for k in range(xa.shape[0]):
        seq = want[k, 2:].tolist()
        seq = seq[: seq.index(EOT)] if EOT in seq else seq
        assert got[k][:n_cmp] == seq[:n_cmp], k
        if n_cmp == len(margins):
            assert got[k] == seq
            # the reference's log-probs come from logits rounded to the activation dtype: besides the fixed tolerance, a
            # result may sit as far from them as the reference's own rounding moved them off its fp32 run (same tokens)
            lp_ref = float(sum_lp[k]) / (len(seq) + 1)
            rounding = abs(lp_ref - float(sum_lp32[k]) / (len(seq) + 1)) if torch.equal(want32[k], want[k]) else 0.0
            assert abs(res[k].avg_logprob - lp_ref) <= 2e-2 * abs(lp_ref) + 1e-3 + 2.0 * rounding
        assert abs(res[k].no_speech_prob - float(nsp[k])) <= 0.05 * float(nsp[k]) + 1e-6
    eng = m.decode_engine(dtype)
    cross = 1 if eng.cross_splits(xa.shape[0]) == 1 else 2
    assert eng.launches_per_step == (6 + 1 + cross) * dims.n_text_layer + 1 + 1 + 2
    one = decode(m, xa[0], DecodingOptions(without_timestamps=True, sample_len=4, fp16=fp16))
    assert one.tokens[:min(4, n_cmp)] == got[0][:min(4, n_cmp)]


def test_batch_size_independence_and_split_paths():
    """1, 5, 20 and 40 concurrent sequences exercise every M-tile variant of the skinny GEMM (16 / 32 / 64 rows) and the
    cross-attention key-range splits (8 -> 1): the same clip must decode to the same ids in every batch."""
    m, sd, dims, OM, xa = _build("tiny", emb_scale=3.0, pos_scale=0.5, n_clips=2)
    eng = m.decode_engine(torch.float16)
    ref = None
    for n in (1, 5, 20, 40):
        feats = xa[:1].repeat(n, 1, 1)
        if n > 1:
            feats[1::2] = xa[1]                                   # odd rows: the other clip
        toks, lps, nsp, replays = eng.greedy(feats, [SOT, NO_TIMESTAMPS], 12, suppress=(50358, 50357, 50257, 50360, 50359, 50361))
        assert toks.shape == (n, 14) and replays == 13
        if ref is None:
            ref = toks[0]
        assert torch.equal(toks[0], ref), n
        assert all(torch.equal(toks[i], toks[i % 2]) for i in range(n)), n
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        assert eng.cross_splits(n) == max(1, min(eng.max_splits, math.ceil(2 * sms / (n * dims.n_text_head))))


def test_sampling_kernel_bookkeeping():
    """dec_sample against a torch statement of SuppressBlank / SuppressTokens / GreedyDecoder.update, including rows that
    already ended (previous token eot: keep emitting eot, log-prob sum frozen), ties (lowest index) and the stop flag."""
    from olmoasr_b200._lib import DecSampleArgs, call, ptr, stream
    import ctypes

    m, sd, dims, OM, xa = _build("tiny", n_clips=1)
    eng = m.decode_engine(torch.float16)
    eng.refresh_weights()
    n, V = 4, eng.V
    g = torch.Generator().manual_seed(11)
    logits = torch.randn(n, V, generator=g).cuda() * 3
    logits[0, 220] = 50.0                 # blank would win at the first sampled position
    logits[1, 7] = 40.0                   # a suppressed id
    logits[2, 123] = logits[2, 4567] = 60.0   # tie -> lowest index
    toks = torch.tensor([[SOT, NO_TIMESTAMPS]] * n, dtype=torch.int32)
    toks[3, 1] = EOT                      # row 3 already ended
    eng.reset(n, toks, suppress=(7, 9), suppress_blank=True)
    eng.pos.fill_(1)                      # the position of the last given token
    eng.logits[:n] = logits
    s = DecSampleArgs()
    s.logits, s.ld_logits = ptr(eng.logits), eng.logits.stride(0)
    s.tokens, s.ld_tokens, s.pos_ptr = ptr(eng.tokens), eng.tokens.stride(0), ptr(eng.pos)
    s.suppress, s.sum_logprobs, s.no_speech_prob = ptr(eng.suppress), ptr(eng.sum_logprobs), ptr(eng.no_speech)
    s.n_unfinished, s.done_flag = ptr(eng.n_unfinished), ptr(eng.done)
    s.scratch, s.counters, s.n_slices = ptr(eng.sample_scratch), ptr(eng.sample_counters), eng.sample_slices
    s.n_seq, s.n_vocab, s.sample_begin, s.sot_index, s.suppress_blank, s.blank, s.eot, s.no_speech = n, V, 2, 0, 1, 220, EOT, 50361
    call("oasr_dec_sample", ctypes.byref(s), stream())
    ref = logits.clone()
    ref[:, [220, EOT]] = -math.inf
    ref[:, [7, 9]] = -math.inf
    nxt = ref.argmax(-1)
    lp = F.log_softmax(ref, -1)[torch.arange(n), nxt]
    out = eng.tokens[:n, 2].cpu()
    assert out[0] == nxt[0] != 220 and out[1] == nxt[1] != 7 and out[2] == 123 and out[3] == EOT
    assert torch.allclose(eng.sum_logprobs[:3].cpu(), lp[:3].cpu(), rtol=1e-4, atol=1e-4) and float(eng.sum_logprobs[3]) == 0.0
    assert int(eng.pos.item()) == 2 and int(eng.done.item()) == 0
    # second step: every row now emits eot -> the stop flag rises
    eng.logits[:n] = -5.0
    eng.logits[:n, EOT] = 30.0
    call("oasr_dec_sample", ctypes.byref(s), stream())
    assert eng.tokens[:n, 3].cpu().tolist() == [EOT] * n and int(eng.done.item()) == 1
    assert int(eng.sample_counters.abs().sum()) == 0            # the slice counters re-arm themselves
    # one slice per row gives the same choices as sixteen
    eng.pos.fill_(1); eng.sum_logprobs.zero_()
    eng.logits[:n] = logits
    s.n_slices = 1
    call("oasr_dec_sample", ctypes.byref(s), stream())
    assert torch.equal(eng.tokens[:n, 2].cpu(), out) and torch.allclose(eng.sum_logprobs[:3].cpu(), lp[:3].cpu(), rtol=1e-4, atol=1e-4)
