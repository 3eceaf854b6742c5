"""Word-level timestamps on the device (csrc/timing.cu, olmoasr_b200/timing.py): `oasr_dtw` against the oracle's float32
DTW (exact paths), `oasr_align_cost` against an fp32 torch restatement of find_alignment's steps 2-7 on the same 16-bit
q / k, `find_alignment` end to end against the oracle run by stock torch on the GPU in fp16, and
`transcribe(word_timestamps=True)` on long synthetic audio."""
import numpy as np
import pytest
import torch

from oracle import timing as OT
from tests.test_decode_engine_gpu import SHARPEN, _build

pytestmark = pytest.mark.gpu

EOT, TB = 50256, 50363


def _dev_dtw(x):
    from olmoasr_b200 import kernels as K

    path, length = K.dtw(torch.from_numpy(x).cuda())
    n = int(length)
    p = path[:, :n].cpu().numpy().astype(np.int64)
    return p[0], p[1]


@pytest.mark.parametrize("shape", [(1, 1), (2, 1500), (47, 750), (225, 1500), (446, 1500)])
def test_dtw_path_equals_the_oracle(shape):
    rng = np.random.default_rng(shape[0] * 7919 + shape[1])
    cases = {"normal": rng.standard_normal(shape).astype(np.float32),
             "ties": (np.round(rng.standard_normal(shape) * 2) / 2).astype(np.float32),   # many equal partial costs
             "flat": np.zeros(shape, dtype=np.float32)}
    r, c = shape
    planted = rng.uniform(0.0, 1.0, shape).astype(np.float32)
    cols = np.sort(rng.choice(c, min(r, c), replace=False))
    planted[np.arange(min(r, c)), cols] = -5.0
    cases["planted"] = planted
    for name, x in cases.items():
        ti, tj = _dev_dtw(x)
        wi, wj = OT.dtw(x)
        assert np.array_equal(ti, wi) and np.array_equal(tj, wj), (shape, name)


def _cost_ref(q, k, heads, n_frames, width=7):
    """fp32 torch restatement of steps 2-7 on the 16-bit q (n_tok, L, H*64) / k (1500, L, H*64)."""
    qks = {}
    for l, h in heads:
        qh = q[:, l, h * 64:(h + 1) * 64].float()
        kh = k[:, l, h * 64:(h + 1) * 64].float()
        qks.setdefault(l, {})[h] = (qh @ kh.T) * 0.125
    return -OT.alignment_matrix(qks, heads, 2 * n_frames, width)


def _align_case(n_tok, n_frames, n_heads, dtype=torch.float16, seed=0):
    from olmoasr_b200 import kernels as K

    g = torch.Generator(device="cuda").manual_seed(seed)
    L, H = (4, 2) if n_heads <= 8 else (24, 16)
    q = torch.randn(n_tok, L, H * 64, device="cuda", generator=g).to(dtype)
    k = torch.randn(1500, L, H * 64, device="cuda", generator=g).to(dtype)
    all_heads = [(l, h) for l in range(L) for h in range(H)]
    pick = sorted(torch.randperm(len(all_heads), generator=torch.Generator().manual_seed(seed))[:n_heads].tolist())
    heads = [all_heads[i] for i in pick]
    pairs = [(q[:, l, h * 64:(h + 1) * 64], k[:, l, h * 64:(h + 1) * 64]) for l, h in heads]
    return K.align_cost(pairs, n_frames), pairs, _cost_ref(q, k, heads, n_frames)


ALIGN_CASES = [(t, f, 7) for t in (3, 37, 227, 448) for f in (1, 3, 4, 750, 1500)] + \
              [(37, 750, 1), (227, 1500, 1), (448, 4, 192), (227, 1500, 192), (448, 1500, 192)]


@pytest.mark.parametrize("n_tok,n_frames,n_heads", ALIGN_CASES)
def test_align_cost_matches_fp32_torch(n_tok, n_frames, n_heads):
    from olmoasr_b200 import kernels as K

    got, pairs, want = _align_case(n_tok, n_frames, n_heads)
    assert got.shape == want.shape == (n_tok - 2, n_frames)
    if n_frames == 1:   # one frame: softmax is 1 everywhere, the std is 0 and both sides give NaN
        assert torch.isnan(got).all() and torch.isnan(want).all()
        return
    err = (got - want).abs().max().item()
    print(f"align_cost n_tok={n_tok} n_frames={n_frames} heads={n_heads}: max-abs {err:.3e}")
    assert err <= 1e-4
    again = K.align_cost(pairs, n_frames)
    assert torch.equal(got, again), "two runs differ"


def test_align_cost_bf16_operands():
    got, _, want = _align_case(37, 750, 7, dtype=torch.bfloat16, seed=3)
    assert (got - want).abs().max().item() <= 1e-4


class SpaceTokenizer:
    """Every id is one word with a leading space, so a segment's words concatenate to its text exactly."""

    def decode(self, ids):
        return "".join(f" w{i % 97}" for i in ids)


@pytest.mark.parametrize("variant", ["tiny", "small"])
def test_find_alignment_end_to_end(variant):
    from olmoasr_b200 import kernels as K
    from olmoasr_b200 import timing as T

    m, sd, dims, OM, xa = _build(variant, *SHARPEN[variant], n_clips=1)
    g = torch.Generator().manual_seed(5)
    text = torch.randint(0, EOT, (40,), generator=g).tolist()
    for num_frames in (3000, 1234):
        cost, probs = T.alignment_cost(m, text, xa[0], num_frames)
        tokens = torch.tensor([[50257, 50362, *text, EOT]], device="cuda")
        with torch.no_grad():
            _, qks = OT.decoder_forward_qk(sd, dims, tokens, xa.half())   # activations in fp16, LayerNorm in fp32
        heads = m.alignment_heads.indices().T.tolist()
        want = -OT.alignment_matrix([q[0] for q in qks], heads, num_frames)
        rel = ((cost - want).norm() / want.norm()).item()
        print(f"{variant} num_frames={num_frames}: cost relative L2 to the fp16 torch oracle {rel:.3e}")
        assert rel <= 2e-2
        path, length = K.dtw(cost)
        n = int(length)
        wi, wj = OT.dtw(cost.cpu().numpy())
        assert np.array_equal(path[0, :n].cpu().numpy(), wi) and np.array_equal(path[1, :n].cpu().numpy(), wj)
        p = probs.cpu()
        assert ((p > 0) & (p <= 1)).all()

        words = T.find_alignment(m, SpaceTokenizer(), text, xa[0], num_frames)
        assert [t for w in words for t in w.tokens] == text
        prev = 0.0
        for w in words:
            assert prev <= w.start <= w.end <= num_frames / 100 + 1e-9 and 0 < w.probability <= 1
            prev = w.start


def test_transcribe_word_timestamps(monkeypatch):
    import olmoasr_b200.timing as TM
    import olmoasr_b200.transcribe as T
    from olmoasr_b200 import synthetic

    m, sd, dims, OM, xa = _build("tiny", emb_scale=3.0, pos_scale=0.5, n_clips=1)
    real_hooks, inside = m.install_kv_cache_hooks, []

    def guarded(*a, **k):        # the alignment forward may install hooks, a decode window may not
        if not inside:
            raise AssertionError("a window took the hook loop")
        return real_hooks(*a, **k)

    real_cost = TM.alignment_cost

    def cost_spy(*a, **k):
        inside.append(1)
        try:
            return real_cost(*a, **k)
        finally:
            inside.pop()

    monkeypatch.setattr(m, "install_kv_cache_hooks", guarded)
    monkeypatch.setattr(TM, "alignment_cost", cost_spy)
    seconds = 75.0
    audio = synthetic.waveforms(1, n_samples=int(seconds * 16000))[0]
    calls = []
    real_decode = T.decode

    def spy(model, segment, options, **kw):
        calls.append(options)
        assert len(calls) < 400, "the seek stopped advancing"
        return real_decode(model, segment, options, **kw)

    monkeypatch.setattr(T, "decode", spy)
    tok = SpaceTokenizer()
    for kw in (dict(), dict(hallucination_silence_threshold=2.0), dict(without_timestamps=False, beam_size=5, best_of=5)):
        calls.clear()
        torch.manual_seed(0)
        out = T.transcribe(m, audio, sample_len=96, tokenizer=tok, word_timestamps=True, **kw)
        assert calls
        prev_seek, n_words = 0, 0
        for seg in out["segments"]:
            assert "words" in seg and seg["seek"] >= prev_seek
            prev_seek = seg["seek"]
            text_ids = [t for t in seg["tokens"] if t < EOT]
            assert "".join(w["word"] for w in seg["words"]) == seg["text"] == tok.decode(text_ids)
            t0 = seg["seek"] / 100
            prev = t0 - 1.4     # the first word after a pause may start up to twice the 0.7 s duration cap early
            for w in seg["words"]:
                assert set(w) == {"word", "start", "end", "probability"}
                assert prev - 1e-6 <= w["start"] <= w["end"] <= t0 + 30.0 + 1e-6 and 0 < w["probability"] <= 1
                prev = w["start"]
            n_words += len(seg["words"])
        print(f"transcribe word_timestamps {kw}: {len(out['segments'])} segments, {n_words} words, {len(calls)} decode calls")
