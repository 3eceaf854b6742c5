"""transcribe_batch() on the device: the batched alignment kernels against the single-window entry points (bits) and
the oracle's DTW, transcribe_batch() against transcribe() per recording at temperature 0, reproducibility and batch-size
independence of the sampled fallback ladder, and the call structure of a round (one encoder call, one engine call per
temperature reached, no window in the hook loop)."""
import numpy as np
import pytest
import torch

from oracle import timing as OT
from tests.test_decode_engine_gpu import _build
from tests.test_timing_gpu import SpaceTokenizer

pytestmark = pytest.mark.gpu

SECONDS = (0.5, 150.0, 37.3, 71.0, 12.0)


def _bits(x):
    return x.contiguous().view(torch.int32)


def test_batched_kernels_equal_the_single_window_entry_points():
    from olmoasr_b200 import kernels as K

    g = torch.Generator(device="cuda").manual_seed(0)
    n_heads = 6
    shapes = [(3, 1), (448, 1500), (37, 3), (227, 750), (5, 2), (448, 1), (3, 1500), (64, 17)]
    windows = []
    for n_tok, n_frames in shapes:
        q = torch.randn(n_tok, n_heads * 64, device="cuda", generator=g).half()
        k = torch.randn(1500, n_heads * 64, device="cuda", generator=g).half()
        windows.append(([(q[:, h * 64:(h + 1) * 64], k[:, h * 64:(h + 1) * 64]) for h in range(n_heads)], n_frames))
    batched = K.align_cost_batched(windows)
    for (heads, n_frames), got in zip(windows, batched):
        want = K.align_cost(heads, n_frames)
        assert got.shape == want.shape and torch.equal(_bits(got), _bits(want)), (heads[0][0].shape[0], n_frames)

    rng = np.random.default_rng(1)
    mats = [rng.standard_normal(s).astype(np.float32) for s in [(1, 1), (2, 1500), (47, 750), (446, 1500), (5, 3), (1, 7), (9, 1)]]
    mats.append((np.round(rng.standard_normal((60, 300)) * 2) / 2).astype(np.float32))     # many ties
    xs = [torch.from_numpy(m).cuda() for m in mats] + [c for c in batched if not torch.isnan(c).any()]
    paths, lengths = K.dtw_batched(xs)
    for w, x in enumerate(xs):
        path, length = K.dtw(x)
        n = int(length)
        assert int(lengths[w]) == n
        assert torch.equal(paths[w, :, :n], path[:, :n])
        wi, wj = OT.dtw(x.cpu().numpy())
        assert np.array_equal(path[0, :n].cpu().numpy(), wi) and np.array_equal(path[1, :n].cpu().numpy(), wj)


@pytest.fixture(scope="module")
def tiny():
    from olmoasr_b200 import synthetic

    m, _, _, _, _ = _build("tiny", 3.0, 0.5, n_clips=1)
    audios = [synthetic.waveforms(1, rank=r, n_samples=int(s * 16000))[0] for r, s in enumerate(SECONDS)]
    return m, audios


def test_encoder_features_do_not_depend_on_the_batch(tiny):
    from olmoasr_b200 import _core
    from olmoasr_b200.audio import N_FRAMES, log_mel_spectrogram, pad_or_trim

    m, audios = tiny
    mels = torch.stack([pad_or_trim(log_mel_spectrogram(a.cuda()), N_FRAMES) for a in audios])
    with torch.no_grad(), _core.bf16_compute():
        together = m.encoder(mels)
        for w in range(mels.shape[0]):
            assert torch.equal(m.encoder(mels[w:w + 1])[0], together[w]), w


def _compare(got, want):
    assert got["text"] == want["text"] and got["language"] == want["language"]
    assert len(got["segments"]) == len(want["segments"])
    for a, b in zip(got["segments"], want["segments"]):
        for key in ("id", "seek", "start", "end", "tokens", "text", "temperature", "compression_ratio"):
            assert a[key] == b[key], key
        for key in ("avg_logprob", "no_speech_prob"):
            assert abs(a[key] - b[key]) <= 1e-4, key
        assert ("words" in a) == ("words" in b)
        for wa, wb in zip(a.get("words", []), b.get("words", [])):
            assert wa == wb
        assert len(a.get("words", [])) == len(b.get("words", []))


@pytest.mark.parametrize("kw", [dict(), dict(without_timestamps=False, beam_size=5, best_of=5), dict(word_timestamps=True),
                                dict(word_timestamps=True, hallucination_silence_threshold=2.0)],
                         ids=["greedy", "eval", "words", "words-hallucination"])
def test_temperature_zero_equals_transcribe(tiny, kw):
    from olmoasr_b200.transcribe import transcribe, transcribe_batch

    m, audios = tiny
    tok = SpaceTokenizer()
    want = [transcribe(m, a, temperature=0.0, sample_len=96, tokenizer=tok, **kw) for a in audios]
    got = transcribe_batch(m, audios, temperature=0.0, sample_len=96, tokenizer=tok, **kw)
    for g, w in zip(got, want):
        _compare(g, w)
    print(f"{kw}: {sum(len(r['segments']) for r in got)} segments, "
          f"{sum(len(s.get('words', [])) for r in got for s in r['segments'])} words")


def test_sampled_ladder_is_reproducible_and_batch_independent(tiny, monkeypatch):
    import olmoasr_b200.transcribe as T

    m, audios = tiny
    temps = []
    real = T.decode_windows

    def spy(model, feats, options, *a, **k):
        temps.append((options.temperature, feats.shape[0]))
        return real(model, feats, options, *a, **k)

    monkeypatch.setattr(T, "decode_windows", spy)

    def run(batch_size):
        torch.manual_seed(21)
        out = T.transcribe_batch(m, audios, batch_size=batch_size, sample_len=96, best_of=5)
        return [[(s["seek"], s["start"], s["end"], s["tokens"], s["temperature"]) for s in r["segments"]] for r in out]

    first = run(None)
    fell_back = sum(n for t, n in temps if t > 0)
    assert run(None) == first
    assert run(1) == first
    print(f"windows decoded at a fallback temperature: {fell_back}; decode calls {len(temps)}")


def test_round_call_structure(tiny, monkeypatch):
    import olmoasr_b200.timing as TM
    import olmoasr_b200.transcribe as T

    m, audios = tiny
    encoder_calls, rounds, engine_calls, per_round_temps = [], [], [], []
    h = m.encoder.register_forward_hook(lambda *_: encoder_calls.append(1))
    real_round = T._decode_round

    def round_spy(model, features, recordings, *a, **k):
        rounds.append(len(recordings))
        before = len(engine_calls)
        out = real_round(model, features, recordings, *a, **k)
        per_round_temps.append((len(set(r.temperature for r in out)), max(T.DEFAULT_TEMPERATURES.index(r.temperature) for r in out) + 1,
                                len(engine_calls) - before))
        return out

    monkeypatch.setattr(T, "_decode_round", round_spy)
    eng = m.decode_engine(torch.float16)
    for name in ("greedy", "sample", "beam_search"):
        real = getattr(eng, name)
        monkeypatch.setattr(eng, name, lambda *a, _real=real, _name=name, **k: (engine_calls.append(_name), _real(*a, **k))[1])
    real_hooks, inside = m.install_kv_cache_hooks, []

    def guarded(*a, **k):
        if not inside:
            raise AssertionError("a window took the hook loop")
        return real_hooks(*a, **k)

    real_forward = TM.alignment_forward

    def forward_spy(*a, **k):
        inside.append(1)
        try:
            return real_forward(*a, **k)
        finally:
            inside.pop()

    monkeypatch.setattr(m, "install_kv_cache_hooks", guarded)
    monkeypatch.setattr(TM, "alignment_forward", forward_spy)
    try:
        torch.manual_seed(3)
        T.transcribe_batch(m, audios, without_timestamps=False, beam_size=5, best_of=5, sample_len=96,
                           word_timestamps=True, tokenizer=SpaceTokenizer())
    finally:
        h.remove()
    assert len(encoder_calls) == len(rounds) >= 1, "one encoder call per round"
    for _, reached, calls in per_round_temps:
        assert calls == reached, "one engine call per temperature a round reaches"
    print(f"rounds {len(rounds)} (windows {rounds}), engine calls {len(engine_calls)}, per round {per_round_temps}")
