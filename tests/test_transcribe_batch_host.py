"""transcribe_batch() against transcribe() on the CPU, with deterministic stand-ins for the log-mel, the encoder, decode and
the device alignment.  Every stand-in result is a function of (recording, seek, temperature), read back from mel values
that encode the recording and the frame, so the two drivers must agree field for field whatever windows share a round.
The recordings cover a clip shorter than a window, pure silence (the no-speech skip), windows that fall back one or more
times, single-timestamp endings, windows without timestamps, and mixed lengths."""
import numpy as np
import pytest
import torch

import olmoasr_b200.timing as TM
import olmoasr_b200.transcribe as T
from olmoasr_b200.decoding import DecodingResult

EOT, TB = 50256, 50363
SILENT = 2                                     # recording id whose windows are silence
SECONDS = [5.0, 95.0, 40.0, 61.3, 200.0, 31.0, 0.004, 130.7]


class _Tok:
    def decode(self, ids):
        return "".join(f" w{i % 97}" for i in ids)


class _Model:
    """dims, device and an encoder whose features carry the window's (recording, seek) from its first mel column."""

    def __init__(self):
        from types import SimpleNamespace

        self.dims = SimpleNamespace(n_mels=80, n_audio_ctx=1500, n_audio_state=8, n_text_ctx=448)
        self.device = torch.device("cpu")
        self.encoded = 0

    def encoder(self, mel):
        self.encoded += 1
        f = torch.zeros(mel.shape[0], 1500, 8)
        f[:, 0, 0], f[:, 0, 1] = mel[:, 0, 0], mel[:, 1, 0]
        return f


def _fake_log_mel(audio, n_mels=80, padding=0, device=None):
    n = (len(audio) + padding) // 160
    mel = torch.zeros(n_mels, n)
    mel[0] = float(audio[0]) if len(audio) else 0.0
    mel[1] = torch.arange(n, dtype=torch.float32)
    return mel


def _tokens(rng):
    """A timestamped window: segments of text between timestamp pairs; ends in a pair, a single timestamp or text."""
    out, t = [], int(rng.integers(0, 40))
    for _ in range(int(rng.integers(1, 4))):
        out += [TB + t] + [int(x) for x in rng.integers(0, 2000, int(rng.integers(1, 8)))]
        t = min(1500, t + int(rng.integers(5, 400)))
        out.append(TB + t)
        if rng.random() < 0.5 and t < 1500:
            out.append(TB + t)        # a closing and an opening timestamp
    ending = rng.integers(0, 3)
    if ending == 1:
        out += [int(x) for x in rng.integers(0, 2000, 3)] + [TB + min(1500, t + 10)]   # single timestamp ending
    elif ending == 2:
        out += [int(x) for x in rng.integers(0, 2000, 2)]                               # text after the last timestamp
    return out


def _result(features_row, options):
    rid, seek = int(features_row[0, 0]), int(features_row[0, 1])
    ti = T.DEFAULT_TEMPERATURES.index(options.temperature)
    rng = np.random.default_rng(rid * 1_000_003 + seek)
    n_fail = int(rng.integers(0, 4))           # this window falls back n_fail times
    if rid == SILENT:
        nsp, lp, toks = 0.9, -2.0, [TB, TB + 20]
    elif rng.random() < 0.15:
        nsp, lp, toks = 0.1, -0.2, [int(x) for x in rng.integers(0, 2000, 6)]         # no timestamps
    else:
        nsp, lp, toks = 0.1, (-1.5 if ti < n_fail else -0.3), _tokens(rng)
        if ti < n_fail:
            toks = toks + [int(rng.integers(0, 2000))]
    text = "".join(f" w{i % 97}" for i in toks if i < EOT).strip()
    return DecodingResult(audio_features=features_row, language="en", tokens=toks, text=text, avg_logprob=lp,
                          no_speech_prob=nsp, temperature=options.temperature)


def _fake_path(model, text_tokens, mel, num_frames, medfilt_width=7):
    rows, cols = len(text_tokens) + 1, num_frames // 2
    ti = np.minimum(np.arange(cols) * rows // cols, rows - 1)
    tj = np.arange(cols)
    if cols < rows:
        ti, tj = np.arange(rows), np.minimum(np.arange(rows) * cols // rows, cols - 1)
    probs = [0.3 + (t % 7) / 10 for t in text_tokens]
    return ti.astype(np.int64), tj.astype(np.int64), probs


@pytest.fixture
def stubs(monkeypatch):
    model = _Model()
    calls = []
    monkeypatch.setattr(T, "log_mel_spectrogram", _fake_log_mel)
    monkeypatch.setattr(T, "decode", lambda m, segment, options, tokenizer=None: _result(m.encoder(segment[None])[0], options))

    def windows(m, feats, options, tokenizer, sample_keys):
        calls.append((options.temperature, [(int(f[0, 0]), int(f[0, 1])) for f in feats], sample_keys))
        return [_result(f, options) for f in feats]

    monkeypatch.setattr(T, "decode_windows", windows)
    monkeypatch.setattr(TM, "_device_alignment", _fake_path)
    monkeypatch.setattr(T, "device_alignments", lambda m, ws: [_fake_path(m, *w) for w in ws])
    audios = [np.full(int(s * 16000), float(rid), dtype=np.float32) for rid, s in enumerate(SECONDS)]
    return model, audios, calls


@pytest.mark.parametrize("kw", [dict(), dict(word_timestamps=True), dict(word_timestamps=True, hallucination_silence_threshold=2.0),
                                dict(beam_size=5, best_of=5)])
@pytest.mark.parametrize("batch_size", [1, 3, None])
def test_batch_equals_sequential(stubs, kw, batch_size):
    model, audios, calls = stubs
    tok = _Tok()
    want = [T.transcribe(model, a, tokenizer=tok, **kw) for a in audios]
    torch.manual_seed(0)
    got = T.transcribe_batch(model, audios, batch_size=batch_size, tokenizer=tok, **kw)
    assert got == want
    assert got[6]["segments"] == [] and got[SILENT]["segments"] == []        # 4 ms: no frame; silence: every window skipped
    assert all(got[i]["segments"] for i in (0, 1, 3, 4, 5, 7))
    temps = [c[0] for c in calls]
    assert any(t > 0 for t in temps), "no window fell back"
    assert len({c[2][0] for c in calls}) == 1                               # one seed per call
    # each decode carries only the windows that still need a result, with one clip id per window
    limit = batch_size or 64 // (5 if "beam_size" in kw else 1)
    for t, wins, (seed, ids) in calls:
        assert len(ids) == len(wins) <= limit and len(set(wins)) == len(wins)


def test_clip_ids_follow_recording_seek_and_temperature(stubs):
    from olmoasr_b200.decode_engine import window_clip_id

    model, audios, calls = stubs
    T.transcribe_batch(model, audios, batch_size=3, tokenizer=_Tok())
    for t, wins, (_, ids) in calls:
        ti = T.DEFAULT_TEMPERATURES.index(t)
        assert ids == [window_clip_id(rid, seek, ti) for rid, seek in wins]
    assert len({window_clip_id(r, s, t) for r in range(8) for s in (0, 3000, 4500) for t in range(6)}) == 8 * 3 * 6


def test_log_mel_is_computed_when_a_recording_joins(stubs, monkeypatch):
    model, audios, _ = stubs
    active, seen = [], []

    def log_mel(audio, *a, **k):
        seen.append(int(audio[0]) if len(audio) else None)
        return _fake_log_mel(audio, *a, **k)

    monkeypatch.setattr(T, "log_mel_spectrogram", log_mel)
    real_encoder = model.encoder

    def encoder(mel):
        active.append(len(seen))
        return real_encoder(mel)

    model.encoder = encoder
    T.transcribe_batch(model, audios, batch_size=2, tokenizer=_Tok())
    assert seen == list(range(len(audios)))
    assert active[0] == 2, "only the first batch_size recordings are prepared before the first round"


def test_rejected_arguments(stubs):
    model, audios, _ = stubs
    with pytest.raises(ValueError, match="batch_size"):
        T.transcribe_batch(model, audios, batch_size=0)
    with pytest.raises(ValueError, match="tokenizer"):
        T.transcribe_batch(model, audios, word_timestamps=True)
    for clip in ("5,10", [3.0, 9.0], "x"):
        with pytest.raises(ValueError, match="clip_timestamps"):
            T.transcribe_batch(model, audios, clip_timestamps=clip)
    assert T.transcribe_batch(model, [], tokenizer=_Tok()) == []
    assert T.transcribe_batch(model, audios[:1], clip_timestamps=[0.0]) == [T.transcribe(model, audios[0])]


def test_models_expose_transcribe_batch():
    from olmoasr_b200 import inf_model, model

    for cls in (model.OLMoASR, inf_model.OLMoASR):
        assert callable(cls.transcribe_batch)


def test_decoding_task_passes_clip_ids_to_the_engine():
    from olmoasr_b200 import decoding as D
    import contextlib

    from tests.test_sampling_host import _StubModel

    m = _StubModel()
    pinned = []
    m.eng.splits_of = lambda rows: (pinned.append(rows), contextlib.nullcontext())[1]
    ids = list(range(100, 113))
    D.decode_windows(m, torch.zeros(13, 1500, 8), D.DecodingOptions(best_of=5, temperature=0.4), None, (77, ids))
    calls = m.eng.calls
    assert [(c[1], c[2]["seed"], c[2]["clip_ids"]) for c in calls] == [(12, 77, ids[:12]), (1, 77, ids[12:])]
    assert pinned == [5]                                        # steps split the cross-attention like a one-clip call
    m2 = _StubModel()
    D.decode(m2, torch.zeros(2, 80, 3000), D.DecodingOptions(best_of=5, temperature=0.4))
    assert "clip_ids" not in m2.eng.calls[0][2]                 # decode() keys clips by their index, as before
