"""Word-level timestamps, CPU side: the oracle (oracle/timing.py) against transformers' independent DTW / median filter
and against the unmodified reference's cross-attention logits; the alignment-head surface of the models; and the host
logic of olmoasr_b200/timing.py (word split, punctuation merge, duration clamps, segment adjustment, hallucination skip)
against the oracle on the same DTW paths and probabilities, with the device calls replaced."""
import base64
import copy
import ctypes
import gzip
import importlib.util
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import logmel, synth
from oracle import model as OM
from oracle import timing as OT

ROOT = Path(__file__).resolve().parents[1]
EOT = 50256


def _make_golden():
    spec = importlib.util.spec_from_file_location("make_golden", ROOT / "tools" / "make_golden.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_oracle_dtw_and_median_filter_equal_transformers(golden_dir):
    gold = np.load(golden_dir / "timing_hf.npz")
    dtw_in, med_in = _make_golden().timing_inputs()
    for k, x in dtw_in.items():
        ti, tj = OT.dtw(x)
        assert np.array_equal(ti, gold[k + "_text"]) and np.array_equal(tj, gold[k + "_time"]), k
    for k, x in med_in.items():
        assert np.array_equal(OT.median_filter(torch.from_numpy(x), 7).numpy(), gold[k]), k


def test_oracle_cross_qk_capture_matches_the_reference(golden_dir):
    g = torch.load(golden_dir / "ref_tiny_cross_qk.pt", weights_only=False)
    dims = OM.variant_dims("tiny")
    sd = OM.init_state_dict(dims, seed=0, train=False)
    gen = torch.Generator().manual_seed(g["pos_seed"])
    sd["decoder.positional_embedding"] = torch.randn(448, dims.n_text_state, generator=gen) * 0.01
    mel = torch.from_numpy(logmel.log_mel_spectrogram(synth.waveforms(1).numpy()))
    with torch.no_grad():
        xa = OM.encoder_forward(sd, dims, mel, sdpa=False)
        _, qks = OT.decoder_forward_qk(sd, dims, g["tokens"][None], xa)
    got = torch.stack([q[0] for q in qks])[..., ::g["frame_step"]]
    assert torch.allclose(got, g["qk_sample"], atol=2e-4, rtol=1e-4)


def test_alignment_heads_default_and_dump_round_trip():
    import olmoasr_b200 as ob
    from olmoasr_b200._core import OLMoASRBase
    from olmoasr_b200.inf_model import OLMoASR

    for name, dims in ob.VARIANT_TO_DIMS.items():
        heads = OLMoASRBase.alignment_heads.fget(SimpleNamespace(dims=dims, _alignment_mask=None))
        assert heads.is_sparse and heads.shape == (dims.n_text_layer, dims.n_text_head)
        assert [tuple(p) for p in heads.indices().T.tolist()] == OT.default_alignment_heads(dims.n_text_layer, dims.n_text_head), name

    m = OLMoASR(ob.VARIANT_TO_DIMS["tiny"])
    keys, bufs = list(m.state_dict().keys()), [(n, b.shape) for n, b in m.named_buffers()]
    mask = torch.zeros(4, 6, dtype=torch.bool)
    mask[1, 2] = mask[3, 0] = mask[3, 5] = True
    dump = base64.b85encode(gzip.compress(mask.numpy().tobytes()))
    m.set_alignment_heads(dump)
    assert m.alignment_heads.indices().T.tolist() == [[1, 2], [3, 0], [3, 5]]
    m.set_alignment_heads(dump.decode())
    assert torch.equal(m.alignment_heads.to_dense(), mask)
    m.set_alignment_heads(mask.numpy())
    assert torch.equal(m.alignment_heads.to_dense(), mask)
    with pytest.raises(ValueError):
        m.set_alignment_heads(torch.ones(3, 6, dtype=torch.bool))
    with pytest.raises(ValueError):
        m.set_alignment_heads(torch.zeros(4, 6, dtype=torch.bool))
    assert list(m.state_dict().keys()) == keys and [(n, b.shape) for n, b in m.named_buffers()] == bufs
    assert "alignment_heads" not in dict(m.named_buffers())


PIECES = [" the", " cat", "s", ".", ",", " sat", "!", " on", "ing", " \"", "mat", "?", " (", ")", " 'em", "-", " dog", ":"]


class FakeTokenizer:
    def decode(self, ids):
        return "".join(PIECES[i % len(PIECES)] for i in ids)


def _random_path(rng, rows, cols):
    """A monotone DTW path from (0, 0) to (rows - 1, cols - 1) with diagonal, down and right steps."""
    i = j = 0
    path = [(0, 0)]
    while (i, j) != (rows - 1, cols - 1):
        step = rng.integers(0, 3)
        if (step == 1 or j == cols - 1) and i < rows - 1:
            i += 1
        elif (step == 2 or i == rows - 1) and j < cols - 1:
            j += 1
        else:
            i, j = i + 1, j + 1
        path.append((i, j))
    p = np.array(path)
    return p[:, 0].astype(np.int64), p[:, 1].astype(np.int64)


def _window(rng, n_segments, seek):
    segs, t = [], seek / 100
    for _ in range(n_segments):
        n = int(rng.integers(1, 9))
        toks = [50364 + int(rng.integers(0, 20))] + [int(x) for x in rng.integers(0, 200, n)] + [50364 + int(rng.integers(20, 60))]
        start = t + float(rng.integers(0, 100)) / 50
        end = start + float(rng.integers(0, 400)) / 50
        segs.append({"id": 0, "seek": seek, "start": start, "end": end, "tokens": toks, "text": ""})
        t = end
    return segs


@pytest.mark.parametrize("seed", range(12))
def test_host_logic_equals_the_oracle(seed, monkeypatch):
    from olmoasr_b200 import timing as T

    rng = np.random.default_rng(seed)
    tok = FakeTokenizer()
    seek = int(rng.integers(0, 5000))
    segs = _window(rng, int(rng.integers(1, 4)), seek)
    text = [t for s in segs for t in s["tokens"] if t < EOT]
    n_frames = int(rng.integers(len(text) + 1, 1501))
    ti, tj = _random_path(rng, len(text) + 1, n_frames)
    probs = rng.uniform(0.01, 1.0, len(text)).tolist()

    ours = T.words_from_path(tok, text, ti, tj, probs)
    ref = OT.words_from_path(tok.decode, text, ti, tj, probs)
    assert [(w.word, w.tokens, w.start, w.end, w.probability) for w in ours] == \
        [(w.word, w.tokens, w.start, w.end, w.probability) for w in ref]

    monkeypatch.setattr(T, "_device_alignment", lambda *a, **k: (ti, tj, probs))
    last = float(rng.uniform(0, seek / 100 + 1))
    a, b = copy.deepcopy(segs), copy.deepcopy(segs)
    T.add_word_timestamps(segments=a, model=None, tokenizer=tok, mel=None, num_frames=2 * n_frames, last_speech_timestamp=last)
    OT.add_word_timestamps(b, OT.words_from_path(tok.decode, text, ti, tj, probs), last)
    assert a == b

    for threshold in (None, 0.5, 2.0):
        for single in (False, True):
            kw = dict(seek=seek + 1234, previous_seek=seek, segment_size=3000, time_offset=seek / 100,
                      window_end_time=(seek + 3000) / 100, segment_duration=30.0, content_frames=seek + 4000,
                      content_duration=(seek + 4000) / 100, last_speech_timestamp=last)
            x, y = copy.deepcopy(a), copy.deepcopy(a)
            got = T.after_word_timestamps(x, single_timestamp_ending=single, hallucination_silence_threshold=threshold, **kw)
            want = OT.window_step(y, kw["seek"], seek, 3000, single, kw["time_offset"], kw["window_end_time"], 30.0,
                                  kw["content_frames"], kw["content_duration"], last, threshold)
            assert got == want and x == y


def test_hallucination_skip_paths():
    """Crafted anomalous segments: a leading one after a long gap skips the window, one surrounded by silence is cut."""
    from olmoasr_b200 import timing as T

    def seg(start, end, words):
        return {"seek": 0, "start": start, "end": end, "tokens": [1], "text": " x",
                "words": [dict(word=" x", start=s, end=e, probability=p) for s, e, p in words]}

    kw = dict(seek=1500, previous_seek=0, segment_size=3000, single_timestamp_ending=False, time_offset=0.0,
              window_end_time=30.0, segment_duration=30.0, content_frames=9000, content_duration=90.0,
              last_speech_timestamp=0.0, hallucination_silence_threshold=2.0)
    lead = [seg(5.0, 5.1, [(5.0, 5.05, 0.01), (5.05, 5.1, 0.01)]), seg(6.0, 8.0, [(6.0, 7.0, 0.9)])]
    for impl in (T.after_word_timestamps, None):
        segs = copy.deepcopy(lead)
        got = impl(segs, **kw) if impl else OT.window_step(segs, 1500, 0, 3000, False, 0.0, 30.0, 30.0, 9000, 90.0, 0.0, 2.0)
        assert got == (True, 500, 0.0)
    mid = [seg(1.0, 3.0, [(1.0, 3.0, 0.9)]), seg(10.0, 10.1, [(10.0, 10.05, 0.01), (10.05, 10.1, 0.01)]),
           seg(20.0, 21.0, [(20.0, 21.0, 0.9)])]
    segs = copy.deepcopy(mid)
    skip, seek, last = T.after_word_timestamps(segs, **kw)
    assert not skip and seek == 1000 and len(segs) == 1 and last == 3.0


def test_word_timestamps_need_a_tokenizer():
    from olmoasr_b200.transcribe import transcribe

    with pytest.raises(ValueError, match="tokenizer"):
        transcribe(None, np.zeros(16000, dtype=np.float32), word_timestamps=True)


def test_timing_entry_points_validate_without_a_gpu():
    from olmoasr_b200 import _lib

    h = _lib.lib()
    p = ctypes.c_void_p(256)
    cases = [
        (lambda: h.oasr_align_cost(None, 1, 64, 8, 10, 7, p, p, 10, 1, None), b"null tensor"),
        (lambda: h.oasr_align_cost(p, 1, 80, 8, 10, 7, p, p, 10, 1, None), b"head_dim"),
        (lambda: h.oasr_align_cost(p, 0, 64, 8, 10, 7, p, p, 10, 1, None), b"at least one head"),
        (lambda: h.oasr_align_cost(p, 1, 64, 2, 10, 7, p, p, 10, 1, None), b"n_tok"),
        (lambda: h.oasr_align_cost(p, 1, 64, 449, 10, 7, p, p, 10, 1, None), b"n_tok"),
        (lambda: h.oasr_align_cost(p, 1, 64, 8, 0, 7, p, p, 10, 1, None), b"n_frames"),
        (lambda: h.oasr_align_cost(p, 1, 64, 8, 1501, 7, p, p, 1501, 1, None), b"n_frames"),
        (lambda: h.oasr_align_cost(p, 1, 64, 8, 10, 6, p, p, 10, 1, None), b"medfilt_width"),
        (lambda: h.oasr_align_cost(p, 1, 64, 8, 10, 9, p, p, 10, 1, None), b"medfilt_width"),
        (lambda: h.oasr_align_cost(p, 1, 64, 8, 10, 7, p, p, 10, 2, None), b"dtype"),
        (lambda: h.oasr_dtw(None, 4, 2, 4, p, p, p, p, None), b"null tensor"),
        (lambda: h.oasr_dtw(p, 4, 0, 4, p, p, p, p, None), b"empty matrix"),
        (lambda: h.oasr_dtw(p, 3, 2, 4, p, p, p, p, None), b"ldx"),
    ]
    for fn, msg in cases:
        rc = fn()
        assert rc == -1 and msg in h.oasr_last_error(), (rc, h.oasr_last_error())
