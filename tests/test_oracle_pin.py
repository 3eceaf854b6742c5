"""Pin the oracle (oracle/*.py) to the reference before anything is compared against it.

  * log-mel restatement  <->  transformers.WhisperFeatureExtractor fixtures (tests/golden/logmel_hf.npz)
  * model restatement    <->  outputs of the UNMODIFIED reference olmoasr/{model,inf_model}.py captured by
                              tools/make_golden.py (tests/golden/model_tiny.pt, inf_tiny.pt, ref_tiny_outputs.pt).
"""
import numpy as np
import pytest
import torch

from oracle import logmel, synth
from oracle import model as OM


def _clips():
    wav = synth.waveforms(2).numpy()
    return {
        "noise": wav[0],
        "short_int16": logmel.pad_or_trim(logmel.int16_to_float(synth.waveforms(2, int16=True).numpy()[1][:51237])),
        "tone": (0.3 * np.sin(2 * np.pi * 440.0 * np.arange(480000) / 16000.0)).astype(np.float32),
    }


def test_mel_filterbank_properties():
    f = logmel.mel_filters(80)
    assert f.shape == (80, 201) and f.dtype == np.float32
    assert int((f != 0).sum()) == 391  # SURVEY.md section 8(c)
    assert abs(float(f.max()) - 0.02588) < 1e-5


def test_logmel_matches_hf_fixture(golden_dir):
    gold = np.load(golden_dir / "logmel_hf.npz")
    for name, w in _clips().items():
        m = logmel.log_mel_spectrogram(w)
        assert m.shape == (80, 3000)
        assert np.abs(m[:, ::7] - gold[name]).max() < 2e-5, name


def test_logmel_batch_is_per_sample():
    w = synth.waveforms(2).numpy()
    w[1] *= 0.01
    mb = logmel.log_mel_spectrogram(w)
    for i in range(2):
        assert np.array_equal(mb[i], logmel.log_mel_spectrogram(w[i]))


def test_pad_or_trim():
    x = np.arange(10, dtype=np.float32)
    assert logmel.pad_or_trim(x, 4).tolist() == [0, 1, 2, 3]
    y = logmel.pad_or_trim(x, 12)
    assert y.shape == (12,) and y[10:].tolist() == [0, 0]
    assert logmel.pad_or_trim(np.zeros((0,), np.float32), 5).shape == (5,)


@pytest.fixture(scope="module")
def tiny_train():
    dims = OM.variant_dims("tiny")
    sd = OM.init_state_dict(dims, seed=0, train=True)
    B = 2
    mel = torch.from_numpy(logmel.log_mel_spectrogram(synth.waveforms(B).numpy()))
    ti, ty, pm, lens = synth.text_batch(B)
    return dims, sd, mel, ti, ty, pm


def test_weights_match_reference_checksums(tiny_train, golden_dir):
    dims, sd, *_ = tiny_train
    g = torch.load(golden_dir / "model_tiny.pt", weights_only=False)
    assert set(g["weight_checksums"]) == set(sd)
    for k, (s, a) in g["weight_checksums"].items():
        assert float(sd[k].double().sum()) == pytest.approx(s, rel=1e-9, abs=1e-9), k
        assert float(sd[k].double().abs().sum()) == pytest.approx(a, rel=1e-9), k


def test_train_forward_matches_reference_golden(tiny_train, golden_dir):
    dims, sd, mel, ti, ty, pm = tiny_train
    g = torch.load(golden_dir / "model_tiny.pt", weights_only=False)
    with torch.no_grad():
        logits = OM.model_forward(sd, dims, mel, ti, pm, train_model=True)
    assert logits.shape == (2, 448, 51865) and logits.dtype == torch.float32
    assert torch.allclose(logits[:, ::16, ::997], g["logits_fp32_sample"], atol=2e-4, rtol=1e-4)
    assert float(OM.token_ce(logits, ty)) == pytest.approx(g["loss_fp32"], rel=1e-5)
    with torch.no_grad():
        l2 = OM.model_forward(sd, dims, mel, ti[:, :20], None, train_model=True)
    assert torch.allclose(l2[:, ::4, ::997], g["logits_2dmask_sample"], atol=2e-4, rtol=1e-4)


def test_train_bf16_autocast_matches_reference_golden(tiny_train, golden_dir):
    """bf16 autocast on the CPU is host-dependent (oneDNN picks different bf16 kernels per CPU), so the golden bf16
    samples of the generating host are a YARDSTICK, not a bit pattern: on any host the bf16 run must sit at the same
    distance from the (host-independent) fp32 golden as the reference's own bf16 run did, and within twice that
    noise of the recorded bf16 sample."""
    dims, sd, mel, ti, ty, pm = tiny_train
    g = torch.load(golden_dir / "model_tiny.pt", weights_only=False)
    with torch.no_grad():
        lb = OM.model_forward(sd, dims, mel, ti, pm, train_model=True, autocast_dtype=torch.bfloat16)
    rel = lambda a, b: float((a - b).norm() / b.norm())
    noise = rel(g["logits_bf16_sample"], g["logits_fp32_sample"])      # the reference's own bf16 error (7.8e-3)
    assert 0.5 * noise <= rel(lb[:, ::16, ::997], g["logits_fp32_sample"]) <= 1.5 * noise
    assert rel(lb[:, ::16, ::997], g["logits_bf16_sample"]) <= 2.0 * noise
    assert float(OM.token_ce(lb, ty)) == pytest.approx(g["loss_fp32"], rel=1e-3)
    assert float(OM.token_ce(lb, ty)) == pytest.approx(g["loss_bf16"], rel=1e-3)


def test_backward_matches_reference_golden(tiny_train, golden_dir):
    dims, sd, mel, ti, ty, pm = tiny_train
    g = torch.load(golden_dir / "model_tiny.pt", weights_only=False)
    p = {k: v.clone().requires_grad_(k != "encoder.positional_embedding") for k, v in sd.items()}
    OM.token_ce(OM.model_forward(p, dims, mel, ti, pm, train_model=True), ty).backward()
    for k, n in g["grad_norms"].items():
        assert float(p[k].grad.double().norm()) == pytest.approx(n, rel=2e-3, abs=1e-7), k
    for k, s in g["grad_samples"].items():
        assert torch.allclose(p[k].grad.flatten()[::1013][:64], s, atol=1e-6, rtol=2e-3), k


def test_inference_model_and_kv_cache_match_reference_golden(golden_dir):
    g = torch.load(golden_dir / "inf_tiny.pt", weights_only=False)
    dims = OM.variant_dims("tiny")
    sd = OM.init_state_dict(dims, seed=0, train=False)
    gen = torch.Generator().manual_seed(g["pos_seed"])
    sd["decoder.positional_embedding"] = torch.randn(448, dims.n_text_state, generator=gen) * 0.01
    mel = torch.from_numpy(logmel.log_mel_spectrogram(synth.waveforms(2).numpy()))
    ti, *_ = synth.text_batch(2)
    with torch.no_grad():
        full = OM.model_forward(sd, dims, mel, ti[:, :20], None, train_model=False)
        xa = OM.encoder_forward(sd, dims, mel, sdpa=False)
        cache = {}
        steps = [OM.decoder_forward(sd, dims, ti[:, a:b], xa, None, False, cache=cache) for a, b in ((0, 3), (3, 4), (4, 5))]
    assert torch.allclose(full[:, ::4, ::997], g["full_logits_sample"], atol=2e-4, rtol=1e-4)
    assert torch.equal(full.argmax(-1), g["argmax_full"])
    assert torch.allclose(xa[:, ::100, ::37], g["xa_sample"], atol=1e-4, rtol=1e-4)
    for s, gs in zip(steps, g["step_logits_sample"]):
        assert torch.allclose(s[:, :, ::997], gs, atol=2e-4, rtol=1e-4)
    # kv-cache steps == full re-forward (the invariant listed in SURVEY.md section 4)
    assert torch.allclose(steps[1][:, 0], full[:, 3], atol=2e-4)
    assert torch.allclose(steps[2][:, 0], full[:, 4], atol=2e-4)


@pytest.mark.parametrize("name", ["base", "medium"])
def test_width_goldens_pin_the_oracle_at_benchmark_widths(name, golden_dir):
    """tests/golden/model_<variant>_2x2.pt: outputs of the unmodified reference at the benchmarked WIDTH (depth 2+2).  The
    oracle must reproduce them before the GPU tests compare the CUDA path with the oracle at those widths."""
    from dataclasses import replace

    g = torch.load(golden_dir / f"model_{name}_2x2.pt", weights_only=False)
    dims = replace(OM.variant_dims(name), n_audio_layer=2, n_text_layer=2)
    sd = OM.init_state_dict(dims, seed=0, train=True)
    for k, (s_, a_) in g["weight_checksums"].items():
        assert float(sd[k].double().sum()) == pytest.approx(s_, rel=1e-9, abs=1e-9), k
    mel = torch.from_numpy(logmel.log_mel_spectrogram(synth.waveforms(2).numpy()))
    ti, ty, pm, _ = synth.text_batch(2)
    p = {k: v.clone().requires_grad_(k != "encoder.positional_embedding") for k, v in sd.items()}
    logits = OM.model_forward(p, dims, mel, ti, pm, train_model=True)
    loss = OM.token_ce(logits, ty)
    assert torch.allclose(logits.detach()[:, ::16, ::997], g["logits_fp32_sample"], atol=2e-4, rtol=1e-4)
    assert float(loss.detach()) == pytest.approx(g["loss_fp32"], rel=1e-5)
    loss.backward()
    for k, n in g["grad_norms"].items():
        assert float(p[k].grad.double().norm()) == pytest.approx(n, rel=2e-3, abs=1e-7), k
    for k, smp in g["grad_samples"].items():
        assert torch.allclose(p[k].grad.flatten()[::1013][:64], smp, atol=1e-6, rtol=2e-3), k


def test_reference_outputs_match_golden(tiny_train, golden_dir):
    """The oracle against the unmodified reference's own forward outputs, stored by tools/make_golden.py (ref_outputs) where
    the reference tree is present: fp32 logits element for element on a dense sample plus whole-tensor sums, and the CPU
    bf16-autocast logits within the reference's own bf16 noise (oneDNN picks host-dependent bf16 kernels)."""
    dims, sd, mel, ti, ty, pm = tiny_train
    g = torch.load(golden_dir / "ref_tiny_outputs.pt", weights_only=False)
    with torch.no_grad():
        l32 = OM.model_forward(sd, dims, mel, ti, pm, train_model=True)
        lbf = OM.model_forward(sd, dims, mel, ti, pm, True, torch.bfloat16)
    assert l32.shape == (2, 448, 51865) and str(lbf.dtype) == g["bf16_dtype"]
    assert torch.allclose(l32[:, ::16, ::97], g["fp32_sample"], atol=1e-5, rtol=1e-5)
    assert float(l32.double().sum()) == pytest.approx(g["fp32_sum"], rel=1e-6)
    assert float(l32.double().abs().sum()) == pytest.approx(g["fp32_abs_sum"], rel=1e-6)
    rel = lambda a, b: float((a.float() - b).norm() / b.norm())
    noise = rel(g["bf16_sample"], g["fp32_sample"])
    assert rel(lbf[:, ::16, ::97], g["bf16_sample"]) <= 2.0 * noise
