"""Generate tests/golden/* from the UNMODIFIED reference.

    OLMOASR_REFERENCE_ROOT=<checkout of allenai/OLMoASR> python tools/make_golden.py

  logmel_hf.npz     transformers.WhisperFeatureExtractor (independent implementation of the upstream
                    whisper log-mel) on seeded waveforms, frame-subsampled.
  model_tiny.pt     outputs of olmoasr/model.py (tiny, seed 0) on the seeded synthetic batch:
                    fp32 and bf16-autocast logits samples, losses, gradient norms; plus per-tensor weight
                    checksums so that the oracle's re-created weights can be pinned on any box.
  inf_tiny.pt       olmoasr/inf_model.py: full-prefix logits sample and kv-cache step logits.
  ref_tiny_outputs.pt  the reference's train-model forward (tiny, seed 0) in fp32 and under CPU bf16 autocast: dense
                    logits samples and whole-tensor sums, what the oracle is compared with element for element.
  timing_hf.npz     transformers' _dynamic_time_warping and _median_filter (independent restatements of upstream
                    whisper/timing.py's dtw and median_filter) on seeded matrices.
  ref_tiny_cross_qk.pt  the reference's inference model (tiny, seed 0, fp32) with forward hooks on every cross_attn
                    reading outs[-1], as whisper.timing does: a sample of the raw cross-attention logits.
"""
import sys
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from oracle import logmel, ref_import, synth  # noqa: E402
from oracle import model as OM  # noqa: E402

OUT = ROOT / "tests" / "golden"
OUT.mkdir(parents=True, exist_ok=True)


def golden_logmel():
    from transformers import WhisperFeatureExtractor

    fe = WhisperFeatureExtractor()
    wav = synth.waveforms(2).numpy()
    clips = {
        "noise": wav[0],
        "short_int16": logmel.pad_or_trim(logmel.int16_to_float(synth.waveforms(2, int16=True).numpy()[1][:51237])),
        "tone": (0.3 * np.sin(2 * np.pi * 440.0 * np.arange(480000) / 16000.0)).astype(np.float32),
    }
    out = {}
    for k, w in clips.items():
        m = fe(w, sampling_rate=16000, return_tensors="np")["input_features"][0]
        out[k] = m[:, ::7].astype(np.float32)
    np.savez_compressed(OUT / "logmel_hf.npz", **out)
    print("logmel_hf.npz", {k: v.shape for k, v in out.items()})


def checksums(sd):
    return {k: (float(v.double().sum()), float(v.double().abs().sum())) for k, v in sd.items()}


def golden_model():
    ref_model, ref_inf, ref_dims = ref_import.load()
    dims = ref_dims.VARIANT_TO_DIMS["tiny"]
    torch.manual_seed(0)
    rm = ref_model.OLMoASR(dims)
    B = 2
    mel = torch.from_numpy(logmel.log_mel_spectrogram(synth.waveforms(B).numpy()))
    ti, ty, pm, lens = synth.text_batch(B)
    logits = rm(mel, ti, pm)
    loss = torch.nn.functional.cross_entropy(logits.view(-1, logits.shape[-1]), ty.view(-1), ignore_index=51864)
    loss.backward()
    gnorm = {k: float(p.grad.double().norm()) for k, p in rm.named_parameters()}
    gsample = {k: rm.get_parameter(k).grad.flatten()[::1013][:64].clone() for k in
               ("encoder.conv1.weight", "encoder.blocks.0.attn.key.weight", "encoder.blocks.3.mlp.0.bias",
                "decoder.token_embedding.weight", "decoder.positional_embedding",
                "decoder.blocks.1.cross_attn.query.weight", "decoder.ln.weight")}
    with torch.no_grad(), torch.autocast("cpu", dtype=torch.bfloat16):
        logits_bf = rm(mel, ti, pm)
    loss_bf = torch.nn.functional.cross_entropy(logits_bf.view(-1, logits_bf.shape[-1]), ty.view(-1), ignore_index=51864)
    with torch.no_grad():
        logits_2d = rm(mel, ti[:, :20], None)
    torch.save({
        "variant": "tiny", "seed": 0, "batch": B,
        "weight_checksums": checksums(rm.state_dict()),
        "logits_fp32_sample": logits.detach()[:, ::16, ::997].clone(),
        "loss_fp32": float(loss),
        "logits_bf16_sample": logits_bf[:, ::16, ::997].clone(),
        "loss_bf16": float(loss_bf),
        "logits_2dmask_sample": logits_2d[:, ::4, ::997].clone(),
        "grad_norms": gnorm, "grad_samples": gsample,
        "torch_version": torch.__version__,
    }, OUT / "model_tiny.pt")
    print("model_tiny.pt loss", float(loss), float(loss_bf))

    torch.manual_seed(0)
    im = ref_inf.OLMoASR(dims)
    sd = im.state_dict()
    g = torch.Generator().manual_seed(7)
    sd["decoder.positional_embedding"] = torch.randn(448, dims.n_text_state, generator=g) * 0.01
    im.load_state_dict(sd)
    with torch.no_grad():
        full = im(mel, ti[:, :20])
        xa = im.encoder(mel)
        cache, hooks = im.install_kv_cache_hooks()
        s1 = im.decoder(ti[:, :3], xa, kv_cache=cache)
        s2 = im.decoder(ti[:, 3:4], xa, kv_cache=cache)
        s3 = im.decoder(ti[:, 4:5], xa, kv_cache=cache)
        for h in hooks:
            h.remove()
    torch.save({
        "variant": "tiny", "seed": 0, "pos_seed": 7,
        "weight_checksums": checksums(im.state_dict()),
        "full_logits_sample": full[:, ::4, ::997].clone(),
        "step_logits_sample": [s1[:, :, ::997].clone(), s2[:, :, ::997].clone(), s3[:, :, ::997].clone()],
        "argmax_full": full.argmax(-1).clone(),
        "xa_sample": xa[:, ::100, ::37].clone(),
    }, OUT / "inf_tiny.pt")
    print("inf_tiny.pt")


def golden_ref_outputs():
    ref_model, ref_inf, ref_dims = ref_import.load()
    torch.manual_seed(0)
    rm = ref_model.OLMoASR(ref_dims.VARIANT_TO_DIMS["tiny"])
    mel = torch.from_numpy(logmel.log_mel_spectrogram(synth.waveforms(2).numpy()))
    ti, ty, pm, _ = synth.text_batch(2)
    with torch.no_grad():
        l32 = rm(mel, ti, pm)
        with torch.autocast("cpu", dtype=torch.bfloat16):
            lbf = rm(mel, ti, pm)
    torch.save({
        "fp32_sample": l32[:, ::16, ::97].clone(), "fp32_sum": float(l32.double().sum()), "fp32_abs_sum": float(l32.double().abs().sum()),
        "bf16_sample": lbf[:, ::16, ::97].float().clone(), "bf16_dtype": str(lbf.dtype),
        "torch_version": torch.__version__,
    }, OUT / "ref_tiny_outputs.pt")
    print("ref_tiny_outputs.pt", tuple(l32.shape), lbf.dtype)


def golden_grad_noise():
    """Per-tensor relative L2 distance between the reference's bf16-autocast gradients and its fp32 gradients
    (tiny, seed 0, the synthetic batch): the yardstick for gradient parity of any bf16 implementation."""
    dims = OM.variant_dims("tiny")
    sd = OM.init_state_dict(dims, 0, True)  # bit-identical to the reference's weights (tests/test_oracle_pin.py)
    B = 2
    mel = torch.from_numpy(logmel.log_mel_spectrogram(synth.waveforms(B).numpy()))
    ti, ty, pm, _ = synth.text_batch(B)

    def grads(ac):
        p = {k: v.clone().requires_grad_(k != "encoder.positional_embedding") for k, v in sd.items()}
        OM.token_ce(OM.model_forward(p, dims, mel, ti, pm, True, ac), ty).backward()
        return {k: v.grad for k, v in p.items() if v.grad is not None}

    g32, gbf = grads(None), grads(torch.bfloat16)
    torch.save({k: float((gbf[k] - g32[k]).norm() / g32[k].norm()) for k in g32}, OUT / "grad_noise_tiny.pt")
    print("grad_noise_tiny.pt")


WIDTHS = {"base": (512, 8), "small": (768, 12), "medium": (1024, 16)}   # olmoasr/config/model_dims.py:28-89


def golden_widths(depth=(2, 2)):
    """The benchmarked variants at their real WIDTH and head count (what selects GEMM tile shapes, attention grids, LN
    vector widths) but depth 2+2 so that the fp32 reference runs in seconds on a CPU.  From the UNMODIFIED reference:
    fp32 loss, logits sample, per-tensor gradient norms and samples, weight checksums.  From the pinned oracle: the
    reference's own bf16-autocast noise (logits rel-L2 and per-tensor gradient rel-L2 against fp32) -- the yardstick a
    bf16 implementation is held to."""
    from dataclasses import replace

    ref_model, ref_inf, ref_dims = ref_import.load()
    B = 2
    mel = torch.from_numpy(logmel.log_mel_spectrogram(synth.waveforms(B).numpy()))
    ti, ty, pm, _ = synth.text_batch(B)
    for name in WIDTHS:
        rd = replace(ref_dims.VARIANT_TO_DIMS[name], n_audio_layer=depth[0], n_text_layer=depth[1])
        torch.manual_seed(0)
        rm = ref_model.OLMoASR(rd)
        logits = rm(mel, ti, pm)
        loss = torch.nn.functional.cross_entropy(logits.view(-1, logits.shape[-1]), ty.view(-1), ignore_index=51864)
        loss.backward()
        gnorm = {k: float(p.grad.double().norm()) for k, p in rm.named_parameters()}
        gsample = {k: p.grad.flatten()[::1013][:64].clone() for k, p in rm.named_parameters()
                   if k.endswith(("conv1.weight", "blocks.0.attn.key.weight", "blocks.1.mlp.0.bias", "token_embedding.weight",
                                  "decoder.positional_embedding", "blocks.1.cross_attn.query.weight", "decoder.ln.weight"))}
        dims = replace(OM.variant_dims(name), n_audio_layer=depth[0], n_text_layer=depth[1])
        sd = OM.init_state_dict(dims, 0, True)
        assert all(torch.equal(sd[k], v) for k, v in rm.state_dict().items())

        def grads(ac):
            p = {k: v.clone().requires_grad_(k != "encoder.positional_embedding") for k, v in sd.items()}
            lg = OM.model_forward(p, dims, mel, ti, pm, True, ac)
            OM.token_ce(lg, ty).backward()
            return lg.detach(), {k: v.grad for k, v in p.items() if v.grad is not None}

        l32, g32 = grads(None)
        lbf, gbf = grads(torch.bfloat16)
        assert torch.equal(l32, logits.detach())
        torch.save({
            "variant": name, "depth": depth, "seed": 0, "batch": B,
            "weight_checksums": checksums(rm.state_dict()),
            "logits_fp32_sample": logits.detach()[:, ::16, ::997].clone(), "loss_fp32": float(loss),
            "loss_bf16": float(OM.token_ce(lbf, ty)),
            "logits_bf16_noise": float((lbf - l32).norm() / l32.norm()),
            "grad_norms": gnorm, "grad_samples": gsample,
            "grad_noise": {k: float((gbf[k] - g32[k]).norm() / g32[k].norm()) for k in g32},
            "torch_version": torch.__version__,
        }, OUT / f"model_{name}_{depth[0]}x{depth[1]}.pt")
        print(f"model_{name}_{depth[0]}x{depth[1]}.pt loss", float(loss), "bf16 logits noise", float((lbf - l32).norm() / l32.norm()))


DTW_SHAPES = ((1, 1), (3, 7), (40, 300), (225, 1500))
MEDFILT_LENGTHS = (2, 3, 4, 750)


def timing_inputs():
    """The seeded DTW and median-filter inputs of timing_hf.npz (tests/test_timing_host.py regenerates them)."""
    g = np.random.default_rng(11)
    dtw = {f"dtw_{r}x{c}": g.standard_normal((r, c)).astype(np.float32) for r, c in DTW_SHAPES}
    planted = g.uniform(0.0, 1.0, (60, 400)).astype(np.float32)
    cols = np.sort(g.choice(400, 60, replace=False))
    planted[np.arange(60), cols] = -5.0
    dtw["dtw_planted"] = planted
    med = {f"med_{n}": g.standard_normal((3, 5, n)).astype(np.float32) for n in MEDFILT_LENGTHS}
    return dtw, med


def golden_timing_hf():
    from transformers.models.whisper.generation_whisper import _dynamic_time_warping, _median_filter

    dtw, med = timing_inputs()
    out = {}
    for k, x in dtw.items():
        ti, tj = _dynamic_time_warping(x)
        out[k + "_text"], out[k + "_time"] = np.asarray(ti, np.int64), np.asarray(tj, np.int64)
    for k, x in med.items():
        out[k] = _median_filter(torch.from_numpy(x), 7).numpy()
    np.savez_compressed(OUT / "timing_hf.npz", **out)
    print("timing_hf.npz", sorted(out))


def golden_cross_qk():
    ref_model, ref_inf, ref_dims = ref_import.load()
    dims = ref_dims.VARIANT_TO_DIMS["tiny"]
    torch.manual_seed(0)
    im = ref_inf.OLMoASR(dims)
    sd = im.state_dict()
    g = torch.Generator().manual_seed(7)
    sd["decoder.positional_embedding"] = torch.randn(448, dims.n_text_state, generator=g) * 0.01
    im.load_state_dict(sd)
    mel = torch.from_numpy(logmel.log_mel_spectrogram(synth.waveforms(1).numpy()))
    tokens = torch.cat([torch.tensor([50257, 50362]), torch.randint(0, 50256, (21,), generator=g), torch.tensor([50256])])
    qks = [None] * dims.n_text_layer
    hooks = [b.cross_attn.register_forward_hook(lambda _, ins, outs, index=i: qks.__setitem__(index, outs[-1][0]))
             for i, b in enumerate(im.decoder.blocks)]
    with torch.no_grad():
        im(mel, tokens[None])
    for h in hooks:
        h.remove()
    torch.save({"variant": "tiny", "seed": 0, "pos_seed": 7, "tokens": tokens,
                "qk_sample": torch.stack(qks)[:, :, :, ::13].clone(), "frame_step": 13,
                "torch_version": torch.__version__}, OUT / "ref_tiny_cross_qk.pt")
    print("ref_tiny_cross_qk.pt", tuple(torch.stack(qks).shape))


if __name__ == "__main__":
    which = sys.argv[1:] or ["logmel", "model", "ref_outputs", "grad_noise", "widths", "timing_hf", "cross_qk"]
    if "logmel" in which:
        golden_logmel()
    if "model" in which:
        golden_model()
    if "ref_outputs" in which:
        golden_ref_outputs()
    if "grad_noise" in which:
        golden_grad_noise()
    if "widths" in which:
        golden_widths()
    if "timing_hf" in which:
        golden_timing_hf()
    if "cross_qk" in which:
        golden_cross_qk()
