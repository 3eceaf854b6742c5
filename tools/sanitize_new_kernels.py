"""Small invocations of the kernels added in round 2, for `compute-sanitizer --tool memcheck|racecheck python tools/sanitize_new_kernels.py`
(the reference has no sanitizer runs, SURVEY.md section 5; out-of-bounds or racy shared-memory accesses in hand-written kernels are
exactly what parity tests can miss)."""
import math
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))


def main():
    import olmoasr_b200 as ob
    from olmoasr_b200 import _core, audio
    from olmoasr_b200 import kernels as K
    from olmoasr_b200 import synthetic as synth
    from olmoasr_b200.config.model_dims import ModelDimensions
    from olmoasr_b200.inf_model import OLMoASR as InfModel
    from olmoasr_b200.model import OLMoASR
    from olmoasr_b200.optim import FusedAdamW

    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    # log-mel: odd length (end reflection inside the padded row), int16 and fp32
    wav = synth.waveforms(2, n_samples=16000 * 3 + 77)
    audio.log_mel_spectrogram(wav.to(dev))
    audio.log_mel_spectrogram(synth.waveforms(1, n_samples=6400, int16=True).to(dev))
    # mask -> key counts
    _, _, pm, _ = synth.text_batch(3)
    _core.kv_len_from_padding_mask(pm.to(dev))
    # attention forward / backward at the mask edges, both dtypes: ragged T, kv_len on and next to the 64-query / 128-key
    # tile edges (the backward's all-visible fast paths switch there), kv_len clamps, strided inputs and outputs
    for dtype in (torch.bfloat16, torch.float16):
        for B, T, Tkv, causal, lens in ((2, 65, 65, True, [65, 1]), (1, 191, 383, False, None),
                                        (6, 257, 257, True, [0, 63, 64, 128, 129, 300]), (2, 129, 300, False, [256, 257])):
            H, d = 2, 128
            qkv = torch.randn(B * T, 3 * d, device=dev).to(dtype)
            kv = torch.randn(B * Tkv, 2 * d, device=dev).to(dtype)
            q, k, v = (qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:]) if causal else (qkv[:, :d], kv[:, :d], kv[:, d:])
            kv_len = torch.tensor(lens, device=dev, dtype=torch.int32) if lens else None
            obuf = torch.zeros(B * T + 1, d + 64, device=dev, dtype=dtype)
            o, lse = K.attention_fwd(q, k, v, B, H, T, Tkv, causal=causal, kv_len=kv_len, out=obuf[1:, 64:])
            gq = torch.zeros(B * T + 1, d + 64, device=dev, dtype=dtype)
            gkv = torch.zeros(B * Tkv + 1, 2 * d + 64, device=dev, dtype=dtype)
            K.attention_bwd(q, k, v, o, torch.randn_like(o), lse, B, H, T, Tkv, causal=causal, kv_len=kv_len,
                            dq=gq[1:, 64:], dk=gkv[1:, :d], dv=gkv[1:, d:2 * d])
    # slab training step on a narrow model (direct gradients, flat optimizer, shadow write)
    dims = ModelDimensions(80, 1500, 64, 1, 1, 51864, 448, 64, 1, 1)
    m = OLMoASR(dims).to(dev)
    slabs = m.use_slabs()
    opt = FusedAdamW(m.parameters(), slabs=slabs)
    mel = ob.log_mel_spectrogram(synth.waveforms(1).to(dev))
    ti, ty, pmask, _ = (t.to(dev) for t in synth.text_batch(1))
    for _ in range(2):
        loss = m(mel, ti, pmask, targets=ty)
        opt.zero_grad()
        loss.backward()
        opt.step()
    # the same step in fp16 with GradScaler: every fp16 instantiation and the device-side unscale / skip
    scaler = torch.amp.GradScaler("cuda")
    for _ in range(2):
        with torch.autocast("cuda", dtype=torch.float16):
            loss = m(mel, ti, pmask, targets=ty)
        opt.zero_grad()
        scaler.scale(loss).backward()
        scaler.step(opt)
        scaler.update()
    # decode engine: direct (3 sequences) and staged (40 sequences) skinny GEMMs, split and fused attention, sampling
    im = InfModel(dims).to(dev)
    with torch.no_grad():
        im.decoder.positional_embedding.normal_(0, 0.02)
    for dtype in (torch.float16, torch.bfloat16):
        eng = im.decode_engine(dtype)
        for n in (3, 40):
            xa = torch.randn(n, 1500, 64, device=dev).bfloat16()
            eng.greedy(xa, [50257, 50362], 3, suppress=(7, 9))
        # beam search: candidates, select, kv reorder, grouped cross-attention; with and without timestamp rules
        xa = torch.randn(3, 1500, 64, device=dev).bfloat16()
        eng.beam_search(xa, [50257, 50362], 4, 5, suppress=(7, 9))
        eng.beam_search(xa[:2], [50257], 4, 3, patience=2.0, suppress=(7, 9), timestamps=True, max_initial_timestamp_index=50)
        # rule-aware sampling: greedy with timestamp rules, best-of sampling (grouped cross-attention) with and without them
        eng.greedy(xa, [50257], 4, suppress=(7, 9), timestamps=True, max_initial_timestamp_index=50)
        eng.sample(xa, [50257, 50362], 4, 0.6, best_of=5, seed=1, suppress=(7, 9))
        eng.sample(xa[:2], [50257], 4, 1.0, best_of=3, seed=2, clip_offset=5, suppress=(7, 9), timestamps=True,
                   max_initial_timestamp_index=50)
    # a training-layout engine (51865 logits per row, the pad row included): the only vocabulary whose last slice ends in a
    # partial float4, so the selection kernels' tail branch runs -- beam search with timestamp rules
    eng = m.decode_engine(torch.float16)
    eng.beam_search(torch.randn(2, 1500, 64, device=dev).bfloat16(), [50257], 4, 5, suppress=(7, 9), timestamps=True,
                    max_initial_timestamp_index=50)
    # word alignment: single-window and batched cost and DTW over ragged windows (edge tiles, one frame, 448 tokens)
    for dtype in (torch.float16, torch.bfloat16):
        windows = []
        for n_tok, n_frames in ((3, 1), (448, 37), (37, 750), (5, 3)):
            q, k = torch.randn(n_tok, 128, device=dev).to(dtype), torch.randn(800, 128, device=dev).to(dtype)
            windows.append(([(q[:, :64], k[:, :64]), (q[:, 64:], k[:, 64:])], n_frames))
        K.align_cost(*windows[1])
        costs = K.align_cost_batched(windows)
    K.dtw(costs[2])
    K.dtw_batched([costs[1], costs[2], costs[3], torch.randn(1, 1, device=dev), torch.randn(9, 1, device=dev)])
    torch.cuda.synchronize()
    print("sanitize run complete; loss", float(loss))


if __name__ == "__main__":
    main()
