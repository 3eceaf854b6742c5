"""Training-step throughput of the fp16 path against the bf16 path and stock PyTorch, in one process on one GPU.

    python tools/time_fp16_step.py [--variant medium] [--batch 16] [--rounds 3] [--steps 5] [--out DIR]

Three steps alternate in rounds, so that clock and co-tenant drift hit all of them alike:
  ours-bf16   model.loss -> backward -> FusedAdamW.step over slabs (what bench.py times);
  ours-fp16   the same under torch.autocast("cuda", torch.float16) with the reference's GradScaler calls
              (scaler.scale(loss).backward(); scaler.step(opt); scaler.update());
  torch-fp16  the stock PyTorch model of baseline/torch_stock.py under autocast(float16) with GradScaler and fused AdamW.
Each round times `steps` steps of each after one untimed step (which absorbs the slab re-cast that a switch between bf16
and fp16 costs).  Prints one JSON line: clips/s per step kind (median over rounds), with the card's name and power limit
read in the same call.
"""
from __future__ import annotations

import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch
import torch.nn.functional as F

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))


def _card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"unavailable ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--variant", default="medium")
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for the JSON result (also printed)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_fp16_step.py measures on a CUDA device; none is available")

    import olmoasr_b200 as ob
    from olmoasr_b200 import audio as A
    from olmoasr_b200 import synthetic as synth
    from olmoasr_b200.model import OLMoASR
    from olmoasr_b200.optim import FusedAdamW
    from baseline.torch_stock import Model, log_mel_torch

    dev = torch.device("cuda", 0)
    dims = ob.VARIANT_TO_DIMS[args.variant]
    B = args.batch
    wav = synth.waveforms(B, int16=True).to(dev)
    ti, ty, pm, _ = (t.to(dev) for t in synth.text_batch(B))

    torch.manual_seed(0)
    with torch.device(dev):
        ours = OLMoASR(dims)
    slabs = ours.use_slabs()
    opt = FusedAdamW(ours.parameters(), lr=1.5e-3, betas=(0.9, 0.98), eps=1e-6, weight_decay=0.1, max_grad_norm=1.0,
                     slabs=slabs)
    scaler = torch.amp.GradScaler("cuda")

    torch.manual_seed(0)
    stock = Model(dims).to(dev)
    sopt = torch.optim.AdamW(stock.parameters(), lr=1.5e-3, betas=(0.9, 0.98), eps=1e-6, weight_decay=0.1, fused=True)
    sscaler = torch.amp.GradScaler("cuda")
    filters = torch.as_tensor(A.mel_filterbank(80), dtype=torch.float32, device=dev)

    def ours_bf16():
        loss = ours(ob.log_mel_spectrogram(wav), ti, pm, targets=ty)
        opt.zero_grad()
        loss.backward()
        opt.step()

    def ours_fp16():
        mel = ob.log_mel_spectrogram(wav)
        with torch.autocast("cuda", dtype=torch.float16):
            loss = ours(mel, ti, pm, targets=ty)
        opt.zero_grad()
        scaler.scale(loss).backward()
        scaler.step(opt)
        scaler.update()

    def torch_fp16():
        mel = log_mel_torch(wav.float() / 32768.0, filters)
        with torch.autocast("cuda", dtype=torch.float16):
            logits = stock(mel, ti, pm)
            loss = F.cross_entropy(logits.view(-1, logits.shape[-1]), ty.view(-1), ignore_index=51864)
        sopt.zero_grad(set_to_none=True)
        sscaler.scale(loss).backward()
        sscaler.unscale_(sopt)
        torch.nn.utils.clip_grad_norm_(stock.parameters(), 1.0)
        sscaler.step(sopt)
        sscaler.update()

    kinds = {"ours-bf16": ours_bf16, "ours-fp16": ours_fp16, "torch-fp16": torch_fp16}
    rates = {k: [] for k in kinds}
    for _ in range(args.rounds):
        for name, fn in kinds.items():
            fn()                                  # untimed: warm-up / dtype switch
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            rates[name].append(B * args.steps / (e0.elapsed_time(e1) / 1e3))
    med = {k: statistics.median(v) for k, v in rates.items()}
    res = {"variant": args.variant, "clips_per_step": B, "card": _card(),
           "clips_per_s": {k: round(v, 2) for k, v in med.items()},
           "clips_per_s_all_rounds": {k: [round(x, 2) for x in v] for k, v in rates.items()},
           "fp16_vs_bf16": round(med["ours-fp16"] / med["ours-bf16"], 4),
           "fp16_vs_torch_fp16": round(med["ours-fp16"] / med["torch-fp16"], 4),
           "ours_skipped_steps": 2 * args.rounds * (args.steps + 1) - opt.applied_steps()}   # GradScaler overflow skips
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / "time_fp16_step.json").write_text(line + "\n")


if __name__ == "__main__":
    main()
