"""Training-step time and memory of LoRA fine-tuning against full fine-tuning, one GPU.

    python tools/time_lora_step.py [--variant medium] [--batch 16] [--rank 32] [--rounds 5] [--steps 5] [--out DIR]

bench.py's workload: the medium model over slabs with FusedAdamW, the 16-clip synthetic batch of olmoasr_b200.synthetic.
Three routes:
    full      every parameter trains
    lora      rank-`rank` adapters on attn.query / attn.value of both stacks, everything else frozen
    lora_dec  the same adapters in the decoder only: the encoder is frozen and runs no backward at all
Memory first: each route alone (its model built, two steps, then freed) reports torch.cuda.max_memory_allocated.  Then
the three routes alternate in rounds so that clock and co-tenant drift hit them alike; each round times `steps` steps of
each after one untimed step.  Reports the median device time per step, with the card's name, power limit and max SM clock
read in the same call.
"""
from __future__ import annotations

import argparse
import gc
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

ROUTES = {"full": None,
          "lora": ("encoder.attn.query", "encoder.attn.value", "decoder.attn.query", "decoder.attn.value"),
          "lora_dec": ("decoder.attn.query", "decoder.attn.value")}


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
    ap.add_argument("--rank", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for the JSON result (also printed)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_lora_step.py measures on a CUDA device; none is available")

    import olmoasr_b200 as ob
    from olmoasr_b200 import synthetic as synth
    from olmoasr_b200.lora import add_lora
    from olmoasr_b200.model import OLMoASR
    from olmoasr_b200.optim import FusedAdamW

    dev = torch.device("cuda", 0)
    B = args.batch
    wav = synth.waveforms(B, int16=True).to(dev)
    ti, ty, pm, _ = synth.text_batch(B)
    ti, ty, pm = ti.to(dev), ty.to(dev), pm.to(dev)

    def build(route):
        torch.manual_seed(0)
        with torch.device(dev):
            m = OLMoASR(ob.VARIANT_TO_DIMS[args.variant])
        if ROUTES[route] is not None:
            add_lora(m, args.rank, 2 * args.rank, targets=ROUTES[route])
        slabs = m.use_slabs()
        opt = FusedAdamW([p for p in m.parameters() if p.requires_grad], lr=1.5e-3, betas=(0.9, 0.98), eps=1e-6,
                         weight_decay=0.1, max_grad_norm=1.0, slabs=slabs)
        n_train = sum(p.numel() for p in m.parameters() if p.requires_grad)

        def step():
            loss = m(ob.log_mel_spectrogram(wav), ti, pm, targets=ty)
            opt.zero_grad()
            loss.backward()
            opt.step()
            return loss
        return m, step, n_train

    memory, trainable = {}, {}
    for route in ROUTES:
        gc.collect()
        torch.cuda.empty_cache()
        torch.cuda.reset_peak_memory_stats(dev)
        m, step, trainable[route] = build(route)
        for _ in range(2):
            step()
        torch.cuda.synchronize()
        memory[route] = torch.cuda.max_memory_allocated(dev)
        del m, step
    gc.collect()
    torch.cuda.empty_cache()

    steps = {route: build(route)[1] for route in ROUTES}
    times = {route: [] for route in ROUTES}
    for _ in range(args.rounds):
        for route, step in steps.items():
            step()                                  # untimed
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                step()
            e1.record()
            torch.cuda.synchronize()
            times[route].append(e0.elapsed_time(e1) / args.steps)
    med = {k: statistics.median(v) for k, v in times.items()}
    res = {"variant": args.variant, "clips_per_step": B, "rank": args.rank, "card": _card(),
           "ms_per_step": {k: round(v, 2) for k, v in med.items()},
           "ms_per_step_all_rounds": {k: [round(x, 2) for x in v] for k, v in times.items()},
           "max_memory_allocated_gib": {k: round(v / 2 ** 30, 2) for k, v in memory.items()},
           "trainable_parameters": trainable}
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / "time_lora_step.json").write_text(line + "\n")


if __name__ == "__main__":
    main()
