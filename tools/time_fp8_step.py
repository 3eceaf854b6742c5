"""Training-step time, memory and loss of FP8 block projections (`fp8_autocast()`) against bf16, one GPU.

    python tools/time_fp8_step.py [--variant medium] [--batch 16] [--rounds 5] [--steps 5] [--profile] [--out DIR]

bench.py's workload: the medium model over slabs with FusedAdamW, the 16-clip synthetic batch of olmoasr_b200.synthetic.
One model; the two routes alternate in rounds so that clock and co-tenant drift hit them alike, each round timing `steps`
steps of each after one untimed step.  Memory first: two steps of each route after a reset of the peak statistics.
Reports the median device time per step, the peak memory and the last loss of each route, with the card's name, power
limit and max SM clock read in the same call.  --profile adds a separate torch.profiler pass over one FP8 step and reports
the device time of the per-row quantiser and of the FP8 GEMMs as shares of the step's kernel time.
"""
from __future__ import annotations

import argparse
import contextlib
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

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
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None, help="directory for the JSON result (also printed)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_fp8_step.py measures on a CUDA device; none is available")

    import olmoasr_b200 as ob
    from olmoasr_b200 import synthetic as synth
    from olmoasr_b200.fp8 import fp8_autocast
    from olmoasr_b200.model import OLMoASR
    from olmoasr_b200.optim import FusedAdamW

    dev = torch.device("cuda", 0)
    B = args.batch
    wav = synth.waveforms(B, int16=True).to(dev)
    ti, ty, pm, _ = synth.text_batch(B)
    ti, ty, pm = ti.to(dev), ty.to(dev), pm.to(dev)
    torch.manual_seed(0)
    with torch.device(dev):
        m = OLMoASR(ob.VARIANT_TO_DIMS[args.variant])
    slabs = m.use_slabs()
    opt = FusedAdamW(list(m.parameters()), lr=1.5e-3, betas=(0.9, 0.98), eps=1e-6, weight_decay=0.1, max_grad_norm=1.0,
                     slabs=slabs)
    ROUTES = {"bf16": contextlib.nullcontext, "fp8": fp8_autocast}
    last = {}

    def step(route):
        with ROUTES[route]():
            loss = m(ob.log_mel_spectrogram(wav), ti, pm, targets=ty)
            opt.zero_grad()
            loss.backward()
        opt.step()
        last[route] = loss.detach()

    memory = {}
    for route in ROUTES:
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        for _ in range(2):
            step(route)
        torch.cuda.synchronize()
        memory[route] = torch.cuda.max_memory_allocated(dev)

    times = {route: [] for route in ROUTES}
    for _ in range(args.rounds):
        for route in ROUTES:
            step(route)                                  # untimed
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                step(route)
            e1.record()
            torch.cuda.synchronize()
            times[route].append(e0.elapsed_time(e1) / args.steps)
    med = {k: statistics.median(v) for k, v in times.items()}
    res = {"variant": args.variant, "clips_per_step": B, "card": _card(),
           "ms_per_step": {k: round(v, 2) for k, v in med.items()},
           "ms_per_step_all_rounds": {k: [round(x, 2) for x in v] for k, v in times.items()},
           "max_memory_allocated_gib": {k: round(v / 2 ** 30, 2) for k, v in memory.items()},
           "last_loss": {k: float(v) for k, v in last.items()}}

    if args.profile:
        from torch.profiler import ProfilerActivity, profile
        step("fp8")
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            step("fp8")
            torch.cuda.synchronize()
        total = quant = gemm8 = 0.0
        for e in prof.key_averages():
            t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            total += t
            if "quantize_" in e.key:
                quant += t
            elif "gemm_fp8_kernel" in e.key:
                gemm8 += t
        res["profile_fp8_step"] = {"kernel_ms": round(total / 1e3, 2), "quantiser_ms": round(quant / 1e3, 2),
                                   "quantiser_share": round(quant / total, 4), "fp8_gemm_ms": round(gemm8 / 1e3, 2),
                                   "fp8_gemm_share": round(gemm8 / total, 4)}
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / "time_fp8_step.json").write_text(line + "\n")


if __name__ == "__main__":
    main()
