"""Time the fp8 device decoder (`DecodingOptions(fp8=True)`) against the 16-bit one, fp16 activations.

    python tools/time_fp8_decode.py [--models small,medium] [--n 1,2,4,8,16,32,64] [--rounds 5] [--json out.json]

For each model and sequence count n, the 16-bit and the fp8 engine of one model are timed alternately in the same
process (rounds x (16-bit, fp8)), and the medians over rounds are reported:
  * step: device time of one greedy step (CUDA events around 40 graph replays at self-attention length ~ 20 .. 60);
  * GB/s: the engine's own `step_bytes` (fp8-aware) at the middle length over the step time;
  * transcribe_batch: wall time of transcribe_batch() over seeded synthetic recordings (greedy, 96 tokens per window),
    once per engine after a warm-up call (small only unless --batch-all).
Weights are random (the model's initialisation); step times do not depend on their values.  The card's name, power
limit and clocks are read in the same run.
"""
import argparse
import json
import statistics
import subprocess
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks.mem"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:   # the timings stand without it; say so
        out = f"nvidia-smi unavailable ({e})"
    return out


def step_ms(eng, xa, n, reps=40):
    """One measurement: 20 warm-up replays, then `reps` timed replays; (ms per step, self-attention length mid-window)."""
    toks = torch.full((n, 1), 50257, dtype=torch.int32)
    eng.prepare(xa[:n])
    eng.reset(n, toks, sample_begin=1)
    eng.suppress.zero_()
    g = eng._graph(n)
    for _ in range(20):
        g.replay()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        g.replay()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps, 20 + reps // 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="small,medium")
    ap.add_argument("--n", default="1,2,4,8,16,32,64")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--recordings", type=int, default=8)
    ap.add_argument("--batch-all", action="store_true")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_fp8_decode.py measures on a CUDA device; none found")
    import olmoasr_b200 as ob
    from olmoasr_b200 import synthetic
    from olmoasr_b200.inf_model import OLMoASR
    from olmoasr_b200.transcribe import transcribe_batch

    info = card()
    print(f"card: {info}")
    results = {"card": info, "models": {}}
    ns = [int(v) for v in args.n.split(",")]
    for name in args.models.split(","):
        torch.manual_seed(0)
        m = OLMoASR(ob.VARIANT_TO_DIMS[name]).cuda()
        engines = {"16-bit": m.decode_engine(torch.float16), "fp8": m.decode_engine(torch.float16, fp8=True)}
        g = torch.Generator(device="cuda").manual_seed(1)
        xa = torch.randn(max(ns), 1500, m.dims.n_audio_state, device="cuda", generator=g).to(torch.bfloat16)
        rows = []
        for n in ns:
            times = {k: [] for k in engines}
            t_mid = 0
            for _ in range(args.rounds):
                for k, eng in engines.items():
                    ms, t_mid = step_ms(eng, xa, n)
                    times[k].append(ms)
            row = {"n": n}
            for k, eng in engines.items():
                med = statistics.median(times[k])
                row[k] = {"step_ms": med, "spread_ms": max(times[k]) - min(times[k]),
                          "step_mb": eng.step_bytes(n, t_mid) / 1e6, "gbs": eng.step_bytes(n, t_mid) / (med * 1e-3) / 1e9}
            row["speedup"] = row["16-bit"]["step_ms"] / row["fp8"]["step_ms"]
            rows.append(row)
            print(f"{name} n={n:2d}: 16-bit {row['16-bit']['step_ms']:.3f} ms ({row['16-bit']['gbs']:.0f} GB/s), "
                  f"fp8 {row['fp8']['step_ms']:.3f} ms ({row['fp8']['gbs']:.0f} GB/s), x{row['speedup']:.2f}", flush=True)
        launches = {k: eng.launches_per_step for k, eng in engines.items()}
        print(f"{name}: launches per step {launches}")
        res = {"steps": rows, "launches_per_step": launches}
        if name == "small" or args.batch_all:
            audios = [synthetic.waveforms(1, rank=r, n_samples=int((20 + 37 * r) * 16000))[0] for r in range(args.recordings)]
            wall = {}
            for k, fp8 in (("16-bit", False), ("fp8", True), ("16-bit", False), ("fp8", True)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                transcribe_batch(m, audios, temperature=0.0, sample_len=96, fp8=fp8)
                torch.cuda.synchronize()
                wall[k] = time.perf_counter() - t0       # the second call of each is kept (the first warms up)
            res["transcribe_batch_s"] = wall
            print(f"{name}: transcribe_batch of {args.recordings} recordings ({sum(a.numel() for a in audios) / 16000:.0f} s "
                  f"of audio): 16-bit {wall['16-bit']:.2f} s, fp8 {wall['fp8']:.2f} s")
        results["models"][name] = res
        del engines, m
        torch.cuda.empty_cache()
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(results, indent=1))


if __name__ == "__main__":
    main()
