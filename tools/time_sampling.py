"""Time greedy decoding with timestamp rules and best-of-5 temperature sampling on the device decoder for the `small` model
in fp16, next to plain greedy decoding, and `transcribe()` with the engine against the hook loop.

    python tools/time_sampling.py [--steps 96] [--clips 1,4,16,64] [--seconds 150] [--reps 2] [--json out.json]

For each clip count n it reports, from CUDA events around graph replays at self-attention length ~64 + steps / 2:
  * greedy n: one plain greedy step over n sequences;
  * greedy+ts n: one greedy step with ApplyTimestampRules over n sequences;
  * best-of-5: one sampling step (temperature 0.6, timestamp rules) over n clips x 5 samples, and greedy 5n, a plain
    greedy step over the same 5 n rows (only where 5 n <= 64, the engine's batch).
Then the wall time of `transcribe()` with default options (temperature fallback 0.0 .. 1.0, timestamps) on a seeded
synthetic recording, with decoding.USE_ENGINE on and off, alternated in the same process.  Weights are random (the
model's initialisation): step times do not depend on their values; the transcribe comparison measures the same windows
and fallbacks on both routes only as far as both routes choose the same tokens.  The card's name, power limit and clocks
are read in the same run.
"""
import argparse
import json
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from tools.time_beam import card, events_ms  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=96)
    ap.add_argument("--clips", default="1,4,16,64")
    ap.add_argument("--seconds", type=float, default=150.0)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_sampling.py measures on a CUDA device; none found")
    import olmoasr_b200 as ob
    from olmoasr_b200 import decoding, synthetic
    from olmoasr_b200.decode_engine import sample_row_key
    from olmoasr_b200.inf_model import OLMoASR
    from olmoasr_b200.transcribe import transcribe

    torch.manual_seed(0)
    m = OLMoASR(ob.VARIANT_TO_DIMS["small"]).cuda()
    eng = m.decode_engine(torch.float16)
    sup = decoding.suppress_token_ids(decoding.DecodingOptions())
    T0, G = 64, 5
    info = card()
    print(f"card: {info}  (torch: {torch.cuda.get_device_name(0)})")

    def step_us(N, init, rules=None, group=1, temperature=0.0):
        """Device time of one step over N rows at self-attention length T0 (graph replays between CUDA events)."""
        eng.prepare((torch.randn(N // group, 1500, eng.d, device="cuda") * 0.5).bfloat16())
        eng.reset(N, torch.tensor([init]).repeat(N, 1), None, sup, True, 0)
        if rules is not None:
            eng._rules_cfg, eng._group = rules, group
            eng.row_keys[:N] = torch.tensor([sample_row_key(0, r // group, r % group) >> 1 for r in range(N)])
            eng.temperature.fill_(temperature)
        g = eng._graph(N)
        eng.pos.fill_(T0)
        return events_ms(g.replay, args.steps) * 1e3

    rows = []
    print(f"{'clips':>5} {'greedy n us':>11} {'greedy+ts n us':>14} {'best-of-5 us':>12} {'greedy 5n us':>12}")
    for n in [int(x) for x in args.clips.split(",")]:
        r = dict(clips=n)
        r["greedy_us"] = step_us(n, [50257, 50362])
        r["greedy_ts_us"] = step_us(n, [50257], rules=(1, 50, 0))
        if n * G <= eng.max_batch:
            r["best_of_5_us"] = step_us(n * G, [50257], rules=(1, 50, 1), group=G, temperature=0.6)
            r["greedy_5n_us"] = step_us(n * G, [50257, 50362])
        rows.append(r)
        fmt = lambda k: f"{r[k]:.1f}" if k in r else "-"
        print(f"{n:>5} {fmt('greedy_us'):>11} {fmt('greedy_ts_us'):>14} {fmt('best_of_5_us'):>12} {fmt('greedy_5n_us'):>12}")

    audio = synthetic.waveforms(1, n_samples=int(args.seconds * 16000))[0]
    walls = {True: [], False: []}
    torch.manual_seed(1)
    transcribe(m, audio)                                  # graphs captured, modules loaded
    for _ in range(args.reps):
        for use in (True, False):
            decoding.USE_ENGINE = use
            torch.manual_seed(1)
            torch.cuda.synchronize()
            t = time.perf_counter()
            out = transcribe(m, audio)
            torch.cuda.synchronize()
            walls[use].append(time.perf_counter() - t)
            print(f"transcribe engine={use}: {walls[use][-1]:.2f} s for {args.seconds:.0f} s of audio, "
                  f"{len(out['segments'])} segments")
    decoding.USE_ENGINE = True
    eng_s, hook_s = min(walls[True]), min(walls[False])
    print(f"transcribe() wall, best of {args.reps}: engine {eng_s:.2f} s, hook loop {hook_s:.2f} s ({hook_s / eng_s:.1f}x)")
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(dict(card=info, model="small", dtype="fp16", rows=rows, seconds=args.seconds,
                                                   transcribe_engine_s=walls[True], transcribe_hook_s=walls[False]), indent=1))


if __name__ == "__main__":
    main()
