"""Time beam search (beam 5) on the device decoder for the `small` model in fp16 against greedy decoding.

    python tools/time_beam.py [--steps 96] [--clips 1,2,4,8,12] [--json out.json]

For each clip count n it reports, from CUDA events around graph replays:
  * beam step: device time of one beam-5 step over n clips (5 n rows) at self-attention length ~64 + steps / 2;
  * reorder: the kv-reorder kernel alone (a permutation of every clip's beams), and its share of the step;
  * greedy n / greedy 5n: one greedy step over n and over 5 n sequences (the rows a beam step decodes);
  * bytes: algorithmic HBM bytes of a beam step (weights once, cross K/V per clip, self K/V per beam, fp32 logits);
  * RTF: decoder wall time of a whole `beam_search` call of `steps` tokens per clip over (n x 30 s) of audio.
Weights are random (the model's initialisation); timings do not depend on their values.  The card's name, power limit and
clocks are read in the same run.
"""
import argparse
import json
import subprocess
import sys
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


def events_ms(fn, reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=96)
    ap.add_argument("--clips", default="1,2,4,8,12")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_beam.py measures on a CUDA device; none found")
    import olmoasr_b200 as ob
    from olmoasr_b200.inf_model import OLMoASR

    torch.manual_seed(0)
    m = OLMoASR(ob.VARIANT_TO_DIMS["small"]).cuda()
    eng = m.decode_engine(torch.float16)
    beam, patience = 5, 6.4          # 32 finished candidates per clip: the decode never stops early
    sot = [50257]
    sup = tuple(range(50357, 50362)) + (50257,)
    T0 = 64
    rows = []
    info = card()
    print(f"card: {info}  (torch: {torch.cuda.get_device_name(0)})")
    hdr = f"{'clips':>5} {'rows':>4} {'beam step us':>12} {'reorder us':>10} {'share':>6} {'greedy n us':>11} " \
          f"{'greedy 5n us':>12} {'MB/step':>8} {'GB/s':>6} {'RTF':>8}"
    print(hdr)
    for C in [int(x) for x in args.clips.split(",")]:
        n = C * beam
        xa = (torch.randn(C, 1500, eng.d, device="cuda") * 0.5).bfloat16()
        # whole decode (graph capture on the first call), then the timed one
        eng.beam_search(xa, sot, 8, beam, patience, sup, timestamps=True, max_initial_timestamp_index=50)
        torch.cuda.synchronize()
        t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t[0].record()
        eng.beam_search(xa, sot, args.steps, beam, patience, sup, timestamps=True, max_initial_timestamp_index=50)
        t[1].record()
        torch.cuda.synchronize()
        rtf = t[0].elapsed_time(t[1]) / 1e3 / (C * 30.0)
        # steady beam steps from position T0
        eng.prepare(xa)
        eng.reset(n, torch.tensor([sot]).repeat(n, 1), None, sup, True, 0)
        eng.reset_beam(C, beam, round(beam * patience), True, 50)
        g = eng._graph(n)
        for _ in range(T0):
            g.replay()
        step_ms = events_ms(g.replay, args.steps)
        # the reorder alone, every clip's beams permuted (the worst case: no identity rows)
        perm = torch.tensor([c * beam + (j + 1) % beam for c in range(C) for j in range(beam)], dtype=torch.int32, device="cuda")
        eng.src_rows[:n] = perm
        eng.pos.fill_(T0 + args.steps // 2)
        reorder_ms = events_ms(lambda: eng.reorder_kv(C, beam), 50)
        # greedy steps over n and 5n sequences at the same length
        greedy = []
        for N in (C, n):
            xg = (torch.randn(N, 1500, eng.d, device="cuda") * 0.5).bfloat16()
            eng.prepare(xg)
            eng.reset(N, torch.tensor([[50257, 50362]]).repeat(N, 1), None, sup, True, 0)
            gg = eng._graph(N)
            eng.pos.fill_(T0)
            greedy.append(events_ms(gg.replay, args.steps))
        e = 2
        d, L = eng.d, eng.L
        t_self = T0 + args.steps // 2
        weights = L * 12 * d * d * e + eng.V * d * e
        nbytes = weights + C * L * 2 * eng.n_audio_ctx * d * e + n * (L * 2 * t_self * d * e + eng.V * 4)
        r = dict(clips=C, rows=n, beam_step_us=step_ms * 1e3, reorder_us=reorder_ms * 1e3, reorder_share=reorder_ms / step_ms,
                 greedy_n_us=greedy[0] * 1e3, greedy_5n_us=greedy[1] * 1e3, bytes_per_step=nbytes,
                 achieved_GBps=nbytes / (step_ms * 1e-3) / 1e9, rtf=rtf)
        rows.append(r)
        print(f"{C:>5} {n:>4} {r['beam_step_us']:>12.1f} {r['reorder_us']:>10.1f} {r['reorder_share']:>6.1%} "
              f"{r['greedy_n_us']:>11.1f} {r['greedy_5n_us']:>12.1f} {nbytes / 1e6:>8.1f} {r['achieved_GBps']:>6.0f} {rtf:>8.5f}")
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(dict(card=info, model="small", dtype="fp16", beam=beam, rows=rows), indent=1))


if __name__ == "__main__":
    main()
