"""Event-timed attention forward / backward at the bench's shapes (medium: 16 heads of 64, 24 encoder and 24 decoder
layers; 16 clips of 30 s), with the decoder's real per-clip key lengths.

    python tools/time_attention.py [--json OUT]

Per use it prints the time per call and TFLOP/s counted two ways: useful (4 B H Tq Tkv 64 for the forward, halved
when causal, and 2.5 x that for the backward) and executed (the backward's kernels run 7 matmuls of 2 B H Tq Tkv 64
where the useful count has 5, because the dQ kernel recomputes S and dP).  The last line is attention time per
training step: per-call time x 24 layers, summed over the three uses.  The card and its power limit head the output."""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from olmoasr_b200 import kernels as K  # noqa: E402
from olmoasr_b200 import synthetic as synth  # noqa: E402

B, H, LAYERS = 16, 16, 24
d = H * 64


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        out = torch.cuda.get_device_name() + ", power limit unknown"
    return out


def timeit(fn, n=20):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--json", default=None, help="also write the table as JSON here")
    args = ap.parse_args()
    print(f"card: {card()}")
    dec_len = synth.text_batch(B)[3].to(torch.int32)   # the bench's decoder key lengths
    rows, step_ms = [], 0.0
    for name, Tq, Tkv, causal in (("encoder self", 1500, 1500, False), ("cross", 448, 1500, False),
                                  ("decoder self", 448, 448, True)):
        torch.manual_seed(0)
        q = torch.randn(B * Tq, d, device="cuda").bfloat16()
        kv = torch.randn(B * Tkv, 2 * d, device="cuda").bfloat16()
        k, v = kv[:, :d], kv[:, d:]
        dout = torch.randn(B * Tq, d, device="cuda").bfloat16()
        kv_len = dec_len.cuda() if causal else None
        o, lse = K.attention_fwd(q, k, v, B, H, Tq, Tkv, causal=causal, kv_len=kv_len)
        fwd_ms = timeit(lambda: K.attention_fwd(q, k, v, B, H, Tq, Tkv, causal=causal, kv_len=kv_len))
        bwd_ms = timeit(lambda: K.attention_bwd(q, k, v, o, dout, lse, B, H, Tq, Tkv, causal=causal, kv_len=kv_len))
        fl = 4.0 * B * H * Tq * Tkv * 64 * (0.5 if causal else 1.0)
        r = dict(use=name, fwd_ms=fwd_ms, bwd_ms=bwd_ms, fwd_tflops=fl / fwd_ms / 1e9,
                 bwd_useful_tflops=2.5 * fl / bwd_ms / 1e9, bwd_executed_tflops=3.5 * fl / bwd_ms / 1e9)
        rows.append(r)
        step_ms += LAYERS * (fwd_ms + bwd_ms)
        print(f"{name:13s} fwd {fwd_ms:7.3f} ms ({r['fwd_tflops']:4.0f} TFLOP/s)   bwd {bwd_ms:7.3f} ms "
              f"({r['bwd_useful_tflops']:4.0f} useful / {r['bwd_executed_tflops']:4.0f} executed TFLOP/s)")
    print(f"attention per training step (x{LAYERS} layers, fwd + bwd, three uses): {step_ms:.1f} ms")
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(dict(card=card(), rows=rows, step_ms=step_ms), indent=1))


if __name__ == "__main__":
    main()
