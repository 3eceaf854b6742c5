"""Training-step time of the packed decoder route (`text_lens=`) against the dense route (`padding_mask`), one GPU.

    python tools/time_packed_step.py [--variant medium] [--batch 16] [--rounds 5] [--steps 5] [--out DIR]

bench.py's workload: the medium model over slabs with FusedAdamW, the 16-clip synthetic batch of olmoasr_b200.synthetic
(transcripts of 31 ... 216 tokens padded to 448).  Dense and packed steps alternate in rounds so that clock and co-tenant
drift hit both alike; each round times `steps` steps of each after one untimed step.  Reports the median device time per
step of each route, with the card's name, power limit and max SM clock read in the same call.

Before timing, both routes run one backward from the same weights: the script reports their losses and the relative
difference of a seeded sample of 1M entries of the gradient slab.
"""
from __future__ import annotations

import argparse
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
    ap.add_argument("--out", default=None, help="directory for the JSON result (also printed)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_packed_step.py measures on a CUDA device; none is available")

    import olmoasr_b200 as ob
    from olmoasr_b200 import synthetic as synth
    from olmoasr_b200.model import OLMoASR
    from olmoasr_b200.optim import FusedAdamW

    dev = torch.device("cuda", 0)
    B = args.batch
    wav = synth.waveforms(B, int16=True).to(dev)
    ti, ty, pm, lens = synth.text_batch(B)
    ti, ty, pm = ti.to(dev), ty.to(dev), pm.to(dev)

    torch.manual_seed(0)
    with torch.device(dev):
        m = OLMoASR(ob.VARIANT_TO_DIMS[args.variant])
    slabs = m.use_slabs()
    opt = FusedAdamW(m.parameters(), lr=1.5e-3, betas=(0.9, 0.98), eps=1e-6, weight_decay=0.1, max_grad_norm=1.0,
                     slabs=slabs)

    def loss_of(packed):
        mel = ob.log_mel_spectrogram(wav)
        return m(mel, ti, targets=ty, text_lens=lens) if packed else m(mel, ti, pm, targets=ty)

    # the two routes' outputs from the same weights
    g = torch.Generator(device=dev).manual_seed(0)
    sample = torch.randint(0, slabs.G.numel(), (1 << 20,), device=dev, generator=g)
    out = {}
    for packed in (False, True):
        opt.zero_grad()
        loss = loss_of(packed)
        loss.backward()
        out[packed] = (loss.item(), slabs.G[sample].clone(), float(slabs.G.norm()))
    (ld, gd, nd), (lp, gp, npk) = out[False], out[True]
    compare = {"loss_dense": ld, "loss_packed": lp, "loss_rel_diff": abs(lp - ld) / abs(ld),
               "grad_sample_rel_l2": float((gp - gd).norm() / gd.norm()), "grad_norm_dense": nd, "grad_norm_packed": npk}

    def step(packed):
        loss = loss_of(packed)
        opt.zero_grad()
        loss.backward()
        opt.step()

    times = {"dense": [], "packed": []}
    for _ in range(args.rounds):
        for name in times:
            step(name == "packed")                # untimed
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.steps):
                step(name == "packed")
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / args.steps)
    med = {k: statistics.median(v) for k, v in times.items()}
    res = {"variant": args.variant, "clips_per_step": B, "text_rows": int(lens.sum()), "dense_rows": B * ti.shape[1],
           "card": _card(), "ms_per_step": {k: round(v, 2) for k, v in med.items()},
           "ms_per_step_all_rounds": {k: [round(x, 2) for x in v] for k, v in times.items()},
           "packed_vs_dense_speedup": round(med["dense"] / med["packed"], 4), "outputs": compare}
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / "time_packed_step.json").write_text(line + "\n")


if __name__ == "__main__":
    main()
