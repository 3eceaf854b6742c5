"""Time transcribe_batch() against sequential transcribe() on synthetic long-form recordings.

    python tools/time_transcribe_batch.py [--variant small] [--recordings 24] [--rounds 3] [--json out.json]

Model: the inference model of `--variant` with the seeded initial weights of oracle/model.py, its token embedding scaled
and its positional embedding redrawn as tests/test_decode_engine_gpu.py::_build does (small: x6.0 and 0.1).  Random
initial weights never emit eot; the sharpened ones end their windows, so the fallback ladder runs as it would on a
checkpoint instead of every window falling through every temperature.  Recordings: `--recordings` seeded Gaussian-noise
waveforms of 60-300 s.

For each option set (greedy with timestamps; the long-form eval options beam_size=5, best_of=5; word_timestamps=True
with a stand-in tokenizer) it alternates sequential transcribe() over every recording and one transcribe_batch() call,
`--rounds` times, with host clocks around synchronised work, and reports audio seconds per wall second, windows, rounds,
device-decoder calls and graph replays, and the mean number of engine rows occupied per replay (how many of the 64 rows
a replay carries; with `live` the rows whose sequence has not ended, for the greedy and sampling calls).  Then it
compares the two drivers' outputs at temperature 0.  The card's name and power limit are read in the same run.
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

SHARPEN = {"tiny": (3.0, 0.5), "small": (6.0, 0.1)}
EOT = 50256


class SpaceTokenizer:
    def decode(self, ids):
        return "".join(f" w{i % 97}" for i in ids)


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:   # the timings stand without it; say so
        return f"nvidia-smi unavailable ({e})"


def build(variant):
    import olmoasr_b200 as ob
    from olmoasr_b200.inf_model import OLMoASR
    from oracle import model as OM

    dims = OM.variant_dims(variant)
    sd = OM.init_state_dict(dims, 0, train=False)
    emb_scale, pos_scale = SHARPEN[variant]
    g = torch.Generator().manual_seed(7)
    sd["decoder.positional_embedding"] = torch.randn(448, dims.n_text_state, generator=g) * pos_scale
    sd["decoder.token_embedding.weight"] = sd["decoder.token_embedding.weight"] * emb_scale
    m = OLMoASR(ob.VARIANT_TO_DIMS[variant])
    m.load_state_dict(sd)
    return m.cuda()


class Counter:
    """Counts engine calls, graph replays and rows per replay by wrapping the engine's decode methods."""

    def __init__(self, eng, transcribe_module):
        self.calls = self.replays = self.row_replays = self.live_replays = self.live_counted = 0
        self.rounds = self.windows = 0
        for name in ("greedy", "sample", "beam_search"):
            setattr(eng, name, self._wrap(getattr(eng, name), name))
        real_round = transcribe_module._decode_round

        def round_spy(model, features, recordings, *a, **k):
            self.rounds += 1
            self.windows += len(recordings)
            return real_round(model, features, recordings, *a, **k)

        transcribe_module._decode_round = round_spy

    def _wrap(self, fn, name):
        def run(feats, init, *a, **k):
            out = fn(feats, init, *a, **k)
            replays = out[-1]
            n_init = len(init)
            if name == "greedy":
                rows = feats.shape[0]
                lens = [self._live(r, n_init, replays) for r in out[0].tolist()]
            elif name == "sample":
                rows = feats.shape[0] * a[2]
                lens = [self._live(r, n_init, replays) for cands in out[0] for r, _ in cands]
            else:
                rows, lens = feats.shape[0] * a[1], None
            self.calls += 1
            self.replays += replays
            self.row_replays += rows * replays
            if lens is not None:
                self.live_replays += sum(lens)
                self.live_counted += replays
            return out
        return run

    @staticmethod
    def _live(row, n_init, replays):
        """Replays in which the row had not yet ended (the teacher-forced prefix, then up to and including its eot)."""
        sampled = row[n_init:]
        n = sampled.index(EOT) + 1 if EOT in sampled else len(sampled)
        return min(replays, n_init - 1 + n)

    def reset(self):
        self.calls = self.replays = self.row_replays = self.live_replays = self.live_counted = 0
        self.rounds = self.windows = 0

    def summary(self):
        return dict(engine_calls=self.calls, replays=self.replays, rounds=self.rounds, windows=self.windows,
                    rows_per_replay=self.row_replays / max(1, self.replays),
                    live_rows_per_replay=(self.live_replays / self.live_counted) if self.live_counted else None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--variant", default="small")
    ap.add_argument("--recordings", type=int, default=24)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--sets", default="greedy,eval,words")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_transcribe_batch.py measures on a CUDA device; none found")
    import numpy as np

    import olmoasr_b200.transcribe as T

    info = card()
    print(f"card: {info}  (torch: {torch.cuda.get_device_name(0)})")
    m = build(args.variant)
    rng = np.random.default_rng(0)
    seconds = rng.uniform(60.0, 300.0, args.recordings)
    g = torch.Generator().manual_seed(1)
    audios = [torch.clamp(torch.randn(int(s * 16000), generator=g) * 0.1, -1.0, 1.0) for s in seconds]
    total = float(sum(seconds))
    print(f"model: {args.variant}, seeded initial weights sharpened as tests/test_decode_engine_gpu.py::_build; "
          f"{len(audios)} recordings, {total:.0f} s of audio")
    counter = Counter(m.decode_engine(torch.float16), T)
    option_sets = {"greedy": dict(), "eval": dict(without_timestamps=False, beam_size=5, best_of=5),
                   "words": dict(word_timestamps=True, tokenizer=SpaceTokenizer())}
    report = dict(card=info, variant=args.variant, recordings=len(audios), audio_seconds=total, sets={})
    for name in args.sets.split(","):
        kw = option_sets[name]
        T.transcribe(m, audios[0][:16000 * 30], **kw)            # graphs captured, kernels loaded
        T.transcribe_batch(m, [a[:16000 * 30] for a in audios[:4]], **kw)
        rates = {"sequential": [], "batch": []}
        counts = {}
        for r in range(args.rounds):
            order = ("sequential", "batch") if r % 2 == 0 else ("batch", "sequential")
            for arm in order:
                counter.reset()
                torch.manual_seed(r)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                if arm == "sequential":
                    for a in audios:
                        T.transcribe(m, a, **kw)
                else:
                    T.transcribe_batch(m, audios, **kw)
                torch.cuda.synchronize()
                wall = time.perf_counter() - t0
                rates[arm].append(total / wall)
                counts[arm] = counter.summary()
                print(f"{name:>6} round {r} {arm:>10}: {total / wall:8.1f} audio s / wall s ({wall:6.1f} s)  {counts[arm]}")
        # the two drivers at temperature 0
        seq = [T.transcribe(m, a, temperature=0.0, **kw) for a in audios]
        bat = T.transcribe_batch(m, audios, temperature=0.0, **kw)
        same = sum(s["text"] == b["text"] and [(x["seek"], x["start"], x["end"], x["tokens"], x.get("words")) for x in s["segments"]]
                   == [(x["seek"], x["start"], x["end"], x["tokens"], x.get("words")) for x in b["segments"]] for s, b in zip(seq, bat))
        med = {k: statistics.median(v) for k, v in rates.items()}
        print(f"{name:>6}: median {med['sequential']:.1f} -> {med['batch']:.1f} audio s / wall s "
              f"(x{med['batch'] / med['sequential']:.2f}); temperature 0: {same}/{len(audios)} recordings identical")
        report["sets"][name] = dict(rates=rates, median=med, counts=counts, identical_at_t0=same)
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(report, indent=1))


if __name__ == "__main__":
    main()
