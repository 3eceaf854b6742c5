"""Time word-level alignment per 30 s window: olmoasr_b200.timing.find_alignment split into its decoder forward,
oasr_align_cost, oasr_dtw and host work, against a stock-torch restatement of upstream whisper/timing.py on the same GPU
(stack, softmax, std_mean, unfold/sort median, then a numpy DTW), with the window's beam-5 decode for scale.

    python tools/time_alignment.py [--variants small medium] [--n-text 32 128 224] [--rounds 3]

Seeded inference models (random weights), num_frames = 3000; CUDA events after warm-up; rounds alternate the two
implementations.  Prints the GPU name and power limit beside the numbers.
"""
import argparse
import statistics
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or torch.cuda.get_device_name()


def events_ms(fn, reps=1):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--variants", nargs="+", default=["small", "medium"])
    ap.add_argument("--n-text", nargs="+", type=int, default=[32, 128, 224])
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_alignment.py needs a CUDA device")

    import olmoasr_b200 as ob
    from olmoasr_b200 import kernels as K
    from olmoasr_b200 import timing as T
    from olmoasr_b200.decoding import DecodingOptions, decode
    from olmoasr_b200.inf_model import OLMoASR
    from olmoasr_b200.synthetic import waveforms
    from oracle import timing as OT

    print(f"GPU: {gpu_info()}")
    num_frames = 3000
    for variant in args.variants:
        dims = ob.VARIANT_TO_DIMS[variant]
        torch.manual_seed(0)
        m = OLMoASR(dims)
        with torch.no_grad():
            m.decoder.positional_embedding.normal_(0, 0.05)
        m = m.cuda().eval()
        mel = ob.log_mel_spectrogram(waveforms(1).cuda(), dims.n_mels)
        with torch.no_grad():
            xa = m.encoder(mel)[0]
        heads = m.alignment_heads.indices().T.tolist()
        blocks = m.decoder.blocks
        layers = sorted({l for l, _ in heads})
        print(f"\n{variant}: {len(heads)} alignment heads")
        for n_text in args.n_text:
            text = torch.randint(0, 50256, (n_text,), generator=torch.Generator().manual_seed(n_text)).tolist()

            def ours():
                cost, probs = T.alignment_cost(m, text, xa, num_frames)
                path, length = K.dtw(cost)
                host = torch.cat([length.float(), path.flatten().float(), probs]).cpu().numpy()
                t1 = time.perf_counter()
                n, w = int(host[0]), path.shape[1]
                T.words_from_path(_Tok(), text, host[1:1 + n].astype(np.int64), host[1 + w:1 + w + n].astype(np.int64),
                                  host[1 + 2 * w:].tolist())
                return (time.perf_counter() - t1) * 1e3

            def split():
                """Device time of each stage (separate event pairs)."""
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
                ev[0].record()
                cache, hooks = m.install_kv_cache_hooks()
                qs = {}
                qh = [blocks[l].cross_attn.query.register_forward_hook(lambda _m, _i, o, l=l: qs.__setitem__(l, o)) for l in layers]
                toks = torch.tensor([[50257, 50362, *text, 50256]], device="cuda")
                with torch.no_grad(), torch.autocast("cuda", torch.float16):
                    logits = m.decoder(toks, xa[None], kv_cache=cache)[0]
                    logits[1:n_text + 1, :50256].float().softmax(-1)
                for h in hooks + qh:
                    h.remove()
                ev[1].record()
                pairs = [(qs[l][0][:, h * 64:(h + 1) * 64], cache[blocks[l].cross_attn.key][0][:, h * 64:(h + 1) * 64])
                         for l, h in heads]
                cost = K.align_cost(pairs, num_frames // 2)
                ev[2].record()
                K.dtw(cost)
                ev[3].record()
                torch.cuda.synchronize()
                return [ev[i].elapsed_time(ev[i + 1]) for i in range(3)]

            def stock():
                t0 = time.perf_counter()
                cache, hooks = m.install_kv_cache_hooks()
                qs = {}
                qh = [blocks[l].cross_attn.query.register_forward_hook(lambda _m, _i, o, l=l: qs.__setitem__(l, o)) for l in layers]
                toks = torch.tensor([[50257, 50362, *text, 50256]], device="cuda")
                with torch.no_grad(), torch.autocast("cuda", torch.float16):
                    logits = m.decoder(toks, xa[None], kv_cache=cache)[0]
                for h in hooks + qh:
                    h.remove()
                with torch.no_grad():
                    qks = {l: {} for l in layers}
                    for l, h in heads:   # upstream's (q hd^-1/4)(k hd^-1/4)^T in fp16, then .float()
                        q = qs[l][0][:, h * 64:(h + 1) * 64] * 0.125 ** 0.5
                        k = cache[blocks[l].cross_attn.key][0][:, h * 64:(h + 1) * 64] * 0.125 ** 0.5
                        qks[l][h] = (q @ k.T).float()
                    matrix = OT.alignment_matrix(qks, heads, num_frames)
                    logits[1:n_text + 1, :50256].float().softmax(-1).cpu()
                    x = (-matrix).cpu().numpy()
                t1 = time.perf_counter()
                OT.dtw(x)
                return t1 - t0, time.perf_counter() - t1

            for _ in range(2):   # warm-up of every shape
                ours(), split(), stock()
            r_ours, r_split, r_stock = [], [], []
            for _ in range(args.rounds):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                host_ms = ours()
                r_ours.append(((time.perf_counter() - t0) * 1e3, host_ms))
                r_split.append(split())
                torch.cuda.synchronize()
                r_stock.append(stock())
            med = statistics.median
            fwd, cost_ms, dtw_ms = (med(s[i] for s in r_split) for i in range(3))
            print(f"  n_text={n_text:3d}: find_alignment {med(r[0] for r in r_ours):7.2f} ms "
                  f"(forward {fwd:.2f}, oasr_align_cost {cost_ms:.3f}, oasr_dtw {dtw_ms:.3f}, host words {med(r[1] for r in r_ours):.2f}) | "
                  f"stock torch device part {med(r[0] for r in r_stock) * 1e3:7.2f} ms + numpy DTW {med(r[1] for r in r_stock) * 1e3:8.1f} ms")
        seg = mel[0]
        decode(m, seg, DecodingOptions(beam_size=5, without_timestamps=False, sample_len=224))
        ms, _ = events_ms(lambda: decode(m, seg, DecodingOptions(beam_size=5, without_timestamps=False, sample_len=224)))
        print(f"  beam-5 decode of the window (timestamps, up to 224 tokens): {ms:.1f} ms")


class _Tok:
    def decode(self, ids):
        return "".join(f" w{i}" for i in ids)


if __name__ == "__main__":
    main()
