"""Per-shape GEMM table of the headline workload: one warm medium training step (16 clips, weight-gradient side stream
off) is run with kernels.GEMM_PROFILE on -- the same mechanism bench.py's roofline pass uses -- and its launches are
grouped by (M, N, K, a_mn, b_mn, epi, split_k, block_n).  Each distinct shape is then timed on its own with CUDA events
over a window of at least --window-ms, on seeded random operands.  One JSON object on stdout.

    python tools/time_gemm.py [--clips 16] [--window-ms 200] [--block-n W] [--fp8]

--block-n replaces every launch's tile width (0: keep what the step asked for), for tile-width comparisons.
--fp8 also profiles one step under fp8_autocast(): the shapes its FP8 launches have -- the block projections' forward
and dgrad, nothing else (the conv stem keeps bf16 GEMMs of similar shapes) -- are timed as kernels.gemm_fp8 with the FP8
tile picker, and the per-row quantisation of their A operand on its own; each such row gains fp8_ms_per_launch,
fp8_tflops, quantise_ms_per_launch and speedup (bf16 time over FP8 GEMM time), over the launches the FP8 step makes.
Select another build of the library with OASR_B200_LIB.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from collections import OrderedDict
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clk = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "clocks_max_sm": clk}
    except (OSError, ValueError, subprocess.TimeoutExpired):
        return {"name": torch.cuda.get_device_name(), "power_limit": None, "clocks_max_sm": None}


def profile_step(clips: int, fp8: bool = False):
    """Launch list of one warm medium training step (under fp8_autocast() with `fp8`): {shape key: launches}, in
    first-launch order."""
    import contextlib

    import olmoasr_b200 as ob
    from olmoasr_b200.fp8 import fp8_autocast
    from olmoasr_b200 import _core
    from olmoasr_b200 import kernels as K
    from olmoasr_b200 import synthetic as synth
    from olmoasr_b200.model import OLMoASR
    from olmoasr_b200.optim import FusedAdamW

    dev = torch.device("cuda", torch.cuda.current_device())
    torch.manual_seed(0)
    with torch.device(dev):
        model = OLMoASR(ob.VARIANT_TO_DIMS["medium"])
    slabs = model.use_slabs(direct_grads=True)
    opt = FusedAdamW(model.parameters(), lr=1.5e-3, betas=(0.9, 0.98), eps=1e-6, weight_decay=0.1, max_grad_norm=1.0, slabs=slabs)
    wav = synth.waveforms(clips, int16=True).to(dev)
    ti, ty, pm, _ = (t.to(dev) for t in synth.text_batch(clips))

    def step():
        with fp8_autocast() if fp8 else contextlib.nullcontext():
            loss = model(ob.log_mel_spectrogram(wav), ti, pm, targets=ty)
            opt.zero_grad()
            loss.backward()
        opt.step()

    _core.SIDE_STREAM = False
    step()
    torch.cuda.synchronize()
    K.GEMM_PROFILE = []
    step()
    torch.cuda.synchronize()
    prof, K.GEMM_PROFILE = K.GEMM_PROFILE, None
    groups = OrderedDict()
    for flops, e0, e1, key in prof:
        g = groups.setdefault(key, {"count": 0, "flops": flops, "step_ms": 0.0})
        g["count"] += 1
        g["step_ms"] += e0.elapsed_time(e1)
    del model, opt, slabs, prof
    torch.cuda.empty_cache()
    return groups


def _operand(rows, cols, gen):
    """bf16 (rows, cols) view with a row stride rounded up to 8 elements (TMA needs 16-byte strides)."""
    ld = (cols + 7) // 8 * 8
    return (torch.randn(rows, ld, device="cuda", generator=gen) * 0.05).bfloat16()[:, :cols]


def _time(run, window_ms):
    for _ in range(3):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    run()
    e1.record()
    torch.cuda.synchronize()
    reps = max(10, int(window_ms / max(e0.elapsed_time(e1), 1e-3)) + 1)
    e0.record()
    for _ in range(reps):
        run()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def fp8_launches(groups8):
    """(M, N, K, b_mn, epi) -> launches per step of the FP8 step's gemm_fp8 calls (an e5m2 A operand is a dgrad, whose
    bf16 form reads B MN-major)."""
    from olmoasr_b200 import kernels as K

    out = {}
    for key, g in groups8.items():
        if key[3] == "fp8":
            M, N, Kd, _, fmt, epi = key[:6]
            k = (M, N, Kd, int(fmt == K.FP8_E5M2), epi)
            out[k] = out.get(k, 0) + g["count"]
    return out


def time_shape_fp8(key, window_ms):
    """(FP8 GEMM ms, quantisation of A ms) of the FP8 form of `key` (A e5m2 for a dgrad, e4m3 for a forward)."""
    from olmoasr_b200 import _core
    from olmoasr_b200 import kernels as K

    M, N, Kd, a_mn, b_mn, epi, split_k, bn = key
    gen = torch.Generator(device="cuda").manual_seed(0)
    a16 = _operand(M, Kd, gen).contiguous()
    a8 = K.quantize_fp8_rows(a16, K.FP8_E5M2 if b_mn else K.FP8_E4M3)
    b8 = K.quantize_fp8_rows(_operand(N, Kd, gen).contiguous(), K.FP8_E4M3)
    out = torch.zeros(M, N, device="cuda", dtype=torch.bfloat16)
    out2 = torch.empty_like(out) if epi == K.EPI_BF16_GELU else None
    bias = None if b_mn else torch.randn(N, device="cuda", generator=gen)
    aux = _operand(M, N, gen).contiguous() if epi in (K.EPI_BF16_RESIDUAL, K.EPI_BF16_GELU_BWD) else None
    bn8 = _core._pick_block_n_fp8(M, N)
    ms = _time(lambda: K.gemm_fp8(a8[0], a8[1], b8[0], b8[1], M, N, Kd, out=out, out2=out2, bias=bias, aux=aux, epi=epi,
                                  block_n=bn8), window_ms)
    qms = _time(lambda: K.quantize_fp8_rows(a16, K.FP8_E5M2 if b_mn else K.FP8_E4M3), window_ms)
    return ms, qms, bn8


def time_shape(key, window_ms, block_n):
    from olmoasr_b200 import kernels as K

    M, N, Kd, a_mn, b_mn, epi, split_k, bn = key
    gen = torch.Generator(device="cuda").manual_seed(0)
    a = _operand(Kd, M, gen) if a_mn else _operand(M, Kd, gen)
    b = _operand(Kd, N, gen) if b_mn else _operand(N, Kd, gen)
    f32 = epi in (K.EPI_F32, K.EPI_F32_ATOMIC_ADD)
    out = torch.zeros(M, N, device="cuda", dtype=torch.float32 if f32 else torch.bfloat16)
    bias = torch.randn(N, device="cuda", generator=gen) if not f32 else None
    aux = _operand(M, N, gen) if epi in (K.EPI_BF16_RESIDUAL, K.EPI_BF16_GELU_BWD) else None
    if aux is not None:
        aux = aux.contiguous()

    def run():
        K.gemm(a, b, M, N, Kd, a_mn=bool(a_mn), b_mn=bool(b_mn), out=out, bias=bias, aux=aux, epi=epi, split_k=split_k,
               block_n=block_n or bn)

    for _ in range(3):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    run()
    e1.record()
    torch.cuda.synchronize()
    reps = max(10, int(window_ms / max(e0.elapsed_time(e1), 1e-3)) + 1)
    e0.record()
    for _ in range(reps):
        run()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    del a, b, out, bias, aux
    return ms, reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=16)
    ap.add_argument("--window-ms", type=float, default=200.0)
    ap.add_argument("--block-n", type=int, default=0)
    ap.add_argument("--fp8", action="store_true")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "time_gemm.py measures on a CUDA device"
    from olmoasr_b200 import _lib

    groups = profile_step(args.clips)
    f8 = fp8_launches(profile_step(args.clips, fp8=True)) if args.fp8 else {}
    rows = []
    for key, g in groups.items():
        ms, reps = time_shape(key, args.window_ms, args.block_n)
        rows.append({"M": key[0], "N": key[1], "K": key[2], "a_mn": key[3], "b_mn": key[4], "epi": key[5], "split_k": key[6],
                     "block_n": args.block_n or key[7], "count": g["count"], "ms_per_launch": ms, "reps": reps,
                     "ms_per_step": ms * g["count"], "tflops": g["flops"] / (ms * 1e-3) / 1e12,
                     "in_step_ms_per_step": g["step_ms"]})
        n8 = f8.get((key[0], key[1], key[2], key[4], key[5]), 0) if not key[3] and key[6] == 1 else 0
        if n8:
            ms8, qms, bn8 = time_shape_fp8(key, args.window_ms)
            rows[-1].update({"fp8_count": n8, "fp8_ms_per_launch": ms8, "fp8_block_n": bn8,
                             "fp8_tflops": g["flops"] / (ms8 * 1e-3) / 1e12, "quantise_ms_per_launch": qms,
                             "speedup": ms / ms8})
    total = sum(r["ms_per_step"] for r in rows)
    for r in rows:
        r["share"] = r["ms_per_step"] / total
    rows.sort(key=lambda r: -r["ms_per_step"])
    flops = sum(g["flops"] * g["count"] for g in groups.values())
    extra = {}
    if args.fp8:
        r8 = [r for r in rows if "fp8_ms_per_launch" in r]     # the projections' launches only
        extra = {"fp8_launches": sum(f8.values()), "fp8_launches_matched": sum(r["fp8_count"] for r in r8),
                 "fp8_shapes_bf16_ms_per_step": sum(r["ms_per_launch"] * r["fp8_count"] for r in r8),
                 "fp8_shapes_fp8_ms_per_step": sum(r["fp8_ms_per_launch"] * r["fp8_count"] for r in r8),
                 "fp8_shapes_quantise_ms_per_step": sum(r["quantise_ms_per_launch"] * r["fp8_count"] for r in r8)}
    print(json.dumps({**extra, "gpu": gpu_info(), "library": str(_lib.lib_path()), "clips": args.clips, "block_n_override": args.block_n,
                      "gemm_ms_per_step": total, "gemm_tflops": flops / (total * 1e-3) / 1e12,
                      "in_step_gemm_ms": sum(g["step_ms"] for g in groups.values()), "shapes": rows}))


if __name__ == "__main__":
    main()
