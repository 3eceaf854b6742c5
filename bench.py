"""Headline benchmark: training throughput in 30 s-clips/s (BASELINE.json metric) for the waveform -> log-mel ->
encoder/decoder fwd+bwd -> token CE -> (DDP all-reduce) -> clip + AdamW step.

    python bench.py --gpus 1 --steps 5 --warmup 3                     # our arm (one process per GPU; torchrun for N > 1)
    python bench.py --impl reference --gpus 1 --steps 2 --warmup 1    # the reference's CPU path (oracle port) on host cores

One JSON line on stdout (rank 0).
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

TRAIN_GFLOP_PER_CLIP = {"tiny": 213.2, "base": 453.2, "small": 1629.8, "medium": 5214.4, "large": 10342.1}  # BASELINE.md section 2
METRIC = "30s-clips/sec training"


def _peaks():
    path = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(path):
        with open(path) as f:
            p = json.load(f)
        return {"bf16_tflops": p["bf16_tflops"], "bf16_tflops_sustained": p["bf16_tflops_sustained"], "hbm_gbs": p["hbm_gbs"],
                "source": "MEASURED_PEAKS.json"}
    # NVIDIA H100 SXM data sheet (700 W board power): dense BF16 and HBM3 bandwidth.  Data-sheet rates, not measured ones.
    return {"bf16_tflops": 989.0, "bf16_tflops_sustained": 989.0, "hbm_gbs": 3350.0, "source": "H100 SXM data sheet"}


# ------------------------------------------------------------------------------------------------------------------
# reference arm / cpu_baseline: the reference's own CPU PyTorch path (restated in oracle/, pinned bit-exact to it)
# ------------------------------------------------------------------------------------------------------------------
def usable_cpus() -> int:
    """Cores this process may actually use: affinity mask capped by the cgroup CPU quota (a 128-thread pool on a
    16-core quota is an order of magnitude slower than 16 threads)."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    try:
        with open("/sys/fs/cgroup/cpu.max") as f:
            quota, period = f.read().split()
        if quota != "max":
            n = min(n, max(1, int(int(quota) / int(period))))
    except (OSError, ValueError):
        pass
    return max(1, n)


def run_cpu_reference(variant: str, clips: int, steps: int, warmup: int, layers=None):
    """The reference's CPU PyTorch path (oracle port, bit-identical model code): fp32, all usable host cores:
    log-mel (numpy) -> model fwd -> CE -> bwd -> clip_grad_norm_ -> AdamW, `clips` clips per step.
    `layers=(Le, Ld)` truncates the encoder / decoder depth (used for the bounded, extrapolated sample)."""
    from dataclasses import replace

    from oracle import logmel
    from oracle import model as OM
    from olmoasr_b200 import synthetic as synth

    threads = usable_cpus()
    torch.set_num_threads(threads)
    dims = OM.variant_dims(variant)
    if layers is not None:
        dims = replace(dims, n_audio_layer=layers[0], n_text_layer=layers[1])
    sd = OM.init_state_dict(dims, seed=0, train=True)
    params = {k: v.requires_grad_(k != "encoder.positional_embedding") for k, v in sd.items()}
    opt = torch.optim.AdamW([p for p in params.values() if p.requires_grad], lr=1.5e-3, betas=(0.9, 0.98), eps=1e-6, weight_decay=0.1)
    wav = synth.waveforms(clips).numpy()
    ti, ty, pm, _ = synth.text_batch(clips)

    def step():
        mel = torch.from_numpy(logmel.log_mel_spectrogram(wav))
        loss = OM.token_ce(OM.model_forward(params, dims, mel, ti, pm, train_model=True), ty)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        torch.nn.utils.clip_grad_norm_([p for p in params.values() if p.requires_grad], 1.0)
        opt.step()
        return float(loss.detach())

    for _ in range(warmup):
        step()
    t0 = time.perf_counter()
    for _ in range(steps):
        step()
    dt = time.perf_counter() - t0
    return clips * steps / dt, dt / steps, threads


def bounded_cpu_sample(variant: str, steps: int = 2, warmup: int = 1):
    """A bounded sample of the workload on the host cores: REAL full-depth optimizer steps of the reference's CPU path
    on ONE clip (the GPU arm's step is --batch-per-gpu clips), nothing extrapolated.  Returns (clips/s, threads, description, seconds per step, steps run)."""
    value, sec, threads = run_cpu_reference(variant, 1, steps, warmup)
    return value, threads, (f"{steps} full-depth optimizer steps of 1 clip each after {warmup} warm-up step(s): {variant}, fp32, torch CPU, "
                            f"{threads} threads, log-mel + fwd + CE + bwd + clip + AdamW ({sec:.2f} s per step)"), sec, steps


def reference_arm(args):
    """`--impl reference`: the reference's own CPU implementation of the path (oracle port, bit-identical model code) on the
    host cores.  Every step is a real full-depth step on a bounded sample (1 clip); at most 3 timed steps and 1 warm-up
    are run whatever --steps / --warmup say, and the line reports the counts actually executed."""
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    steps = max(1, min(args.steps, 3))
    warmup = max(0, min(args.warmup, 1))
    value, threads, sample, sec, _ = bounded_cpu_sample(args.variant, steps, warmup)
    line = {
        "impl": "reference", "metric": METRIC, "value": value, "unit": "clips/s", "n_gpus": args.gpus, "steps": steps,
        "warmup": warmup, "steps_requested": args.steps, "warmup_requested": args.warmup,
        "ms_per_step": sec * 1e3, "higher_is_better": True, "scaling": "weak",
        "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": {"workload": f"{args.variant} training step, 30 s synthetic clips (reference CPU path, 1 clip per step)",
                   "global_batch": 1, "parallelism": "cpu"},
        "cpu_baseline": {"value": value, "unit": "clips/s", "cores": threads, "kind": "port", "sample": sample},
        "e2e": {"value": value, "unit": "clips/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }
    print(json.dumps(line), flush=True)


# ------------------------------------------------------------------------------------------------------------------
class ClockSampler:
    """nvidia-smi clock / throttle-reason samples during the timed region (read-only queries)."""

    FIELDS = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.active,clocks_event_reasons.hw_slowdown,"
              "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, gpu_index: int):
        self.proc = None
        self.lines = []
        self.gpu_index = gpu_index

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.FIELDS}", "--format=csv,noheader,nounits", "-lms", "200",
                                          "-i", str(self.gpu_index)], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.thread = threading.Thread(target=self._read, daemon=True)
            self.thread.start()
        except OSError:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.lines.append(line.strip())

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=5)
        except subprocess.TimeoutExpired:
            self.proc.kill()
        sm, mx, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for ln in self.lines:
            f = [x.strip() for x in ln.split(",")]
            if len(f) < 9:
                continue
            try:
                sm.append(float(f[1])); mx.append(float(f[2]))
            except ValueError:
                continue
            for n, v in zip(names, f[5:9]):
                if v.lower().startswith("active"):
                    reasons.add(n)
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": max(mx) if mx else None, "reasons": sorted(reasons),
                "samples": len(sm)}


def _setup_dist():
    import torch.distributed as dist

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1 and not dist.is_initialized():
        dist.init_process_group("nccl", device_id=dev)
    return world, rank, local_rank, dev


def gpu_baseline_leg(args, world, rank, dev, steps=None):
    """The reference's GPU path (stock PyTorch: cuBLASLt / cuDNN / ATen SDPA, autocast bf16, DDP, clip_grad_norm_, fused
    torch AdamW) on the same synthetic batch, same box, same N -- the denominator north_star names.  Run after our own
    arm has released its memory."""
    import gc

    from baseline import torch_stock

    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    steps = steps or max(2, min(args.steps, 5))
    B = args.batch_per_gpu
    note = ""
    try:
        r = torch_stock.run(args.variant, B, steps, 2, dev, rank=rank, world=world)
    except torch.OutOfMemoryError:
        gc.collect()
        torch.cuda.empty_cache()
        note = f"out of memory at {B} clips per GPU"
        return {"value": None, "unit": "clips/s", "impl": "stock PyTorch", "unavailable": note}
    return {"value": r["clips_per_s"], "unit": "clips/s", "ms_per_step": r["ms_per_step"], "steps": steps, "warmup": 2,
            "impl": f"stock PyTorch {torch.__version__} (baseline/torch_stock.py): nn.Linear / Conv1d / fp32 F.layer_norm / "
                    "F.scaled_dot_product_attention with the dense float mask / fp32 logits + F.cross_entropy, autocast bf16, "
                    + ("DistributedDataParallel, " if world > 1 else "") + "clip_grad_norm_ + fused torch.optim.AdamW; log-mel by "
                    "torch.stft on the GPU (the reference computes it in CPU workers, outside its step time)",
            "clips_per_gpu": B, "loss": r["loss"], "peak_mem_gib": r["peak_mem_gib"]}


def torch_gpu_arm(args):
    """`--impl torch_gpu`: the stock-PyTorch GPU arm alone, same JSON shape."""
    import torch.distributed as dist

    world, rank, local_rank, dev = _setup_dist()
    g = gpu_baseline_leg(args, world, rank, dev, steps=args.steps)
    if rank == 0:
        line = {"impl": "torch_gpu", "metric": METRIC, "value": g.get("value"), "unit": "clips/s", "n_gpus": world,
                "steps": g.get("steps"), "warmup": g.get("warmup"), "ms_per_step": g.get("ms_per_step"), "higher_is_better": True,
                "scaling": "weak", "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
                "config": {"workload": f"{args.variant} model DDP training bf16, {args.batch_per_gpu} x 30 s synthetic clips per GPU",
                           "global_batch": args.batch_per_gpu * world, "parallelism": f"dp{world}"},
                "gpu_baseline": g}
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()


DUMP_SAMPLE = 1 << 21   # elements per sampled slab: 2 x 8 MB of float32


def dump_outputs(out_dir: str, loss: float, slabs) -> None:
    """What a caller of the training step holds after the last timed step: its loss, the updated fp32 master weights and
    the gradients it applied.  The slabs hold ~10^9 elements, so both are sampled at the same fixed, seeded positions
    (identical from run to run and build to build for the same --variant)."""
    import numpy as np

    os.makedirs(out_dir, exist_ok=True)
    gen = torch.Generator().manual_seed(20240607)
    n = slabs.P.numel()
    idx = torch.randint(0, n, (min(DUMP_SAMPLE, n),), generator=gen).sort().values.to(slabs.P.device)
    np.save(os.path.join(out_dir, "loss.npy"), np.array([loss], dtype=np.float64))
    np.save(os.path.join(out_dir, "weights_sample.npy"), slabs.P[idx].float().cpu().numpy())
    np.save(os.path.join(out_dir, "grads_sample.npy"), slabs.G[idx].float().cpu().numpy())


def our_arm(args):
    import torch.distributed as dist

    import olmoasr_b200 as ob
    from olmoasr_b200 import _lib
    from olmoasr_b200 import kernels as K
    from olmoasr_b200.model import OLMoASR
    from olmoasr_b200.optim import FusedAdamW
    from olmoasr_b200 import synthetic as synth

    world, rank, local_rank, dev = _setup_dist()
    assert world == args.gpus, f"--gpus {args.gpus} but WORLD_SIZE={world} (launch with torch.distributed.run)"

    dims = ob.VARIANT_TO_DIMS[args.variant]
    B = args.batch_per_gpu
    torch.manual_seed(0)
    with torch.device(dev):
        model = OLMoASR(dims)
    net = model
    sync = None
    # gradient synchronisation: "slab" (default) = olmoasr_b200.ddp.SlabGradSync over the flat gradient slab;
    # "torch" = torch DistributedDataParallel (the reference's wrapper) for A/B runs
    ddp_impl = os.environ.get("OASR_DDP_IMPL", "slab")
    slabs = model.use_slabs(direct_grads=(ddp_impl == "slab"))
    if world > 1 and ddp_impl == "slab":
        from olmoasr_b200.ddp import SlabGradSync
        sync = SlabGradSync(model, slabs, bucket_bytes=int(os.environ.get("OASR_BUCKET_MB", "256")) << 20,
                            tail_bucket_bytes=int(os.environ.get("OASR_TAIL_BUCKET_MB", "32")) << 20)
    elif world > 1:
        net = torch.nn.parallel.DistributedDataParallel(model, device_ids=[local_rank], output_device=local_rank)
        slabs.invalidate()      # DDP's constructor broadcast rank 0's weights into the masters behind autograd's back
    opt = FusedAdamW(model.parameters(), lr=1.5e-3, betas=(0.9, 0.98), eps=1e-6, weight_decay=0.1, max_grad_norm=1.0, slabs=slabs)

    # synthetic batch of SURVEY.md 8(d); host copies are pinned (what a DataLoader with pin_memory hands over)
    wav_h = synth.waveforms(B, rank=rank, int16=True).pin_memory()
    ti_h, ty_h, pm_h, _ = synth.text_batch(B, rank=rank)
    ti_h, ty_h, pm_h = ti_h.pin_memory(), ty_h.pin_memory(), pm_h.pin_memory()
    h2d_bytes = sum(t.numel() * t.element_size() for t in (wav_h, ti_h, ty_h, pm_h))
    dev_in = [t.to(dev) for t in (wav_h, ti_h, ty_h, pm_h)]

    def train_step(wav, ti, ty, pm):
        mel = ob.log_mel_spectrogram(wav)
        loss = net(mel, ti, pm, targets=ty)
        opt.zero_grad()
        loss.backward()
        opt.step(inv_scale=sync.finish() if sync is not None else 1.0)
        return loss.detach()

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def timed(n_steps, e2e):
        barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record()
        last = None
        for _ in range(n_steps):
            if e2e:
                ins = [t.to(dev, non_blocking=True) for t in (wav_h, ti_h, ty_h, pm_h)]
                last = train_step(*ins).item()  # device->host read of the step's loss, every step
            else:
                last = train_step(*dev_in)
        e1.record()
        barrier()
        ms = e0.elapsed_time(e1)
        wall_ms = (time.perf_counter() - t0) * 1e3
        ms = max(ms, wall_ms) if e2e else ms
        if world > 1:
            t = torch.tensor([ms], device=dev)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            ms = float(t.item())
        return ms, (last if e2e else float(last.item()))

    for _ in range(args.warmup):
        train_step(*dev_in)
    torch.cuda.synchronize()

    sampler = ClockSampler(local_rank)
    if rank == 0:
        sampler.start()
    launches0 = _lib.LAUNCH_COUNT
    ms, loss = timed(args.steps, e2e=False)
    launches = _lib.LAUNCH_COUNT - launches0
    clocks = sampler.stop() if rank == 0 else None
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, loss, slabs)
    ms_e2e, loss_e2e = timed(args.steps, e2e=True)
    # roofline pass: the same K steps with every GEMM launch bracketed by CUDA events.  The weight-gradient side stream
    # is switched off for this pass so that launches do not overlap and a launch's event time is its own duration.
    from olmoasr_b200 import _core
    side_prev, _core.SIDE_STREAM = _core.SIDE_STREAM, False
    K.GEMM_PROFILE = []
    ms_serial, _ = timed(args.steps, e2e=False)
    prof, K.GEMM_PROFILE = K.GEMM_PROFILE, None
    _core.SIDE_STREAM = side_prev
    gemm_flops = sum(p[0] for p in prof)
    gemm_ms = sum(p[1].elapsed_time(p[2]) for p in prof)
    n_gemm = len(prof)
    applied = opt.applied_steps()
    peak_mem = torch.cuda.max_memory_allocated() / 2**30

    # release everything of ours before the stock-PyTorch leg
    if sync is not None:
        sync.remove()
    del prof, net, model, opt, slabs, sync, dev_in
    gpu_base = None
    if not args.no_gpu_baseline:
        gpu_base = gpu_baseline_leg(args, world, rank, dev)

    if rank != 0:
        if world > 1:
            dist.destroy_process_group()
        return
    global_batch = B * world
    value = global_batch * args.steps / (ms / 1e3)
    e2e_value = global_batch * args.steps / (ms_e2e / 1e3)
    peaks = _peaks()
    gemm_tflops = gemm_flops / (gemm_ms / 1e3) / 1e12 if gemm_ms > 0 else 0.0
    step_tflops = value * TRAIN_GFLOP_PER_CLIP[args.variant] / 1e3 / world
    line = {
        "metric": METRIC, "value": value, "unit": "clips/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "bf16",
        "data": "synthetic",
        "config": {"workload": f"{args.variant} model DDP training bf16, {B} x 30 s synthetic clips per GPU "
                               f"(BASELINE.json configs[2] at {world} GPU(s)): int16 waveform -> log-mel -> fwd/bwd -> CE -> "
                               f"{'NCCL all-reduce -> ' if world > 1 else ''}clip + AdamW",
                   "global_batch": global_batch, "parallelism": f"dp{world}",
                   "grad_sync": ("none" if world == 1 else ("olmoasr_b200.ddp.SlabGradSync (flat fp32 gradient slab, segment all-reduces)"
                                                            if ddp_impl == "slab" else "torch DistributedDataParallel")),
                   "state_layout": "parameter / gradient / moment / bf16-shadow slabs (olmoasr_b200/slab.py); AdamW refreshes the bf16 weights",
                   "l2": "no flush needed: the per-step working set (tens of GB of activations) is >> the 50 MB L2",
                   "loss": loss, "optimizer_steps_applied": applied, "peak_mem_gib": peak_mem},
        "e2e": {"value": e2e_value, "unit": "clips/s", "h2d_bytes_per_step": h2d_bytes, "d2h_bytes_per_step": 4,
                "ms_per_step": ms_e2e / args.steps, "loss": loss_e2e},
        "gpu_launches": launches,
        "clocks": clocks,
        "roofline": {"bound": "tensor", "kernel": "gemm_wgmma_kernel (all GEMM launches of K steps)",
                     "achieved": gemm_tflops, "peak": peaks["bf16_tflops_sustained"], "unit": "TFLOP/s",
                     "frac": gemm_tflops / peaks["bf16_tflops_sustained"], "traffic": None,
                     "peak_source": peaks["source"] + " (sustained: kernel timed inside a long step)",
                     "measured_in": "a second pass of the same K steps with the weight-gradient side stream off (launches "
                                    "serialised, so each launch's CUDA-event time is its own duration)",
                     "serial_ms_per_step": ms_serial / args.steps,
                     "gemm_share_of_step": gemm_ms / ms_serial, "gemm_launches": n_gemm,
                     "whole_step_tflops_per_gpu": step_tflops, "whole_step_frac": step_tflops / peaks["bf16_tflops_sustained"]},
    }
    if gpu_base is not None:
        line["gpu_baseline"] = gpu_base
        if gpu_base.get("value"):
            line["gpu_baseline"]["ours_over_stock"] = value / gpu_base["value"]
    if world == 1 and not args.no_cpu_baseline:
        v, threads, sample, _, _ = bounded_cpu_sample(args.variant)
        line["cpu_baseline"] = {"value": v, "unit": "clips/s", "cores": threads, "kind": "port", "sample": sample}
    print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()


# ------------------------------------------------------------------------------------------------------------------
# second half of BASELINE.json's metric: greedy-decode real-time factor (config 5: small, kv-cache decode, 1 GPU,
# 1..64 concurrent 30 s clips; scripts/eval/eval.py:1846-1847 calls model.decode(mel, DecodingOptions(language="en",
# without_timestamps=True)) -> up to n_text_ctx // 2 = 224 sampled tokens per clip)
# ------------------------------------------------------------------------------------------------------------------
RTF_METRIC = "greedy-decode RTF"
RTF_BATCHES = (1, 2, 4, 8, 16, 32, 64)


def cpu_decode_reference(variant: str, n_clips: int = 1, sample_len: int = 224):
    """The reference's CPU path for config 5 (oracle port of inf_model.py + the upstream greedy loop), fp32, all host
    threads: log-mel + encoder + `sample_len` kv-cache steps for `n_clips` clips.  Returns (RTF, seconds, threads)."""
    from oracle import decoding as OD
    from oracle import logmel
    from oracle import model as OM
    from olmoasr_b200 import synthetic as synth

    threads = usable_cpus()
    torch.set_num_threads(threads)
    dims = OM.variant_dims(variant)
    sd = OM.init_state_dict(dims, 0, train=False)
    sd["decoder.positional_embedding"] = torch.randn(dims.n_text_ctx, dims.n_text_state, generator=torch.Generator().manual_seed(7)) * 0.01
    wav = synth.waveforms(n_clips).numpy()
    t0 = time.perf_counter()
    with torch.no_grad():
        mel = torch.from_numpy(logmel.log_mel_spectrogram(wav))
        OD.greedy_decode(sd, dims, mel, sample_len=sample_len, dtype=torch.float32)
    sec = time.perf_counter() - t0
    return sec / (n_clips * 30.0), sec, threads


def rtf_reference_arm(args):
    if int(os.environ.get("RANK", "0")) != 0:
        return
    rtf, sec, threads = cpu_decode_reference(args.variant_rtf, 1, 224)
    line = {"impl": "reference", "metric": RTF_METRIC, "value": rtf, "unit": "s per s of audio", "n_gpus": args.gpus, "steps": 1,
            "warmup": 0, "steps_requested": args.steps, "ms_per_step": sec * 1e3, "higher_is_better": False, "scaling": "weak",
            "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": {"workload": f"{args.variant_rtf} greedy kv-cache decode of 1 x 30 s synthetic clip, 224 sampled tokens (reference CPU path)",
                       "parallelism": "cpu"},
            "cpu_baseline": {"value": rtf, "unit": "s per s of audio", "cores": threads, "kind": "port",
                             "sample": f"1 clip, log-mel + encoder + 224 greedy steps, fp32, {threads} threads ({sec:.1f} s)"},
            "e2e": {"value": rtf, "unit": "s per s of audio", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
    print(json.dumps(line), flush=True)


def rtf_arm(args):
    """`--metric rtf`: the RTF sweep on one GPU.  A "step" here is one complete decode of N concurrent clips (int16
    waveform in pinned host memory -> H2D -> log-mel -> encoder -> cross K/V -> 1 + 224 graph replays -> token ids D2H)."""
    import olmoasr_b200 as ob
    from olmoasr_b200 import _lib
    from olmoasr_b200 import synthetic as synth
    from olmoasr_b200.decoding import DecodingOptions, DecodingTask
    from olmoasr_b200.inf_model import OLMoASR

    world, rank, local_rank, dev = _setup_dist()
    variant = args.variant_rtf
    dims = ob.VARIANT_TO_DIMS[variant]
    torch.manual_seed(0)
    with torch.device(dev):
        model = OLMoASR(dims)
    with torch.no_grad():
        model.decoder.positional_embedding.normal_(0, 0.01)   # inf_model.py:307 leaves it uninitialised (checkpoints fill it)
    dtype = torch.float16 if args.dtype == "fp16" else torch.bfloat16
    eng = model.decode_engine(dtype)
    opts = DecodingOptions(language="en", without_timestamps=True, fp16=(dtype == torch.float16))
    task = DecodingTask(model, opts)
    sample_len = task.sample_len
    peaks = _peaks()
    sweep = []
    sampler = ClockSampler(local_rank)
    sampler.start()
    launches0 = _lib.LAUNCH_COUNT
    for n in RTF_BATCHES:
        wav_h = synth.waveforms(n, rank=rank, int16=True).pin_memory()

        def full_decode():
            wav = wav_h.to(dev, non_blocking=True)
            mel = ob.log_mel_spectrogram(wav)
            with torch.no_grad():
                xa = model.encoder(mel)
            toks, lps, nsp, replays = eng.greedy(xa, task.initial_tokens, sample_len, task.suppress, opts.suppress_blank, task.sot_index)
            return toks, replays

        for _ in range(max(1, min(args.warmup, 2))):
            full_decode()
        torch.cuda.synchronize()
        reps = max(1, min(args.steps, 3))
        t0 = time.perf_counter()
        for _ in range(reps):
            toks, replays = full_decode()       # ends with a D2H copy of the token ids: wall clock covers everything
        wall = (time.perf_counter() - t0) / reps
        # the replay loop alone (device time): graph replays back to back from a prepared state
        eng.reset(n, torch.tensor([list(task.initial_tokens)], dtype=torch.int32).repeat(n, 1), None, task.suppress, opts.suppress_blank, task.sot_index)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(replays):
            eng.replay(n)
        e1.record()
        torch.cuda.synchronize()
        step_ms = e0.elapsed_time(e1) / replays
        t_mid = len(task.initial_tokens) + sample_len // 2
        gbs = eng.step_bytes(n, t_mid) / (step_ms * 1e-3) / 1e9
        sweep.append({"n_clips": n, "rtf": wall / (n * 30.0), "wall_s": wall, "replays": replays, "ms_per_step": step_ms,
                      "step_gb": eng.step_bytes(n, t_mid) / 1e9, "hbm_gbs": gbs, "hbm_frac": gbs / peaks["hbm_gbs"],
                      "tokens_per_s": n * 1e3 / step_ms})
    launches = _lib.LAUNCH_COUNT - launches0
    clocks = sampler.stop()
    best = sweep[-1]
    line = {"metric": RTF_METRIC, "value": best["rtf"], "unit": "s per s of audio", "n_gpus": 1, "steps": max(1, min(args.steps, 3)),
            "warmup": max(1, min(args.warmup, 2)), "ms_per_step": best["wall_s"] * 1e3, "higher_is_better": False, "scaling": "weak",
            "vs_baseline": None, "dtype": args.dtype, "data": "synthetic",
            "config": {"workload": f"{variant} greedy kv-cache decode (BASELINE.json configs[4]): N concurrent 30 s synthetic clips, "
                                   f"{sample_len} sampled tokens each (random-init weights never emit eot), value = RTF at N = {best['n_clips']}",
                       "sweep": sweep, "launches_per_decode_step": eng.launches_per_step,
                       "l2": "every step re-reads the decoder weights (278 MB) and N x 55 MB of cross K/V: > 50 MB L2 from N = 1"},
            "e2e": {"value": best["rtf"], "unit": "s per s of audio", "h2d_bytes_per_step": best["n_clips"] * 480000 * 2,
                    "d2h_bytes_per_step": best["n_clips"] * (len(task.initial_tokens) + sample_len) * 8},
            "gpu_launches": launches, "clocks": clocks,
            "roofline": {"bound": "hbm", "kernel": "decode step (dec_linear / dec_attn_scores / dec_attn_pv / dec_sample graph replay)",
                         "achieved": best["hbm_gbs"], "peak": peaks["hbm_gbs"], "unit": "GB/s", "frac": best["hbm_frac"], "traffic": None,
                         "peak_source": peaks["source"], "algorithmic_bytes": "weights once + per sequence cross K/V of every layer + "
                                                                                "self K/V so far + fp32 logits row (SURVEY.md 8(d))"}}
    if not args.no_cpu_baseline:
        rtf, sec, threads = cpu_decode_reference(variant, 1, 224)
        line["cpu_baseline"] = {"value": rtf, "unit": "s per s of audio", "cores": threads, "kind": "port",
                                "sample": f"1 clip, log-mel + encoder + 224 greedy steps, fp32, {threads} threads ({sec:.1f} s)"}
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference", "torch_gpu"])
    ap.add_argument("--variant", default="medium", choices=list(TRAIN_GFLOP_PER_CLIP))
    # 16 clips of the medium model fit the 80 GB of an H100 with room for the stock-PyTorch leg that follows
    ap.add_argument("--batch-per-gpu", type=int, default=16)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-gpu-baseline", action="store_true")
    ap.add_argument("--metric", default="train", choices=["train", "rtf"], help="train: clips/s (default); "
                    "rtf: greedy-decode real-time factor sweep (BASELINE.json metric, second half)")
    ap.add_argument("--variant-rtf", default="small")
    ap.add_argument("--dtype", default="fp16", choices=["fp16", "bf16"], help="decode activation dtype for --metric rtf")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="train arm: after the timed steps write what the last timed step computed to DIR/<name>.npy "
                         "(loss, and fixed seeded samples of the updated fp32 weights and of the gradients)")
    args = ap.parse_args()
    if args.metric == "rtf":
        (rtf_reference_arm if args.impl == "reference" else rtf_arm)(args)
    elif args.impl == "reference":
        reference_arm(args)
    elif args.impl == "torch_gpu":
        torch_gpu_arm(args)
    else:
        our_arm(args)


if __name__ == "__main__":
    main()
