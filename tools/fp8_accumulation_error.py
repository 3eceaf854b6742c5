"""How far the FP8 GEMM's accumulation is from fp64, in units of sum |a b|: the figure behind FP8_ACC in
tests/test_fp8_gpu.py.

    python tools/fp8_accumulation_error.py [--k 1024 4096] [--out DIR]
    OASR_B200_LIB=olmoasr_b200/csrc/_ab/nopromote.so python tools/fp8_accumulation_error.py   # the unpromoted sum

(the second library: python -m olmoasr_b200.build --variant nopromote -DOASR_FP8_NO_PROMOTE).  For each K, the
operands of tests/test_fp8_gpu.py's K = 4096 case (M = 1024, N = 1280, randn rows quantised to e4m3 per row) go through
kernels.gemm_fp8 (bf16 output) and through the fp64 product of the dequantised operands.  Per element, what the bf16
output's one ulp and the fp32 stage bound of tests/training_reference.py do not explain, over sum_k |a b|, is the
accumulation's own relative error; its maximum is the smallest FP8_ACC the test's rule 1 accepts.  One JSON line, with
the card read in the same call.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--k", type=int, nargs="+", default=[1024, 4096])
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fp8_accumulation_error.py measures on a CUDA device; none is available")
    from olmoasr_b200 import _lib
    from olmoasr_b200 import kernels as K
    from tests import training_reference as tr

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    res = {"library": str(_lib.lib_path()), "card": card, "k": {}}
    for Kd in args.k:
        g = torch.Generator(device="cuda").manual_seed(Kd)
        M, N = 1024, 1280
        a8 = K.quantize_fp8_rows((torch.randn((M, Kd), device="cuda", generator=g)).bfloat16(), K.FP8_E4M3)
        b8 = K.quantize_fp8_rows((torch.randn((N, Kd), device="cuda", generator=g) * Kd ** -0.5).bfloat16(), K.FP8_E4M3)
        got = K.gemm_fp8(a8[0], a8[1], b8[0], b8[1], M, N, Kd).double()
        A = a8[0].double() * a8[1].double()[:, None]
        B = b8[0].double() * b8[1].double()[:, None]
        ref = A @ B.t()
        mag = A.abs() @ B.abs().t()
        r16 = tr.rnd(ref, torch.bfloat16)
        explained = tr.ulp(torch.maximum(got.abs(), r16.abs()), torch.bfloat16) + tr.gemm_stages(Kd) * 2.0 ** -23 * mag
        excess = ((got - r16).abs() - explained).clamp_min(0) / mag
        res["k"][Kd] = {"max_excess_over_sum_abs": float(excess.max()), "mean_abs_err_over_sum_abs": float(((got - ref).abs() / mag).mean()),
                        "max_abs_err_over_sum_abs": float(((got - ref).abs() / mag).max())}
    line = json.dumps(res)
    print(line)
    if args.out:
        Path(args.out).mkdir(parents=True, exist_ok=True)
        (Path(args.out) / ("fp8_accumulation_error_" + Path(res["library"]).stem + ".json")).write_text(line + "\n")


if __name__ == "__main__":
    main()
