"""Regenerate the kernel / yardstick error-ratio table of tests/attention_reference.py on a GPU:

    python tools/attention_error_table.py [extra pytest arguments]

runs tests/test_attention_parity_gpu.py with OASR_ATTN_REPORT pointing at a temporary file, then prints, per case
group, dtype and tensor, the largest max-row and mean-row ratios that attention_reference.check() measured, and the
largest lse error in LSE_TOL units.  Re-run it after an attention kernel change before touching ALPHA or BETA."""
import collections
import json
import os
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
GROUPS = {"test_production_shapes": "production", "test_medium_bench_shape": "production",
          "test_kv_len_on_tile_edges": "mask edges", "test_ragged_lengths": "mask edges",
          "test_kv_len_without_causal": "mask edges", "test_kv_len_clamps": "mask edges",
          "test_score_regimes": "score regimes", "test_uniform_softmax_is_the_mean_of_v": "score regimes",
          "test_non_default_scale": "scale"}


def main():
    with tempfile.TemporaryDirectory() as tmp:
        report = os.path.join(tmp, "report.jsonl")
        env = dict(os.environ, OASR_ATTN_REPORT=report)
        cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider",
               "tests/test_attention_parity_gpu.py", *sys.argv[1:]]
        rc = subprocess.call(cmd, cwd=ROOT, env=env)
        lines = Path(report).read_text().splitlines() if os.path.exists(report) else []
    worst = collections.defaultdict(lambda: [0.0, 0.0])
    lse, power = 0.0, float("inf")
    for line in lines:
        rec = json.loads(line)
        test = rec["test"].split("::")[-1].split("[")[0]
        if test == "test_check_catches_an_off_by_one_kv_len" and rec["kind"] == "rows":
            power = min(power, max(rec["worst_ratio"], rec["mean_ratio"]))
        group = GROUPS.get(test)
        if group is None:             # the power test and the bit-exact tests are not calibration cases
            continue
        if rec["kind"] == "lse":
            lse = max(lse, rec["lse_tol_units"])
            continue
        w = worst[(group, rec["dtype"], rec["name"])]
        w[0], w[1] = max(w[0], rec["worst_ratio"]), max(w[1], rec["mean_ratio"])
    print(f"\n    {'group':16} dtype   " + "  ".join(f"{t:11}" for t in ("O", "dQ", "dK", "dV")))
    for group in dict.fromkeys(GROUPS.values()):
        for dt in ("bfloat16", "float16"):
            cells = "  ".join(f"{worst[(group, dt, t)][0]:.2f} / {worst[(group, dt, t)][1]:.2f}" for t in ("o", "dq", "dk", "dv"))
            print(f"    {group if dt == 'bfloat16' else '':16} {'bf16' if dt == 'bfloat16' else 'fp16'}    {cells}")
    print(f"\nworst lse error: {lse:.2f} x LSE_TOL")
    print(f"kernels fed kv_len - 1: smallest ratio {power:.1f} (must stay well above ALPHA)")
    sys.exit(rc)


if __name__ == "__main__":
    main()
