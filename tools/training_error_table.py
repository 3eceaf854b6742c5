"""Regenerate the kernel / yardstick table of tests/training_reference.py on a GPU:

    python tools/training_error_table.py [extra pytest arguments]

runs tests/test_training_parity_gpu.py with OASR_ATTN_REPORT pointing at a temporary file, then prints, per test and
dtype, the largest rule-1 value (worst error over its bound), the largest rule-2 value (unexplained differing elements
over ALPHA x the yardstick's + SLACK) with the largest kernel / yardstick count ratio, the fp32 outputs' largest
element-bound value and max-row / mean-row ratios to the yardstick, and the worst lse and loss errors in units of
their bounds.  Re-run it after a GEMM, LayerNorm or cross-entropy kernel change before touching ALPHA, F32_ALPHA or
LSE_TOL."""
import collections
import json
import os
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from tests import decode_reference as dr          # noqa: E402
from tests import training_reference as tr        # noqa: E402


def main(test_file="tests/test_training_parity_gpu.py"):
    """Run `test_file` with the report on and print its table (tools/step_error_table.py passes its own file)."""
    with tempfile.TemporaryDirectory() as tmp:
        report = os.path.join(tmp, "report.jsonl")
        env = dict(os.environ, OASR_ATTN_REPORT=report)
        cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider",
               test_file, *sys.argv[1:]]
        rc = subprocess.call(cmd, cwd=ROOT, env=env)
        lines = Path(report).read_text().splitlines() if os.path.exists(report) else []
    table = collections.defaultdict(lambda: collections.defaultdict(float))
    for line in lines:
        rec = json.loads(line)
        test = rec["test"].split("::")[-1].split("[")[0]
        row = table[(test, rec.get("dtype", ""))]
        kind = rec["kind"]
        if kind == "t16":
            row["rule 1"] = max(row["rule 1"], rec["worst"])
            alpha = rec.get("alpha", tr.ALPHA)
            row["rule 2"] = max(row["rule 2"], rec["n_diff"] / (alpha * rec["emu_diff"] + dr.slack(rec["numel"])))
            row["diff ratio"] = max(row["diff ratio"], rec["n_diff"] / max(rec["emu_diff"], 1))
        elif kind == "f32":
            row["f32 bound"] = max(row["f32 bound"], rec["worst"])
            row["f32 max"] = max(row["f32 max"], rec["worst_ratio"])
            row["f32 mean"] = max(row["f32 mean"], rec["mean_ratio"])
        elif kind == "lse":
            row["lse"] = max(row["lse"], rec["lse_tol_units"])
            row["loss"] = max(row["loss"], rec["loss_units"])
        elif kind == "scalar":
            row["scalar"] = max(row["scalar"], rec["worst"])
        elif kind == "step":
            row["rows max"] = max(row["rows max"], rec["worst_ratio"])
            row["rows mean"] = max(row["rows mean"], rec["mean_ratio"])
    for (test, dtype), row in sorted(table.items()):
        print(f"{test:45s} {dtype:9s} " + "  ".join(f"{k} {v:.3g}" for k, v in row.items()))
    sys.exit(rc)


if __name__ == "__main__":
    main()
