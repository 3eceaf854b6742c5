"""Regenerate the kernel / yardstick table of tests/decode_reference.py on a GPU:

    python tools/decode_error_table.py [extra pytest arguments]

runs tests/test_decode_parity_gpu.py with OASR_ATTN_REPORT pointing at a temporary file, then prints, per test and
dtype, the largest rule-1 value (worst error over its bound), the largest ratio of differing elements to the
yardstick's (rule 2), the composed step's largest max-row / mean-row ratios and the decode-attention launches' worst
error in units of u.  Re-run it after a decoder-step kernel change before touching ALPHA, SLACK or STEP_ALPHA."""
import collections
import json
import os
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]


def main():
    with tempfile.TemporaryDirectory() as tmp:
        report = os.path.join(tmp, "report.jsonl")
        env = dict(os.environ, OASR_ATTN_REPORT=report)
        cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider",
               "tests/test_decode_parity_gpu.py", *sys.argv[1:]]
        rc = subprocess.call(cmd, cwd=ROOT, env=env)
        lines = Path(report).read_text().splitlines() if os.path.exists(report) else []
    table = collections.defaultdict(lambda: collections.defaultdict(float))
    for line in lines:
        rec = json.loads(line)
        test = rec["test"].split("::")[-1].split("[")[0]
        row = table[(test, rec.get("dtype", ""))]
        if rec["kind"] == "linear":
            row["rule 1"] = max(row["rule 1"], rec["worst"])
            row["diff ratio"] = max(row["diff ratio"], rec["n_diff"] / max(rec["emu_diff"], 1))
            row["diff share"] = max(row["diff share"], rec["n_diff"] / max(rec["numel"], 1))
        elif rec["kind"] == "step":
            row["step max"] = max(row["step max"], rec["worst_ratio"])
            row["step mean"] = max(row["step mean"], rec["mean_ratio"])
        elif rec["kind"] == "attention":
            row["attention / u"] = max(row["attention / u"], rec["worst_u"])
        elif rec["kind"] == "prepare":
            row["fp16 gap share"] = max(row["fp16 gap share"], rec["share_differing"])
            row["fp16 gap row"] = max(row["fp16 gap row"], rec["worst_row_rel"])
    for (test, dtype), row in sorted(table.items()):
        print(f"{test:45s} {dtype:9s} " + "  ".join(f"{k} {v:.3g}" for k, v in row.items()))
    sys.exit(rc)


if __name__ == "__main__":
    main()
