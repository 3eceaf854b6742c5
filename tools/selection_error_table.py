"""Regenerate the error-to-bound figures of tests/selection_reference.py on a GPU:

    python tools/selection_error_table.py [extra pytest arguments]

runs tests/test_selection_parity_gpu.py and prints, per selection form and vocabulary width, the largest ratio of a
log-prob sum's (or no-speech probability's) error to its derived bound, as the test module collects them."""
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]

if __name__ == "__main__":
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-s", "tests/test_selection_parity_gpu.py", *sys.argv[1:]],
                       cwd=ROOT, capture_output=True, text=True)
    lines = [l for l in r.stdout.splitlines() if l.startswith(("selection error", "harvested"))]
    for l in lines:
        print(l)
    sys.exit(r.returncode)
