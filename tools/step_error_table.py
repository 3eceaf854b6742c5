"""Regenerate the kernel / yardstick table of tests/step_reference.py on a GPU:

    python tools/step_error_table.py [extra pytest arguments]

runs tests/test_step_parity_gpu.py with OASR_ATTN_REPORT pointing at a temporary file and prints, per test and dtype,
training_error_table's columns: the largest rule-1 value (worst error over its bound) and rule-2 value (unexplained
differing elements over ALPHA x the yardstick's + SLACK) of the outputs rounded to T, the fp32 outputs' largest
element-bound value and row ratios to the yardstick, and the optimizer state's largest error over its bound
("scalar").  Re-run it after a change to the conv-stem glue, embedding, column-sum or optimizer kernels before
touching a bound of tests/step_reference.py."""
from training_error_table import main

if __name__ == "__main__":
    main("tests/test_step_parity_gpu.py")
