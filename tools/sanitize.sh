#!/bin/bash
# compute-sanitizer passes over the hand-written kernels ; summaries go to the output directory (default sanitizer_out/).
set -u
OUT=${1:-sanitizer_out}
mkdir -p "$OUT"
FILES="tests/test_gpu_parity.py tests/test_gpu_ozaki.py tests/test_gpu_ozaki2.py tests/test_gpu_tf32.py tests/test_gpu_spmm.py tests/test_gpu_grid.py"
run() {  # tool, tag, pytest -k expression
  timeout 900 compute-sanitizer --tool "$1" --print-limit 5 python -m pytest $FILES -m gpu -x -q -k "$3" > "$OUT/sanitizer_$1_$2.log" 2>&1
  echo "== $1 $2: exit $? ; $(grep -E 'ERROR SUMMARY|RACECHECK SUMMARY|passed|failed' "$OUT/sanitizer_$1_$2.log" | tr '\n' ' ')"
}
run memcheck dmma    "multiply_dense_vs_oracle and (131 or 300 or 40-40)"
run memcheck ozaki   "ozaki_multiply_vs_oracle and (131 or 300)"
run memcheck crt     "crt_multiply_vs_oracle and (131 or 300 or 1024) or crt_is_bit_exact"          # engine: 1-SM (blk 64/128) and CTA-pair (blk 256) kernels
run memcheck crtjobs "crt_pipelined or crt_panelled or corrects_isolated"           # + outlier records and the fix-up kernel                                                # pipelined groups, panelled scratch
run memcheck tf32    "tf32x3_multiply and (300 or 512)"
run memcheck sparse  "sparse_blocks or sparse_op_sparse or aggregates or project"
run memcheck spsp    "sparse_times_sparse"
run memcheck spmm2   "spmm2_vs_oracle and (700 or 0.05 or False) or spmm2_accumulates"               # ragged strips, global-entry path, unsorted rows
run memcheck sprand  "device_sprand and 512"
run memcheck grid    "grid_multiply_matches_oracle and 1-4-1024 or sharded_put_block"
run synccheck crt    "crt_multiply_vs_oracle and (256-256-256 or 1024)"
run synccheck spmm2  "spmm2_vs_oracle and 700"
run racecheck crt2sm "crt_multiply_vs_oracle and 1024"
