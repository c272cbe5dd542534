#!/bin/bash
# compute-sanitizer passes over the hand-written kernels ; summaries go to the output directory (default sanitizer_out/).
set -u
OUT=${1:-sanitizer_out}
mkdir -p "$OUT"
FILES="tests/test_gpu_parity.py tests/test_gpu_ozaki.py tests/test_gpu_ozaki2.py tests/test_gpu_tf32.py tests/test_gpu_spmm.py tests/test_gpu_grid.py"
run() {  # tool, tag, pytest -k expression [, test files instead of $FILES]
  timeout 900 compute-sanitizer --tool "$1" --print-limit 5 python -m pytest ${4:-$FILES} -m gpu -x -q -k "$3" > "$OUT/sanitizer_$1_$2.log" 2>&1
  echo "== $1 $2: exit $? ; $(grep -E 'ERROR SUMMARY|RACECHECK SUMMARY|passed|failed' "$OUT/sanitizer_$1_$2.log" | tr '\n' ' ')"
}
run memcheck dmma    "multiply_dense_vs_oracle and (131 or 300 or 40-40)"
run memcheck ozaki   "ozaki_multiply_vs_oracle and (131 or 300)"
run memcheck ozaki1  "irregular_shapes and (130x120x140 or 300x31x260)" tests/test_gpu_ozaki1_edges.py   # Ozaki-I: blk 50 (byte-wise digit stores), outer product with K % 4 != 0
run memcheck crt     "crt_multiply_vs_oracle and (131 or 300 or 1024) or crt_is_bit_exact"          # engine: 1-SM (blk 64/128) and CTA-pair (blk 256) kernels
run memcheck crtjobs "crt_pipelined or crt_panelled or corrects_isolated"           # + outlier records and the fix-up kernel                                                # pipelined groups, panelled scratch
run memcheck crtedge "irregular_shapes and (563x563x563-blk200-sparse or 356x300x356)" tests/test_gpu_ozaki2_edges.py   # CTA pairs on ragged slots: padding tile, absent blocks
run memcheck tf32   "tf32x3_multiply and (300 or 512)"
run memcheck tf32edge "exact_regime_is_bit_exact and 256x512x128 or more_than_65535_blocks" tests/test_gpu_tf32_edges.py   # stats / slice chunks, ordered reductions
run racecheck tf32edge "exact_regime_is_bit_exact and 256x512x128" tests/test_gpu_tf32_edges.py                              # the slice pass's per-warp line sums in shared memory
run memcheck sparse  "sparse_blocks or sparse_op_sparse or aggregates or project"
run memcheck spsp    "sparse_times_sparse"
run memcheck spgemm  "format_pairs_bit_exact and 0.02 or absent_and_empty or block_heights and (blk64 or blk8192) and csc_csr" tests/test_gpu_spgemm.py  # smem and global accumulators, CSR<->CSC conversion, dense and sparse fills
run memcheck spmm2   "spmm2_vs_oracle and (700 or 0.05 or False) or spmm2_accumulates"               # ragged strips, global-entry path, unsorted rows
run memcheck spmmedge "segment_capacity or extreme_values and pipelined or grid_multiply_rows and sparse and 2-2 or multi_block and 700" tests/test_gpu_spmm_edges.py  # E_CAP +- 1, global window, nnz = 0, ragged strips, grid rows
run memcheck sprand  "device_sprand and 512"
run memcheck grid    "grid_multiply_matches_oracle and 1-4-1024 or sharded_put_block"
run memcheck ksplit  "ksplit_matches_oracle and (1-1-gram or 2-1-odd or 2-4-k3 or 8-1-single)" tests/test_gpu_grid_ksplit.py  # world 1 and multi-GPU, 128-bit and scalar reduce paths
run memcheck stream  "ragged_absent_and_transposed_blocks and 1 or sparse_times_sparse_keeps" tests/test_gpu_streamed.py  # tiled, double-buffered panels, write-back of dense and sparse C blocks
run synccheck crt    "crt_multiply_vs_oracle and (256-256-256 or 1024)"
run synccheck spmm2  "spmm2_vs_oracle and 700"
run synccheck spmmcap "segment_capacity" tests/test_gpu_spmm_edges.py              # shared-memory and global segments in one tile
run racecheck spmmcap "segment_capacity" tests/test_gpu_spmm_edges.py
run racecheck crt2sm "crt_multiply_vs_oracle and 1024"
run memcheck dspmm   "density_around_tau or nonfinite_left or repeated_coordinates or streamed_matches_resident and AB" tests/test_gpu_dspmm.py  # dense x sparse route, flag pass and fix-up
run racecheck dspmm  "density_around_tau" tests/test_gpu_dspmm.py                 # shared-memory and global segments, empty segments skipped
run memcheck gram    "bit_for_bit and (640 or 700) or outliers_on_both_lines or absent_blocks" tests/test_gpu_gram.py  # shared residues, triangular tiles, upper-only fix-up, mirror
run initcheck gram   "bit_for_bit and (640 or 700) or outliers_on_both_lines" tests/test_gpu_gram.py    # nothing reads a lower element no engine stored
run racecheck gram   "bit_for_bit and 640" tests/test_gpu_gram.py                                        # the mirror kernel's shared tile
run memcheck spgram  "layouts_and_densities and (0.004 or 0.06) and mixed or blk40 or absent_and_empty or single_block_8192 and 0.0004 or shuffled and csr" tests/test_gpu_sparse_gram.py  # triangular chains, sym completion, mirrors, fallback
run racecheck spgram "layouts_and_densities and 0.02 and mixed" tests/test_gpu_sparse_gram.py            # per-level counters in shared memory
