#!/bin/bash
# memcheck + racecheck + synccheck on the paths that changed last (row compaction, staged ingest, layout partitions,
# async packed results, ingest against its restatement, every tick result form, snapshot / restore of the active set)
mkdir -p gpurun_out
K='leftovers_in_most_rows or staged or async or packed or (window_parity and (2049 or 70001)) or (random_pool and (4097 or 70001)) or config2 or dedupe or leaver or persistent or multi_tick or (test_ingest and not 5242883 and not wrap and not tombstones) or (test_tick_forms and (few_rows or lob8193 or wide_group or restore or remove_after_take))'
timeout 420 compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests -m gpu -q -x -k "$K" > gpurun_out/memcheck.log 2>&1; echo "memcheck rc=$?"; grep -E "ERROR SUMMARY|passed|failed" gpurun_out/memcheck.log | tail -3
K2='(leftovers_in_most_rows and dense) or staged or (window_parity and 2049 and not 100000) or (random_pool and 4097) or packed_rejects or (test_ingest and (1023 or 1025 or repeat_of_a_cut or reject_list or refusal)) or (test_tick_forms and (one_row or (lob8193 and not s1)))'
timeout 300 compute-sanitizer --tool racecheck --error-exitcode 9 python -m pytest tests -m gpu -q -x -k "$K2" > gpurun_out/racecheck.log 2>&1; echo "racecheck rc=$?"; grep -E "RACECHECK SUMMARY|passed|failed" gpurun_out/racecheck.log | tail -3
timeout 200 compute-sanitizer --tool synccheck --error-exitcode 9 python -m pytest tests -m gpu -q -x -k "$K2" > gpurun_out/synccheck.log 2>&1; echo "synccheck rc=$?"; grep -E "ERROR SUMMARY|passed|failed" gpurun_out/synccheck.log | tail -3
