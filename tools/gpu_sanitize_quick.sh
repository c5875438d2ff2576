#!/bin/bash
# memcheck + racecheck + synccheck on the paths that changed last (row compaction, staged ingest, layout partitions,
# async packed results)
mkdir -p gpurun_out
K='leftovers_in_most_rows or staged or async or packed or (window_parity and (2049 or 70001)) or (random_pool and (4097 or 70001)) or config2 or dedupe or leaver or persistent or multi_tick'
timeout 420 compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests -m gpu -q -x -k "$K" > gpurun_out/memcheck.log 2>&1; echo "memcheck rc=$?"; grep -E "ERROR SUMMARY|passed|failed" gpurun_out/memcheck.log | tail -3
K2='(leftovers_in_most_rows and dense) or staged or (window_parity and 2049 and not 100000) or (random_pool and 4097) or packed_rejects'
timeout 300 compute-sanitizer --tool racecheck --error-exitcode 9 python -m pytest tests -m gpu -q -x -k "$K2" > gpurun_out/racecheck.log 2>&1; echo "racecheck rc=$?"; grep -E "RACECHECK SUMMARY|passed|failed" gpurun_out/racecheck.log | tail -3
timeout 200 compute-sanitizer --tool synccheck --error-exitcode 9 python -m pytest tests -m gpu -q -x -k "$K2" > gpurun_out/synccheck.log 2>&1; echo "synccheck rc=$?"; grep -E "ERROR SUMMARY|passed|failed" gpurun_out/synccheck.log | tail -3
