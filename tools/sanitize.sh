#!/bin/bash
# compute-sanitizer passes over the GPU parity tests (run on the GPU box); logs under gpurun_out/san/,
# one-line summaries are copied to profiles/ by hand.  memcheck: out-of-bounds / misaligned accesses;
# racecheck: shared-memory hazards (the matcher's lock-free pipeline polls shared flags on purpose:
# every reported hazard is listed by source line in the log).
mkdir -p gpurun_out/san
K1='rank_and_match_parity_random or constraint_kernel or rank_golden or quota_and_rate'
K2='rebalanc or next_state or pending_job or below_quota or off_grid or placement_failure or exchange_device or state_offers'
timeout 1500 compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests -m gpu -x -q -k "$K1" > gpurun_out/san/memcheck_rank_match.log 2>&1
echo "memcheck rank+match rc=$?"; grep -E "ERROR SUMMARY|passed|failed" gpurun_out/san/memcheck_rank_match.log | tail -3
timeout 1500 compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests -m gpu -x -q -k "$K2" > gpurun_out/san/memcheck_rebalance_misc.log 2>&1
echo "memcheck rebalance+misc rc=$?"; grep -E "ERROR SUMMARY|passed|failed" gpurun_out/san/memcheck_rebalance_misc.log | tail -3
timeout 1500 compute-sanitizer --tool racecheck --racecheck-report analysis python -m pytest tests/test_gpu_parity.py -x -q -k "rank_and_match_parity_random and (11 or 12 or 16)" > gpurun_out/san/racecheck_match.log 2>&1
echo "racecheck match rc=$?"; grep -E "RACECHECK SUMMARY|passed|failed" gpurun_out/san/racecheck_match.log | tail -3
grep -E "Race reported|hazard" gpurun_out/san/racecheck_match.log | sed -E 's/0x[0-9a-f]+/ADDR/g' | sort | uniq -c | sort -rn | head -20
