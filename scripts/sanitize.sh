#!/bin/bash
# Race / memory checking of the single-GPU kernels (run on a GPU box).
# Multi-rank kernels spin on peers and cannot be replayed under the sanitizer; their
# ordering contract is covered by the SPMD suites instead.
set -u
export PYTHONPATH=$PWD
OUT=gpurun_out; mkdir -p $OUT
timeout 900 compute-sanitizer --tool memcheck --log-file $OUT/memcheck_gemm.log python -m pytest tests/test_gpu_gemm.py -x -q -k "shape0 or shape5" 2>&1 | tail -3
timeout 900 compute-sanitizer --tool racecheck --log-file $OUT/racecheck_gemm.log python -m pytest tests/test_gpu_gemm.py -x -q -k "shape0" 2>&1 | tail -3
M4T_TEST_DEVICE=cuda timeout 900 compute-sanitizer --tool memcheck --log-file $OUT/memcheck_np1.log python -m mpi4torch_b200.launch -np 1 tests/spmd/run_all.py "spmd_collectives.py" 2>&1 | tail -3
grep -h "ERROR SUMMARY" $OUT/memcheck_*.log $OUT/racecheck_*.log
