#!/bin/bash
# Round-2 closing GPU session (about 4 minutes): the --treat_multiallelics kernels on a real GPU.
#   gpurun --timeout 330 -- 'bash scripts/gpu_session_r2p.sh'
# 1. their parity tests + the CLI tests of the branch (stops here when they fail: the remaining budget is for a re-test)
# 2. memcheck of one small contig through the index pass, build and merge
# 3. device split / merge against the Python model on one dense contig (scripts/bench_multiallelic.py)
set -u
cd "$(dirname "$0")/.."
out=gpurun_out/r2p
mkdir -p "$out"
nvidia-smi --query-gpu=name,clocks.max.sm --format=csv > "$out/box.txt" 2>&1
timeout 200 python -m pytest tests/test_gpu_z_multiallelic_device.py tests/test_gpu_multiallelics.py \
    "tests/test_gpu_cli.py::test_index_ends_records_at_info_end" -q -m gpu -x -p no:cacheprovider > "$out/tests.log" 2>&1
rc=$?
tail -4 "$out/tests.log"
echo "tests rc=$rc"
if [ $rc -ne 0 ]; then grep -n "Error\|error\|assert" "$out/tests.log" | head -20; exit 1; fi
timeout 90 compute-sanitizer --tool memcheck --error-exitcode 9 python scripts/bench_multiallelic.py 30000 > "$out/memcheck.log" 2>&1
echo "memcheck rc=$?"; tail -6 "$out/memcheck.log"
timeout 150 python scripts/bench_multiallelic.py ${MA_BP:-800000} > "$out/ma_bench.json" 2> "$out/ma_bench.err"
echo "bench rc=$?"; cat "$out/ma_bench.json"; tail -3 "$out/ma_bench.err"
