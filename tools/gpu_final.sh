#!/bin/bash
# Round-end GPU pass (what the driver runs, plus the extra bench lines): the whole -m gpu suite in one process, smoke(), the default
# bench line (batched + single-chunk record + CPU leg), the reference arm, the int8 line, the phase-by-phase check of the many-row kernel.
# tools/gpu_profile.sh is the ncu half; tools/make_profiles.py turns gpurun_out/ into profiles/.
cd "$(dirname "$0")/.."
mkdir -p gpurun_out
timeout 1500 python -m pytest tests/ -x -q -m gpu -p no:cacheprovider > gpurun_out/test_all_gpu.log 2>&1; echo "pytest -m gpu exit $?"
tail -n 6 gpurun_out/test_all_gpu.log | cut -c1-300
timeout 300 python __graft_entry__.py --smoke > gpurun_out/smoke.log 2>&1; echo "smoke exit $?"; tail -n 2 gpurun_out/smoke.log
( time timeout 1500 python bench.py > gpurun_out/bench_default.json 2> gpurun_out/bench_default.err ) 2> gpurun_out/bench_default.time; echo "bench default exit $?"; grep real gpurun_out/bench_default.time
( time timeout 1200 python bench.py --impl reference --steps 2 --warmup 1 > gpurun_out/bench_reference.json 2> gpurun_out/bench_reference.err ) 2> gpurun_out/bench_reference.time; echo "bench reference exit $?"; grep real gpurun_out/bench_reference.time
timeout 900 python bench.py --compute-type int8_float16 --no-secondary --no-cpu-baseline --steps 3 > gpurun_out/bench_b16_int8.json 2> gpurun_out/bench_b16_int8.err; echo "bench int8 exit $?"
python tools/show_bench.py gpurun_out/bench_default.json gpurun_out/bench_reference.json gpurun_out/bench_b16_int8.json 2>&1 | cut -c1-700 | tail -30
timeout 900 python -m pytest tests/test_gpu_decode_phases.py -q -s -m gpu -k phase -p no:cacheprovider 2>&1 | grep -E "ratio|passed|failed" | awk '{print ($(NF-1) == "ratio" ? $NF : 9), $0}' | sort -g | tail -n 8 | cut -c1-200; echo "decode phases exit ${PIPESTATUS[0]}"
