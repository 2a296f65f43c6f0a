#!/bin/bash
# ncu evidence for the round: launch list of the default bench line + full captures of the two persistent step kernels, and the
# per-phase device timers (ticks build).  tools/make_profiles.py turns gpurun_out/ into profiles/.
cd "$(dirname "$0")/.."
mkdir -p gpurun_out
timeout 900 ncu --metrics gpu__time_duration.sum --clock-control none -c 40000 --csv --log-file gpurun_out/launches_batched.csv \
  python bench.py --steps 1 --warmup 3 --no-cpu-baseline --no-secondary > gpurun_out/ncu_bench.log 2>&1; echo "ncu list exit $?"
python tools/ncu_summary.py gpurun_out/launches_batched.csv 2>/dev/null | head -12
timeout 600 ncu --set full --clock-control none --import-source on -k bstep_kernel -s 14 -c 1 -f -o gpurun_out/full_bstep \
  python tools/profile_step.py --batch 16 --new-tokens 24 > gpurun_out/full_bstep.log 2>&1; echo "ncu full bstep exit $?"
timeout 400 ncu --set full --clock-control none --import-source on -k regex:dstep_kernel -s 10 -c 1 -f -o gpurun_out/full_dstep \
  python tools/profile_step.py --batch 1 --new-tokens 16 > gpurun_out/full_dstep.log 2>&1; echo "ncu full dstep exit $?"
python tools/ncu_full_summary.py gpurun_out/full_bstep.ncu-rep gpurun_out/full_dstep.ncu-rep 2>&1 | cut -c1-700 | head -30
if [ -f faster_whisper_b200/libb200whisper_ticks.so ]; then
  B2W_LIBRARY=$PWD/faster_whisper_b200/libb200whisper_ticks.so timeout -s KILL 300 python tools/step_ab.py --repeat 1 --prof > gpurun_out/step_prof.log 2>&1; echo "step_prof exit $?"
  grep "bstep prof\|decode" gpurun_out/step_prof.log | tail -n 20 | cut -c1-260
  B2W_LIBRARY=$PWD/faster_whisper_b200/libb200whisper_ticks.so timeout -s KILL 300 python tools/step_ab.py --batch 1 --repeat 1 --prof > gpurun_out/step_prof_single.log 2>&1; echo "step_prof single exit $?"
  grep "dstep prof\|decode" gpurun_out/step_prof_single.log | tail -n 16 | cut -c1-260
fi
timeout -s KILL 300 python tools/step_ab.py --batch 1 --configs "B2W_STEP=dstep;B2W_STEP=bstep" 2>&1 | grep decode | cut -c1-200; echo "single ab exit ${PIPESTATUS[0]}"
ls -la gpurun_out/*.ncu-rep
