#!/bin/bash
# One gpurun call's worth of verification + measurement, in the order that matters if the call is cut short.
#   /usr/local/graft/bin/gpurun --timeout 1500 -- 'tools/gpu_session.sh r02'              (1 GPU)
#   /usr/local/graft/bin/gpurun --gpus 8 --timeout 900 -- 'tools/gpu_session.sh r02 node' (N GPUs: node-level only)
# Everything lands under gpurun_out/<tag>/; copy what should be judged into profiles/.
set -uo pipefail
TAG=${1:-rXX}
MODE=${2:-single}
OUT=gpurun_out/$TAG
mkdir -p $OUT
nvidia-smi --query-gpu=name,clocks.sm,clocks.max.sm,clocks_throttle_reasons.active --format=csv > $OUT/clocks_before.csv 2>&1
N=$(nvidia-smi -L | wc -l)

# what the round-end driver does around bench.py: an nvidia-smi sampler polling NVML while the bench runs (this is what
# made a per-cycle NVML query cost 2.3 ms in BENCH_r01); ours must hold its e2e with it running
sampler_start() { nvidia-smi --query-gpu=index,clocks.sm,power.draw,utilization.gpu --format=csv,noheader -lms 100 > $OUT/$1 2>&1 & SAMPLER=$!; }
sampler_stop() { kill $SAMPLER 2>/dev/null; wait $SAMPLER 2>/dev/null; }

if [ "$MODE" = scale ]; then
  # both arms at N with the driver's command line under a driver-style sampler, nothing else
  sampler_start smi_ref_${N}gpu.csv
  timeout 300 python bench.py --impl reference --gpus $N --steps 20 --warmup 5 --no-allocate > $OUT/bench_reference_${N}gpu.json 2> $OUT/bench_reference_${N}gpu.err
  sampler_stop
  sampler_start smi_ours_${N}gpu.csv
  timeout 600 python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port 29511 \
    bench.py --gpus $N --steps 20 --warmup 5 > $OUT/bench_${N}gpu_sampled.json 2> $OUT/bench_${N}gpu_sampled.err
  sampler_stop
  tail -c 300 $OUT/bench_${N}gpu_sampled.json
  exit 0
fi
if [ "$MODE" = node ]; then
  # multi-device correctness under one process: the tests that SKIP on a 1-GPU box
  timeout 600 python -m pytest tests/test_cycle_gpu.py tests/test_daemon_gpu.py -m gpu -x -q -k "probe_all or node_cycle or native-transient" -rs \
    > $OUT/pytest_multi_${N}gpu.log 2>&1; echo "pytest rc=$?" >> $OUT/pytest_multi_${N}gpu.log
  # both arms at N, with the driver-style sampler running, the reference first (as the driver orders them)
  sampler_start smi_ref_${N}gpu.csv
  timeout 300 python bench.py --impl reference --gpus $N --steps 20 --warmup 5 --no-allocate > $OUT/bench_reference_${N}gpu.json 2> $OUT/bench_reference_${N}gpu.err
  sampler_stop
  sampler_start smi_ours_${N}gpu.csv
  timeout 600 python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port 29511 \
    bench.py --gpus $N --steps 20 --warmup 5 > $OUT/bench_${N}gpu_sampled.json 2> $OUT/bench_${N}gpu_sampled.err
  sampler_stop
  timeout 600 python -m torch.distributed.run --nnodes=1 --nproc-per-node $N --master-addr 127.0.0.1 --master-port 29512 \
    bench.py --gpus $N --steps 200 --warmup 5 > $OUT/bench_${N}gpu.json 2> $OUT/bench_${N}gpu.err
  # the round-1 behaviour for contrast: NVML inside every cycle of all N devices of one process
  GSB_INVENTORY_POLICY=live timeout 300 python tools/node_cycle.py > $OUT/node_cycle_${N}gpu_live.json 2> $OUT/node_cycle_${N}gpu.err
  timeout 300 python tools/node_cycle.py > $OUT/node_cycle_${N}gpu_snapshot.json 2>> $OUT/node_cycle_${N}gpu.err
  tail -3 $OUT/pytest_multi_${N}gpu.log
  exit 0
fi
if [ "$MODE" = lab ]; then
  # kernel lab work (needs build/direct_anomaly, built on the builder and shipped)
  timeout 120 build/direct_anomaly > $OUT/direct_anomaly.json 2> $OUT/direct_anomaly.err
  # one full capture of the shipped refill kernel on a 1 GiB window (profiles/ncu_window_r02_*), and of the shipped VERIFY
  timeout 600 ncu --set full --clock-control none --import-source on -k regex:probe_bulk_dyn -c 2 -o $OUT/ncu_window_dyn_r02 \
    python tools/profile_target.py 5 4 > $OUT/ncu_full.log 2>&1
  timeout 600 ncu --set full --clock-control none --import-source on -k regex:probe_bulk -c 4 -o $OUT/ncu_transient_r02 \
    python tools/profile_target.py 0 2 transient > $OUT/ncu_transient.log 2>&1
  ncu -i $OUT/ncu_transient_r02.ncu-rep --page raw --csv > $OUT/ncu_transient_r02_raw.csv 2>/dev/null
  ncu -i $OUT/ncu_window_dyn_r02.ncu-rep --page raw --csv > $OUT/ncu_window_dyn_r02_raw.csv 2>/dev/null
  ncu -i $OUT/ncu_window_dyn_r02.ncu-rep --page details --csv > $OUT/ncu_window_dyn_r02_details.csv 2>/dev/null
  tail -c 300 $OUT/direct_anomaly.json
  exit 0
fi
timeout 900 python -m pytest tests -m gpu -x -q -rs > $OUT/pytest_gpu.log 2>&1; echo "pytest rc=$?" >> $OUT/pytest_gpu.log
python __graft_entry__.py smoke-only > $OUT/smoke.log 2>&1
# the driver's own command lines (steps 20, warmup 5), reference first, each under a driver-style sampler
sampler_start smi_ref.csv
timeout 400 python bench.py --impl reference --steps 20 --warmup 5 > $OUT/bench_reference_1gpu_sampled.json 2> $OUT/bench_reference_1gpu.err
sampler_stop
sampler_start smi_ours.csv
timeout 400 python bench.py --steps 20 --warmup 5 > $OUT/bench_1gpu_sampled.json 2> $OUT/bench_1gpu_sampled.err
sampler_stop
# longer, quiet run: the numbers DESIGN.md quotes
timeout 400 python bench.py --steps 200 --warmup 5 --quick-allocate > $OUT/bench_1gpu.json 2> $OUT/bench_1gpu.err
# launch list of the same command (shares, not absolutes: ncu serialises and runs cold)
timeout 600 ncu --metrics gpu__time_duration.sum --clock-control none -c 400 --csv --log-file $OUT/launches.csv \
  python bench.py --steps 20 --warmup 3 --no-allocate --no-cpu-baseline > $OUT/bench_under_ncu.log 2>&1
# the DIRECT control: the same headline on the unstaged load -> store path
timeout 400 python bench.py --variant direct --steps 20 --warmup 5 --no-allocate --no-cpu-baseline > $OUT/bench_direct.json 2> $OUT/bench_direct.err
# memcheck + racecheck of every data path on a small arena (the smoke), this round's kernels
GSB_PROBE_WATCHDOG_MS=0 timeout 600 compute-sanitizer --tool memcheck --error-exitcode 3 python __graft_entry__.py smoke-only > $OUT/memcheck_smoke.log 2>&1; echo "memcheck rc=$?" >> $OUT/memcheck_smoke.log
GSB_PROBE_WATCHDOG_MS=0 timeout 600 compute-sanitizer --tool racecheck --error-exitcode 3 python tools/profile_target.py 5 2 > $OUT/racecheck_bulkd.log 2>&1; echo "racecheck rc=$?" >> $OUT/racecheck_bulkd.log
nvidia-smi --query-gpu=name,clocks.sm,clocks.max.sm,clocks_throttle_reasons.active --format=csv > $OUT/clocks_after.csv 2>&1
tail -3 $OUT/pytest_gpu.log
