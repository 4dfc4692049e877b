#!/bin/bash
# Runs on the GPU box under gpurun: parity tests (one process per file so a faulting kernel cannot
# poison the others), smoke, a short bench.  Everything is logged under gpurun_out/.
mkdir -p gpurun_out
nvidia-smi > gpurun_out/nvsmi.txt 2>&1
python -c "import torch; print(torch.cuda.get_device_name(0), torch.cuda.get_device_capability(0))" > gpurun_out/dev.txt 2>&1
# default: every GPU module, in sorted order (the z / zz prefixes put the slow or device-hungry ones last)
DEFAULT_FILES=$(cd tests && ls test_gpu_*.py | LC_ALL=C sort | sed 's/\.py$//')
for f in ${TEST_FILES:-$DEFAULT_FILES}; do
  echo "=== $f ===" 
  timeout 900 python -m pytest tests/$f.py -q -m gpu --tb=short -p no:cacheprovider ${PYTEST_ARGS} > gpurun_out/$f.log 2>&1
  echo "rc=$?" >> gpurun_out/$f.log
  tail -n 25 gpurun_out/$f.log
done
echo "=== smoke ==="
timeout 300 python __graft_entry__.py --smoke > gpurun_out/smoke.log 2>&1; echo "rc=$?" >> gpurun_out/smoke.log; tail -n 5 gpurun_out/smoke.log
echo "=== bench ==="
timeout 600 python bench.py --steps ${BENCH_STEPS:-10} --warmup 3 > gpurun_out/bench.log 2>&1; echo "rc=$?" >> gpurun_out/bench.log; tail -n 5 gpurun_out/bench.log | cut -c1-3000
