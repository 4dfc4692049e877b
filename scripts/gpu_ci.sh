#!/bin/bash
# Runs on the GPU box under gpurun: parity tests (one process per file so a faulting kernel cannot
# poison the others), smoke, a short bench.  Everything is logged under gpurun_out/.
mkdir -p gpurun_out
nvidia-smi > gpurun_out/nvsmi.txt 2>&1
python -c "import torch; print(torch.cuda.get_device_name(0), torch.cuda.get_device_capability(0))" > gpurun_out/dev.txt 2>&1
for f in ${TEST_FILES:-test_gpu_linear test_gpu_recurrent test_gpu_model test_gpu_train test_gpu_train_fullsize test_gpu_decoder_envelope test_gpu_z_audio test_gpu_z_data test_gpu_z_features test_gpu_z_resample test_gpu_z_summary test_gpu_z_trim test_gpu_z_longform test_gpu_zz_decoder_budget test_gpu_speaker_decoder test_gpu_guided_attention}; do
  echo "=== $f ===" 
  timeout 900 python -m pytest tests/$f.py -q -m gpu --tb=short -p no:cacheprovider ${PYTEST_ARGS} > gpurun_out/$f.log 2>&1
  echo "rc=$?" >> gpurun_out/$f.log
  tail -n 25 gpurun_out/$f.log
done
echo "=== smoke ==="
timeout 300 python __graft_entry__.py --smoke > gpurun_out/smoke.log 2>&1; echo "rc=$?" >> gpurun_out/smoke.log; tail -n 5 gpurun_out/smoke.log
echo "=== bench ==="
timeout 600 python bench.py --steps ${BENCH_STEPS:-10} --warmup 3 > gpurun_out/bench.log 2>&1; echo "rc=$?" >> gpurun_out/bench.log; tail -n 5 gpurun_out/bench.log | cut -c1-3000
