#!/bin/bash
# decoder kernel times against the number of frames in one launch (latency floor vs throughput)
TAG=${1:-s1}
mkdir -p gpurun_out
sms=$(python -c "import torch; print(torch.cuda.get_device_properties(0).multi_processor_count)")
for n in $sms $((8 * sms)) $((32 * sms)) 8192 16384; do
  echo "== n=$n" >> gpurun_out/dec_sweep_$TAG.log
  timeout 300 python scripts/gpu_dec.py $n 2 2>&1 | grep -E "^rep 1|roles" >> gpurun_out/dec_sweep_$TAG.log
done
cat gpurun_out/dec_sweep_$TAG.log
