#!/bin/bash
# k_parse / k_entropy time against the number of frames in one launch (wave quantisation, tail)
TAG=${1:-s1}
mkdir -p gpurun_out
sms=$(python -c "import torch; print(torch.cuda.get_device_properties(0).multi_processor_count)")
for n in $((8 * sms)) $((16 * sms)) $((32 * sms)) 6144 8192 $((64 * sms)) 16384; do
  echo "== n=$n" >> gpurun_out/enc_sweep_$TAG.log
  timeout 300 python scripts/gpu_enc.py $n 2 3 2>&1 | tail -2 >> gpurun_out/enc_sweep_$TAG.log
done
cat gpurun_out/enc_sweep_$TAG.log
