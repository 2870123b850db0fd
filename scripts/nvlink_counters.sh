#!/bin/bash
# NVLink byte counters of the fused step at 2 GPUs: rank 0 runs under ncu with single-pass metrics only (no kernel
# replay, so the peer's flag exchange keeps working), rank 1 runs plain.  Launch it on 2 GPUs with bench.py's
# arguments: torchrun --nproc_per_node 2 --no-python scripts/nvlink_counters.sh --gpus 2 --gather p2p
if [ "$LOCAL_RANK" = "0" ]; then
  exec ncu --metrics nvltx__bytes.sum,nvlrx__bytes.sum,gpu__time_duration.sum --clock-control none -k regex:step_kernel_gather -s 20 -c 4 --csv --log-file gpurun_out/r2b_nvlink_rank0.csv python bench.py "$@"
else
  exec python bench.py "$@"
fi
