#!/bin/bash
# Where the time of the CartPole step goes on one H100 (DESIGN §4.1): the memory floor (scripts/membench.cu, the
# step's bytes with no arithmetic), the compute floor (scripts/cartpole_floors.py, state resident in L2), and the
# kernels themselves (bench.py headline and 2^23 strong-scaling line): kernel P and the default (kernel B).
# Usage, from the repository root after build(): scripts/h100_floors.sh OUT_DIR
OUT="${1:?usage: scripts/h100_floors.sh OUT_DIR}"
mkdir -p "$OUT"
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv | tee "$OUT/floors_gpu.txt"
T=$(mktemp -d)
nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o "$T/membench" scripts/membench.cu && "$T/membench" | tee "$OUT/floors_membench.txt"
rm -rf "$T"
for k in l b; do
  B200GYM_KERNEL=$k timeout 300 python scripts/cartpole_floors.py | tee -a "$OUT/floors_compute.jsonl"
done
# "l": kernel P; "default": kernel B (bench.py labels only the letters a|p|l)
for v in l default; do
  if [ "$v" = default ]; then
    timeout 600 python bench.py --steps 400 --warmup 50 --no-cpu-baseline --no-e2e 2>/dev/null | tail -1 > "$OUT/floors_bench_$v.json"
  else
    B200GYM_KERNEL=l timeout 600 python bench.py --steps 400 --warmup 50 --no-cpu-baseline --no-e2e \
      2>/dev/null | tail -1 > "$OUT/floors_bench_$v.json"
  fi
  python -c "
import json, sys
d = json.load(open(sys.argv[1]))
s = d.get('strong_scaling') or {}
print(sys.argv[2], 'headline_us', round(d['ms_per_step'] * 1e3, 2),
      'p10/p90', round(d['ms_per_step_p10'] * 1e3, 2), round(d['ms_per_step_p90'] * 1e3, 2),
      'strong_us', round(s.get('ms_per_step', 0) * 1e3, 1), 'clocks', json.dumps(d.get('clocks')))
" "$OUT/floors_bench_$v.json" $v
done
