#!/bin/bash
# Smoke, GPU parity tests and one bench line in one go.  Usage (repo root):  bash tools/gpu_check.sh [OUT_DIR]
set -u
OUT=${1:-gpu_check_out}
mkdir -p "$OUT"
nvidia-smi --query-gpu=name,power.limit,clocks.sm,clocks.max.sm,power.draw --format=csv > "$OUT/gpu.txt" 2>&1
echo "== smoke" ; timeout 200 python __graft_entry__.py --smoke 2>&1 | tail -3
echo "== pytest gpu" ; timeout 1200 python -m pytest tests -m gpu -q 2>&1 | tail -6 | tee "$OUT/pytest_gpu.txt"
echo "== bench" ; timeout 900 python bench.py --steps 20 --warmup 5 2>"$OUT/bench.err" | tee "$OUT/bench.json" | cut -c1-400
tail -3 "$OUT/bench.err"
