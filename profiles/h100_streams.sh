#!/bin/bash
# One H100 session for the stream / graph / thread tests: the card, tests/test_gpu_streams.py (with its wall
# time), the unqueried window's generic-kernel fallback against the queried window's tile kernel
# (unqueried_window_times.py), smoke() and two bench lines; with "suite" as the second argument the whole
# GPU suite instead (the two halves fit one session each).
# usage: profiles/h100_streams.sh <out dir> [suite]
out=${1:?usage: profiles/h100_streams.sh <out dir> [suite]}
mkdir -p "$out"
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv > "$out/gpu.txt" 2>&1
cat "$out/gpu.txt"
python -c "import __graft_entry__ as g; g.build()" > "$out/build.txt" 2>&1 || { tail -40 "$out/build.txt"; exit 1; }
if [ "$2" = "suite" ]; then
    # (the stream tests first, so that the routing tests that profile in this process run after them)
    timeout 560 python -m pytest tests/test_gpu_streams.py tests -q -p no:cacheprovider -m gpu -rs > "$out/pytest_gpu.txt" 2>&1
    tail -12 "$out/pytest_gpu.txt"
    exit 0
fi
start=$(date +%s.%N)
timeout 600 python -m pytest tests/test_gpu_streams.py -q -p no:cacheprovider -m gpu -rfs > "$out/pytest_streams.txt" 2>&1
end=$(date +%s.%N)
tail -5 "$out/pytest_streams.txt"
echo "test_gpu_streams.py wall time: $(python -c "print(round($end - $start, 1))") s (python start-up included)"
timeout 300 python profiles/unqueried_window_times.py --n 30 > "$out/unqueried_window_times.jsonl" 2> "$out/unqueried_window_times.err"
cat "$out/unqueried_window_times.jsonl"; tail -3 "$out/unqueried_window_times.err"
timeout 300 python -c "import __graft_entry__ as g; g.smoke()" > "$out/smoke.txt" 2>&1
tail -1 "$out/smoke.txt"
for run in 1 2; do
    timeout 300 python bench.py --gpus 1 --steps 20 --warmup 3 --no-cpu-baseline > "$out/bench_$run.json" 2> "$out/bench_$run.err"
    cut -c1-200 "$out/bench_$run.json"
done
