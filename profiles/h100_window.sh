#!/bin/bash
# One H100 session for destination windows: the card, the window tests, window against whole-image times
# (window_times.py), the whole suite, smoke() and the bench line -- alternating with a checkout of the parent
# commit when its (built) tree is given.
# usage: profiles/h100_window.sh <out dir> [<parent tree>]
out=${1:?usage: profiles/h100_window.sh <out dir> [<parent tree>]}
parent=$2
mkdir -p "$out"
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv > "$out/gpu.txt" 2>&1
cat "$out/gpu.txt"
python -c "import __graft_entry__ as g; g.build()" > "$out/build.txt" 2>&1 || { tail -40 "$out/build.txt"; exit 1; }
timeout 1200 python -m pytest tests/test_gpu_window.py -q -p no:cacheprovider -m gpu -rs > "$out/pytest_window.txt" 2>&1
tail -2 "$out/pytest_window.txt"
timeout 300 python profiles/window_times.py --n 30 > "$out/window_times.jsonl" 2> "$out/window_times.err"
cat "$out/window_times.jsonl"
for run in 1 2 3; do
    timeout 300 python bench.py --gpus 1 --steps 20 --warmup 3 --no-cpu-baseline --no-extras > "$out/bench_new_$run.json" 2> "$out/bench_new_$run.err"
    cut -c1-200 "$out/bench_new_$run.json"
    if [ -n "$parent" ]; then
        (cd "$parent" && timeout 300 python bench.py --gpus 1 --steps 20 --warmup 3 --no-cpu-baseline --no-extras) > "$out/bench_parent_$run.json" 2> "$out/bench_parent_$run.err"
        cut -c1-200 "$out/bench_parent_$run.json"
    fi
done
timeout 300 python -c "import __graft_entry__ as g; g.smoke()" > "$out/smoke.txt" 2>&1
tail -1 "$out/smoke.txt"
timeout 1500 python -m pytest tests -q -p no:cacheprovider > "$out/pytest_full.txt" 2>&1
tail -2 "$out/pytest_full.txt"
