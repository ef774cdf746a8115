#!/bin/bash
# One H100 session for the change that gives each workspace / mailbox / streaming-parameter decision one
# definition: the card, the GPU tests, the whole suite, smoke() and the bench line.
# usage: profiles/h100_single_layouts.sh <out dir>
out=${1:?usage: profiles/h100_single_layouts.sh <out dir>}
mkdir -p "$out"
nvidia-smi --query-gpu=name,power.limit --format=csv > "$out/gpu.txt" 2>&1
cat "$out/gpu.txt"
python -c "import __graft_entry__ as g; g.build()" > "$out/build.txt" 2>&1 || { tail -40 "$out/build.txt"; exit 1; }
timeout 900 python -m pytest tests -q -p no:cacheprovider -m gpu -rs > "$out/pytest_gpu.txt" 2>&1
tail -3 "$out/pytest_gpu.txt"
timeout 1500 python -m pytest tests -q -p no:cacheprovider > "$out/pytest_full.txt" 2>&1
tail -3 "$out/pytest_full.txt"
timeout 300 python -c "import __graft_entry__ as g; g.smoke()" > "$out/smoke.txt" 2>&1
tail -2 "$out/smoke.txt"
for run in 1 2; do
    timeout 900 python bench.py --gpus 1 --steps 20 --warmup 3 > "$out/bench_n1_$run.json" 2> "$out/bench_n1_$run.err"
    cut -c1-400 "$out/bench_n1_$run.json"
done
