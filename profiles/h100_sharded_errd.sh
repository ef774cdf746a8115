#!/bin/bash
# One H100 session for double buffers and error diffusion on the sharded and per-pass entry points: the card,
# tests/test_gpu_sharded_errd.py, sharded_errd_times.py, smoke() and the bench line; with "suite" as the second
# argument the rest of the GPU suite instead.  The test runs write their progress unbuffered into the out dir.
# usage: profiles/h100_sharded_errd.sh <out dir> [suite]
out=${1:?usage: profiles/h100_sharded_errd.sh <out dir> [suite]}
mkdir -p "$out"
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv > "$out/gpu.txt" 2>&1
cat "$out/gpu.txt"
start=$(date +%s)
python -c "import __graft_entry__ as g; g.build()" > "$out/build.txt" 2>&1 || { tail -40 "$out/build.txt"; exit 1; }
echo "build: $(( $(date +%s) - start )) s"
if [ "$2" = "suite" ]; then
    timeout 900 python -u -m pytest tests -q -p no:cacheprovider -m gpu -rs --ignore=tests/test_gpu_sharded_errd.py > "$out/pytest_gpu.txt" 2>&1
    tail -12 "$out/pytest_gpu.txt"
    exit 0
fi
timeout 900 python -u -m pytest tests/test_gpu_sharded_errd.py -q -p no:cacheprovider -m gpu -rfs --durations=5 > "$out/pytest_sharded_errd.txt" 2>&1
tail -25 "$out/pytest_sharded_errd.txt"
timeout 300 python -u profiles/sharded_errd_times.py --n 20 > "$out/sharded_errd_times.jsonl" 2> "$out/sharded_errd_times.err"
cat "$out/sharded_errd_times.jsonl"; tail -3 "$out/sharded_errd_times.err"
timeout 300 python -c "import __graft_entry__ as g; g.smoke()" > "$out/smoke.txt" 2>&1
tail -1 "$out/smoke.txt"
timeout 300 python bench.py --gpus 1 --steps 20 --warmup 3 --no-cpu-baseline > "$out/bench.json" 2> "$out/bench.err"
cut -c1-200 "$out/bench.json"
