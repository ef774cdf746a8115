#!/bin/bash
# One H100 session for row-sharded CLancIR: the card and its power limit, the new CPU and GPU tests, the
# sharded_local times (lancir_sharded_times.py), three bench lines (their lancir block), smoke() and the GPU
# suite.  With two or more visible GPUs the multi-GPU worker test runs inside the GPU suite; strong scaling
# of lancirb200_resize_sharded is not timed by this script.
# usage: profiles/h100_lancir_sharded.sh <out dir>
out=${1:?usage: profiles/h100_lancir_sharded.sh <out dir>}
mkdir -p "$out"
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv > "$out/gpu.txt" 2>&1
cat "$out/gpu.txt"
python -c "import __graft_entry__ as g; g.build()" > "$out/build.txt" 2>&1 || { tail -40 "$out/build.txt"; exit 1; }
timeout 1200 python -m pytest tests/test_gpu_lancir_sharded.py tests/test_lancir_sharding.py -q -p no:cacheprovider -rs -x \
    > "$out/pytest_lancir_sharded.txt" 2>&1
tail -15 "$out/pytest_lancir_sharded.txt"
timeout 300 python profiles/lancir_sharded_times.py --n 30 > "$out/lancir_sharded_times.jsonl" 2> "$out/lancir_sharded_times.err"
cat "$out/lancir_sharded_times.jsonl"; tail -3 "$out/lancir_sharded_times.err"
lancir() { python -c "import json,sys; d=json.loads(sys.stdin.read().strip().splitlines()[-1]); l=d.get('lancir', {}); print(json.dumps({'lancir_ms': l.get('ms_per_frame'), 'error': l.get('error')}))"; }
for run in 1 2 3; do
    timeout 600 python bench.py --gpus 1 --steps 20 --warmup 3 --no-cpu-baseline > "$out/bench_new_$run.json" 2> "$out/bench_new_$run.err"
    cut -c1-160 "$out/bench_new_$run.json"; lancir < "$out/bench_new_$run.json"
done
timeout 300 python -c "import __graft_entry__ as g; g.smoke()" > "$out/smoke.txt" 2>&1
tail -1 "$out/smoke.txt"
timeout 2400 python -m pytest tests -q -p no:cacheprovider -m gpu > "$out/pytest_gpu.txt" 2>&1
tail -3 "$out/pytest_gpu.txt"
