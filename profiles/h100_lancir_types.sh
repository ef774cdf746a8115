#!/bin/bash
# One H100 session for CLancIR's double and uint32_t buffers: the card, the GPU suite (the new
# test_gpu_lancir_types.py included), smoke(), per-pair times (lancir_types_times.py) of this change with the
# parent commit's u8 -> u8 alternating when its built tree is given, and the bench line (its lancir block) of
# both, alternating.
# usage: profiles/h100_lancir_types.sh <out dir> [<parent tree>]
out=${1:?usage: profiles/h100_lancir_types.sh <out dir> [<parent tree>]}
parent=$2
mkdir -p "$out"
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv > "$out/gpu.txt" 2>&1
cat "$out/gpu.txt"
python -c "import __graft_entry__ as g; g.build()" > "$out/build.txt" 2>&1 || { tail -40 "$out/build.txt"; exit 1; }
timeout 2400 python -m pytest tests -q -p no:cacheprovider -m gpu -rs > "$out/pytest_gpu.txt" 2>&1
grep -E "FAILED|ERROR" "$out/pytest_gpu.txt" | head -20
tail -3 "$out/pytest_gpu.txt"
grep -c "test_gpu_lancir_types" "$out/pytest_gpu.txt"
timeout 300 python -c "import __graft_entry__ as g; g.smoke()" > "$out/smoke.txt" 2>&1
tail -1 "$out/smoke.txt"
for run in 1 2 3; do
    timeout 300 python profiles/lancir_types_times.py --n 30 > "$out/types_times_new_$run.jsonl" 2> "$out/types_times_new_$run.err"
    cat "$out/types_times_new_$run.jsonl"
    if [ -n "$parent" ]; then
        timeout 300 python profiles/lancir_types_times.py --n 30 --pairs u8-u8 --root "$parent" > "$out/types_times_parent_$run.jsonl" 2> "$out/types_times_parent_$run.err"
        cat "$out/types_times_parent_$run.jsonl"
    fi
done
lancir() { python -c "import json,sys; d=json.loads(sys.stdin.read().strip().splitlines()[-1]); l=d.get('lancir', {}); print(json.dumps({'ms_per_step': d.get('ms_per_step'), 'lancir_ms': l.get('ms_per_frame'), 'error': l.get('error')}))"; }
for run in 1 2; do
    timeout 600 python bench.py --gpus 1 --steps 20 --warmup 3 --no-cpu-baseline > "$out/bench_new_$run.json" 2> "$out/bench_new_$run.err"
    echo -n "change "; lancir < "$out/bench_new_$run.json"
    if [ -n "$parent" ]; then
        (cd "$parent" && timeout 600 python bench.py --gpus 1 --steps 20 --warmup 3 --no-cpu-baseline) > "$out/bench_parent_$run.json" 2> "$out/bench_parent_$run.err"
        echo -n "parent "; lancir < "$out/bench_parent_$run.json"
    fi
done
