#!/bin/bash
# One H100 session for CLancIR destination windows: the card, the LANCIR window tests, window against
# whole-image times (lancir_window_times.py), the bench line (its lancir block) of this change and -- when
# its built tree is given -- of the parent commit, alternating, one bench line with the host baselines
# (the lancir block's parity against upstream), smoke() and the GPU suite.
# usage: profiles/h100_lancir_window.sh <out dir> [<parent tree>]
out=${1:?usage: profiles/h100_lancir_window.sh <out dir> [<parent tree>]}
parent=$2
mkdir -p "$out"
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv > "$out/gpu.txt" 2>&1
cat "$out/gpu.txt"
python -c "import __graft_entry__ as g; g.build()" > "$out/build.txt" 2>&1 || { tail -40 "$out/build.txt"; exit 1; }
timeout 1200 python -m pytest tests/test_gpu_lancir_window.py tests/test_lancir_window.py -q -p no:cacheprovider -m gpu -rs -x > "$out/pytest_lancir_window.txt" 2>&1
tail -15 "$out/pytest_lancir_window.txt"
timeout 300 python profiles/lancir_window_times.py --n 30 > "$out/lancir_window_times.jsonl" 2> "$out/lancir_window_times.err"
cat "$out/lancir_window_times.jsonl"
lancir() { python -c "import json,sys; d=json.loads(sys.stdin.read().strip().splitlines()[-1]); l=d.get('lancir', {}); print(json.dumps({'lancir_ms': l.get('ms_per_frame'), 'parity': l.get('parity_vs_reference'), 'error': l.get('error')}))"; }
for run in 1 2 3; do
    timeout 600 python bench.py --gpus 1 --steps 20 --warmup 3 --no-cpu-baseline > "$out/bench_new_$run.json" 2> "$out/bench_new_$run.err"
    cut -c1-160 "$out/bench_new_$run.json"; lancir < "$out/bench_new_$run.json"
    if [ -n "$parent" ]; then
        (cd "$parent" && timeout 600 python bench.py --gpus 1 --steps 20 --warmup 3 --no-cpu-baseline) > "$out/bench_parent_$run.json" 2> "$out/bench_parent_$run.err"
        echo -n "parent "; cut -c1-160 "$out/bench_parent_$run.json"; lancir < "$out/bench_parent_$run.json"
    fi
done
# once with the host baselines: the lancir block's parity against upstream
timeout 900 python bench.py --gpus 1 --steps 20 --warmup 3 > "$out/bench_new_parity.json" 2> "$out/bench_new_parity.err"
lancir < "$out/bench_new_parity.json"
timeout 300 python -c "import __graft_entry__ as g; g.smoke()" > "$out/smoke.txt" 2>&1
tail -1 "$out/smoke.txt"
timeout 2400 python -m pytest tests -q -p no:cacheprovider -m gpu > "$out/pytest_gpu.txt" 2>&1
tail -3 "$out/pytest_gpu.txt"
