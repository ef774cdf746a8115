#!/bin/bash
# One H100 session for the pass-request refactor (one PassRequest per pass, one run_pass, one family decision):
# the card, the GPU tests (the rest of the suite needs no GPU), smoke(), the bench line of this change and its parent commit
# alternating, and the per-pass times of the tile and generic families (pass_times.py --family 2 / 1, which the
# bench barely exercises) on both trees with their output hashes.
# usage: profiles/h100_pass_request.sh <out dir> [<parent tree, built>] [tests | perf]  (default: both parts)
out=${1:?usage: profiles/h100_pass_request.sh <out dir> [<parent tree>] [tests | perf]}
parent=$2
part=${3:-all}
mkdir -p "$out"
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm,clocks.sm --format=csv > "$out/gpu.txt" 2>&1
cat "$out/gpu.txt"
python -c "import __graft_entry__ as g; g.build()" > "$out/build.txt" 2>&1 || { tail -40 "$out/build.txt"; exit 1; }
if [ "$part" != perf ]; then
timeout 1500 python -m pytest tests -q -p no:cacheprovider -m gpu -rs > "$out/pytest_gpu.txt" 2>&1
tail -2 "$out/pytest_gpu.txt"
fi
[ "$part" = tests ] && exit 0
timeout 300 python -c "import __graft_entry__ as g; g.smoke(); print('smoke ok')" > "$out/smoke.txt" 2>&1
tail -1 "$out/smoke.txt"
for run in 1 2 3; do
    timeout 300 python bench.py --gpus 1 --steps 20 --warmup 3 --no-cpu-baseline > "$out/bench_new_$run.json" 2> "$out/bench_new_$run.err"
    cut -c1-200 "$out/bench_new_$run.json"
    if [ -n "$parent" ]; then
        (cd "$parent" && timeout 300 python bench.py --gpus 1 --steps 20 --warmup 3 --no-cpu-baseline) > "$out/bench_parent_$run.json" 2> "$out/bench_parent_$run.err"
        cut -c1-200 "$out/bench_parent_$run.json"
    fi
done
for fam in 1 2; do
    for cfg in cfg3 rgb; do
        timeout 300 python profiles/pass_times.py --cfg $cfg --family $fam --n 20 > "$out/pass_new_${cfg}_f$fam.json" 2>&1
        tail -1 "$out/pass_new_${cfg}_f$fam.json"
        if [ -n "$parent" ]; then
            (cd "$parent" && timeout 300 python profiles/pass_times.py --cfg $cfg --family $fam --n 20) > "$out/pass_parent_${cfg}_f$fam.json" 2>&1
            tail -1 "$out/pass_parent_${cfg}_f$fam.json"
        fi
    done
done
