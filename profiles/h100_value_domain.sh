#!/bin/bash
# One H100 session for the value-domain tests: the card, tests/test_value_domain.py alone, the whole
# suite, smoke() and the bench line.
# usage: profiles/h100_value_domain.sh <out dir>
out=${1:?usage: profiles/h100_value_domain.sh <out dir>}
mkdir -p "$out"
nvidia-smi --query-gpu=name,power.limit --format=csv > "$out/gpu.txt" 2>&1
python -c "import __graft_entry__ as g; g.build()" > "$out/build.txt" 2>&1 || { tail -40 "$out/build.txt"; exit 1; }
timeout 600 python -m pytest -q -p no:cacheprovider -m gpu -rs tests/test_value_domain.py > "$out/pytest_value_domain.txt" 2>&1
tail -3 "$out/pytest_value_domain.txt"
timeout 1500 python -m pytest -q -p no:cacheprovider > "$out/pytest_full.txt" 2>&1
tail -3 "$out/pytest_full.txt"
timeout 300 python -c "import __graft_entry__ as g; g.smoke()" > "$out/smoke.txt" 2>&1
tail -2 "$out/smoke.txt"
timeout 900 python bench.py --gpus 1 --steps 20 --warmup 3 > "$out/bench_n1.json" 2> "$out/bench_n1.err"
cut -c1-600 "$out/bench_n1.json"
