#!/bin/bash
# One H100 session for the shared halo exchange (avir_b200/csrc/peer_mailbox.cu: band partition, PeerExchange,
# push_rows), run as parts in the order given:
#   tests:   the card and the GPUs visible, the sharded tests of both resizers, the host calls, the sharded cases of
#            the parity, stream and layout tests, tests/test_shard_partition.py, the multi-GPU tests (they skip
#            with fewer GPUs than they need), smoke()
#   suite:   the GPU suite except tests/test_gpu_extents.py
#   extents: tests/test_gpu_extents.py
#   bench:   bench lines of this change and its parent commit, alternating (the first of each round alternating
#            too), 2 of each
# usage: profiles/h100_shard_exchange.sh <out dir> <parent tree> <part>...
#   <parent tree>: a built copy of the parent commit's files
out=${1:?usage: profiles/h100_shard_exchange.sh <out dir> <parent tree> <part>...}
parent=${2:?usage: profiles/h100_shard_exchange.sh <out dir> <parent tree> <part>...}
shift 2
mkdir -p "$out"
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv > "$out/gpu.txt" 2>&1
nvidia-smi -L >> "$out/gpu.txt" 2>&1
cat "$out/gpu.txt"
python -c "import __graft_entry__ as g; g.build()" > "$out/build.txt" 2>&1 || { tail -40 "$out/build.txt"; exit 1; }
for part in "$@"; do
case "$part" in
tests)
    timeout 600 python -m pytest -q -p no:cacheprovider -m gpu -rfs \
        tests/test_gpu_lancir_sharded.py tests/test_gpu_sharded_errd.py tests/test_gpu_host_calls.py \
        tests/test_shard_partition.py tests/test_gpu_nccl.py > "$out/pytest_sharded.txt" 2>&1
    tail -12 "$out/pytest_sharded.txt"
    timeout 600 python -m pytest -q -p no:cacheprovider -m gpu -rfs -k "shard" \
        tests/test_gpu_parity.py tests/test_gpu_streams.py tests/test_gpu_layouts.py > "$out/pytest_sharded_k.txt" 2>&1
    tail -4 "$out/pytest_sharded_k.txt"
    timeout 120 python -c "import __graft_entry__ as g; g.smoke()" > "$out/smoke.txt" 2>&1
    tail -1 "$out/smoke.txt"
    ;;
suite)
    timeout 900 python -m pytest tests -q -p no:cacheprovider -m gpu -rfs --ignore=tests/test_gpu_extents.py \
        > "$out/pytest_gpu.txt" 2>&1
    tail -16 "$out/pytest_gpu.txt"
    ;;
extents)
    timeout 540 python -m pytest tests/test_gpu_extents.py -q -p no:cacheprovider -m gpu -rfs \
        > "$out/pytest_extents.txt" 2>&1
    tail -3 "$out/pytest_extents.txt"
    ;;
bench)
    for run in 1 2; do
        order="this parent"; [ $((run % 2)) = 0 ] && order="parent this"
        for tree in $order; do
            dir=.; [ "$tree" = parent ] && dir=$parent
            (cd "$dir" && timeout 240 python bench.py --gpus 1 --steps 20 --warmup 3 --no-cpu-baseline) \
                > "$out/bench_${tree}_$run.json" 2> "$out/bench_${tree}_$run.err"
            echo "$tree $run: $(cut -c1-200 "$out/bench_${tree}_$run.json")"
        done
    done
    ;;
esac
done
