#!/bin/bash
# One H100 session, in four parts, for the shared host-call path (avir_b200/csrc/host_call.cu):
#   tests:   the card, tests/test_gpu_host_calls.py on the parent commit's library and on this one, the host-call
#            tests of tests/test_gpu_streams.py, smoke()
#   suite:   the GPU suite except tests/test_gpu_extents.py
#   extents: tests/test_gpu_extents.py
#   bench:   bench lines of this change and its parent commit, alternating (the first of each round
#            alternating too), [rounds] of each (default 2)
#   pageable: the bench's pageable_f32 call alone (CImageResizer::resizeImage, 8K -> 4K RGBA float from and to
#            pageable numpy buffers, 15 row bands through the bounce buffers): [rounds] processes per tree,
#            alternating, 2 warm-up and 15 timed calls each
# usage: profiles/h100_host_call.sh <out dir> <parent tree> tests|suite|extents|bench [rounds]
#   <parent tree>: a copy of the parent commit's files, with tests/test_gpu_host_calls.py copied into its tests/
out=${1:?usage: profiles/h100_host_call.sh <out dir> <parent tree> tests|suite|extents|bench}
parent=${2:?usage: profiles/h100_host_call.sh <out dir> <parent tree> tests|suite|extents|bench}
mkdir -p "$out"
nvidia-smi --query-gpu=name,power.limit,clocks.max.sm --format=csv > "$out/gpu_$3.txt" 2>&1
cat "$out/gpu_$3.txt"
python -c "import __graft_entry__ as g; g.build()" > "$out/build_$3.txt" 2>&1 || { tail -40 "$out/build_$3.txt"; exit 1; }
case "$3" in
tests)
    (cd "$parent" && python -c "import __graft_entry__ as g; g.build()") > "$out/build_parent.txt" 2>&1 \
        || { tail -40 "$out/build_parent.txt"; exit 1; }
    (cd "$parent" && timeout 200 python -m pytest tests/test_gpu_host_calls.py -q -p no:cacheprovider -m gpu -rfs) \
        > "$out/pytest_host_calls_parent.txt" 2>&1
    grep -E "^FAILED|passed|failed" "$out/pytest_host_calls_parent.txt" | cut -c1-160
    timeout 200 python -m pytest tests/test_gpu_host_calls.py tests/test_gpu_streams.py -q -p no:cacheprovider -m gpu \
        -k "host" -rfs > "$out/pytest_host_calls.txt" 2>&1
    tail -4 "$out/pytest_host_calls.txt"
    timeout 120 python -c "import __graft_entry__ as g; g.smoke()" > "$out/smoke.txt" 2>&1
    tail -1 "$out/smoke.txt"
    ;;
suite)
    timeout 540 python -m pytest tests -q -p no:cacheprovider -m gpu -rfs --ignore=tests/test_gpu_extents.py \
        > "$out/pytest_gpu.txt" 2>&1
    tail -6 "$out/pytest_gpu.txt"
    ;;
extents)
    timeout 540 python -m pytest tests/test_gpu_extents.py -q -p no:cacheprovider -m gpu -rfs \
        > "$out/pytest_extents.txt" 2>&1
    tail -3 "$out/pytest_extents.txt"
    ;;
bench)
    for run in $(seq "${4:-2}"); do
        order="this parent"; [ $((run % 2)) = 0 ] && order="parent this"
        for tree in $order; do
            dir=.; [ "$tree" = parent ] && dir=$parent
            (cd "$dir" && timeout 240 python bench.py --gpus 1 --steps 20 --warmup 3 --no-cpu-baseline) \
                > "$out/bench_${tree}_$run.json" 2> "$out/bench_${tree}_$run.err"
            echo "$tree $run: $(cut -c1-160 "$out/bench_${tree}_$run.json")"
        done
    done
    ;;
pageable)
    code='import sys, time, numpy as np; sys.path[:0] = [".", "tests"]; import avir_b200 as ab
rs = ab.CImageResizer(16, 0, 0, 2)  # fpclass_float8_dil, as the bench
src = np.random.default_rng(1).random((4320, 7680, 4), dtype=np.float32); dst = np.empty((2160, 3840, 4), np.float32)
ts = []
for i in range(17):
    t0 = time.perf_counter(); rs.resizeImage(src, 3840, 2160, 0.0, NewBuf=dst); ts.append(time.perf_counter() - t0)
ts = sorted(ts[2:]); print("%.2f %.2f %.2f" % (ts[len(ts) // 2] * 1e3, ts[0] * 1e3, ts[-1] * 1e3))'
    for run in $(seq "${4:-2}"); do
        order="this parent"; [ $((run % 2)) = 0 ] && order="parent this"
        for tree in $order; do
            dir=.; [ "$tree" = parent ] && dir=$parent
            echo "$tree $run: ms per call median min max $(cd "$dir" && timeout 120 python -c "$code" 2>&1 | tail -1)" \
                | tee -a "$out/pageable.txt"
        done
    done
    ;;
esac
