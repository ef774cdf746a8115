"""Generates the committed CLancIR element-type fixtures types_*.npz from UPSTREAM ITSELF
(oracle/_ref/liblancir_types_ref.so: lancir.h compiled with the pinned flags -O2 -mavx2 -ffp-contract=off by
oracle/types.mk).

Run in the build container (where the reference headers exist):
    python tests/golden/make_types_golden.py
Each types_*.npz holds: geometry, source kind (test_lancir_types.TYPE_FIXTURES), input, upstream CLancIR output,
for double and uint32_t buffers as source and as destination.  Their float outputs carry NaN: they are compared
NaN-aware (cases.value_mismatch).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import lancir_types_oracle as lo  # noqa: E402
from test_lancir_types import TYPE_FIXTURES, fixture_source  # noqa: E402


def main():
    assert lo.have_ref(), "build oracle/_ref first (make -C oracle -f types.mk ref)"
    for i, c in enumerate(TYPE_FIXTURES):
        sw, sh, nw, nh, ch, ti, to, kind = c
        src = fixture_source(c, seed=400 + i)
        r, out = lo.lancir_ref(src, nw, nh, to)
        assert r == nh
        np.savez_compressed(os.path.join(HERE, "types_%02d.npz" % i), src=src, out=out,
                            geom=np.array([sw, sh, nw, nh]), kind=kind)
    print("wrote", len(TYPE_FIXTURES), "CLancIR element-type fixtures")


if __name__ == "__main__":
    main()
