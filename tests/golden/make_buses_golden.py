#!/usr/bin/env python
"""Write tests/golden/buses.npz from the REFERENCE ITSELF: Synth::processVector (source/app/MLSynth.h:36-60) compiled in
place (oracle/_ref/libmlsynth.so).  Run only where the reference tree exists:

    python -c "from oracle import bus_bindings as b; b.build('ref')" && python tests/golden/make_buses_golden.py

Only buses.npz is written; no other golden file is touched.  Contents (tests/bus_cases.py):
  first, count     [9] i32            the bus layout over 40 voices: counts 0, 1, 3, 16, gaps and overlaps
  rows_p1, rows_p3 [2][P][40][64]     voice rows with -0, +-inf, NaN, subnormals and cancelling large magnitudes
  bus_p1, bus_p3   [2][P][9][64]      the reference Synth's outputs, one Synth(count) and AudioContext(0, P, 48000) per bus
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))

from oracle.bus_bindings import ref_buses  # noqa: E402
from tests.bus_cases import GOLDEN_COUNT, GOLDEN_FIRST, GOLDEN_V, special_rows  # noqa: E402


def main():
    out = {"first": GOLDEN_FIRST, "count": GOLDEN_COUNT}
    for P, seed in ((1, 31), (3, 32)):
        rows = special_rows(2, P, GOLDEN_V, seed)
        out["rows_p%d" % P] = rows
        out["bus_p%d" % P] = ref_buses(rows, GOLDEN_FIRST, GOLDEN_COUNT)
    path = os.path.join(HERE, "buses.npz")
    np.savez_compressed(path, **out)
    print("buses.npz", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
