#!/usr/bin/env python
"""Write tests/golden/fdtd.npz from the REFERENCE ITSELF: the text of examples/audio-and-midi/fdtd.cpp compiled in place
(oracle/_ref/libmlfdtd.so).  Run only where the reference tree exists:

    python -c "from oracle import fdtd_bindings as f; f.build('ref')" && python tests/golden/make_fdtd_golden.py

Only fdtd.npz is written; no other golden file is touched.  Contents:
  in                 [12][2][4][64]  excitation (seeded noise) and frequency rows (workloads.fdtd_inputs) of 4 membranes
  out_ftz0/1         [12][2][4][64]  processFDTDModel's two rows, IEEE / under UsingFlushDenormalsToZero
  state_ftz0/1       [4][2][16][16]  the z^-1 and z^-2 surfaces afterwards
  example_head       [16][2][64]     the first 16 vectors of the example's own processFDTD (AudioContext(0, 2, 48000))
  example_sha256     [32] u8         SHA-256 of all 800 vectors ([800][2][64] little-endian f32; three impulses), which
                                     keeps the file small
"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))

from madronalib_b200 import workloads as wl  # noqa: E402
from oracle.fdtd_bindings import RefFdtd  # noqa: E402

FDTD_V, FDTD_T, FDTD_EXAMPLE_VECTORS = 4, 12, 800


def main():
    R = RefFdtd()
    inp = wl.fdtd_inputs(FDTD_V, FDTD_T, t0=0)
    inp[:, 0] = np.random.default_rng(21).uniform(-0.1, 0.1, (FDTD_T, FDTD_V, 64)).astype(np.float32)
    out = {"in": inp}
    for ftz in (0, 1):
        y, st, _ = R.run(inp, ftz=bool(ftz))
        out["out_ftz%d" % ftz], out["state_ftz%d" % ftz] = y, st
    ex = np.ascontiguousarray(R.example(FDTD_EXAMPLE_VECTORS), "<f4")
    out["example_head"] = ex[:16]
    out["example_sha256"] = np.frombuffer(hashlib.sha256(ex.tobytes()).digest(), np.uint8)
    np.savez_compressed(os.path.join(HERE, "fdtd.npz"), **out)
    print("fdtd.npz", os.path.getsize(os.path.join(HERE, "fdtd.npz")), "bytes")


if __name__ == "__main__":
    main()
