#!/usr/bin/env python
"""Write tests/golden/controllers.npz from the REFERENCE ITSELF: one complete EventsToSignals per instrument
(source/app/MLEventsToSignals.cpp), compiled in place (oracle/_ref/libmlctrl.so).  Run only where the reference tree
exists:

    python -c "from oracle import ctrl_bindings as c; c.build('ref')" && python tests/golden/make_controllers_golden.py

Only controllers.npz is written; no other golden file is touched.  Contents, for each case k (tests/ctrl_cases.py):
  ctrl_k      [C] i32              the requested controllers
  sr_k, proto_k                    sample rate, protocol (0 MIDI, 1 MPE)
  offsets_k   [T][G + 1] i32       the CSR change list of the case's events, in the order the reference applies them
  changes_k   [n] u2, u2, f4       (controller, pad, value)
  out_k       [T][C][G][64] f32    getController(n).output of the reference after every processVector
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))

from oracle.ctrl_bindings import changes_from_events, ref_controllers  # noqa: E402
from tests.ctrl_cases import ALL_CONTROLLERS, special_phrases  # noqa: E402

CASES = (  # (sample rate, protocol, G, T, seed, controllers)
    (44100.0, 0, 5, 24, 41, ALL_CONTROLLERS),
    (48000.0, 1, 4, 20, 42, [128, 74, 1, 123, 0, 7]),
    (96000.0, 0, 3, 40, 43, [7, 128, 120]),
)


def main():
    out = {}
    for k, (sr, proto, G, T, seed, ctrl) in enumerate(CASES):
        phrases = special_phrases(G, T, seed)
        offsets, changes = changes_from_events(phrases, T, protocol=proto)
        out.update({"ctrl_%d" % k: np.array(ctrl, np.int32), "sr_%d" % k: np.float32(sr), "proto_%d" % k: proto,
                    "offsets_%d" % k: offsets, "changes_%d" % k: changes,
                    "out_%d" % k: ref_controllers(phrases, ctrl, T, sr, protocol=proto)})
    path = os.path.join(HERE, "controllers.npz")
    np.savez_compressed(path, **out)
    print("controllers.npz", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
