"""ctypes bindings for the end-to-end checker of a traced Synth that overrides processVector -- TEST INFRASTRUCTURE ONLY.

  ref_synth  oracle/_ref/libmlfxsynth.so: G complete reference AudioContext + Synth objects running the Synth subclass
             of tests/cpp/fx_synth_body.h (oracle/ref/mlfxsynth.cpp); only where the reference tree existed at build
             time.

Built by oracle/fxsynth.mk (`build()` below).  Only tests/, tools/ and __graft_entry__ may import this module.  Nothing
under madronalib_b200/ does.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

from madronalib_b200.api import EVENT_DTYPE, TRANSPORT_DTYPE
from madronalib_b200.graph import BLOCK

_HERE = os.path.dirname(os.path.abspath(__file__))
REF_LIB = os.path.join(_HERE, "_ref", "libmlfxsynth.so")

VARIANTS = {"midi": 0, "mpe": 1}  # fxSynthSetup's variants
N_OUT = 3

_ref = None


def build(target: str = "ref") -> None:
    """The reference-backed checker: a no-op without the reference tree."""
    assert target == "ref"
    subprocess.run(["make", "-f", os.path.join(_HERE, "fxsynth.mk"), "fxsynth-ref"], check=True,
                   stdout=subprocess.DEVNULL)


def ref_available() -> bool:
    return os.path.exists(REF_LIB)


def ref_synth(case: str, n_voices: int, offsets, events, time_offsets, transports, sample_rate: int = 48000,
              nthreads: int = 0):
    """G reference AudioContext + FxSynth pairs set up as `case`: offsets / time_offsets [T][G + 1] into events
    (EVENT_DTYPE, times within the vector) and transports (TRANSPORT_DTYPE) -> (bus [T][3][G][64], seconds)."""
    global _ref
    if _ref is None:
        f = ctypes.CDLL(REF_LIB).mlfxsynth_run
        f.restype = ctypes.c_double
        f.argtypes = [ctypes.c_int] * 5 + [ctypes.c_void_p] * 5 + [ctypes.c_int]
        _ref = f
    off = np.ascontiguousarray(offsets, np.int32)
    toff = np.ascontiguousarray(time_offsets, np.int32)
    T, G = off.shape[0], off.shape[1] - 1
    assert toff.shape == off.shape
    ev = np.ascontiguousarray(events, EVENT_DTYPE)
    tr = np.ascontiguousarray(transports, TRANSPORT_DTYPE)
    bus = np.zeros((T, N_OUT, G, BLOCK), np.float32)
    sec = _ref(G, T, VARIANTS[case], n_voices, sample_rate, off.ctypes.data, ev.ctypes.data if ev.size else None,
               toff.ctypes.data, tr.ctypes.data if tr.size else None, bus.ctypes.data, nthreads)
    return bus, float(sec)
