"""ctypes bindings for the two CPU checkers of kernel K10, the per-instrument output buses of the reference's
Synth::processVector (source/app/MLSynth.h:36-60) -- TEST INFRASTRUCTURE ONLY.

  port_buses  oracle/_port/libmlport_bus.so: plain-C strict-order restatement (oracle/port/mlport_bus.c), any bus size.
  ref_buses   oracle/_ref/libmlsynth.so: the reference's own Synth compiled in place (oracle/ref/mlsynth.cpp); buses of
              at most 16 voices (a Synth reads at most EventsToSignals::kMaxVoices); only where the reference tree
              existed at build time.

Both are built by oracle/synth.mk (`build()` below).  Only tests/, __graft_entry__ and the benchmark tools' parity
legs may import this module.  Nothing under madronalib_b200/ does.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

from madronalib_b200.graph import BLOCK

_HERE = os.path.dirname(os.path.abspath(__file__))
PORT_LIB = os.path.join(_HERE, "_port", "libmlport_bus.so")
SYNTH_LIB = os.path.join(_HERE, "_ref", "libmlsynth.so")
MAX_REF_VOICES = 16  # EventsToSignals::kMaxVoices (MLEventsToSignals.h:47)

_vp = ctypes.c_void_p
_ARGS = [ctypes.c_int] * 4 + [_vp] * 4


def build(target: str = "port") -> None:
    """target "port": the plain-C checker (anywhere).  target "ref": the reference's Synth -- a no-op without the
    reference tree."""
    mk = os.path.join(_HERE, "synth.mk")
    subprocess.run(["make", "-f", mk, {"port": "bus-port", "ref": "synth-ref"}[target]], check=True,
                   stdout=subprocess.DEVNULL)


def synth_ref_available() -> bool:
    return os.path.exists(SYNTH_LIB)


def _shapes(rows, first, count):
    rows = np.ascontiguousarray(rows, np.float32)
    assert rows.ndim == 4 and rows.shape[3] == BLOCK, rows.shape
    fv, vc = np.ascontiguousarray(first, np.int32), np.ascontiguousarray(count, np.int32)
    assert fv.ndim == 1 and fv.shape == vc.shape
    assert (fv >= 0).all() and (vc >= 0).all() and (fv.astype(np.int64) + vc <= rows.shape[2]).all()
    T, P, V, _ = rows.shape
    return rows, fv, vc, np.zeros((T, P, fv.shape[0], BLOCK), np.float32)


_port = None
_ref = None


def port_buses(rows: np.ndarray, first, count) -> np.ndarray:
    """rows [T][P][V][64] -> bus [T][P][G][64], bus g the strict-order sum from +0 of rows [first[g], +count[g])."""
    global _port
    rows, fv, vc, bus = _shapes(rows, first, count)
    if _port is None:
        if not os.path.exists(PORT_LIB):
            build("port")
        f = ctypes.CDLL(PORT_LIB).mlport_buses
        f.restype = None
        f.argtypes = _ARGS
        _port = f
    T, P, V, _ = rows.shape
    _port(V, fv.shape[0], P, T, fv.ctypes.data, vc.ctypes.data, rows.ctypes.data, bus.ctypes.data)
    return bus


def ref_buses(rows: np.ndarray, first, count, sample_rate: int = 48000) -> np.ndarray:
    """The reference's Synth::processVector per bus, one Synth(count) and AudioContext(0, P, sample_rate) each.
    Raises ValueError, having run nothing, when a bus has more than 16 voices."""
    global _ref
    rows, fv, vc, bus = _shapes(rows, first, count)
    if _ref is None:
        if not os.path.exists(SYNTH_LIB):
            raise FileNotFoundError(SYNTH_LIB + " not built; run oracle.bus_bindings.build('ref') where the reference "
                                    "tree exists")
        f = ctypes.CDLL(SYNTH_LIB).mlsynth_buses
        f.restype = ctypes.c_int
        f.argtypes = _ARGS + [ctypes.c_int]
        _ref = f
    T, P, V, _ = rows.shape
    rc = _ref(V, fv.shape[0], P, T, fv.ctypes.data, vc.ctypes.data, rows.ctypes.data, bus.ctypes.data,
              int(sample_rate))
    if rc != 0:
        g = -1 - rc
        raise ValueError(f"bus {g} has {int(vc[g])} voices: a Synth reads at most {MAX_REF_VOICES}")
    return bus
