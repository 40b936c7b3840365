"""ctypes bindings for the two CPU checkers of kernel K11, the smoothed MIDI controllers of the reference's
EventsToSignals (source/app/MLEventsToSignals.cpp:264-285, 431-435) -- TEST INFRASTRUCTURE ONLY.

  port_controllers  oracle/_port/libmlport_ctrl.so: plain-C restatement fed by the CSR change list
                    (oracle/port/mlport_ctrl.c), with the device bank's state layout.
  ref_controllers   oracle/_ref/libmlctrl.so: one complete reference EventsToSignals per instrument
                    (oracle/ref/mlctrl.cpp), fed by events; only where the reference tree existed at build time.

Both are built by oracle/ctrl.mk (`build()` below).  Only tests/, __graft_entry__ and the benchmark tools' parity
legs may import this module.  Nothing under madronalib_b200/ does.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

from madronalib_b200.graph import BLOCK

_HERE = os.path.dirname(os.path.abspath(__file__))
PORT_LIB = os.path.join(_HERE, "_port", "libmlport_ctrl.so")
REF_LIB = os.path.join(_HERE, "_ref", "libmlctrl.so")

_vp = ctypes.c_void_p

CHANGE_DTYPE = np.dtype([("controller", "<u2"), ("pad", "<u2"), ("value", "<f4")])  # mlb_controller_change
EVENT_DTYPE = np.dtype([("type", "u1"), ("channel", "u1"), ("source_idx", "<u2"), ("time", "<i4"),
                        ("value1", "<f4"), ("value2", "<f4")])                           # mlb_event
N_WORDS = 4  # inputValue, target, vectorsRemaining, step


def build(target: str = "port") -> None:
    """target "port": the plain-C checker (anywhere).  target "ref": the reference's EventsToSignals -- a no-op
    without the reference tree."""
    mk = os.path.join(_HERE, "ctrl.mk")
    subprocess.run(["make", "-f", mk, {"port": "ctrl-port", "ref": "ctrl-ref"}[target]], check=True,
                   stdout=subprocess.DEVNULL)


def ref_available() -> bool:
    return os.path.exists(REF_LIB)


def initial_state(G: int, C: int):
    """The state of a fresh bank: words [4][C][G] (vectorsRemaining -1), rows [C][G][64] of +0."""
    words = np.zeros((N_WORDS, C, G), np.uint32)
    words[2] = 0xFFFFFFFF
    return words, np.zeros((C, G, BLOCK), np.float32)


_port = None
_ref = None


def port_controllers(G: int, controllers, offsets: np.ndarray, changes: np.ndarray, sample_rate: float,
                     state=None):
    """offsets [T][G + 1], changes (CHANGE_DTYPE) -> (out [T][C][G][64], words, rows); `state` = (words, rows) to
    start from (copied), else a fresh bank's."""
    global _port
    ctrl = np.ascontiguousarray(controllers, np.int32)
    C = int(ctrl.shape[0])
    off = np.ascontiguousarray(offsets, np.int32)
    assert off.ndim == 2 and off.shape[1] == G + 1, off.shape
    ch = np.ascontiguousarray(changes, CHANGE_DTYPE)
    words, rows = initial_state(G, C) if state is None else (np.array(state[0], np.uint32), np.array(state[1], np.float32))
    assert words.shape == (N_WORDS, C, G) and rows.shape == (C, G, BLOCK)
    T = int(off.shape[0])
    out = np.zeros((T, C, G, BLOCK), np.float32)
    if _port is None:
        if not os.path.exists(PORT_LIB):
            build("port")
        f = ctypes.CDLL(PORT_LIB).mlport_controllers
        f.restype = None
        f.argtypes = [ctypes.c_int] * 3 + [ctypes.c_float] + [_vp] * 6
        _port = f
    _port(G, C, T, float(sample_rate), ctrl.ctypes.data, off.ctypes.data, ch.ctypes.data if ch.size else None,
          words.ctypes.data, rows.ctypes.data, out.ctypes.data)
    return out, words, rows


def ref_controllers(events_per_instrument, controllers, T: int, sample_rate: float, protocol: int = 0,
                    polyphony: int = 4) -> np.ndarray:
    """One reference EventsToSignals per instrument: events_per_instrument[g] is a list of (type, channel,
    source_idx, time, value1[, value2]) with times from the start of vector 0 -> out [T][C][G][64]."""
    global _ref
    ctrl = np.ascontiguousarray(controllers, np.int32)
    G, C = len(events_per_instrument), int(ctrl.shape[0])
    flat = [tuple(e) + (0.0,) * (6 - len(e)) for evs in events_per_instrument for e in evs]
    ev = np.array(flat, EVENT_DTYPE) if flat else np.zeros(1, EVENT_DTYPE)
    ev_off = np.zeros(G + 1, np.int32)
    ev_off[1:] = np.cumsum([len(evs) for evs in events_per_instrument])
    out = np.zeros((T, C, G, BLOCK), np.float32)
    if _ref is None:
        if not os.path.exists(REF_LIB):
            raise FileNotFoundError(REF_LIB + " not built; run oracle.ctrl_bindings.build('ref') where the reference "
                                    "tree exists")
        f = ctypes.CDLL(REF_LIB).mlctrl_run
        f.restype = None
        f.argtypes = [ctypes.c_int] * 3 + [ctypes.c_double] + [ctypes.c_int] * 2 + [_vp] * 4
        _ref = f
    _ref(G, C, int(T), float(sample_rate), int(protocol), int(polyphony), ctrl.ctypes.data, ev_off.ctypes.data,
         ev.ctypes.data, out.ctypes.data)
    return out


def changes_from_events(events_per_instrument, T: int, protocol: int = 0):
    """The CSR change list a router would emit for these events (controller events, and channel pressure in MIDI
    mode), each vector's writes in the order the reference applies them: addEvent inserts at the lower bound of
    (time, type), so of two events with equal time and type the later one added comes first.
    Returns (offsets [T][G + 1], changes)."""
    G = len(events_per_instrument)
    per = [[[] for _ in range(G)] for _ in range(T)]
    for g, evs in enumerate(events_per_instrument):
        for i, e in sorted(enumerate(evs), key=lambda ie: (ie[1][3], ie[1][0], -ie[0])):
            typ, _, src, time, v1 = e[:5]
            t = time // BLOCK
            if not 0 <= t < T:
                continue
            if typ == 6:
                per[t][g].append((min(src, 128), 0, v1))
            elif typ == 9 and protocol == 0:
                per[t][g].append((128, 0, v1))
    offsets = np.zeros((T, G + 1), np.int32)
    flat = []
    for t in range(T):
        for g in range(G):
            offsets[t, g] = len(flat)
            flat += per[t][g]
        offsets[t, G] = len(flat)
    return offsets, np.array(flat, CHANGE_DTYPE)
