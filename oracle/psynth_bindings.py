"""ctypes bindings for the end-to-end checker of published signals of mlb::tr::TracedSynth -- TEST INFRASTRUCTURE ONLY.

  ref_psynth  oracle/_ref/libmlpsynth.so: G complete reference AudioContext + Synth objects running the Synth subclass
              of tests/cpp/published_body.h (oracle/ref/mlpsynth.cpp), with the reads of that file after every call;
              only where the reference tree existed at build time.
  ref_signal  one reference PublishedSignal through given writeQuick calls and reads (the same library).

Built by oracle/psynth.mk (`build()` below).  Only tests/ and __graft_entry__ may import this module.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

from madronalib_b200.api import EVENT_DTYPE
from madronalib_b200.graph import BLOCK

_HERE = os.path.dirname(os.path.abspath(__file__))
REF_LIB = os.path.join(_HERE, "_ref", "libmlpsynth.so")

VARIANTS = {"midi": 0, "mpe": 1}  # publishBodySetup's variants
SIGNALS = 3                       # kPublishSignals
READ_WIDTH = 200                  # kPublishReadWidth

_ref = None


def build(target: str = "ref") -> None:
    """The reference-backed checker: a no-op without the reference tree."""
    assert target == "ref"
    subprocess.run(["make", "-f", os.path.join(_HERE, "psynth.mk"), "psynth-ref"], check=True,
                   stdout=subprocess.DEVNULL)


def ref_available() -> bool:
    return os.path.exists(REF_LIB)


def ref_psynth(case: str, n_voices: int, offsets, events, splits, sample_rate: int = 48000, nthreads: int = 0):
    """G reference AudioContext + PublishSynth pairs set up as `case`, run in calls of `splits` vectors: offsets
    [T][G + 1] into events (EVENT_DTYPE, times within the vector) -> (bus [T][2][G][64], counts [calls][3][G],
    dest [calls][3][G][READ_WIDTH])."""
    global _ref
    if _ref is None:
        f = ctypes.CDLL(REF_LIB).mlpsynth_run
        f.restype = None
        f.argtypes = [ctypes.c_int] * 4 + [ctypes.c_void_p] * 3 + [ctypes.c_int] + [ctypes.c_void_p] * 3 + [ctypes.c_int]
        _ref = f
    off = np.ascontiguousarray(offsets, np.int32)
    T, G = off.shape[0], off.shape[1] - 1
    sp = np.ascontiguousarray(splits, np.int32)
    assert sp.sum() == T
    ev = np.ascontiguousarray(events, EVENT_DTYPE)
    bus = np.zeros((T, 2, G, BLOCK), np.float32)
    counts = np.zeros((len(sp), SIGNALS, G), np.int32)
    dest = np.zeros((len(sp), SIGNALS, G, READ_WIDTH), np.float32)
    _ref(G, VARIANTS[case], n_voices, sample_rate, off.ctypes.data, ev.ctypes.data if ev.size else None, sp.ctypes.data,
         len(sp), bus.ctypes.data, counts.ctypes.data, dest.ctypes.data, nthreads)
    return bus, counts, dest


def ref_signal(max_frames: int, max_voices: int, channels: int, octaves: int, calls):
    """One reference SignalProcessor::PublishedSignal.  calls: a list of (stores, mode, frames), stores a list of
    (rows [channels][64] float32, frames) written with writeQuick in order, then one read (mode as publishReadMode's)
    of `frames` frames -> a list of (count, dest [frames * channels]) per call."""
    f = ctypes.CDLL(REF_LIB).mlpsynth_signal_run
    f.restype = ctypes.c_int
    f.argtypes = [ctypes.c_int] * 5 + [ctypes.c_void_p] * 7
    n_stores = np.array([len(st) for st, _, _ in calls], np.int32)
    frames = np.array([fr for st, _, _ in calls for _, fr in st] or [0], np.int32)
    rows = np.ascontiguousarray(np.array([r for st, _, _ in calls for r, _ in st] or np.zeros((1, channels, BLOCK)),
                                         np.float32))
    modes = np.array([m for _, m, _ in calls], np.int32)
    req = np.array([n for _, _, n in calls], np.int32)
    counts = np.zeros(len(calls), np.int32)
    dest = np.zeros(int(req.sum()) * channels + 1, np.float32)
    assert f(max_frames, max_voices, channels, octaves, len(calls), n_stores.ctypes.data, frames.ctypes.data,
             rows.ctypes.data, modes.ctypes.data, req.ctypes.data, counts.ctypes.data, dest.ctypes.data) == 0
    out, at = [], 0
    for c in range(len(calls)):
        n = int(req[c]) * channels
        out.append((int(counts[c]), dest[at:at + n]))
        at += n
    return out
