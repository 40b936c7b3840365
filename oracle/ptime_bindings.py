"""ctypes bindings for the two CPU checkers of kernel K13, the host-transport beat phase of the reference's
AudioContext::ProcessTime (source/app/MLAudioContext.cpp:16-101) -- TEST INFRASTRUCTURE ONLY.

  port_process_time  oracle/_port/libmlport_ptime.so: plain-C restatement fed by the CSR transport list
                     (oracle/port/mlport_ptime.c), with the device bank's state layout.
  ref_process_time   oracle/_ref/libmlptime.so: one complete reference AudioContext per instrument
                     (oracle/ref/mlptime.cpp); only where the reference tree existed at build time.

Both are built by oracle/ptime.mk (`build()` below).  Only tests/, __graft_entry__ and the benchmark tools' parity
legs may import this module.  Nothing under madronalib_b200/ does.
"""
from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

from madronalib_b200.api import TRANSPORT_DTYPE  # mlb_transport
from madronalib_b200.graph import BLOCK

_HERE = os.path.dirname(os.path.abspath(__file__))
PORT_LIB = os.path.join(_HERE, "_port", "libmlport_ptime.so")
REF_LIB = os.path.join(_HERE, "_ref", "libmlptime.so")

_vp = ctypes.c_void_p

N_WORDS = 10  # MLB_PT_WORDS
OMEGA, DPDT, PPQ_POS1, PPQ_PHASE1, PLAYING1, ACTIVE1, SAMPLES_PREV, SAMPLES_START, BPM, SAMPLE_RATE = range(N_WORDS)
FLOAT_WORDS, DOUBLE_WORDS = (OMEGA,), (DPDT, PPQ_POS1, PPQ_PHASE1, BPM, SAMPLE_RATE)


def build(target: str = "port") -> None:
    """target "port": the plain-C checker (anywhere).  target "ref": the reference's AudioContext -- a no-op without
    the reference tree."""
    mk = os.path.join(_HERE, "ptime.mk")
    subprocess.run(["make", "-f", mk, {"port": "ptime-port", "ref": "ptime-ref"}[target]], check=True,
                   stdout=subprocess.DEVNULL)


def ref_available() -> bool:
    return os.path.exists(REF_LIB)


def initial_state(G: int, sample_rate: float) -> np.ndarray:
    """The words [10][G] uint64 of AudioContext(nIn, nOut, sample_rate): ppqPos1_ = -1, sampleRate, the rest 0."""
    w = np.zeros((N_WORDS, G), np.uint64)
    w[PPQ_POS1] = np.float64(-1.0).view(np.uint64)
    w[SAMPLE_RATE] = np.float64(sample_rate).view(np.uint64)
    return w


_port = None
_port_clear = None
_ref = None


def _port_lib():
    global _port, _port_clear
    if _port is None:
        if not os.path.exists(PORT_LIB):
            build("port")
        L = ctypes.CDLL(PORT_LIB)
        _port = L.mlport_process_time
        _port.restype = None
        _port.argtypes = [ctypes.c_int] * 2 + [_vp] * 4
        _port_clear = L.mlport_process_time_clear
        _port_clear.restype = None
        _port_clear.argtypes = [ctypes.c_int, _vp]
    return _port, _port_clear


def port_process_time(G: int, offsets: np.ndarray, transports: np.ndarray, sample_rate: float = 48000.0,
                      state=None):
    """offsets [T][G + 1], transports (TRANSPORT_DTYPE) -> (out [T][G][64], words [10][G]); `state` = words to start
    from (copied), else a fresh bank's."""
    run, _ = _port_lib()
    off = np.ascontiguousarray(offsets, np.int32)
    assert off.ndim == 2 and off.shape[1] == G + 1, off.shape
    tr = np.ascontiguousarray(transports, TRANSPORT_DTYPE)
    words = initial_state(G, sample_rate) if state is None else np.array(state, np.uint64)
    assert words.shape == (N_WORDS, G)
    T = int(off.shape[0])
    out = np.zeros((T, G, BLOCK), np.float32)
    run(G, T, off.ctypes.data, tr.ctypes.data if tr.size else None, words.ctypes.data, out.ctypes.data)
    return out, words


def port_clear(words: np.ndarray) -> np.ndarray:
    """ProcessTime::clear() of every clock, on a copy of words [10][G]."""
    _, clear = _port_lib()
    w = np.array(words, np.uint64)
    clear(int(w.shape[1]), w.ctypes.data)
    return w


def ref_process_time(G: int, offsets: np.ndarray, transports: np.ndarray, sample_rate: int = 48000,
                     clear_before=None):
    """One reference AudioContext(0, 0, sample_rate) per instrument -> (out [T][G][64], words [10][G]);
    clear_before[t] true: AudioContext::clear() before vector t's updates."""
    global _ref
    off = np.ascontiguousarray(offsets, np.int32)
    tr = np.ascontiguousarray(transports, TRANSPORT_DTYPE)
    T = int(off.shape[0])
    clr = None if clear_before is None else np.ascontiguousarray(clear_before, np.int32)
    out = np.zeros((T, G, BLOCK), np.float32)
    words = np.zeros((N_WORDS, G), np.uint64)
    if _ref is None:
        if not os.path.exists(REF_LIB):
            raise FileNotFoundError(REF_LIB + " not built; run oracle.ptime_bindings.build('ref') where the reference "
                                    "tree exists")
        f = ctypes.CDLL(REF_LIB).mlptime_run
        f.restype = None
        f.argtypes = [ctypes.c_int] * 3 + [_vp] * 5
        _ref = f
    _ref(G, T, int(sample_rate), off.ctypes.data, tr.ctypes.data if tr.size else None,
         None if clr is None else clr.ctypes.data, out.ctypes.data, words.ctypes.data)
    return out, words


def same_words(got: np.ndarray, want: np.ndarray) -> np.ndarray:
    """Per word, equal bits, or both NaN for the float and double words (x86 and sm_90 NaN payloads differ)."""
    got, want = np.asarray(got, np.uint64), np.asarray(want, np.uint64)
    eq = got == want
    for k in FLOAT_WORDS:
        a = (got[k] & 0xFFFFFFFF).astype(np.uint32).view(np.float32)
        b = (want[k] & 0xFFFFFFFF).astype(np.uint32).view(np.float32)
        eq[k] |= np.isnan(a) & np.isnan(b)
    for k in DOUBLE_WORDS:
        eq[k] |= np.isnan(got[k].view(np.float64)) & np.isnan(want[k].view(np.float64))
    return eq
