"""ctypes bindings for the two CPU checkers of kernel K9 (the FDTD membrane of the reference's
examples/audio-and-midi/fdtd.cpp) -- TEST INFRASTRUCTURE ONLY.

  port_fdtd   oracle/_port/libmlport_fdtd.so: plain-C restatement (oracle/port/mlport_fdtd.c), any sample rate.
  RefFdtd     oracle/_ref/libmlfdtd.so: the example's own text compiled against the reference (oracle/ref/mlfdtd.cpp),
              48 kHz as the example fixes it; only where the reference tree existed at build time.

Both are built by oracle/fdtd.mk (`build()` below).  Only tests/, __graft_entry__ and the benchmark tools' parity and
CPU legs may import this module.  Nothing under madronalib_b200/ does.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
import sys
from typing import Optional

import numpy as np

from madronalib_b200.graph import BLOCK

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
PORT_LIB = os.path.join(_HERE, "_port", "libmlport_fdtd.so")
FDTD_LIB = os.path.join(_HERE, "_ref", "libmlfdtd.so")

_vp = ctypes.c_void_p


def build(target: str = "port") -> None:
    """target "port": the plain-C checker (anywhere).  target "ref": extract the example's text from the reference tree
    (tests/cpp/make_fdtd_body.py, git-ignored output) and compile it against the reference -- a no-op without the
    reference tree."""
    mk = os.path.join(_HERE, "fdtd.mk")
    if target == "port":
        subprocess.run(["make", "-f", mk, "fdtd-port"], check=True, stdout=subprocess.DEVNULL)
    elif target == "ref":
        subprocess.run([sys.executable, os.path.join(_ROOT, "tests", "cpp", "make_fdtd_body.py")], check=True,
                       stdout=subprocess.DEVNULL)
        subprocess.run(["make", "-f", mk, "fdtd-ref"], check=True, stdout=subprocess.DEVNULL)
    else:
        raise ValueError(target)


def fdtd_ref_available() -> bool:
    return os.path.exists(FDTD_LIB)


def _ptr(a: Optional[np.ndarray]):
    return None if a is None else a.ctypes.data_as(_vp)


def _fdtd_shapes(inp, state, V, in_planes):
    inp = np.ascontiguousarray(inp, np.float32)
    assert inp.ndim == 4 and inp.shape[1:] == (in_planes, V, BLOCK), inp.shape
    st = np.zeros((V, 2, 16, 16), np.float32) if state is None else np.array(state, np.float32, order="C")
    assert st.shape == (V, 2, 16, 16), st.shape
    return inp, st


_port = None


def port_fdtd(inp: np.ndarray, state: Optional[np.ndarray] = None, ftz: bool = False, sample_rate: float = 48000.0,
              excite_plane: int = 0, freq_plane: int = 1):
    """The plain-C port of FDTDState + processFDTDModel for V instances: inp [T][in_planes][V][64] ->
    (out [T][2][V][64], state after [V][2][16][16]).  state None = all surfaces zero."""
    global _port
    T, P, V = inp.shape[0], inp.shape[1], inp.shape[2]
    inp, st = _fdtd_shapes(inp, state, V, P)
    out = np.zeros((T, 2, V, BLOCK), np.float32)
    if _port is None:
        if not os.path.exists(PORT_LIB):
            build("port")
        f = ctypes.CDLL(PORT_LIB).mlport_fdtd
        f.restype = None
        f.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_float, ctypes.c_int, ctypes.c_int, ctypes.c_int, _vp, _vp,
                      _vp, ctypes.c_int]
        _port = f
    _port(V, T, sample_rate, P, excite_plane, freq_plane, _ptr(inp), _ptr(st), _ptr(out), int(ftz))
    return out, st


class RefFdtd:
    """The reference's own FDTD example text compiled in place (oracle/_ref/libmlfdtd.so); 48 kHz only."""

    def __init__(self):
        if not os.path.exists(FDTD_LIB):
            raise FileNotFoundError(FDTD_LIB + " not built; run oracle.fdtd_bindings.build('ref') where the "
                                    "reference tree exists")
        self.lib = L = ctypes.CDLL(FDTD_LIB)
        L.mlfdtd_run.restype = ctypes.c_double
        L.mlfdtd_run.argtypes = [ctypes.c_int, ctypes.c_int, _vp, _vp, _vp, _vp, ctypes.c_int, ctypes.c_int]
        L.mlfdtd_example.restype = None
        L.mlfdtd_example.argtypes = [ctypes.c_int, _vp]

    def run(self, inp: np.ndarray, state: Optional[np.ndarray] = None, ftz: bool = False, nthreads: int = 1):
        """processFDTDModel on V instances: inp [T][2][V][64] (excitation, frequency) ->
        (out [T][2][V][64], state after [V][2][16][16], seconds)."""
        T, V = inp.shape[0], inp.shape[2]
        inp, st = _fdtd_shapes(inp, state, V, 2)
        out = np.zeros((T, 2, V, BLOCK), np.float32)
        sec = self.lib.mlfdtd_run(V, T, _ptr(inp), _ptr(st), _ptr(st), _ptr(out), int(ftz), int(nthreads))
        return out, st, float(sec)

    def example(self, n_vectors: int) -> np.ndarray:
        """The example's own processFDTD with an AudioContext(0, 2, 48000): -> [n_vectors][2][64]."""
        out = np.zeros((n_vectors, 2, BLOCK), np.float32)
        self.lib.mlfdtd_example(n_vectors, _ptr(out))
        return out
