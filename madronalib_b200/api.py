"""Python host mirror of the C ABI in ``include/mlb200.h`` (ctypes over libmlb200.so).

The library is the product; this module only marshals pointers.  There is NO CPU
fallback: if ``libmlb200.so`` is missing, or no sm_90 GPU is visible, calls raise.

``VoiceGraph`` is the batched analogue of the reference's ``Bank<T, ROWS>``
(reference: source/DSP/MLDSPFunctional.h:321-360) with ``ROWS`` chosen at run time:
``process`` = n_blocks successive ``Bank::operator()`` calls fused in one launch.
"""
from __future__ import annotations

import ctypes
import os
from typing import Optional

import numpy as np

from .graph import BLOCK, GraphSpec, Layout, Node, OP_ID

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmlb200.so")

_vp = ctypes.c_void_p
_cf = ctypes.c_float

FLAG_EXACT = 0
FLAG_FAST = 1
FLAG_FORCE_GENERIC = 2
FLAG_SINGLE_STAGE = 4


class MlbError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"mlb200 error {code}: {msg}")
        self.code = code


_lib = None


def lib() -> ctypes.CDLL:
    """Load libmlb200.so (built by ``python -m madronalib_b200.build``); fail loudly if absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise FileNotFoundError(
            f"{LIB_PATH} not found: build it with `python -m madronalib_b200.build` "
            "(there is no CPU fallback)")
    L = ctypes.CDLL(LIB_PATH)
    L.mlb_last_error.restype = ctypes.c_char_p
    L.mlb_op_name.restype = ctypes.c_char_p
    L.mlb_op_name.argtypes = [ctypes.c_int]
    L.mlb_op_info.argtypes = [ctypes.c_int, _vp, _vp, _vp]
    L.mlb_graph_layout.argtypes = [_vp, ctypes.c_int, _vp, _vp, _vp]
    L.mlb_kernel_launches.restype = ctypes.c_longlong
    L.mlb_init.argtypes = [ctypes.c_int]
    L.mlb_graph_create.argtypes = [_vp, ctypes.c_int, _vp, ctypes.c_int, ctypes.c_int,
                                   ctypes.c_uint, ctypes.POINTER(_vp)]
    L.mlb_graph_destroy.argtypes = [_vp]
    L.mlb_graph_layout_of.argtypes = [_vp, _vp]
    L.mlb_graph_plan.argtypes = [_vp, ctypes.c_int, _vp, ctypes.c_int, ctypes.c_int, ctypes.c_uint, _vp, _vp, _vp]
    L.mlb_graph_kernel_name.restype = ctypes.c_char_p
    L.mlb_graph_kernel_name.argtypes = [_vp]
    L.mlb_graph_set_coefs.argtypes = [_vp, _vp]
    L.mlb_graph_set_state.argtypes = [_vp, _vp]
    L.mlb_graph_get_state.argtypes = [_vp, _vp]
    L.mlb_graph_clear_delays.argtypes = [_vp]
    L.mlb_graph_delay_bytes.restype = ctypes.c_size_t
    L.mlb_graph_delay_bytes.argtypes = [_vp]
    L.mlb_graph_reserve_sms.argtypes = [_vp, ctypes.c_int]
    L.mlb_graph_set_input_planes.argtypes = [_vp, ctypes.c_int]
    L.mlb_router_create.restype = _vp
    L.mlb_router_create.argtypes = [ctypes.c_int, ctypes.c_int]
    L.mlb_router_destroy.argtypes = [_vp]
    L.mlb_router_destroy.restype = None
    L.mlb_router_set_unison.argtypes = [_vp, ctypes.c_int]
    L.mlb_router_set_unison.restype = None
    L.mlb_router_add_event.argtypes = [_vp, _vp]
    L.mlb_router_add_event.restype = None
    L.mlb_router_clear_events.argtypes = [_vp]
    L.mlb_router_clear_events.restype = None
    L.mlb_router_record_count.argtypes = [_vp]
    L.mlb_router_unsupported_count.argtypes = [_vp]
    L.mlb_router_set_mod_cc.argtypes = [_vp, ctypes.c_int]
    L.mlb_router_set_mod_cc.restype = None
    L.mlb_router_process_vector.argtypes = [_vp, ctypes.c_int, _vp]
    L.mlb_router_controller_changes.argtypes = [_vp, _vp, ctypes.c_int]
    L.mlb_controllers_create.argtypes = [ctypes.c_int, _cf, ctypes.c_int, _vp, ctypes.c_int, _vp]
    L.mlb_controllers_destroy.argtypes = [_vp]
    L.mlb_controllers_clear.argtypes = [_vp]
    L.mlb_controllers_get_state.argtypes = [_vp, _vp, _vp]
    L.mlb_controllers_set_state.argtypes = [_vp, _vp, _vp]
    L.mlb_controllers_set_voice_map.argtypes = [_vp, _vp, ctypes.c_int]
    L.mlb_controllers_process_device.argtypes = [_vp, _vp, _vp, _vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, _vp]
    L.mlb_controllers_process_host.argtypes = [_vp, _vp, _vp, ctypes.c_int, _vp, ctypes.c_int, ctypes.c_int,
                                               ctypes.c_int]
    L.mlb_resampler_create.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, _vp]
    L.mlb_resampler_destroy.argtypes = [_vp]
    L.mlb_resampler_clear.argtypes = [_vp]
    L.mlb_resampler_process_host.argtypes = [_vp, _vp, _vp, ctypes.c_int, _vp]
    L.mlb_resampler_process_device.argtypes = [_vp, _vp, _vp, ctypes.c_int, _vp, _vp]
    L.mlb_fdtd_create.argtypes = [ctypes.c_int, _cf, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_uint, _vp]
    L.mlb_fdtd_destroy.argtypes = [_vp]
    L.mlb_fdtd_clear.argtypes = [_vp]
    L.mlb_fdtd_get_state.argtypes = [_vp, _vp]
    L.mlb_fdtd_set_state.argtypes = [_vp, _vp]
    L.mlb_fdtd_process_device.argtypes = [_vp, _vp, _vp, ctypes.c_int, _vp]
    L.mlb_fdtd_process_host.argtypes = [_vp, _vp, _vp, ctypes.c_int]
    L.mlb_voices_create.argtypes =[ctypes.c_int, _cf, _vp, _vp, _vp, _vp, ctypes.c_uint, _vp]
    L.mlb_voices_destroy.argtypes = [_vp]
    L.mlb_voices_set_main_voices.argtypes = [_vp, _vp]
    L.mlb_voices_process_host.argtypes = [_vp, _vp, _vp, ctypes.c_int, ctypes.c_uint]
    L.mlb_voices_process_device.argtypes = [_vp, _vp, _vp, ctypes.c_int, ctypes.c_uint, _vp]
    L.mlb_graph_process_device.argtypes = [_vp, _vp, _vp, _vp, ctypes.c_int, _vp]
    L.mlb_synth_process_host.argtypes = [_vp, _vp, _vp, _vp, _vp, ctypes.c_int]
    L.mlb_buses_create.argtypes = [ctypes.c_int, ctypes.c_int, _vp, _vp, _vp]
    L.mlb_buses_destroy.argtypes = [_vp]
    L.mlb_buses_sum_device.argtypes = [_vp, _vp, _vp, ctypes.c_int, ctypes.c_int, _vp]
    L.mlb_synth_process_buses_host.argtypes = [_vp, _vp, _vp, _vp, _vp, ctypes.c_int]
    L.mlb_synth_process_controllers_host.argtypes = [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, ctypes.c_int]
    L.mlb_graph_process_host.argtypes = [_vp, _vp, _vp, _vp, ctypes.c_int]
    L.mlb_graph_last_kernel_ms.argtypes = [_vp, _vp]
    L.mlb_graph_last_host_slices.argtypes = [_vp]
    L.mlb_mixbus_create.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_size_t, ctypes.POINTER(_vp)]
    L.mlb_mixbus_handle.argtypes = [_vp, _vp]
    L.mlb_mixbus_connect.argtypes = [_vp, _vp]
    L.mlb_mixbus_destroy.argtypes = [_vp]
    L.mlb_graph_attach_mixbus.argtypes = [_vp, _vp]
    L.mlb_mixbus_set_async.argtypes = [_vp, ctypes.c_int]
    L.mlb_graph_mix_wait.argtypes = [_vp, _vp]
    L.mlb_graph_set_mix_async.argtypes = [_vp, ctypes.c_int]
    L.mlb_map_device.argtypes = [ctypes.c_int, _vp, _vp, _vp, _vp, ctypes.c_size_t, _vp]
    L.mlb_map_host.argtypes = [ctypes.c_int, _vp, _vp, _vp, _vp, ctypes.c_size_t]
    L.mlb_map_host_allocations.restype = ctypes.c_longlong
    for name, n in (("lopass", 2), ("hipass", 2), ("bandpass", 2), ("loshelf", 3), ("hishelf", 3),
                    ("bell", 3), ("onepole", 1), ("peak", 1), ("rms", 1), ("adsr", 5), ("glide", 1),
                    ("sample_glide", 1)):
        fn = getattr(L, "mlb_coeffs_" + name)
        fn.argtypes = [_cf] * n + [_vp]
        fn.restype = None
    L.mlb_coeffs_batch.argtypes = [ctypes.c_int, ctypes.c_size_t, _vp, _vp, _vp, _vp]
    L.mlb_coeffs_lopass_vec.argtypes = [_vp, _vp, _vp]
    L.mlb_coeffs_lopass_vec.restype = None
    L.mlb_coeffs_lopass_vec_n.argtypes = [_vp, _vp, _vp, ctypes.c_size_t]
    L.mlb_coeffs_lopass_vec_n.restype = None
    L.mlb_interpolate_coeffs_linear.argtypes = [_vp, _vp, ctypes.c_int, _vp]
    L.mlb_interpolate_coeffs_linear.restype = None
    L.mlb_coeffs_dcblocker.argtypes = [_cf]
    L.mlb_coeffs_dcblocker.restype = _cf
    L.mlb_impulse_table.argtypes = [_vp]
    L.mlb_impulse_table.restype = None
    L.mlb_coeffs_allpass1.argtypes = [_cf]
    L.mlb_coeffs_allpass1.restype = _cf
    L.mlb_db_to_gain.argtypes = [_cf]
    L.mlb_db_to_gain.restype = _cf
    L.mlb_coeffs_fdn8.argtypes = [_vp, _vp, _vp, _vp]
    L.mlb_coeffs_fdn8.restype = None
    _lib = L
    return L


def _check(rc: int) -> None:
    if rc != 0:
        raise MlbError(rc, lib().mlb_last_error().decode())


def _ptr(a) -> Optional[int]:
    """Raw address of a numpy array / torch tensor / int / None."""
    if a is None:
        return None
    if isinstance(a, int):
        return a
    if isinstance(a, np.ndarray):
        return a.ctypes.data
    if hasattr(a, "data_ptr"):
        return a.data_ptr()
    raise TypeError(type(a))


def device_count() -> int:
    return int(lib().mlb_device_count())


def init(device: int = 0) -> None:
    _check(lib().mlb_init(device))


def kernel_launches() -> int:
    return int(lib().mlb_kernel_launches())


def live_handles() -> int:
    """Graphs, voice banks, bus layouts, controller banks, resamplers, FDTD banks and mix buses alive in this
    process."""
    return int(lib().mlb_live_handles())


# ---- coefficient design (host libm; same calls as the reference's makeCoeffs) ----
_NCOEF = {"lopass": 3, "hipass": 4, "bandpass": 3, "loshelf": 5, "hishelf": 6, "bell": 4, "onepole": 2,
          "peak": 2, "rms": 2, "adsr": 4, "glide": 2, "sample_glide": 2}


def coeffs(kind: str, *args: float) -> np.ndarray:
    out = np.zeros(_NCOEF[kind], np.float32)
    getattr(lib(), "mlb_coeffs_" + kind)(*[_cf(a) for a in args], out.ctypes.data)
    return out


def coeffs_batch(kind: str, omega, k=None, A=None) -> np.ndarray:
    """makeCoeffs of `kind` for n voices at once -> [n_coef][n] (one C call, host libm)."""
    om = np.ascontiguousarray(omega, np.float32)
    n = om.shape[0]
    kk = None if k is None else np.ascontiguousarray(np.broadcast_to(np.asarray(k, np.float32), (n,)))
    aa = None if A is None else np.ascontiguousarray(np.broadcast_to(np.asarray(A, np.float32), (n,)))
    out = np.zeros((_NCOEF[kind], n), np.float32)
    _check(lib().mlb_coeffs_batch(OP_ID[kind.upper()], n, om.ctypes.data, _ptr(kk), _ptr(aa), out.ctypes.data))
    return out


def coeffs_lopass_vec(omega, k) -> np.ndarray:
    """Lopass::makeCoeffsVec for rows of 64 samples: omega, k of shape [..., 64] -> [..., 3, 64]
    (rows g0, g1, g2 = inputs 1..3 of a LOPASS_V node).  Host libm, one C call."""
    om = np.ascontiguousarray(omega, np.float32)
    kk = np.ascontiguousarray(np.broadcast_to(np.asarray(k, np.float32), om.shape))
    assert om.shape[-1] == BLOCK
    out = np.empty(om.shape[:-1] + (3, BLOCK), np.float32)
    lib().mlb_coeffs_lopass_vec_n(om.ctypes.data, kk.ctypes.data, out.ctypes.data, om.size // BLOCK)
    return out


def interpolate_coeffs_linear(c0, c1) -> np.ndarray:
    """interpolateCoeffsLinear(c0, c1): [n_coeffs] x 2 -> [n_coeffs][64] ramps (LoShelf/HiShelf::vcoeffs when
    c0 / c1 come from coeffs('loshelf' / 'hishelf', ...))."""
    a, b = np.ascontiguousarray(c0, np.float32), np.ascontiguousarray(c1, np.float32)
    assert a.shape == b.shape and a.ndim == 1
    out = np.empty((a.shape[0], BLOCK), np.float32)
    lib().mlb_interpolate_coeffs_linear(a.ctypes.data, b.ctypes.data, a.shape[0], out.ctypes.data)
    return out


def coeffs_dcblocker(omega: float) -> float:
    return float(lib().mlb_coeffs_dcblocker(omega))


def impulse_table() -> np.ndarray:
    """ImpulseGen's 17-tap table as the library builds it on the host."""
    out = np.zeros(17, np.float32)
    lib().mlb_impulse_table(out.ctypes.data)
    return out


def coeffs_allpass1(d: float) -> float:
    return float(lib().mlb_coeffs_allpass1(d))


def db_to_gain(db: float) -> float:
    return float(lib().mlb_db_to_gain(db))


def coeffs_fdn8(times, cutoffs, gains) -> np.ndarray:
    t = np.ascontiguousarray(times, np.float32)
    c = np.ascontiguousarray(cutoffs, np.float32)
    g = np.ascontiguousarray(gains, np.float32)
    out = np.zeros(32, np.float32)
    lib().mlb_coeffs_fdn8(t.ctypes.data, c.ctypes.data, g.ctypes.data, out.ctypes.data)
    return out


# ---- stateless elementwise ops (every DEFINE_OP* of MLDSPOps.h) ----
def map_host(op: str, x1: np.ndarray, x2: Optional[np.ndarray] = None,
             x3: Optional[np.ndarray] = None) -> np.ndarray:
    """y = op(x1[, x2[, x3]]) on arrays of shape [n_rows, 64] (host in, host out, GPU compute)."""
    x1 = np.ascontiguousarray(x1, np.float32)
    assert x1.size % BLOCK == 0
    xs = [None if x is None else np.ascontiguousarray(x, np.float32) for x in (x2, x3)]
    for x in xs:
        if x is not None and x.shape != x1.shape:
            raise ValueError(f"map_host: operand shapes differ ({x.shape} vs {x1.shape})")
    y = np.empty_like(x1)
    _check(lib().mlb_map_host(OP_ID[op.upper()], x1.ctypes.data, _ptr(xs[0]), _ptr(xs[1]),
                              y.ctypes.data, x1.size // BLOCK))
    return y


def map_device(op: str, x1, x2, x3, y, n_rows: int, stream: int = 0) -> None:
    _check(lib().mlb_map_device(OP_ID[op.upper()], _ptr(x1), _ptr(x2), _ptr(x3), _ptr(y), n_rows,
                                stream or None))


def plan(spec: GraphSpec, n_voices: int, flags: int = 0):
    """The graph interpreter's host-side plan, no device needed (mlb_graph_plan): (stage of every node -- -1 for PARAM
    and the like --, number of stages, number of shared-memory row slots)."""
    n = spec.n_nodes
    stage = (ctypes.c_int32 * max(1, n))()
    ns, rows = ctypes.c_int32(), ctypes.c_int32()
    _check(lib().mlb_graph_plan(spec.c_nodes(), n, spec.c_outs(), spec.n_out, int(n_voices), int(flags), stage,
                                ctypes.byref(ns), ctypes.byref(rows)))
    return list(stage)[:n], int(ns.value), int(rows.value)


class _Handle:
    """Owner of one library handle ``_h``: ``close()`` (a no-op once closed) or the garbage collector hands it to the
    library function named ``_destroy``."""

    _h = None
    _destroy = ""

    def close(self) -> None:
        if self._h:
            getattr(lib(), self._destroy)(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class VoiceGraph(_Handle):
    """Device-resident bank of ``n_voices`` identical graphs (one voice per CUDA lane)."""

    _destroy = "mlb_graph_destroy"

    def __init__(self, spec: GraphSpec, n_voices: int, flags: int = FLAG_EXACT):
        self.spec = spec
        self.n_voices = int(n_voices)
        self._h = _vp()
        L = lib()
        nodes, outs = spec.c_nodes(), spec.c_outs()
        _check(L.mlb_graph_create(nodes, spec.n_nodes, outs, spec.n_out, self.n_voices, flags,
                                  ctypes.byref(self._h)))
        lay = Layout()
        _check(L.mlb_graph_layout_of(self._h, ctypes.byref(lay)))
        assert (lay.n_state_words, lay.n_coef_words, lay.n_inputs) == (spec.n_state, spec.n_coef,
                                                                       spec.n_in)

    @property
    def kernel_name(self) -> str:
        return lib().mlb_graph_kernel_name(self._h).decode()

    @property
    def delay_bytes(self) -> int:
        return int(lib().mlb_graph_delay_bytes(self._h))

    def set_coefs(self, coef: np.ndarray) -> None:
        coef = np.ascontiguousarray(coef, np.float32)
        assert coef.shape == (self.spec.n_coef, self.n_voices), coef.shape
        _check(lib().mlb_graph_set_coefs(self._h, coef.ctypes.data if coef.size else None))

    def set_state(self, state: np.ndarray) -> None:
        state = np.ascontiguousarray(state, np.uint32)
        assert state.shape == (self.spec.n_state, self.n_voices), state.shape
        _check(lib().mlb_graph_set_state(self._h, state.ctypes.data if state.size else None))

    def get_state(self) -> np.ndarray:
        st = np.zeros((self.spec.n_state, self.n_voices), np.uint32)
        _check(lib().mlb_graph_get_state(self._h, st.ctypes.data if st.size else None))
        return st

    def clear_delays(self) -> None:
        _check(lib().mlb_graph_clear_delays(self._h))

    def process_host(self, inp: Optional[np.ndarray], n_blocks: int, want_out: bool = True,
                     want_mix: bool = False, out: Optional[np.ndarray] = None,
                     mix: Optional[np.ndarray] = None):
        """Host buffers in, host buffers out; H2D + one kernel + D2H inside the call."""
        s, V, T = self.spec, self.n_voices, int(n_blocks)
        if s.n_in:
            assert inp is not None and inp.dtype == np.float32 and inp.flags["C_CONTIGUOUS"]
            assert inp.shape == (T, s.n_in, V, BLOCK), inp.shape
        if want_out and out is None:
            out = np.empty((T, s.n_out, V, BLOCK), np.float32)
        if want_mix and mix is None:
            mix = np.empty((T, s.n_out, BLOCK), np.float32)
        for name, a, shape in (("out", out if want_out else None, (T, s.n_out, V, BLOCK)),
                               ("mix", mix if want_mix else None, (T, s.n_out, BLOCK))):
            if a is not None and not (isinstance(a, np.ndarray) and a.dtype == np.float32 and
                                      a.flags["C_CONTIGUOUS"] and a.shape == shape):
                raise ValueError(f"process_host: `{name}` must be a C-contiguous float32 array of shape {shape}")
        _check(lib().mlb_graph_process_host(self._h, _ptr(inp) if s.n_in else None,
                                            _ptr(out) if want_out else None,
                                            _ptr(mix) if want_mix else None, T))
        return out, mix

    def process_events_host(self, bank: "VoiceBank", events: np.ndarray, want_out: bool = True,
                            want_mix: bool = False, out: Optional[np.ndarray] = None,
                            mix: Optional[np.ndarray] = None):
        """Contract E (mlb_synth_process_host): event records [T][V] in, the graph's rows / mix bus out.
        The graph's INPUT plane r is Voice row r of ``bank``; the rows never leave the device."""
        s, V = self.spec, self.n_voices
        if not (isinstance(events, np.ndarray) and events.ndim == 2 and events.shape[1] == V and
                events.dtype.itemsize == 72 and events.flags["C_CONTIGUOUS"]):
            raise ValueError("process_events_host: `events` must be a C-contiguous [T][V] array of 72-byte records")
        T = int(events.shape[0])
        if want_out and out is None:
            out = np.empty((T, s.n_out, V, BLOCK), np.float32)
        if want_mix and mix is None:
            mix = np.empty((T, s.n_out, BLOCK), np.float32)
        for name, a, shape in (("out", out if want_out else None, (T, s.n_out, V, BLOCK)),
                               ("mix", mix if want_mix else None, (T, s.n_out, BLOCK))):
            if a is not None and not (isinstance(a, np.ndarray) and a.dtype == np.float32 and
                                      a.flags["C_CONTIGUOUS"] and a.shape == shape):
                raise ValueError(f"process_events_host: `{name}` must be a C-contiguous float32 array of shape {shape}")
        _check(lib().mlb_synth_process_host(bank._h, self._h, events.ctypes.data,
                                            _ptr(out) if want_out else None,
                                            _ptr(mix) if want_mix else None, T))
        return out, mix

    def process_events_controllers_host(self, bank: "VoiceBank", controllers: "ControllerBank", events: np.ndarray,
                                        offsets: np.ndarray, changes: np.ndarray, want_out: bool = True,
                                        want_mix: bool = False):
        """Contract E with controller planes (mlb_synth_process_controllers_host): event records [T][V] and a controller
        change list (offsets [T][G + 1], changes) in, the graph's rows / mix bus out.  INPUT planes 0..7 are the
        Voice rows of ``bank``, plane 8 + k controller k of ``controllers`` (which needs a voice map of this graph's
        voices); nothing but records and changes crosses PCIe on the way in."""
        s, V = self.spec, self.n_voices
        if not (isinstance(events, np.ndarray) and events.ndim == 2 and events.shape[1] == V and
                events.dtype.itemsize == 72 and events.flags["C_CONTIGUOUS"]):
            raise ValueError("process_events_controllers_host: `events` must be a C-contiguous [T][V] array of 72-byte "
                             "records")
        T = int(events.shape[0])
        off = np.ascontiguousarray(offsets, np.int32)
        if off.shape != (T, controllers.n_instruments + 1):
            raise ValueError(f"process_events_controllers_host: offsets must be [{T}][{controllers.n_instruments + 1}], "
                             f"got {off.shape}")
        ch = np.ascontiguousarray(changes, CONTROLLER_CHANGE_DTYPE)
        out = np.empty((T, s.n_out, V, BLOCK), np.float32) if want_out else None
        mix = np.empty((T, s.n_out, BLOCK), np.float32) if want_mix else None
        _check(lib().mlb_synth_process_controllers_host(bank._h, controllers._h, self._h, events.ctypes.data,
                                                        off.ctypes.data, ch.ctypes.data if ch.size else None,
                                                        _ptr(out), _ptr(mix), T))
        return out, mix

    def process_events_buses_host(self, bank: "VoiceBank", buses: "Buses", events: np.ndarray,
                                  out: Optional[np.ndarray] = None) -> np.ndarray:
        """Contract E with per-instrument output (mlb_synth_process_buses_host): event records [T][V] in, the bus rows
        [T][n_out][G][64] out -- each bus the strict-order sum of its voices' output rows (Synth::processVector).
        The voice rows never leave the device."""
        s, V = self.spec, self.n_voices
        if not (isinstance(events, np.ndarray) and events.ndim == 2 and events.shape[1] == V and
                events.dtype.itemsize == 72 and events.flags["C_CONTIGUOUS"]):
            raise ValueError("process_events_buses_host: `events` must be a C-contiguous [T][V] array of 72-byte "
                             "records")
        T = int(events.shape[0])
        shape = (T, s.n_out, buses.n_buses, BLOCK)
        if out is None:
            out = np.empty(shape, np.float32)
        if not (isinstance(out, np.ndarray) and out.dtype == np.float32 and out.flags["C_CONTIGUOUS"] and
                out.shape == shape):
            raise ValueError(f"process_events_buses_host: `out` must be a C-contiguous float32 array of shape {shape}")
        _check(lib().mlb_synth_process_buses_host(bank._h, self._h, buses._h, events.ctypes.data, _ptr(out), T))
        return out

    def process_device(self, inp, out, mix, n_blocks: int, stream: int = 0) -> None:
        """Device pointers (torch tensors / ints); asynchronous on ``stream`` (cudaStream_t)."""
        _check(lib().mlb_graph_process_device(self._h, _ptr(inp), _ptr(out), _ptr(mix), int(n_blocks),
                                              stream or None))

    def set_input_planes(self, n_planes: int) -> None:
        """The input buffer carries n_planes planes per block (more than the graph reads)."""
        _check(lib().mlb_graph_set_input_planes(self._h, int(n_planes)))

    def attach_mixbus(self, bus: Optional["MixBus"]) -> None:
        """From now on `mix` is the sum over all ranks of the bus (reduced in-kernel over NVLink)."""
        _check(lib().mlb_graph_attach_mixbus(self._h, bus._h if bus is not None else None))

    def set_mix_async(self, on: bool = True) -> None:
        """mix_reduce (and the multi-GPU exchange) on the graph's own stream, overlapping the next call; a call's
        `mix` is complete after mix_wait(stream)."""
        _check(lib().mlb_graph_set_mix_async(self._h, int(on)))

    def mix_wait(self, stream: int = 0) -> None:
        """Make `stream` wait for the most recent call's mix bus (async mix bus only; else a no-op)."""
        _check(lib().mlb_graph_mix_wait(self._h, stream or None))

    def reserve_sms(self, n_sms: int) -> None:
        """Keep n_sms SMs out of the persistent chain grid (room for an overlapped collective)."""
        _check(lib().mlb_graph_reserve_sms(self._h, int(n_sms)))

    @property
    def last_host_slices(self) -> int:
        """Voice slices the most recent process_host call was pipelined over (1 = one launch)."""
        return int(lib().mlb_graph_last_host_slices(self._h))

    def last_kernel_ms(self) -> float:
        ms = ctypes.c_float(0)
        _check(lib().mlb_graph_last_kernel_ms(self._h, ctypes.byref(ms)))
        return float(ms.value)


class MixBus:
    """Multi-GPU mix bus over peer memory (mlb_mixbus_*): after ``connect`` + ``graph.attach_mixbus(bus)`` the
    ``mix`` output of every process call is the sum over all ranks, reduced inside the kernel over NVLink."""

    def __init__(self, rank: int, world: int, max_floats: int):
        self._h = _vp()
        self.rank, self.world = rank, world
        _check(lib().mlb_mixbus_create(rank, world, max_floats, ctypes.byref(self._h)))

    def handle(self) -> bytes:
        buf = ctypes.create_string_buffer(64)
        _check(lib().mlb_mixbus_handle(self._h, buf))
        return buf.raw

    def set_async(self, on: bool = True) -> None:
        """Completion (wait for peers + sum) on the bus's own stream; see mlb_mixbus_set_async."""
        _check(lib().mlb_mixbus_set_async(self._h, int(on)))

    def connect(self, handles) -> None:
        """handles: the 64-byte handle of every rank, in rank order."""
        blob = b"".join(bytes(h) for h in handles)
        assert len(blob) == 64 * self.world
        _check(lib().mlb_mixbus_connect(self._h, blob))

    def close(self) -> None:
        if self._h:
            lib().mlb_mixbus_destroy(self._h)
            self._h = _vp()


class VoiceBank(_Handle):
    """V x EventsToSignals::Voice on the device (SURVEY 8f row 3): per-voice event records in,
    the 8 control rows (pitch, gate, voice, z, x, y, mod, elapsed time) out."""

    _destroy = "mlb_voices_destroy"

    ROWS = 8

    MIDI = 1  # MLB_VOICES_MIDI: z row += smoothed channel pressure

    def __init__(self, sample_rate: float, voice_index, pitch_glide_seconds, drift_amount, pitch_bend,
                 flags: int = 0):
        vi = np.ascontiguousarray(voice_index, np.int32)
        gs, da, pb = (np.ascontiguousarray(a, np.float32) for a in (pitch_glide_seconds, drift_amount, pitch_bend))
        self.n_voices = int(vi.shape[0])
        assert gs.shape == da.shape == pb.shape == vi.shape
        h = ctypes.c_void_p()
        _check(lib().mlb_voices_create(self.n_voices, sample_rate, vi.ctypes.data, gs.ctypes.data, da.ctypes.data,
                                       pb.ctypes.data, flags, ctypes.byref(h)))
        self._h = h

    def set_main_voices(self, main_voice) -> None:
        """MPE: main_voice[v] = bank index of voice v's main voice, or -1."""
        mv = np.ascontiguousarray(main_voice, np.int32)
        assert mv.shape == (self.n_voices,)
        _check(lib().mlb_voices_set_main_voices(self._h, mv.ctypes.data))

    def process_host(self, events: np.ndarray, row_mask: int = 0xFF) -> np.ndarray:
        """events: [T][V] array of workloads.VOICE_EVENTS_DTYPE; returns out [T][8][V][64] f32
        (planes whose bit is clear in row_mask are left zero)."""
        assert events.ndim == 2 and events.shape[1] == self.n_voices and events.dtype.itemsize == 72
        ev = np.ascontiguousarray(events)
        out = np.zeros((ev.shape[0], self.ROWS, self.n_voices, BLOCK), np.float32)
        _check(lib().mlb_voices_process_host(self._h, ev.ctypes.data, out.ctypes.data, ev.shape[0], row_mask))
        return out

    def process_device(self, events, out, n_blocks: int, row_mask: int = 0xFF, stream: int = 0) -> None:
        _check(lib().mlb_voices_process_device(self._h, _ptr(events), _ptr(out), int(n_blocks), row_mask,
                                               stream or None))


class Buses(_Handle):
    """G per-instrument output buses over a V-voice bank (mlb_buses_*): bus g is the strict left-to-right sum, from
    +0, of the voice rows [first[g], first[g] + count[g]) -- Synth::processVector (MLSynth.h:36-60) per instrument.
    Ranges may be empty, leave gaps (MPE main voices) and overlap."""

    _destroy = "mlb_buses_destroy"

    def __init__(self, n_voices: int, first, count):
        fv = np.ascontiguousarray(first, np.int32)
        vc = np.ascontiguousarray(count, np.int32)
        if fv.ndim != 1 or fv.shape != vc.shape:
            raise ValueError(f"Buses: `first` and `count` must be 1-D of one length, got {fv.shape} and {vc.shape}")
        self.n_voices, self.n_buses = int(n_voices), int(fv.shape[0])
        h = ctypes.c_void_p()
        _check(lib().mlb_buses_create(self.n_voices, self.n_buses, fv.ctypes.data, vc.ctypes.data, ctypes.byref(h)))
        self._h = h

    def sum_device(self, rows, out, n_planes: int, n_blocks: int, stream: int = 0) -> None:
        """Device buffers (torch tensors / ints): rows [T][P][V][64] -> out [T][P][G][64]; asynchronous on ``stream``,
        one kernel launch, no allocation or synchronisation (capturable into a CUDA graph)."""
        _check(lib().mlb_buses_sum_device(self._h, _ptr(rows), _ptr(out), int(n_planes), int(n_blocks),
                                          stream or None))


CONTROLLER_CHANGE_DTYPE = np.dtype([("controller", "<u2"), ("pad", "<u2"), ("value", "<f4")])  # mlb_controller_change


class ControllerBank(_Handle):
    """G instruments x C requested MIDI controllers (mlb_controllers_*): the SmoothedControllers of one reference
    EventsToSignals per instrument (MLEventsToSignals.h:170-180), i.e. what AudioContext::getInputController(n)
    returns, bit for bit.  Input per block: a CSR change list, offsets [T][G + 1] into changes
    (CONTROLLER_CHANGE_DTYPE), each instrument's writes in event order; output [T][n_planes][N][64] with controller
    k of the list in plane plane0 + k and N = G, or N = V after set_voice_map (every voice gets its instrument's row,
    a voice of instrument -1 gets +0)."""

    _destroy = "mlb_controllers_destroy"

    MIDI, MPE = 0, 1
    N_WORDS = 4  # state words: inputValue, target, vectorsRemaining, step

    def __init__(self, n_instruments: int, controllers, sample_rate: float = 48000.0, protocol: int = 0):
        ctrl = np.ascontiguousarray(controllers, np.int32)
        if ctrl.ndim != 1:
            raise ValueError(f"ControllerBank: `controllers` must be a 1-D list of numbers, got shape {ctrl.shape}")
        self.n_instruments, self.controllers = int(n_instruments), [int(c) for c in ctrl]
        self.n_controllers, self.protocol, self.n_voices = len(self.controllers), int(protocol), 0
        h = ctypes.c_void_p()
        _check(lib().mlb_controllers_create(self.n_instruments, sample_rate, self.protocol, ctrl.ctypes.data,
                                            self.n_controllers, ctypes.byref(h)))
        self._h = h

    def clear(self) -> None:
        _check(lib().mlb_controllers_clear(self._h))

    def get_state(self):
        """(words [4][C][G] uint32, rows [C][G][64] f32); an idle glide's row is its target."""
        C, G = self.n_controllers, self.n_instruments
        words = np.zeros((self.N_WORDS, C, G), np.uint32)
        rows = np.zeros((C, G, BLOCK), np.float32)
        _check(lib().mlb_controllers_get_state(self._h, words.ctypes.data, rows.ctypes.data))
        return words, rows

    def set_state(self, words: np.ndarray, rows: np.ndarray) -> None:
        C, G = self.n_controllers, self.n_instruments
        w = np.ascontiguousarray(words, np.uint32)
        r = np.ascontiguousarray(rows, np.float32)
        if w.shape != (self.N_WORDS, C, G) or r.shape != (C, G, BLOCK):
            raise ValueError(f"set_state: words must be [4][{C}][{G}] and rows [{C}][{G}][64], got {w.shape} and "
                             f"{r.shape}")
        _check(lib().mlb_controllers_set_state(self._h, w.ctypes.data, r.ctypes.data))

    def set_voice_map(self, voice_instrument) -> None:
        """voice_instrument[V]: each voice's instrument or -1; None goes back to instrument rows."""
        if voice_instrument is None:
            _check(lib().mlb_controllers_set_voice_map(self._h, None, 0))
            self.n_voices = 0
            return
        vm = np.ascontiguousarray(voice_instrument, np.int32)
        _check(lib().mlb_controllers_set_voice_map(self._h, vm.ctypes.data, int(vm.shape[0])))
        self.n_voices = int(vm.shape[0])

    def process_host(self, offsets: np.ndarray, changes: np.ndarray, out: Optional[np.ndarray] = None,
                     plane0: int = 0, n_planes: Optional[int] = None) -> np.ndarray:
        """offsets [T][G + 1] int32, changes (CONTROLLER_CHANGE_DTYPE) -> out [T][n_planes][N][64]; planes outside
        [plane0, plane0 + C) of a given `out` are left as they are."""
        off = np.ascontiguousarray(offsets, np.int32)
        if off.ndim != 2 or off.shape[1] != self.n_instruments + 1:
            raise ValueError(f"process_host: offsets must be [T][{self.n_instruments + 1}], got {off.shape}")
        ch = np.ascontiguousarray(changes, CONTROLLER_CHANGE_DTYPE)
        T = int(off.shape[0])
        P = self.n_controllers if n_planes is None else int(n_planes)
        shape = (T, P, self.n_voices or self.n_instruments, BLOCK)
        if out is None:
            out = np.zeros(shape, np.float32)
        if not (isinstance(out, np.ndarray) and out.dtype == np.float32 and out.flags["C_CONTIGUOUS"] and
                out.shape == shape):
            raise ValueError(f"process_host: `out` must be a C-contiguous float32 array of shape {shape}")
        _check(lib().mlb_controllers_process_host(self._h, off.ctypes.data, ch.ctypes.data if ch.size else None,
                                                  int(ch.size), out.ctypes.data, int(plane0), P, T))
        return out

    def process_device(self, offsets, changes, out, n_blocks: int, plane0: int = 0, n_planes: Optional[int] = None,
                       stream: int = 0) -> None:
        """Device buffers (torch tensors / ints); asynchronous on ``stream``, one kernel launch, no allocation or
        synchronisation (capturable into a CUDA graph)."""
        P = self.n_controllers if n_planes is None else int(n_planes)
        _check(lib().mlb_controllers_process_device(self._h, _ptr(offsets), _ptr(changes), _ptr(out), int(plane0), P,
                                                    int(n_blocks), stream or None))


class ResamplerBank(_Handle):
    """Upsampler(octaves) / Downsampler(octaves) x V (SURVEY 8f row 4).  direction: 0 up, 1 down."""

    _destroy = "mlb_resampler_destroy"

    UP, DOWN = 0, 1

    def __init__(self, direction: int, octaves: int, n_voices: int):
        self.direction, self.octaves, self.n_voices = direction, octaves, n_voices
        h = ctypes.c_void_p()
        _check(lib().mlb_resampler_create(direction, octaves, n_voices, ctypes.byref(h)))
        self._h = h

    def clear(self) -> None:
        _check(lib().mlb_resampler_clear(self._h))

    def process_host(self, x: np.ndarray) -> np.ndarray:
        """x [T][V][64] -> [T << octaves][V][64] (up) or the completed groups (down)."""
        x = np.ascontiguousarray(x, np.float32)
        assert x.ndim == 3 and x.shape[1] == self.n_voices and x.shape[2] == BLOCK
        T = x.shape[0]
        cap = T << self.octaves if self.direction == self.UP else T
        out = np.zeros((max(cap, 1), self.n_voices, BLOCK), np.float32)
        n = ctypes.c_int(0)
        _check(lib().mlb_resampler_process_host(self._h, x.ctypes.data, out.ctypes.data, T, ctypes.byref(n)))
        return out[:n.value]


class FDTDBank(_Handle):
    """V x the reference's FDTD membrane (FDTDState + processFDTDModel, examples/audio-and-midi/fdtd.cpp): per
    block, an excitation row and a frequency row (cycles per sample) in, the two pickup rows L, R out."""

    _destroy = "mlb_fdtd_destroy"

    FTZ = 1  # MLB_FDTD_FTZ: every FP op flushes subnormals, as under UsingFlushDenormalsToZero
    SIZE = 16

    def __init__(self, n_instances: int, sample_rate: float = 48000.0, in_planes: int = 2, excite_plane: int = 0,
                 freq_plane: int = 1, flags: int = 0):
        self.n_instances, self.in_planes = int(n_instances), int(in_planes)
        h = ctypes.c_void_p()
        _check(lib().mlb_fdtd_create(self.n_instances, sample_rate, self.in_planes, excite_plane, freq_plane, flags,
                                     ctypes.byref(h)))
        self._h = h

    def clear(self) -> None:
        _check(lib().mlb_fdtd_clear(self._h))

    def get_state(self) -> np.ndarray:
        """[V][2][16][16]: the z^-1 surface, then z^-2."""
        st = np.zeros((self.n_instances, 2, self.SIZE, self.SIZE), np.float32)
        _check(lib().mlb_fdtd_get_state(self._h, st.ctypes.data))
        return st

    def set_state(self, state: np.ndarray) -> None:
        st = np.ascontiguousarray(state, np.float32)
        assert st.shape == (self.n_instances, 2, self.SIZE, self.SIZE), st.shape
        _check(lib().mlb_fdtd_set_state(self._h, st.ctypes.data))

    def process_host(self, inp: np.ndarray) -> np.ndarray:
        """inp [T][in_planes][V][64] -> out [T][2][V][64] (pickups L, R)."""
        inp = np.ascontiguousarray(inp, np.float32)
        if inp.ndim != 4 or inp.shape[1:] != (self.in_planes, self.n_instances, BLOCK):
            raise ValueError(f"process_host: inp must be [T][{self.in_planes}][{self.n_instances}][64], got {inp.shape}")
        out = np.empty((inp.shape[0], 2, self.n_instances, BLOCK), np.float32)
        _check(lib().mlb_fdtd_process_host(self._h, inp.ctypes.data, out.ctypes.data, inp.shape[0]))
        return out

    def process_device(self, inp, out, n_blocks: int, stream: int = 0) -> None:
        """Device buffers (torch tensors / ints): inp [T][in_planes][V][64], out [T][2][V][64]; asynchronous on
        ``stream``, one kernel launch, no allocation or synchronisation (capturable into a CUDA graph)."""
        _check(lib().mlb_fdtd_process_device(self._h, _ptr(inp), _ptr(out), int(n_blocks), stream or None))


class _Event(ctypes.Structure):
    """struct mlb_event"""
    _fields_ = [("type", ctypes.c_uint8), ("channel", ctypes.c_uint8), ("source_idx", ctypes.c_uint16),
                ("time", ctypes.c_int32), ("value1", ctypes.c_float), ("value2", ctypes.c_float)]


class EventRouter(_Handle):
    """EventsToSignals' event routing (host only, no GPU needed): events in, per-voice records out."""

    _destroy = "mlb_router_destroy"

    MIDI, MPE = 0, 1
    NOTE_ON, NOTE_OFF, SUSTAIN_PEDAL, CONTROLLER, PITCH_BEND, NOTE_PRESSURE, CHANNEL_PRESSURE = 1, 4, 5, 6, 7, 8, 9

    def __init__(self, polyphony: int, protocol: int = 0, unison: bool = False):
        self._h = lib().mlb_router_create(polyphony, protocol)
        if not self._h:
            raise MlbError(1, "bad router arguments")
        if unison:
            lib().mlb_router_set_unison(self._h, 1)
        self.n_records = lib().mlb_router_record_count(self._h)

    def add_event(self, type: int, channel: int, source_idx: int, time: int, value1: float = 0.0,
                  value2: float = 0.0) -> None:
        e = _Event(type, channel, source_idx, time, value1, value2)
        lib().mlb_router_add_event(self._h, ctypes.byref(e))

    @property
    def unsupported_events(self) -> int:
        """Events seen but not routed (CC 120 all-sound-off) since creation."""
        return int(lib().mlb_router_unsupported_count(self._h))

    def set_mod_cc(self, cc: int) -> None:
        lib().mlb_router_set_mod_cc(self._h, int(cc))

    def process_vector(self, start_time: int, records: np.ndarray) -> int:
        """records: array of n_records elements of workloads.VOICE_EVENTS_DTYPE (written in place)."""
        assert records.dtype.itemsize == 72 and records.size == self.n_records and records.flags["C_CONTIGUOUS"]
        return int(lib().mlb_router_process_vector(self._h, start_time, records.ctypes.data))

    def controller_changes(self) -> np.ndarray:
        """The controller writes of the last process_vector, in the order they were applied (CONTROLLER_CHANGE_DTYPE):
        controller events (numbers above 128 read as 128) and, in MIDI mode, channel pressure as controller 128."""
        n = int(lib().mlb_router_controller_changes(self._h, None, 0))
        out = np.zeros(n, CONTROLLER_CHANGE_DTYPE)
        if n:
            lib().mlb_router_controller_changes(self._h, out.ctypes.data, n)
        return out
