"""The live-handle count (mlb_live_handles) without a device: a refused create leaves no handle behind, destroying
NULL is harmless, and the interpreter's host-only plan is never counted.  The Python wrapper of the host-only event
router releases its handle on close() and on garbage collection."""
import ctypes
import gc
import os

import numpy as np
import pytest

from madronalib_b200 import api, graph

_vp = ctypes.c_void_p


@pytest.fixture(scope="module")
def L():
    if not os.path.exists(api.LIB_PATH):
        from madronalib_b200 import build
        build.build()
    return api.lib()


def _creates(L, ok):
    """Every create entry point, with valid arguments when `ok`, else refused on its arguments."""
    g = graph.graph_sine_lopass_gain()
    h = _vp()
    vi = np.ones(4, np.int32)
    f4 = np.zeros(4, np.float32)
    first, count = np.array([0], np.int32), np.array([4 if ok else 5], np.int32)
    return {
        "mlb_graph_create": lambda: L.mlb_graph_create(g.c_nodes(), g.n_nodes, g.c_outs(), g.n_out, 4 if ok else 0, 0,
                                                       ctypes.byref(h)),
        "mlb_voices_create": lambda: L.mlb_voices_create(4 if ok else 0, 48000.0, vi.ctypes.data, f4.ctypes.data,
                                                         f4.ctypes.data, f4.ctypes.data, 0, ctypes.byref(h)),
        "mlb_buses_create": lambda: L.mlb_buses_create(4, 1, first.ctypes.data, count.ctypes.data, ctypes.byref(h)),
        "mlb_resampler_create": lambda: L.mlb_resampler_create(0 if ok else 2, 1, 4, ctypes.byref(h)),
        "mlb_fdtd_create": lambda: L.mlb_fdtd_create(4 if ok else 0, 48000.0, 2, 0, 1, 0, ctypes.byref(h)),
        "mlb_mixbus_create": lambda: L.mlb_mixbus_create(0, 1 if ok else 0, 64, ctypes.byref(h)),
    }


def test_refused_creates_leave_no_live_handle(L):
    n0 = api.live_handles()
    if api.device_count() == 0:
        assert n0 == 0
    for name, create in _creates(L, ok=False).items():
        assert create() == 1, name
        assert api.live_handles() == n0, name


def test_creates_without_a_device_leave_no_live_handle(L):
    if api.device_count() > 0:
        pytest.skip("a GPU is visible here")
    for name, create in _creates(L, ok=True).items():
        assert create() == 3, (name, L.mlb_last_error())
        assert b"no CPU fallback" in L.mlb_last_error()
        assert api.live_handles() == 0, name


@pytest.mark.parametrize("kind", ["graph", "voices", "buses", "resampler", "fdtd", "mixbus"])
def test_destroying_null_is_harmless(L, kind):
    n0 = api.live_handles()
    assert getattr(L, "mlb_%s_destroy" % kind)(None) == 0
    assert api.live_handles() == n0


def test_the_interpreter_plan_is_not_a_live_handle(L):
    n0 = api.live_handles()
    assert api.plan(graph.graph_fdn(6)[0], 45)[1] == 1
    with pytest.raises(api.MlbError):
        api.plan(graph.graph_fdn(24)[0], 45)
    assert api.live_handles() == n0


def test_mix_bus_has_no_finaliser():
    """mlb_mixbus_destroy synchronises the device and unmaps the peers' buffers: only an explicit close() does that."""
    assert not hasattr(api.MixBus, "__del__")


def test_router_handle_is_released_once(L, monkeypatch):
    freed = []
    destroy = L.mlb_router_destroy
    monkeypatch.setattr(L, "mlb_router_destroy", lambda h: (freed.append(h), destroy(h)))
    r = api.EventRouter(4)
    h = r._h
    r.close()
    r.close()
    assert freed == [h]
    r = api.EventRouter(4)
    h2 = r._h
    del r
    gc.collect()
    assert freed == [h, h2]
