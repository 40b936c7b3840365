"""K12 without a GPU: the workload's CSR, the host checker (route_on_host) against the reference's complete
EventsToSignals, and every argument error of mlb_routers_create refused before any device is touched."""
import os

import numpy as np
import pytest

from madronalib_b200 import api, workloads as wl
from tests.router_cases import route_on_host


@pytest.mark.parametrize("mpe", [False, True])
def test_workload_csr_is_valid(mpe):
    G, T = 50, 30
    offsets, ev = wl.midi_performance(G, T, 6, mpe, density=0.5, seed=1)
    assert offsets.shape == (T, G + 1) and offsets[0, 0] == 0 and offsets[-1, -1] == ev.size
    assert (np.diff(offsets, axis=1) >= 0).all() and (offsets[1:, 0] == offsets[:-1, -1]).all()
    assert ((ev["time"] >= 0) & (ev["time"] < 64)).all()
    types = set(ev["type"].tolist())
    assert {1, 4, 5, 6, 7, 8, 9} <= types
    assert (ev["source_idx"][ev["type"] == 6] == 123).any()
    same = (np.diff(ev["time"]) == 0) & (np.diff(ev["type"]) == 0)
    assert same.any(), "equal times and types arrive"
    lay = wl.midi_layout(G, 6, mpe, gap=1)
    assert lay["n_voices"] == G * (7 if mpe else 6) + G


@pytest.mark.parametrize("mpe", [False, True])
def test_route_on_host_plus_port_bank_equals_reference(mpe):
    """route_on_host's CSR binning and tie order, through the port Voice bank, equal the complete reference
    EventsToSignals fed the same events."""
    from oracle import bindings
    if not os.path.exists(bindings.E2S_LIB):
        pytest.skip("oracle/_ref/libmle2s.so not built")
    import ctypes
    G, T, P, sr = 3, 60, 4, 48000.0
    offsets, ev = wl.midi_performance(G, T, P, mpe, density=0.7, seed=12)
    lay = wl.midi_layout(G, P, mpe)
    rec, _, _, _, _ = route_on_host(offsets, ev, lay, mpe)
    port = bindings.port_voice_bank()
    L = port.lib
    L.mlport_bank_create.restype = ctypes.c_void_p
    L.mlport_bank_set_main_voices.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    L.mlport_bank_process.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
    L.mlport_bank_process.restype = ctypes.c_double
    L.mlport_bank_destroy.argtypes = [ctypes.c_void_p]
    for g in range(G):
        ref = bindings.RefEventsToSignals(sr, P, 0.02, 0.5, mpe=mpe)
        for t in range(T):
            for e in ev[offsets[t, g]:offsets[t, g + 1]]:
                ref.add_event(int(e["type"]), int(e["channel"]), int(e["source_idx"]), t * 64 + int(e["time"]),
                              float(e["value1"]), float(e["value2"]))
        want = np.stack([ref.process_vector(t * 64) for t in range(T)])
        ref.close()
        f, NR = int(lay["first_voice"][g]), P + (1 if mpe else 0)
        r = np.ascontiguousarray(rec[:, f:f + NR])
        idx = np.arange(NR, dtype=np.int32) + (0 if mpe else 1)
        bend = np.full(NR, 24.0 if mpe else 7.0, np.float32)
        if mpe:
            bend[0] = 7.0
        gs, da = np.full(NR, 0.02, np.float32), np.full(NR, 0.5, np.float32)
        vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
        h = L.mlport_bank_create(NR, ctypes.c_float(sr), vp(idx), vp(gs), vp(da), vp(bend), 0 if mpe else 1)
        if mpe:
            mainv = np.zeros(NR, np.int32)
            mainv[0] = -1
            L.mlport_bank_set_main_voices(h, vp(mainv))
        got = np.zeros((T, 8, NR, 64), np.float32)
        L.mlport_bank_process(h, T, vp(r), vp(got), 1)
        L.mlport_bank_destroy(h)
        got = got[:, :, 1 if mpe else 0:, :].transpose(0, 2, 1, 3)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"instrument {g}"
        assert want[:, :, 1].max() > 0.1


CASES = [
    (dict(polyphony=[4, 17]), "instrument 1: polyphony 17 is not in 0..16"),
    (dict(polyphony=[4, -1]), "instrument 1: polyphony -1"),
    (dict(first_voice=[0, 3]), "instrument 1: voice 3 belongs to instrument 0"),
    (dict(first_voice=[0, 6]), r"instrument 1: voices \[6, 10\) are not within the 8 voices"),
    (dict(first_voice=[-1, 4]), "instrument 0: voices"),
    (dict(protocol=2), "protocol must be 0"),
    (dict(mod_cc=[16, 129]), "instrument 1: mod CC 129"),
    (dict(mod_cc=[-1, 16]), "instrument 0: mod CC -1"),
    (dict(unison=[0, 2]), "instrument 1: unison 2"),
    (dict(n_voices=0), "n_voices must be positive"),
    (dict(protocol=1), r"instrument 1: voices \[4, 9\) are not within the 8 voices"),
]


@pytest.mark.parametrize("kw,msg", CASES)
def test_create_argument_errors_without_device(kw, msg):
    args = dict(polyphony=[4, 4], first_voice=[0, 4], n_voices=8, protocol=0, unison=None, mod_cc=None)
    args.update(kw)
    n0 = api.live_handles()
    with pytest.raises(api.MlbError, match=msg):
        api.RouterBank(**args)
    assert api.live_handles() == n0
