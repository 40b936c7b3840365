"""K11, CPU side: the plain-C port of the smoothed MIDI controllers (oracle/port/mlport_ctrl.c) against the committed
golden and, where oracle/_ref was built, against one complete reference EventsToSignals per instrument
(oracle/_ref/libmlctrl.so); the router's controller change lists fed to the port; the host-side checks of
mlb_controllers_create.  NaN equals NaN (DESIGN.md 5)."""
import ctypes
import os

import numpy as np
import pytest

from tests.common import assert_same_bits
from tests.ctrl_cases import (ALL_CONTROLLERS, CHANNEL_PRESSURE, CONTROLLER, GLIDE_VECTORS, NOTE_OFF, NOTE_ON,
                              SAMPLE_RATES, special_phrases)

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "controllers.npz")


@pytest.fixture(scope="module")
def ctrl_ref():
    """One reference EventsToSignals per instrument, compiled in place; built here where the reference tree exists."""
    from oracle import bindings, ctrl_bindings
    if not ctrl_bindings.ref_available() and bindings.reference_dir():
        ctrl_bindings.build("ref")
    if not ctrl_bindings.ref_available():
        pytest.skip("oracle/_ref/libmlctrl.so not built (no reference tree here)")
    return ctrl_bindings.ref_controllers


def _port(G, ctrl, offsets, changes, sr, state=None):
    from oracle.ctrl_bindings import port_controllers
    return port_controllers(G, ctrl, offsets, changes, sr, state)


def test_port_equals_golden():
    g = np.load(GOLDEN)
    for k in range(3):
        offsets = g["offsets_%d" % k]
        out, _, _ = _port(offsets.shape[1] - 1, g["ctrl_%d" % k], offsets, g["changes_%d" % k], float(g["sr_%d" % k]))
        assert_same_bits(out, g["out_%d" % k], "case %d" % k)
    o = g["out_0"]
    assert np.isnan(o).any() and np.isinf(o).any() and ((o != 0) & (np.abs(o) < np.finfo(np.float32).tiny)).any()


@pytest.mark.parametrize("sr", SAMPLE_RATES)
def test_glide_length(sr):
    """int(sr * 0.02f) in double, truncated to whole vectors (SmoothedController::process, .cpp:274-285)."""
    from oracle import ctrl_bindings
    lib = ctypes.CDLL(ctrl_bindings.PORT_LIB) if os.path.exists(ctrl_bindings.PORT_LIB) else None
    if lib is None:
        ctrl_bindings.build("port")
        lib = ctypes.CDLL(ctrl_bindings.PORT_LIB)
    per, dy = ctypes.c_float(), ctypes.c_float()
    lib.mlport_ctrl_glide(ctypes.c_float(sr), ctypes.byref(per), ctypes.byref(dy))
    assert per.value == GLIDE_VECTORS[sr]
    # a step from 0 to 1 lands after exactly that many vectors
    from oracle.ctrl_bindings import CHANGE_DTYPE
    T = GLIDE_VECTORS[sr] + 3
    offsets = np.zeros((T, 2), np.int32)
    offsets[:, 1] = 1
    offsets[0, 0] = 0
    offsets[1:, 0] = 1
    out, _, _ = _port(1, [1], offsets, np.array([(1, 0, 1.0)], CHANGE_DTYPE), sr)
    ends = out[:, 0, 0, 63]
    assert (ends[:GLIDE_VECTORS[sr] - 1] < 1).all() and (out[GLIDE_VECTORS[sr]:, 0, 0] == 1).all()


@pytest.mark.parametrize("sr", SAMPLE_RATES)
@pytest.mark.parametrize("protocol", [0, 1])
def test_port_equals_reference(ctrl_ref, sr, protocol):
    from oracle.ctrl_bindings import changes_from_events
    G, T = 9, 48
    phrases = special_phrases(G, T, seed=int(sr) + protocol)
    want = ctrl_ref(phrases, ALL_CONTROLLERS, T, sr, protocol=protocol)
    offsets, changes = changes_from_events(phrases, T, protocol=protocol)
    got, _, _ = _port(G, ALL_CONTROLLERS, offsets, changes, sr)
    assert_same_bits(got, want, "port vs EventsToSignals, sr %g, protocol %d" % (sr, protocol))
    assert np.isnan(want).any() and (want != 0).mean() > 0.01


def test_port_split_calls_and_state():
    """A run split in two, the second half from the state the first left, equals the run in one piece."""
    from madronalib_b200 import workloads as wl
    G, T, ctrl = 40, 30, [1, 7, 11, 128, 74]
    offsets, changes = wl.controller_changes(G, T, density=0.3, seed=5)
    whole, words, rows = _port(G, ctrl, offsets, changes, 48000.0)
    a, w1, r1 = _port(G, ctrl, offsets[:11], changes, 48000.0)
    b, w2, r2 = _port(G, ctrl, offsets[11:], changes, 48000.0, state=(w1, r1))
    assert_same_bits(np.concatenate([a, b]), whole, "split")
    assert (w2 == words).all() and (r2.view(np.uint32) == rows.view(np.uint32)).all()


def _router_changes(phrase, T, protocol):
    """The router's change list for one instrument: ([T] lists of (controller, value)), via api.EventRouter."""
    from madronalib_b200 import api
    r = api.EventRouter(4, protocol)
    records = np.zeros(r.n_records, np.dtype((np.void, 72)))
    for e in phrase:
        r.add_event(*e)
    per = []
    for t in range(T):
        r.process_vector(t * 64, records)
        per.append(r.controller_changes())
    r.close()
    return per


def _csr(per_instrument, T):
    from oracle.ctrl_bindings import CHANGE_DTYPE
    G = len(per_instrument)
    offsets = np.zeros((T, G + 1), np.int32)
    flat = []
    for t in range(T):
        for g in range(G):
            offsets[t, g] = len(flat)
            flat += [tuple(c) for c in per_instrument[g][t]]
        offsets[t, G] = len(flat)
    return offsets, np.array(flat, CHANGE_DTYPE)


def _phrases():
    """CC sweeps, channel pressure, CC > 128, CC 123, CC 120 (not 0, see ctrl_cases), notes, writes at one instant."""
    sweep = [(CONTROLLER, 1, 1, 7 * i, i / 40.0) for i in range(40)]
    pressure = [(CHANNEL_PRESSURE, 2, 0, 50 * i, (i % 5) / 4.0) for i in range(20)]
    mixed = [(NOTE_ON, 1, 60, 0, 60.0, 0.9), (CONTROLLER, 1, 300, 64, 0.7), (CONTROLLER, 1, 123, 64, 0.0),
             (CONTROLLER, 1, 120, 200, 0.5), (CONTROLLER, 1, 74, 300, 0.25), (CONTROLLER, 1, 74, 300, 0.75),
             (CONTROLLER, 3, 74, 300, 0.5), (NOTE_OFF, 1, 60, 400, 60.0), (CHANNEL_PRESSURE, 1, 0, 400, -0.0),
             (CONTROLLER, 1, 128, 600, 1e-40), (CONTROLLER, 1, 11, 700, float("nan")), (CONTROLLER, 1, 11, 1200, 1.0)]
    return [sweep, pressure, mixed, []] + special_phrases(4, 24, seed=77)


@pytest.mark.parametrize("protocol", [0, 1])
def test_router_changes_through_port_equal_reference(ctrl_ref, protocol):
    T, sr = 24, 48000.0
    phrases = _phrases()
    offsets, changes = _csr([_router_changes(p, T, protocol) for p in phrases], T)
    got, _, _ = _port(len(phrases), ALL_CONTROLLERS, offsets, changes, sr)
    want = ctrl_ref(phrases, ALL_CONTROLLERS, T, sr, protocol=protocol)
    assert_same_bits(got, want, "router -> port vs EventsToSignals, protocol %d" % protocol)
    assert (want[:, 128, 1] != 0).any() == (protocol == 0), "channel pressure is controller 128 in MIDI mode only"


def test_router_change_order_and_clamp():
    from madronalib_b200 import api
    r = api.EventRouter(2, 0)
    records = np.zeros(r.n_records, np.dtype((np.void, 72)))
    for e in [(CONTROLLER, 1, 7, 5, 0.25), (CONTROLLER, 1, 7, 5, 0.5), (CONTROLLER, 1, 999, 3, 0.125),
              (CHANNEL_PRESSURE, 1, 0, 5, 0.75), (CONTROLLER, 1, 120, 70, 0.0)]:
        r.add_event(*e)
    r.process_vector(0, records)
    got = [(int(c["controller"]), float(c["value"])) for c in r.controller_changes()]
    # (time, type) order; of equal events the one added later comes first (addEvent's lower bound)
    assert got == [(128, 0.125), (7, 0.5), (7, 0.25), (128, 0.75)]
    r.process_vector(64, records)
    assert [(int(c["controller"]), float(c["value"])) for c in r.controller_changes()] == [(120, 0.0)]
    assert r.unsupported_events == 1, "CC 120 stays unsupported; its controller write is routed"
    r.close()
    r = api.EventRouter(2, 1)
    r.add_event(CHANNEL_PRESSURE, 2, 0, 0, 0.5)
    r.process_vector(0, np.zeros(r.n_records, np.dtype((np.void, 72))))
    assert r.controller_changes().size == 0, "MPE channel pressure writes no controller"
    r.close()


def test_workload_controller_changes():
    from madronalib_b200 import workloads as wl
    G, T = 300, 16
    offsets, changes = wl.controller_changes(G, T, density=0.2, seed=9)
    assert offsets.shape == (T, G + 1) and offsets[0, 0] == 0 and offsets[-1, -1] == changes.size
    assert (np.diff(offsets, axis=1) >= 0).all() and (offsets[1:, 0] == offsets[:-1, -1]).all()
    assert changes.itemsize == 8 and (changes["controller"] <= 128).all()
    # some blocks carry several writes to one controller
    dup = 0
    for t in range(T):
        for g in range(G):
            c = changes["controller"][offsets[t, g]:offsets[t, g + 1]]
            dup += len(c) != len(set(c.tolist()))
    assert dup > 0


def test_create_argument_errors():
    """Checked on the host before any device is touched: each error names the offending value."""
    from madronalib_b200 import api
    cases = [((0, [1]), "n_instruments"), ((4, [1], 0.0), "sample_rate"), ((4, [1], 48000.0, 2), "protocol"),
             ((4, []), "n_controllers"), ((4, list(range(129)) + [5]), "n_controllers"),
             ((4, [1, 129]), "controller 129 \\(list index 1\\)"), ((4, [3, -1]), "controller -1"),
             ((4, [7, 1, 7]), "controller 7 is requested twice \\(list indexes 0 and 2\\)")]
    for args, msg in cases:
        with pytest.raises(api.MlbError, match=msg) as e:
            api.ControllerBank(*args)
        assert e.value.code == 1
    with pytest.raises(ValueError):
        api.ControllerBank(4, [[1, 2]])
