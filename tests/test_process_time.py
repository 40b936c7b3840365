"""K13, CPU side: the plain-C port of AudioContext::ProcessTime (oracle/port/mlport_ptime.c) against one complete
reference AudioContext per instrument (oracle/_ref/libmlptime.so, where it was built), phase rows and every state word,
NaN equal to NaN; the transport workload; the host-side checks of mlb_process_time_create."""
import numpy as np
import pytest

from madronalib_b200 import api, workloads as wl
from tests.common import assert_same_bits


@pytest.fixture(scope="module")
def pt_ref():
    """One reference AudioContext per instrument, compiled in place; built here where the reference tree exists."""
    from oracle import bindings, ptime_bindings
    if not ptime_bindings.ref_available() and bindings.reference_dir():
        ptime_bindings.build("ref")
    if not ptime_bindings.ref_available():
        pytest.skip("oracle/_ref/libmlptime.so not built (no reference tree here)")
    return ptime_bindings.ref_process_time


def _port(G, offsets, transports, sr, state=None):
    from oracle.ptime_bindings import port_process_time
    return port_process_time(G, offsets, transports, sr, state)


def assert_same_words(got, want, what):
    from oracle.ptime_bindings import same_words
    eq = same_words(got, want)
    assert eq.all(), f"{what}: state words differ at (word, instrument) {np.argwhere(~eq)[:4].tolist()}"


def _csr(per_block):
    """per_block[t] = list of (ppq, bpm, sr, playing) for one instrument -> (offsets [T][2], transports)."""
    off = np.zeros((len(per_block), 2), np.int32)
    flat = []
    for t, ups in enumerate(per_block):
        off[t, 0] = len(flat)
        flat += [(p, b, s, int(pl), 0) for p, b, s, pl in ups]
        off[t, 1] = len(flat)
    return off, np.array(flat, api.TRANSPORT_DTYPE)


def edge_script(sr=48000.0):
    """One instrument through every branch of setTimeAndRate: start, a steady run, two updates in one vector (dPhase /
    0: +inf clamped to 1, and 0 / 0 = NaN, which ml::clamp lets through), vectors without updates, a stop, a restart,
    a backwards jump, zero, -0 and negative positions, a tempo and a sample-rate change, a sample rate of 0, NaN and
    infinite updates (ignored), and an is_playing of 2."""
    q = 120.0 * 64 / (60.0 * sr)  # quarter notes per vector at 120 bpm
    nan, inf = float("nan"), float("inf")
    s = [[(3.0, 120.0, sr, 1)], [(3.0 + q, 120.0, sr, 1)], [(3.0 + 2 * q, 120.0, sr, 1)], [], [],
         [(3.0 + 5 * q, 120.0, sr, 1), (3.0 + 5 * q + 0.01, 120.0, sr, 1)],  # dPhase / 0 = +inf -> 1
         [(3.5, 120.0, sr, 1), (3.5, 120.0, sr, 1)],                         # the same position: inactive
         [(3.6, 120.0, sr, 1), (3.61, 120.0, sr, 1), (3.61 - 1e-9, 120.0, sr, 1)],
         [(3.75, 120.0, sr, 1), (4.75, 120.0, sr, 1)], [(5.0, 120.0, sr, 1)],  # dPhase 0 / 0 samples: NaN
         [(nan, 120.0, sr, 1)], [(4.0, inf, sr, 1)], [(-inf, 120.0, sr, 1)], [(4.5, nan, sr, 0)],
         [(4.0, 120.0, sr, 0)], [], [(4.0, 120.0, sr, 1)], [(4.0 + q, 120.0, sr, 1)],  # stop, then play again
         [(1.25, 120.0, sr, 1)],                                                      # backwards jump
         [(0.0, 120.0, sr, 1)], [(-0.0, 120.0, sr, 1)], [(-0.75, 120.0, sr, 1)], [(-2.25, 97.0, sr, 1)],
         [(-2.0, 97.0, 44100.0, 1)], [(-1.5, 200.0, 96000.0, 2)], [(0.0, 200.0, 96000.0, 0)],
         [(0.5, 150.0, 0.0, 1)], [(0.75, 150.0, 0.0, 1)], [(0.0, 150.0, 0.0, 0)], [(1.0, 150.0, sr, 1)],
         [(1.0 + 4 * q, 150.0, sr, 1)], [(1.0 + 4 * q, 150.0, sr, 1), (1.0 + 4 * q, 150.0, sr, 1)],
         [(2.0, 150.0, sr, 1)]] + [[]] * 40 + [[(9.0, 133.0, sr, 1)]] + [[(9.0 + 0.06 * k, 133.0, sr, 1)] for k in
                                                                         range(1, 8)]
    return _csr(s)


@pytest.mark.parametrize("sr", [44100, 48000, 96000])
def test_edge_script_equals_reference(pt_ref, sr):
    off, tr = edge_script(float(sr))
    want, want_w = pt_ref(1, off, tr, sr)
    got, got_w = _port(1, off, tr, float(sr))
    assert_same_bits(got, want, "edge script rows, sr %d" % sr)
    assert_same_words(got_w, want_w, "edge script state, sr %d" % sr)
    # the script reaches the wrapped, the inactive (-1), the NaN and the infinite phase
    assert np.isnan(want).any() and np.isinf(want).any() and (want == -1).any() and (want > 0.5).any()


@pytest.mark.parametrize("every,chaos", [(1, 0.0), (1, 0.15), (3, 0.3), (1, 0.6), (7, 0.0)])
@pytest.mark.parametrize("sr", [44100, 48000, 96000])
def test_port_equals_reference(pt_ref, sr, every, chaos):
    G, T = 23, 96
    off, tr = wl.transport_updates(G, T, float(sr), seed=sr + every + int(chaos * 100), every=every, chaos=chaos)
    want, want_w = pt_ref(G, off, tr, sr)
    got, got_w = _port(G, off, tr, float(sr))
    assert_same_bits(got, want, "rows, sr %d, every %d, chaos %g" % (sr, every, chaos))
    assert_same_words(got_w, want_w, "state, sr %d, every %d, chaos %g" % (sr, every, chaos))
    assert (want > 0).mean() > 0.2


def test_clear_mid_stream(pt_ref):
    """AudioContext::clear() between vectors resets dpdt_, active1_ and playing1_ only: the phase holds its last value
    until the next update, which then counts as a fresh start."""
    from oracle.ptime_bindings import port_clear
    G, T, sr = 11, 60, 48000
    off, tr = wl.transport_updates(G, T, float(sr), seed=5, every=2, chaos=0.2)
    cuts = [7, 8, 31]
    clear_before = np.zeros(T, np.int32)
    clear_before[cuts] = 1
    want, want_w = pt_ref(G, off, tr, sr, clear_before=clear_before)
    rows, w = [], None
    for t0, t1 in zip([0] + cuts, cuts + [T]):
        if t0:
            w = port_clear(w)
        o, w = _port(G, off[t0:t1], tr, float(sr), state=w)
        rows.append(o)
    got = np.concatenate(rows)
    assert_same_bits(got, want, "rows with clear()")
    assert_same_words(w, want_w, "state with clear()")
    plain, _ = pt_ref(G, off, tr, sr)
    assert not np.array_equal(plain.view(np.uint32), want.view(np.uint32))  # clear() did change something


def test_split_calls_carry_state():
    G, T, sr = 37, 50, 96000.0
    off, tr = wl.transport_updates(G, T, sr, seed=9, every=1, chaos=0.3)
    whole, w_whole = _port(G, off, tr, sr)
    parts, w = [], None
    for t0, t1 in ((0, 1), (1, 17), (17, 18), (18, 50)):
        o, w = _port(G, off[t0:t1], tr, sr, state=w)
        parts.append(o)
    assert_same_bits(np.concatenate(parts), whole, "split calls")
    assert_same_words(w, w_whole, "split calls, state")


def test_transport_workload():
    """The CSR layout, a steady host (one update per vector, nothing special) and the chaos kinds."""
    G, T, sr = 64, 40, 48000.0
    off, tr = wl.transport_updates(G, T, sr, seed=3)
    assert off.shape == (T, G + 1) and (np.diff(off.reshape(-1)) >= 0).all() and off[-1, -1] == tr.size == G * T
    assert (tr["is_playing"] == 1).all() and np.isfinite(tr["ppq_pos"]).all()
    rows, _ = _port(G, off, tr, sr)
    assert (rows[1:] >= 0).all() and (rows[1:] <= 1).all()  # a steady clock: phases in [0, 1] once started
    off, tr = wl.transport_updates(G, T, sr, seed=4, every=1, chaos=0.5)
    n = np.diff(off[:, :G + 1], axis=1)
    assert (n == 0).any() and (n == 2).any()
    assert np.isnan(tr["ppq_pos"]).any() and np.isnan(tr["bpm"]).any() and np.isinf(tr["ppq_pos"]).any()
    assert (tr["ppq_pos"] < 0).any() and (tr["is_playing"] == 0).any() and (tr["sample_rate"] != sr).any()
    # a restart is a stop followed by play from the top at the same instrument's next update
    inst = np.concatenate([np.repeat(np.arange(G), np.diff(off[t])) for t in range(T)])
    restarts = 0
    for g in range(G):
        mine = tr[inst == g]
        restarts += int(((mine["is_playing"][:-1] == 0) & (mine["is_playing"][1:] == 1) &
                         (mine["ppq_pos"][1:] == 0.0)).sum())
    assert restarts >= 5, restarts
    off3, tr3 = wl.transport_updates(G, T, sr, seed=4, every=3)
    assert off3[-1, -1] == tr3.size == G * len(range(0, T, 3))


def test_create_argument_errors():
    """Checked on the host before any device is touched: each error names the offending value.  The rate is whole
    hertz, as the reference's AudioContext(nIn, nOut, int rate) takes it."""
    for args, msg in (((0,), "n_instruments"), ((-3, 48000.0), "n_instruments"), ((4, 0.0), "sample_rate"),
                      ((4, -48000.0), "sample_rate"), ((4, float("nan")), "sample_rate"),
                      ((4, float("inf")), "sample_rate"), ((4, 44100.5), "whole number of hertz .*44100.5"),
                      ((4, 0.5), "sample_rate"), ((4, 2.0 ** 31), "sample_rate")):
        with pytest.raises(api.MlbError, match=msg) as e:
            api.ProcessTimeBank(*args)
        assert e.value.code == 1
