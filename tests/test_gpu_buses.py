"""K10 on the GPU: per-instrument output buses (mlb_buses_*), bit-exact against the strict-order port
(oracle/port/mlport_bus.c, itself pinned to the reference's Synth::processVector by tests/test_buses.py), NaN == NaN.
Also contract E with bus output (mlb_synth_process_buses_host) against port(bank) -> port(graph) -> port(buses), and
bus rows fed as they are into a per-instrument effect graph."""
import os

import numpy as np
import pytest

from madronalib_b200 import workloads as wl
from tests.bus_cases import random_layout, special_rows
from tests.common import assert_same_bits, assert_state_equal

pytestmark = pytest.mark.gpu

NTHREADS = max(1, len(os.sched_getaffinity(0)))


def port_buses(rows, first, count):
    from oracle.bus_bindings import port_buses as f
    return f(rows, first, count)


@pytest.fixture(scope="module")
def port_bank():
    from oracle import bindings
    return bindings.port_voice_bank()


def _layout(name):
    """(V, first, count) of the layouts the device sum is checked on."""
    rng = np.random.default_rng(len(name))
    if name == "g1_all":  # the weak case: one long serial chain per (t, p)
        V = 3001
        return V, np.array([0], np.int32), np.array([V], np.int32)
    if name == "g7_counts":
        V = 1200
        count = np.array([0, 1, 16, 17, 33, 1000, V], np.int32)
        first = np.array([rng.integers(0, V - c + 1) for c in count], np.int32)
        return V, first, count
    if name == "g4096_random":  # gaps and overlaps
        V = 5000
        first, count = random_layout(rng, V, 4096, 33)
        return V, first, count
    if name == "g4096_mpe":  # main voices skipped
        first, count = wl.instrument_buses(4096, 2, mpe=True)
        return 4096 * 3, first, count
    raise KeyError(name)


def _sum_on_device(gpu, V, first, count, rows):
    import torch
    T, P = rows.shape[:2]
    b = gpu.Buses(V, first, count)
    try:
        x = torch.from_numpy(rows).cuda()
        y = torch.full((T, P, len(first), 64), float("nan"), device="cuda")
        b.sum_device(x, y, P, T, torch.cuda.current_stream().cuda_stream)
        return y.cpu().numpy()
    finally:
        b.close()


@pytest.mark.parametrize("layout", ["g1_all", "g7_counts", "g4096_random", "g4096_mpe"])
@pytest.mark.parametrize("P,T", [(1, 64), (2, 5), (8, 1)])
def test_sum_device_equals_port(gpu, layout, P, T):
    """Layouts with buses of 1 000 voices and more get finite special values: with inf and NaN in the rows every
    column of such a bus would be NaN, and its order would go unchecked."""
    V, first, count = _layout(layout)
    nonfinite = int(count.max()) <= 33
    rows = special_rows(T, P, V, seed=7 * P + T, nonfinite=nonfinite)
    got = _sum_on_device(gpu, V, first, count, rows)
    want = port_buses(rows, first, count)
    assert_same_bits(got, want, f"{layout}, P = {P}, T = {T}")
    assert np.isfinite(want).all() != nonfinite


def test_one_launch_per_call_and_graph_replay(gpu):
    import torch
    V, first, count = _layout("g7_counts")
    T, P = 5, 2
    rows = special_rows(T, P, V, seed=3)
    b = gpu.Buses(V, first, count)
    try:
        x = torch.from_numpy(rows).cuda()
        y = torch.empty((T, P, len(first), 64), device="cuda")
        n0 = gpu.kernel_launches()
        b.sum_device(x, y, P, T, torch.cuda.current_stream().cuda_stream)
        assert gpu.kernel_launches() - n0 == 1
        torch.cuda.synchronize()
        direct = y.cpu().numpy().copy()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            b.sum_device(x, y, P, T, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        y.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert_same_bits(y.cpu().numpy(), direct, "graph replay vs direct call")
    finally:
        b.close()
    assert_same_bits(direct, port_buses(rows, first, count), "direct call vs port")


def _expect(port, port_bank, w, ev, prm, planes, first, count):
    T, V = ev.shape
    rows, _ = port_bank.run(48000.0, *prm, ev, nthreads=NTHREADS)
    out, _, st = port.run(w.spec, V, T, np.ascontiguousarray(rows[:, planes]), w.state, w.coef, nthreads=NTHREADS)
    return port_buses(out, first, count), st


@pytest.mark.parametrize("chunk,calls", [(8, (20,)), (0, (20,)), (3, (7, 13))])
def test_events_to_buses_fused_chain(gpu, port, port_bank, monkeypatch, chunk, calls):
    """Config A reading the bank's kPitch row, 19 instruments x 16 voices; time chunks of 8 / one chunk / two
    successive calls with ragged chunks (bank and chain state carry across chunks and calls)."""
    if chunk:
        monkeypatch.setenv("MLB_SYNTH_CHUNK_BLOCKS", str(chunk))
    else:
        monkeypatch.delenv("MLB_SYNTH_CHUNK_BLOCKS", raising=False)
    first, count = wl.instrument_buses(19, 16)
    V, T = 19 * 16, sum(calls)
    w = wl.config_a(V)
    ev = wl.synth_events(V, T, seed=21, density=0.3, ctl=0.2)
    prm = wl.synth_bank_params(V)
    want, want_st = _expect(port, port_bank, w, ev, prm, [0], first, count)
    vb = gpu.VoiceBank(48000.0, *prm)
    g = gpu.VoiceGraph(w.spec, V)
    b = gpu.Buses(V, first, count)
    try:
        assert g.kernel_name.startswith("fused:")
        g.set_coefs(w.coef)
        g.set_state(w.state)
        outs, t0 = [], 0
        for n in calls:
            outs.append(g.process_events_buses_host(vb, b, np.ascontiguousarray(ev[t0:t0 + n])))
            t0 += n
            if chunk:
                assert g.last_host_slices == (n + chunk - 1) // chunk
        st = g.get_state()
    finally:
        for h in (g, vb, b):
            h.close()
    got = np.concatenate(outs)
    assert got.shape == (T, 1, 19, 64)
    assert_same_bits(got, want, "events -> chain A -> buses")
    assert_state_equal(st, want_st, "events -> chain A -> buses: state")
    assert np.abs(want).max() > 0.01


def test_events_to_buses_interpreted_graph(gpu, port, port_bank, monkeypatch):
    """A graph reading pitch and gate (pitch x 2^-2 -> SineGen -> x gate) through the interpreter, MPE layout
    (each instrument's main voice outside its bus)."""
    from madronalib_b200.graph import GraphSpec, SINE_ZERO_PHASE
    monkeypatch.setenv("MLB_SYNTH_CHUNK_BLOCKS", "6")
    first, count = wl.instrument_buses(9, 7, mpe=True)
    V, T = 9 * 8, 16
    gs = GraphSpec()
    pitch, gate = gs.input(0), gs.input(1)
    k = gs.param()
    gs.output(gs.node("MULTIPLY", gs.node("SINE", gs.node("MULTIPLY", pitch, k)), gate))
    coef, state = gs.new_coefs(V), gs.new_state(V)
    coef[0] = np.float32(0.25)
    state[0] = SINE_ZERO_PHASE
    w = wl.Workload("pitch_sine_gate", gs, V, coef, state)
    ev = wl.synth_events(V, T, seed=23, density=0.3, ctl=0.2)
    prm = wl.synth_bank_params(V)
    want, want_st = _expect(port, port_bank, w, ev, prm, [0, 1], first, count)
    vb = gpu.VoiceBank(48000.0, *prm)
    g = gpu.VoiceGraph(gs, V)
    b = gpu.Buses(V, first, count)
    try:
        assert not g.kernel_name.startswith("fused:")
        g.set_coefs(coef)
        g.set_state(state)
        got = g.process_events_buses_host(vb, b, ev)
        st = g.get_state()
    finally:
        for h in (g, vb, b):
            h.close()
    assert_same_bits(got, want, "events -> interpreted graph -> buses")
    assert_state_equal(st, want_st, "state")
    assert np.abs(want).max() > 0.01


def test_bus_rows_feed_a_per_instrument_reverb(gpu, port):
    """A two-output voice graph's rows -> sum_device with P = 2 -> config 6 (Aaltoverb) with one voice per
    instrument, reading the two bus planes as its inputs: all on the device, against the same chain of checkers."""
    import torch
    from madronalib_b200.graph import GraphSpec
    n_inst, poly, T = 6, 16, 12
    V = n_inst * poly
    first, count = wl.instrument_buses(n_inst, poly)
    vg = GraphSpec()
    x0, x1 = vg.input(0), vg.input(1)
    k0, k1 = vg.param(), vg.param()
    vg.output(vg.node("MULTIPLY", x0, k0), vg.node("ADD", vg.node("MULTIPLY", x1, k1), x0))
    vcoef = vg.new_coefs(V)
    vcoef[vg.coef_slot(k0)] = np.float32(0.3) + np.float32(0.01) * np.arange(V, dtype=np.float32)
    vcoef[vg.coef_slot(k1)] = np.float32(-0.7)
    vstate = vg.new_state(V)
    inp = wl.config_6(V).inputs(T)
    fx = wl.config_6(n_inst)
    g1, g2 = gpu.VoiceGraph(vg, V), gpu.VoiceGraph(fx.spec, n_inst)
    b = gpu.Buses(V, first, count)
    try:
        g1.set_coefs(vcoef)
        g1.set_state(vstate)
        g2.set_coefs(fx.coef)
        g2.set_state(fx.state)
        s = torch.cuda.current_stream().cuda_stream
        d_in = torch.from_numpy(np.ascontiguousarray(inp)).cuda()
        d_rows = torch.empty((T, 2, V, 64), device="cuda")
        d_bus = torch.empty((T, 2, n_inst, 64), device="cuda")
        d_out = torch.empty((T, 2, n_inst, 64), device="cuda")
        g1.process_device(d_in, d_rows, None, T, s)
        b.sum_device(d_rows, d_bus, 2, T, s)
        g2.process_device(d_bus, d_out, None, T, s)
        torch.cuda.synchronize()
        got_bus, got = d_bus.cpu().numpy(), d_out.cpu().numpy()
        st = g2.get_state()
    finally:
        for h in (g1, g2, b):
            h.close()
    rows, _, _ = port.run(vg, V, T, inp, vstate, vcoef, nthreads=NTHREADS)
    want_bus = port_buses(rows, first, count)
    want, _, want_st = port.run(fx.spec, n_inst, T, want_bus, fx.state, fx.coef, nthreads=NTHREADS)
    assert_same_bits(got_bus, want_bus, "voice graph -> buses")
    assert_same_bits(got, want, "buses -> per-instrument Aaltoverb")
    assert_state_equal(st, want_st, "Aaltoverb state")
    assert np.abs(want).max() > 0.01


def test_events_to_buses_full_size(gpu, port, port_bank, monkeypatch):
    """65 536 voices x 64 vectors as 4 096 instruments x 16 voices, default time chunks: a stride of buses against
    port(bank) -> port(graph) -> port(buses) on those buses' voices (voices are independent)."""
    monkeypatch.delenv("MLB_SYNTH_CHUNK_BLOCKS", raising=False)
    V, T, n_inst, poly = 65536, 64, 4096, 16
    first, count = wl.instrument_buses(n_inst, poly)
    w = wl.config_a(V)
    ev = wl.synth_events(V, T)
    prm = wl.synth_bank_params(V)
    vb = gpu.VoiceBank(48000.0, *prm)
    g = gpu.VoiceGraph(w.spec, V)
    b = gpu.Buses(V, first, count)
    try:
        g.set_coefs(w.coef)
        g.set_state(w.state)
        got = g.process_events_buses_host(vb, b, ev)
        assert g.last_host_slices == 8
    finally:
        for h in (g, vb, b):
            h.close()
    sel = np.arange(0, n_inst, 37)
    voices = (first[sel, None] + np.arange(poly)[None, :]).reshape(-1)
    rows, _ = port_bank.run(48000.0, *(p[voices] for p in prm), np.ascontiguousarray(ev[:, voices]),
                            nthreads=NTHREADS)
    out, _, _ = port.run(w.spec, len(voices), T, np.ascontiguousarray(rows[:, 0:1]),
                         np.ascontiguousarray(w.state[:, voices]), np.ascontiguousarray(w.coef[:, voices]),
                         nthreads=NTHREADS)
    sub_first, sub_count = wl.instrument_buses(len(sel), poly)
    want = port_buses(out, sub_first, sub_count)
    assert_same_bits(got[:, :, sel], want, "contract E with buses, 65536 x 64 (%d-bus sample)" % len(sel))
    assert np.abs(want).max() > 0.01


def test_argument_errors(gpu):
    import torch
    from madronalib_b200.graph import GraphSpec
    V = 64
    first, count = wl.instrument_buses(4, 16)
    w = wl.config_a(V)
    prm = wl.synth_bank_params(V)
    vb = gpu.VoiceBank(48000.0, *prm)
    vb_small = gpu.VoiceBank(48000.0, *wl.voice_bank_params(32))
    g = gpu.VoiceGraph(w.spec, V)
    no_in = GraphSpec()
    no_in.output(no_in.node("NOISE"))
    g2 = gpu.VoiceGraph(no_in, V)
    far = GraphSpec()
    far.output(far.node("SINE", far.input(9)))
    g3 = gpu.VoiceGraph(far, V)
    no_out = GraphSpec()
    no_out.node("SINE", no_out.input(0))
    g4 = gpu.VoiceGraph(no_out, V)
    b = gpu.Buses(V, first, count)
    b_small = gpu.Buses(32, *wl.instrument_buses(2, 16))
    ev = wl.synth_events(V, 2)
    x = torch.zeros((2, 1, V, 64), device="cuda")
    y = torch.zeros((2, 1, 4, 64), device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    try:
        g.set_coefs(w.coef)
        # sum_device
        for rows, out, P, T in ((0, y, 1, 2), (x, 0, 1, 2), (x, y, 0, 2), (x, y, 1, 0), (x, y, -1, 2)):
            with pytest.raises(gpu.MlbError) as e:
                b.sum_device(rows, out, P, T, s)
            assert e.value.code == 1
        # process_events_buses_host
        with pytest.raises(gpu.MlbError, match="voices"):
            g.process_events_buses_host(vb_small, b, ev)
        with pytest.raises(gpu.MlbError, match="buses are laid over 32 voices"):
            g.process_events_buses_host(vb, b_small, ev)
        with pytest.raises(gpu.MlbError, match="no Voice row"):
            g2.process_events_buses_host(vb, b, ev)
        with pytest.raises(gpu.MlbError, match="not a Voice row"):
            g3.process_events_buses_host(vb, b, ev)
        with pytest.raises(gpu.MlbError, match="no outputs"):
            g4.process_events_buses_host(vb, b, ev)
        with pytest.raises(ValueError):
            g.process_events_buses_host(vb, b, ev[:, :10])
        with pytest.raises(ValueError):
            g.process_events_buses_host(vb, b, ev, out=np.zeros((2, 1, 5, 64), np.float32))
        with pytest.raises(gpu.MlbError, match="n_blocks"):
            g.process_events_buses_host(vb, b, ev[:0])
    finally:
        for h in (g, g2, g3, g4, vb, vb_small, b, b_small):
            h.close()
