"""K12 on the GPU: the event routing of many instruments (mlb_routers_*), checked record byte for record byte, change
list and counters against G host routers (tests/router_cases.route_on_host); and contract E from raw events
(mlb_synth_process_routed_host) bit for bit against the record path fed by the host routers."""
import numpy as np
import pytest

from madronalib_b200 import workloads as wl
from tests.common import assert_same_bits
from tests.router_cases import csr, edge_blocks, route_on_host, unison_release_blocks

pytestmark = pytest.mark.gpu


def _bytes(a):
    return np.ascontiguousarray(a).view(np.uint8)


def run_split(gpu, layout, offsets, events, mpe, unison=None, mod_cc=None, splits=()):
    """Route on the device in calls split at `splits` -> (records, change_offsets, changes, overflow, unsupported)."""
    r = gpu.RouterBank(layout["polyphony"], layout["first_voice"], layout["n_voices"], 1 if mpe else 0, unison, mod_cc)
    try:
        recs, coffs, chs, base = [], [], [], 0
        cuts = [0] + list(splits) + [offsets.shape[0]]
        for a, b in zip(cuts[:-1], cuts[1:]):
            rec, coff, ch = r.process_host(offsets[a:b], events)
            recs.append(rec)
            coffs.append(coff + base)
            chs.append(ch)
            base += ch.size
        ovf, uns = r.counters()
    finally:
        r.close()
    return np.concatenate(recs), np.concatenate(coffs), np.concatenate(chs), ovf, uns


def check_equal(got, want, what):
    rec, coff, ch, ovf, uns = got
    wrec, wcoff, wch, wovf, wuns = want
    assert np.array_equal(_bytes(rec), _bytes(wrec)), what + ": records"
    assert np.array_equal(coff, wcoff), what + ": change offsets"
    assert np.array_equal(_bytes(ch), _bytes(wch)), what + ": changes"
    assert np.array_equal(ovf, wovf), what + ": overflow"
    assert np.array_equal(uns, wuns), what + ": unsupported"


@pytest.mark.parametrize("G", [1, 33, 4096])
@pytest.mark.parametrize("mode", ["midi", "mpe", "unison"])
def test_records_changes_counters_equal_host_routers(gpu, G, mode):
    mpe = mode == "mpe"
    T = 24 if G < 4096 else 10
    rng = np.random.default_rng(G * 7 + len(mode))
    poly = rng.integers(1, 17, G).astype(np.int32) if G > 1 else np.array([4], np.int32)
    lay = wl.midi_layout(G, poly, mpe, gap=1 if G == 33 else 0)
    unison = (rng.random(G) < 0.5).astype(np.int32) if mode == "unison" else None
    mod_cc = rng.choice([1, 16, 73, 74], G).astype(np.int32)
    offsets, ev = wl.midi_performance(G, T, poly, mpe, density=0.6 if G < 4096 else 0.1, seed=G + 5)
    want = route_on_host(offsets, ev, lay, mpe, unison, mod_cc)
    got = run_split(gpu, lay, offsets, ev, mpe, unison, mod_cc, splits=(T // 3, T // 3 + 1))
    check_equal(got, want, f"G {G} {mode}")
    assert want[2].size > 0 and (want[0]["n_events"] > 0).any()


def test_polyphony_0_to_16_and_gaps(gpu):
    G, T = 17, 30
    poly = np.arange(17, dtype=np.int32)
    lay = wl.midi_layout(G, poly, False, gap=2)
    offsets, ev = wl.midi_performance(G, T, np.maximum(poly, 1), False, density=0.8, seed=3)
    mod_cc = np.arange(G, dtype=np.int32) * 7 % 129
    want = route_on_host(offsets, ev, lay, False, None, mod_cc)
    got = run_split(gpu, lay, offsets, ev, False, None, mod_cc)
    check_equal(got, want, "polyphony 0..16")
    assert not _bytes(got[0][:, lay["voice_instrument"] < 0]).any(), "voices of no instrument get zero records"


@pytest.mark.parametrize("mpe", [False, True])
def test_200_events_in_one_vector_with_overflow(gpu, mpe):
    G, T = 3, 4
    lay = wl.midi_layout(G, [16, 2, 5], mpe)
    offsets, ev = wl.midi_performance(G, T, [16, 2, 5], mpe, density=1.0, seed=9)
    rng = np.random.default_rng(1)
    many = np.concatenate([wl.midi_performance(1, 1, 2, mpe, density=1.0, seed=100 + s)[1] for s in range(80)])[:200]
    many["time"] = rng.integers(0, 4, many.size)  # many equal times
    assert many.size == 200
    # block 2, instrument 1 gets the 200 events
    rows = [ev[offsets[t, g]:offsets[t, g + 1]] if (t, g) != (2, 1) else many for t in range(T) for g in range(G)]
    offsets2 = np.zeros((T, G + 1), np.int32)
    sizes = np.array([r.size for r in rows]).reshape(T, G)
    ends = np.cumsum(sizes.ravel()).reshape(T, G)
    offsets2[:, 1:] = ends
    offsets2[:, 0] = np.concatenate(([0], ends[:-1, -1]))
    ev2 = np.concatenate(rows)
    want = route_on_host(offsets2, ev2, lay, mpe)
    got = run_split(gpu, lay, offsets2, ev2, mpe)
    check_equal(got, want, "200 events")
    assert want[3][1] > 0, "overflow happened"


@pytest.mark.parametrize("mpe", [False, True])
def test_edge_cases(gpu, mpe):
    G = 2
    lay = wl.midi_layout(G, [2, 3], mpe)
    offsets, ev = csr(edge_blocks(), G)
    if mpe:  # the key is the channel in MPE: keys >= 128 do not exist there, channels >= 128 do
        ev["channel"] = np.where(ev["source_idx"] >= 128, 200, ev["channel"] + (ev["source_idx"] % 7))
    want = route_on_host(offsets, ev, lay, mpe)
    got = run_split(gpu, lay, offsets, ev, mpe, splits=(2,))
    check_equal(got, want, "edge cases")
    assert want[4][0] == 1, "CC 120 with value 0 counted"


def test_unison_release_and_voice_0(gpu):
    G = 2
    lay = wl.midi_layout(G, [3, 1], False)
    offsets, ev = csr(unison_release_blocks(), G)
    unison = np.array([1, 0], np.int32)
    want = route_on_host(offsets, ev, lay, False, unison)
    got = run_split(gpu, lay, offsets, ev, False, unison)
    check_equal(got, want, "unison release")
    assert (want[0]["n_events"] > 0).any()


def test_clear_mid_performance_equals_fresh_bank(gpu):
    G, T = 40, 20
    lay = wl.midi_layout(G, 6, False)
    offsets, ev = wl.midi_performance(G, T, 6, False, density=0.7, seed=4)
    r = gpu.RouterBank(lay["polyphony"], lay["first_voice"], lay["n_voices"])
    fresh = gpu.RouterBank(lay["polyphony"], lay["first_voice"], lay["n_voices"])
    try:
        r.process_host(offsets[:10], ev)
        ovf0, uns0 = r.counters()
        r.clear()
        assert np.array_equal(r.counters()[0], ovf0) and np.array_equal(r.counters()[1], uns0), "counters kept"
        a = r.process_host(offsets[10:], ev)
        b = fresh.process_host(offsets[10:], ev)
    finally:
        r.close()
        fresh.close()
    for x, y in zip(a, b):
        assert np.array_equal(_bytes(x), _bytes(y))


def test_three_launches_per_call_and_graph_replay(gpu):
    import torch
    G, T = 50, 8
    lay = wl.midi_layout(G, 5, True)
    offsets, ev = wl.midi_performance(G, T, 5, True, density=0.7, seed=6)
    want = route_on_host(offsets, ev, lay, True)
    r = gpu.RouterBank(lay["polyphony"], lay["first_voice"], lay["n_voices"], 1)
    try:
        d_off = torch.from_numpy(offsets).cuda()
        d_ev = torch.from_numpy(ev.view(np.uint8)).cuda()
        d_rec = torch.empty((T, lay["n_voices"], 72), dtype=torch.uint8, device="cuda")
        d_coff = torch.empty((T, G + 1), dtype=torch.int32, device="cuda")
        d_ch = torch.empty((max(ev.size, 1), 8), dtype=torch.uint8, device="cuda")
        s = torch.cuda.Stream()
        n0 = gpu.kernel_launches()
        with torch.cuda.stream(s):
            r.process_device(d_off, d_ev, d_rec, d_coff, d_ch, T, s.cuda_stream)
        s.synchronize()
        assert gpu.kernel_launches() - n0 == 3
        n = int(d_coff[-1, -1])
        assert np.array_equal(d_rec.cpu().numpy().ravel(), _bytes(want[0]).ravel())
        assert np.array_equal(d_coff.cpu().numpy(), want[1])
        assert np.array_equal(d_ch[:n].cpu().numpy().ravel(), _bytes(want[2]).ravel())
        # captured into a CUDA graph from a cleared bank and replayed: the same bytes
        r.clear()
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, stream=s):
            r.process_device(d_off, d_ev, d_rec, d_coff, d_ch, T, s.cuda_stream)
        r.clear()
        d_rec.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert np.array_equal(d_rec.cpu().numpy().ravel(), _bytes(want[0]).ravel())
        assert np.array_equal(d_coff.cpu().numpy(), want[1])
    finally:
        r.close()


def _graphs(gpu, V, n_ctrl):
    from madronalib_b200.graph import GraphSpec
    gs = GraphSpec()
    pitch, gate = gs.input(0), gs.input(1)
    k = gs.param()
    y = gs.node("MULTIPLY", gs.node("SINE", gs.node("MULTIPLY", pitch, k)), gate)
    if n_ctrl:
        y = gs.node("MULTIPLY", y, gs.node("ADD", gs.input(8), gs.input(8 + n_ctrl - 1)))
    gs.output(gs.node("ADD", y, gs.input(5)))
    coef, state = gs.new_coefs(V), gs.new_state(V)
    coef[0] = np.float32(0.01)
    g = gpu.VoiceGraph(gs, V)
    g.set_coefs(coef)
    g.set_state(state)
    return g, coef, state


def _fused(gpu, V):
    w = wl.config_a(V)
    g = gpu.VoiceGraph(w.spec, V)
    g.set_coefs(w.coef)
    g.set_state(w.state)
    assert g.kernel_name.startswith("fused:")
    return g, w.coef, w.state


@pytest.mark.parametrize("mpe", [False, True])
@pytest.mark.parametrize("kind", ["fused", "interpreted", "interpreted+controllers", "buses"])
def test_routed_contract_e_equals_record_path(gpu, mpe, kind):
    G, P, T = (4096, 16, 64) if (kind == "buses" and not mpe) else (37, 5, 20)
    lay = wl.midi_layout(G, P, mpe)
    V = lay["n_voices"]
    offsets, ev = wl.midi_performance(G, T, P, mpe, density=0.1 if G == 4096 else 0.6, seed=G + T)
    rec, coff, ch, _, _ = route_on_host(offsets, ev, lay, mpe)
    vi, gs_, da, pb = wl.synth_bank_params(V)
    vi = lay["voice_index"]
    ctrl = [1, 74, 128] if kind == "interpreted+controllers" else []

    def make():
        vb = gpu.VoiceBank(48000.0, vi, gs_, da, pb, flags=0 if mpe else gpu.VoiceBank.MIDI)
        if mpe:
            vb.set_main_voices(lay["main_voice"])
        cb = None
        if ctrl:
            cb = gpu.ControllerBank(G, ctrl, 48000.0, 1 if mpe else 0)
            cb.set_voice_map(lay["voice_instrument"])
        g, _, _ = _fused(gpu, V) if kind == "fused" else _graphs(gpu, V, len(ctrl))
        return vb, cb, g

    vb, cb, g = make()
    r = gpu.RouterBank(lay["polyphony"], lay["first_voice"], V, 1 if mpe else 0)
    buses = gpu.Buses(V, lay["bus_first"], lay["bus_count"]) if kind == "buses" else None
    try:
        if buses is not None:
            got = g.process_routed_host(r, vb, offsets[:T // 2], ev, buses=buses)
            got = np.concatenate([got, g.process_routed_host(r, vb, offsets[T // 2:], ev, buses=buses)])
        else:
            got, got_mix = g.process_routed_host(r, vb, offsets, ev, controllers=cb, want_mix=True)
        got_st = g.get_state()
    finally:
        for h in (vb, cb, g, r):
            if h is not None:
                h.close()
    vb, cb, g = make()
    try:
        if buses is not None:
            want = g.process_events_buses_host(vb, buses, np.ascontiguousarray(rec))
        elif cb is not None:
            want, want_mix = g.process_events_controllers_host(vb, cb, rec, coff, ch, want_mix=True)
        else:
            want, want_mix = g.process_events_host(vb, rec, want_mix=True)
        want_st = g.get_state()
    finally:
        for h in (vb, cb, g, buses):
            if h is not None:
                h.close()
    assert_same_bits(got, want, f"routed contract E, {kind}")
    if buses is None:
        assert_same_bits(got_mix, want_mix, "mix bus")
    assert np.array_equal(got_st, want_st), "graph state"
    assert np.abs(want).max() > 0


def test_argument_errors(gpu):
    G, T = 4, 3
    lay = wl.midi_layout(G, 4, False)
    V = lay["n_voices"]
    offsets, ev = wl.midi_performance(G, T, 4, False, density=1.0, seed=2)
    r = gpu.RouterBank(lay["polyphony"], lay["first_voice"], V)
    r_mpe = gpu.RouterBank(lay["polyphony"], np.arange(G, dtype=np.int32) * 5, G * 5, 1)
    vi, gs_, da, pb = wl.synth_bank_params(V)
    vb = gpu.VoiceBank(48000.0, vi, gs_, da, pb, flags=gpu.VoiceBank.MIDI)
    vb_mpe = gpu.VoiceBank(48000.0, vi, gs_, da, pb)
    g, _, _ = _graphs(gpu, V, 0)
    g2, _, _ = _graphs(gpu, V + 1, 0)
    try:
        bad = offsets.copy()
        bad[1, 2] = bad[1, 3] + 1
        with pytest.raises(gpu.MlbError, match="block 1, instrument 2"):
            r.process_host(bad, ev)
        badt = ev.copy()
        badt["time"][offsets[2, 1]] = 64
        with pytest.raises(gpu.MlbError, match=f"block 2, instrument 1, event {offsets[2, 1]}: time 64"):
            r.process_host(offsets, badt)
        with pytest.raises(gpu.MlbError, match="block 1, instrument 2"):
            g.process_routed_host(r, vb, bad, ev)
        with pytest.raises(gpu.MlbError, match="time 64"):
            g.process_routed_host(r, vb, offsets, badt)
        with pytest.raises(gpu.MlbError, match="voice bank has 16 voices, graph has 17"):
            g2.process_routed_host(r, vb, offsets, ev)
        with pytest.raises(gpu.MlbError, match="router bank protocol MIDI, voice bank without MLB_VOICES_MIDI"):
            g.process_routed_host(r, vb_mpe, offsets, ev)
        with pytest.raises(gpu.MlbError, match="router bank writes 20 voices, graph has 16"):
            g.process_routed_host(r_mpe, vb_mpe, offsets, ev)
        cb = gpu.ControllerBank(G, [1], 48000.0, 1)
        cb.set_voice_map(lay["voice_instrument"])
        with pytest.raises(gpu.MlbError, match="router bank protocol MIDI, controller bank MPE"):
            g.process_routed_host(r, vb, offsets, ev, controllers=cb)
        cb.close()
        out, _ = g.process_routed_host(r, vb, offsets, ev)
        assert out.shape == (T, 1, V, 64)
    finally:
        for h in (r, r_mpe, vb, vb_mpe, g, g2):
            h.close()


def test_same_range_in_two_blocks_and_capacity(gpu):
    """Offsets may reference one range in several blocks: its writes count once per reference, the wrapper sizes the
    change list from the library's count, and a host call with too small a capacity is refused before any copy."""
    import ctypes
    from tests.router_cases import CC
    G = 2
    lay = wl.midi_layout(G, 3, False)
    offsets, ev = csr([{0: [(CC, 1, 1, t, 0.1 * t, 0.0) for t in range(4)]}], G)
    offsets = np.ascontiguousarray(np.repeat(offsets, 2, axis=0))  # [[0, 4, 4], [0, 4, 4]]
    want = route_on_host(offsets, ev, lay)
    assert want[2].size == 8
    check_equal(run_split(gpu, lay, offsets, ev, False), want, "one range in two blocks")
    r = gpu.RouterBank(lay["polyphony"], lay["first_voice"], lay["n_voices"])
    try:
        rec = np.zeros((2, lay["n_voices"]), wl.VOICE_EVENTS_DTYPE)
        coff = np.full((2, G + 1), -7, np.int32)
        ch = np.zeros(4, gpu.CONTROLLER_CHANGE_DTYPE)
        n = ctypes.c_int(-1)
        rc = gpu.lib().mlb_routers_process_host(r._h, offsets.ctypes.data, ev.ctypes.data, int(ev.size),
                                                rec.ctypes.data, coff.ctypes.data, ch.ctypes.data, int(ch.size),
                                                ctypes.byref(n), 2)
        assert rc == 1 and "make 8 controller writes, changes has room for 4" in gpu.lib().mlb_last_error().decode()
        assert (coff == -7).all() and not _bytes(ch).any(), "nothing copied"
    finally:
        r.close()


def test_mpe_polyphony_0_main_voice_record(gpu):
    """An MPE instrument of polyphony 0 has one record, its main voice: a note-on finds no free voice and the nearest
    voice is voice 0 (retrigger); channel-1 bend and pressure; CC 123 writes a note-off.  No host router of polyphony 0
    exists, so the record is written out here."""
    from tests.router_cases import BEND, CC, CPRESS, ON
    G = 2
    lay = wl.midi_layout(G, [0, 2], True)
    blocks = [{0: [(ON, 3, 60, 5, 5.0, 0.75), (BEND, 1, 0, 9, -0.5, 0.0), (CPRESS, 1, 0, 9, 0.25, 0.0),
                   (CC, 3, 123, 20, 0.0, 0.0)], 1: [(ON, 2, 61, 1, 5.1, 0.5)]}]
    offsets, ev = csr(blocks, G)
    got = run_split(gpu, lay, offsets, ev, True)
    r = got[0][0, 0]
    assert r["n_events"] == 2 and r["set_mask"] == 1 | 16
    assert list(r["time"][:2]) == [5, 20] and list(r["type"][:2]) == [2, 4] and list(r["flags"][:2]) == [3, 2]
    assert r["value1"][0] == np.float32(5.0) and r["value2"][0] == np.float32(0.75)
    assert r["bend"] == np.float32(-0.5) and r["z"] == np.float32(0.25)
    assert got[2].size == 1 and got[2]["controller"][0] == 123
    # the second instrument is unaffected and equals a host router's routing
    sub = wl.midi_layout(1, [2], True)
    want = route_on_host(*csr([{0: blocks[0][1]}], 1), sub, True)
    assert np.array_equal(_bytes(got[0][:, 1:]), _bytes(want[0]))


def test_refused_call_leaves_routing_state(gpu):
    G, T = 6, 8
    lay = wl.midi_layout(G, 4, False)
    offsets, ev = wl.midi_performance(G, T, 4, False, density=0.9, seed=17)
    bad = ev.copy()
    bad["time"][offsets[3, 2]] = -1
    r = gpu.RouterBank(lay["polyphony"], lay["first_voice"], lay["n_voices"])
    fresh = gpu.RouterBank(lay["polyphony"], lay["first_voice"], lay["n_voices"])
    try:
        r.process_host(offsets[:4], ev)
        fresh.process_host(offsets[:4], ev)
        with pytest.raises(gpu.MlbError, match="time -1"):
            r.process_host(offsets[3:], bad)
        a, b = r.process_host(offsets[4:], ev), fresh.process_host(offsets[4:], ev)
    finally:
        r.close()
        fresh.close()
    for x, y in zip(a, b):
        assert np.array_equal(_bytes(x), _bytes(y))


def test_routed_refusals_of_buses_and_controllers(gpu):
    G, T = 4, 3
    lay = wl.midi_layout(G, 4, False)
    V = lay["n_voices"]
    offsets, ev = wl.midi_performance(G, T, 4, False, density=1.0, seed=2)
    r = gpu.RouterBank(lay["polyphony"], lay["first_voice"], V)
    vi, gs_, da, pb = wl.synth_bank_params(V)
    vb = gpu.VoiceBank(48000.0, vi, gs_, da, pb, flags=gpu.VoiceBank.MIDI)
    g, _, _ = _graphs(gpu, V, 1)
    g0, _, _ = _graphs(gpu, V, 0)
    b = gpu.Buses(V + 2, [0], [4])
    cb_unmapped = gpu.ControllerBank(G, [1], 48000.0)
    cb_g = gpu.ControllerBank(G + 1, [1], 48000.0)
    cb_g.set_voice_map(np.append(lay["voice_instrument"], []).astype(np.int32))
    try:
        with pytest.raises(gpu.MlbError, match="buses are laid over 18 voices, graph has 16"):
            g0.process_routed_host(r, vb, offsets, ev, buses=b)
        with pytest.raises(gpu.MlbError, match="voice map has 0 voices, graph has 16"):
            g.process_routed_host(r, vb, offsets, ev, controllers=cb_unmapped)
        with pytest.raises(gpu.MlbError, match="router bank has 4 instruments, controller bank 5"):
            g.process_routed_host(r, vb, offsets, ev, controllers=cb_g)
    finally:
        for h in (r, vb, g, g0, b, cb_unmapped, cb_g):
            h.close()
