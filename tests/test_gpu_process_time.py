"""K13 on the GPU: the host-transport beat phase (mlb_process_time_*), bit-exact against the plain-C port
(oracle/port/mlport_ptime.c, itself pinned to the reference's AudioContext by tests/test_process_time.py), NaN equal
to NaN: instrument rows and voice maps, ragged calls carrying state, state round trips and clear(), one launch per
call and CUDA-graph replay, every argument error; and contract E with every AudioContext signal
(mlb_synth_process_context_host) against its stages run one by one on the device."""
import numpy as np
import pytest

from madronalib_b200 import workloads as wl
from tests.common import assert_same_bits

pytestmark = pytest.mark.gpu


def port_pt(G, offsets, tr, sr=48000.0, state=None):
    from oracle.ptime_bindings import port_process_time
    return port_process_time(G, offsets, tr, sr, state)


def assert_same_words(got, want, what):
    from oracle.ptime_bindings import same_words
    eq = same_words(got, want)
    assert eq.all(), f"{what}: state words differ at (word, instrument) {np.argwhere(~eq)[:4].tolist()}"


def voice_rows(inst_rows, voice_instrument):
    """[T][G][64] instrument rows -> [T][V][64] voice rows (+0 for a voice of no instrument)."""
    vi = np.asarray(voice_instrument)
    out = inst_rows[:, np.maximum(vi, 0)].copy()
    out[:, vi < 0] = 0.0
    return out


@pytest.mark.parametrize("G", [1, 37, 4096 + 5])
def test_device_equals_port_ragged_calls(gpu, G):
    import torch
    sr, T = 48000.0, 64
    off, tr = wl.transport_updates(G, T, sr, seed=G, every=1, chaos=0.3)
    want, want_w = port_pt(G, off, tr, sr)
    bank = gpu.ProcessTimeBank(G, sr)
    try:
        d_tr = torch.from_numpy(tr.view(np.uint8)).cuda()
        s = torch.cuda.current_stream().cuda_stream
        got = []
        for t0, t1 in ((0, 1), (1, 14), (14, 15), (15, 64)):
            d_off = torch.from_numpy(np.ascontiguousarray(off[t0:t1])).cuda()
            y = torch.full((t1 - t0, 1, G, 64), 7.0, device="cuda")
            bank.process_device(d_off, d_tr, y, t1 - t0, stream=s)
            torch.cuda.synchronize()
            got.append(y.cpu().numpy()[:, 0])
            _, w = port_pt(G, off[:t1], tr, sr)
            assert_same_words(bank.get_state(), w, f"state after block {t1}")
    finally:
        bank.close()
    assert_same_bits(np.concatenate(got), want, f"G {G}, instrument rows")
    assert (want == -1).any() and (want > 0.5).any()


@pytest.mark.parametrize("sr", [44100, 48000, 96000])
def test_edge_script(gpu, sr):
    """Every branch of setTimeAndRate, NaN and infinite phases included (tests/test_process_time.edge_script)."""
    from tests.test_process_time import edge_script
    off, tr = edge_script(float(sr))
    want, want_w = port_pt(1, off, tr, float(sr))
    bank = gpu.ProcessTimeBank(1, float(sr))
    try:
        got = bank.process_host(off, tr)
        assert_same_words(bank.get_state(), want_w, "edge script state")
    finally:
        bank.close()
    assert_same_bits(got[:, 0], want, "edge script rows")
    assert np.isnan(want).any() and np.isinf(want).any()


@pytest.mark.parametrize("mpe", [False, True])
def test_voice_map_and_untouched_planes(gpu, mpe):
    G, T, sr = 37, 12, 44100.0
    lay = wl.midi_layout(G, 5, mpe, gap=1)
    off, tr = wl.transport_updates(G, T, sr, seed=3, every=2, chaos=0.2)
    want, _ = port_pt(G, off, tr, sr)
    bank = gpu.ProcessTimeBank(G, sr)
    try:
        bank.set_voice_map(lay["voice_instrument"])
        out = np.full((T, 3, lay["n_voices"], 64), 5.0, np.float32)
        first = np.ascontiguousarray(out[:5])
        bank.process_host(off[:5], tr, out=first, plane0=1, n_planes=3)
        rest = np.ascontiguousarray(out[5:])
        bank.process_host(off[5:], tr, out=rest, plane0=1, n_planes=3)
        got = np.concatenate([first, rest])
        assert (got[:, 0] == 5.0).all() and (got[:, 2] == 5.0).all(), "planes other than plane0 were written"
        assert_same_bits(got[:, 1], voice_rows(want, lay["voice_instrument"]), "voice rows")
        bank.set_voice_map(None)
        bank.clear()
    finally:
        bank.close()


def test_state_round_trip_and_clear(gpu):
    from oracle.ptime_bindings import port_clear
    G, T, sr = 200, 30, 96000.0
    off, tr = wl.transport_updates(G, T, sr, seed=17, every=1, chaos=0.25)
    _, w10 = port_pt(G, off[:10], tr, sr)
    want, want_w = port_pt(G, off[10:], tr, sr, state=port_clear(w10))
    bank = gpu.ProcessTimeBank(G, sr)
    other = gpu.ProcessTimeBank(G, 8000.0)
    try:
        bank.process_host(off[:10], tr)
        w = bank.get_state()
        assert_same_words(w, w10, "after 10 blocks")
        other.set_state(w)
        other.clear()
        assert_same_words(other.get_state(), port_clear(w10), "clear()")
        got = other.process_host(off[10:], tr)
        assert_same_words(other.get_state(), want_w, "after clear() and 20 more blocks")
    finally:
        bank.close()
        other.close()
    assert_same_bits(got[:, 0], want, "rows after set_state and clear()")


def test_one_launch_per_call_and_graph_replay(gpu):
    import torch
    G, T, sr = 100, 8, 48000.0
    off, tr = wl.transport_updates(G, T, sr, seed=11, every=1, chaos=0.3)
    want, _ = port_pt(G, off, tr, sr)
    base = gpu.live_handles()
    bank = gpu.ProcessTimeBank(G, sr)
    assert gpu.live_handles() == base + 1
    try:
        d_off = torch.from_numpy(off).cuda()
        d_tr = torch.from_numpy(tr.view(np.uint8)).cuda()
        y = torch.empty((T, 1, G, 64), device="cuda")
        w0 = bank.get_state()
        n0 = gpu.kernel_launches()
        bank.process_device(d_off, d_tr, y, T, stream=torch.cuda.current_stream().cuda_stream)
        assert gpu.kernel_launches() - n0 == 1
        torch.cuda.synchronize()
        direct = y.cpu().numpy().copy()
        bank.set_state(w0)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            bank.process_device(d_off, d_tr, y, T, stream=torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        bank.set_state(w0)
        y.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert_same_bits(y.cpu().numpy(), direct, "graph replay vs direct call")
        del g
    finally:
        bank.close()
    assert gpu.live_handles() == base
    assert_same_bits(direct[:, 0], want, "direct call vs port")


def test_argument_errors(gpu):
    import torch
    G = 8
    off, tr = wl.transport_updates(G, 4, seed=1)
    bank = gpu.ProcessTimeBank(G)
    try:
        w0 = bank.get_state()
        bad = off.copy()
        bad[2, 3] = bad[2, 4] + 1
        with pytest.raises(gpu.MlbError, match="block 2, instrument 3"):
            bank.process_host(bad, tr)
        with pytest.raises(gpu.MlbError, match="block 3, instrument 7"):
            bank.process_host(off, tr[:-1])
        with pytest.raises(gpu.MlbError, match="output planes"):
            bank.process_host(off, tr, plane0=1, n_planes=1)
        with pytest.raises(gpu.MlbError, match="voice 2: instrument 8"):
            bank.set_voice_map([0, 1, 8])
        with pytest.raises(gpu.MlbError, match="voice 0: instrument -2"):
            bank.set_voice_map([-2])
        with pytest.raises(gpu.MlbError, match="n_blocks"):
            bank.process_device(torch.zeros(9, dtype=torch.int32, device="cuda"), None,
                                torch.zeros(64 * G, device="cuda"), 0)
        with pytest.raises(gpu.MlbError, match="output planes"):
            bank.process_device(torch.zeros(9, dtype=torch.int32, device="cuda"), None,
                                torch.zeros(64 * G, device="cuda"), 1, plane0=-1)
        with pytest.raises(ValueError):
            bank.set_state(np.zeros((10, G + 1), np.uint64))
        assert np.array_equal(bank.get_state(), w0), "a refused call changed the state"
    finally:
        bank.close()


# ---- contract E with every AudioContext signal -------------------------------------------------------------------

def _graph(gpu, V, C, phase):
    """Voice rows 0, 1 and 5, controller planes 8 and 8 + C - 1, and the beat phase (plane 8 + C) into one output."""
    from madronalib_b200.graph import GraphSpec
    gs = GraphSpec()
    pitch, gate = gs.input(0), gs.input(1)
    k = gs.param()
    y = gs.node("MULTIPLY", gs.node("SINE", gs.node("MULTIPLY", pitch, k)), gate)
    if C:
        y = gs.node("MULTIPLY", y, gs.node("ADD", gs.input(8), gs.input(8 + C - 1)))
    if phase:
        y = gs.node("ADD", y, gs.node("MULTIPLY", gs.input(8 + C), k))
    gs.output(gs.node("ADD", y, gs.input(5)))
    coef, state = gs.new_coefs(V), gs.new_state(V)
    coef[0] = np.float32(0.01)
    g = gpu.VoiceGraph(gs, V)
    g.set_coefs(coef)
    g.set_state(state)
    return g, gs.n_in


@pytest.mark.parametrize("mpe", [False, True])
@pytest.mark.parametrize("ctrl,phase", [([1, 74, 128], True), ([], True), ([7, 1], False), ([], False)])
def test_context_contract_e_equals_stages(gpu, mpe, ctrl, phase):
    """mlb_synth_process_context_host, in two calls, against K12 -> K7 -> K11 -> K13 -> the graph run one by one
    through their own host entry points, and (without a process-time bank) against the routed entry point."""
    G, P, T, sr = 37, 5, 24, 48000.0
    C = len(ctrl)
    lay = wl.midi_layout(G, P, mpe)
    V = lay["n_voices"]
    offsets, ev = wl.midi_performance(G, T, P, mpe, density=0.6, seed=G + T + C)
    toff, tr = wl.transport_updates(G, T, sr, seed=5, every=1, chaos=0.1)
    vi, gs_, da, pb = wl.synth_bank_params(V)
    vi = lay["voice_index"]
    proto = 1 if mpe else 0

    def banks():
        r = gpu.RouterBank(lay["polyphony"], lay["first_voice"], V, proto)
        vb = gpu.VoiceBank(sr, vi, gs_, da, pb, flags=0 if mpe else gpu.VoiceBank.MIDI)
        if mpe:
            vb.set_main_voices(lay["main_voice"])
        cb = pt = None
        if C:
            cb = gpu.ControllerBank(G, ctrl, sr, proto)
            cb.set_voice_map(lay["voice_instrument"])
        if phase:
            pt = gpu.ProcessTimeBank(G, sr)
            pt.set_voice_map(lay["voice_instrument"])
        g, n_in = _graph(gpu, V, C, phase)
        return [r, vb, cb, pt, g], n_in

    (r, vb, cb, pt, g), n_in = banks()
    try:
        h = T // 3
        kw = dict(controllers=cb, times=pt, want_mix=True)
        o1, m1 = g.process_context_host(r, vb, offsets[:h], ev, time_offsets=toff[:h], transports=tr, **kw)
        o2, m2 = g.process_context_host(r, vb, offsets[h:], ev, time_offsets=toff[h:], transports=tr, **kw)
        got, got_mix, got_st = np.concatenate([o1, o2]), np.concatenate([m1, m2]), g.get_state()
    finally:
        for x in (r, vb, cb, pt, g):
            if x is not None:
                x.close()
    (r, vb, cb, pt, g), _ = banks()
    try:
        rec, coff, ch = r.process_host(offsets, ev)
        inp = np.zeros((T, max(n_in, 8), V, 64), np.float32)
        inp[:, :8] = vb.process_host(rec)
        if C:
            cb.process_host(coff, ch, out=inp, plane0=8, n_planes=n_in)
        if phase:
            pt.process_host(toff, tr, out=inp, plane0=8 + C, n_planes=n_in)
        want, want_mix = g.process_host(np.ascontiguousarray(inp[:, :n_in]), T, want_out=True, want_mix=True)
        want_st = g.get_state()
    finally:
        for x in (r, vb, cb, pt, g):
            if x is not None:
                x.close()
    assert_same_bits(got, want, f"context contract E, C {C}, phase {phase}")
    assert_same_bits(got_mix, want_mix, "mix bus")
    assert np.array_equal(got_st, want_st), "graph state"
    if phase:
        assert np.abs(inp[:, 8 + C]).max() > 0
    if not phase:
        (r, vb, cb, pt, g), _ = banks()
        try:
            routed, _ = g.process_routed_host(r, vb, offsets, ev, controllers=cb)
        finally:
            for x in (r, vb, cb, pt, g):
                if x is not None:
                    x.close()
        assert_same_bits(routed, want, "routed entry point")


def test_context_contract_e_buses_full_size(gpu):
    """4 096 instruments x 16 voices x 64 vectors, bus rows out, against the stages one by one (sampled buses)."""
    G, P, T, sr = 4096, 16, 64, 48000.0
    lay = wl.midi_layout(G, P, False)
    V = lay["n_voices"]
    offsets, ev = wl.midi_performance(G, T, P, False, density=0.1, seed=7)
    toff, tr = wl.transport_updates(G, T, sr, seed=8)
    vi, gs_, da, pb = wl.synth_bank_params(V)
    vi = lay["voice_index"]
    r = gpu.RouterBank(lay["polyphony"], lay["first_voice"], V)
    vb = gpu.VoiceBank(sr, vi, gs_, da, pb, flags=gpu.VoiceBank.MIDI)
    pt = gpu.ProcessTimeBank(G, sr)
    pt.set_voice_map(lay["voice_instrument"])
    g, n_in = _graph(gpu, V, 0, True)
    buses = gpu.Buses(V, lay["bus_first"], lay["bus_count"])
    try:
        got = g.process_context_host(r, vb, offsets, ev, times=pt, time_offsets=toff, transports=tr, buses=buses)
    finally:
        for x in (r, vb, pt, g, buses):
            x.close()
    # the same instruments through the stages, on a bank of 8 sampled instruments with their voices' parameters
    inst = np.array([0, 1, 31, 1000, 2047, 4000, 4094, 4095])
    sub_off, sub_ev = _sub_csr(offsets, ev, inst)
    sub_toff, sub_tr = _sub_csr(toff, tr, inst)
    lay8 = wl.midi_layout(len(inst), P, False)
    V8 = lay8["n_voices"]
    sel = (lay["first_voice"][inst][:, None] + np.arange(P)).reshape(-1)
    r = gpu.RouterBank(lay8["polyphony"], lay8["first_voice"], V8)
    vb = gpu.VoiceBank(sr, vi[sel], gs_[sel], da[sel], pb[sel], flags=gpu.VoiceBank.MIDI)
    pt = gpu.ProcessTimeBank(len(inst), sr)
    pt.set_voice_map(lay8["voice_instrument"])
    g, n_in = _graph(gpu, V8, 0, True)
    buses = gpu.Buses(V8, lay8["bus_first"], lay8["bus_count"])
    try:
        rec, _, _ = r.process_host(sub_off, sub_ev)
        inp = np.zeros((T, n_in, V8, 64), np.float32)
        inp[:, :8] = vb.process_host(rec)
        pt.process_host(sub_toff, sub_tr, out=inp, plane0=8, n_planes=n_in)
        rows, _ = g.process_host(inp, T)
        import torch
        d_bus = torch.empty((T, 1, len(inst), 64), device="cuda")
        buses.sum_device(torch.from_numpy(rows).cuda(), d_bus, 1, T, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        want = d_bus.cpu().numpy()
    finally:
        for x in (r, vb, pt, g, buses):
            x.close()
    assert_same_bits(got[:, :, inst], want, "4 096 instruments, sampled buses")
    assert np.abs(want).max() > 0


def test_context_contract_e_refusals(gpu):
    """Each mismatch is refused before anything is copied, and names itself."""
    G, T = 4, 3
    lay = wl.midi_layout(G, 4, False)
    V = lay["n_voices"]
    offsets, ev = wl.midi_performance(G, T, 4, False, density=1.0, seed=2)
    toff, tr = wl.transport_updates(G, T, seed=2)
    vi, gs_, da, pb = wl.synth_bank_params(V)
    r = gpu.RouterBank(lay["polyphony"], lay["first_voice"], V)
    vb = gpu.VoiceBank(48000.0, lay["voice_index"], gs_, da, pb, flags=gpu.VoiceBank.MIDI)
    pt = gpu.ProcessTimeBank(G)
    pt.set_voice_map(lay["voice_instrument"])
    pt_g = gpu.ProcessTimeBank(G + 1)
    pt_unmapped = gpu.ProcessTimeBank(G)
    g, _ = _graph(gpu, V, 0, True)
    g_beyond, _ = _graph(gpu, V, 1, True)  # reads planes 8 and 9: one past the beat phase without controllers
    try:
        w0 = pt.get_state()
        kw = dict(time_offsets=toff, transports=tr)
        with pytest.raises(gpu.MlbError, match="router bank has 4 instruments, process-time bank 5"):
            g.process_context_host(r, vb, offsets, ev, times=pt_g, **kw)
        with pytest.raises(gpu.MlbError, match="process-time bank's voice map has 0 voices, graph has 16"):
            g.process_context_host(r, vb, offsets, ev, times=pt_unmapped, **kw)
        bad = toff.copy()
        bad[1, 2] = bad[1, 3] + 1
        with pytest.raises(gpu.MlbError, match="block 1, instrument 2: transport range"):
            g.process_context_host(r, vb, offsets, ev, times=pt, time_offsets=bad, transports=tr)
        with pytest.raises(gpu.MlbError, match="INPUT plane 9 is not a Voice row, controller plane or the beat-phase "
                                               "plane \\(0..8\\)"):
            g_beyond.process_context_host(r, vb, offsets, ev, times=pt, **kw)
        with pytest.raises(ValueError):
            g.process_context_host(r, vb, offsets, ev, times=pt)
        assert np.array_equal(pt.get_state(), w0), "a refused call changed the beat-phase state"
        out, _ = g.process_context_host(r, vb, offsets, ev, times=pt, **kw)
        assert out.shape == (T, 1, V, 64)
    finally:
        for x in (r, vb, pt, pt_g, pt_unmapped, g, g_beyond):
            x.close()


def _sub_csr(offsets, items, inst):
    """The CSR list (events or transport updates) of the instruments `inst` only."""
    T = offsets.shape[0]
    off = np.zeros((T, len(inst) + 1), np.int32)
    parts, n = [], 0
    for t in range(T):
        for j, g in enumerate(inst):
            off[t, j] = n
            seg = items[offsets[t, g]:offsets[t, g + 1]]
            parts.append(seg)
            n += seg.size
        off[t, len(inst)] = n
    return off, np.concatenate(parts)
