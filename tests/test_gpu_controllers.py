"""K11 on the GPU: the smoothed MIDI controllers (mlb_controllers_*), bit-exact against the plain-C port
(oracle/port/mlport_ctrl.c, itself pinned to the reference's EventsToSignals by tests/test_controllers.py), NaN == NaN:
instrument and voice layouts, split calls, state round trips, special values, one launch per call and CUDA-graph
replay, the full 4 096 x 129 x 64 size, and every argument error."""
import numpy as np
import pytest

from madronalib_b200 import workloads as wl
from tests.common import assert_same_bits, assert_state_equal
from tests.ctrl_cases import ALL_CONTROLLERS

pytestmark = pytest.mark.gpu

SPECIAL = np.array([-0.0, np.inf, -np.inf, np.nan, 1e-40, -1e-42, 1.4e-45, 3e38, 0.0], np.float32)


def port_ctrl(G, ctrl, offsets, changes, sr=48000.0, state=None):
    from oracle.ctrl_bindings import port_controllers
    return port_controllers(G, ctrl, offsets, changes, sr, state)


def special_changes(G, T, seed, density=0.3, ctrl=(0, 1, 7, 64, 74, 127, 128)):
    """Fader moves with duplicates in a block over (up to 8 of) the requested controllers `ctrl`, plus NaN / +-inf /
    -0 / subnormal values, controller numbers the bank does not request and numbers above 128."""
    unrequested = [n for n in range(129) if n not in ctrl][:2]
    pool = list(ctrl)[:8] + unrequested + [129, 999]
    offsets, ch = wl.controller_changes(G, T, density=density, seed=seed, pool=pool)
    rng = np.random.default_rng(seed)
    k = rng.random(ch.size) < 0.15
    ch["value"][k] = SPECIAL[rng.integers(0, len(SPECIAL), int(k.sum()))]
    return offsets, ch


def controller_list(C, seed):
    rng = np.random.default_rng(seed)
    return rng.permutation(129)[:C].tolist()  # any order


@pytest.mark.parametrize("G", [1, 33, 4096])
@pytest.mark.parametrize("C", [1, 9, 32, 33, 129])
def test_device_equals_port_split_calls(gpu, G, C):
    T = 24 if G < 4096 else 12
    ctrl = controller_list(C, G * 131 + C)
    offsets, ch = special_changes(G, T, seed=G + C, density=0.6 if G < 4096 else 0.2, ctrl=ctrl)
    want, words, rows = port_ctrl(G, ctrl, offsets, ch)
    bank = gpu.ControllerBank(G, ctrl, 48000.0)
    try:
        t1 = T // 3
        a = bank.process_host(offsets[:t1], ch)
        b = bank.process_host(offsets[t1:], ch)
        got_w, got_r = bank.get_state()
    finally:
        bank.close()
    assert_same_bits(np.concatenate([a, b]), want, "G %d, C %d" % (G, C))
    assert_state_equal(got_w, words, "state words")
    assert_same_bits(got_r, rows, "rows")
    assert (want != 0).any() and (np.isnan(want).any() or G < 4096)


@pytest.mark.parametrize("sr", [44100.0, 96000.0])
def test_set_state_mid_stream_and_interrupted_glides(gpu, sr):
    """From a random mid-stream state (moving, landing and idle glides, special targets) set through set_state;
    new targets arrive while glides move."""
    G, T, ctrl = 70, 40, [74, 1, 128, 7, 0]
    offsets, ch = special_changes(G, T, seed=3, density=0.5, ctrl=ctrl)
    _, w0, r0 = port_ctrl(G, ctrl, offsets[:9], ch, sr)
    rem = w0[2].view(np.int32)
    assert (rem > 0).any() and (rem < 0).any(), "the state holds moving and idle glides"
    want, words, rows = port_ctrl(G, ctrl, offsets[9:], ch, sr, state=(w0, r0))
    bank = gpu.ControllerBank(G, ctrl, sr)
    try:
        bank.set_state(w0, r0)
        w_back, r_back = bank.get_state()
        assert_state_equal(w_back, w0, "state round trip")
        assert_same_bits(r_back, r0, "rows round trip")
        got = bank.process_host(offsets[9:], ch)
        got_w, got_r = bank.get_state()
        bank.clear()
        cw, cr = bank.get_state()
    finally:
        bank.close()
    assert_same_bits(got, want, "from set_state")
    assert_state_equal(got_w, words, "state words")
    assert_same_bits(got_r, rows, "rows")
    from oracle.ctrl_bindings import initial_state
    iw, ir = initial_state(G, len(ctrl))
    assert (cw == iw).all() and (cr.view(np.uint32) == 0).all(), "clear"


def test_voice_planes_with_gaps(gpu):
    G, T, ctrl = 37, 10, [128, 11, 1]
    V = 200
    rng = np.random.default_rng(7)
    vmap = rng.integers(-1, G, V).astype(np.int32)
    vmap[:5] = -1
    vmap[5:21] = 3  # one instrument with 16 voices
    offsets, ch = special_changes(G, T, seed=8, density=0.5, ctrl=ctrl)
    inst, _, _ = port_ctrl(G, ctrl, offsets, ch)
    P, plane0 = len(ctrl) + 4, 3
    sentinel = np.float32(12345.0)
    bank = gpu.ControllerBank(G, ctrl, 48000.0)
    try:
        bank.set_voice_map(vmap)
        out = np.full((T, P, V, 64), sentinel, np.float32)
        bank.process_host(offsets, ch, out=out, plane0=plane0, n_planes=P)
        bank.set_voice_map(None)
        bank.clear()
        back = bank.process_host(offsets, ch)
    finally:
        bank.close()
    want = np.where((vmap >= 0)[None, None, :, None], inst[:, :, np.maximum(vmap, 0)], np.float32(0))
    assert_same_bits(out[:, plane0:plane0 + len(ctrl)], want, "voice planes")
    assert not np.signbit(out[:, plane0:plane0 + len(ctrl), vmap < 0]).any(), "a voice of no instrument gets +0"
    assert (out[:, :plane0] == sentinel).all() and (out[:, plane0 + len(ctrl):] == sentinel).all(), "other planes kept"
    assert_same_bits(back, inst, "instrument rows again")


def test_one_launch_per_call_and_graph_replay(gpu):
    import torch
    G, T, ctrl = 100, 8, [1, 7, 74, 128]
    offsets, ch = special_changes(G, T, seed=11, density=0.5, ctrl=ctrl)
    want, _, _ = port_ctrl(G, ctrl, offsets, ch)
    base = gpu.live_handles()
    bank = gpu.ControllerBank(G, ctrl, 48000.0)
    assert gpu.live_handles() == base + 1
    try:
        d_off = torch.from_numpy(offsets).cuda()
        d_ch = torch.from_numpy(ch.view(np.int64)).cuda()
        y = torch.empty((T, len(ctrl), G, 64), device="cuda")
        s = torch.cuda.current_stream().cuda_stream
        w0, r0 = bank.get_state()
        n0 = gpu.kernel_launches()
        bank.process_device(d_off, d_ch, y, T, stream=s)
        assert gpu.kernel_launches() - n0 == 1
        torch.cuda.synchronize()
        direct = y.cpu().numpy().copy()
        bank.set_state(w0, r0)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            bank.process_device(d_off, d_ch, y, T, stream=torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        bank.set_state(w0, r0)
        y.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert_same_bits(y.cpu().numpy(), direct, "graph replay vs direct call")
        del g
    finally:
        bank.close()
    assert gpu.live_handles() == base
    assert_same_bits(direct, want, "direct call vs port")


def _sub_csr(offsets, changes, inst):
    """The change list of the instruments `inst` only."""
    T = offsets.shape[0]
    off = np.zeros((T, len(inst) + 1), np.int32)
    parts, n = [], 0
    for t in range(T):
        for j, g in enumerate(inst):
            off[t, j] = n
            seg = changes[offsets[t, g]:offsets[t, g + 1]]
            parts.append(seg)
            n += seg.size
        off[t, len(inst)] = n
    return off, np.concatenate(parts)


def test_full_size(gpu):
    """4 096 instruments x 129 controllers x 64 vectors in one call; sampled instruments against the port."""
    import torch
    G, T, C = 4096, 64, 129
    offsets, ch = special_changes(G, T, seed=21, density=0.05)
    bank = gpu.ControllerBank(G, ALL_CONTROLLERS, 48000.0)
    try:
        d_off = torch.from_numpy(offsets).cuda()
        d_ch = torch.from_numpy(ch.view(np.int64)).cuda()
        y = torch.empty((T, C, G, 64), device="cuda")
        bank.process_device(d_off, d_ch, y, T, stream=torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        inst = np.array([0, 1, 31, 32, 1000, 2047, 4064, 4095])
        got = y[:, :, torch.from_numpy(inst).cuda()].cpu().numpy()
        del y
    finally:
        bank.close()
    off, sub = _sub_csr(offsets, ch, inst)
    want, _, _ = port_ctrl(len(inst), ALL_CONTROLLERS, off, sub)
    assert_same_bits(got, want, "full size, sampled instruments")


def test_argument_errors(gpu):
    import torch
    G, ctrl = 8, [1, 128]
    bank = gpu.ControllerBank(G, ctrl, 48000.0)
    offsets, ch = wl.controller_changes(G, 4, density=0.5, seed=2)
    try:
        bad = offsets.copy()
        bad[2, 3] = bad[2, 4] + 1
        with pytest.raises(gpu.MlbError, match="block 2, instrument 3"):
            bank.process_host(bad, ch)
        bad = offsets.copy()
        bad[3, G] = ch.size + 1
        with pytest.raises(gpu.MlbError, match="block 3, instrument 7"):
            bank.process_host(bad, ch)
        with pytest.raises(gpu.MlbError, match="output planes"):
            bank.process_host(offsets, ch, plane0=1, n_planes=2)
        with pytest.raises(gpu.MlbError, match="voice 2: instrument 8"):
            bank.set_voice_map(np.array([0, -1, 8], np.int32))
        with pytest.raises(gpu.MlbError, match="voice 0: instrument -2"):
            bank.set_voice_map(np.array([-2], np.int32))
        with pytest.raises(ValueError):
            bank.set_state(np.zeros((4, 2, G + 1), np.uint32), np.zeros((2, G, 64), np.float32))
        y = torch.zeros((1, 2, G, 64), device="cuda")
        d_off = torch.from_numpy(offsets[:1]).cuda()
        s = torch.cuda.current_stream().cuda_stream
        for args in ((None, None, y, 1), (d_off, None, None, 1), (d_off, None, y, 0)):
            with pytest.raises(gpu.MlbError) as e:
                bank.process_device(*args, stream=s)
            assert e.value.code == 1
        with pytest.raises(gpu.MlbError, match="output planes"):
            bank.process_device(d_off, None, y, 1, plane0=-1, stream=s)
    finally:
        bank.close()


# ---- contract E with controller planes: records + change lists in, graph rows / mix out ----

def _n_inputs(api, g):
    from madronalib_b200.graph import Layout
    import ctypes
    lay = Layout()
    api._check(api.lib().mlb_graph_layout_of(g._h, ctypes.byref(lay)))
    return int(lay.n_inputs)


def _expect_e(port, port_bank, w, ev, prm, flags, ctrl, vmap, offsets, changes, protocol):
    """port(bank) + port(controllers) -> port(graph): the graph's input is [T][8 + C][V][64]."""
    T, V = ev.shape
    rows, _ = port_bank.run(48000.0, *prm, ev, flags=flags)
    inst, _, _ = port_ctrl(len(offsets[0]) - 1, ctrl, offsets, changes)
    cplanes = np.where((vmap >= 0)[None, None, :, None], inst[:, :, np.maximum(vmap, 0)], np.float32(0))
    inp = np.ascontiguousarray(np.concatenate([rows, cplanes], axis=1)[:, :w.spec.n_in])  # the planes it reads
    out, mix, st = port.run(w.spec, V, T, inp, w.state, w.coef, want_mix=True)
    return out, mix, st


@pytest.fixture(scope="module")
def port_bank():
    from oracle import bindings
    return bindings.port_voice_bank()


@pytest.mark.parametrize("chunk", [0, 5])
def test_events_with_controllers_fused_chain(gpu, port, port_bank, monkeypatch, chunk):
    """Config A (reads kPitch) behind 8 + 4 input planes, MIDI: the graph's layout is untouched, the Voice rows land
    where they did."""
    if chunk:
        monkeypatch.setenv("MLB_SYNTH_CHUNK_BLOCKS", str(chunk))
    else:
        monkeypatch.delenv("MLB_SYNTH_CHUNK_BLOCKS", raising=False)
    G, poly = 12, 16
    V, T, ctrl = G * poly, 14, [1, 7, 11, 128]
    vmap = np.repeat(np.arange(G, dtype=np.int32), poly)
    w = wl.config_a(V)
    ev = wl.synth_events(V, T, seed=31, density=0.3, ctl=0.2)
    prm = wl.synth_bank_params(V)
    offsets, ch = special_changes(G, T, seed=32, density=0.4, ctrl=ctrl)
    want, want_mix, want_st = _expect_e(port, port_bank, w, ev, prm, wl.VOICES_MIDI, ctrl, vmap, offsets, ch, 0)
    vb = gpu.VoiceBank(48000.0, *prm, flags=wl.VOICES_MIDI)
    cb = gpu.ControllerBank(G, ctrl, 48000.0, protocol=0)
    g = gpu.VoiceGraph(w.spec, V)
    try:
        assert g.kernel_name.startswith("fused:")
        n_in = _n_inputs(gpu, g)
        cb.set_voice_map(vmap)
        g.set_coefs(w.coef)
        g.set_state(w.state)
        out, mix = g.process_events_controllers_host(vb, cb, ev, offsets, ch, want_mix=True)
        st = g.get_state()
        assert _n_inputs(gpu, g) == n_in, "the graph's plane count is unchanged"
        if chunk:
            assert g.last_host_slices == (T + chunk - 1) // chunk
    finally:
        for h in (g, vb, cb):
            h.close()
    assert_same_bits(out, want, "events + controllers -> chain A")
    assert_state_equal(st, want_st, "state")
    assert np.abs(want).max() > 0.01
    np.testing.assert_allclose(mix, want_mix, rtol=1e-4, atol=1e-4)  # the mix bus keeps its own order (DESIGN.md 5)


def test_events_with_controllers_interpreted_graph(gpu, port, port_bank, monkeypatch):
    """SineGen(pitch x 2^-2) x gate x (mod wheel + expression), MPE, a voice map with main voices outside (-1);
    split into two calls: bank, controller and graph state carry across."""
    from madronalib_b200.graph import GraphSpec, SINE_ZERO_PHASE
    monkeypatch.setenv("MLB_SYNTH_CHUNK_BLOCKS", "4")
    G, poly = 7, 5
    V, T, ctrl = G * (poly + 1), 18, [128, 1, 11]
    vmap = np.repeat(np.arange(G, dtype=np.int32), poly + 1)
    vmap[::poly + 1] = -1
    gs = GraphSpec()
    pitch, gate, mod, expr = gs.input(0), gs.input(1), gs.input(9), gs.input(10)
    k = gs.param()
    sine = gs.node("MULTIPLY", gs.node("SINE", gs.node("MULTIPLY", pitch, k)), gate)
    gs.output(gs.node("MULTIPLY", sine, gs.node("ADD", mod, expr)))
    coef, state = gs.new_coefs(V), gs.new_state(V)
    coef[0] = np.float32(0.25)
    state[0] = SINE_ZERO_PHASE
    w = wl.Workload("pitch_sine_gate_ctrl", gs, V, coef, state)
    ev = wl.synth_events(V, T, seed=33, density=0.3, ctl=0.2)
    prm = wl.synth_bank_params(V)
    offsets, ch = wl.controller_changes(G, T, density=0.5, seed=34, pool=(1, 11, 128, 74))
    want, _, want_st = _expect_e(port, port_bank, w, ev, prm, 0, ctrl, vmap, offsets, ch, 1)
    vb = gpu.VoiceBank(48000.0, *prm)
    cb = gpu.ControllerBank(G, ctrl, 48000.0, protocol=1)
    g = gpu.VoiceGraph(gs, V)
    try:
        assert not g.kernel_name.startswith("fused:")
        cb.set_voice_map(vmap)
        g.set_coefs(coef)
        g.set_state(state)
        a, _ = g.process_events_controllers_host(vb, cb, np.ascontiguousarray(ev[:7]), offsets[:7], ch)
        b, _ = g.process_events_controllers_host(vb, cb, np.ascontiguousarray(ev[7:]), offsets[7:], ch)
        st = g.get_state()
    finally:
        for h in (g, vb, cb):
            h.close()
    assert_same_bits(np.concatenate([a, b]), want, "events + controllers -> interpreted graph")
    assert_state_equal(st, want_st, "state")
    assert np.abs(want).max() > 0.01


def test_events_with_controllers_argument_errors(gpu):
    from madronalib_b200.graph import GraphSpec
    G, V, T = 4, 64, 3
    prm = wl.synth_bank_params(V)
    vb = gpu.VoiceBank(48000.0, *prm, flags=wl.VOICES_MIDI)
    cb = gpu.ControllerBank(G, [1, 7], 48000.0)
    cb_mpe = gpu.ControllerBank(G, [1, 7], 48000.0, protocol=1)
    gs = GraphSpec()
    gs.output(gs.node("MULTIPLY", gs.input(0), gs.input(9)))
    g = gpu.VoiceGraph(gs, V)
    far = GraphSpec()
    far.output(far.node("SINE", far.input(10)))
    g_far = gpu.VoiceGraph(far, V)
    ev = wl.synth_events(V, T)
    offsets, ch = wl.controller_changes(G, T, density=0.5, seed=1)
    try:
        with pytest.raises(gpu.MlbError, match="voice map has 0 voices"):
            g.process_events_controllers_host(vb, cb, ev, offsets, ch)
        vm = np.repeat(np.arange(G, dtype=np.int32), V // G)
        cb.set_voice_map(vm)
        cb_mpe.set_voice_map(vm)
        with pytest.raises(gpu.MlbError, match="protocol MPE"):
            g.process_events_controllers_host(vb, cb_mpe, ev, offsets, ch)
        with pytest.raises(gpu.MlbError, match="INPUT plane 10 is not a Voice row or controller plane \\(0..9\\)"):
            g_far.process_events_controllers_host(vb, cb, ev, offsets, ch)
        bad = offsets.copy()
        bad[1, 2] = -1
        with pytest.raises(gpu.MlbError, match="block 1, instrument 1"):
            g.process_events_controllers_host(vb, cb, ev, bad, ch)
        out, _ = g.process_events_controllers_host(vb, cb, ev, offsets, ch)
        assert out.shape == (T, 1, V, 64)
    finally:
        for h in (g, g_far, vb, cb, cb_mpe):
            h.close()
