"""Kernel launches per time chunk of the contract-E entry points that feed the graph more than the Voice rows: controller
planes from the host, and raw events routed on the device with controller planes, the beat phase and bus rows.  The
record and bus entry points are counted in test_gpu_host_paths.py."""
import pytest

from madronalib_b200 import workloads as wl

pytestmark = pytest.mark.gpu

# launches per time chunk of each stage
ROUTER, VOICE, K11, K13, GRAPH, BUS, MIX = 3, 1, 1, 1, 1, 1, 1


def _launches(gpu, call):
    n0 = gpu.kernel_launches()
    call()
    return gpu.kernel_launches() - n0


def test_contract_e_launches_per_chunk_controllers_routed_context(gpu, monkeypatch):
    """Three chunks of 3 blocks: each chunk runs the router (raw events), the bank, K11 and K13 if given, the graph,
    and the mix reduction or the bus sum."""
    monkeypatch.setenv("MLB_SYNTH_CHUNK_BLOCKS", "3")
    G, P, T = 20, 16, 9
    lay = wl.midi_layout(G, P)
    V = lay["n_voices"]
    w = wl.config_a(V)
    ev = wl.synth_events(V, T, seed=31, density=0.3, ctl=0.2)
    coff, ch = wl.controller_changes(G, T, density=0.5, seed=32)
    offsets, raw = wl.midi_performance(G, T, P, density=0.5, seed=33)
    toff, tr = wl.transport_updates(G, T, seed=34)
    vb = gpu.VoiceBank(48000.0, *wl.synth_bank_params(V), flags=gpu.VoiceBank.MIDI)
    g = gpu.VoiceGraph(w.spec, V)
    b = gpu.Buses(V, *wl.instrument_buses(G, P))
    cb = gpu.ControllerBank(G, [1, 7], 48000.0)
    pt = gpu.ProcessTimeBank(G, 48000.0)
    r = gpu.RouterBank(lay["polyphony"], lay["first_voice"], V)
    try:
        g.set_coefs(w.coef)
        g.set_state(w.state)
        cb.set_voice_map(lay["voice_instrument"])
        pt.set_voice_map(lay["voice_instrument"])
        assert _launches(gpu, lambda: g.process_events_controllers_host(vb, cb, ev, coff, ch)) == \
            3 * (VOICE + K11 + GRAPH)
        assert _launches(gpu, lambda: g.process_events_controllers_host(vb, cb, ev, coff, ch, want_mix=True)) == \
            3 * (VOICE + K11 + GRAPH + MIX)
        assert g.last_host_slices == 3
        assert _launches(gpu, lambda: g.process_routed_host(r, vb, offsets, raw)) == 3 * (ROUTER + VOICE + GRAPH)
        assert _launches(gpu, lambda: g.process_routed_host(r, vb, offsets, raw, controllers=cb, want_out=False,
                                                            want_mix=True)) == 3 * (ROUTER + VOICE + K11 + GRAPH + MIX)
        assert _launches(gpu, lambda: g.process_routed_host(r, vb, offsets, raw, buses=b)) == \
            3 * (ROUTER + VOICE + GRAPH + BUS)
        assert g.last_host_slices == 3
        ctx = dict(times=pt, time_offsets=toff, transports=tr)
        assert _launches(gpu, lambda: g.process_context_host(r, vb, offsets, raw, **ctx)) == \
            3 * (ROUTER + VOICE + K13 + GRAPH)
        assert _launches(gpu, lambda: g.process_context_host(r, vb, offsets, raw, controllers=cb, want_mix=True,
                                                             **ctx)) == 3 * (ROUTER + VOICE + K11 + K13 + GRAPH + MIX)
        assert _launches(gpu, lambda: g.process_context_host(r, vb, offsets, raw, controllers=cb, buses=b, **ctx)) \
            == 3 * (ROUTER + VOICE + K11 + K13 + GRAPH + BUS)
        assert g.last_host_slices == 3
    finally:
        for h in (r, pt, cb, b, g, vb):
            h.close()
