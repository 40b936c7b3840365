"""The host entry points of a graph: kernel launches per call on every path (one launch, voice slices, time
chunks), a pipeline that fails part-way, and the input plane count a graph keeps across contract E."""
import ctypes
import os

import numpy as np
import pytest

from madronalib_b200 import workloads as wl
from tests.common import assert_same_bits, assert_state_equal

pytestmark = pytest.mark.gpu

NTHREADS = max(1, len(os.sched_getaffinity(0)))


def _launches(gpu, call):
    n0 = gpu.kernel_launches()
    call()
    return gpu.kernel_launches() - n0


def _n_inputs(gpu, g):
    lay = gpu.Layout()
    gpu._check(gpu.lib().mlb_graph_layout_of(g._h, ctypes.byref(lay)))
    return lay.n_inputs


def test_process_host_launches(gpu, monkeypatch):
    """One launch, plus the mix reduction; over voice slices, one launch per slice plus one reduction."""
    monkeypatch.setenv("MLB_HOST_SLICES", "5")
    monkeypatch.setenv("MLB_HOST_SLICE_MIN_MB", "1")
    for V, T, slices in ((300, 4, 1), (4207, 9, 5)):
        w = wl.config_a(V)
        inp = w.inputs(T)
        g = gpu.VoiceGraph(w.spec, V)
        try:
            g.set_coefs(w.coef)
            g.set_state(w.state)
            assert _launches(gpu, lambda: g.process_host(inp, T, want_out=True, want_mix=False)) == slices
            assert g.last_host_slices == slices
            assert _launches(gpu, lambda: g.process_host(inp, T, want_out=True, want_mix=True)) == slices + 1
            assert g.last_host_slices == slices
        finally:
            g.close()


@pytest.mark.parametrize("case,flags,launches", [("fused", 0, 2), ("fdn", 0, 3), ("generic", 2, 2)])
def test_process_device_launches_with_mix(gpu, case, flags, launches):
    """The graph's kernel and the mix reduction; the FDN kernel adds the partials of its two output planes."""
    import torch
    V, T = 96, 3
    w = wl.config_4(V) if case == "fdn" else wl.config_a(V)
    dev = torch.device("cuda", 0)
    g = gpu.VoiceGraph(w.spec, V, flags)
    try:
        assert g.kernel_name.startswith("generic" if case == "generic" else "fused:"), g.kernel_name
        g.set_coefs(w.coef)
        g.set_state(w.state)
        d_in = torch.from_numpy(w.inputs(T)).to(dev)
        d_out = torch.empty((T, w.spec.n_out, V, 64), dtype=torch.float32, device=dev)
        d_mix = torch.empty((T, w.spec.n_out, 64), dtype=torch.float32, device=dev)
        s = torch.cuda.current_stream().cuda_stream
        assert _launches(gpu, lambda: g.process_device(d_in, d_out, d_mix, T, s)) == launches
        torch.cuda.synchronize()
    finally:
        g.close()


def test_contract_e_launches_per_chunk(gpu, monkeypatch):
    """Per time chunk: the bank, the graph, and the mix reduction or the bus sum."""
    monkeypatch.setenv("MLB_SYNTH_CHUNK_BLOCKS", "3")
    V, T = 320, 9
    w = wl.config_a(V)
    ev = wl.synth_events(V, T, seed=31, density=0.3, ctl=0.2)
    vb = gpu.VoiceBank(48000.0, *wl.synth_bank_params(V))
    g = gpu.VoiceGraph(w.spec, V)
    b = gpu.Buses(V, *wl.instrument_buses(V // 16, 16))
    try:
        g.set_coefs(w.coef)
        g.set_state(w.state)
        assert _launches(gpu, lambda: g.process_events_host(vb, ev, want_out=True)) == 3 * 2
        assert g.last_host_slices == 3
        assert _launches(gpu, lambda: g.process_events_host(vb, ev, want_out=True, want_mix=True)) == 3 * 3
        assert _launches(gpu, lambda: g.process_events_host(vb, ev, want_out=False, want_mix=True)) == 3 * 3
        assert _launches(gpu, lambda: g.process_events_buses_host(vb, b, ev)) == 3 * 3
        assert g.last_host_slices == 3
    finally:
        for h in (b, g, vb):
            h.close()


def test_contract_e_failing_part_way_leaves_graph_and_bank_as_they_were(gpu, port, monkeypatch):
    """The bank refuses its launch after the first chunk's records went up: the call fails naming the cause, the
    graph keeps its input plane count, and the same call afterwards is bit-exact from the initial state."""
    from oracle import bindings
    monkeypatch.setenv("MLB_SYNTH_CHUNK_BLOCKS", "3")
    V, T = 200, 9
    w = wl.config_a(V)
    ev = wl.synth_events(V, T, seed=32, density=0.3, ctl=0.2)
    prm = wl.synth_bank_params(V)
    rows, _ = bindings.port_voice_bank().run(48000.0, *prm, ev, nthreads=NTHREADS)
    want, want_mix, want_st = port.run(w.spec, V, T, np.ascontiguousarray(rows[:, :1]), w.state, w.coef,
                                       want_mix=True, mix_mode=1, nthreads=NTHREADS)
    vb = gpu.VoiceBank(48000.0, *prm)
    g = gpu.VoiceGraph(w.spec, V)
    try:
        g.set_coefs(w.coef)
        g.set_state(w.state)
        monkeypatch.setenv("MLB_VOICE_WARPS", "8")
        with pytest.raises(gpu.MlbError, match="MLB_VOICE_WARPS"):
            g.process_events_host(vb, ev, want_out=True, want_mix=True)
        assert _n_inputs(gpu, g) == 1
        monkeypatch.delenv("MLB_VOICE_WARPS")
        o, m = g.process_events_host(vb, ev, want_out=True, want_mix=True)
        st = g.get_state()
    finally:
        g.close()
        vb.close()
    assert_same_bits(o, want, "rows after a failed call")
    assert_same_bits(m, want_mix, "mix after a failed call")
    assert_state_equal(st, want_st, "state after a failed call")


def test_contract_e_keeps_the_graph_input_planes(gpu, port):
    """Contract E reads the bank's 8 Voice rows without changing the plane count the graph was given: a later
    process_device call still reads [T][3][V][64] (plane 0 the frequencies, planes 1 and 2 junk)."""
    import torch
    V, T, T2 = 130, 5, 4
    w = wl.config_a(V)
    ev = wl.synth_events(V, T, seed=33, density=0.3, ctl=0.2)
    vb = gpu.VoiceBank(48000.0, *wl.synth_bank_params(V))
    g = gpu.VoiceGraph(w.spec, V)
    try:
        g.set_coefs(w.coef)
        g.set_state(w.state)
        g.set_input_planes(3)
        g.process_events_host(vb, ev, want_out=True)
        assert _n_inputs(gpu, g) == 3
        st = g.get_state()
        inp = w.inputs(T2)
        junk = np.random.default_rng(7).standard_normal((T2, 2, V, 64)).astype(np.float32)
        dev = torch.device("cuda", 0)
        d_in = torch.from_numpy(np.ascontiguousarray(np.concatenate([inp, junk], axis=1))).to(dev)
        d_out = torch.empty((T2, 1, V, 64), dtype=torch.float32, device=dev)
        g.process_device(d_in, d_out, None, T2, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        got, got_st = d_out.cpu().numpy(), g.get_state()
    finally:
        g.close()
        vb.close()
    want, _, want_st = port.run(w.spec, V, T2, inp, st, w.coef)
    assert_same_bits(got, want, "plane 0 of three")
    assert_state_equal(got_st, want_st)
