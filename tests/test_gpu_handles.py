"""Every handle the library creates is counted while it lives and only then (mlb_live_handles, the count mlb_init's
one-device rule reads): one per kind, none left by a create refused after its first allocations, none left by a graph
that grew every buffer it has, and none left by a Python wrapper that was never closed."""
import gc

import numpy as np
import pytest

from madronalib_b200 import graph, workloads as wl
from madronalib_b200.graph import OP_ID
from tests.common import assert_same_bits, assert_state_equal, run_gpu

pytestmark = pytest.mark.gpu

V = 40
# one handle of each kind, and the kernel each graph must run
KINDS = {
    "graph_fused": lambda api: api.VoiceGraph(graph.graph_sine_lopass_gain(), V),
    "graph_fm3_fdn8": lambda api: api.VoiceGraph(graph.graph_fm3_fdn8(), V),
    "graph_interpreter": lambda api: api.VoiceGraph(graph.graph_sine_lopass_gain(), V, api.FLAG_FORCE_GENERIC),
    "voice_bank": lambda api: api.VoiceBank(48000.0, *wl.voice_bank_params(V)),
    "buses": lambda api: api.Buses(V, *wl.instrument_buses(V // 8, 8)),
    "upsampler": lambda api: api.ResamplerBank(api.ResamplerBank.UP, 2, V),
    "downsampler": lambda api: api.ResamplerBank(api.ResamplerBank.DOWN, 2, V),
    "fdtd": lambda api: api.FDTDBank(V),
    "mixbus": lambda api: api.MixBus(0, 1, 8 * 64),
}
KERNELS = {"graph_fused": "fused:MLB_OP_SINE", "graph_fm3_fdn8": "fused:fm3_fdn8", "graph_interpreter": "generic"}


@pytest.mark.parametrize("kind", list(KINDS))
def test_create_counts_one_handle_and_destroy_gives_it_back(gpu, kind):
    n0 = gpu.live_handles()
    h = KINDS[kind](gpu)
    assert gpu.live_handles() == n0 + 1
    if kind in KERNELS:
        assert h.kernel_name.startswith(KERNELS[kind]), h.kernel_name
    h.close()
    assert gpu.live_handles() == n0


def test_a_graph_refused_after_allocating_leaves_no_handle(gpu, port):
    """FDN<24> passes validation and gets its voice state, streams and events before the interpreter's planner finds
    28 live rows too many for shared memory; the graph created next runs as if nothing had happened."""
    n0 = gpu.live_handles()
    with pytest.raises(gpu.MlbError) as e:
        gpu.VoiceGraph(graph.graph_fdn(24)[0], 45)
    assert e.value.code == 5 and "live rows" in str(e.value)
    assert gpu.live_handles() == n0
    w, _, _, _ = wl.fdn_case(16, 45)
    T = 12
    inp = w.inputs(T)
    po, _, ps = port.run(w.spec, w.n_voices, T, inp, w.state, w.coef)
    go, _, gs, kname = run_gpu(gpu, w, T, inp, splits=(5, 7))
    assert_same_bits(go, po, "fdn16 after a refused fdn24 (%s)" % kname)
    assert_state_equal(gs, ps, "fdn16 after a refused fdn24")
    assert gpu.live_handles() == n0


def test_graphs_that_grew_every_buffer_give_their_handle_back(gpu):
    n0 = gpu.live_handles()
    # host staging with out and mix, then the asynchronous mix bus, then staging regrown by a larger T
    w = wl.config_a(96)
    g = gpu.VoiceGraph(w.spec, w.n_voices)
    g.set_coefs(w.coef)
    g.set_state(w.state)
    g.process_host(w.inputs(2), 2, want_out=True, want_mix=True)
    g.set_mix_async(True)
    g.process_host(w.inputs(7), 7, want_out=True, want_mix=True)
    assert gpu.live_handles() == n0 + 1
    g.close()
    assert gpu.live_handles() == n0
    # FDN8 delay memory, reallocated by set_coefs for two larger rings
    w = wl.config_4(V)
    g = gpu.VoiceGraph(w.spec, w.n_voices)
    g.set_state(w.state)
    lengths = w.spec.coef_slot(w.spec.ops.index(OP_ID["FDN8"])) + 24
    sizes = []
    for scale in (1, 4, 16):
        coef = w.coef.copy()
        coef[lengths:lengths + 8] *= np.float32(scale)
        g.set_coefs(coef)
        sizes.append(g.delay_bytes)
        g.process_host(w.inputs(3), 3, want_out=True, want_mix=True)
    assert sizes[0] < sizes[1] < sizes[2], sizes
    g.close()
    assert gpu.live_handles() == n0
    # functors with delay memory through the interpreter, channel planes regrown by a larger T
    w = wl.config_6(33)
    g = gpu.VoiceGraph(w.spec, w.n_voices)
    g.set_coefs(w.coef)
    g.set_state(w.state)
    assert g.kernel_name.startswith("generic") and g.delay_bytes > 0
    g.process_host(w.inputs(2), 2, want_out=True, want_mix=True)
    g.process_host(w.inputs(6), 6, want_out=True, want_mix=True)
    g.close()
    assert gpu.live_handles() == n0


@pytest.mark.parametrize("kind", [k for k in KINDS if k != "mixbus"])
def test_an_unclosed_wrapper_is_released_by_the_garbage_collector(gpu, kind):
    n0 = gpu.live_handles()
    h = KINDS[kind](gpu)
    assert gpu.live_handles() == n0 + 1
    del h
    gc.collect()
    assert gpu.live_handles() == n0
    h = KINDS[kind](gpu)
    h.close()
    h.close()
    assert gpu.live_handles() == n0
