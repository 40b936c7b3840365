"""mlb::tr::TracedSynth through a Synth::processVector override, on the GPU: tests/cpp/test_fx_synth runs the Synth
subclass of tests/cpp/fx_synth_body.h for G instruments from raw events and transport updates (K12 -> K7 -> K11 -> K13
-> voice graph -> assembly kernel -> instrument graph, one mlb_synth_process_instrument_host call per split), and its bus
rows equal G reference AudioContext + FxSynth objects (oracle/_ref/libmlfxsynth.so) bit for bit."""
import numpy as np
import pytest

from tests import fx_synth_cases as fc
from tests import restart_cases as rc
from tests import synth_cases as sc
from tests.common import assert_same_bits


def _ref():
    from oracle import fxsynth_bindings
    if not fxsynth_bindings.ref_available():
        pytest.skip("oracle/_ref/libmlfxsynth.so not built (no reference tree where build() ran)")
    return fxsynth_bindings


@pytest.mark.gpu
@pytest.mark.parametrize("case,G,T,splits", [("midi", 1, 40, (40,)), ("midi", 37, 48, (5, 17, 1, 25)),
                                             ("midi", 4096, 64, (64,)), ("mpe", 1, 24, (24,)),
                                             ("mpe", 37, 40, (13, 27)), ("mpe", 4096, 32, (11, 21))])
def test_fx_synth_equals_reference_synths(gpu, tmp_path, case, G, T, splits):
    ref = _ref()
    d = fc.dump(case)
    late, never = (G // 2, G - 1) if G > 2 else (None, None)
    off, ev, toff, tr = sc.performance(d, G, T, seed=G + T, late=late, never=never, density=0.3)
    got, _, out = fc.run(tmp_path, case, G, T, off, ev, toff, tr, splits)
    want, _ = ref.ref_synth(case, d["n_voices"], off, ev, toff, tr)
    assert_same_bits(got, want, f"traced {case} FxSynth, {G} instruments, calls of {splits} vectors")
    assert np.nanmax(np.abs(want)) > 0.1
    print(out.strip().split("\n")[0])


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["midi", "mpe"])
def test_launches_are_the_context_call_plus_one_per_chunk(gpu, tmp_path, monkeypatch, case):
    """One call forced into 4 time chunks (MLB_SYNTH_CHUNK_BLOCKS=9 over 30 vectors): the traced synth equals its
    banks wired by hand through VoiceGraph.process_instrument_host, bit for bit and launch for launch, and that call
    takes the launches of process_context_host on the same voice graph plus exactly one per chunk (the assembly kernel
    takes the bus sum's place; the instrument graph is one launch)."""
    monkeypatch.setenv("MLB_SYNTH_CHUNK_BLOCKS", "9")
    d = fc.dump(case)
    G, T = 21, 30
    off, ev, toff, tr = sc.performance(d, G, T, seed=4)
    got, launches, _ = fc.run(tmp_path, case, G, T, off, ev, toff, tr, (T,))
    b = fc.banks(gpu, d, G)
    try:
        n0 = gpu.kernel_launches()
        want = b["graph"].process_instrument_host(b["instrument"], b["routers"], b["bank"], b["buses"], off, ev,
                                                  controllers=b["controllers"], times=b["times"], time_offsets=toff,
                                                  transports=tr)
        inst = gpu.kernel_launches() - n0
        n0 = gpu.kernel_launches()
        b["graph"].process_context_host(b["routers"], b["bank"], off, ev, controllers=b["controllers"], times=b["times"],
                                        time_offsets=toff, transports=tr, buses=b["buses"])
        ctx = gpu.kernel_launches() - n0
    finally:
        fc.close(b)
    assert_same_bits(got, want, f"traced {case} FxSynth vs the hand-wired instrument call")
    assert launches == [inst] and inst == ctx + 4, (launches, inst, ctx)


@pytest.mark.gpu
def test_base_only_override_takes_todays_launches_and_bits(gpu, tmp_path):
    """BodySynth with an override that only calls the base runs exactly as BodySynth: same bus rows, same launches per
    call (mlb_synth_process_context_host, no instrument graph)."""
    d = sc.dump("midi")
    G, T = 37, 40
    off, ev, toff, tr = sc.performance(d, G, T, seed=9, density=0.3)
    want, want_l, out = fc.run(tmp_path, "body", G, T, off, ev, toff, tr, (13, 27))
    got, got_l, out2 = fc.run(tmp_path, "bodybase", G, T, off, ev, toff, tr, (13, 27))
    assert_same_bits(got, want, "base-only override vs no override")
    assert got_l == want_l and "instrument graph on (none)" in out2, (got_l, want_l, out2)
    from oracle import tsynth_bindings
    if tsynth_bindings.ref_available():
        ref, _ = tsynth_bindings.ref_synth("midi", d["n_voices"], off, ev, toff, tr)
        assert_same_bits(got, ref, "base-only override vs reference AudioContext + BodySynth")


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["midi", "mpe"])
def test_restart_at_vector_37_equals_fresh_reference_synths(gpu, tmp_path, case):
    """Instruments 3, 11 and 20 restarted after vector 37 equal fresh reference objects fed only what follows; the
    others are unchanged bit for bit.  The restart is six launches: routers, Voice rows, controllers, beat phase, voice
    graph, instrument graph."""
    ref = _ref()
    d = fc.dump(case)
    G, T = 23, 60
    off, ev, toff, tr = sc.performance(d, G, T, seed=37, density=0.3)
    restart = [3, 11, 20]
    got, _, out = fc.run(tmp_path, case, G, T, off, ev, toff, tr, (37, 23), restart=restart)
    want = rc.expected(lambda o, e, to, r: ref.ref_synth(case, d["n_voices"], o, e, to, r)[0], off, ev, toff, tr,
                       {37: restart})
    assert_same_bits(got, want, f"traced {case} FxSynth restarted at vector 37")
    full, _ = ref.ref_synth(case, d["n_voices"], off, ev, toff, tr)
    assert not np.array_equal(full[37:, :, restart].view(np.uint32), want[37:, :, restart].view(np.uint32))
    assert int(out.split("restart launches: ")[1].split()[0]) == 6


@pytest.mark.gpu
def test_instrument_call_argument_errors_write_nothing(gpu, tmp_path):
    """Each refused call (an instrument graph over other lanes, one reading a plane past the beat phase, buses of
    another instrument count) raises before anything is copied: the bus rows keep their sentinel, and the next good
    call equals the traced synth's first call."""
    d = fc.dump("midi")
    G, T = 9, 12
    off, ev, toff, tr = sc.performance(d, G, T, seed=5)
    want, _, _ = fc.run(tmp_path, "midi", G, T, off, ev, toff, tr, (T,))
    b = fc.banks(gpu, d, G)
    ispec = fc.instrument_graph(d)[0]
    wide = gpu.VoiceGraph(ispec, G + 1)
    far = fc.instrument_graph(d)[0]
    far.iargs = [d["instrument"]["planes"] if a == 0 and op == 0 else a for op, a in zip(far.ops, far.iargs)]
    far_g = gpu.VoiceGraph(far, G)
    lay = sc.layout(d, G)
    first = (lay["first_voice"] + d["mpe"]).astype(np.int32)
    other = gpu.Buses(b["graph"].n_voices, first[:G - 1], np.full(G - 1, d["n_voices"], np.int32))
    kw = dict(controllers=b["controllers"], times=b["times"], time_offsets=toff, transports=tr)
    try:
        for gi, buses, msg in ((wide, b["buses"], "instrument graph has"), (far_g, b["buses"], "INPUT plane"),
                               (b["instrument"], other, "buses have")):
            sentinel = np.full((T, gi.spec.n_out, buses.n_buses, 64), np.nan, np.float32)
            with pytest.raises(gpu.MlbError, match=msg):
                b["graph"].process_instrument_host(gi, b["routers"], b["bank"], buses, off, ev, bus=sentinel, **kw)
            assert np.isnan(sentinel).all()
        got = b["graph"].process_instrument_host(b["instrument"], b["routers"], b["bank"], b["buses"], off, ev, **kw)
    finally:
        fc.close(b)
        for x in (wide, far_g, other):
            x.close()
    assert_same_bits(got, want, "the first good call after refused ones vs the traced synth")
