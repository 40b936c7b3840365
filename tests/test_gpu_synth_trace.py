"""mlb::tr::TracedSynth on the GPU: tests/cpp/test_synth_trace runs the Synth subclass of tests/cpp/synth_body.h for G
instruments from raw events and transport updates (K12 -> K7 -> K11 -> K13 -> graph -> bus sum, one
mlb_synth_process_context_host call per split), and its bus rows equal G reference AudioContext + Synth objects
(oracle/_ref/libmltsynth.so) bit for bit, and the same graph wired by hand through VoiceGraph.process_context_host."""
import subprocess

import numpy as np
import pytest

from tests import synth_cases as sc
from tests.common import assert_same_bits


def _run(tmp_path, case, G, T, off, ev, toff, tr, splits):
    sc.build_exe()
    for name, a in (("offsets", off), ("events", ev), ("toff", toff), ("tr", tr)):
        np.ascontiguousarray(a).tofile(str(tmp_path / (name + ".bin")))
    r = subprocess.run([sc.EXE, "run", case, str(G), str(T), str(tmp_path), ",".join(map(str, splits))],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    launches = [int(n) for n in r.stdout.split("launches per call: ")[1].split()[0].split(",")]
    return np.fromfile(str(tmp_path / "bus.bin"), np.float32).reshape(T, 2, G, 64), launches


@pytest.mark.gpu
@pytest.mark.parametrize("case,G,T,splits", [("midi", 1, 40, (40,)), ("midi", 37, 48, (5, 17, 1, 25)),
                                             ("midi", 4096, 64, (64,)), ("mpe", 33, 40, (13, 27)),
                                             ("unison", 37, 40, (7, 33)), ("modcc", 37, 24, (24,))])
def test_traced_synth_equals_reference_synths(gpu, tmp_path, case, G, T, splits):
    from oracle import tsynth_bindings
    if not tsynth_bindings.ref_available():
        pytest.skip("oracle/_ref/libmltsynth.so not built (no reference tree where build() ran)")
    d = sc.dump(case)
    late, never = (G // 2, G - 1) if G > 2 else (None, None)
    off, ev, toff, tr = sc.performance(d, G, T, seed=G + T, late=late, never=never, density=0.3)
    got, _ = _run(tmp_path, case, G, T, off, ev, toff, tr, splits)
    want, _ = tsynth_bindings.ref_synth(case, d["n_voices"], off, ev, toff, tr)
    assert_same_bits(got, want, f"traced {case} synth, {G} instruments, calls of {splits} vectors")
    assert np.abs(want).max() > 0.1


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["midi", "mpe"])
def test_traced_synth_equals_hand_wired_context_call(gpu, tmp_path, case):
    """The traced bank equals its graph wired by hand: RouterBank, VoiceBank, ControllerBank, ProcessTimeBank and Buses
    built from the dump's settings, through VoiceGraph.process_context_host -- the same bus rows from the same number
    of kernel launches (TracedSynth::process is that one call)."""
    d = sc.dump(case)
    G, T = 21, 30
    off, ev, toff, tr = sc.performance(d, G, T, seed=4)
    got, launches = _run(tmp_path, case, G, T, off, ev, toff, tr, (T,))
    lay = sc.layout(d, G)
    V, mpe = lay["n_voices"], bool(d["mpe"])
    spec, coef, state = sc.graph(d, G)
    pb = np.full(V, d["pitch_bend"], np.float32)
    if mpe:
        pb[lay["main_voice"] >= 0] = np.float32(d["mpe_pitch_bend"])
    r = gpu.RouterBank(lay["polyphony"], lay["first_voice"], V, int(mpe), unison=np.full(G, d["unison"]),
                       mod_cc=np.full(G, d["mod_cc"]))
    vb = gpu.VoiceBank(float(sc.SR), lay["voice_index"], np.full(V, d["glide_seconds"], np.float32),
                       np.full(V, d["drift_amount"], np.float32), pb, flags=0 if mpe else gpu.VoiceBank.MIDI)
    if mpe:
        vb.set_main_voices(lay["main_voice"])
    cb = gpu.ControllerBank(G, d["controllers"], float(sc.SR), int(mpe))
    cb.set_voice_map(lay["voice_instrument"])
    pt = gpu.ProcessTimeBank(G, float(sc.SR))
    pt.set_voice_map(lay["voice_instrument"])
    g = gpu.VoiceGraph(spec, V)
    g.set_coefs(coef)
    g.set_state(state)
    buses = gpu.Buses(V, (lay["first_voice"] + d["mpe"]).astype(np.int32), np.full(G, d["n_voices"], np.int32))
    try:
        n0 = gpu.kernel_launches()
        want = g.process_context_host(r, vb, off, ev, controllers=cb, times=pt, time_offsets=toff, transports=tr,
                                      buses=buses)
        hand = gpu.kernel_launches() - n0
    finally:
        for x in (r, vb, cb, pt, g, buses):
            x.close()
    assert_same_bits(got, want, f"traced {case} synth vs the hand-wired context call")
    assert launches == [hand], (launches, hand)


@pytest.mark.gpu
def test_record_overflow_is_refused_after_the_call(gpu, tmp_path):
    """Unison with the full event mix: more than MLB_VOICE_MAX_EVENTS note events reach a voice in one vector, the
    router drops them, and TracedSynth::process says so by instrument instead of returning rows that differ from
    the reference."""
    from madronalib_b200 import workloads as wl
    d = sc.dump("unison")
    G, T = 7, 44
    off, ev = wl.midi_performance(G, T, d["polyphony"], False, density=0.5, seed=3)
    toff, tr = wl.transport_updates(G, T, float(sc.SR), seed=4, every=1, chaos=0.2)
    for name, a in (("offsets", off), ("events", ev), ("toff", toff), ("tr", tr)):
        np.ascontiguousarray(a).tofile(str(tmp_path / (name + ".bin")))
    sc.build_exe()
    r = subprocess.run([sc.EXE, "run", "unison", str(G), str(T), str(tmp_path), str(T)], capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 1 and "note events found their voice's record full (4 per voice and vector)" in r.stdout, \
        r.stdout + r.stderr
