"""mlb::tr::TracedSynth on the CPU: the Synth subclass of tests/cpp/synth_body.h, traced with only the namespace changed
(tests/cpp/test_synth_trace.cpp), run through the CPU stages (host routers -> port Voice bank -> port controllers ->
port beat phase -> port graph -> port buses) equals G complete reference AudioContext + Synth objects running the same
source (oracle/_ref/libmltsynth.so) bit for bit; and every construct TracedSynth cannot run is refused by name."""
import subprocess

import numpy as np
import pytest

from madronalib_b200.graph import OP_NAME
from tests import synth_cases as sc
from tests.common import assert_same_bits


@pytest.fixture(scope="module")
def tsynth():
    from oracle import tsynth_bindings
    if not tsynth_bindings.ref_available():
        pytest.skip("oracle/_ref/libmltsynth.so not built (no reference tree where build() ran)")
    return tsynth_bindings


def test_traced_graph_layout():
    """Voice rows at planes 0..7 (only those read), controllers 1 and 74 at 8 and 9, the beat phase at 10; one carried
    row; two outputs; per-voice words where the cutoff and detune depend on voiceIndex."""
    d = sc.dump("midi")
    assert d["controllers"] == [1, 74] and d["phase"] == 1 and d["n_voices"] == d["polyphony"] == 16
    planes = sorted(n["iarg"] for n in d["nodes"] if OP_NAME[n["op"]] == "INPUT")
    assert planes == [0, 1, 3, 6, 8, 9, 10] and d["drift_amount"] == 0
    names = [OP_NAME[n["op"]] for n in d["nodes"]]
    assert names.count("FEEDBACK_READ") == 1 and names.count("FEEDBACK_WRITE") == 1 and len(d["outs"]) == 2
    lp = next(n for n in d["nodes"] if OP_NAME[n["op"]] == "LOPASS")
    assert len({tuple(c) for c in lp["coef"]}) == 16  # one cutoff per voice
    sine = next(n for n in d["nodes"] if OP_NAME[n["op"]] == "SINE")
    assert len({tuple(s) for s in sine["state"]}) == 1


@pytest.mark.parametrize("case", ["midi", "mpe", "modcc", "unison"])
def test_port_stages_equal_reference_synths(tsynth, port, case):
    """7 instruments x 44 vectors of raw MIDI / MPE (stealing, glide, pedal, bend, note and channel pressure, CC 1 / 74
    moves, CC 123) and a host transport with stops and jumps; instrument 5 gets its first event at vector 14 and
    instrument 6 none at all."""
    d = sc.dump(case)
    G, T = 7, 44
    off, ev, toff, tr = sc.performance(d, G, T, seed=3, late=5, never=6)
    want, _ = tsynth.ref_synth(case, d["n_voices"], off, ev, toff, tr)
    got = sc.port_stages(d, G, off, ev, toff, tr, port)
    assert_same_bits(got, want, f"traced {case} synth through the CPU stages vs reference AudioContext + Synth")
    assert np.abs(want).max() > 0.1
    assert not want[:, :, 6].any()
    assert not want[:T // 3, :, 5].any() and want[T // 3:, :, 5].any()


def test_unison_differs_exactly_where_records_overflow(tsynth, port):
    """In unison every note event goes to every voice, whose record holds MLB_VOICE_MAX_EVENTS (4) note events per
    vector; the router drops and counts the rest (TracedSynth::process then throws).  With the full event mix, the
    instruments that differ from the reference are exactly those whose records overflowed."""
    from madronalib_b200 import workloads as wl
    from tests.router_cases import route_on_host
    d = sc.dump("unison")
    G, T = 7, 44
    off, ev = wl.midi_performance(G, T, d["polyphony"], False, density=0.5, seed=3)
    toff, tr = wl.transport_updates(G, T, float(sc.SR), seed=4, every=1, chaos=0.2)
    _, _, _, overflow, _ = route_on_host(off, ev, sc.layout(d, G), unison=np.ones(G), mod_cc=np.full(G, 16))
    want, _ = tsynth.ref_synth("unison", d["n_voices"], off, ev, toff, tr)
    got = sc.port_stages(d, G, off, ev, toff, tr, port)
    same = (got.view(np.uint32) == want.view(np.uint32)).all(axis=(0, 1, 3))
    assert overflow.any() and [bool(x) for x in same] == [int(n) == 0 for n in overflow]


REFUSALS = [
    ("rescale", "reads or rescales the accumulator outputs\\[0\\]; only outputs\\[0\\] \\+= x"),
    ("twice", "adds twice into outputs\\[0\\]"),
    ("assign", "assigns outputs\\[0\\] = x"),
    ("other", "voice 0 reads the rows of voice 1"),
    ("differ", "voice 1 records a different graph from voice 0"),
    ("inactive", "voice 2 is not active"),
    ("inputs", "the synth has audio inputs"),
    ("controller", "controller 129 is above 128"),
    ("polyphony", "polyphony 3 must be in \\[getNumVoices\\(\\) = 4, 16\\]"),
    ("shared", "a functor object is called by voice 0 and voice 1"),
    ("sharedrow", "voice 1 reads a DSPVector of another voice \\(a member shared between voices"),
    ("heldvoice", "voice 1 reads a DSPVector of another voice"),
    ("drift", "drift amount 0.500000 is not 0: EventsToSignals starts an instrument's voices, drift included, only at "
              "its first event \\(awake_\\)"),
]


@pytest.mark.parametrize("case,msg", REFUSALS)
def test_refusals_name_the_construct(case, msg):
    import re
    sc.build_exe()
    r = subprocess.run([sc.EXE, "dump", case], capture_output=True, text=True, timeout=60)
    assert r.returncode == 1 and re.search(msg, r.stdout), r.stdout + r.stderr
