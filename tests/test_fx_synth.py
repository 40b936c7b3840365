"""mlb::tr::TracedSynth through a Synth::processVector override, on the CPU: the Synth subclass of
tests/cpp/fx_synth_body.h, traced with only the namespace changed (tests/cpp/test_fx_synth.cpp), run through the CPU
stages (the voice graph through the port, the bus sum, the instrument graph through the port) equals G complete
reference AudioContext + FxSynth objects (whose section reads its carried member before and after the base call) running the same source (oracle/_ref/libmlfxsynth.so) bit for bit; an
override that only calls the base traces exactly as no override; and every override TracedSynth cannot run is refused
by name."""
import re
import subprocess

import numpy as np
import pytest

from madronalib_b200.graph import OP_NAME
from tests import fx_synth_cases as fc
from tests import synth_cases as sc
from tests.common import assert_same_bits


@pytest.fixture(scope="module")
def fxsynth():
    from oracle import fxsynth_bindings
    if not fxsynth_bindings.ref_available():
        pytest.skip("oracle/_ref/libmlfxsynth.so not built (no reference tree where build() ran)")
    return fxsynth_bindings


def test_instrument_graph_layout():
    """Controllers in first-use order across processVector (73 before the base call, 1 in the voices, 74 after); the
    voice graph has the two bus rows the base call was handed, the instrument graph three outputs over the bus rows, the
    three controller planes and the beat phase, with one carried row."""
    d = fc.dump("midi")
    assert d["controllers"] == [73, 1, 74] and d["phase"] == 1 and len(d["outs"]) == 2
    # the carried delay output is read before the base call (a tap) and after it (the feedback): one feedback edge
    ig = d["instrument"]
    assert ig["bus_planes"] == 2 and ig["planes"] == 6 and len(ig["outs"]) == 3
    planes = sorted(n["iarg"] for n in ig["nodes"] if OP_NAME[n["op"]] == "INPUT")
    assert planes == [0, 1, 2, 3, 4, 5]
    names = [OP_NAME[n["op"]] for n in ig["nodes"]]
    assert names.count("FEEDBACK_READ") == 1 and names.count("FEEDBACK_WRITE") == 1
    assert {"LOPASS", "FRACTIONAL_DELAY", "ALLPASS_INT", "SIN"} <= set(names)
    # the voice graph reads only its own controller (1, plane 9) and no beat phase
    vplanes = sorted(n["iarg"] for n in d["nodes"] if OP_NAME[n["op"]] == "INPUT")
    assert vplanes == [0, 1, 3, 9]
    # the pass-through output is a copy of bus row 0
    last = ig["nodes"][ig["outs"][2]]
    assert OP_NAME[last["op"]] == "SELECT" and ig["nodes"][last["in"][0]]["iarg"] == 0


def test_base_only_override_dumps_as_no_override():
    """An override that only hands `outputs` to the base call: the same dump, byte for byte, as the synth without it,
    and as that synth traced by tests/cpp/test_synth_trace -- no instrument graph."""
    body, base = fc.dump_text("body"), fc.dump_text("bodybase")
    assert body == base and '"instrument"' not in base
    sc.build_exe()
    r = subprocess.run([sc.EXE, "dump", "midi"], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and r.stdout == body


@pytest.mark.parametrize("case", ["midi", "mpe"])
def test_port_stages_equal_reference_synths(fxsynth, port, case):
    """7 instruments x 44 vectors of raw MIDI / MPE (stealing, glide, pedal, bend, pressure, CC 1 / 73 / 74 moves,
    CC 123) and a host transport with stops, jumps and tempo changes; instrument 5 gets its first event at vector 14 and
    instrument 6 none at all."""
    d = fc.dump(case)
    G, T = 7, 44
    off, ev, toff, tr = sc.performance(d, G, T, seed=3, late=5, never=6)
    assert len(np.unique(tr["bpm"])) > 2
    want, _ = fxsynth.ref_synth(case, d["n_voices"], off, ev, toff, tr)
    got = fc.port_stages(d, G, off, ev, toff, tr, port)
    assert_same_bits(got, want, f"traced {case} FxSynth through the CPU stages vs reference AudioContext + FxSynth")
    assert np.abs(want).max() > 0.1
    # the instrument section is audible: the wet path differs from the plain bus row 0 (output 2)
    assert not np.array_equal(want[:, 0], want[:, 2])
    assert not want[:, :, 6].any()
    assert not want[:T // 3, :, 5].any() and want[T // 3:, :, 5].any()


REFUSALS = [
    ("nobase", "Synth::processVector does not call the base Synth::processVector"),
    ("twice", "calls the base Synth::processVector more than once in a vector"),
    ("voice", "getInputVoice\\(0\\) outside the base Synth::processVector call"),
    ("heldvoice", "Synth::processVector reads, outside the base Synth::processVector call, a DSPVector made in "
                  "processVoice \\(a Voice& kept past the call"),
    ("pre", "voice 0 reads a DSPVector made outside processVoice \\(before the base Synth::processVector call"),
    ("member", "voice 0 reads a DSPVector made outside processVoice \\(before the base Synth::processVector call, or "
               "by the instrument section\\)"),
    ("shared", "a functor object is called by voice 0 and by the instrument section"),
    ("store", "storePublishedSignal\\(level\\): outside processVoice"),
    ("unassigned", "leaves outputs\\[1\\] unassigned: it is neither handed to the base Synth::processVector nor "
                   "assigned after it"),
    ("stale", "reads outputs\\[1\\] before assigning it"),
    ("param", "tr::param\\(wet\\) in Synth::processVector outside the base call"),
]


@pytest.mark.parametrize("case,msg", REFUSALS)
def test_refusals_name_the_construct(case, msg):
    fc.build_exe()
    r = subprocess.run([fc.EXE, "dump", case], capture_output=True, text=True, timeout=60)
    assert r.returncode == 1 and re.search(msg, r.stdout), r.stdout + r.stderr


def test_outputs_handed_to_the_base_call_pass_through():
    """When `outputs` itself goes to the base call, an output the section does not assign is its bus row."""
    fc.build_exe()
    r = subprocess.run([fc.EXE, "dump", "passed"], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0 and "not refused" in r.stdout, r.stdout + r.stderr
