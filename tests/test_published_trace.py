"""Published signals in the tracing layer (CPU): the Synth subclass of tests/cpp/published_body.h traced with only the
namespace changed records its declarations, store items and the stored rows as extra graph outputs; every store
TracedSynth cannot run is refused by name; and a numpy model of the closed-form selection and ring that K14 and the
batched reads implement equals the reference's SignalProcessor::PublishedSignal across the parameter space."""
import ctypes

import numpy as np
import pytest

from madronalib_b200.graph import OP_NAME
from tests import published_cases as pc


def test_traced_body_records_declarations_and_stores():
    d = pc.dump("midi")
    assert [(p["name"], p["max_frames"], p["max_voices"], p["channels"], p["octaves_down"]) for p in d["published"]] == \
        [("scope", 64, 2, 2, 1), ("voices", 64, 4, 1, 7), ("pitch", 17, 16, 1, 3)]
    # the store into "nowhere" records nothing
    assert [(s["signal"], s["frames"], len(s["rows"])) for s in d["stores"]] == [(0, 64, 2), (1, 64, 1), (2, 17, 1)]
    nodes = d["nodes"]
    # the gate Voice row is stored as it is: an INPUT node
    gate = d["stores"][1]["rows"][0]
    assert OP_NAME[nodes[gate]["op"]] == "INPUT" and nodes[gate]["iarg"] == 1
    # one select(x, x, x) copy per stored row, after the audio outputs
    rows = [r for s in d["stores"] for r in s["rows"]]
    assert len(d["published_outs"]) == len(rows) == 4 and len(d["outs"]) == 2
    for o, r in zip(d["published_outs"], rows):
        assert OP_NAME[nodes[o]["op"]] == "SELECT" and nodes[o]["in"][:3] == [r, r, r]
    assert not set(d["published_outs"]) & set(d["outs"])


def test_synth_without_stores_dumps_as_before():
    d = pc.dump("nostore")
    assert d["stores"] == [] and d["published_outs"] == []
    assert not any(OP_NAME[n["op"]] == "SELECT" for n in d["nodes"])


@pytest.mark.parametrize("case,message", [
    ("channels", "a DSPVectorArray<1> into a signal of 2 channels"),
    ("frames", "frames 65 is not in 0..64"),
    ("maxframes", "frames 33 is above maxFrames 32"),
    ("vert", "storePublishedSignalVert(sig) takes a host pointer"),
    ("differ", "a different number of published stores"),
])
def test_refusals_name_the_store(case, message):
    rc, out = pc.trace(case)
    assert rc == 1 and message in out, out


# ---------------------------------------------------------------- the closed form, in numpy
class Model:
    """One instrument's published signal as K14 and the read kernel compute it: the written frames in closed form,
    the ring by its final indices."""

    def __init__(self, max_frames, max_voices, channels, octaves):
        size = 64
        while size < max_frames * channels * max_voices:
            size *= 2
        self.size, self.ch, self.od = size, channels, octaves
        self.ring = np.zeros(size, np.float32)
        self.w = self.r = self.c = 0

    def store_chunk(self, rows):
        """rows: the chunk's stores in order, each a [channels][frames] array."""
        seq = np.concatenate([np.asarray(x, np.float32).T for x in rows]) if rows else np.zeros((0, self.ch))
        total = len(seq)
        n = (self.c + total) >> self.od
        k = (np.arange(1, n + 1) << self.od) - self.c - 1  # the written frames
        flat = seq[k].reshape(-1)
        W, size, dist = len(flat), self.size, 2 * self.size - 1
        j = np.arange(max(0, W - size), W)
        self.ring[(self.w + j) % size] = flat[j]
        avail = min(((self.w - self.r) & dist) + W, size)
        self.w = (self.w + W) & dist
        self.r = (self.w - avail) & dist
        self.c = (self.c + total) & ((1 << self.od) - 1)

    def avail(self):
        return (self.w - self.r) & (2 * self.size - 1)

    def _copy(self, start, n):
        return self.ring[(start + np.arange(n)) % self.size]

    def read(self, frames, latest=False):
        want, av = frames * self.ch, self.avail()
        if latest and av > want:
            self.r = (self.r + av - want) & (2 * self.size - 1)
            av = want
        n = min(av, want)
        out = self._copy(self.r, n)
        self.r = (self.r + n) & (2 * self.size - 1)
        return out

    def peek(self, frames):
        want, av = frames * self.ch, self.avail()
        return self._copy(self.r + av - want, want) if av >= want else None


@pytest.fixture(scope="module")
def psynth():
    from oracle import psynth_bindings
    if not psynth_bindings.ref_available():
        pytest.skip("oracle/_ref/libmlpsynth.so not built (no reference tree where build() ran)")
    return psynth_bindings


def _model_calls(m, calls):
    out = []
    for stores, mode, frames in calls:
        m.store_chunk([r[:, :fr] for r, fr in stores])
        dest = np.zeros(frames * m.ch, np.float32)
        if mode in (0, 1):
            x = m.read(frames, latest=mode == 0)
            dest[:len(x)] = x
            out.append((len(x), dest))
        elif mode == 2:
            x = m.peek(frames)
            if x is not None:
                dest[:] = x
            out.append((int(x is not None), dest))
        else:
            out.append((m.avail() // m.ch, dest))
    return out


@pytest.mark.parametrize("octaves", range(9))
def test_closed_form_model_equals_reference_published_signal(psynth, octaves):
    """For voices 1..16 storing 0, 1, 17 or 64 frames per vector, in calls of 1..3 vectors with one read after each
    (every mode, interleaved): rings from 64 floats (overflowed within one call) up, 1 to 3 channels."""
    rng = np.random.default_rng(octaves)
    for voices in range(1, 17):
        for frames in (0, 1, 17, 64):
            for channels, max_voices in ((1, 1), (2, 3), (3, 1)):
                max_frames = max(frames, 1)
                calls = []
                for c in range(7):
                    vectors = int(rng.integers(1, 4))
                    stores = [(rng.standard_normal((channels, 64)).astype(np.float32), frames)
                              for _ in range(vectors * voices)]
                    calls.append((stores, (c + voices) % 4, int(rng.integers(0, 90))))
                want = psynth.ref_signal(max_frames, max_voices, channels, octaves, calls)
                got = _model_calls(Model(max_frames, max_voices, channels, octaves), calls)
                for c, ((n0, d0), (n1, d1)) in enumerate(zip(got, want)):
                    what = f"octaves {octaves}, {voices} voices x {frames} frames, {channels} ch, call {c}"
                    assert n0 == n1, what
                    assert np.array_equal(d0.view(np.uint32), d1.view(np.uint32)), what
