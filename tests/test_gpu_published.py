"""Published signals of a traced Synth on the GPU: tests/cpp/test_published_trace runs the Synth subclass of
tests/cpp/published_body.h for G instruments from raw events (K12 -> K7 -> graph -> bus sum -> K14 per time chunk),
and after every call reads each instrument's signals (readLatest, read, peekLatest, getAvailableFrames).  Bus rows,
counts and frames equal G reference AudioContext + Synth objects (oracle/_ref/libmlpsynth.so) bit for bit, rings that
overflow within one vector and frames that rotate between voices included."""
import numpy as np
import pytest

from tests import published_cases as pc
from tests import synth_cases as sc
from tests.common import assert_same_bits


def _performance(d, G, T, seed):
    off, ev, _, _ = sc.performance(d, G, T, seed=seed, late=G // 2 if G > 2 else None, density=0.3)
    return off, ev


@pytest.mark.gpu
@pytest.mark.parametrize("case,G,T,splits", [("midi", 1, 24, (24,)), ("midi", 37, 40, (5, 17, 1, 17)),
                                             ("mpe", 37, 30, (13, 3, 14)), ("midi", 4096, 16, (7, 9))])
def test_published_signals_equal_reference_synths(gpu, tmp_path, case, G, T, splits):
    from oracle import psynth_bindings
    if not psynth_bindings.ref_available():
        pytest.skip("oracle/_ref/libmlpsynth.so not built (no reference tree where build() ran)")
    d = pc.dump(case)
    off, ev = _performance(d, G, T, seed=G + T)
    bus, counts, dest, _ = pc.run(tmp_path, case, G, T, off, ev, splits, chunk_blocks=4)
    want_bus, want_counts, want_dest = psynth_bindings.ref_psynth(case, d["n_voices"], off, ev, splits)
    what = f"published {case} synth, {G} instruments, calls of {splits} vectors"
    assert_same_bits(bus, want_bus, what + ": bus rows")
    assert np.array_equal(counts, want_counts), what + ": counts"
    assert_same_bits(dest, want_dest, what + ": frames read")
    assert np.abs(want_dest).max() > 0.1 and want_counts.max() > 0


@pytest.mark.gpu
def test_publishing_leaves_audio_alone_and_adds_one_launch_per_chunk(gpu, tmp_path):
    """The same synth with its stores removed: the same bus rows, and one launch fewer in every time chunk."""
    d = pc.dump("midi")
    G, T, splits, chunk = 21, 30, (5, 17, 8), 4
    off, ev = _performance(d, G, T, seed=5)
    bus, _, _, launches = pc.run(tmp_path, "midi", G, T, off, ev, splits, chunk_blocks=chunk)
    bus0, _, _, launches0 = pc.run(tmp_path, "nostore", G, T, off, ev, splits, chunk_blocks=chunk)
    assert_same_bits(bus, bus0, "bus rows with and without published stores")
    assert np.abs(bus).max() > 0.1
    assert launches == [n0 + -(-n // chunk) for n0, n in zip(launches0, splits)], (launches, launches0)


@pytest.mark.gpu
def test_published_bank_from_python_equals_the_model(gpu):
    """api.PublishedBank on hand-made device rows: two signals, three stores, 5 instruments of 3 voices, two chunks;
    every read equals the numpy model of tests/test_published_trace.py."""
    import torch
    from tests.test_published_trace import Model, _model_calls
    G, NV, T = 5, 3, 6
    signals, stores = [(40, 2, 2, 0), (64, 1, 1, 7)], [(0, 40), (1, 64), (0, 17)]
    bank = gpu.PublishedBank(G * NV, np.arange(G) * NV, np.full(G, NV), signals, stores)
    try:
        assert bank.planes == 5
        rng = np.random.default_rng(1)
        rows = rng.standard_normal((T, 1 + bank.planes, G * NV, 64)).astype(np.float32)  # plane 0: audio
        dev = torch.from_numpy(rows).cuda()
        for t0, t1 in ((0, 2), (2, T)):
            bank.process_device(dev[t0:t1], 1, 1 + bank.planes, t1 - t0)
        torch.cuda.synchronize()
        for s, (mf, mv, ch, od) in enumerate(signals):
            # the signal's stores in call order, with the first published plane of each (plane 0 is the audio output)
            items = [(fr, 1 + sum(signals[x][2] for x, _ in stores[:k])) for k, (sig, fr) in enumerate(stores) if sig == s]
            models = [Model(mf, mv, ch, od) for _ in range(G)]
            for g, m in enumerate(models):
                seq = [(rows[t, p:p + ch, g * NV + v, :], fr) for t in range(T) for v in range(NV) for fr, p in items]
                _model_calls(m, [(seq, 3, 0)])
            for mode, n in ((2, 30), (0, 25), (1, 9), (3, 0), (1, 200)):
                dest, counts = bank.read(s, mode, n)
                for g, m in enumerate(models):
                    c, d = _model_calls(m, [([], mode, n)])[0]
                    assert counts[g] == c, (s, g, mode)
                    assert np.array_equal(dest[g].view(np.uint32), d.view(np.uint32)), (s, g, mode)
    finally:
        bank.close()
