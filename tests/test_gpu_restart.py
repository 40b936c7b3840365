"""Restarting instruments of a running bank on the GPU (mlb_*_reset, TracedSynth::restart): a restarted instrument
equals objects constructed at the restart and fed only what follows, bit for bit, and every other instrument equals a
run with no restart.  The traced Synth of tests/cpp/synth_body.h against the reference (oracle/_ref/libmltsynth.so)
over slices of the performance; each bank against a fresh bank fed the same slice; the graph at a delay write index
(blocks_done = 37) that is no multiple of any ring length."""
import numpy as np
import pytest

from madronalib_b200 import workloads as wl
from tests import restart_cases as rc
from tests import synth_cases as sc
from tests.common import assert_same_bits

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------- TracedSynth::restart
@pytest.mark.parametrize("case,G,T,splits,restarts", [
    ("midi", 37, 48, (5, 12, 1, 20, 10), {5: [0, 36], 17: [], 18: [7, 36, 7], 38: [20]}),
    ("midi", 4096, 40, (13, 27), {13: [0, 1, 2000, 4095]}),
    ("mpe", 33, 40, (13, 14, 13), {13: [4, 32], 27: [4]})])
def test_traced_synth_restart_equals_fresh_reference_synths(gpu, tmp_path, case, G, T, splits, restarts):
    from oracle import tsynth_bindings
    if not tsynth_bindings.ref_available():
        pytest.skip("oracle/_ref/libmltsynth.so not built (no reference tree where build() ran)")
    d = sc.dump(case)
    off, ev, toff, tr = sc.performance(d, G, T, seed=G + T, density=0.3)
    got, launches, restart_launches = rc.run(tmp_path, case, G, T, off, ev, toff, tr, splits, restarts)
    plain, plain_launches, _ = rc.run(tmp_path, case, G, T, off, ev, toff, tr, splits, {})
    want = rc.expected(lambda *a: tsynth_bindings.ref_synth(case, d["n_voices"], *a)[0], off, ev, toff, tr, restarts)
    what = f"traced {case} synth, {G} instruments, restarts {restarts}"
    assert_same_bits(got, want, what)
    hit = sorted({g for gs in restarts.values() for g in gs})
    others = np.setdiff1d(np.arange(G), hit)
    assert_same_bits(got[:, :, others], plain[:, :, others], what + ": instruments not restarted vs no restart")
    assert not np.array_equal(got[:, :, hit], plain[:, :, hit])
    # one launch per stateful bank: routers, Voice rows, graph, controllers and beat phase when built; none when empty
    per = 3 + (1 if d["controllers"] else 0) + (1 if d["phase"] else 0)
    assert restart_launches == [per if restarts[t] else 0 for t in sorted(restarts)]
    assert launches == plain_launches


# ---------------------------------------------------------------------------------------- the graph
def _graph(gpu, w, V):
    g = gpu.VoiceGraph(w.spec, V)
    g.set_coefs(w.coef)
    g.set_state(w.state)
    return g


def _inputs(w, T, t0):
    x = w.inputs(T, t0)
    return None if x is None else np.ascontiguousarray(x, np.float32)


@pytest.mark.parametrize("config,V", [("a", 2048), ("4", 256), ("6", 64)])
def test_graph_reset_voices_equals_fresh_graph(gpu, config, V):
    w = {"a": wl.config_a, "4": wl.config_4, "6": wl.config_6}[config](V)
    T0, T1 = 37, 45
    R = [1, 5, 5, V - 1, V // 2]
    keep = np.setdiff1d(np.arange(V), R)
    plain, reset, fresh = _graph(gpu, w, V), _graph(gpu, w, V), _graph(gpu, w, V)
    try:
        name = reset.kernel_name
        for g in (plain, reset):
            g.process_host(_inputs(w, T0, 0), T0)
        n0 = gpu.kernel_launches()
        reset.reset_voices([])
        assert gpu.kernel_launches() == n0
        reset.reset_voices(R)
        assert gpu.kernel_launches() == n0 + 1
        x = _inputs(w, T1, T0)
        want_keep, _ = plain.process_host(x, T1)
        got, _ = reset.process_host(x, T1)  # immediately after the reset, on the pipeline's other streams
        want_r, _ = fresh.process_host(x, T1)
        st, st_keep, st_r = reset.get_state(), plain.get_state(), fresh.get_state()
        assert reset.kernel_name == name
    finally:
        for g in (plain, reset, fresh):
            g.close()
    what = f"config {config}, {V} voices, reset at block {T0}"
    assert_same_bits(got[:, :, R], want_r[:, :, R], what + ": reset voices vs a fresh graph")
    assert_same_bits(got[:, :, keep], want_keep[:, :, keep], what + ": other voices vs no reset")
    assert np.array_equal(st[:, R], st_r[:, R]) and np.array_equal(st[:, keep], st_keep[:, keep])
    assert not np.array_equal(got[:, :, R], want_keep[:, :, R])


def test_refused_reset_writes_nothing(gpu):
    w = wl.config_6(32)
    plain, g = _graph(gpu, w, 32), _graph(gpu, w, 32)
    try:
        for h in (plain, g):
            h.process_host(_inputs(w, 9, 0), 9)
        n0 = gpu.kernel_launches()
        for bad, named in (([0, 32], "voice 32"), ([-1], "voice -1"), ([3, 40, 2], "voice 40")):
            with pytest.raises(gpu.MlbError, match=named):
                g.reset_voices(bad)
        assert gpu.kernel_launches() == n0
        x = _inputs(w, 11, 9)
        want, _ = plain.process_host(x, 11)
        got, _ = g.process_host(x, 11)
    finally:
        plain.close(), g.close()
    assert_same_bits(got, want, "a refused reset")


# ---------------------------------------------------------------------------------------- the other banks
def test_voice_bank_reset_after_drift_redraw_equals_fresh_bank(gpu):
    V, T0, T1 = 40, 9, 23
    vi, gs, _, pb = wl.voice_bank_params(V)
    da = np.full(V, 0.5, np.float32)
    ev = wl.voice_events(V, T0 + T1, seed=5)
    R = [0, 17, 17, 39]
    keep = np.setdiff1d(np.arange(V), R)
    banks = [gpu.VoiceBank(48000.0, vi, gs, da, pb) for _ in range(3)]
    plain, reset, fresh = banks
    try:
        for b in (plain, reset):
            b.process_host(ev[:T0])
        reset.reset(R)
        got = reset.process_host(ev[T0:])
        want_keep = plain.process_host(ev[T0:])
        want_r = fresh.process_host(np.ascontiguousarray(ev[T0:]))
    finally:
        for b in banks:
            b.close()
    assert_same_bits(got[:, :, R], want_r[:, :, R], "Voice bank: reset voices vs a fresh bank")
    assert_same_bits(got[:, :, keep], want_keep[:, :, keep], "Voice bank: other voices vs no reset")
    assert not np.array_equal(got[:, :, R], want_keep[:, :, R])


def _bank_case(make, feed, G, off, items, T0, R):
    """(got, want_fresh, want_plain) of a bank fed blocks [0, T0), reset on R, fed the rest; a fresh bank fed the
    rest; a bank never reset."""
    plain, reset, fresh = make(), make(), make()
    try:
        o0, i0 = off[:T0], items[:off[T0, 0]]
        feed(plain, o0, i0), feed(reset, o0, i0)
        reset.reset(R)
        o1, i1 = rc.slice_from(off, items, T0)
        return feed(reset, o1, i1), feed(fresh, o1, i1), feed(plain, o1, i1)
    finally:
        for b in (plain, reset, fresh):
            b.close()


def _check_instruments(got, fresh, plain, R, axis, what):
    G = got.shape[axis]
    keep = np.setdiff1d(np.arange(G), R)
    take = lambda a, ix: np.take(a, ix, axis=axis)  # noqa: E731
    assert_same_bits(take(got, R), take(fresh, R), what + ": reset instruments vs a fresh bank")
    assert_same_bits(take(got, keep), take(plain, keep), what + ": other instruments vs no reset")


def test_controller_bank_reset(gpu):
    G, T0, T = 37, 13, 40
    off, ch = wl.controller_changes(G, T, density=0.3, seed=3)
    ctrl = [1, 7, 74]
    R = [0, 12, 36]
    got, fresh, plain = _bank_case(lambda: gpu.ControllerBank(G, ctrl), lambda b, o, c: b.process_host(o, c),
                                   G, off, ch, T0, R)
    _check_instruments(got, fresh, plain, R, 2, "ControllerBank")


def test_process_time_bank_reset(gpu):
    G, T0, T = 37, 13, 40
    off, tr = wl.transport_updates(G, T, 48000.0, seed=9, every=1, chaos=0.3)
    R = [2, 30, 30]
    got, fresh, plain = _bank_case(lambda: gpu.ProcessTimeBank(G), lambda b, o, t: b.process_host(o, t),
                                   G, off, tr, T0, R)
    _check_instruments(got, fresh, plain, R, 2, "ProcessTimeBank")


@pytest.mark.parametrize("mpe", [False, True])
def test_router_bank_reset_keeps_counters(gpu, mpe):
    G, T0, T = 21, 11, 36
    lay = wl.midi_layout(G, 6, mpe)
    off, ev = wl.midi_performance(G, T, 6, mpe, density=0.5, seed=7)
    R = [0, 9, 20]

    def make():
        return gpu.RouterBank(lay["polyphony"], lay["first_voice"], lay["n_voices"], int(mpe))
    plain, reset, fresh = make(), make(), make()
    try:
        o0, e0 = off[:T0], ev[:off[T0, 0]]
        plain.process_host(o0, e0), reset.process_host(o0, e0)
        before = reset.counters()
        reset.reset(R)
        assert all(np.array_equal(a, b) for a, b in zip(reset.counters(), before))
        o1, e1 = rc.slice_from(off, ev, T0)
        got, want_r, want_keep = (b.process_host(o1, e1) for b in (reset, fresh, plain))
    finally:
        for b in (plain, reset, fresh):
            b.close()
    first, n = lay["first_voice"], lay["polyphony"] + (1 if mpe else 0)
    voices = lambda gs: np.concatenate([np.arange(first[g], first[g] + n[g]) for g in gs])  # noqa: E731
    keep = np.setdiff1d(np.arange(G), R)
    rec = lambda r, vs: r[0][:, vs].tobytes()  # noqa: E731
    assert rec(got, voices(R)) == rec(want_r, voices(R)), "RouterBank: reset instruments' records"
    assert rec(got, voices(keep)) == rec(want_keep, voices(keep)), "RouterBank: other records"

    def changes(r, g):
        coff, ch = r[1], r[2]
        return [ch[coff[t, g]:coff[t, g + 1]].tobytes() for t in range(coff.shape[0])]
    for g in R:
        assert changes(got, g) == changes(want_r, g), f"RouterBank: controller writes of instrument {g}"
    for g in keep:
        assert changes(got, g) == changes(want_keep, g), f"RouterBank: controller writes of instrument {g}"


def test_published_bank_reset(gpu):
    import torch
    G, per, T0, T1 = 9, 3, 5, 7
    V = G * per
    first, count = np.arange(G, dtype=np.int32) * per, np.full(G, per, np.int32)
    signals = [(256, 4, 1, 0), (64, 4, 2, 2)]
    stores = [(0, 64), (1, 17)]
    rng = np.random.default_rng(2)
    rows = torch.from_numpy(rng.standard_normal((T0 + T1, 3, V, 64)).astype(np.float32)).cuda()
    R = [0, 4, 4, 8]

    def make():
        return gpu.PublishedBank(V, first, count, signals, stores)
    plain, reset, fresh = make(), make(), make()
    try:
        for b in (plain, reset):
            b.process_device(rows[:T0], 0, 3, T0)
        torch.cuda.synchronize()
        reset.reset(R)
        for b in (plain, reset, fresh):
            b.process_device(rows[T0:], 0, 3, T1)
        torch.cuda.synchronize()
        reads = []
        for b in (reset, fresh, plain):
            r = []
            for s in (0, 1):
                for mode, frames in ((b.AVAILABLE, 0), (b.PEEK, 5), (b.READ_LATEST, 9), (b.READ, 30), (b.AVAILABLE, 0)):
                    r.append(b.read(s, mode, frames))
            reads.append(r)
    finally:
        for b in (plain, reset, fresh):
            b.close()
    for k, (got, want_r, want_keep) in enumerate(zip(*reads)):
        for part in (0, 1):
            _check_instruments(got[part], want_r[part], want_keep[part], R, 0, f"PublishedBank read {k}")
