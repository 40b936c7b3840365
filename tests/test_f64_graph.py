"""The float64 evaluator (tests/f64_graph.py) pinned against the port before it judges fast mode on the GPU.

For every case of tests/fast_cases.py: the exact port stays within its case's bound of the evaluator, phase and seed
words match the port bit for bit, and the bound fast mode is held to rejects a 1e-4 coefficient fault and two
swapped voices."""
import functools

import numpy as np
import pytest

from madronalib_b200 import workloads as wl
from madronalib_b200.graph import GraphSpec
from tests import f64_graph as fg
from tests import fast_cases as fc

V, T = 40, 16


@functools.lru_cache(maxsize=None)
def _run(port, name):
    case = fc.BY_NAME[name]
    p = fc.prepare(port, case, V, T)
    out, _, st = port.run(p.spec, V, T, p.inp, p.state, p.coef)
    return p, out, st, fg.evaluate(p.spec, V, T, p.inp, p.state, p.coef)


def test_case_table_covers_every_fused_entry():
    """One case per X( row of MLB_FUSED_LIST, so that a new fused entry needs a new case."""
    rows = fc.fused_rows()
    assert len(rows) == 20, rows  # the regex reads the list as mlb200.cu writes it
    assert len(fc.FUSED) == len(rows)
    assert sorted(c.row for c in fc.FUSED) == sorted(rows)
    assert set(fc.BOUND) == set(fc.BY_NAME)


@pytest.mark.parametrize("name", [c.name for c in fc.CASES])
def test_port_against_f64(port, name):
    p, out, st, r = _run(port, name)
    err, serr = fg.rel_err(out, r.out), fg.state_err(st, r, p.spec)
    assert err < fc.BOUND[name] and serr < fc.BOUND[name], (err, serr, fc.BOUND[name])
    assert np.abs(r.out).max() > 1e-3  # the case really makes a signal
    np.testing.assert_allclose(r.mix, r.out.sum(axis=2))


@pytest.mark.parametrize("name", [c.name for c in fc.CASES if c.name != "fm3_fdn8"])
def test_integer_state_bit_exact(port, name):
    """Phase accumulators and noise seeds of generators fed straight from INPUT / PARAM equal the port's.  (FM3's
    carrier frequency is a product computed in float64 here, so its phase may differ by rounding.)"""
    p, _, st, r = _run(port, name)
    ints = fg.int_slots(p.spec)
    assert np.array_equal(r.state_int[ints], st[ints])


@pytest.mark.parametrize("name", [c.name for c in fc.CASES])
def test_negative_controls(port, name):
    """A fault of 1e-4 in one coefficient word of one voice, and two voices' states swapped, are both rejected by
    the bounds the GPU test applies: the case's bound and max(4 * err_exact, 2^-20)."""
    p, out, _, r = _run(port, name)
    bound = min(fc.BOUND[name], fc.fast_bound(fg.rel_err(out, r.out)))
    v = V // 2
    slot = fc.probe_slot(fc.BY_NAME[name], p.spec)
    if slot is not None or p.spec.n_in:
        coef, inp = p.coef.copy(), None if p.inp is None else p.inp.copy()
        if slot is not None:
            coef[slot, v] *= np.float32(1 + 1e-4)
        else:  # no coefficient words: the frequency input instead
            inp[:, 0, v] *= np.float32(1 + 1e-4)
        bad, _, _ = port.run(p.spec, V, T, inp, p.state, coef)
        assert fg.rel_err(bad, r.out) > bound
    else:
        assert name == "noise"  # nothing to scale: the swap below is its control
    st = p.state.copy()
    st[:, [0, V - 1]] = st[:, [V - 1, 0]]
    bad, _, _ = port.run(p.spec, V, T, p.inp, st, p.coef)
    assert fg.rel_err(bad, r.out) > bound


def test_phase_decisions_at_the_edges(port):
    """cvtps2dq's out-of-range rule (NaN, infinities, |freq| >= 0.5) and negative frequencies: the evaluator's phase
    words follow the port's through all of them, for SineGen, PhasorGen and SawGen."""
    bad = np.array([0.5, 0.75, -0.5, 1e9, -1e9, np.inf, -np.inf, np.nan, 2.0 ** -40, -0.0, -0.01], np.float32)
    for op in ("SINE", "PHASOR", "SAW"):
        g = GraphSpec()
        g.output(g.node(op, g.input(0)))
        n = 8
        inp = wl.freq_rows(n, 3) * np.float32(10.0)
        inp[1, 0, :, 10:10 + bad.size] = bad
        st = (np.arange(n, dtype=np.uint32) * np.uint32(0x9E3779B9))[None]
        _, _, ps = port.run(g, n, 3, inp, st, g.new_coefs(n))
        r = fg.evaluate(g, n, 3, inp, st, g.new_coefs(n))
        assert np.array_equal(r.state_int, ps), op
        assert np.isfinite(r.out[0]).all() and np.isfinite(r.out[2]).all(), op


@pytest.mark.parametrize("build", [lambda g: g.node("TICK", g.input(0)), lambda g: g.node("PULSE", g.input(0), g.input(1)),
                                   lambda g: g.node("INTEGER_DELAY", g.input(0)),
                                   lambda g: g.again(g.node("LOPASS", g.input(0)), g.input(1))])
def test_evaluator_refuses_other_ops(build):
    g = GraphSpec()
    g.output(build(g))
    with pytest.raises(ValueError):
        fg.evaluate(g, 2, 1, np.zeros((1, max(1, g.n_in), 2, 64), np.float32), g.new_state(2), g.new_coefs(2))
