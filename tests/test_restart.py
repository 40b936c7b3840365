"""Restarting instruments without a device: the expected output of a restart needs no new reference code, and the
argument checks of the reset entry points come before anything touches the device.

A restarted instrument at vector t is the reference run of the performance's slice [t, T) (offsets rebased, event
times unchanged, as they are frames within the vector).  Here the traced midi / mpe banks run through the CPU stages
(tests/synth_cases.port_stages), with fresh port objects for every slice, and equal those reference slices bit for
bit."""
import ctypes

import numpy as np
import pytest

from madronalib_b200 import api
from tests import restart_cases as rc
from tests import synth_cases as sc
from tests.common import assert_same_bits

RESETS = ("mlb_graph_reset_voices", "mlb_voices_reset", "mlb_routers_reset", "mlb_controllers_reset",
          "mlb_process_time_reset", "mlb_published_reset")


@pytest.fixture(scope="module")
def L():
    from madronalib_b200 import build
    build.build()
    return api.lib()


@pytest.mark.parametrize("fn", RESETS)
def test_reset_arguments_are_checked_first(L, fn):
    one = np.zeros(1, np.int32)
    f = getattr(L, fn)
    assert f(None, None, 1) == 1 and b"null" in L.mlb_last_error() and b"list of 1" in L.mlb_last_error()
    assert f(None, one.ctypes.data, -1) == 1 and b"must not be negative" in L.mlb_last_error()
    assert f(None, None, 0) == 1 and b"null" in L.mlb_last_error()  # no bank
    assert f(None, one.ctypes.data, 1) == 1 and b"null" in L.mlb_last_error()


@pytest.mark.parametrize("case,G,T,restarts", [("midi", 7, 40, {13: [2, 5], 29: [5, 0]}),
                                               ("mpe", 7, 36, {9: [6], 21: [1, 6, 1]})])
def test_port_stages_over_slices_equal_reference_slices(port, case, G, T, restarts):
    from oracle import tsynth_bindings
    if not tsynth_bindings.ref_available():
        pytest.skip("oracle/_ref/libmltsynth.so not built (no reference tree where build() ran)")
    d = sc.dump(case)
    off, ev, toff, tr = sc.performance(d, G, T, seed=T + 3, density=0.4)
    want = rc.expected(lambda *a: tsynth_bindings.ref_synth(case, d["n_voices"], *a)[0], off, ev, toff, tr, restarts)
    got = rc.expected(lambda o, e, to, r: sc.port_stages(d, G, o, e, to, r, port), off, ev, toff, tr, restarts)
    assert_same_bits(got, want, f"{case}: port stages vs reference, restarts {restarts}")
    full, _ = tsynth_bindings.ref_synth(case, d["n_voices"], off, ev, toff, tr)
    for gs in restarts.values():
        assert not np.array_equal(want[:, :, gs], full[:, :, gs])
