"""K10, CPU side: the plain-C strict-order port of the per-instrument output buses against the committed golden and,
where oracle/_ref was built, against the reference's own Synth::processVector (source/app/MLSynth.h:36-60) compiled
in place (oracle/_ref/libmlsynth.so).  Also the bus layouts of workloads.instrument_buses and the host-side checks
of mlb_buses_create.  NaN equals NaN (DESIGN.md 5)."""
import os

import numpy as np
import pytest

from tests.bus_cases import random_layout, special_rows
from tests.common import assert_same_bits

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "buses.npz")


@pytest.fixture(scope="module")
def synth_ref():
    """The reference's Synth compiled in place; built here where the reference tree exists."""
    from oracle import bindings, bus_bindings
    if not bus_bindings.synth_ref_available() and bindings.reference_dir():
        bus_bindings.build("ref")
    if not bus_bindings.synth_ref_available():
        pytest.skip("oracle/_ref/libmlsynth.so not built (no reference tree here)")
    return bus_bindings.ref_buses


def test_port_equals_golden():
    from oracle.bus_bindings import port_buses
    g = np.load(GOLDEN)
    for P in (1, 3):
        assert_same_bits(port_buses(g["rows_p%d" % P], g["first"], g["count"]), g["bus_p%d" % P], "P = %d" % P)
    b = g["bus_p3"]
    assert np.isnan(b).any() and np.isinf(b).any() and ((b != 0) & (np.abs(b) < np.finfo(np.float32).tiny)).any()
    assert not (np.signbit(b) & (b == 0)).any(), "a sum from +0 is never -0 under round to nearest"
    assert (b[:, :, 0] == 0).all() and not np.signbit(b[:, :, 0]).any(), "an empty bus is +0"


@pytest.mark.parametrize("P,seed", [(1, 41), (2, 42), (3, 43)])
def test_port_equals_reference_random_layouts(synth_ref, P, seed):
    from oracle.bus_bindings import port_buses
    rng = np.random.default_rng(seed)
    V = 57
    first, count = random_layout(rng, V, 23, 16)
    first[:2], count[:2] = (0, V - 16), (16, 16)
    rows = special_rows(5, P, V, seed)
    want = synth_ref(rows, first, count)
    assert_same_bits(port_buses(rows, first, count), want, "port vs Synth, P = %d" % P)
    assert np.isfinite(want).mean() > 0.5


def test_reference_synth_refuses_17_voices(synth_ref):
    rows = special_rows(1, 1, 20, 44)
    with pytest.raises(ValueError, match="17 voices"):
        synth_ref(rows, np.array([0, 1], np.int32), np.array([3, 17], np.int32))
    synth_ref(rows, np.array([0, 1], np.int32), np.array([3, 16], np.int32))


def test_instrument_buses_layouts():
    from madronalib_b200 import workloads as wl
    f, c = wl.instrument_buses(4096, 16)
    assert f.dtype == c.dtype == np.int32 and f.shape == c.shape == (4096,)
    assert (f == np.arange(4096) * 16).all() and (c == 16).all() and f[-1] + c[-1] == 65536
    f, c = wl.instrument_buses(3, 4, mpe=True)
    assert f.tolist() == [1, 6, 11] and c.tolist() == [4, 4, 4]
    # every voice that is not a main voice is in exactly one bus, and the main voices in none
    cover = np.zeros(15, int)
    for a, n in zip(f, c):
        cover[a:a + n] += 1
    assert cover.tolist() == [0, 1, 1, 1, 1] * 3


def test_create_rejects_bad_arguments_without_touching_a_device():
    from madronalib_b200 import api
    api.lib()
    for V, first, count, where in ((8, [], [], None), (0, [0], [1], None), (8, [0, -1], [1, 1], "bus 1"),
                                   (8, [0, 2], [1, -2], "bus 1"), (8, [0, 0, 5], [8, 1, 4], "bus 2"),
                                   (8, [8], [1], "bus 0"), (8, [2**31 - 1], [1], "bus 0")):
        with pytest.raises(api.MlbError) as e:
            api.Buses(V, first, count)
        assert e.value.code == 1, (V, first, count)
        if where:
            assert where in str(e.value), str(e.value)
    with pytest.raises(ValueError):
        api.Buses(8, [0, 1], [1])


def test_create_fails_loudly_without_a_device():
    from madronalib_b200 import api
    if api.device_count() > 0:
        pytest.skip("a GPU is visible here")
    with pytest.raises(api.MlbError) as e:
        api.Buses(8, [0, 4], [4, 4])
    assert e.value.code == 3 and "no CPU fallback" in str(e.value)
