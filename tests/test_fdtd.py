"""K9, CPU side: the plain-C port of the reference's FDTD membrane example (examples/audio-and-midi/fdtd.cpp)
against the committed golden and, where oracle/_ref was built, against the example's own text compiled in place
(oracle/_ref/libmlfdtd.so) in both floating-point modes: IEEE, and flush-to-zero as under
UsingFlushDenormalsToZero.  NaN equals NaN (DESIGN.md 5)."""
import hashlib
import os

import numpy as np
import pytest

from tests.common import assert_same_bits

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "fdtd.npz")


@pytest.fixture(scope="module")
def fdtd_ref():
    """The example's own text compiled against the reference; built here where the reference tree exists."""
    from oracle import bindings, fdtd_bindings
    if not fdtd_bindings.fdtd_ref_available() and bindings.reference_dir():
        fdtd_bindings.build("ref")
    if not fdtd_bindings.fdtd_ref_available():
        pytest.skip("oracle/_ref/libmlfdtd.so not built (no reference tree here)")
    return fdtd_bindings.RefFdtd()


def noise_case(V, T, seed, amp=0.1, f_lo=0.002, f_hi=0.05):
    """Noise excitation, per-instance frequencies swept over [f_lo, f_hi] cycles per sample."""
    rng = np.random.default_rng(seed)
    inp = np.zeros((T, 2, V, 64), np.float32)
    inp[:, 0] = (rng.uniform(-1, 1, (T, V, 64)) * amp).astype(np.float32)
    n = np.arange(T * 64, dtype=np.float64).reshape(T, 1, 64)
    f = np.linspace(f_lo, f_hi, V)[None, :, None] * (1.0 + 0.2 * np.sin(n / 700.0 + np.arange(V)[None, :, None]))
    inp[:, 1] = f.astype(np.float32)
    return inp


def port(inp, state=None, ftz=False, sr=48000.0):
    from oracle.fdtd_bindings import port_fdtd
    return port_fdtd(inp, state, ftz=ftz, sample_rate=sr)


def test_port_equals_golden():
    g = np.load(GOLDEN)
    for ftz in (0, 1):
        y, st = port(g["in"], ftz=bool(ftz))
        assert_same_bits(y, g["out_ftz%d" % ftz], "port vs golden, ftz=%d" % ftz)
        assert_same_bits(st, g["state_ftz%d" % ftz], "port state vs golden, ftz=%d" % ftz)
    assert np.abs(g["out_ftz0"]).max() > 1e-3


def test_example_graph_and_port_equal_golden_example():
    """The example's processFDTD as workloads.fdtd_example's graph (through the port oracle) feeding the port in FTZ
    mode gives the bits the reference's own processFDTD gave for 800 vectors."""
    from madronalib_b200 import workloads as wl
    from oracle.bindings import PortOracle
    g = np.load(GOLDEN)
    w = wl.fdtd_example(1)
    rows, _, _ = PortOracle().run(w.spec, 1, 800, None, w.state, w.coef)
    y, _ = port(rows, ftz=True)
    ex = np.ascontiguousarray(y[:, :, 0], "<f4")
    assert_same_bits(ex[:16], g["example_head"], "example head")
    assert hashlib.sha256(ex.tobytes()).digest() == g["example_sha256"].tobytes()


@pytest.mark.parametrize("ftz", [False, True])
def test_port_equals_reference_noise_sweep(fdtd_ref, ftz):
    inp = noise_case(7, 20, seed=3)
    want, want_st, _ = fdtd_ref.run(inp, ftz=ftz)
    got, got_st = port(inp, ftz=ftz)
    assert_same_bits(got, want, "noise sweep")
    assert_same_bits(got_st, want_st, "noise sweep state")
    assert np.abs(want).max() > 0.01


def test_port_equals_reference_subnormal(fdtd_ref):
    """Excitation around 1e-37: the surface goes subnormal; IEEE and FTZ must then give different bits."""
    inp = noise_case(5, 16, seed=4, amp=1e-37)
    outs = {}
    for ftz in (False, True):
        want, want_st, _ = fdtd_ref.run(inp, ftz=ftz)
        got, got_st = port(inp, ftz=ftz)
        assert_same_bits(got, want, "subnormal, ftz=%s" % ftz)
        assert_same_bits(got_st, want_st, "subnormal state, ftz=%s" % ftz)
        outs[ftz] = want
    a, b = outs[False], outs[True]
    assert not np.array_equal(a.view(np.uint32), b.view(np.uint32)), "FTZ made no difference: not exercised"
    sub = (a != 0) & (np.abs(a) < np.finfo(np.float32).tiny)
    assert sub.any(), "no subnormal output in IEEE mode"


@pytest.mark.parametrize("ftz", [False, True])
def test_port_equals_reference_split_and_random_state(fdtd_ref, ftz):
    rng = np.random.default_rng(5)
    V = 6
    state = rng.uniform(-0.5, 0.5, (V, 2, 16, 16)).astype(np.float32)
    inp = noise_case(V, 12, seed=6)
    want, want_st, _ = fdtd_ref.run(inp, state, ftz=ftz)
    y1, s1 = port(inp[:5], state, ftz=ftz)
    y2, s2 = port(inp[5:], s1, ftz=ftz)
    assert_same_bits(np.concatenate([y1, y2]), want, "5 + 7 blocks from a random state")
    assert_same_bits(s2, want_st, "state after 5 + 7 blocks")


@pytest.mark.parametrize("ftz", [False, True])
def test_port_equals_reference_unstable(fdtd_ref, ftz):
    """Frequencies past the stable limit (T^2 > 3/5, Fs > ~0.057) blow up to inf / NaN."""
    inp = noise_case(4, 40, seed=7, f_lo=0.06, f_hi=0.2)
    want, want_st, _ = fdtd_ref.run(inp, ftz=ftz)
    got, got_st = port(inp, ftz=ftz)
    assert_same_bits(got, want, "unstable")
    assert_same_bits(got_st, want_st, "unstable state")
    assert not np.isfinite(want).all()


def test_port_equals_reference_example(fdtd_ref):
    """The reference's own processFDTD (with its AudioContext) equals the example graph through both checkers."""
    from madronalib_b200 import workloads as wl
    from oracle.bindings import PortOracle
    want = fdtd_ref.example(800)
    w = wl.fdtd_example(1)
    rows, _, _ = PortOracle().run(w.spec, 1, 800, None, w.state, w.coef)
    got, _ = port(rows, ftz=True)
    assert_same_bits(got[:, :, 0], want, "example: graph + port vs processFDTD")
    ref_rows, _, _ = fdtd_ref.run(rows, ftz=True)
    assert_same_bits(ref_rows[:, :, 0], want, "example: graph + processFDTDModel vs processFDTD")


def test_port_other_sample_rate_differs():
    """The port takes the sample rate (isr and SK depend on it); at 44.1 kHz the bits must change."""
    inp = noise_case(3, 4, seed=8)
    a, _ = port(inp, sr=48000.0)
    b, _ = port(inp, sr=44100.0)
    assert np.isfinite(b).all() and not np.array_equal(a, b)


def test_create_rejects_bad_arguments_without_touching_a_device():
    from madronalib_b200 import api
    api.lib()
    for args in ((0, 48000.0, 2, 0, 1, 0), (-3, 48000.0, 2, 0, 1, 0), (4, 0.0, 2, 0, 1, 0), (4, -1.0, 2, 0, 1, 0),
                 (4, float("inf"), 2, 0, 1, 0), (4, float("nan"), 2, 0, 1, 0), (4, 48000.0, 0, 0, 0, 0),
                 (4, 48000.0, 2, 2, 1, 0), (4, 48000.0, 2, 0, -1, 0), (4, 48000.0, 2, 0, 1, 2)):
        with pytest.raises(api.MlbError) as e:
            api.FDTDBank(args[0], args[1], args[2], args[3], args[4], args[5])
        assert e.value.code == 1, args


def test_create_fails_loudly_without_a_device():
    from madronalib_b200 import api
    if api.device_count() > 0:
        pytest.skip("a GPU is visible here")
    with pytest.raises(api.MlbError) as e:
        api.FDTDBank(4)
    assert e.value.code == 3 and "no CPU fallback" in str(e.value)
