"""K9 on the GPU: the FDTD membrane bank (mlb_fdtd_*) bit for bit against the checkers -- the plain-C port, which
tests/test_fdtd.py pins to the reference's own example text, and that text itself (oracle/_ref/libmlfdtd.so) where it
was built -- in both floating-point modes."""
import ctypes
import hashlib
import os

import numpy as np
import pytest

from tests.common import assert_same_bits
from tests.test_fdtd import GOLDEN, noise_case

pytestmark = pytest.mark.gpu


def port(inp, state=None, ftz=False, **kw):
    from oracle.fdtd_bindings import port_fdtd
    return port_fdtd(inp, state, ftz=ftz, **kw)


def flags(api, ftz):
    return api.FDTDBank.FTZ if ftz else 0


@pytest.mark.parametrize("ftz", [False, True])
@pytest.mark.parametrize("T", [1, 5, 64])
@pytest.mark.parametrize("V", [1, 33, 4097])
def test_gpu_fdtd_bit_exact(gpu, V, T, ftz):
    inp = noise_case(V, T, seed=V * 7 + T)
    want, want_st = port(inp, ftz=ftz)
    b = gpu.FDTDBank(V, flags=flags(gpu, ftz))
    try:
        got = b.process_host(inp)
        st = b.get_state()
    finally:
        b.close()
    assert_same_bits(got, want, "V=%d T=%d ftz=%s" % (V, T, ftz))
    assert_same_bits(st, want_st, "state V=%d T=%d ftz=%s" % (V, T, ftz))


@pytest.mark.parametrize("ftz", [False, True])
def test_gpu_fdtd_subnormal(gpu, ftz):
    """Excitation around 1e-37: the surfaces cross the subnormal range many times."""
    inp = noise_case(33, 8, seed=11, amp=1e-37)
    want, want_st = port(inp, ftz=ftz)
    b = gpu.FDTDBank(33, flags=flags(gpu, ftz))
    try:
        got = b.process_host(inp)
        st = b.get_state()
    finally:
        b.close()
    assert_same_bits(got, want, "subnormal, ftz=%s" % ftz)
    assert_same_bits(st, want_st, "subnormal state, ftz=%s" % ftz)


@pytest.mark.parametrize("ftz", [False, True])
def test_gpu_fdtd_state_split_and_unstable(gpu, ftz):
    rng = np.random.default_rng(12)
    V = 37
    state = rng.uniform(-0.5, 0.5, (V, 2, 16, 16)).astype(np.float32)
    inp = noise_case(V, 12, seed=13)
    inp[:, 1, :5] = np.float32(0.12)  # five instances past the stable limit: inf / NaN
    want, want_st = port(inp, state, ftz=ftz)
    b = gpu.FDTDBank(V, flags=flags(gpu, ftz))
    try:
        b.set_state(state)
        assert np.array_equal(b.get_state().view(np.uint32), state.view(np.uint32))  # round trip
        got = np.concatenate([b.process_host(inp[:5]), b.process_host(inp[5:])])
        st = b.get_state()
        b.clear()
        assert not b.get_state().any()
    finally:
        b.close()
    assert_same_bits(got, want, "5 + 7 blocks from a random state")
    assert_same_bits(st, want_st, "state after 5 + 7 blocks")
    assert not np.isfinite(want[:, :, :5]).all()


def test_gpu_fdtd_input_planes(gpu):
    V, T = 19, 4
    base = noise_case(V, T, seed=14)
    inp = np.random.default_rng(15).standard_normal((T, 8, V, 64)).astype(np.float32)  # other planes: garbage
    inp[:, 3], inp[:, 6] = base[:, 0], base[:, 1]
    want, want_st = port(inp, ftz=True, excite_plane=3, freq_plane=6)
    want2, _ = port(base, ftz=True)
    assert_same_bits(want, want2, "port: planes 3 and 6 of 8")
    b = gpu.FDTDBank(V, in_planes=8, excite_plane=3, freq_plane=6, flags=gpu.FDTDBank.FTZ)
    try:
        got = b.process_host(inp)
        st = b.get_state()
    finally:
        b.close()
    assert_same_bits(got, want, "in_planes = 8")
    assert_same_bits(st, want_st, "in_planes = 8, state")


def test_gpu_fdtd_argument_errors(gpu):
    L = gpu.lib()
    h = ctypes.c_void_p()
    for args in ((0, 48000.0, 2, 0, 1, 0), (4, 0.0, 2, 0, 1, 0), (4, float("nan"), 2, 0, 1, 0),
                 (4, float("inf"), 2, 0, 1, 0), (4, 48000.0, 2, 2, 1, 0), (4, 48000.0, 2, 0, 2, 0),
                 (4, 48000.0, 0, 0, 0, 0), (4, 48000.0, 2, -1, 1, 0), (4, 48000.0, 2, 0, 1, 6)):
        assert L.mlb_fdtd_create(*args, ctypes.byref(h)) == 1, args
        assert L.mlb_last_error()
    assert L.mlb_fdtd_create(4, 48000.0, 2, 0, 1, 0, None) == 1
    b = gpu.FDTDBank(4)
    try:
        import torch
        x = torch.zeros((2, 2, 4, 64), device="cuda")
        y = torch.zeros((2, 2, 4, 64), device="cuda")
        hb = b._h
        assert L.mlb_fdtd_process_device(None, x.data_ptr(), y.data_ptr(), 2, None) == 1
        assert L.mlb_fdtd_process_device(hb, None, y.data_ptr(), 2, None) == 1
        assert L.mlb_fdtd_process_device(hb, x.data_ptr(), None, 2, None) == 1
        assert L.mlb_fdtd_process_device(hb, x.data_ptr(), y.data_ptr(), 0, None) == 1
        assert L.mlb_fdtd_process_device(hb, x.data_ptr(), y.data_ptr(), -1, None) == 1
        hx = np.zeros((2, 2, 4, 64), np.float32)
        assert L.mlb_fdtd_process_host(hb, None, hx.ctypes.data, 2) == 1
        assert L.mlb_fdtd_process_host(hb, hx.ctypes.data, None, 2) == 1
        assert L.mlb_fdtd_process_host(hb, hx.ctypes.data, hx.ctypes.data, 0) == 1
        assert L.mlb_fdtd_get_state(hb, None) == 1 and L.mlb_fdtd_set_state(hb, None) == 1
        assert L.mlb_fdtd_get_state(None, hx.ctypes.data) == 1 and L.mlb_fdtd_clear(None) == 1
        with pytest.raises(ValueError):
            b.process_host(np.zeros((2, 3, 4, 64), np.float32))
    finally:
        b.close()


def test_gpu_fdtd_one_launch_and_graph_capture(gpu):
    import torch
    V, T = 40, 6
    inp = noise_case(V, T, seed=16)
    st0 = np.random.default_rng(17).uniform(-0.3, 0.3, (V, 2, 16, 16)).astype(np.float32)
    b = gpu.FDTDBank(V, flags=gpu.FDTDBank.FTZ)
    try:
        x = torch.from_numpy(inp).cuda()
        y = torch.empty((T, 2, V, 64), device="cuda")
        b.set_state(st0)
        n0 = gpu.kernel_launches()
        b.process_device(x, y, T, stream=torch.cuda.current_stream().cuda_stream)
        assert gpu.kernel_launches() - n0 == 1
        torch.cuda.synchronize()
        direct, direct_st = y.cpu().numpy().copy(), b.get_state()

        g = torch.cuda.CUDAGraph()
        y.zero_()
        b.set_state(st0)
        with torch.cuda.graph(g):
            b.process_device(x, y, T, stream=torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        b.set_state(st0)
        g.replay()
        torch.cuda.synchronize()
        assert_same_bits(y.cpu().numpy(), direct, "graph replay vs direct call")
        assert_same_bits(b.get_state(), direct_st, "graph replay state")
    finally:
        b.close()
    want, _ = port(inp, st0, ftz=True)
    assert_same_bits(direct, want, "direct call vs port")


def test_gpu_fdtd_example_end_to_end(gpu):
    """The example itself: processFDTD's generators as a graph, whose output buffer is the bank's input with no copy,
    V = 3 identical instances, 800 vectors (three impulses); every instance equals the reference's own processFDTD."""
    import torch
    from madronalib_b200 import workloads as wl
    from oracle import fdtd_bindings as bindings
    V, T = 3, 800
    w = wl.fdtd_example(V)
    g = gpu.VoiceGraph(w.spec, V)
    b = gpu.FDTDBank(V, 48000.0, in_planes=2, excite_plane=0, freq_plane=1, flags=gpu.FDTDBank.FTZ)
    try:
        g.set_coefs(w.coef)
        g.set_state(w.state)
        rows = torch.empty((T, 2, V, 64), device="cuda")
        out = torch.empty((T, 2, V, 64), device="cuda")
        s = torch.cuda.current_stream().cuda_stream
        g.process_device(None, rows, None, T, stream=s)
        b.process_device(rows, out, T, stream=s)
        torch.cuda.synchronize()
        got = out.cpu().numpy()
    finally:
        g.close()
        b.close()
    gold = np.load(GOLDEN)
    want = bindings.RefFdtd().example(T) if bindings.fdtd_ref_available() else None
    for v in range(V):
        y = np.ascontiguousarray(got[:, :, v], "<f4")
        assert_same_bits(y[:16], gold["example_head"], "example head, instance %d" % v)
        assert hashlib.sha256(y.tobytes()).digest() == gold["example_sha256"].tobytes(), "instance %d" % v
        if want is not None:
            assert_same_bits(y, want, "example vs processFDTD, instance %d" % v)
    assert np.abs(got).max() > 0.1


def test_gpu_fdtd_full_size(gpu):
    """16 384 membranes x 64 vectors in FTZ mode against the compiled example text on all host threads (or the port
    where oracle/_ref was not built)."""
    from madronalib_b200 import workloads as wl
    from oracle import fdtd_bindings as bindings
    V, T = 16384, 64
    inp = wl.fdtd_inputs(V, T)
    if bindings.fdtd_ref_available():
        want, want_st, _ = bindings.RefFdtd().run(inp, ftz=True, nthreads=os.cpu_count() or 1)
    else:
        want, want_st = port(inp, ftz=True)
    b = gpu.FDTDBank(V, flags=gpu.FDTDBank.FTZ)
    try:
        got = b.process_host(inp)
        st = b.get_state()
    finally:
        b.close()
    assert_same_bits(got, want, "16384 x 64")
    assert_same_bits(st, want_st, "16384 x 64 state")
    assert np.abs(want).max() > 1e-3
