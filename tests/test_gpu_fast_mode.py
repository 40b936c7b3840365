"""Fast mode (MLB_GRAPH_FAST) against the float64 evaluator, for every kernel family that has a fast instance.

Every case runs one graph, state and input twice, exactly and with FLAG_FAST, and measures both against
tests/f64_graph.py.  The contract: the kernel names are the exact one and the same ending in "(fast)"; the exact run
stays within its case's bound (pinned on the CPU by test_f64_graph.py); err_fast <= max(4 * err_exact, 2^-20), for
the output rows and for the float state words; and where a recurrence is written with an explicit FMA in fast mode,
the fast bits really differ from the exact ones.  Runs go through mlb_graph_process_device, one launch per call, so
that the bank size alone picks the fused chain's launch regime."""
import numpy as np
import pytest

from tests import f64_graph as fg
from tests import fast_cases as fc

pytestmark = pytest.mark.gpu

T = 16
EPS32 = 2.0 ** -24
# filters whose fast recurrence is an explicit fmaf (A<false>::mul_add_mul / mad in ops.cuh): their fast bits differ
FMA_OPS = {"LOPASS", "HIPASS", "BANDPASS", "LOSHELF", "HISHELF", "BELL", "ONEPOLE", "LOPASS_V", "FDN8"}


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def run_device(gpu, p, flags, splits, want_mix=False):
    """Run a prepared case through mlb_graph_process_device, one call per entry of `splits`."""
    import torch
    dev = torch.device("cuda", 0)
    g = gpu.VoiceGraph(p.spec, p.V, flags)
    try:
        g.set_coefs(p.coef)
        g.set_state(p.state)
        stream = torch.cuda.current_stream().cuda_stream
        outs, mixes, t0 = [], [], 0
        for n in splits:
            d_in = None if p.inp is None else torch.from_numpy(np.ascontiguousarray(p.inp[t0:t0 + n])).to(dev)
            d_out = torch.empty((n, p.spec.n_out, p.V, 64), dtype=torch.float32, device=dev)
            d_mix = torch.zeros((n, p.spec.n_out, 64), dtype=torch.float32, device=dev) if want_mix else None
            g.process_device(d_in, d_out, d_mix, n, stream)
            torch.cuda.synchronize()
            outs.append(d_out.cpu().numpy())
            mixes.append(None if d_mix is None else d_mix.cpu().numpy())
            t0 += n
        assert t0 == p.T
        st, name = g.get_state(), g.kernel_name
    finally:
        g.close()
    return np.concatenate(outs), (np.concatenate(mixes) if want_mix else None), st, name


def judge(what, p, exact, fast, voices, bound):
    """Both runs against the evaluator on `voices`; returns (err_exact, err_fast) of the outputs."""
    r = fg.evaluate(p.spec, p.V, p.T, p.inp, p.state, p.coef, voices)
    (eo, _, es, _), (fo, _, fs, _) = exact, fast
    e_ex, e_fa = fg.rel_err(eo[:, :, voices], r.out), fg.rel_err(fo[:, :, voices], r.out)
    s_ex, s_fa = fg.state_err(es[:, voices], r, p.spec), fg.state_err(fs[:, voices], r, p.spec)
    print(f"fast-mode {what}: err_exact {e_ex:.3e} err_fast {e_fa:.3e} ratio {e_fa / max(e_ex, 1e-30):.2f} | "
          f"state exact {s_ex:.3e} fast {s_fa:.3e}")
    assert e_ex < bound and s_ex < bound, (what, e_ex, s_ex, bound)
    assert e_fa <= fc.fast_bound(e_ex), (what, e_fa, e_ex)
    assert s_fa <= fc.fast_bound(s_ex), (what, s_fa, s_ex)
    return e_ex, e_fa


def _has_fma_filter(spec):
    from madronalib_b200.graph import OP_NAME
    return any(OP_NAME[op] in FMA_OPS for op in spec.ops)


def _pair(gpu, p, flags, splits, want_mix=False):
    return (run_device(gpu, p, flags, splits, want_mix),
            run_device(gpu, p, flags | gpu.FLAG_FAST, splits, want_mix))


@pytest.mark.parametrize("size", [0, 1, 2])
@pytest.mark.parametrize("name", [c.name for c in fc.FUSED])
def test_fused_entry_fast(gpu, port, name, size):
    """Every fast fused entry at 97 voices (the team kernel where the chain has one), at 32 * 6 * SMs + 13 voices
    (one warp per group; the four-plane swept chains already take the chunked grid) and at 32 * 10 * SMs + 29
    voices (the chunked persistent grid; one unsplit call of 16 blocks is cut into time chunks)."""
    case = fc.BY_NAME[name]
    V = fc.chain_sizes(_sms())[size]
    splits = (5, 11) if size < 2 else (T,)
    p = fc.prepare(port, case, V, T)
    exact, fast = _pair(gpu, p, 0, splits)
    want = fc.fused_name(case.row)
    assert exact[3] == want and fast[3] == want + "(fast)", (exact[3], fast[3])
    judge(f"{name} V={V}", p, exact, fast, fc.sample_voices(V), fc.BOUND[name])
    ints = fg.int_slots(p.spec)
    assert np.array_equal(fast[2][ints], exact[2][ints]), "integer state words differ between fast and exact"
    if _has_fma_filter(p.spec):
        assert not np.array_equal(fast[0], exact[0]), "fast bits equal the exact bits: the fast instance did not run"


@pytest.mark.parametrize("size", [1, 2])
def test_mix_bus_fast(gpu, port, size):
    """Config A's mix bus in both modes against the float64 sum of the float64 rows of all voices:
    |mix - sum y64| <= (V - 1) eps sum |y| + sum |y - y64|, sample by sample."""
    V = fc.chain_sizes(_sms())[size]
    p = fc.prepare(port, fc.BY_NAME["config_a"], V, T)
    r = fg.evaluate(p.spec, V, T, p.inp, p.state, p.coef)
    for flags in (0, gpu.FLAG_FAST):
        out, mix, _, name = run_device(gpu, p, flags, (T,), want_mix=True)
        y = out.astype(np.float64)
        tol = (V - 1) * EPS32 * np.abs(y).sum(axis=2) + np.abs(y - r.out).sum(axis=2)
        err = np.abs(mix - r.mix)
        print(f"fast-mode mix {name} V={V}: max |mix - sum y64| {err.max():.3e}, at most {(err / tol).max():.3f} "
              f"of its bound")
        assert (err <= tol).all(), (name, float(err.max()))


def test_fm3_fdn8_fast(gpu, port):
    """FM3 -> FDN8 on its fused kernel and on the interpreter, fast against exact, 130 voices, two calls (the ring
    write index carries across)."""
    case = fc.BY_NAME["fm3_fdn8"]
    p = fc.prepare(port, case, 130, 14)
    for flags, kind in ((0, "fused:fm3_fdn8"), (gpu.FLAG_FORCE_GENERIC, "generic")):
        exact, fast = _pair(gpu, p, flags, (5, 9))
        assert exact[3].startswith(kind) and fast[3] == exact[3].replace(kind, kind + "(fast)", 1), (exact[3], fast[3])
        judge(f"fm3_fdn8 {exact[3]}", p, exact, fast, np.arange(p.V), fc.BOUND["fm3_fdn8"])
        assert not np.array_equal(fast[0], exact[0])
        assert np.abs(exact[0]).max() > 0.1  # the reverb tail is there


@pytest.mark.parametrize("name", ["config_a", "config_2_lopass", "config_2_hipass", "config_2_bandpass",
                                  "config_2_loshelf", "config_2_hishelf", "config_2_bell", "config_3", "lopass_v",
                                  "chain256"])
def test_interpreter_fast(gpu, port, name):
    """The graph interpreter's fast instance (FLAG_FAST | FLAG_FORCE_GENERIC); config 5 at 1024 voices x 4 blocks on
    its default multi-stage pipeline."""
    case = fc.BY_NAME[name]
    if name == "chain256":
        p, splits = fc.prepare(port, case, 1024, 4), (4,)
    else:
        p, splits = fc.prepare(port, case, 200, T), (5, 11)
    exact, fast = _pair(gpu, p, gpu.FLAG_FORCE_GENERIC, splits)
    assert exact[3].startswith("generic[") and fast[3] == exact[3].replace("generic", "generic(fast)", 1), \
        (exact[3], fast[3])
    judge(f"interpreter {name} V={p.V}", p, exact, fast, fc.sample_voices(p.V), fc.BOUND[name])
    ints = fg.int_slots(p.spec)
    assert np.array_equal(fast[2][ints], exact[2][ints])
    assert not np.array_equal(fast[0], exact[0]), "fast bits equal the exact bits: the fast instance did not run"
