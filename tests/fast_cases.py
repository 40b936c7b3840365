"""The graphs fast mode is checked on, shared by tests/test_f64_graph.py (CPU) and tests/test_gpu_fast_mode.py.

One case per row of MLB_FUSED_LIST (madronalib_b200/csrc/mlb200.cu), plus config 4 (FM3 -> FDN8) and config 5 (the
256-node chain).  Every case starts from a warm state -- WARM blocks run through the port from the workload's own
start -- so that voices differ in phase and filter state, and its inputs continue from block WARM.
"""
from __future__ import annotations

import os
import re
from dataclasses import dataclass
from typing import Callable, Optional, Tuple

import numpy as np

from madronalib_b200 import api, workloads as wl
from madronalib_b200.graph import BLOCK, OP_NAME, GraphSpec

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WARM = 2


def fused_rows() -> list:
    """The (GEN, SRC, F1, F2, GAIN) rows of MLB_FUSED_LIST, as written in mlb200.cu."""
    with open(os.path.join(ROOT, "madronalib_b200", "csrc", "mlb200.cu")) as f:
        text = f.read()
    body = text[text.index("#define MLB_FUSED_LIST(X)"):text.index("static const FusedEntry g_fused[]")]
    return re.findall(r"X\(\s*(\w+)\s*,\s*(\w+)\s*,\s*(\w+)\s*,\s*(\w+)\s*,\s*(\w+)\s*\)", body)


def fused_name(row: Tuple[str, ...]) -> str:
    """The kernel name of a row's exact entry (`#G "+" #F1 "+" #F2 "+" #GN`); the fast entry adds "(fast)"."""
    g, _, f1, f2, gn = row
    return "fused:%s+%s+%s+%s" % (g, f1, f2, gn)


@dataclass
class Case:
    name: str
    make: Callable[[int], wl.Workload]       # n_voices -> workload (inputs(T, t0) continue in time)
    row: Optional[Tuple[str, ...]] = None    # the MLB_FUSED_LIST row that runs it, or None
    probe: Optional[int] = None              # coefficient word of the negative control (default: probe_slot)


def _noise_inputs(w: wl.Workload, seed: int, scale: float = 0.5) -> wl.Workload:
    """Seeded Gaussian audio on input plane 0, block by block, so that inputs(T, t0) continue in time."""
    V = w.n_voices

    def inputs(n_blocks, t0=0, v0=0, v1=None, out=None):
        x = np.empty((n_blocks, 1, V, BLOCK), np.float32)
        for t in range(n_blocks):
            x[t, 0] = np.random.default_rng(seed * 100003 + t0 + t).standard_normal((V, BLOCK)) * scale
        return np.ascontiguousarray(x[:, :, v0:v1])
    w.inputs = inputs  # type: ignore[assignment]
    return w


def _omega(V: int) -> np.ndarray:
    """The cutoffs of config 2's filters: 0.02 + 0.2 v / V."""
    return (np.float32(0.02) + np.float32(0.2) * np.arange(V, dtype=np.float32) / np.float32(V)).astype(np.float32)


def config_2(kind: str) -> Callable[[int], wl.Workload]:
    """Config 2 with each voice's sine at 0.5, 0.7, 1 or 1.4 times its filter's cutoff (cycling over the voices), with
    the workload's slow vibrato: the same conditioning at every bank size.  (At the workload's own 110 Hz a hipass
    far above its input leaves an output 1e-4 of its states, all rounding noise.)"""
    def make(V: int) -> wl.Workload:
        w = wl.config_2(kind, V)
        ratio = np.array([0.5, 0.7, 1.0, 1.4], np.float32)[np.arange(V) % 4]
        scale = (_omega(V) * ratio / wl.base_freq(V)).astype(np.float32)
        w.inputs = lambda n_blocks, t0=0, v0=0, v1=None, out=None: \
            wl.freq_rows(V, n_blocks, t0, v0, v1) * scale[v0:v1, None]  # type: ignore[assignment]
        return w
    return make


def spread_freq(V: int) -> np.ndarray:
    """0.002 .. 0.102 cycles per sample spread over the voices (golden-ratio steps), the same range at every size."""
    return (np.float32(0.002) + np.float32(0.1) * ((np.arange(V) * 0.6180339887) % 1.0).astype(np.float32))


def contract_s(V: int) -> wl.Workload:
    g = GraphSpec()
    s = g.node("SINE", g.param())
    g.output(g.node("MULTIPLY", g.node("LOPASS", s), g.param()))
    coef = g.new_coefs(V)
    coef[0] = spread_freq(V)
    coef[1:4] = api.coeffs_batch("lopass", _omega(V), 0.5)
    coef[4] = 0.1
    st = g.new_state(V)
    st[0] = wl.SINE_ZERO_PHASE
    return wl.Workload("contract_s", g, V, coef, st)


def bare_generator(op: str) -> Callable[[int], wl.Workload]:
    def make(V: int) -> wl.Workload:
        g = GraphSpec()
        g.output(g.node(op) if op == "NOISE" else g.node(op, g.input(0)))
        st = g.new_state(V)
        st[0] = np.arange(V, dtype=np.uint32) * np.uint32(2654435761)
        w = wl.Workload(op.lower(), g, V, g.new_coefs(V), st)
        if op != "NOISE":  # spread_freq with the workload's slow vibrato: up to six wraps (and polyBLEP
            # corrections) per block
            scale = (spread_freq(V) / wl.base_freq(V)).astype(np.float32)
            w.inputs = lambda n_blocks, t0=0, v0=0, v1=None, out=None: \
                wl.freq_rows(V, n_blocks, t0, v0, v1) * scale[v0:v1, None]  # type: ignore[assignment]
        return w
    return make


def noise_lopass_gain(V: int) -> wl.Workload:
    g = GraphSpec()
    g.output(g.node("MULTIPLY", g.node("LOPASS", g.node("NOISE")), g.param()))
    coef = g.new_coefs(V)
    coef[0:3] = api.coeffs_batch("lopass", _omega(V), 0.7)
    coef[3] = 0.25
    st = g.new_state(V)
    st[0] = np.arange(V, dtype=np.uint32)
    return wl.Workload("noise_lopass_gain", g, V, coef, st)


def bare_filter(op: str) -> Callable[[int], wl.Workload]:
    def make(V: int) -> wl.Workload:
        g = GraphSpec()
        g.output(g.node(op, g.input(0)))
        coef = g.new_coefs(V)
        if op == "LOPASS":
            coef[:] = api.coeffs_batch("lopass", _omega(V), 0.5)
        elif op == "ONEPOLE":
            coef[:] = api.coeffs_batch("onepole", _omega(V) * np.float32(0.25))
        else:
            table = np.array([api.coeffs_dcblocker(0.005 + 0.004 * k) for k in range(16)], np.float32)
            coef[0] = table[np.arange(V) % 16]
        return _noise_inputs(wl.Workload(op.lower(), g, V, coef, g.new_state(V)), seed=41)
    return make


def swept_param_sine(V: int) -> wl.Workload:
    """PARAM frequency -> SineGen -> Lopass with coefficient rows on input planes 0..2 -> gain."""
    g = GraphSpec()
    s = g.node("SINE", g.param())
    lp = g.node("LOPASS_V", s, g.input(0), g.input(1), g.input(2))
    g.output(g.node("MULTIPLY", lp, g.param()))
    coef = g.new_coefs(V)
    coef[0] = spread_freq(V)
    coef[1] = 0.1
    st = g.new_state(V)
    st[0] = wl.SINE_ZERO_PHASE
    w = wl.Workload("swept_param_sine", g, V, coef, st)

    def inputs(n_blocks, t0=0, v0=0, v1=None, out=None):
        om, k = wl.swept_omega_k(V, n_blocks, t0)
        rows = api.coeffs_lopass_vec(om, k)  # [T][V][3][64]
        return np.ascontiguousarray(rows.transpose(0, 2, 1, 3)[:, :, v0:v1])
    w.inputs = inputs  # type: ignore[assignment]
    return w


def _row(g, s, f1, f2, gn):
    return (g, s, f1, f2, gn)


N_ = "N_"
CASES = [
    Case("config_a", wl.config_a, _row("MLB_OP_SINE", "SRC_INPUT", "MLB_OP_LOPASS", N_, "true")),
    Case("contract_s", contract_s, _row("MLB_OP_SINE", "SRC_PARAM", "MLB_OP_LOPASS", N_, "true")),
] + [
    Case("config_2_" + k, config_2(k),
         _row("MLB_OP_SINE", "SRC_INPUT", "MLB_OP_" + k.upper(), N_, "false"))
    for k in ("lopass", "hipass", "bandpass", "loshelf", "hishelf", "bell")
] + [
    Case("config_3", wl.config_3, _row("MLB_OP_PHASOR", "SRC_INPUT", "MLB_OP_LOPASS", "MLB_OP_ONEPOLE",
                                                 "false")),
    Case("sine", bare_generator("SINE"), _row("MLB_OP_SINE", "SRC_INPUT", N_, N_, "false")),
    Case("phasor", bare_generator("PHASOR"), _row("MLB_OP_PHASOR", "SRC_INPUT", N_, N_, "false")),
    Case("saw", bare_generator("SAW"), _row("MLB_OP_SAW", "SRC_INPUT", N_, N_, "false")),
    Case("noise", bare_generator("NOISE"), _row("MLB_OP_NOISE", "SRC_NONE", N_, N_, "false")),
    Case("noise_lopass_gain", noise_lopass_gain, _row("MLB_OP_NOISE", "SRC_NONE", "MLB_OP_LOPASS", N_,
                                                                "true")),
    Case("lopass", bare_filter("LOPASS"), _row(N_, "SRC_INPUT", "MLB_OP_LOPASS", N_, "false")),
    Case("onepole", bare_filter("ONEPOLE"), _row(N_, "SRC_INPUT", "MLB_OP_ONEPOLE", N_, "false")),
    Case("dcblocker", bare_filter("DCBLOCKER"), _row(N_, "SRC_INPUT", "MLB_OP_DCBLOCKER", N_, "false")),
    Case("sine_lopass_v_gain", lambda V: wl.swept_filter_case("sine_lopass_v_gain", V),
         _row("MLB_OP_SINE", "SRC_INPUT", "MLB_OP_LOPASS_V", N_, "true")),
    Case("swept_param_sine", swept_param_sine, _row("MLB_OP_SINE", "SRC_PARAM", "MLB_OP_LOPASS_V", N_,
                                                             "true")),
    Case("lopass_v", lambda V: wl.swept_filter_case("lopass_v", V),
         _row(N_, "SRC_INPUT", "MLB_OP_LOPASS_V", N_, "false")),
    Case("fm3_fdn8", wl.config_4),
    # the last word is the last Lopass's g2, which the clamp / abs / lerp tail all but hides: probe the gain of the
    # 32 MULTIPLY nodes instead
    Case("chain256", lambda V: wl.config_5(V, 256), probe=0),
]
BY_NAME = {c.name: c for c in CASES}
FUSED = [c for c in CASES if c.row is not None]

# The bound of each case on the exact port's error against the float64 evaluator (f64_graph.rel_err of the outputs
# and f64_graph.state_err of the float state words): twice the largest value measured, over 40 and 97 voices and the
# sampled voices of the chain sizes of a 132-SM H100 (25 357 and 42 269 voices), 16 blocks after the warm-up; 130 and
# 200 voices for fm3_fdn8, 200 and 1024 voices x 4 blocks for chain256.  The measured maximum is in the comment.
BOUND = {
    "config_a": 1.2e-5,            # 5.77e-6 (state, 97 voices)
    "contract_s": 5.6e-6,          # 2.76e-6
    "config_2_lopass": 3.0e-6,     # 1.48e-6
    "config_2_hipass": 5.6e-6,     # 2.80e-6
    "config_2_bandpass": 1.9e-6,   # 9.48e-7
    "config_2_loshelf": 2.6e-6,    # 1.31e-6
    "config_2_hishelf": 3.8e-6,    # 1.87e-6
    "config_2_bell": 1.5e-6,       # 7.38e-7 (state)
    "config_3": 9.7e-6,            # 4.86e-6 (state)
    "sine": 1.2e-6,                # 5.58e-7
    "phasor": 6.1e-8,              # 3.05e-8
    "saw": 3.1e-5,                 # 1.53e-5
    "noise": 1e-12,                # 0: u * 2 - 3 is exact in binary32
    "noise_lopass_gain": 4.6e-7,   # 2.26e-7
    "lopass": 5.0e-7,              # 2.50e-7
    "onepole": 6.1e-7,             # 3.05e-7
    "dcblocker": 2.7e-6,           # 1.36e-6
    "sine_lopass_v_gain": 1.9e-5,  # 9.15e-6 (state)
    "swept_param_sine": 3.5e-6,    # 1.72e-6
    "lopass_v": 1.2e-6,            # 5.87e-7
    "fm3_fdn8": 9.4e-7,            # 4.70e-7
    "chain256": 3.9e-5,            # 1.94e-5 (state)
}
FLOOR = 2.0 ** -20  # fast mode may always be this far off, whatever the exact error
FAST_RATIO = 4.0    # err_fast <= max(FAST_RATIO * err_exact, FLOOR)


def fast_bound(err_exact: float) -> float:
    return max(FAST_RATIO * err_exact, FLOOR)


def chain_sizes(n_sms: int) -> Tuple[int, int, int]:
    """Bank sizes that reach the fused chain's launch regimes by size alone on a GPU with n_sms SMs: the team kernel
    (or one warp per group), between 4 and 8 groups per SM, and more than 8 groups per SM (the chunked grid)."""
    return 97, 32 * 6 * n_sms + 13, 32 * 10 * n_sms + 29


def sample_voices(V: int, n: int = 256) -> np.ndarray:
    """About n voices of a bank of V: voice 0, the last voice, both sides of 40 group boundaries, the rest at random."""
    if V <= n:
        return np.arange(V)
    G = (V + 31) // 32
    picks = {0, V - 1}
    for g in np.linspace(1, G - 1, 40).astype(np.int64):
        picks.update(v for v in (32 * int(g) - 1, 32 * int(g)) if v < V)
    rng = np.random.default_rng(V)
    while len(picks) < n:
        picks.add(int(rng.integers(V)))
    return np.array(sorted(picks), np.int64)


@dataclass
class Prepared:
    spec: GraphSpec
    V: int
    T: int
    coef: np.ndarray
    state: np.ndarray
    inp: Optional[np.ndarray]


def prepare(port, case: Case, V: int, T: int, voices: Optional[np.ndarray] = None) -> Prepared:
    """The case's workload at V voices, warmed for WARM blocks by the port, with T blocks of inputs after those;
    restricted to `voices` (a smaller bank of the same voices) when given."""
    w = case.make(V)
    spec = w.spec
    sl = slice(None) if voices is None else voices
    coef = np.ascontiguousarray(w.coef[:, sl])
    state = np.ascontiguousarray(w.state[:, sl])
    warm = w.inputs(WARM + T) if spec.n_in else None
    if warm is not None:
        warm = np.ascontiguousarray(warm[:, :, sl])
    n = coef.shape[1]
    _, _, state = port.run(spec, n, WARM, None if warm is None else np.ascontiguousarray(warm[:WARM]), state, coef,
                           want_out=False, nthreads=8)
    inp = None if warm is None else np.ascontiguousarray(warm[WARM:])
    return Prepared(spec, n, T, coef, state, inp)


def probe_slot(case: Case, spec: GraphSpec) -> Optional[int]:
    """The coefficient word the negative control scales: the case's own choice, else the last one that is not an FDN
    delay length (a length is truncated to an integer, so a small scaling need not change it); None when the graph
    has none."""
    if case.probe is not None:
        return case.probe
    co_off = spec.offsets()[1]
    skip = set()
    for i, op in enumerate(spec.ops):
        if OP_NAME[op] == "FDN8":
            skip.update(range(co_off[i] + 24, co_off[i] + 32))
    slots = [s for s in range(spec.n_coef) if s not in skip]
    return slots[-1] if slots else None

