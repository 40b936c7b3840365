"""Synthetic workloads for the BASELINE.json configurations (SURVEY.md section 8d).

Deterministic formulas only (no RNG except NoiseGen's own LCG).  Coefficients come from
the library's host-side ``mlb_coeffs_*`` (glibc libm, the same calls as the reference's
``makeCoeffs``); tests check those against both oracles.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import numpy as np

from . import api
from .graph import (BLOCK, OP_ID, SINE_ZERO_PHASE, GraphSpec, graph_chain256, graph_fm3_fdn8,
                    graph_phasor_lopass_onepole, graph_sine_lopass_gain, graph_sine_svf)

SR = 48000.0


@dataclass
class Workload:
    name: str
    spec: GraphSpec
    n_voices: int
    coef: np.ndarray   # [n_coef][V] f32
    state: np.ndarray  # [n_state][V] u32

    def inputs(self, n_blocks: int, t0: int = 0, v0: int = 0, v1: Optional[int] = None,
               out: Optional[np.ndarray] = None) -> Optional[np.ndarray]:
        """Contract R input planes [T][n_in][V'][64] for voices [v0, v1), blocks [t0, t0+T)."""
        if self.spec.n_in == 0:
            return None
        v1 = self.n_voices if v1 is None else v1
        return freq_rows(self.n_voices, n_blocks, t0, v0, v1, out)

    def shard(self, rank: int, world: int) -> "Workload":
        """Contiguous voice range [rank*V/world, (rank+1)*V/world) (SURVEY 8e)."""
        v0, v1 = self.n_voices * rank // world, self.n_voices * (rank + 1) // world
        w = Workload(self.name, self.spec, v1 - v0, np.ascontiguousarray(self.coef[:, v0:v1]),
                     np.ascontiguousarray(self.state[:, v0:v1]))
        w._v0, w._V = v0, self.n_voices  # type: ignore[attr-defined]
        return w


def base_freq(n_voices: int, v0: int = 0, v1: Optional[int] = None) -> np.ndarray:
    """f_v = (110 + 0.25 v) / 48000 cycles per sample (max 0.344 at V = 65536)."""
    v1 = n_voices if v1 is None else v1
    v = np.arange(v0, v1, dtype=np.float32)
    return ((np.float32(110.0) + np.float32(0.25) * v) / np.float32(SR)).astype(np.float32)


def freq_rows(n_voices: int, n_blocks: int, t0: int = 0, v0: int = 0, v1: Optional[int] = None,
              out: Optional[np.ndarray] = None) -> np.ndarray:
    """Time-varying per-voice frequency rows (SURVEY 8d, contract R):
    freq_v[n] = f_v * (1 + 0.002 * tri(((n*7 + v*13) mod 512) / 512)), n = absolute sample index,
    tri = 0..1..0 triangle.  Shape [T][1][V'][64] f32."""
    v1 = n_voices if v1 is None else v1
    nv = v1 - v0
    if out is None:
        out = np.empty((n_blocks, 1, nv, BLOCK), np.float32)
    f = base_freq(n_voices, v0, v1)[:, None]
    vv = (np.arange(v0, v1, dtype=np.int64) * 13)[:, None]
    for t in range(n_blocks):
        n = (np.arange(BLOCK, dtype=np.int64) + (t0 + t) * BLOCK)[None, :] * 7
        ph = ((n + vv) % 512).astype(np.float32) / np.float32(512.0)
        tri = np.float32(1.0) - np.abs(np.float32(2.0) * ph - np.float32(1.0))
        out[t, 0] = f * (np.float32(1.0) + np.float32(0.002) * tri)
    return out


def _set(coef: np.ndarray, spec: GraphSpec, node: int, values) -> None:
    values = np.asarray(values, np.float32)
    base = spec.coef_slot(node)
    if values.ndim == 1:
        values = values[:, None]
    coef[base:base + values.shape[0]] = values


def _svf_coefs(kind: str, n_voices: int) -> np.ndarray:
    """omega_v = 0.02 + 0.2 v/V, k = 0.5 (Bell/shelves: A = dBToGain(6)); [n_coef][V]."""
    v = np.arange(n_voices, dtype=np.float32)
    omega = np.float32(0.02) + np.float32(0.2) * v / np.float32(n_voices)
    if kind in ("lopass", "hipass", "bandpass"):
        return api.coeffs_batch(kind, omega, 0.5)
    return api.coeffs_batch(kind, omega, 0.5, api.db_to_gain(6.0))


def config_a(n_voices: int = 65536, gain: float = 0.1) -> Workload:
    """Headline: SineGen.clear() -> Lopass(fixed coeffs) -> gain (also config 1 at V=1)."""
    spec = graph_sine_lopass_gain()
    coef = spec.new_coefs(n_voices)
    _set(coef, spec, 2, _svf_coefs("lopass", n_voices))
    coef[spec.coef_slot(3)] = np.float32(gain)
    state = spec.new_state(n_voices)
    state[spec.state_slot(1)] = SINE_ZERO_PHASE
    return Workload("sine_lopass_gain", spec, n_voices, coef, state)


def config_1() -> Workload:
    """Plumbing: 1 voice, freq 440/48000 constant, Lopass::makeCoeffs(0.1, 1.0), gain 0.5."""
    w = config_a(1, gain=0.5)
    _set(w.coef, w.spec, 2, api.coeffs("lopass", 0.1, 1.0))
    w.name = "config1"
    w.inputs = lambda n_blocks, t0=0, v0=0, v1=None, out=None: np.full(  # type: ignore[assignment]
        (n_blocks, 1, 1, BLOCK), np.float32(440.0) / np.float32(48000.0), np.float32)
    return w


def config_2(kind: str = "lopass", n_voices: int = 4096) -> Workload:
    """SineGen -> SVF ("Biquad" stand-in, SURVEY D2)."""
    spec = graph_sine_svf(kind)
    coef = spec.new_coefs(n_voices)
    _set(coef, spec, 2, _svf_coefs(kind, n_voices))
    state = spec.new_state(n_voices)
    state[spec.state_slot(1)] = SINE_ZERO_PHASE
    return Workload("sine_" + kind, spec, n_voices, coef, state)


def config_3(n_voices: int = 65536) -> Workload:
    """PhasorGen.clear(0) -> Lopass -> OnePole(0.001 + 0.01 v/V)."""
    spec = graph_phasor_lopass_onepole()
    coef = spec.new_coefs(n_voices)
    _set(coef, spec, 2, _svf_coefs("lopass", n_voices))
    vv = np.arange(n_voices, dtype=np.float32)
    om = np.float32(0.001) + np.float32(0.01) * vv / np.float32(n_voices)
    _set(coef, spec, 3, api.coeffs_batch("onepole", om))
    return Workload("phasor_lopass_onepole", spec, n_voices, coef, spec.new_state(n_voices))


FDN_TIMES = np.array([67, 73, 91, 103, 127, 151, 173, 199], np.float32)
FDN_CUTOFFS = np.array([0.1, 0.2, 0.3, 0.4, 0.1, 0.2, 0.3, 0.4], np.float32)


def config_4(n_voices: int = 16384) -> Workload:
    """3-op FM (r1=2, r2=3.5, i1=0.3, i2=0.1) -> FDN<8>, delays {67..199}+64*(v mod 8),
    cutoffs {0.1,0.2,0.3,0.4}x2, feedback 0.5, stereo out."""
    spec = graph_fm3_fdn8()
    coef = spec.new_coefs(n_voices)
    for node, val in zip(range(1, 6), (2.0, 3.5, 0.3, 0.1, 1.0)):
        coef[spec.coef_slot(node)] = np.float32(val)
    fdn = spec.ops.index(OP_ID["FDN8"])
    gains = np.full(8, 0.5, np.float32)
    per = [api.coeffs_fdn8(FDN_TIMES + np.float32(64 * m), FDN_CUTOFFS, gains) for m in range(8)]
    block = np.stack([per[v % 8] for v in range(n_voices)], axis=1)  # [32][V]
    _set(coef, spec, fdn, block)
    state = spec.new_state(n_voices)
    for i, op in enumerate(spec.ops):
        if op == OP_ID["SINE"]:
            state[spec.state_slot(i)] = SINE_ZERO_PHASE
    w = Workload("fm3_fdn8", spec, n_voices, coef, state)
    w.inputs = lambda n_blocks, t0=0, v0=0, v1=None, out=None: np.ascontiguousarray(  # type: ignore
        np.broadcast_to(base_freq(n_voices, v0, v1)[None, None, :, None],
                        (n_blocks, 1, (n_voices if v1 is None else v1) - v0, BLOCK)))
    return w


def fdn_case(size: int, n_voices: int = 40):
    """FDN<size> written out with IntegerDelay / OnePole / feedback-edge nodes (graph.graph_fdn): per-voice delay
    times, cutoffs and gains; a noise burst in.  Returns (workload, times [size][V], cutoffs [size], gains [size])."""
    from .graph import graph_fdn
    V = n_voices
    g, idx = graph_fdn(size)
    coef, state = g.new_coefs(V), g.new_state(V)
    base = np.array([67, 73, 91, 103, 127, 149, 173, 199, 211, 233, 257, 281, 307, 331, 353, 379], np.float32)[:size]
    times = base[:, None] + np.float32(37.0) * (np.arange(V, dtype=np.float32) % 5)[None, :]      # [size][V]
    cutoffs = (np.float32(0.08) + np.float32(0.05) * (np.arange(size, dtype=np.float32) % 5)).astype(np.float32)
    gains = (np.float32(0.55) - np.float32(0.01) * np.arange(size, dtype=np.float32)).astype(np.float32)
    coef[g.coef_slot(idx["zero"][0])] = np.float32(0.0)
    coef[g.coef_slot(idx["k"][0])] = np.float32(2.0) / np.float32(size)
    for n in range(size):
        length = np.maximum(1, (times[n] - np.float32(BLOCK)).astype(np.int32)).astype(np.float32)  # FDN::setDelaysInSamples
        coef[g.coef_slot(idx["delay"][n])] = length         # IntegerDelay::setDelayInSamples(len)
        coef[g.coef_slot(idx["delay"][n], 1)] = length      # ... sized for exactly that delay (SURVEY D7 shim)
        _set(coef, g, idx["filter"][n], np.repeat(api.coeffs("onepole", float(cutoffs[n]))[:, None], V, 1))
        coef[g.coef_slot(idx["gain"][n])] = gains[n]
    w = Workload("fdn%d" % size, g, V, coef, state)
    noise = _noise_rows(31 + size, V, 0.5)

    def fn(T, t0=0, v0=0, v1=None, out=None):
        x = noise(T, t0)
        x[6:] = 0  # a burst, then the tail
        return x
    w.inputs = fn  # type: ignore[assignment]
    return w, times, cutoffs, gains


def config_5(n_instances: int = 1024, n_nodes: int = 256) -> Workload:
    """256-node chain cycling 8 node kinds, fed by NoiseGen seeded with the instance index."""
    spec = graph_chain256(n_nodes)
    coef = spec.new_coefs(n_instances)
    for node, val in zip(range(5), (0.999, 1e-3, -1.0, 1.0, 0.5)):
        coef[spec.coef_slot(node)] = np.float32(val)
    c_op, c_lp = api.coeffs("onepole", 0.01), api.coeffs("lopass", 0.1, 1.0)
    for i, op in enumerate(spec.ops):
        if op == OP_ID["ONEPOLE"]:
            _set(coef, spec, i, np.repeat(c_op[:, None], n_instances, 1))
        elif op == OP_ID["LOPASS"]:
            _set(coef, spec, i, np.repeat(c_lp[:, None], n_instances, 1))
    state = spec.new_state(n_instances)
    state[spec.state_slot(spec.ops.index(OP_ID["NOISE"]))] = np.arange(n_instances, dtype=np.uint32)
    return Workload("chain%d" % n_nodes, spec, n_instances, coef, state)


# ---- SURVEY 8(f) row 2: one small workload per functor of the rest of the L2 set ----

def _rows_inputs(fn):
    """Wrap fn(T, t0) -> [T][n_in][V][64] into the Workload.inputs signature (voice slicing included)."""
    def inputs(n_blocks, t0=0, v0=0, v1=None, out=None):
        x = fn(n_blocks, t0)
        return np.ascontiguousarray(x[:, :, v0:v1])
    return inputs


def _noise_rows(seed: int, n_voices: int, scale: float = 1.0):
    def fn(T, t0):
        out = np.empty((T, 1, n_voices, BLOCK), np.float32)
        for t in range(T):
            rng = np.random.default_rng(seed * 100003 + t0 + t)
            out[t, 0] = (rng.standard_normal((n_voices, BLOCK)) * scale).astype(np.float32)
        return out
    return fn


def functor_case(name: str, n_voices: int = 40) -> Workload:
    """name in FUNCTOR_CASES.  Inputs are seeded noise / gates / slowly moving delay times."""
    V = n_voices
    g = GraphSpec()
    vv = np.arange(V, dtype=np.float32)
    noise = _noise_rows(11, V)

    def two_planes(a, b):
        return lambda T, t0: np.concatenate([a(T, t0), b(T, t0)], axis=1)

    def delay_rows(lo, hi, rate):
        # per-voice triangle sweep of the delay time between lo and hi samples
        def fn(T, t0):
            n = (np.arange(T * BLOCK, dtype=np.float64) + t0 * BLOCK)[None, :]
            ph = (n * rate * (1.0 + 0.01 * vv[:, None].astype(np.float64)) + 0.37 * vv[:, None]) % 1.0
            tri = 1.0 - np.abs(2.0 * ph - 1.0)
            d = (lo + (hi - lo) * tri).astype(np.float32)              # [V][T*64]
            return np.ascontiguousarray(d.reshape(V, T, BLOCK).transpose(1, 0, 2))[:, None]
        return fn

    if name == "impulse":
        y = g.node("IMPULSE", g.input(0))
        g.output(y)
        coef, state = g.new_coefs(V), g.new_state(V)
        fn = lambda T, t0: np.broadcast_to(((1.0 + vv) / np.float32(150.0)).astype(np.float32)[None, None, :, None],
                                           (T, 1, V, BLOCK)).copy()
    elif name == "oneshot":
        y = g.node("ONESHOT", g.input(0))
        g.output(y)
        coef, state = g.new_coefs(V), g.new_state(V)
        state[1, ::2] = 1  # every other voice triggered (mGate = 1)
        fn = lambda T, t0: np.broadcast_to(((1.0 + vv) / np.float32(300.0)).astype(np.float32)[None, None, :, None],
                                           (T, 1, V, BLOCK)).copy()
    elif name in ("peak", "rms"):
        y = g.node(name.upper(), g.input(0))
        g.output(y)
        coef, state = g.new_coefs(V), g.new_state(V)
        for v in range(V):
            c = api.coeffs(name, 0.0005 + 0.001 * v)
            coef[0:2, v] = c
        if name == "peak":
            coef[2] = np.float32(100 + 7 * np.arange(V))

        def fn(T, t0):  # bursts: noise gated by a slow square so that the hold/decay paths both run
            x = noise(T, t0)
            n = (np.arange(T * BLOCK) + t0 * BLOCK).reshape(T, 1, 1, BLOCK)
            return (x * ((n // 150) % 3 == 0)).astype(np.float32)
    elif name == "adsr":
        y = g.node("ADSR", g.input(0))
        g.output(y)
        coef, state = g.new_coefs(V), g.new_state(V)
        for v in range(V):
            coef[:, v] = api.coeffs("adsr", 0.0005 + 0.0001 * v, 0.001 + 0.0002 * v, 0.25 + 0.5 * v / V,
                                    0.002, SR)

        def fn(T, t0):  # gate: amplitude 0.5+v/V while ((n + 17 v) mod 700) < 400, else 0
            n = (np.arange(T * BLOCK) + t0 * BLOCK).reshape(T, 1, 1, BLOCK)
            on = ((n + 17 * np.arange(V).reshape(1, 1, V, 1)) % 700) < 400
            amp = (np.float32(0.5) + vv / np.float32(V)).reshape(1, 1, V, 1)
            return (on * amp).astype(np.float32)
    elif name == "allpass1":
        y = g.node("ALLPASS1", g.input(0))
        g.output(y)
        coef, state = g.new_coefs(V), g.new_state(V)
        coef[0] = [api.coeffs_allpass1(0.618 + v / V) for v in range(V)]
        fn = noise
    elif name in ("glide", "interpolator1", "sample_glide"):
        y = g.node(name.upper(), g.input(0))
        g.output(y)
        coef, state = g.new_coefs(V), g.new_state(V)
        if name == "glide":
            for v in range(V):
                coef[:, v] = api.coeffs("glide", 64.0 * (1 + v % 5))
        if name == "sample_glide":
            for v in range(V):
                coef[:, v] = api.coeffs("sample_glide", 10.0 + 13 * v)

        def fn(T, t0):  # a staircase: the target moves every (3 + v mod 4) blocks (every 90 samples for sample_glide)
            out = np.empty((T, 1, V, BLOCK), np.float32)
            for t in range(T):
                if name == "sample_glide":
                    n = (np.arange(BLOCK) + (t0 + t) * BLOCK)[None, :]
                    out[t, 0] = (((n // 90 + np.arange(V)[:, None]) * 37 % 11) / np.float32(11.0)).astype(np.float32)
                else:
                    step = (t0 + t) // (3 + np.arange(V) % 4)
                    out[t, 0] = (((step * 29 + np.arange(V)) % 13) / np.float32(13.0)).astype(np.float32)[:, None]
            return out
    elif name == "integer_delay":
        y = g.node("INTEGER_DELAY", g.input(0))
        g.output(y)
        coef, state = g.new_coefs(V), g.new_state(V)
        coef[0] = np.float32((np.arange(V) * 23) % 301)
        coef[1] = np.float32(300 + (np.arange(V) % 3) * 400)   # rings of 512 / 1024 / 2048 samples
        fn = noise
    elif name == "integer_delay_var":
        y = g.node("INTEGER_DELAY_VAR", g.input(0), g.input(1))
        g.output(y)
        coef, state = g.new_coefs(V), g.new_state(V)
        coef[0] = np.float32(500)
        fn = two_planes(noise, delay_rows(0.0, 500.0, 1.0 / 900.0))
    elif name == "fractional_delay":
        y = g.node("FRACTIONAL_DELAY", g.input(0))
        g.output(y)
        coef, state = g.new_coefs(V), g.new_state(V)
        coef[0] = (np.float32(0.3) + vv * np.float32(7.77)).astype(np.float32)
        coef[1] = np.float32(400)
        fn = noise
    elif name in ("fractional_delay_var", "pitchbend_delay"):
        y = g.node(name.upper(), g.input(0), g.input(1))
        g.output(y)
        coef, state = g.new_coefs(V), g.new_state(V)
        coef[0] = np.float32(1000)
        fn = two_planes(noise, delay_rows(0.0, 1000.0, 1.0 / 5000.0))
    elif name in ("allpass_int", "allpass_frac"):
        y = g.node(name.upper(), g.input(0))
        g.output(y)
        coef, state = g.new_coefs(V), g.new_state(V)
        coef[0] = (np.float32(0.3) + np.float32(0.5) * vv / np.float32(V)).astype(np.float32)
        coef[1] = (np.float32(64.0) + vv * np.float32(11.37)).astype(np.float32)
        coef[2] = np.float32(64 + 12 * V)
        fn = noise
    elif name == "allpass_pb":
        y = g.node("ALLPASS_PB", g.input(0), g.input(1))
        g.output(y)
        coef, state = g.new_coefs(V), g.new_state(V)
        coef[0] = (np.float32(0.3) + np.float32(0.5) * vv / np.float32(V)).astype(np.float32)
        coef[1] = np.float32(1000)
        fn = two_planes(noise, delay_rows(64.0, 1000.0, 1.0 / 5000.0))
    elif name in ("halfband_up", "halfband_roundtrip", "upsample2x_clip"):
        # up: both 2x rows out; roundtrip: down(up(x)); upsample2x_clip: Upsample2xFunction with the
        # stateless fn(v) = clamp(v * drive, -1, 1) (MLDSPFunctional.h:114-160)
        x = g.input(0)
        up1 = g.node("HALFBAND_UP", x)
        up2 = g.node("HALFBAND_UP_2", up1)
        if name == "halfband_up":
            g.output(up1, up2)
        elif name == "halfband_roundtrip":
            g.output(g.node("HALFBAND_DOWN", up1, up2))
        else:
            drive, lo, hi = g.param(), g.param(), g.param()
            f1 = g.node("CLAMP", g.node("MULTIPLY", up1, drive), lo, hi)
            f2 = g.node("CLAMP", g.node("MULTIPLY", up2, drive), lo, hi)
            g.output(g.node("HALFBAND_DOWN", f1, f2))
        coef, state = g.new_coefs(V), g.new_state(V)
        if name == "upsample2x_clip":
            coef[0] = (np.float32(0.5) + vv / np.float32(V) * np.float32(3.0)).astype(np.float32)
            coef[1], coef[2] = np.float32(-1.0), np.float32(1.0)
        fn = noise
    elif name == "upsample2x_osc":
        # Upsample2xFunction<1> with a STATEFUL process function, fn(v) = lp(osc(v * 0.5)): the SineGen and the
        # Lopass are called twice per vector (MLB_AGAIN), as in the reference's tutorial
        # (examples/tutorial/dspOpsExample.cpp:100-102 wraps a sine generator this way)
        x = g.input(0)
        up1 = g.node("HALFBAND_UP", x)
        up2 = g.node("HALFBAND_UP_2", up1)
        half = g.param()
        s1 = g.node("SINE", g.node("MULTIPLY", up1, half))
        l1 = g.node("LOPASS", s1)
        s2 = g.again(s1, g.node("MULTIPLY", up2, half))
        l2 = g.again(l1, s2)
        g.output(g.node("HALFBAND_DOWN", l1, l2))
        coef, state = g.new_coefs(V), g.new_state(V)
        coef[g.coef_slot(half)] = np.float32(0.5)
        _set(coef, g, l1, _svf_coefs("lopass", V))
        state[g.state_slot(s1)] = SINE_ZERO_PHASE
        fn = lambda T, t0: freq_rows(V, T, t0, 0, V)
    elif name == "downsample2x_clip":
        # Downsample2xFunction with the stateless fn(v) = clamp(v * drive, -1, 1) (MLDSPFunctional.h:166-223)
        x = g.input(0)
        drive, lo, hi = g.param(), g.param(), g.param()
        half = g.node("DOWN2X_IN", x)
        f = g.node("CLAMP", g.node("MULTIPLY", half, drive), lo, hi)
        g.output(g.node("DOWN2X_OUT", f))
        coef, state = g.new_coefs(V), g.new_state(V)
        coef[0] = (np.float32(0.5) + vv / np.float32(V) * np.float32(3.0)).astype(np.float32)
        coef[1], coef[2] = np.float32(-1.0), np.float32(1.0)
        fn = noise
    elif name == "tempo_lock":
        # input clock phasor (PhasorGen) -> TempoLock at ratio dydx_v; a few voices start stopped (-1)
        # plane 1 is a bit mask: all-ones rows replace the clock by -1 ("stopped", F:1503-1507) for a
        # block now and then, so the stop and restart paths run too
        f, mask = g.input(0), g.input(1)
        ph = g.node("PHASOR", f)
        ratio, minus_one = g.param(), g.param()
        clock = g.node("SELECT", minus_one, ph, mask)
        tl = g.node("TEMPO_LOCK", clock, ratio)
        g.output(tl)
        coef, state = g.new_coefs(V), g.new_state(V)
        ratios = np.array([1.0, 2.0, 0.5, 3.0, 1.5, 0.25, 4.0, 0.3337], np.float32)
        coef[g.coef_slot(ratio)] = ratios[np.arange(V) % 8]
        coef[g.coef_slot(minus_one)] = np.float32(-1.0)
        coef[g.coef_slot(tl)] = np.float32(1.0 / SR)

        def fn(T, t0):
            out = np.zeros((T, 2, V, BLOCK), np.float32)
            out[:, 0] = ((2.0 + vv) / np.float32(3000.0)).astype(np.float32)[None, :, None]
            stop = ((np.arange(T)[:, None] + t0 + np.arange(V)[None, :]) % 9) == 4
            out[:, 1].view(np.uint32)[stop] = 0xFFFFFFFF
            return out
    elif name == "feedback":
        # y = x + 0.5 * y[previous block]: a 64-sample comb through the feedback edge
        x = g.input(0)
        k = g.param()
        fb = g.feedback_read()
        y = g.node("ADD", x, g.node("MULTIPLY", fb, k))
        g.feedback_write(fb, y)
        g.output(y)
        coef, state = g.new_coefs(V), g.new_state(V)
        coef[0] = (np.float32(0.2) + np.float32(0.7) * vv / np.float32(V)).astype(np.float32)
        fn = noise
    else:
        raise KeyError(name)
    w = Workload("functor_" + name, g, V, coef, state)
    w.inputs = _rows_inputs(fn)  # type: ignore[assignment]
    return w


FUNCTOR_CASES = ("impulse", "oneshot", "peak", "rms", "adsr", "allpass1", "glide", "interpolator1", "sample_glide",
                 "integer_delay", "integer_delay_var", "fractional_delay", "fractional_delay_var",
                 "pitchbend_delay", "allpass_int", "allpass_frac", "allpass_pb", "feedback",
                 "halfband_up", "halfband_roundtrip", "upsample2x_clip", "downsample2x_clip", "tempo_lock")
# functor cases with MLB_AGAIN nodes (a functor called again in the same vector): kept apart so that their GPU tests
# can be collected last (tests/test_zz_gpu_again.py)
AGAIN_CASES = ("upsample2x_osc",)


def aaltoverb_feedback(size_u: float, decay_u: float) -> float:
    """reverb.cpp:18-19,76-83: decayTime = unityToLogParam({0.8, 20})(decayU) (MLDSPProjections.h:105-123,176-195:
    intervalMap({0,1}, {a,b}, log{a,b})), decayIterations = decayTime / (sizeU * 0.5),
    feedback = powf(0.001, 1 / decayIterations) -- host-side scalar maths in float, step by step as written there."""
    f = np.float32
    a, b = f(0.8), f(20.0)
    x = f(decay_u) * (f(1.0) / (f(1.0) - f(0.0))) + (-f(0.0)) / (f(1.0) - f(0.0))
    c = a * (np.power(b / a, x, dtype=np.float32) - f(1.0)) / (b - a)
    decay_time = c * (b - a) + a
    iters = f(decay_time / (float(f(size_u)) * 0.5))  # double product, like `sizeU*0.5` with a double literal
    if decay_u >= 1.0:
        return 1.0
    return float(np.power(f(0.001), f(1.0) / iters, dtype=np.float32))


def config_6(n_voices: int = 4096) -> Workload:
    """Aaltoverb (examples/audio-and-midi/reverb.cpp) x n_voices independent stereo reverbs.
    sizeU = 0.25 + 0.5 v/V, decayU = 0.5; glide time 0.1 s; input = noise bursts on both channels."""
    from .graph import (AALTOVERB_AP_GAINS, AALTOVERB_AP_MAX, AALTOVERB_AP_SCALE, AALTOVERB_DELAY_MAX,
                        AALTOVERB_DELAY_SCALE, graph_aaltoverb)
    V = n_voices
    spec, n = graph_aaltoverb()
    coef, state = spec.new_coefs(V), spec.new_state(V)
    size_u = (np.float32(0.25) + np.float32(0.5) * np.arange(V, dtype=np.float32) / np.float32(V)).astype(np.float32)
    coef[spec.coef_slot(n["size2"])] = size_u * np.float32(2.0)
    coef[spec.coef_slot(n["feedback"])] = [aaltoverb_feedback(float(s), 0.5) for s in size_u]
    coef[spec.coef_slot(n["sr"])] = np.float32(SR)
    coef[spec.coef_slot(n["vmin"])] = np.float32(BLOCK)
    for i in range(10):
        coef[spec.coef_slot(n["apscale%d" % i])] = np.float32(AALTOVERB_AP_SCALE[i])
        coef[spec.coef_slot(n["ap%d" % (i + 1)], 0)] = np.float32(AALTOVERB_AP_GAINS[i])
        coef[spec.coef_slot(n["ap%d" % (i + 1)], 1)] = np.float32(AALTOVERB_AP_MAX[i])
    coef[spec.coef_slot(n["dscaleL"])] = np.float32(AALTOVERB_DELAY_SCALE[0])
    coef[spec.coef_slot(n["dscaleR"])] = np.float32(AALTOVERB_DELAY_SCALE[1])
    coef[spec.coef_slot(n["delayL"])] = coef[spec.coef_slot(n["delayR"])] = np.float32(AALTOVERB_DELAY_MAX)
    glide = api.coeffs("glide", 0.1 * SR)
    for key in ("glideDelay", "glideFeedback"):
        _set(coef, spec, n[key], np.repeat(glide[:, None], V, 1))
    w = Workload("aaltoverb", spec, V, coef, state)
    nl, nr = _noise_rows(5, V, 0.25), _noise_rows(6, V, 0.25)

    def fn(T, t0):  # a burst of noise for 6 blocks out of every 40, then the tail rings
        x = np.concatenate([nl(T, t0), nr(T, t0)], axis=1)
        on = ((np.arange(T) + t0) % 40 < 6).reshape(T, 1, 1, 1)
        return (x * on).astype(np.float32)
    w.inputs = _rows_inputs(fn)  # type: ignore[assignment]
    return w


# ---- coefficient-ROW (modulated / swept) filters: MLDSPFilters.h:97-115,136-152,283-286,304-319,385-400 ----

SWEPT_CASES = ("lopass_v", "sine_lopass_v_gain", "lopass_v_const", "lopass_mod", "loshelf_v", "hishelf_v",
               "loshelf_ramp")


def swept_omega_k(n_voices: int, n_blocks: int, t0: int = 0):
    """Per-voice cutoff / resonance sweeps (signal rate): omega in [0.02, 0.32], k in [0.05, 1.55]; [T][V][64]."""
    n = (np.arange(n_blocks * BLOCK, dtype=np.float64) + t0 * BLOCK)[None, :]
    v = np.arange(n_voices, dtype=np.float64)[:, None]
    omega = 0.02 + 0.3 * (0.5 + 0.5 * np.sin(n * (0.0021 + 1e-5 * v) + 0.37 * v))
    k = 0.05 + 1.5 * (0.5 + 0.5 * np.cos(n * 0.0013 + 0.11 * v))
    shp = (n_voices, n_blocks, BLOCK)
    return (np.ascontiguousarray(omega.astype(np.float32).reshape(shp).transpose(1, 0, 2)),
            np.ascontiguousarray(k.astype(np.float32).reshape(shp).transpose(1, 0, 2)))


def shelf_endpoints(kind: str, n_voices: int, n_points: int, t0: int = 0) -> np.ndarray:
    """Block-rate shelf coefficients {makeCoeffs(p_t)}: p_t = (omega, k, A) moving slowly; [n_points][n_coef][V]."""
    out = np.zeros((n_points, api._NCOEF[kind], n_voices), np.float32)
    v = np.arange(n_voices, dtype=np.float64)
    for i in range(n_points):
        t = t0 + i
        omega = (0.03 + 0.2 * (0.5 + 0.5 * np.sin(0.31 * t + 0.2 * v))).astype(np.float32)
        k = (0.4 + 0.8 * (0.5 + 0.5 * np.cos(0.17 * t + 0.05 * v))).astype(np.float32)
        db = -9.0 + 18.0 * (0.5 + 0.5 * np.sin(0.23 * t + 0.4 * v))
        A = np.power(np.float32(10.0), (db / 40.0).astype(np.float32)).astype(np.float32)
        out[i] = api.coeffs_batch(kind, omega, k, A)
    return out


def swept_filter_case(name: str, n_voices: int = 40, n_blocks: int = 8, x=None, omega=None, k=None) -> Workload:
    """name in SWEPT_CASES.  Audio = seeded noise (or `x` [T][V][64]); coefficient rows designed on the host
    with the library's own mlb_coeffs_* calls; `omega`, `k` override the sweeps."""
    V = n_voices
    g = GraphSpec()
    noise = _noise_rows(21, V, 0.5)
    audio = (lambda T, t0: noise(T, t0)[:, 0]) if x is None else (lambda T, t0: np.asarray(x, np.float32)[t0:t0 + T])

    def sweeps(T, t0):
        if omega is not None:
            return np.asarray(omega, np.float32)[t0:t0 + T], np.asarray(k, np.float32)[t0:t0 + T]
        return swept_omega_k(V, T, t0)

    coef = state = None
    if name in ("lopass_v", "sine_lopass_v_gain"):
        src = g.input(0)
        if name == "sine_lopass_v_gain":
            src = g.node("SINE", src)
        lp = g.node("LOPASS_V", src, g.input(1), g.input(2), g.input(3))
        if name == "sine_lopass_v_gain":
            lp = g.node("MULTIPLY", lp, g.param())
        g.output(lp)
        coef, state = g.new_coefs(V), g.new_state(V)
        if name == "sine_lopass_v_gain":
            coef[0] = np.float32(0.1)
            state[0] = SINE_ZERO_PHASE

        def fn(T, t0):
            om, kk = sweeps(T, t0)
            rows = api.coeffs_lopass_vec(om, kk)                        # [T][V][3][64]
            first = freq_rows(V, T, t0)[:, 0] if name == "sine_lopass_v_gain" else audio(T, t0)
            return np.ascontiguousarray(np.concatenate([first[:, None], rows.transpose(0, 2, 1, 3)], axis=1))
    elif name == "lopass_v_const":
        lp = g.node("LOPASS_V", g.input(0), g.param(), g.param(), g.param())
        g.output(lp)
        coef, state = g.new_coefs(V), g.new_state(V)
        coef[0:3] = _svf_coefs("lopass", V)
        fn = lambda T, t0: np.ascontiguousarray(audio(T, t0)[:, None])
    elif name == "lopass_mod":
        g.output(g.node("LOPASS_MOD", g.input(0), g.input(1), g.input(2)))
        coef, state = g.new_coefs(V), g.new_state(V)

        def fn(T, t0):
            om, kk = sweeps(T, t0)
            return np.ascontiguousarray(np.stack([audio(T, t0), om, kk], axis=1))
    elif name in ("loshelf_v", "hishelf_v"):
        kind = name[:-2]
        nco = api._NCOEF[kind]
        g.output(g.node(name.upper(), g.input(0), *[g.input(1 + i) for i in range(nco)]))
        coef, state = g.new_coefs(V), g.new_state(V)

        def fn(T, t0):
            ep = shelf_endpoints(kind, V, T + 1, t0)                    # block t ramps from ep[t] to ep[t+1]
            rows = np.empty((T, nco, V, BLOCK), np.float32)
            for t in range(T):
                for v in range(V):
                    rows[t, :, v] = api.interpolate_coeffs_linear(ep[t, :, v], ep[t + 1, :, v])
            return np.ascontiguousarray(np.concatenate([audio(T, t0)[:, None], rows], axis=1))
    elif name == "loshelf_ramp":
        # interpolateCoeffsLinear on the device: one RAMP per coefficient from two endpoint rows (sample 0 is read)
        ramps = [g.node("RAMP", g.input(1 + 2 * i), g.input(2 + 2 * i)) for i in range(5)]
        g.output(g.node("LOSHELF_V", g.input(0), *ramps))
        coef, state = g.new_coefs(V), g.new_state(V)

        def fn(T, t0):
            ep = shelf_endpoints("loshelf", V, T + 1, t0)
            planes = np.zeros((T, 11, V, BLOCK), np.float32)
            planes[:, 0] = audio(T, t0)
            for i in range(5):
                planes[:, 1 + 2 * i, :, 0] = ep[:T, i]
                planes[:, 2 + 2 * i, :, 0] = ep[1:T + 1, i]
            return planes
    else:
        raise ValueError(name)
    w = Workload("swept_" + name, g, V, coef, state)
    w.inputs = _rows_inputs(fn)  # type: ignore[assignment]
    return w


# ---- SURVEY 8(f) row 3: per-voice event records for the EventsToSignals::Voice bank ----

VOICE_EVENTS_DTYPE = np.dtype([("n_events", "u1"), ("set_mask", "u1"), ("pad", "u1", (2,)),
                               ("time", "u1", (4,)), ("type", "u1", (4,)), ("flags", "u1", (4,)),
                               ("value1", "f4", (4,)), ("value2", "f4", (4,)),
                               ("bend", "f4"), ("mod", "f4"), ("x", "f4"), ("y", "f4"), ("z", "f4"),
                               ("pressure", "f4")])
assert VOICE_EVENTS_DTYPE.itemsize == 72  # struct mlb_voice_events (include/mlb200.h)
VOICES_MIDI = 1

EV_NOTE_ON, EV_NOTE_RETRIG, EV_NOTE_SUSTAIN, EV_NOTE_OFF = 1, 2, 3, 4
EVF_GLIDE, EVF_RESET = 1, 2


def voice_bank_params(n_voices: int):
    """voice_index, pitch_glide_seconds, drift_amount, pitch_bend (semitones) per voice."""
    v = np.arange(n_voices)
    return ((v % 16 + 1).astype(np.int32), (np.float32(0.0) + np.float32(0.01) * (v % 7)).astype(np.float32),
            (np.float32(0.25) * (v % 5)).astype(np.float32), np.where(v % 3 == 0, 24.0, 7.0).astype(np.float32))


def voice_events(n_voices: int, n_blocks: int, seed: int = 1, density: float = 0.35, ctl: float = 0.3) -> np.ndarray:
    """A seeded performance: [T][V] records.  Each voice plays notes (on / retrigger / off, with and
    without glide and age reset, sometimes several per vector, sometimes two at the same frame) while
    bend / mod / x / y / z move now and then."""
    rng = np.random.default_rng(seed)
    ev = np.zeros((n_blocks, n_voices), VOICE_EVENTS_DTYPE)
    held = np.zeros(n_voices, bool)
    for t in range(n_blocks):
        for v in range(n_voices):
            r = ev[t, v]
            if rng.random() < density:
                n = int(rng.integers(1, 5))
                times = np.sort(rng.integers(0, 65, n))  # 64 = "end of vector", clamped by the voice
                if rng.random() < 0.2 and n > 1:
                    times[1] = times[0]
                for k in range(n):
                    if held[v] and rng.random() < 0.5:
                        typ = EV_NOTE_OFF
                    else:
                        typ = EV_NOTE_ON if rng.random() < 0.7 else EV_NOTE_RETRIG
                    if rng.random() < 0.05:
                        typ = EV_NOTE_SUSTAIN  # ignored by the voice
                    held[v] = typ in (EV_NOTE_ON, EV_NOTE_RETRIG) or (held[v] and typ == EV_NOTE_SUSTAIN)
                    r["time"][k] = times[k]
                    r["type"][k] = typ
                    r["flags"][k] = int(rng.integers(0, 4))
                    r["value1"][k] = np.float32(rng.integers(36, 96)) / np.float32(12.0)
                    r["value2"][k] = np.float32(rng.random() * 0.9 + 0.1)
                r["n_events"] = n
            if rng.random() < ctl:
                m = int(rng.integers(1, 64))
                r["set_mask"] = m
                r["pressure"] = np.float32(rng.random())
                r["bend"], r["mod"] = np.float32(rng.random() * 2 - 1), np.float32(rng.random())
                r["x"], r["y"], r["z"] = np.float32(rng.random()), np.float32(rng.random()), np.float32(rng.random())
    return ev


def synth_bank_params(n_voices: int):
    """voice_bank_params with a pitch-bend range of 0 semitones: the kPitch row is then the glided note
    pitch plus drift, usable as a SineGen frequency row as it stands (see synth_events)."""
    vi, gs, da, pb = voice_bank_params(n_voices)
    return vi, gs, da, np.zeros_like(pb)


def synth_events(n_voices: int, n_blocks: int, seed: int = 2, density: float = 0.10, ctl: float = 0.05,
                 pitch_scale: float = 2.0 ** -5) -> np.ndarray:
    """Contract-E performance for a bank of any size: a 256-voice seeded performance repeated across the
    bank, note pitches scaled so that the kPitch row can drive SineGen directly (note / 12 * 2^-5 =
    0.09 .. 0.25 cycles per sample; the reference leaves the pitch -> frequency mapping to the client,
    MLSynth.h:67-71)."""
    base = voice_events(min(n_voices, 256), n_blocks, seed=seed, density=density, ctl=ctl)
    base["value1"] *= np.float32(pitch_scale)
    reps = (n_voices + base.shape[1] - 1) // base.shape[1]
    return np.ascontiguousarray(np.tile(base, (1, reps))[:, :n_voices])


def instrument_buses(n_instruments: int, polyphony: int, mpe: bool = False):
    """The bus layout (first voice, voice count; int32 [G] each) of a bank of n_instruments Synths with `polyphony`
    voices each, for api.Buses.  MIDI: instrument k is voices [k poly, (k + 1) poly).  MPE: instrument k owns
    poly + 1 voices, of which the first, k (poly + 1), is its main voice; Synth sums getInputVoice(v) = voices[v + 1]
    (MLEventsToSignals.h:184), so the bus skips it: [k (poly + 1) + 1, (k + 1) (poly + 1))."""
    k = np.arange(n_instruments, dtype=np.int64)
    stride = polyphony + 1 if mpe else polyphony
    first = (k * stride + (1 if mpe else 0)).astype(np.int32)
    return first, np.full(n_instruments, polyphony, np.int32)


CONTROLLER_POOL = (1, 2, 7, 10, 11, 16, 64, 71, 73, 74, 128)  # mod wheel, breath, volume, pan, expression, ...


def controller_changes(n_instruments: int, n_blocks: int, density: float = 0.05, seed: int = 11,
                       pool=CONTROLLER_POOL):
    """A MIDI-fader-like controller stream for api.ControllerBank: in a fraction `density` of the (block, instrument)
    pairs a fader moves, sending 1 to 4 writes in the block, mostly to one controller of `pool` (so that some
    blocks hold several writes to one controller, the last of which counts) with 7-bit values (k / 127) walking
    from where the fader was.  Returns (offsets [T][G + 1] int32, changes of api.CONTROLLER_CHANGE_DTYPE)."""
    from .api import CONTROLLER_CHANGE_DTYPE
    rng = np.random.default_rng(seed)
    G, T = int(n_instruments), int(n_blocks)
    pool = np.asarray(pool, np.uint16)
    n = np.where(rng.random((T, G)) < density, rng.integers(1, 5, (T, G)), 0)
    offsets = np.zeros((T, G + 1), np.int32)
    ends = np.cumsum(n.ravel()).reshape(T, G)
    offsets[:, 1:] = ends
    offsets[:, 0] = np.concatenate(([0], ends[:-1, -1]))
    total = int(n.sum())
    burst = np.repeat(np.arange(n.size), n.ravel())                # the (block, instrument) pair of each write
    fader = rng.integers(0, len(pool), n.size)[burst]               # the burst's controller ...
    other = rng.random(total) < 0.25                                 # ... or, now and then, another one
    ctrl = np.where(other, rng.integers(0, len(pool), total), fader)
    start = rng.integers(0, 128, n.size)[burst]
    pos = np.arange(total) - np.repeat(np.cumsum(n.ravel()) - n.ravel(), n.ravel())
    step = rng.integers(-6, 7, n.size)[burst]
    value = np.clip(start + pos * step, 0, 127).astype(np.float32) / np.float32(127)
    changes = np.zeros(total, CONTROLLER_CHANGE_DTYPE)
    changes["controller"] = pool[ctrl]
    changes["value"] = value
    return offsets, changes


# ---- random voice graphs (tests): any DAG of the op table, for checker-vs-checker and GPU-vs-checker runs ----

def random_graph_workload(seed: int, n_voices: int = 37, n_nodes: int = 24, hw_approx: bool = True,
                          again_prob: float = 0.0) -> Workload:
    """A random DAG over most of the op table (generators, filters, functors with delay memory, elementwise
    ops), two external input planes, random but sane coefficients; two outputs.  hw_approx=False leaves out
    Peak / RMS, whose outputs go through the CPU-defined rsqrt approximation (compared with a tolerance only).
    again_prob > 0: generators, filters and glides are, with that probability, called AGAIN in the same vector on
    other inputs (MLB_AGAIN; the default 0 leaves the graphs of a seed as they always were)."""
    from .graph import OP_INFO, OP_NAME
    rng = np.random.default_rng(seed)
    V = n_voices
    g = GraphSpec()
    rows = [g.input(0), g.input(1)]           # audio-ish rows in [-1, 1] and positive "control" rows
    params = [g.param() for _ in range(4)]
    unary = ["ABS", "SIN_APPROX", "COS", "SIGN", "FRACTIONAL_PART", "EXP_APPROX", "SQRT"]
    binary = ["ADD", "SUBTRACT", "MULTIPLY", "MIN", "MAX", "GREATER_THAN", "DIVIDE"]
    ternary = ["LERP", "CLAMP", "SELECT"]
    filt = ["LOPASS", "HIPASS", "BANDPASS", "BELL", "ONEPOLE", "DCBLOCKER", "INTEGRATOR", "DIFFERENTIATOR", "RMS",
            "PEAK", "ALLPASS1", "ADSR", "SAMPLE_GLIDE"]
    if not hw_approx:
        filt = [f for f in filt if f not in ("RMS", "PEAK")]
    gens = ["SINE", "PHASOR", "SAW", "TICK", "ONESHOT", "IMPULSE"]
    delays1 = ["INTEGER_DELAY", "FRACTIONAL_DELAY", "ALLPASS_INT", "ALLPASS_FRAC", "GLIDE", "INTERPOLATOR1"]
    delays2 = ["INTEGER_DELAY_VAR", "FRACTIONAL_DELAY_VAR", "PITCHBEND_DELAY", "ALLPASS_PB"]
    node_kind = {}

    def pick(allow_param=True):
        pool = rows + (params if allow_param else [])
        return pool[int(rng.integers(len(pool)))]

    fb = g.feedback_read() if rng.random() < 0.5 else None
    if fb is not None:
        rows.append(fb)
    while g.n_nodes < n_nodes:
        r = rng.random()
        if r < 0.2:
            y = g.node(unary[int(rng.integers(len(unary)))], pick(False))
        elif r < 0.45:
            y = g.node(binary[int(rng.integers(len(binary)))], pick(False), pick())
        elif r < 0.55:
            y = g.node(ternary[int(rng.integers(len(ternary)))], pick(False), pick(), pick())
        elif r < 0.75:
            y = g.node(filt[int(rng.integers(len(filt)))], pick(False))
        elif r < 0.83:
            y = g.node(gens[int(rng.integers(len(gens)))], rows[1] if rng.random() < 0.7 else params[0])
        elif r < 0.93:
            y = g.node(delays1[int(rng.integers(len(delays1)))], pick(False))
        else:
            y = g.node(delays2[int(rng.integers(len(delays2)))], pick(False), rows[1])
        node_kind[y] = OP_NAME[g.ops[y]]
        rows.append(y)
        name = node_kind[y]
        if again_prob and (name in filt or name in gens or name in ("GLIDE", "INTERPOLATOR1")) and \
                rng.random() < again_prob:
            if name in gens:
                rows.append(g.again(y, rows[1] if rng.random() < 0.5 else params[0]))
            else:
                rows.append(g.again(y, pick(False)))
    if fb is not None:
        g.feedback_write(fb, g.node("MULTIPLY", rows[-1], params[1]))
    g.output(rows[-1], rows[len(rows) // 2])
    coef, state = g.new_coefs(V), g.new_state(V)
    vv = np.arange(V, dtype=np.float32)
    coef[g.coef_slot(params[0])] = np.float32(0.01) + np.float32(0.002) * vv      # a frequency
    coef[g.coef_slot(params[1])] = np.float32(0.3)
    coef[g.coef_slot(params[2])] = np.float32(-0.5) + vv / np.float32(V)
    coef[g.coef_slot(params[3])] = np.float32(1.5)
    for i, name in node_kind.items():
        c0 = g.coef_slot(i)
        n_co = OP_INFO[g.ops[i]][2]
        om = float(0.01 + 0.2 * rng.random())
        if name in ("LOPASS", "HIPASS", "BANDPASS"):
            coef[c0:c0 + n_co] = api.coeffs(name.lower(), om, 0.7)[:, None]
        elif name == "BELL":
            coef[c0:c0 + n_co] = api.coeffs("bell", om, 0.7, 1.3)[:, None]
        elif name in ("ONEPOLE", "RMS"):
            coef[c0:c0 + n_co] = api.coeffs(name.lower(), om * 0.1)[:, None]
        elif name == "PEAK":
            coef[c0:c0 + 2] = api.coeffs("peak", om * 0.01)[:, None]
            coef[c0 + 2] = np.float32(150)
        elif name == "DCBLOCKER":
            coef[c0] = np.float32(api.coeffs_dcblocker(0.045))
        elif name == "INTEGRATOR":
            coef[c0] = np.float32(0.01)
        elif name == "ALLPASS1":
            coef[c0] = np.float32(api.coeffs_allpass1(0.618 + rng.random()))
        elif name == "ADSR":
            coef[c0:c0 + 4] = api.coeffs("adsr", 0.001, 0.002, 0.5, 0.003, SR)[:, None]
        elif name == "SAMPLE_GLIDE":
            coef[c0:c0 + 2] = api.coeffs("sample_glide", 40.0)[:, None]
        elif name == "GLIDE":
            coef[c0:c0 + 2] = api.coeffs("glide", 192.0)[:, None]
        elif name == "INTEGER_DELAY":
            coef[c0] = np.float32((np.arange(V) * 7) % 200)
            coef[c0 + 1] = np.float32(200)
        elif name == "FRACTIONAL_DELAY":
            coef[c0] = (np.float32(3.3) + vv * np.float32(2.1)).astype(np.float32)
            coef[c0 + 1] = np.float32(200)
        elif name in ("ALLPASS_INT", "ALLPASS_FRAC"):
            coef[c0] = np.float32(0.5)
            coef[c0 + 1] = (np.float32(70.0) + vv * np.float32(3.3)).astype(np.float32)
            coef[c0 + 2] = np.float32(64 + 4 * V)
        elif name in ("INTEGER_DELAY_VAR", "FRACTIONAL_DELAY_VAR", "PITCHBEND_DELAY"):
            coef[c0] = np.float32(300)
        elif name == "ALLPASS_PB":
            coef[c0] = np.float32(0.6)
            coef[c0 + 1] = np.float32(400)
        if name == "ONESHOT":
            state[g.state_slot(i, 1)] = 1
        if name == "SINE":
            state[g.state_slot(i)] = SINE_ZERO_PHASE
    w = Workload("random%d" % seed, g, V, coef, state)
    audio = _noise_rows(seed + 1000, V, 0.5)

    def fn(T, t0):  # plane 0: noise with gaps (gates for ADSR); plane 1: positive, slowly moving (frequencies / delay times)
        x = audio(T, t0)
        n = (np.arange(T * BLOCK, dtype=np.float64) + t0 * BLOCK)
        ctl = (0.004 + 0.003 * np.sin(n[None, :] * 0.001 * (1.0 + 0.01 * vv[:, None].astype(np.float64)))).astype(np.float32)
        ctl = np.ascontiguousarray(ctl.reshape(V, T, BLOCK).transpose(1, 0, 2))[:, None]
        gate = (((n.reshape(T, 1, 1, BLOCK) // 200) % 2) == 0)
        return np.concatenate([(x * gate).astype(np.float32), ctl * np.float32(60.0)], axis=1)
    w.inputs = _rows_inputs(fn)  # type: ignore[assignment]
    return w


# ---- K9: the FDTD membrane of examples/audio-and-midi/fdtd.cpp ----

def fdtd_example(n_instances: int) -> Workload:
    """The first lines of the example's processFDTD (fdtd.cpp:165-170) as a graph, per instance:
        ticks = ImpulseGen(2/sr) * 0.1;  freq = (220 + SineGen(0.15/sr) * 40) / sr   (sr = 48000)
    with freshly constructed generators.  Outputs [ticks, freq]: the graph's [T][2][V][64] output buffer is the
    input of an FDTDBank(V, in_planes=2, excite_plane=0, freq_plane=1, flags=FTZ) as it stands."""
    V = n_instances
    g = GraphSpec()
    f_imp, gain, f_sin, depth, center, rate = (g.param() for _ in range(6))
    ticks = g.node("MULTIPLY", g.node("IMPULSE", f_imp), gain)
    freq = g.node("DIVIDE", g.node("ADD", center, g.node("MULTIPLY", g.node("SINE", f_sin), depth)), rate)
    g.output(ticks, freq)
    coef, state = g.new_coefs(V), g.new_state(V)
    sr = np.float32(SR)
    for node, value in ((f_imp, np.float32(2.0) / sr), (gain, np.float32(0.1)), (f_sin, np.float32(0.15) / sr),
                        (depth, np.float32(40.0)), (center, np.float32(220.0)), (rate, sr)):
        coef[g.coef_slot(node)] = value
    return Workload("fdtd_example", g, V, coef, state)


FDTD_BURST_PERIOD = 375  # vectors between two excitations of one membrane (the example's impulse rate at 48 kHz)


def fdtd_inputs(n_instances: int, n_blocks: int, t0: int = 0, v0: int = 0, v1: Optional[int] = None) -> np.ndarray:
    """Excitation and frequency rows for a bank of FDTD membranes, [T][2][V'][64] f32 for instances [v0, v1):
      excitation: one vector of noise (uniform in +-0.1, a seeded function of instance and vector) every
                  FDTD_BURST_PERIOD vectors, instance v firing at vectors t = (53 v) mod FDTD_BURST_PERIOD + k P;
      frequency:  Fs_v[n] = (100 + 900 v / V) / 48000 * (1 + 0.1 tri(((n + 97 v) mod 4800) / 4800)) cycles per sample,
                  n = absolute sample index, tri = 0..1..0 -- at most 0.0229, inside the stable range (T^2 < 3/5,
                  i.e. Fs below ~0.057)."""
    V = n_instances
    v1 = V if v1 is None else v1
    vv = np.arange(v0, v1, dtype=np.int64)
    out = np.zeros((n_blocks, 2, v1 - v0, BLOCK), np.float32)
    base = ((np.float32(100.0) + np.float32(900.0) * vv.astype(np.float32) / np.float32(V)) / np.float32(SR))[:, None]
    for t in range(n_blocks):
        ta = t0 + t
        fire = np.nonzero((ta - 53 * vv) % FDTD_BURST_PERIOD == 0)[0]
        for i in fire:
            rng = np.random.default_rng((int(vv[i]) << 20) ^ ta)
            out[t, 0, i] = rng.uniform(-0.1, 0.1, BLOCK).astype(np.float32)
        n = np.arange(BLOCK, dtype=np.int64)[None, :] + ta * BLOCK + 97 * vv[:, None]
        ph = (n % 4800).astype(np.float32) / np.float32(4800.0)
        tri = np.float32(1.0) - np.abs(np.float32(2.0) * ph - np.float32(1.0))
        out[t, 1] = base * (np.float32(1.0) + np.float32(0.1) * tri)
    return out
