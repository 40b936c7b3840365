"""Float64 evaluation of the voice graphs the fast-mode kernels run -- TEST INFRASTRUCTURE ONLY.

Fast mode (MLB_GRAPH_FAST) lets the compiler contract multiplies and adds into FMAs, so its bits differ from the
reference's.  Its accuracy is judged here against this evaluator: the same formulas as the plain-C port
(oracle/port/mlport.c) -- phasorToSine with the Newton sqrt2 constants, polyBLEP, the cephes-style sinApprox, the SVF
cores, FDN<8> -- with the same binary32 constants and coefficient words, evaluated in binary64.  A difference from it
is rounding error and nothing else.

The discrete decisions are the reference's own: phase accumulators are uint32 sums of cvtps2dq(freq * 2^32)
(0x80000000 when out of range), the phasor that polyBLEP compares is the binary32 value the reference compares,
NoiseGen is its LCG bit for bit, and the FDN delay lengths are the port's integers.

Only the ops the fast kernels instantiate are covered; any other op is refused.
"""
from __future__ import annotations

from typing import NamedTuple, Optional, Sequence

import numpy as np

from madronalib_b200.graph import BLOCK, OP_INFO, OP_NAME, GraphSpec

SUPPORTED = frozenset(("INPUT", "PARAM", "NOISE", "PHASOR", "SINE", "SAW", "LOPASS", "HIPASS", "BANDPASS", "LOSHELF",
                       "HISHELF", "BELL", "ONEPOLE", "DCBLOCKER", "LOPASS_V", "MULTIPLY", "ADD", "FDN8", "FDN8_R",
                       "SIN_APPROX", "CLAMP", "ABS", "LERP"))
INT_STATE_OPS = frozenset(("NOISE", "PHASOR", "SINE", "SAW"))  # mSeed, mOmega32


def _c(hexfloat: str) -> float:
    return float.fromhex(hexfloat)


def _f(x: float) -> float:
    """A binary32 constant of the reference, as a binary64 value."""
    return float(np.float32(x))


# phasorToSine (G:316-338): the reference's constexpr Newton sqrt2, not sqrt(2)
K_SQRT2 = _c("0x1.6a0a0ap+0")
K_DOMAIN = _c("0x1.6a0a0ap+2")
K_FLIP = _c("0x1.6a0a0ap+1")
K_INV_RANGE = _c("0x1.0f876cp+0")
K_ONE_SIXTH = _c("0x1.555556p-3")
# sinApprox (M:758-772)
SIN_APPROX_C = tuple(_f(x) for x in (0.99997937679290771484375, -0.166624367237091064453125,
                                       8.30897875130176544189453125e-3, -1.92649182281456887722015380859375e-4,
                                       2.147840177713078446686267852783203125e-6))


class F64Run(NamedTuple):
    out: np.ndarray          # [T][n_out][V'][64] float64
    state_int: np.ndarray    # [n_state][V'] uint32; integer words (phases, seeds), 0 in the float slots
    state_float: np.ndarray  # [n_state][V'] float64; float words, NaN in the integer slots
    mix: np.ndarray          # [T][n_out][64] float64: the float64 sum of the float64 rows of the evaluated voices


def int_slots(spec: GraphSpec) -> np.ndarray:
    """Boolean [n_state]: True where the state word is an integer (phase accumulator or noise seed)."""
    st_off = spec.offsets()[0]
    m = np.zeros(spec.n_state, bool)
    for i, op in enumerate(spec.ops):
        if OP_NAME[op] in INT_STATE_OPS:
            m[st_off[i]:st_off[i] + OP_INFO[op][1]] = True
    return m


def check_supported(spec: GraphSpec) -> None:
    for i, op in enumerate(spec.ops):
        name = OP_NAME[op]
        if name not in SUPPORTED:
            raise ValueError(f"f64_graph: node {i} is {name}, which this evaluator does not cover")
        if spec.again_target(i) >= 0:
            raise ValueError(f"f64_graph: node {i} calls another node's functor again; not covered")


# ---- generators ----

def _phases(phase0: np.ndarray, freq: np.ndarray) -> np.ndarray:
    """The phase after each sample, uint64 holding uint32 values: phase += cvtps2dq(freq * 2^32) (G:190-199)."""
    steps = freq * 4294967296.0
    ok = np.abs(steps) < 2147483648.0  # False for NaN too: "integer indefinite"
    inc = np.where(ok, np.rint(np.where(ok, steps, 0.0)), -2147483648.0).astype(np.int64) & 0xFFFFFFFF
    return (phase0.astype(np.uint64)[:, None] + np.cumsum(inc.astype(np.uint64), axis=1)) & 0xFFFFFFFF


def _phasor(ph: np.ndarray) -> np.ndarray:
    """unsignedIntToFloat(phase) * 2^-32 in binary64: (phase >> 1) * 2^-31."""
    return (ph >> 1).astype(np.float64) * 2.0 ** -31


def _phasor32(ph: np.ndarray) -> np.ndarray:
    """The same value as the reference holds it: (float)(int)(phase >> 1) * 2^-31, binary32."""
    return (ph >> 1).astype(np.float32) * np.float32(2.0 ** -31)


def _phasor_to_sine(p: np.ndarray) -> np.ndarray:
    omega = p * K_DOMAIN - K_SQRT2
    tri = np.where(omega > K_SQRT2, K_FLIP - omega, omega)
    return (K_INV_RANGE * tri) * (1.0 - (tri * tri) * K_ONE_SIXTH)


def _saw(ph: np.ndarray, freq: np.ndarray) -> np.ndarray:
    """phasorToSaw (G:362-369) with polyBLEP (G:285-311); the branches are taken on the binary32 values compared."""
    t, t32 = _phasor(ph), _phasor32(ph)
    dt, dt32 = freq, freq.astype(np.float32)
    lo = t32 < dt32
    hi = ~lo & (t32 > np.float32(1.0) - dt32)
    with np.errstate(divide="ignore", invalid="ignore"):
        u = t / dt
        w = (t - 1.0) / dt
    c = np.where(lo, u + u - u * u - 1.0, np.where(hi, w * w + w + w + 1.0, 0.0))
    return (t * 2.0 - 1.0) - c


def _noise(seed: np.ndarray):
    """NoiseGen (G:115,132-142): the LCG bit for bit; u * 2 - 3 is exact in binary32 already."""
    s = seed.copy()
    y = np.empty((s.shape[0], BLOCK))
    for j in range(BLOCK):
        s = s * np.uint32(0x0019660D) + np.uint32(0x3C6EF35F)
        u = (((s >> np.uint32(9)) & np.uint32(0x007FFFFF)) | np.uint32(0x3F800000)).view(np.float32)
        y[:, j] = u.astype(np.float64) * 2.0 - 3.0
    return y, s


# ---- filters: c[k] is coefficient k as a [V'][64] row (constant words broadcast) ----

def _svf_g(kind, x, c, st):
    """Lopass / Hipass / Bandpass (F:121-131, 183-194, 227-237) and Lopass with coefficient rows (F:141-149)."""
    ic1, ic2 = st
    y = np.empty_like(x)
    g0, g1, g2 = c[0], c[1], c[2]
    for j in range(BLOCK):
        v0 = x[:, j]
        t0 = v0 - ic2
        t1 = g0[:, j] * t0 + g1[:, j] * ic1
        t2 = g2[:, j] * t0 + g0[:, j] * ic1
        v1 = t1 + ic1
        v2 = t2 + ic2
        ic1 = ic1 + 2.0 * t1
        ic2 = ic2 + 2.0 * t2
        if kind == "HIPASS":
            y[:, j] = v0 - c[3][:, j] * v1 - v2
        elif kind == "BANDPASS":
            y[:, j] = v1
        else:
            y[:, j] = v2
    return y, [ic1, ic2]


def _svf_a(kind, x, c, st):
    """LoShelf / HiShelf / Bell (F:293-299, 374-380, 432-438)."""
    ic1, ic2 = st
    y = np.empty_like(x)
    a1, a2, a3 = c[0], c[1], c[2]
    for j in range(BLOCK):
        v0 = x[:, j]
        v3 = v0 - ic2
        v1 = a1[:, j] * ic1 + a2[:, j] * v3
        v2 = ic2 + a2[:, j] * ic1 + a3[:, j] * v3
        ic1 = 2.0 * v1 - ic1
        ic2 = 2.0 * v2 - ic2
        if kind == "LOSHELF":
            y[:, j] = v0 + c[3][:, j] * v1 + c[4][:, j] * v2
        elif kind == "HISHELF":
            y[:, j] = c[3][:, j] * v0 + c[4][:, j] * v1 + c[5][:, j] * v2
        else:
            y[:, j] = v0 + c[3][:, j] * v1
    return y, [ic1, ic2]


def _onepole(x, c, st):
    """OnePole (F:466-475)."""
    (y1,) = st
    y = np.empty_like(x)
    for j in range(BLOCK):
        y1 = c[0][:, j] * x[:, j] + c[1][:, j] * y1
        y[:, j] = y1
    return y, [y1]


def _dcblocker(x, c, st):
    """DCBlocker (F:500-512); state x1, y1."""
    x1, y1 = st
    y = np.empty_like(x)
    for j in range(BLOCK):
        y1 = x[:, j] - x1 + c[0][:, j] * y1
        x1 = x[:, j]
        y[:, j] = y1
    return y, [x1, y1]


class _Fdn8:
    """FDN<8> (F:1162-1239) for the evaluated voices: eight IntegerDelays of the port's integer lengths, read from
    the history of their inputs, the stereo sums, the Householder step, eight OnePoles and the feedback gains."""

    def __init__(self, co: np.ndarray, n_blocks: int):
        # co [32][V']: a0[8] b1[8] gain[8] len[8]; the length is C's (int) truncation of the word
        self.a0, self.b1, self.gain = co[0:8], co[8:16], co[16:24]
        self.len = np.trunc(co[24:32]).astype(np.int64)
        n = co.shape[1]
        self.hist = np.zeros((8, n, n_blocks * BLOCK))  # what each delay line was given, sample by sample
        self.carry = np.zeros((8, n, BLOCK))            # FDN::mDelayInputVectors, written at the end of a block
        self.t = 0

    def __call__(self, x: np.ndarray, st):
        n = x.shape[0]
        t0 = self.t * BLOCK
        self.hist[:, :, t0:t0 + BLOCK] = self.carry
        idx = t0 + np.arange(BLOCK)[None, None, :] - self.len[:, :, None]   # [8][V'][64]
        d = np.take_along_axis(self.hist, np.maximum(idx, 0), axis=2)
        d = np.where(idx >= 0, d, 0.0)
        out_r = d[0] + d[2] + d[4] + d[6]
        out_l = d[1] + d[3] + d[5] + d[7]
        d = d - d.sum(axis=0)[None] * 0.25
        y1 = np.stack(st)  # [8][V']
        for j in range(BLOCK):
            y1 = self.a0 * d[:, :, j] + self.b1 * y1
            self.carry[:, :, j] = y1 * self.gain + x[None, :, j]
        self.t += 1
        assert n == y1.shape[1]
        return out_l, out_r, list(y1)


def evaluate(spec: GraphSpec, n_voices: int, n_blocks: int, inp: Optional[np.ndarray], state: np.ndarray,
             coef: np.ndarray, voices: Optional[Sequence[int]] = None) -> F64Run:
    """Run `n_blocks` blocks of the graph from `state` in binary64 (arguments as PortOracle.run takes them), for the
    voices listed in `voices` (all by default); voices are independent.  Outputs and state columns follow `voices`."""
    check_supported(spec)
    V, T = n_voices, n_blocks
    vs = np.arange(V) if voices is None else np.asarray(voices, np.int64)
    n = vs.shape[0]
    st_off, co_off, n_state, _ = spec.offsets()
    state = np.asarray(state, np.uint32)
    coef = np.asarray(coef, np.float32)
    assert state.shape == (n_state, V) and coef.shape == (spec.n_coef, V)
    if spec.n_in:
        assert inp is not None and inp.shape == (T, spec.n_in, V, BLOCK), None if inp is None else inp.shape
    co = coef[:, vs].astype(np.float64)
    st0 = state[:, vs]
    is_int = int_slots(spec)
    words = [st0[s].copy() if is_int[s] else st0[s].view(np.float32).astype(np.float64) for s in range(n_state)]
    fdn = {i: _Fdn8(co[co_off[i]:co_off[i] + 32], T) for i, op in enumerate(spec.ops) if OP_NAME[op] == "FDN8"}

    def row(k):  # coefficient word k as a [V'][64] row
        return np.broadcast_to(co[k][:, None], (n, BLOCK))

    out = np.empty((T, spec.n_out, n, BLOCK))
    for t in range(T):
        rows, second = [None] * spec.n_nodes, {}
        for i, op in enumerate(spec.ops):
            name = OP_NAME[op]
            _, nst, nco = OP_INFO[op]
            a, b, c = [rows[j] if j >= 0 else None for j in (list(spec.ins[i]) + [-1, -1, -1])[:3]]
            st = words[st_off[i]:st_off[i] + nst]
            cw = [row(co_off[i] + k) for k in range(nco)]
            if name == "INPUT":
                y = inp[t, spec.iargs[i]][vs].astype(np.float64)
            elif name == "PARAM":
                y = cw[0]
            elif name == "NOISE":
                y, s = _noise(st[0])
                st = [s]
            elif name in ("PHASOR", "SINE", "SAW"):
                ph = _phases(st[0], a)
                st = [ph[:, -1].astype(np.uint32)]
                y = _phasor(ph) if name == "PHASOR" else _phasor_to_sine(_phasor(ph)) if name == "SINE" else _saw(ph, a)
            elif name in ("LOPASS", "HIPASS", "BANDPASS"):
                y, st = _svf_g(name, a, cw, st)
            elif name == "LOPASS_V":
                y, st = _svf_g(name, a, [b, c, rows[spec.ins[i][3]]], st)
            elif name in ("LOSHELF", "HISHELF", "BELL"):
                y, st = _svf_a(name, a, cw, st)
            elif name == "ONEPOLE":
                y, st = _onepole(a, cw, st)
            elif name == "DCBLOCKER":
                y, st = _dcblocker(a, cw, st)
            elif name == "FDN8":
                y, second[i], st = fdn[i](a, st)
            elif name == "FDN8_R":
                y = second[spec.ins[i][0]]
            elif name == "MULTIPLY":
                y = a * b
            elif name == "ADD":
                y = a + b
            elif name == "SIN_APPROX":
                x2 = a * a
                k0, k1, k2, k3, k4 = SIN_APPROX_C
                y = a * (k0 + x2 * (k1 + x2 * (k2 + x2 * (k3 + x2 * k4))))
            elif name == "CLAMP":  # _mm_min_ps(_mm_max_ps(a, b), c): second operand when unordered or equal
                m = np.where(a > b, a, b)
                y = np.where(m < c, m, c)
            elif name == "ABS":
                y = np.abs(a)
            elif name == "LERP":
                y = a + c * (b - a)
            else:  # pragma: no cover -- check_supported refused it
                raise AssertionError(name)
            words[st_off[i]:st_off[i] + nst] = st
            rows[i] = y
        for k, o in enumerate(spec.outs):
            out[t, k] = rows[o]
    state_int = np.zeros((n_state, n), np.uint32)
    state_float = np.full((n_state, n), np.nan)
    for s in range(n_state):
        if is_int[s]:
            state_int[s] = words[s]
        else:
            state_float[s] = words[s]
    return F64Run(out, state_int, state_float, out.sum(axis=2))


# ---- the error metric ----

def rel_err_per_voice(y: np.ndarray, y64: np.ndarray) -> np.ndarray:
    """[V']: per voice and output plane, max |y - y64| over the run over max |y64| of that voice and plane over the
    run (the absolute error where that peak is 0); the largest over the planes.  NaN wherever y is not finite."""
    y = np.asarray(y, np.float64)
    assert y.shape == y64.shape, (y.shape, y64.shape)
    e = np.abs(y - y64).max(axis=(0, 3))
    p = np.abs(y64).max(axis=(0, 3))
    r = np.where(p > 0, e / np.where(p > 0, p, 1.0), e)
    return np.where(np.isfinite(y).all(axis=(0, 3)), r, np.nan).max(axis=0)


def rel_err(y: np.ndarray, y64: np.ndarray) -> float:
    """The error of a run: the largest per-voice error (NaN if any output is not finite, so no bound accepts it)."""
    r = rel_err_per_voice(y, y64)
    return float(np.nan) if np.isnan(r).any() else float(r.max())


def state_err(state: np.ndarray, run: F64Run, spec: GraphSpec) -> float:
    """The float state words against the float64 final state: per word, max over voices of |s - s64| over the peak
    |s64| of that word (absolute where the peak is 0); the largest over the words.  0 when there are none."""
    fl = ~int_slots(spec)
    if not fl.any():
        return 0.0
    s = np.asarray(state, np.uint32)[fl].view(np.float32).astype(np.float64)
    s64 = run.state_float[fl]
    if not np.isfinite(s).all():
        return float(np.nan)
    e = np.abs(s - s64).max(axis=1)
    p = np.abs(s64).max(axis=1)
    return float(np.where(p > 0, e / np.where(p > 0, p, 1.0), e).max())
