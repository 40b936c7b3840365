"""Shared by tests/test_synth_trace.py and tests/test_gpu_synth_trace.py: the traced Synth subclass of
tests/cpp/synth_body.h (tests/cpp/test_synth_trace), its performances, and its bank run through the CPU stages."""
import ctypes
import json
import os
import subprocess

import numpy as np

from madronalib_b200 import api, workloads as wl
from madronalib_b200.graph import GraphSpec

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "cpp", "test_synth_trace")
SR = 48000


def build_exe():
    from madronalib_b200 import build
    if not os.path.exists(api.LIB_PATH):
        build.build()
    libdir = os.path.dirname(api.LIB_PATH)
    src = os.path.join(ROOT, "tests", "cpp", "test_synth_trace.cpp")
    deps = [src, os.path.join(ROOT, "tests", "cpp", "synth_body.h")]
    deps += [os.path.join(ROOT, "include", h) for h in ("mlb200_trace.hpp", "mlb200.hpp", "mlb200_host.hpp", "mlb200.h")]
    if os.path.exists(EXE) and all(os.path.getmtime(EXE) > os.path.getmtime(p) for p in deps):
        return
    cmd = ["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), src, "-o", EXE,
           "-L", libdir, "-lmlb200", "-Wl,-rpath," + libdir]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]


def dump(case: str) -> dict:
    build_exe()
    r = subprocess.run([EXE, "dump", case], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stdout + r.stderr
    return json.loads(r.stdout)


def layout(d: dict, G: int):
    return wl.midi_layout(G, d["polyphony"], bool(d["mpe"]))


def lane_voice(d: dict, G: int) -> np.ndarray:
    """The synth voice whose words each lane gets (the MPE main voice and voices past getNumVoices(): voice 0)."""
    NR = d["polyphony"] + d["mpe"]
    v = np.tile(np.arange(NR) - d["mpe"], G)
    return np.where((v >= 0) & (v < d["n_voices"]), v, 0)


def graph(d: dict, G: int):
    """-> (GraphSpec, coef [n_coef][V], state [n_state][V]) of the traced bank over every lane of G instruments."""
    g = GraphSpec()
    coef_rows, state_rows = [], []
    for n in d["nodes"]:
        g.ops.append(n["op"])
        g.ins.append(tuple(n["in"]))
        g.iargs.append(n["iarg"])
        coef_rows += [list(w) for w in zip(*n["coef"])]    # [word][voice]
        state_rows += [list(w) for w in zip(*n["state"])]
    g.outs = list(d["outs"])
    lv = lane_voice(d, G)
    coef = np.array(coef_rows, np.uint32).reshape(-1, d["n_voices"])[:, lv].view(np.float32)
    state = np.array(state_rows, np.uint32).reshape(-1, d["n_voices"])[:, lv]
    assert coef.shape[0] == g.n_coef and state.shape[0] == g.n_state
    return g, np.ascontiguousarray(coef), np.ascontiguousarray(state)


def _rebuild(offsets, events, fn):
    """The CSR list with block t's events of instrument g replaced by fn(t, g, events)."""
    T, G = offsets.shape[0], offsets.shape[1] - 1
    off = np.zeros_like(offsets)
    parts, n = [np.zeros(0, api.EVENT_DTYPE)], 0
    for t in range(T):
        for g in range(G):
            off[t, g] = n
            seg = fn(t, g, events[offsets[t, g]:offsets[t, g + 1]])
            parts.append(seg)
            n += seg.size
        off[t, G] = n
    return off, np.concatenate(parts)


def performance(d: dict, G: int, T: int, seed: int, late=None, never=None, density=0.5):
    """A performance of G instruments for the traced case `d`: raw events (stealing, pedal, bend, pressure, CC 1 / 74
    moves, CC 123), a host transport with stops and jumps, instrument `late` silent before vector T // 3, `never`
    silent throughout.  In unison every note event goes to every voice, whose record holds MLB_VOICE_MAX_EVENTS (4)
    per vector: there a vector keeps at most 2 note-ons and note-offs and no CC 123 or pedal (a pedal release or a
    CC 123 writes note-offs of its own).  Returns (offsets, events, time_offsets, transports)."""
    mpe = bool(d["mpe"])
    offsets, ev = wl.midi_performance(G, T, d["polyphony"], mpe, density=density, seed=seed)

    def fn(t, g, seg):
        if g == never or (g == late and t < T // 3):
            return seg[:0]
        if d["unison"]:
            seg = seg[(seg["type"] != 5) & ~((seg["type"] == 6) & (seg["source_idx"] == 123))]
            note = (seg["type"] == 1) | (seg["type"] == 4)
            seg = seg[~note | (np.cumsum(note) <= 2)]
        return seg
    offsets, ev = _rebuild(offsets, ev, fn)
    toff, tr = wl.transport_updates(G, T, float(SR), seed=seed + 1, every=1, chaos=0.2)
    return offsets, ev, toff, tr


def _port_voice_rows(d, lay, rec):
    from oracle import bindings
    L = bindings.port_voice_bank().lib
    L.mlport_bank_create.restype = ctypes.c_void_p
    L.mlport_bank_create.argtypes = [ctypes.c_int, ctypes.c_float] + [ctypes.c_void_p] * 4 + [ctypes.c_uint]
    L.mlport_bank_set_main_voices.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    L.mlport_bank_process.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
    L.mlport_bank_process.restype = ctypes.c_double
    L.mlport_bank_destroy.argtypes = [ctypes.c_void_p]
    V, T = lay["n_voices"], rec.shape[0]
    vi = np.ascontiguousarray(lay["voice_index"], np.int32)
    gs = np.full(V, d["glide_seconds"], np.float32)
    da = np.full(V, d["drift_amount"], np.float32)
    pb = np.full(V, d["pitch_bend"], np.float32)
    if d["mpe"]:
        pb[lay["main_voice"] >= 0] = np.float32(d["mpe_pitch_bend"])
    vp = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    h = L.mlport_bank_create(V, float(SR), vp(vi), vp(gs), vp(da), vp(pb), 0 if d["mpe"] else wl.VOICES_MIDI)
    try:
        if d["mpe"]:
            L.mlport_bank_set_main_voices(h, vp(np.ascontiguousarray(lay["main_voice"], np.int32)))
        out = np.zeros((T, 8, V, 64), np.float32)
        r = np.ascontiguousarray(rec)
        L.mlport_bank_process(h, T, vp(r), vp(out), 1)
    finally:
        L.mlport_bank_destroy(h)
    return out


def port_stages(d: dict, G: int, offsets, events, time_offsets, transports, port):
    """The traced bank through the CPU stages one after another: host routers -> port Voice bank -> port controllers ->
    port beat phase -> port graph -> port buses.  -> bus [T][n_out][G][64]."""
    from oracle import bus_bindings, ctrl_bindings, ptime_bindings
    from tests.router_cases import route_on_host
    lay = layout(d, G)
    V, T = lay["n_voices"], offsets.shape[0]
    mpe = bool(d["mpe"])
    rec, coff, ch, _, _ = route_on_host(offsets, events, lay, mpe, unison=np.full(G, d["unison"]),
                                        mod_cc=np.full(G, d["mod_cc"]))
    spec, coef, state = graph(d, G)
    C = len(d["controllers"])
    inp = np.zeros((T, spec.n_in, V, 64), np.float32)
    rows = _port_voice_rows(d, lay, rec)
    inp[:, :min(8, spec.n_in)] = rows[:, :min(8, spec.n_in)]
    inst = lay["voice_instrument"]
    if C:
        c, _, _ = ctrl_bindings.port_controllers(G, d["controllers"], coff, ch, float(SR))
        inp[:, 8:8 + C] = c[:, :, inst]
    if d["phase"]:
        p, _ = ptime_bindings.port_process_time(G, time_offsets, transports, float(SR))
        inp[:, 8 + C] = p[:, inst]
    out, _, _ = port.run(spec, V, T, inp, state, coef)
    first = (lay["first_voice"] + d["mpe"]).astype(np.int32)
    return bus_bindings.port_buses(out, first, np.full(G, d["n_voices"], np.int32))
