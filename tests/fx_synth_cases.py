"""Shared by tests/test_fx_synth.py and tests/test_gpu_fx_synth.py: the traced Synth subclass of
tests/cpp/fx_synth_body.h, which overrides processVector (tests/cpp/test_fx_synth), and its banks run through the CPU
stages: the voice graph through the port, the bus sum, the instrument graph through the port."""
import json
import os
import subprocess

import numpy as np

from madronalib_b200 import api
from madronalib_b200.graph import OP_NAME, GraphSpec
from tests import synth_cases as sc

ROOT = sc.ROOT
EXE = os.path.join(ROOT, "tests", "cpp", "test_fx_synth")
SR = sc.SR


def build_exe():
    from madronalib_b200 import build
    if not os.path.exists(api.LIB_PATH):
        build.build()
    libdir = os.path.dirname(api.LIB_PATH)
    src = os.path.join(ROOT, "tests", "cpp", "test_fx_synth.cpp")
    deps = [src] + [os.path.join(ROOT, "tests", "cpp", h) for h in ("fx_synth_body.h", "synth_body.h")]
    deps += [os.path.join(ROOT, "include", h) for h in ("mlb200_trace.hpp", "mlb200.hpp", "mlb200_host.hpp", "mlb200.h")]
    if os.path.exists(EXE) and all(os.path.getmtime(EXE) > os.path.getmtime(p) for p in deps):
        return
    cmd = ["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), src, "-o", EXE,
           "-L", libdir, "-lmlb200", "-Wl,-rpath," + libdir]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]


def dump_text(case: str) -> str:
    build_exe()
    r = subprocess.run([EXE, "dump", case], capture_output=True, text=True, timeout=60)
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout


def dump(case: str) -> dict:
    return json.loads(dump_text(case))


def instrument_graph(d: dict):
    """-> (GraphSpec, coef [n_coef][G], state [n_state][G]) of the instrument graph of the dump, for G = 1 (the words
    are the same for every instrument)."""
    ig = d["instrument"]
    g = GraphSpec()
    coef, state = [], []
    for n in ig["nodes"]:
        g.ops.append(n["op"])
        g.ins.append(tuple(n["in"]))
        g.iargs.append(n["iarg"])
        coef += n["coef"]
        state += n["state"]
    g.outs = list(ig["outs"])
    coef = np.array(coef, np.uint32).view(np.float32).reshape(-1, 1)
    state = np.array(state, np.uint32).reshape(-1, 1)
    assert coef.shape[0] == g.n_coef and state.shape[0] == g.n_state
    return g, coef, state


def instrument_inputs(d: dict, bus, time_offsets, transports, offsets, events):
    """The instrument graph's input planes [T][P + C + phase][G][64]: the bus rows, then each instrument's controllers
    and beat phase, as the port computes them."""
    from oracle import ctrl_bindings, ptime_bindings
    from tests.router_cases import route_on_host
    T, P, G = bus.shape[0], bus.shape[1], bus.shape[2]
    C = len(d["controllers"])
    inp = np.zeros((T, d["instrument"]["planes"], G, 64), np.float32)
    inp[:, :P] = bus
    if C:
        lay = sc.layout(d, G)
        _, coff, ch, _, _ = route_on_host(offsets, events, lay, bool(d["mpe"]), unison=np.full(G, d["unison"]),
                                          mod_cc=np.full(G, d["mod_cc"]))
        c, _, _ = ctrl_bindings.port_controllers(G, d["controllers"], coff, ch, float(SR))
        inp[:, P:P + C] = c
    if d["phase"]:
        p, _ = ptime_bindings.port_process_time(G, time_offsets, transports, float(SR))
        inp[:, P + C] = p
    return inp


def port_stages(d: dict, G: int, offsets, events, time_offsets, transports, port):
    """The traced synth through the CPU stages: synth_cases.port_stages (routers -> Voice bank -> controllers -> beat
    phase -> voice graph -> buses), then the instrument graph through the port.  -> [T][outputs][G][64]."""
    # synth_cases.port_stages feeds the voice graph every plane up to the beat phase; here the voice graph may read
    # fewer (the instrument section reads the others), so it gets the controllers up to the last one it reads
    C = len(d["controllers"])
    planes = [n["iarg"] for n in d["nodes"] if OP_NAME[n["op"]] == "INPUT"]
    vd = dict(d)
    if 8 + C not in planes:
        vd["phase"], vd["controllers"] = 0, d["controllers"][:max(0, max(planes) + 1 - 8)]
    bus = sc.port_stages(vd, G, offsets, events, time_offsets, transports, port)
    spec, coef, state = instrument_graph(d)
    inp = instrument_inputs(d, bus, time_offsets, transports, offsets, events)
    out, _, _ = port.run(spec, G, bus.shape[0], inp, np.repeat(state, G, axis=1), np.repeat(coef, G, axis=1))
    return out


def run(tmp_path, case, G, T, off, ev, toff, tr, splits, restart=None, env=None):
    """TracedSynth over calls of `splits` vectors (restarting the instruments `restart` after the first call) ->
    (bus [T][outputs][G][64], launches per call, stdout)."""
    build_exe()
    for name, a in (("offsets", off), ("events", ev), ("toff", toff), ("tr", tr)):
        np.ascontiguousarray(a).tofile(str(tmp_path / (name + ".bin")))
    args = [EXE, "run", case, str(G), str(T), str(tmp_path), ",".join(map(str, splits))]
    if restart is not None:
        args.append(",".join(map(str, restart)))
    r = subprocess.run(args, capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0, r.stdout + r.stderr
    launches = [int(n) for n in r.stdout.split("launches per call: ")[1].split()[0].split(",")]
    bus = np.fromfile(str(tmp_path / "bus.bin"), np.float32)
    return bus.reshape(T, -1, G, 64), launches, r.stdout


def banks(gpu, d: dict, G: int) -> dict:
    """The banks of the traced synth built by hand from its dump, as TracedSynth::compile builds them (`gpu`: the api
    module): routers, Voice bank, controllers, beat phase, voice graph, buses, and the instrument graph if any."""
    lay = sc.layout(d, G)
    V, mpe = lay["n_voices"], bool(d["mpe"])
    spec, coef, state = sc.graph(d, G)
    pb = np.full(V, d["pitch_bend"], np.float32)
    if mpe:
        pb[lay["main_voice"] >= 0] = np.float32(d["mpe_pitch_bend"])
    r = gpu.RouterBank(lay["polyphony"], lay["first_voice"], V, int(mpe), unison=np.full(G, d["unison"]),
                       mod_cc=np.full(G, d["mod_cc"]))
    vb = gpu.VoiceBank(float(sc.SR), lay["voice_index"], np.full(V, d["glide_seconds"], np.float32),
                       np.full(V, d["drift_amount"], np.float32), pb, flags=0 if mpe else gpu.VoiceBank.MIDI)
    if mpe:
        vb.set_main_voices(lay["main_voice"])
    cb = gpu.ControllerBank(G, d["controllers"], float(sc.SR), int(mpe))
    cb.set_voice_map(lay["voice_instrument"])
    pt = gpu.ProcessTimeBank(G, float(sc.SR))
    pt.set_voice_map(lay["voice_instrument"])
    g = gpu.VoiceGraph(spec, V)
    g.set_coefs(coef)
    g.set_state(state)
    buses = gpu.Buses(V, (lay["first_voice"] + d["mpe"]).astype(np.int32), np.full(G, d["n_voices"], np.int32))
    b = dict(routers=r, bank=vb, controllers=cb, times=pt, graph=g, buses=buses)
    if "instrument" in d:
        ispec, icoef, istate = instrument_graph(d)
        b["instrument"] = gpu.VoiceGraph(ispec, G)
        b["instrument"].set_coefs(np.repeat(icoef, G, axis=1))
        b["instrument"].set_state(np.repeat(istate, G, axis=1))
    return b


def close(banks: dict) -> None:
    for b in banks.values():
        b.close()
