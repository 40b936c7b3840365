"""Wall time of restarting instruments of a running synth bank, beside the time of one 64-vector call.

The traced `synth_body` Synth (tests/cpp/synth_body.h, case midi: 16 voices) for 4 096 instruments, wired by hand from
its dump as TracedSynth::compile wires it.  After a warm-up call, each of the banks that TracedSynth::restart resets
(routers, Voice rows, controllers, beat phase, graph) is reset for the first 1, 64 and 4 096 instruments, as
TracedSynth::restart does: five synchronous calls, one launch each.  The time is the host clock around those calls
(each returns when its launch has finished), the median of `--reps`.  The bytes are the state words the resets write,
from the banks' layouts (DESIGN.md "Restart").  Prints one JSON line with the card's name and power limit.

    python tools/restart_timing.py [--instruments 4096] [--reps 20]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from madronalib_b200 import api  # noqa: E402
from tests import synth_cases as sc  # noqa: E402

VS_COUNT, VG_COUNT = 47, 7        # Voice bank state words and LinearGlide rows per voice (voice_kernel.cuh)
ROUTER_WORDS = 14 * 32 + 31       # every router word of an instrument but its two counters (router_kernel.cuh)
CTRL_WORDS, PT_WORDS = 4 + 64, 20  # per controller: 4 state words and a row; 10 64-bit clock words


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--instruments", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    api.lib()
    assert api.device_count() > 0, "no CUDA device: restart timings are measured on the GPU only"
    api.init(0)
    d = sc.dump("midi")
    G, T = args.instruments, 64
    lay = sc.layout(d, G)
    V = lay["n_voices"]
    spec, coef, state = sc.graph(d, G)
    off, ev, toff, tr = sc.performance(d, G, T, seed=1, density=0.3)
    r = api.RouterBank(lay["polyphony"], lay["first_voice"], V, 0, unison=np.full(G, d["unison"]),
                       mod_cc=np.full(G, d["mod_cc"]))
    vb = api.VoiceBank(float(sc.SR), lay["voice_index"], np.full(V, d["glide_seconds"], np.float32),
                       np.full(V, d["drift_amount"], np.float32), np.full(V, d["pitch_bend"], np.float32),
                       flags=api.VoiceBank.MIDI)
    cb = api.ControllerBank(G, d["controllers"], float(sc.SR), 0)
    cb.set_voice_map(lay["voice_instrument"])
    pt = api.ProcessTimeBank(G, float(sc.SR))
    pt.set_voice_map(lay["voice_instrument"])
    g = api.VoiceGraph(spec, V)
    g.set_coefs(coef)
    g.set_state(state)
    buses = api.Buses(V, lay["first_voice"].astype(np.int32), np.full(G, d["n_voices"], np.int32))
    NR = V // G

    def call():
        t0 = time.perf_counter()
        g.process_context_host(r, vb, off, ev, controllers=cb, times=pt, time_offsets=toff, transports=tr,
                               buses=buses)
        return time.perf_counter() - t0

    def restart(inst):
        lanes = (inst[:, None] * NR + np.arange(NR)[None, :]).reshape(-1)
        t0 = time.perf_counter()
        r.reset(inst)
        vb.reset(lanes)
        cb.reset(inst)
        pt.reset(inst)
        g.reset_voices(lanes)
        return time.perf_counter() - t0

    call()
    call_ms = 1e3 * float(np.median([call() for _ in range(max(3, args.reps // 4))]))
    per_lane = VS_COUNT + VG_COUNT * 64 + spec.n_state + g.delay_bytes // (4 * V)
    per_inst = ROUTER_WORDS + len(d["controllers"]) * CTRL_WORDS + PT_WORDS + NR * per_lane
    out = {"card": card(), "instruments": G, "voices_per_instrument": NR, "call_64_vectors_ms": round(call_ms, 3),
           "restart": []}
    for n in (1, 64, G):
        inst = np.arange(n, dtype=np.int32)
        restart(inst)
        n0 = api.kernel_launches()
        ms = 1e3 * float(np.median([restart(inst) for _ in range(args.reps)]))
        launches = (api.kernel_launches() - n0) // args.reps
        out["restart"].append({"instruments": n, "wall_ms": round(ms, 4), "bytes": int(n * per_inst * 4),
                               "launches": int(launches)})
    for h in (r, vb, cb, pt, g, buses):
        h.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
