"""What the instrument stage costs in one 64-vector call of a synth with an instrument section.

The traced FxSynth (tests/cpp/fx_synth_body.h, case midi: 16 voices, an instrument section after the voice sum) for
4 096 instruments, wired by hand from its dump as TracedSynth::compile wires it, and the same voices reading the same
controllers and beat phase without a section (case fxplain: the same banks, planes and time chunks, the bus rows as
outputs).  FxSynth runs through mlb_synth_process_instrument_host, the plain synth through
mlb_synth_process_context_host with buses, so the two calls differ exactly by the instrument stage: the assembly kernel
in the bus sum's place, the instrument graph, and a third output plane.
  * The stages: the instrument graph alone on 64 vectors of its input planes, from CUDA events around it (the median
    of `--reps`); the assembly kernel (instrument_inputs_kernel) of one FxSynth call and the bus sum (bus_sum_kernel)
    of one plain call, summed over the call's time chunks, from torch.profiler's kernel records -- the assembly kernel
    has no entry point of its own to put events around.
  * The calls: after `--warmup` calls of each, the two alternate `--reps` times; the call time is the host clock around
    a call (it returns when its streams have drained), the median.
Prints one JSON line with the card's name and power limit.

    python tools/fx_synth_timing.py [--instruments 4096] [--blocks 64] [--reps 10] [--warmup 2]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from madronalib_b200 import api  # noqa: E402
from tests import fx_synth_cases as fc  # noqa: E402
from tests import synth_cases as sc  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--instruments", type=int, default=4096)
    ap.add_argument("--blocks", type=int, default=64)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import torch

    if api.device_count() < 1:
        raise SystemExit("fx_synth_timing: no CUDA device")
    api.init(0)
    G, T = a.instruments, a.blocks
    fx, base = fc.dump("midi"), fc.dump("fxplain")
    assert base["controllers"] == fx["controllers"] and base["phase"] == fx["phase"] and "instrument" not in base
    off, ev, toff, tr = sc.performance(fx, G, T, seed=1, density=0.3)
    bf, bb = fc.banks(api, fx, G), fc.banks(api, base, G)
    kw_f = dict(controllers=bf["controllers"], times=bf["times"], time_offsets=toff, transports=tr)
    kw_b = dict(controllers=bb["controllers"], times=bb["times"], time_offsets=toff, transports=tr)

    def call_fx():
        return bf["graph"].process_instrument_host(bf["instrument"], bf["routers"], bf["bank"], bf["buses"], off, ev,
                                                   **kw_f)

    def call_base():
        return bb["graph"].process_context_host(bb["routers"], bb["bank"], off, ev, buses=bb["buses"], **kw_b)

    try:
        for _ in range(a.warmup):
            call_fx(), call_base()
        t_fx, t_base = [], []
        for _ in range(a.reps):
            for f, acc in ((call_fx, t_fx), (call_base, t_base)):
                t0 = time.perf_counter()
                f()
                acc.append((time.perf_counter() - t0) * 1e3)
        n0 = api.kernel_launches()
        call_fx()
        launches_fx = api.kernel_launches() - n0
        n0 = api.kernel_launches()
        call_base()
        launches_base = api.kernel_launches() - n0

        # the instrument graph alone, on 64 vectors of input planes, CUDA events around it
        gi = bf["instrument"]
        planes = fx["instrument"]["planes"]
        inp = torch.randn((T, planes, G, 64), device="cuda") * 0.1
        out = torch.empty((T, gi.spec.n_out, G, 64), device="cuda")
        stream = torch.cuda.current_stream().cuda_stream
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        gi_ms = []
        for k in range(a.warmup + a.reps):
            e0.record()
            gi.process_device(inp, out, None, T, stream)
            e1.record()
            e1.synchronize()
            if k >= a.warmup:
                gi_ms.append(e0.elapsed_time(e1))

        # the assembly kernel and the bus sum of one call each, from the profiler's kernel records
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call_fx()
            call_base()
            torch.cuda.synchronize()
        kern = {}
        for e in prof.events():
            if e.device_type.name == "CUDA":
                for key in ("instrument_inputs_kernel", "bus_sum_kernel"):
                    if key in e.name:
                        kern[key] = kern.get(key, 0.0) + e.device_time_total / 1e3
        kernel = gi.kernel_name
    finally:
        fc.close(bf), fc.close(bb)
    print(json.dumps({
        "card": card(), "instruments": G, "voices": fx["n_voices"], "blocks": T,
        "instrument_graph_ms": statistics.median(gi_ms), "instrument_kernel": kernel,
        "assembly_kernel_ms": kern.get("instrument_inputs_kernel"), "bus_sum_kernel_ms": kern.get("bus_sum_kernel"),
        "fx_call_ms": statistics.median(t_fx), "plain_call_ms": statistics.median(t_base),
        "fx_launches": launches_fx, "plain_launches": launches_base,
        "instrument_planes": planes, "reps": a.reps,
    }))


if __name__ == "__main__":
    main()
