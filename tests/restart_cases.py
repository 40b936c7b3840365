"""Shared by tests/test_restart.py and tests/test_gpu_restart.py: what a restarted instrument must produce, built from
runs of the unchanged reference (or port) over slices of a performance, and the driver of TracedSynth::restart."""
import os
import subprocess

import numpy as np

from madronalib_b200 import api
from tests import synth_cases as sc

ROOT = sc.ROOT
EXE = os.path.join(ROOT, "tests", "cpp", "test_synth_restart")


def slice_from(offsets, items, t0: int):
    """Blocks [t0, T) of a CSR list, offsets [T][G + 1] into items: (offsets rebased to 0, items from there)."""
    return offsets[t0:] - offsets[t0, 0], items[offsets[t0, 0]:]


def expected(run, off, ev, toff, tr, restarts):
    """The bus rows of G instruments with restarts {t: [instruments]} before vector t.  run(off, ev, toff, tr) -> bus
    [T][n_out][G][64] runs objects created at the first vector of what it is fed, so a restarted instrument g at t is
    run's instrument g over the slice [t, T): its rows before t come from the run over everything (or an earlier
    slice), the rest from the slice."""
    want = run(off, ev, toff, tr).copy()
    for t in sorted(restarts):
        if not restarts[t]:
            continue
        o, e = slice_from(off, ev, t)
        to, r = slice_from(toff, tr, t)
        part = run(o, e, to, r)
        for g in set(restarts[t]):
            want[t:, :, g] = part[:, :, g]
    return want


def build_exe():
    sc.build_exe()
    libdir = os.path.dirname(api.LIB_PATH)
    src = os.path.join(ROOT, "tests", "cpp", "test_synth_restart.cpp")
    deps = [src, os.path.join(ROOT, "tests", "cpp", "synth_body.h")]
    deps += [os.path.join(ROOT, "include", h) for h in ("mlb200_trace.hpp", "mlb200.hpp", "mlb200_host.hpp", "mlb200.h")]
    if os.path.exists(EXE) and all(os.path.getmtime(EXE) > os.path.getmtime(p) for p in deps):
        return
    cmd = ["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), src, "-o", EXE,
           "-L", libdir, "-lmlb200", "-Wl,-rpath," + libdir]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]


def run(tmp_path, case, G, T, off, ev, toff, tr, splits, restarts):
    """TracedSynth over calls of `splits` vectors, restarting {t: [instruments]} before the call that starts at t ->
    (bus [T][2][G][64], launches per call, launches per restart)."""
    build_exe()
    for name, a in (("offsets", off), ("events", ev), ("toff", toff), ("tr", tr)):
        np.ascontiguousarray(a).tofile(str(tmp_path / (name + ".bin")))
    spec = ",".join(f"{t}:" + "+".join(map(str, gs)) for t, gs in sorted(restarts.items()))
    r = subprocess.run([EXE, "run", case, str(G), str(T), str(tmp_path), ",".join(map(str, splits)), spec],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr

    def counts(key):
        s = r.stdout.split(key)[1].split("\n")[0].strip()
        return [int(n) for n in s.split(",")] if s else []
    bus = np.fromfile(str(tmp_path / "bus.bin"), np.float32).reshape(T, 2, G, 64)
    return bus, counts("launches per call: "), counts("launches per restart: ")
