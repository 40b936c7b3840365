"""Shared helpers of the published-signal tests: the traced body of tests/cpp/published_body.h
(tests/cpp/test_published_trace.cpp) and a run of it on the GPU."""
import json
import os
import subprocess

import numpy as np

from madronalib_b200 import api

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "cpp", "test_published_trace")
SIGNALS, READ_WIDTH = 3, 200  # kPublishSignals, kPublishReadWidth


def build_exe():
    from madronalib_b200 import build
    if not os.path.exists(api.LIB_PATH):
        build.build()
    libdir = os.path.dirname(api.LIB_PATH)
    src = os.path.join(ROOT, "tests", "cpp", "test_published_trace.cpp")
    deps = [src, os.path.join(ROOT, "tests", "cpp", "published_body.h")]
    deps += [os.path.join(ROOT, "include", h) for h in ("mlb200_trace.hpp", "mlb200.hpp", "mlb200_host.hpp", "mlb200.h")]
    if os.path.exists(EXE) and all(os.path.getmtime(EXE) > os.path.getmtime(p) for p in deps):
        return
    cmd = ["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), src, "-o", EXE,
           "-L", libdir, "-lmlb200", "-Wl,-rpath," + libdir]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]


def trace(case: str):
    """(returncode, stdout) of `test_published_trace dump <case>`."""
    build_exe()
    r = subprocess.run([EXE, "dump", case], capture_output=True, text=True, timeout=60)
    return r.returncode, r.stdout + r.stderr


def dump(case: str) -> dict:
    rc, out = trace(case)
    assert rc == 0, out
    return json.loads(out)


def run(tmp_path, case, G, T, off, ev, splits, chunk_blocks=None):
    """The traced synth on the GPU in calls of `splits` vectors -> (bus, counts, dest, launches per call)."""
    build_exe()
    for name, a in (("offsets", off), ("events", ev)):
        np.ascontiguousarray(a).tofile(str(tmp_path / (name + ".bin")))
    env = dict(os.environ)
    if chunk_blocks:
        env["MLB_SYNTH_CHUNK_BLOCKS"] = str(chunk_blocks)
    r = subprocess.run([EXE, "run", case, str(G), str(T), str(tmp_path), ",".join(map(str, splits))],
                       capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0, r.stdout + r.stderr
    launches = [int(n) for n in r.stdout.split("launches per call: ")[1].split()[0].split(",")]
    bus = np.fromfile(str(tmp_path / "bus.bin"), np.float32).reshape(T, 2, G, 64)
    counts = np.fromfile(str(tmp_path / "counts.bin"), np.int32)
    dest = np.fromfile(str(tmp_path / "dest.bin"), np.float32)
    if case != "nostore":
        counts = counts.reshape(len(splits), SIGNALS, G)
        dest = dest.reshape(len(splits), SIGNALS, G, READ_WIDTH)
    return bus, counts, dest, launches
