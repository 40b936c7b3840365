#!/usr/bin/env python
"""Config A's chain kernel against the copy ceiling of its own access pattern, in one run on one card.

    python tools/chain_ceiling.py [--launches 20] [--variants] [--kernel-only]

Prints JSON lines:
  * the card: name, power limit, current and maximum SM clock;
  * `tools/ubench/tma_copy.cu` (compiled into a temporary directory) at V = 65 536, T = 64: the full-block ring
    (mode 1, W = 12, S = 2: the chunked grid's shape) and the half-tile ring (mode 3, W = 16, S = 3: every group
    resident), each as a pure copy and with the kernel's LDS/STS row walk, and the spread of the warps' finish times;
  * `chain_kernel` on config A (65 536 voices x 64 blocks, contract R, mix bus on), exact and fast, with the planner's
    default launch shape: mean of `--launches` event-timed launches after 5 warm-ups.
    `--variants` adds launch shapes forced through the MLB_CHAIN_* overrides.
Bytes are the algorithmic ones of bench.py (8 B per voice-sample plus state and coefficients) over the data-sheet
3.35 TB/s of a 700 W H100 SXM.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

DATASHEET_GBS = 3350.0
V, T = 65536, 64
COPIES = [(1, 0, 12, 2), (1, 1, 12, 2), (3, 0, 16, 3), (3, 1, 16, 3), (3, 1, 12, 4)]
VARIANTS = [("resident, two time chunks", {"MLB_CHAIN_CHUNKS": "2"}),
            ("chunked grid: W = 12, five time chunks", {"MLB_CHAIN_WARPS": "12", "MLB_CHAIN_CHUNKS": "5"})]


def copy_ceiling(tmp):
    exe = os.path.join(tmp, "tma_copy")
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-o", exe,
                    os.path.join(ROOT, "tools", "ubench", "tma_copy.cu"), "-lcuda"], check=True)
    for mode, touch, w, s in COPIES:
        r = subprocess.run([exe, str(mode), str(touch), str(w), str(s), str(V), str(T)], capture_output=True,
                           text=True, check=True)
        line = json.loads(r.stdout.strip().splitlines()[-1])
        line["what"] = "tma_copy " + ("full-block ring" if mode == 1 else "half-tile ring") + \
            (" + LDS/STS row walk" if touch else "")
        line["frac_of_datasheet"] = line["gbs"] / DATASHEET_GBS
        print(json.dumps(line), flush=True)


def chain_kernel_ms(api, wl, torch, fast, launches, env):
    saved = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        dev = torch.device("cuda", 0)
        w = wl.config_a(V)
        g = api.VoiceGraph(w.spec, V, api.FLAG_FAST if fast else api.FLAG_EXACT)
        try:
            g.set_coefs(w.coef)
            g.set_state(w.state)
            d_in = torch.from_numpy(w.inputs(T)).to(dev)
            d_out = torch.empty((T, 1, V, 64), dtype=torch.float32, device=dev)
            d_mix = torch.empty((T, 1, 64), dtype=torch.float32, device=dev)
            sh = torch.cuda.current_stream().cuda_stream
            for _ in range(5):
                g.process_device(d_in, d_out, d_mix, T, sh)
            ms = []
            for _ in range(launches):
                g.process_device(d_in, d_out, d_mix, T, sh)
                ms.append(g.last_kernel_ms())
            torch.cuda.synchronize()
            return g.kernel_name, ms
        finally:
            g.close()
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=20)
    ap.add_argument("--variants", action="store_true", help="also time launch shapes forced through MLB_CHAIN_*")
    ap.add_argument("--kernel-only", action="store_true", help="skip the copy ceiling")
    args = ap.parse_args()
    from bench_configs import gpu_facts
    print(json.dumps(gpu_facts()), flush=True)
    if not args.kernel_only:
        with tempfile.TemporaryDirectory() as tmp:
            copy_ceiling(tmp)
    import torch

    from madronalib_b200 import api, workloads as wl
    api.init(0)
    alg = 2 * V * T * 64 * 4 + V * (2 * 3 * 4 + 4 * 4)
    shapes = [("planner default", {})] + (VARIANTS if args.variants else [])
    for label, env in shapes:
        for fast in (False, True):
            name, ms = chain_kernel_ms(api, wl, torch, fast, args.launches, env)
            mean = float(np.mean(ms))
            print(json.dumps({"what": "chain_kernel config A", "shape": label, "env": env, "kernel": name,
                              "ms_mean": mean, "ms_min": float(np.min(ms)), "ms_max": float(np.max(ms)),
                              "gbs": alg / (mean * 1e-3) / 1e9,
                              "frac_of_datasheet": alg / (mean * 1e-3) / 1e9 / DATASHEET_GBS}), flush=True)


if __name__ == "__main__":
    main()
