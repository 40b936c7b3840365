#!/usr/bin/env python
"""Kernel-resident timing of everything except the headline: BASELINE.json configurations 2-5, the
SURVEY 8(f) workloads (config 6 = Aaltoverb x V, the EventsToSignals::Voice bank) and the elementwise maps.

    python tools/bench_configs.py [--steps K] [--only 2,3,4,5,6,voices,map,fdtd,buses,controllers,router,routed,
                                   process_time,context] [--generic] [--cpu]

Prints one JSON line per configuration: kernel name, mean CUDA-event kernel time, algorithmic
bytes per launch (SURVEY.md 8d / DESIGN.md), achieved GB/s and fraction of the measured HBM peak.
--cpu also times the reference (oracle/_ref) on the box's host cores for config 6, the Voice bank and the FDTD
membranes.  The FDTD lines (K9) are compute-bound: they report instance-samples/s and the share of the FP32 issue
ceiling instead of bytes.  The bus lines (K10) report bytes against the data-sheet HBM bandwidth, and contract E
with bus output against the rows-out and mix-only paths in voice-samples/s.  The beat-phase lines (K13) report
voice-samples/s and bytes against the data-sheet HBM bandwidth, and contract E with every AudioContext signal against
the routed entry point on the same performance.
Not the headline benchmark (that is bench.py / config A).
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch

    from madronalib_b200 import api, workloads as wl
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--only", default="2,3,swept,4,5,6,voices,map,fdtd,buses,controllers,router,routed,process_time,"
                                      "context")
    ap.add_argument("--generic", action="store_true", help="force the graph interpreter kernel")
    ap.add_argument("--cpu", action="store_true",
                    help="also time the reference (oracle/_ref, all host threads) on config 6, the Voice bank "
                         "and the FDTD membranes")
    args = ap.parse_args()
    only = set(args.only.split(","))
    api.init(0)
    try:
        peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]
    except Exception:
        peak = 6650.0
    dev = torch.device("cuda", 0)
    cfgs = []
    if "2" in only:
        for kind in ("lopass", "hipass", "bell"):
            cfgs.append(("config2_" + kind, wl.config_2(kind, 4096), 64, lambda V, T: 8.0 * V * T * 64))
    if "3" in only:
        cfgs.append(("config3", wl.config_3(65536), 64, lambda V, T: 8.0 * V * T * 64))
    if "swept" in only:
        # the swept headline chain: SineGen -> Lopass(coefficient ROWS g0, g1, g2) -> gain; per voice-sample
        # 4 B freq + 3 x 4 B coefficient rows in + 4 B out = 20 B (MLDSPFilters.h:136-152 after makeCoeffsVec)
        cfgs.append(("configA_swept", wl.swept_filter_case("sine_lopass_v_gain", 65536, 16), 16,
                     lambda V, T: 20.0 * V * T * 64))
    if "4" in only:
        # ring 8 x (256 B r + 256 B w) + freq row in + 2 rows out per voice-block = 4864 B
        cfgs.append(("config4", wl.config_4(16384), 16, lambda V, T: 4864.0 * V * T))
    if "5" in only:
        cfgs.append(("config5", wl.config_5(1024, 256), 16, lambda V, T: 256.0 * V * T))
    if "6" in only:
        # Aaltoverb x V (SURVEY 8f row 2).  Per reverb-block: 12 rings x (256 B write + 256 B read: the two
        # taps of a PitchbendableDelay sit within a sample of each other) + 10 vy1 rows r/w + 2 feedback
        # rows r/w + 2 glide rows read + 2 rows in + 2 rows out = 13824 B
        for V6 in (4096, 16384):
            cfgs.append(("config6_aaltoverb", wl.config_6(V6), 16, lambda V, T: 13824.0 * V * T))
    if "map" in only:
        # K3: stateless elementwise ops, n_rows x 64 elements resident in HBM
        n_rows = 1 << 20  # 64 Mi elements = 256 MB per operand (> L2)
        x1 = torch.rand((n_rows, 64), dtype=torch.float32, device=dev) * 4 - 2
        x2 = torch.rand((n_rows, 64), dtype=torch.float32, device=dev) + 0.5
        x3 = torch.rand((n_rows, 64), dtype=torch.float32, device=dev)
        y = torch.empty_like(x1)
        sh = torch.cuda.current_stream().cuda_stream
        for op, nin in (("multiply", 2), ("sin", 1), ("exp", 1), ("log", 1), ("sin_approx", 1),
                        ("pow", 2), ("lerp", 3), ("clamp", 3)):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            for _ in range(3):
                api.map_device(op, x1, x2 if nin > 1 else None, x3 if nin > 2 else None, y, n_rows, sh)
            e0.record()
            for _ in range(args.steps):
                api.map_device(op, x1, x2 if nin > 1 else None, x3 if nin > 2 else None, y, n_rows, sh)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / args.steps
            b = (nin + 1) * n_rows * 64 * 4.0
            print(json.dumps({"config": "map_" + op, "kernel": "map_kernel", "rows": n_rows, "kernel_ms": ms,
                              "algorithmic_bytes": b, "achieved_gbs": b / (ms * 1e-3) / 1e9,
                              "frac_of_measured_hbm_peak": b / (ms * 1e-3) / 1e9 / peak}), flush=True)
        del x1, x2, x3, y
    if "voices" in only:
        # K7: EventsToSignals::Voice x V (SURVEY 8f row 3).  Per voice-block: 72 B record in, selected rows out.
        V7, T7 = 65536, 64
        # a busy performance: a voice gets note events in 10 % of its vectors, controller moves in 5 %
        ev = wl.voice_events(256, T7, seed=2, density=0.10, ctl=0.05)
        ev = np.ascontiguousarray(np.tile(ev, (1, V7 // 256)))
        prm = wl.voice_bank_params(V7)
        d_ev = torch.from_numpy(ev.view(np.uint8).reshape(T7, V7, 72)).to(dev)
        d_rows = torch.empty((T7, 8, V7, 64), dtype=torch.float32, device=dev)
        sh = torch.cuda.current_stream().cuda_stream
        for mask, label in ((0x03, "pitch+gate"), (0xFF, "all 8 rows")):
            vb = api.VoiceBank(48000.0, *prm)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            for _ in range(2):
                vb.process_device(d_ev, d_rows, T7, mask, sh)
            e0.record()
            for _ in range(args.steps):
                vb.process_device(d_ev, d_rows, T7, mask, sh)
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / args.steps
            b = (72.0 + 256.0 * bin(mask).count("1")) * V7 * T7
            print(json.dumps({"config": "voices_" + label, "kernel": "voice_bank_kernel", "voices": V7, "blocks": T7,
                              "kernel_ms": ms, "voice_samples_per_s": V7 * T7 * 64 / (ms * 1e-3),
                              "algorithmic_bytes": b, "achieved_gbs": b / (ms * 1e-3) / 1e9,
                              "frac_of_measured_hbm_peak": b / (ms * 1e-3) / 1e9 / peak}), flush=True)
            vb.close()
        del d_ev, d_rows
    if "fdtd" in only:
        bench_fdtd(api, wl, torch, dev, args.steps, args.cpu)
    if "buses" in only:
        bench_buses(api, wl, torch, dev, args.steps)
    if "controllers" in only:
        bench_controllers(api, wl, torch, dev, args.steps)
    if "router" in only:
        bench_router(api, wl, torch, dev, args.steps)
    if "routed" in only:
        bench_routed(api, wl, torch)
    if "process_time" in only:
        bench_process_time(api, wl, torch, dev, args.steps)
    if "context" in only:
        bench_context(api, wl, torch)
    if args.cpu:
        # the reference itself on this box's host cores (oracle/_ref; checker code, used here only as a baseline)
        import time
        from oracle import bindings as ob
        cores = os.cpu_count() or 1
        if "6" in only:
            R = ob.RefOracle()
            w = wl.config_6(1024)
            inp = w.inputs(16)
            best = 1e30
            for _ in range(3):
                t0 = time.perf_counter()
                R.run(w.spec, w.n_voices, 16, inp, w.state, w.coef, want_out=True, nthreads=cores)
                best = min(best, time.perf_counter() - t0)
            print(json.dumps({"config": "config6_aaltoverb_reference_cpu", "threads": cores, "voices": 1024, "blocks": 16,
                              "seconds": best, "voice_samples_per_s": 1024 * 16 * 64 / best,
                              "note": "reference functors behind the graph interpreter of oracle/ref/mlref.cpp, "
                                      "includes building the per-voice functor objects"}), flush=True)
        if "voices" in only:
            B = ob.ref_voice_bank()
            Vc, Tc = 8192, 64
            ev = np.ascontiguousarray(np.tile(wl.voice_events(256, Tc, seed=2, density=0.10, ctl=0.05), (1, Vc // 256)))
            out, sec = B.run(48000.0, *wl.voice_bank_params(Vc), ev, nthreads=cores)
            print(json.dumps({"config": "voices_reference_cpu", "threads": cores, "voices": Vc, "blocks": Tc,
                              "seconds": sec, "voice_samples_per_s": Vc * Tc * 64 / sec,
                              "note": "the reference's own EventsToSignals::Voice (oracle/_ref/libmle2s.so)"}), flush=True)
    for name, w, T, alg in cfgs:
        V = w.n_voices
        g = api.VoiceGraph(w.spec, V, api.FLAG_FORCE_GENERIC if args.generic else 0)
        g.set_coefs(w.coef)
        g.set_state(w.state)
        inp = w.inputs(T)
        d_in = torch.from_numpy(inp).to(dev) if inp is not None else None
        d_out = torch.empty((T, w.spec.n_out, V, 64), dtype=torch.float32, device=dev)
        torch.cuda.synchronize()
        sh = torch.cuda.current_stream().cuda_stream
        for _ in range(3):
            g.process_device(d_in, d_out, None, T, sh)
        ms = []
        for _ in range(args.steps):
            g.process_device(d_in, d_out, None, T, sh)
            ms.append(g.last_kernel_ms())
        kms = float(np.mean(ms))
        b = alg(V, T)
        print(json.dumps({"config": name, "kernel": g.kernel_name, "voices": V, "blocks": T,
                          "kernel_ms": kms, "voice_samples_per_s": V * T * 64 / (kms * 1e-3),
                          "algorithmic_bytes": b, "achieved_gbs": b / (kms * 1e-3) / 1e9,
                          "frac_of_measured_hbm_peak": b / (kms * 1e-3) / 1e9 / peak,
                          "delay_memory_mb": g.delay_bytes / 1e6}), flush=True)
        g.close()
        del d_in, d_out


# K9's arithmetic, counted from the example's text (fdtd.cpp:85-129 and doFDTDStep2D :64-69) rather than typed in:
# the stencil is a sum of terms coefficient * (sum of n cells); the coefficient design and the exciter are
# lists of (multiplies, adds) per step.
FDTD_STENCIL_TERMS = (("kc", 1), ("ke", 4), ("kk", 4), ("kc2", 1), ("ke2", 4))
FDTD_DESIGN_STEPS = (("c = kSize Fs", 1, 0), ("T = 3/5 c", 1, 0), ("T T", 1, 0), ("kk", 1, 0), ("ke", 1, 0),
                     ("kc = 2 - 4 (kk + ke)", 1, 2), ("ks1 = s1 T isr", 2, 0), ("ke += ks1", 0, 1),
                     ("kc += -4 ks1", 1, 1), ("ke2 = -1 ks1", 1, 0), ("kc2 = s0 isr + 4 ks1 - 1", 2, 2),
                     ("5 x *= SK", 5, 0), ("exciter += in kInputGain", 1, 1))


def fdtd_ops_per_sample():
    """(stencil ops per cell, design + exciter ops per sample, total FP32 ops per instance-sample)."""
    cell = sum(1 + (n - 1) for _, n in FDTD_STENCIL_TERMS) + (len(FDTD_STENCIL_TERMS) - 1)
    design = sum(m + a for _, m, a in FDTD_DESIGN_STEPS)
    return cell, design, 16 * 16 * cell + design


def gpu_facts():
    """Card name, power limit (W) and SM clocks (MHz, current and maximum), read in this run (read-only query)."""
    import subprocess
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30)
        name, pl, sm, smax = [x.strip() for x in r.stdout.strip().split("\n")[0].split(",")]
        return {"gpu": name, "power_limit_w": float(pl), "sm_clock_mhz": float(sm), "sm_clock_max_mhz": float(smax)}
    except Exception as e:  # noqa: BLE001
        return {"gpu": "unknown (%s)" % e}


def bench_fdtd(api, wl, torch, dev, steps, cpu):
    """K9: V FDTD membranes x 64 vectors, inputs resident on the device, both floating-point modes.  Mean of `steps`
    CUDA-event-timed launches after 3 warm-up launches; parity of 64 instances of the last timed launch against the
    checker (the example's text where oracle/_ref was built, else the plain-C port)."""
    from oracle import fdtd_bindings as ob
    T = 64
    cell, design, ops = fdtd_ops_per_sample()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for V in (4096, 16384):
        inp = wl.fdtd_inputs(V, T)
        d_in = torch.from_numpy(inp).to(dev)
        d_out = torch.empty((T, 2, V, 64), dtype=torch.float32, device=dev)
        sample = np.linspace(0, V - 1, 64).astype(np.int64)
        for ftz in (False, True):
            b = api.FDTDBank(V, 48000.0, flags=api.FDTDBank.FTZ if ftz else 0)
            sh = torch.cuda.current_stream().cuda_stream
            for _ in range(3):
                b.process_device(d_in, d_out, T, sh)
            times = []
            for i in range(steps):
                if i == steps - 1:
                    torch.cuda.synchronize()
                    st_before = b.get_state()[sample]
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                b.process_device(d_in, d_out, T, sh)
                e1.record()
                torch.cuda.synchronize()
                times.append(e0.elapsed_time(e1))
            facts = gpu_facts()
            got = d_out[:, :, torch.from_numpy(sample).to(dev)].cpu().numpy()
            sub_in = np.ascontiguousarray(inp[:, :, sample])
            if ob.fdtd_ref_available():
                want, _, _ = ob.RefFdtd().run(sub_in, st_before, ftz=ftz)
                checker = "reference example text (oracle/_ref/libmlfdtd.so)"
            else:
                want, _ = ob.port_fdtd(sub_in, st_before, ftz=ftz)
                checker = "plain-C port"
            both_nan = np.isnan(got) & np.isnan(want)
            mism = int(((got.view(np.uint32) != want.view(np.uint32)) & ~both_nan).sum())
            b.close()
            ms = float(np.mean(times))
            rate = V * T * 64 / (ms * 1e-3)
            clock = facts.get("sm_clock_max_mhz")
            ceiling = sms * 128 * clock * 1e6 if clock else None
            print(json.dumps({
                "config": "fdtd_" + ("ftz" if ftz else "ieee"), "kernel": "fdtd_kernel<%s>" % ("true" if ftz else "false"),
                "instances": V, "blocks": T, "kernel_ms": ms, "instance_samples_per_s": rate,
                "membranes_realtime_48k": rate / 48000.0,
                "fp32_ops_per_instance_sample": ops, "stencil_ops_per_cell": cell, "design_ops_per_sample": design,
                "achieved_fp32_ops_per_s": rate * ops,
                "non_fma_fp32_ceiling_ops_per_s": ceiling,
                "frac_of_non_fma_ceiling": rate * ops / ceiling if ceiling else None,
                "ceiling_note": "%d SMs x 128 FP32 lanes x max SM clock, one op per lane per clock: exact mode "
                                "cannot fuse multiplies and adds, so the FMA data-sheet figure does not apply" % sms,
                **facts, "parity_instances": 64, "parity_checker": checker, "mismatches": mism}), flush=True)
        if cpu and ob.fdtd_ref_available():
            cores = os.cpu_count() or 1
            best = 1e30
            for _ in range(2):
                _, _, sec = ob.RefFdtd().run(inp, ftz=True, nthreads=cores)
                best = min(best, sec)
            print(json.dumps({"config": "fdtd_reference_cpu", "threads": cores, "instances": V, "blocks": T,
                              "seconds": best, "instance_samples_per_s": V * T * 64 / best,
                              "note": "the example's own processFDTDModel under UsingFlushDenormalsToZero "
                                      "(oracle/_ref/libmlfdtd.so), same inputs"}), flush=True)
        del d_in, d_out


HBM_DATASHEET_GBS = 3350.0  # H100 SXM data sheet (700 W card), not a measured peak


def bench_buses(api, wl, torch, dev, steps):
    """K10 alone, rows resident on the device: mean of `steps` CUDA-event-timed launches after 3 warm-up launches;
    algorithmic bytes = every voice row of every bus read once + the bus rows written.  Parity of up to 64 sampled
    buses (all blocks; for G = 1, the first and last block) against the plain-C port.  Then contract E at
    65 536 voices x 64 vectors as 4 096 instruments x 16 voices: rows out, mix bus only, and bus rows out."""
    from oracle import bus_bindings as bb
    T = 64
    facts = gpu_facts()
    shapes = [(4096, 16, 1), (4096, 16, 2), (16384, 4, 1), (16384, 4, 2), (1, 65536, 1)]
    for G, poly, P in shapes:
        V = G * poly
        first, count = wl.instrument_buses(G, poly)
        rows = torch.randn((T, P, V, 64), dtype=torch.float32, device=dev)
        bus = torch.empty((T, P, G, 64), dtype=torch.float32, device=dev)
        b = api.Buses(V, first, count)
        sh = torch.cuda.current_stream().cuda_stream
        for _ in range(3):
            b.sum_device(rows, bus, P, T, sh)
        times = []
        for _ in range(steps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            b.sum_device(rows, bus, P, T, sh)
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
        b.close()
        sel = np.unique(np.linspace(0, G - 1, min(G, 64)).astype(np.int64))
        sel_t = np.arange(T) if G > 1 else np.array([0, T - 1])
        voices = (first[sel, None] + np.arange(poly)[None, :]).reshape(-1)
        sub = rows[torch.from_numpy(sel_t).to(dev)][:, :, torch.from_numpy(voices).to(dev)].cpu().numpy()
        want = bb.port_buses(sub, *wl.instrument_buses(len(sel), poly))
        got = bus[torch.from_numpy(sel_t).to(dev)][:, :, torch.from_numpy(sel).to(dev)].cpu().numpy()
        mism = int(((got.view(np.uint32) != want.view(np.uint32)) & ~(np.isnan(got) & np.isnan(want))).sum())
        ms = float(np.mean(times))
        nbytes = 4.0 * 64 * T * P * (V + G)
        print(json.dumps({
            "config": "buses_%dx%d_p%d" % (G, poly, P), "kernel": "bus_sum_kernel", "buses": G, "voices_per_bus": poly,
            "planes": P, "blocks": T, "kernel_ms": ms, "algorithmic_bytes": nbytes,
            "achieved_gbs": nbytes / (ms * 1e-3) / 1e9,
            "frac_of_datasheet_hbm": nbytes / (ms * 1e-3) / 1e9 / HBM_DATASHEET_GBS,
            "datasheet_note": "3.35 TB/s, H100 SXM data sheet", **facts,
            "parity_buses": int(len(sel)), "parity_blocks": int(len(sel_t)), "parity_checker": "plain-C port",
            "mismatches": mism}), flush=True)
        del rows, bus
        torch.cuda.empty_cache()
    bench_contract_e_buses(api, wl, torch, facts)


def bench_contract_e_buses(api, wl, torch, facts, n_calls=5):
    """Contract E, 65 536 voices x 64 vectors of config A, pinned host buffers, host clock around calls that return
    finished: rows + mix out, mix only, bus rows of 4 096 x 16 instruments out.  Parity of 16 buses of the last
    call against port(bank) -> port(graph) -> port(buses), the events replayed for every call made."""
    import time
    from oracle import bindings, bus_bindings as bb
    V, T, G, poly = 65536, 64, 4096, 16
    w = wl.config_a(V)
    prm = wl.synth_bank_params(V)
    ev_np = wl.synth_events(V, T)
    h_ev = torch.empty(ev_np.nbytes, dtype=torch.uint8).pin_memory()
    h_ev.numpy()[:] = ev_np.view(np.uint8).reshape(-1)
    ev = h_ev.numpy().view(ev_np.dtype).reshape(T, V)
    h_out = torch.empty((T, 1, V, 64), dtype=torch.float32).pin_memory().numpy()
    h_mix = torch.empty((T, 1, 64), dtype=torch.float32).pin_memory().numpy()
    h_bus = torch.empty((T, 1, G, 64), dtype=torch.float32).pin_memory().numpy()
    first, count = wl.instrument_buses(G, poly)
    vb = api.VoiceBank(48000.0, *prm)
    g = api.VoiceGraph(w.spec, V)
    b = api.Buses(V, first, count)
    g.set_coefs(w.coef)
    g.set_state(w.state)
    legs = (("contract_E_rows", lambda: g.process_events_host(vb, ev, want_out=True, want_mix=True, out=h_out, mix=h_mix),
             h_out.nbytes + h_mix.nbytes),
            ("contract_E_mix", lambda: g.process_events_host(vb, ev, want_out=False, want_mix=True, mix=h_mix),
             h_mix.nbytes),
            ("contract_E_buses", lambda: g.process_events_buses_host(vb, b, ev, out=h_bus), h_bus.nbytes))
    calls = 0
    for name, call, down in legs:
        call()
        t0 = time.perf_counter()
        for _ in range(n_calls):
            call()
        dt = time.perf_counter() - t0
        calls += 1 + n_calls
        print(json.dumps({"config": name, "voices": V, "blocks": T, "ms_per_call": 1e3 * dt / n_calls,
                          "voice_samples_per_s": V * T * 64 * n_calls / dt, "h2d_bytes_per_call": int(ev.nbytes),
                          "d2h_bytes_per_call": int(down), "time_chunks": g.last_host_slices,
                          "kernels": "voice_bank_kernel -> " + g.kernel_name +
                                     (" -> bus_sum_kernel" if name.endswith("buses") else ""), **facts}), flush=True)
    for h in (g, vb, b):
        h.close()
    sel = np.linspace(0, G - 1, 16).astype(np.int64)
    voices = (first[sel, None] + np.arange(poly)[None, :]).reshape(-1)
    rows, _ = bindings.port_voice_bank().run(48000.0, *(p_[voices] for p_ in prm),
                                             np.ascontiguousarray(np.tile(ev[:, voices], (calls, 1))),
                                             nthreads=os.cpu_count() or 1)
    out, _, _ = bindings.PortOracle().run(w.spec, len(voices), T * calls, np.ascontiguousarray(rows[:, 0:1]),
                                          np.ascontiguousarray(w.state[:, voices]),
                                          np.ascontiguousarray(w.coef[:, voices]), nthreads=os.cpu_count() or 1)
    want = bb.port_buses(np.ascontiguousarray(out[T * (calls - 1):]), *wl.instrument_buses(len(sel), poly))
    got = np.ascontiguousarray(h_bus[:, :, sel])
    mism = int(((got.view(np.uint32) != want.view(np.uint32)) & ~(np.isnan(got) & np.isnan(want))).sum())
    print(json.dumps({"config": "contract_E_buses_parity", "buses": int(len(sel)), "blocks": T,
                      "calls_replayed": calls, "checker": "port bank -> port graph -> port buses",
                      "mismatches": mism}), flush=True)


def bench_controllers(api, wl, torch, dev, steps):
    """K11 alone, change lists resident on the device: 4 096 instruments x 129 and x 9 controllers x 64 vectors of
    fader moves (density 0.05), mean of `steps` CUDA-event-timed launches after 3 warm-up launches.  Bytes written =
    the controller rows (the bound: idle rows are stored without being read).  Parity of 16 sampled instruments of
    the first launch against the plain-C port.  Then contract E at 65 536 voices x 64 vectors of config A with 4
    controller planes (4 096 instruments x 16 voices), host clock around calls that return finished."""
    import time
    from oracle import ctrl_bindings as cbind
    T, G = 64, 4096
    facts = gpu_facts()
    offsets, ch = wl.controller_changes(G, T, density=0.05, seed=40)
    d_off = torch.from_numpy(offsets).to(dev)
    d_ch = torch.from_numpy(ch.view(np.int64)).to(dev)
    sel = np.linspace(0, G - 1, 16).astype(np.int64)
    for C in (129, 9):
        ctrl = list(range(129)) if C == 129 else list(wl.CONTROLLER_POOL[:9])
        out = torch.empty((T, C, G, 64), dtype=torch.float32, device=dev)
        bank = api.ControllerBank(G, ctrl, 48000.0)
        sh = torch.cuda.current_stream().cuda_stream
        bank.process_device(d_off, d_ch, out, T, stream=sh)
        torch.cuda.synchronize()
        got = out[:, :, torch.from_numpy(sel).to(dev)].cpu().numpy()
        for _ in range(2):
            bank.process_device(d_off, d_ch, out, T, stream=sh)
        times = []
        for _ in range(steps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            bank.process_device(d_off, d_ch, out, T, stream=sh)
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
        bank.close()
        sub_off = np.zeros((T, len(sel) + 1), np.int32)
        parts, n = [], 0
        for t in range(T):
            for j, g in enumerate(sel):
                sub_off[t, j] = n
                parts.append(ch[offsets[t, g]:offsets[t, g + 1]])
                n += parts[-1].size
            sub_off[t, -1] = n
        want, _, _ = cbind.port_controllers(len(sel), ctrl, sub_off, np.concatenate(parts), 48000.0)
        mism = int(((got.view(np.uint32) != want.view(np.uint32)) & ~(np.isnan(got) & np.isnan(want))).sum())
        ms = float(np.mean(times))
        nbytes = 256.0 * T * C * G
        print(json.dumps({
            "config": "controllers_%dx%d" % (G, C), "kernel": "controller_bank_kernel", "instruments": G,
            "controllers": C, "blocks": T, "changes": int(ch.size), "kernel_ms": ms, "bytes_written": nbytes,
            "achieved_gbs": nbytes / (ms * 1e-3) / 1e9,
            "frac_of_datasheet_hbm": nbytes / (ms * 1e-3) / 1e9 / HBM_DATASHEET_GBS,
            "datasheet_note": "3.35 TB/s, H100 SXM data sheet", **facts,
            "parity_instruments": int(len(sel)), "parity_checker": "plain-C port", "mismatches": mism}), flush=True)
        del out
        torch.cuda.empty_cache()
    del d_off, d_ch
    V, poly, n_calls = 65536, 16, 5
    ctrl = [1, 7, 11, 128]
    w = wl.config_a(V)
    prm = wl.synth_bank_params(V)
    ev_np = wl.synth_events(V, T)
    h_ev = torch.empty(ev_np.nbytes, dtype=torch.uint8).pin_memory()
    h_ev.numpy()[:] = ev_np.view(np.uint8).reshape(-1)
    ev = h_ev.numpy().view(ev_np.dtype).reshape(T, V)
    vb = api.VoiceBank(48000.0, *prm)
    cb = api.ControllerBank(V // poly, ctrl, 48000.0, protocol=api.ControllerBank.MPE)
    cb.set_voice_map(np.repeat(np.arange(V // poly, dtype=np.int32), poly))
    offsets, ch = wl.controller_changes(V // poly, T, density=0.05, seed=41, pool=ctrl)
    g = api.VoiceGraph(w.spec, V)
    g.set_coefs(w.coef)
    g.set_state(w.state)
    g.process_events_controllers_host(vb, cb, ev, offsets, ch, want_out=False, want_mix=True)
    t0 = time.perf_counter()
    for _ in range(n_calls):
        g.process_events_controllers_host(vb, cb, ev, offsets, ch, want_out=False, want_mix=True)
    dt = time.perf_counter() - t0
    print(json.dumps({"config": "contract_E_controllers_mix", "voices": V, "blocks": T, "controller_planes": len(ctrl),
                      "ms_per_call": 1e3 * dt / n_calls, "voice_samples_per_s": V * T * 64 * n_calls / dt,
                      "h2d_bytes_per_call": int(ev.nbytes + offsets.nbytes + ch.nbytes),
                      "time_chunks": g.last_host_slices,
                      "kernels": "voice_bank_kernel -> controller_bank_kernel -> " + g.kernel_name, **facts}),
          flush=True)
    for h in (g, vb, cb):
        h.close()



def bench_router(api, wl, torch, dev, steps):
    """K12 alone, events resident on the device: 4 096 instruments x 16 voices x 64 vectors of midi_performance at
    its density (0.1) and at 10x, mean of `steps` CUDA-event-timed calls (three launches each) after 2 warm-up calls.
    Bytes written = the records.  Parity of 16 sampled instruments of a fresh bank's first call against host routers."""
    import sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    from tests.router_cases import route_on_host
    G, P, T = 4096, 16, 64
    facts = gpu_facts()
    lay = wl.midi_layout(G, P)
    V = lay["n_voices"]
    sel = np.linspace(0, G - 1, 16).astype(np.int64)
    for density in (0.1, 1.0):
        offsets, ev = wl.midi_performance(G, T, P, density=density, seed=50)
        d_off = torch.from_numpy(offsets).to(dev)
        d_ev = torch.from_numpy(ev.view(np.uint8)).to(dev)
        d_rec = torch.empty((T, V, 72), dtype=torch.uint8, device=dev)
        d_coff = torch.empty((T, G + 1), dtype=torch.int32, device=dev)
        d_ch = torch.empty((max(ev.size, 1), 8), dtype=torch.uint8, device=dev)
        r = api.RouterBank(lay["polyphony"], lay["first_voice"], V)
        sh = torch.cuda.current_stream().cuda_stream
        r.process_device(d_off, d_ev, d_rec, d_coff, d_ch, T, stream=sh)
        torch.cuda.synchronize()
        got = d_rec.cpu().numpy()
        for _ in range(2):
            r.process_device(d_off, d_ev, d_rec, d_coff, d_ch, T, stream=sh)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            r.process_device(d_off, d_ev, d_rec, d_coff, d_ch, T, stream=sh)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / steps
        r.close()
        sub_off = np.zeros((T, len(sel) + 1), np.int32)
        parts, n = [], 0
        for t in range(T):
            for j, g in enumerate(sel):
                sub_off[t, j] = n
                parts.append(ev[offsets[t, g]:offsets[t, g + 1]])
                n += parts[-1].size
            sub_off[t, -1] = n
        sub_lay = wl.midi_layout(len(sel), P)
        want = route_on_host(sub_off, np.concatenate(parts), sub_lay)[0]
        voices = (lay["first_voice"][sel, None] + np.arange(P)[None, :]).reshape(-1)
        mism = int((got[:, voices].reshape(-1) != np.ascontiguousarray(want).view(np.uint8).reshape(-1)).sum())
        nbytes = 72.0 * T * V
        print(json.dumps({
            "config": "router_%dx%d_density_%g" % (G, P, density), "kernels": "router_count_kernel -> "
            "router_bank_kernel -> router_total_kernel", "instruments": G, "voices": V, "blocks": T,
            "events": int(ev.size), "ms_per_call": ms, "record_bytes_written": nbytes,
            "achieved_gbs": nbytes / (ms * 1e-3) / 1e9,
            "frac_of_datasheet_hbm": nbytes / (ms * 1e-3) / 1e9 / HBM_DATASHEET_GBS,
            "datasheet_note": "3.35 TB/s, H100 SXM data sheet", **facts,
            "parity_instruments": int(len(sel)), "parity_checker": "host routers (mlb::VoiceRouter)",
            "mismatched_bytes": mism}), flush=True)


def host_router_timing(wl, lay, offsets, ev, reps=3):
    """Compile tools/host_router_timing.cpp into a temporary directory and run it on the performance: one
    mlb::VoiceRouter per instrument on one host thread.  Returns its JSON line plus the records it produced."""
    import subprocess
    import tempfile
    here = os.path.dirname(os.path.abspath(__file__))
    G, T = offsets.shape[1] - 1, offsets.shape[0]
    with tempfile.TemporaryDirectory() as d:
        exe, inp, out = os.path.join(d, "hrt"), os.path.join(d, "in.bin"), os.path.join(d, "rec.bin")
        subprocess.run(["g++", "-O2", "-std=c++17", "-I", os.path.join(os.path.dirname(here), "include"),
                        os.path.join(here, "host_router_timing.cpp"), "-o", exe], check=True)
        with open(inp, "wb") as f:
            f.write(np.array([G, T, 0, reps], np.int32).tobytes())
            f.write(lay["polyphony"].astype(np.int32).tobytes() + lay["first_voice"].astype(np.int32).tobytes())
            f.write(np.array([lay["n_voices"]], np.int32).tobytes() + offsets.astype(np.int32).tobytes())
            f.write(np.array([ev.size], np.int32).tobytes() + ev.tobytes())
        line = json.loads(subprocess.run([exe, inp, out], check=True, capture_output=True, text=True).stdout)
        line["records"] = np.fromfile(out, wl.VOICE_EVENTS_DTYPE).reshape(T, lay["n_voices"])
    return line


def bench_routed(api, wl, torch, n_calls=5):
    """Contract E from raw events against contract E from host-routed records, same performance (4 096 instruments x
    16 voices x 64 vectors of midi_performance, config A, bus rows out), pinned host buffers, host clock around calls
    that return finished.  The host-routed line adds the wall time of the 4 096 host routers (one thread, this
    machine's host, timed in C++ by tools/host_router_timing.cpp) that produce its records.  Parity: the two paths' bus rows of the first call, bit for bit."""
    import ctypes
    import time
    from madronalib_b200.api import EVENT_DTYPE
    G, P, T = 4096, 16, 64
    facts = gpu_facts()
    lay = wl.midi_layout(G, P)
    V = lay["n_voices"]
    w = wl.config_a(V)
    vi, gs, da, pb = wl.synth_bank_params(V)
    offsets, ev = wl.midi_performance(G, T, P, density=0.1, seed=51)
    L = api.lib()
    rec = torch.empty((T * V * 72,), dtype=torch.uint8).pin_memory().numpy().view(wl.VOICE_EVENTS_DTYPE).reshape(T, V)
    host = host_router_timing(wl, lay, offsets, ev, reps=3)
    rec[:] = host.pop("records")
    h_bus = [torch.empty((T, 1, G, 64), dtype=torch.float32).pin_memory().numpy() for _ in range(2)]
    ev_pin = torch.empty((max(ev.size, 1) * 16,), dtype=torch.uint8).pin_memory().numpy().view(EVENT_DTYPE)
    ev_pin[:ev.size] = ev
    off_pin = torch.empty(offsets.shape, dtype=torch.int32).pin_memory().numpy()
    off_pin[:] = offsets
    results = {}
    for name in ("host_routed", "routed"):
        vb = api.VoiceBank(48000.0, lay["voice_index"], gs, da, pb, flags=api.VoiceBank.MIDI)
        g = api.VoiceGraph(w.spec, V)
        g.set_coefs(w.coef)
        g.set_state(w.state)
        b = api.Buses(V, lay["bus_first"], lay["bus_count"])
        r = api.RouterBank(lay["polyphony"], lay["first_voice"], V)
        out = h_bus[0 if name == "host_routed" else 1]
        if name == "host_routed":
            call = lambda: L.mlb_synth_process_buses_host(vb._h, g._h, b._h, rec.ctypes.data, out.ctypes.data, T)  # noqa
            up = rec.nbytes
        else:
            call = lambda: L.mlb_synth_process_routed_host(r._h, vb._h, None, g._h, b._h, off_pin.ctypes.data,  # noqa
                                                           ev_pin.ctypes.data, int(ev.size), None, None,
                                                           out.ctypes.data, T)
            up = offsets.nbytes + ev.nbytes
        assert call() == 0, api.lib().mlb_last_error()
        first = out.copy()
        t0 = time.perf_counter()
        for _ in range(n_calls):
            call()
        dt = (time.perf_counter() - t0) / n_calls
        results[name] = first
        for h in (vb, g, b, r):
            h.close()
        line = {"config": "contract_E_%s_buses" % name, "instruments": G, "voices": V, "blocks": T,
                "events": int(ev.size), "ms_per_call": 1e3 * dt, "calls_per_s": 1.0 / dt,
                "voice_samples_per_s": V * T * 64 / dt, "h2d_bytes_per_call": int(up), **facts}
        if name == "host_routed":
            line["host_routing_ms"] = host["host_routing_ms"]
            line["host_routing_note"] = "4 096 mlb::VoiceRouter on one host thread, C++ (tools/host_router_timing.cpp), best of 3"
            line["ms_per_call_with_host_routing"] = 1e3 * dt + host["host_routing_ms"]
        print(json.dumps(line), flush=True)
    a, b_ = results["host_routed"], results["routed"]
    mism = int(((a.view(np.uint32) != b_.view(np.uint32)) & ~(np.isnan(a) & np.isnan(b_))).sum())
    print(json.dumps({"config": "contract_E_routed_parity", "checker": "contract E fed by the host routers",
                      "blocks": T, "mismatches": mism}), flush=True)


def bench_process_time(api, wl, torch, dev, steps):
    """K13 alone, transport updates resident on the device: 4 096 instruments x 64 vectors of a steady host transport
    (one update per vector), as instrument rows and through a 65 536-voice map (16 voices each), mean of `steps`
    CUDA-event-timed calls after 2 warm-up calls.  Bytes = the rows written (the updates read are 0.05 % of them).
    Parity of a fresh bank's first call against the port (oracle/port/mlport_ptime.c), every row."""
    from oracle.ptime_bindings import port_process_time
    G, P, T, sr = 4096, 16, 64, 48000.0
    facts = gpu_facts()
    lay = wl.midi_layout(G, P)
    offsets, tr = wl.transport_updates(G, T, sr, seed=60)
    want, _ = port_process_time(G, offsets, tr, sr)
    d_off = torch.from_numpy(offsets).to(dev)
    d_tr = torch.from_numpy(tr.view(np.uint8)).to(dev)
    sh = torch.cuda.current_stream().cuda_stream
    for vmap in (None, lay["voice_instrument"]):
        N = G if vmap is None else lay["n_voices"]
        d_out = torch.empty((T, 1, N, 64), dtype=torch.float32, device=dev)
        pt = api.ProcessTimeBank(G, sr)
        pt.set_voice_map(vmap)
        w0 = pt.get_state()
        pt.process_device(d_off, d_tr, d_out, T, stream=sh)
        torch.cuda.synchronize()
        got = d_out[:, 0].cpu().numpy()
        ref = want if vmap is None else want[:, vmap]
        mism = int(((got.view(np.uint32) != ref.view(np.uint32)) & ~(np.isnan(got) & np.isnan(ref))).sum())
        for _ in range(2):
            pt.set_state(w0)
            pt.process_device(d_off, d_tr, d_out, T, stream=sh)
        pt.set_state(w0)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            pt.process_device(d_off, d_tr, d_out, T, stream=sh)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / steps
        pt.close()
        nbytes = 256.0 * N * T
        print(json.dumps({
            "config": "process_time_%dx%d_%s" % (G, T, "instrument_rows" if vmap is None else "voice_map_%d" % N),
            "kernel": "process_time_kernel", "instruments": G, "rows": N, "blocks": T, "ms_per_call": ms,
            "voice_samples_per_s": N * T * 64 / (ms * 1e-3), "row_bytes_written": nbytes,
            "achieved_gbs": nbytes / (ms * 1e-3) / 1e9,
            "frac_of_datasheet_hbm": nbytes / (ms * 1e-3) / 1e9 / HBM_DATASHEET_GBS,
            "datasheet_note": "3.35 TB/s, H100 SXM data sheet", **facts,
            "parity_checker": "oracle/port/mlport_ptime.c", "mismatched_words": mism}), flush=True)
        del d_out


def bench_context(api, wl, torch, n_calls=5):
    """Contract E with every AudioContext signal (mlb_synth_process_context_host: routers, Voice rows, controllers 1
    and 74, the beat phase, config A, bus rows out) against the routed entry point on the same performance (4 096
    instruments x 16 voices x 64 vectors of midi_performance, one transport update per instrument and vector), pinned
    host buffers, host clock around calls that return finished, the two alternated.  Config A reads only the Voice
    rows, so the bus rows of the two paths must match bit for bit; the difference in time is K11 + K13."""
    import time
    from madronalib_b200.api import EVENT_DTYPE, TRANSPORT_DTYPE
    G, P, T, sr = 4096, 16, 64, 48000.0
    facts = gpu_facts()
    lay = wl.midi_layout(G, P)
    V = lay["n_voices"]
    w = wl.config_a(V)
    vi, gs, da, pb = wl.synth_bank_params(V)
    offsets, ev = wl.midi_performance(G, T, P, density=0.1, seed=51)
    toff, tr = wl.transport_updates(G, T, sr, seed=61)
    L = api.lib()

    def pinned(a, dtype):
        p = torch.empty((max(a.nbytes, 1),), dtype=torch.uint8).pin_memory().numpy()
        p[:a.nbytes] = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
        return p[:a.nbytes].view(dtype).reshape(a.shape)

    ev_pin, off_pin = pinned(ev, EVENT_DTYPE), pinned(offsets, np.int32)
    tr_pin, toff_pin = pinned(tr, TRANSPORT_DTYPE), pinned(toff, np.int32)
    h_bus = {k: torch.empty((T, 1, G, 64), dtype=torch.float32).pin_memory().numpy() for k in ("routed", "context")}
    hs = {}
    for name in ("routed", "context"):
        vb = api.VoiceBank(sr, lay["voice_index"], gs, da, pb, flags=api.VoiceBank.MIDI)
        g = api.VoiceGraph(w.spec, V)
        g.set_coefs(w.coef)
        g.set_state(w.state)
        b = api.Buses(V, lay["bus_first"], lay["bus_count"])
        r = api.RouterBank(lay["polyphony"], lay["first_voice"], V)
        cb = api.ControllerBank(G, [1, 74], sr)
        cb.set_voice_map(lay["voice_instrument"])
        pt = api.ProcessTimeBank(G, sr)
        pt.set_voice_map(lay["voice_instrument"])
        hs[name] = (vb, g, b, r, cb, pt)
    out_first = {}

    def call(name):
        vb, g, b, r, cb, pt = hs[name]
        out = h_bus[name]
        if name == "routed":
            return L.mlb_synth_process_routed_host(r._h, vb._h, None, g._h, b._h, off_pin.ctypes.data,
                                                   ev_pin.ctypes.data, int(ev.size), None, None, out.ctypes.data, T)
        return L.mlb_synth_process_context_host(r._h, vb._h, cb._h, pt._h, g._h, b._h, off_pin.ctypes.data,
                                                ev_pin.ctypes.data, int(ev.size), toff_pin.ctypes.data,
                                                tr_pin.ctypes.data, int(tr.size), None, None, out.ctypes.data, T)

    for name in hs:
        assert call(name) == 0, L.mlb_last_error()
        out_first[name] = h_bus[name].copy()
    dt = {k: 0.0 for k in hs}
    for _ in range(n_calls):
        for name in hs:
            t0 = time.perf_counter()
            call(name)
            dt[name] += (time.perf_counter() - t0) / n_calls
    for hh in hs.values():
        for h in hh:
            h.close()
    for name in hs:
        print(json.dumps({"config": "context_pair_%s_buses" % name, "instruments": G, "voices": V, "blocks": T,
                          "events": int(ev.size), "transport_updates": int(tr.size) if name == "context" else 0,
                          "planes": 8 + (3 if name == "context" else 0), "ms_per_call": 1e3 * dt[name],
                          "voice_samples_per_s": V * T * 64 / dt[name], **facts}), flush=True)
    a, b_ = out_first["routed"], out_first["context"]
    mism = int(((a.view(np.uint32) != b_.view(np.uint32)) & ~(np.isnan(a) & np.isnan(b_))).sum())
    print(json.dumps({"config": "contract_E_context_parity", "checker": "the routed entry point", "blocks": T,
                      "mismatches": mism}), flush=True)


if __name__ == "__main__":
    main()
