#!/usr/bin/env python
"""Loop points bound from device memory versus the alternatives (GPU).  N graphs of a 1.5 s device-input background -> looping
AudioBufferSource -> lowpass biquad -> gain -> destination, 2 channels x L frames at 48 kHz (the README workload).  Per run a new loop
region (start in [0, 0.5] s, end in [0.9, 1.5] s), playback rate in [0.9, 1.1], lowpass frequency and gain are drawn per graph.  With the
card's name and power limit read in the same run, medians over --runs timed runs after --warmup untimed ones, the variants alternated run
by run:
  (a) loop points and rate bound (wae_batch_bind_loops + wae_batch_bind_params) + run + sync: the bound slow track;
  (b) the same graphs with host-built loop points and a bound rate + run + sync: today's serial kernel;
  (c) host-built graphs with the drawn values: build + prepare + bind the background + run + sync;
then per-stage kernel times of (a) and (b) (CUDA events, runs of their own), the device time of a loop bind (k_bind_loops and
k_absn_loop_schedule, with the item table's copy; CUDA events on the engine stream), and the largest difference between (a) and (c) for
the same values.  Prints one JSON line.  Writes nothing."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
BG = 1.5  # seconds of background


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # (reported, not fatal)
        return "unknown (%s)" % e


def graph(pkg, be, length, sr, mode, vals=None):
    """mode 'loops': loop points, rate, frequency and gain bound; 'serial': the loop points host-built (0.25, 1.2), the rest bound;
    'host': vals = (loop_start, loop_end, rate, frequency, gain) host-built"""
    ls, le, rate, freq, gain = vals if vals is not None else (0.25, 1.2, 1.0, 2000.0, 0.5)
    c = pkg.OfflineAudioContext(2, length, sr, be)
    src = c.create_buffer_source(playback_rate=rate, loop=True)
    src.set_device_input(2, int(BG * sr), sr)
    src.set_loop_start(ls)
    src.set_loop_end(le)
    bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=freq)
    gn = c.create_gain(gain)
    src.connect(bq)
    bq.connect(gn)
    gn.connect(c.destination())
    src.start()
    params = []
    if mode != "host":
        src.playback_rate.set_device_value(0.9, 1.1)
        bq.frequency.set_device_value()
        gn.gain.set_device_value(0.05, 2.0)
        params = [src.playback_rate, bq.frequency, gn.gain]
    if mode == "loops":
        src.set_device_loop((0.0, 0.5), (0.9, 1.5))
    return c, src, params


def median(xs):
    return float(np.median(np.asarray(xs, np.float64)))


def stage_times(batch):
    batch.set_timing(True)
    batch.run()
    batch.sync()
    out = {}
    for k, t, _ in batch.stage_times():
        out[k] = out.get(k, 0.0) + t
    batch.set_timing(False)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--graphs", type=int, default=1000)
    ap.add_argument("--frames", type=int, default=480000)
    ap.add_argument("--sr", type=float, default=48000.0)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--seed", type=int, default=11)
    a = ap.parse_args()
    import torch
    import conftest
    if not torch.cuda.is_available():
        raise SystemExit("loop_bind_bench: no CUDA device")
    pkg = conftest.load_package()
    eng = pkg.Engine(0)
    be = eng.backend
    n, L, sr = a.graphs, a.frames, a.sr
    gen = torch.Generator(device="cuda").manual_seed(a.seed)
    bg = torch.rand((n, 2, int(BG * sr)), generator=gen, device="cuda") * 2.0 - 1.0

    def draw():
        u = lambda lo, hi: torch.rand(n, generator=gen, device="cuda", dtype=torch.float64) * (hi - lo) + lo
        ls, le = u(0.0, 0.5), u(0.9, 1.5)
        rate = u(0.9, 1.1).float()
        freq = torch.exp(u(np.log(200.0), np.log(8000.0))).float()
        gain = u(0.1, 0.9).float()
        return ls, le, torch.stack([rate, freq, gain], dim=1)

    def prepared(ctxs):
        b = pkg.Batch([c for c, _, _ in ctxs])
        b.bind_sources(ctxs[0][1], bg)
        return b, ctxs[0][1], ctxs[0][2]

    loops, lnode, lparams = prepared([graph(pkg, be, L, sr, "loops") for _ in range(n)])
    serial, _, sparams = prepared([graph(pkg, be, L, sr, "serial") for _ in range(n)])
    res = {"graphs": n, "frames": L, "channels": 2, "sample_rate": sr, "background_s": BG, "runs": a.runs,
           "kinds_a": pkg.plan_batch([graph(pkg, be, L, sr, "loops")[0]])["kinds"],
           "kinds_b": pkg.plan_batch([graph(pkg, be, L, sr, "serial")[0]])["kinds"]}

    t_a, t_b, t_c = [], [], []
    for r in range(a.warmup + a.runs):
        ls, le, vals = draw()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        loops.bind_loops(lnode, ls, le)
        loops.bind_params(lparams, vals)
        loops.run()
        loops.sync()
        t1 = time.perf_counter()
        serial.bind_params(sparams, vals)
        serial.run()
        serial.sync()
        t2 = time.perf_counter()
        hv = torch.cat([ls[:, None], le[:, None], vals.double()], dim=1).cpu().numpy()
        host, _, _ = prepared([graph(pkg, be, L, sr, "host", tuple(float(x) for x in hv[i])) for i in range(n)])
        host.run()
        host.sync()
        t3 = time.perf_counter()
        if r >= a.warmup:
            t_a.append((t1 - t0) * 1e3)
            t_b.append((t2 - t1) * 1e3)
            t_c.append((t3 - t2) * 1e3)
        if r + 1 < a.warmup + a.runs:
            host.destroy()
    res["a_bind_loops_params_run_sync_ms"] = round(median(t_a), 2)
    res["b_serial_bind_params_run_sync_ms"] = round(median(t_b), 2)
    res["c_build_prepare_run_sync_ms"] = round(median(t_c), 2)
    res["max_abs_diff_a_vs_c"] = float((loops.output_tensor() - host.output_tensor()).abs().max().item())

    # per-stage kernel times (runs of their own) and the device time of a loop bind
    sa, sb = [], []
    for r in range(a.warmup + a.runs):
        sa.append(stage_times(loops))
        sb.append(stage_times(serial))
    for key, acc in (("a", sa), ("b", sb)):
        res[f"{key}_stage_ms"] = {k: round(median([s.get(k, 0.0) for s in acc[a.warmup:]]), 3) for k in acc[-1]}
    stream = loops._engine_stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    tb = []
    for r in range(a.warmup + a.runs):
        ls, le, _ = draw()
        torch.cuda.synchronize()
        e0.record(stream)
        loops.bind_loops(lnode, ls, le)
        e1.record(stream)
        e1.synchronize()
        if r >= a.warmup:
            tb.append(e0.elapsed_time(e1))
    res["bind_loops_device_ms"] = round(median(tb), 3)
    res["card"] = card()
    print(json.dumps(res))
    for b in (loops, serial, host):
        b.destroy()
    eng.close()


if __name__ == "__main__":
    main()
