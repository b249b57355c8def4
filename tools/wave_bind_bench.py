#!/usr/bin/env python
"""A new set of periodic waves for a prepared batch, bound from device memory versus built again (GPU).  Workload: N graphs of 1 s, each
a custom OscillatorNode whose wave of H harmonics is declared bound from device memory (wae_oscillator_set_device_periodic_wave, 8192-point
wavetable, normalised) -> lowpass (frequency declared with set_device_value) -> gain (declared) -> destination, run at each --harmonics.
Per new wave set (random real / imag [N][H] tensors with 1/k amplitudes drawn on the GPU, new lowpass and gain values beside them) it
times, with the card's name and power limit read in the same run (medians over --runs timed runs after --warmup untimed ones):
  (a) wae_batch_bind_periodic_waves alone (CUDA events on the engine stream around the item-table copy, k_bind_waves and
      k_wave_normalize), the host side of the bind call, and the kernels' device times (torch.profiler), with the synthesis terms
      (N x 8192 x (H - 1)) per second of k_bind_waves;
  (b) bind_periodic_waves + bind_params + run + sync on the host clock;
  (c) what a caller does without it: copy the coefficients and values to the host, make each wavetable with wae_periodic_wave_table (on
      every host core), build the N contexts with them given to set_periodic_wave and the values set, prepare the batch, run, sync
      (--rebuild-runs timed runs: the host synthesis takes seconds);
and the largest difference between (b)'s and (c)'s renders of the last set.  Prints one JSON line.  Writes nothing."""
import argparse
import ctypes
import gc
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
TABLE_LEN = 8192


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # (reported, not fatal)
        return "unknown (%s)" % e


def graph(pkg, be, g, length, harmonics, sr, table=None, vals=None):
    """table None: the wave bound from device memory and the lowpass frequency and gain declared; else the wavetable given to
    set_periodic_wave and vals = (frequency, gain)"""
    c = pkg.OfflineAudioContext(2, length, sr, be)
    o = c.create_oscillator(frequency=55.0 * 2.0 ** ((g % 48) / 12.0))
    bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=2000.0 if vals is None else float(vals[0]), q=1.0)
    gn = c.create_gain(0.5 if vals is None else float(vals[1]))
    if table is None:
        o.set_device_periodic_wave(harmonics, TABLE_LEN)
        bq.frequency.set_device_value()
        gn.gain.set_device_value()
    else:
        o.set_periodic_wave(table)
    o.connect(bq)
    bq.connect(gn)
    gn.connect(c.destination())
    o.start()
    return c, o, bq, gn


def median(xs):
    return float(np.median(np.asarray(xs, np.float64)))


def host_tables(api, real, imag):
    """wae_periodic_wave_table of every row, on every host core (the call releases the GIL)"""
    fp = ctypes.POINTER(ctypes.c_float)
    n, h = real.shape
    out = np.zeros((n, TABLE_LEN), np.float32)

    def one(g):
        api.check(api.periodic_wave_table(real[g].ctypes.data_as(fp), imag[g].ctypes.data_as(fp), h, 0, out[g].ctypes.data_as(fp), TABLE_LEN))
    with ThreadPoolExecutor(max_workers=os.cpu_count() or 1) as ex:
        list(ex.map(one, range(n)))
    return out


def bench(pkg, eng, torch, n, L, harmonics, sr, runs, warmup, rebuild_runs, seed):
    be = eng.backend
    api = pkg.api()
    gen = torch.Generator(device="cuda").manual_seed(seed)
    k = torch.arange(1, harmonics + 1, device="cuda", dtype=torch.float32)[None, :]

    def draw():
        real = (torch.rand((n, harmonics), generator=gen, device="cuda") * 2.0 - 1.0) / k
        imag = (torch.rand((n, harmonics), generator=gen, device="cuda") * 2.0 - 1.0) / k
        vals = torch.stack([200.0 + 7800.0 * torch.rand(n, generator=gen, device="cuda"),
                            0.1 + 0.8 * torch.rand(n, generator=gen, device="cuda")], dim=1)
        return real, imag, vals

    made = [graph(pkg, be, g, L, harmonics, sr) for g in range(n)]
    batch = pkg.Batch([m[0] for m in made])
    _, o, bq, gn = made[0]
    es = batch._engine_stream()
    terms = n * TABLE_LEN * (harmonics - 1)
    res = {"graphs": n, "frames": L, "harmonics": harmonics, "table_len": TABLE_LEN, "sample_rate": sr, "runs": runs}

    # (a) the bind alone: the caller's stream sleeps while the host validates, so e0 -> e1 spans the item-table copy and the kernels
    side = torch.cuda.Stream()
    bind_ms, host_ms = [], []
    for r in range(warmup + runs):
        real, imag, _ = draw()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        with torch.cuda.stream(side):
            torch.cuda._sleep(40_000_000)
            e0.record(side)
            t0 = time.perf_counter()
            batch.bind_periodic_waves(o, real, imag)
            t1 = time.perf_counter()
        e1.record(es)
        e1.synchronize()
        if r >= warmup:
            bind_ms.append(e0.elapsed_time(e1))
            host_ms.append((t1 - t0) * 1e3)
    res.update({"bind_ms": round(median(bind_ms), 4), "bind_call_host_ms": round(median(host_ms), 3)})

    # the kernels on their own (device time per launch, averaged over --runs binds)
    from torch.profiler import ProfilerActivity, profile
    real, imag, _ = draw()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(runs):
            batch.bind_periodic_waves(o, real, imag)
        torch.cuda.synchronize()
    for ev in prof.key_averages():
        for name in ("k_bind_waves", "k_wave_normalize"):
            if name in ev.key and ev.count:
                t = getattr(ev, "device_time_total", None)
                if t is None:
                    t = ev.cuda_time_total
                res[name + "_ms"] = round(t / ev.count / 1e3, 4)
    if "k_bind_waves_ms" in res:
        res["synthesis_terms_per_s"] = float("%.3g" % (terms / (res["k_bind_waves_ms"] * 1e-3)))

    # (b) bind_periodic_waves + bind_params + run + sync
    e2e = []
    for r in range(warmup + runs):
        real, imag, vals = draw()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        batch.bind_periodic_waves(o, real, imag)
        batch.bind_params([bq.frequency, gn.gain], vals)
        batch.run()
        batch.sync()
        t1 = time.perf_counter()
        if r >= warmup:
            e2e.append((t1 - t0) * 1e3)
    res["b_bind_run_sync_ms"] = round(median(e2e), 2)
    last = (real, imag, vals)
    bound_out = batch.output_tensor().clone()
    torch.cuda.synchronize()
    batch.destroy()
    del made, batch
    gc.collect()

    # (c) coefficients to the host + host wavetables + build + prepare + run + sync per wave set
    rebuild = []
    for r in range(rebuild_runs):
        real, imag, vals = last if r == rebuild_runs - 1 else draw()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        hr, hi, hv = real.cpu().numpy(), imag.cpu().numpy(), vals.cpu().numpy()
        tables = host_tables(api, hr, hi)
        ctxs = [graph(pkg, be, g, L, harmonics, sr, tables[g], hv[g])[0] for g in range(n)]
        b = pkg.Batch(ctxs)
        b.run()
        b.sync()
        t1 = time.perf_counter()
        rebuild.append((t1 - t0) * 1e3)
        if r == rebuild_runs - 1:
            rebuilt = b.output_tensor()
            res["bit_equal"] = bool(torch.equal(rebuilt, bound_out))
            res["max_abs_diff_b_vs_c"] = float((rebuilt - bound_out).abs().max().item())
            torch.cuda.synchronize()
        b.destroy()
        del ctxs, b
        gc.collect()
    res["c_host_tables_build_prepare_run_sync_ms"] = round(median(rebuild), 2)
    res["host_cores"] = os.cpu_count()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--graphs", type=int, default=1000)
    ap.add_argument("--frames", type=int, default=48000)
    ap.add_argument("--harmonics", type=int, nargs="+", default=[64, 512])
    ap.add_argument("--sr", type=float, default=48000.0)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rebuild-runs", type=int, default=1)
    ap.add_argument("--seed", type=int, default=5)
    a = ap.parse_args()
    import torch
    import conftest
    if not torch.cuda.is_available():
        raise SystemExit("wave_bind_bench: no CUDA device")
    pkg = conftest.load_package()
    eng = pkg.Engine(0)
    out = {}
    for h in a.harmonics:
        out["h%d" % h] = bench(pkg, eng, torch, a.graphs, a.frames, h, a.sr, a.runs, a.warmup, a.rebuild_runs, a.seed)
    out["card"] = card()
    print(json.dumps(out))
    eng.close()


if __name__ == "__main__":
    main()
