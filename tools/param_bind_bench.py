#!/usr/bin/env python
"""A new parameter set for a prepared batch, bound from device memory versus built again (GPU).  The C2 shape of BASELINE configs[1]: N
graphs of AudioBufferSource -> lowpass biquad -> gain -> destination, 2 channels x L frames at 48 kHz, each source a device input
(wae_buffer_source_set_device_input) and the biquad's frequency and Q and the gain bound from device memory (wae_param_set_device_value).
Per new parameter set (a [N][3] tensor drawn on the GPU) it times, with the card's name and power limit read in the same run (medians
over --runs timed runs after --warmup untimed ones):
  (a) wae_batch_bind_params + run + sync on the host clock, the bind alone (CUDA events on the engine stream around k_bind_params and
      k_derive_params with their item-table copy) and the host side of the bind call;
  (b) what a caller does without it: build the N contexts with the new values, prepare the batch, bind the same device audio, run, sync;
and the largest difference between the two renders of the last parameter set.  Prints one JSON line.  Writes nothing."""
import argparse
import gc
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # (reported, not fatal)
        return "unknown (%s)" % e


def c2(pkg, be, length, sr, vals=None):
    """vals None: the parameters bound from device memory; else (frequency, Q, gain) as constants"""
    c = pkg.OfflineAudioContext(2, length, sr, be)
    src = c.create_buffer_source()
    src.set_device_input(2, length, sr)
    f, q, g = vals if vals is not None else (1000.0, 1.0, 0.5)
    bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=f, q=q)
    gn = c.create_gain(g)
    src.connect(bq)
    bq.connect(gn)
    gn.connect(c.destination())
    src.start()
    if vals is None:
        bq.frequency.set_device_value()
        bq.q.set_device_value()
        gn.gain.set_device_value(0.05, 2.0)
    return c, src, [bq.frequency, bq.q, gn.gain]


def median(xs):
    return float(np.median(np.asarray(xs, np.float64)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--graphs", type=int, default=1000)
    ap.add_argument("--frames", type=int, default=480000)
    ap.add_argument("--sr", type=float, default=48000.0)
    ap.add_argument("--runs", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=5)
    a = ap.parse_args()
    import torch
    import conftest
    if not torch.cuda.is_available():
        raise SystemExit("param_bind_bench: no CUDA device")
    pkg = conftest.load_package()
    eng = pkg.Engine(0)
    be = eng.backend
    n, L, sr = a.graphs, a.frames, a.sr
    gen = torch.Generator(device="cuda").manual_seed(a.seed)
    pcm = torch.rand((n, 2, L), generator=gen, device="cuda") * 2.0 - 1.0

    def draw():
        return torch.stack([torch.exp(torch.rand(n, generator=gen, device="cuda") * (np.log(8000.0) - np.log(100.0)) + np.log(100.0)),
                            torch.rand(n, generator=gen, device="cuda") * 3.5 + 0.5, torch.rand(n, generator=gen, device="cuda") * 0.8 + 0.1], dim=1)

    made = [c2(pkg, be, L, sr) for _ in range(n)]
    batch = pkg.Batch([c for c, _, _ in made])
    node, params = made[0][1], made[0][2]
    batch.bind_sources(node, pcm)
    es = batch._engine_stream()
    res = {"graphs": n, "frames": L, "channels": 2, "sample_rate": sr, "runs": a.runs, "bound_params_per_graph": 3}

    # the bind alone: as in device_sources_bench, the caller's stream sleeps while the host validates, so e0 -> e1 spans the item-table
    # copy and the two kernels
    side = torch.cuda.Stream()
    bind_ms, host_ms = [], []
    for r in range(a.warmup + a.runs):
        vals = draw()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        with torch.cuda.stream(side):
            torch.cuda._sleep(40_000_000)
            e0.record(side)
            t0 = time.perf_counter()
            batch.bind_params(params, vals)
            t1 = time.perf_counter()
        e1.record(es)
        e1.synchronize()
        if r >= a.warmup:
            bind_ms.append(e0.elapsed_time(e1))
            host_ms.append((t1 - t0) * 1e3)
    res.update({"bind_kernels_ms": round(median(bind_ms), 4), "bind_call_host_ms": round(median(host_ms), 3)})

    # (a) bind_params + run + sync
    e2e = []
    for r in range(a.warmup + a.runs):
        vals = draw()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        batch.bind_params(params, vals)
        batch.run()
        batch.sync()
        t1 = time.perf_counter()
        if r >= a.warmup:
            e2e.append((t1 - t0) * 1e3)
    res["a_bind_run_sync_ms"] = round(median(e2e), 2)
    last = vals.cpu().numpy()
    bound_out = batch.output_tensor().clone()
    torch.cuda.synchronize()
    batch.destroy()
    del made, batch
    gc.collect()

    # (b) build + prepare + bind_sources + run + sync per parameter set
    rebuild = []
    for r in range(a.warmup + a.runs):
        v = last if r == a.warmup + a.runs - 1 else draw().cpu().numpy()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ctxs = [c2(pkg, be, L, sr, tuple(float(x) for x in v[i])) for i in range(n)]
        b = pkg.Batch([c for c, _, _ in ctxs])
        b.bind_sources(ctxs[0][1], pcm)
        b.run()
        b.sync()
        t1 = time.perf_counter()
        if r >= a.warmup:
            rebuild.append((t1 - t0) * 1e3)
        if r == a.warmup + a.runs - 1:
            res["max_abs_diff_a_vs_b"] = float((b.output_tensor() - bound_out).abs().max().item())
            torch.cuda.synchronize()
        b.destroy()
        del ctxs, b
        gc.collect()
    res["b_build_prepare_bind_run_sync_ms"] = round(median(rebuild), 2)
    res["card"] = card()
    print(json.dumps(res))
    eng.close()


if __name__ == "__main__":
    main()
