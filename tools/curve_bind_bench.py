#!/usr/bin/env python
"""A new set of WaveShaper curves for a prepared batch, bound from device memory versus built again (GPU).  Two workloads, each source a
device input (wae_buffer_source_set_device_input) and each curve declared bound from device memory (wae_wave_shaper_set_device_curve):
  c2: N graphs of C2's shape with a distortion stage: stereo AudioBufferSource -> WaveShaper (1024 points, fused into k_chain) ->
      Biquad (lowpass, seeded f0 / Q) -> Gain -> destination;
  x4: M graphs of stereo AudioBufferSource -> WaveShaper (1024 points, oversample 4x) -> destination.
Per new curve set (a [N][1024] tensor of tanh curves of random drive and offset drawn on the GPU; about half map 0 to 0) it times, with
the card's name and power limit read in the same run (medians over --runs timed runs after --warmup untimed ones):
  (a) wae_batch_bind_curves alone (CUDA events on the engine stream around the item-table copy and k_bind_curves) and the host side
      of the bind call;
  (b) bind_curves + run + sync on the host clock;
  (c) what a caller does without it: copy the curves to the host, build the N contexts with them given to set_curve, prepare the batch,
      bind the same device audio, run, sync;
and the largest difference between (b)'s and (c)'s renders of the last curve set.  Prints one JSON line.  Writes nothing."""
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


def graph(pkg, G, be, workload, g, length, points, sr, curve=None):
    """curve None: the curve bound from device memory; else the points given to set_curve"""
    c = pkg.OfflineAudioContext(2, length, sr, be)
    src = c.create_buffer_source()
    src.set_device_input(2, length, sr)
    sh = c.create_wave_shaper(oversample=2 if workload == "x4" else 0)
    if curve is None:
        sh.set_device_curve(points)
    else:
        sh.set_curve(curve)
    src.connect(sh)
    if workload == "c2":
        _, f0, q, gain = G.c2_params(g)
        bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=f0, q=q)
        gn = c.create_gain(gain)
        sh.connect(bq)
        bq.connect(gn)
        gn.connect(c.destination())
    else:
        sh.connect(c.destination())
    src.start()
    return c, src, sh


def median(xs):
    return float(np.median(np.asarray(xs, np.float64)))


def bench(pkg, G, eng, torch, workload, n, L, points, sr, runs, warmup, seed):
    be = eng.backend
    gen = torch.Generator(device="cuda").manual_seed(seed)
    pcm = torch.rand((n, 2, L), generator=gen, device="cuda") * 2.0 - 1.0
    x = torch.linspace(-1.0, 1.0, points, device="cuda")

    def draw():
        drive = 0.5 + 4.0 * torch.rand((n, 1), generator=gen, device="cuda")
        lift = (torch.rand((n, 1), generator=gen, device="cuda") < 0.5).float() * 0.05
        return torch.tanh(drive * x[None, :]) + lift

    made = [graph(pkg, G, be, workload, g, L, points, sr) for g in range(n)]
    batch = pkg.Batch([c for c, _, _ in made])
    src_node, sh_node = made[0][1], made[0][2]
    batch.bind_sources(src_node, pcm)
    es = batch._engine_stream()
    res = {"graphs": n, "frames": L, "points": points, "channels": 2, "sample_rate": sr, "runs": runs}

    # (a) the bind alone: the caller's stream sleeps while the host validates, so e0 -> e1 spans the item-table copy and the kernel
    side = torch.cuda.Stream()
    bind_ms, host_ms = [], []
    for r in range(warmup + runs):
        curves = draw()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        with torch.cuda.stream(side):
            torch.cuda._sleep(40_000_000)
            e0.record(side)
            t0 = time.perf_counter()
            batch.bind_curves(sh_node, curves)
            t1 = time.perf_counter()
        e1.record(es)
        e1.synchronize()
        if r >= warmup:
            bind_ms.append(e0.elapsed_time(e1))
            host_ms.append((t1 - t0) * 1e3)
    res.update({"bind_ms": round(median(bind_ms), 4), "bind_call_host_ms": round(median(host_ms), 3)})

    # the kernel on its own (device time per launch, averaged over --runs binds)
    from torch.profiler import ProfilerActivity, profile
    curves = draw()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(runs):
            batch.bind_curves(sh_node, curves)
        torch.cuda.synchronize()
    for ev in prof.key_averages():
        if "k_bind_curves" in ev.key and ev.count:
            t = getattr(ev, "device_time_total", None)
            if t is None:
                t = ev.cuda_time_total
            res["k_bind_curves_ms"] = round(t / ev.count / 1e3, 4)

    # (b) bind_curves + run + sync
    e2e = []
    for r in range(warmup + runs):
        curves = draw()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        batch.bind_curves(sh_node, curves)
        batch.run()
        batch.sync()
        t1 = time.perf_counter()
        if r >= warmup:
            e2e.append((t1 - t0) * 1e3)
    res["b_bind_run_sync_ms"] = round(median(e2e), 2)
    last = curves
    bound_out = batch.output_tensor().clone()
    torch.cuda.synchronize()
    batch.destroy()
    del made, batch
    gc.collect()

    # (c) curves to the host + build + prepare + bind_sources + run + sync per curve set
    rebuild = []
    for r in range(warmup + runs):
        curves = last if r == warmup + runs - 1 else draw()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        host = curves.cpu().numpy()
        ctxs = [graph(pkg, G, be, workload, g, L, points, sr, host[g]) for g in range(n)]
        b = pkg.Batch([c for c, _, _ in ctxs])
        b.bind_sources(ctxs[0][1], pcm)
        b.run()
        b.sync()
        t1 = time.perf_counter()
        if r >= warmup:
            rebuild.append((t1 - t0) * 1e3)
        if r == warmup + runs - 1:
            rebuilt = b.output_tensor()
            res["bit_equal"] = bool(torch.equal(rebuilt, bound_out))
            res["max_abs_diff_b_vs_c"] = float((rebuilt - bound_out).abs().max().item())
            torch.cuda.synchronize()
        b.destroy()
        del ctxs, b
        gc.collect()
    res["c_host_build_prepare_run_sync_ms"] = round(median(rebuild), 2)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--c2-graphs", type=int, default=1000)
    ap.add_argument("--x4-graphs", type=int, default=256)
    ap.add_argument("--frames", type=int, default=48000)
    ap.add_argument("--points", type=int, default=1024)
    ap.add_argument("--sr", type=float, default=48000.0)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=5)
    a = ap.parse_args()
    import torch
    import conftest
    import graphs as G
    if not torch.cuda.is_available():
        raise SystemExit("curve_bind_bench: no CUDA device")
    pkg = conftest.load_package()
    eng = pkg.Engine(0)
    out = {}
    for workload, n in (("c2", a.c2_graphs), ("x4", a.x4_graphs)):
        out[workload] = bench(pkg, G, eng, torch, workload, n, a.frames, a.points, a.sr, a.runs, a.warmup, a.seed)
    out["card"] = card()
    print(json.dumps(out))
    eng.close()


if __name__ == "__main__":
    main()
