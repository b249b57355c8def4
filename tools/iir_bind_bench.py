#!/usr/bin/env python
"""A new set of IIRFilterNode coefficients for a prepared batch, bound from device memory versus built again (GPU).  Two workloads of
N graphs (default 1000), each stereo, --frames long at --sr: a device input (wae_buffer_source_set_device_input) -> IIRFilterNode
(coefficients declared bound from device memory, wae_iir_filter_set_device_coefficients) -> destination, with
  order2: 3 feedforward / 3 feedback coefficients (the k_chain scan);
  coef8: 8 / 8 coefficients (k_iir_serial, one thread per graph and channel).
Per new coefficient set (f64 [N][nff] / [N][nfb] tensors of Butterworth low-passes of random cutoff, made on the host once and scaled by
a random factor on the GPU per set) it times, with the card's name and power limit read in the same run (medians over --runs timed runs
after --warmup untimed ones):
  (a) wae_batch_bind_iir_coefficients alone (CUDA events on the engine stream around the item-table copy and k_bind_iir), k_bind_iir per
      launch (torch.profiler), and the host side of the bind call;
  (b) bind_iir_coefficients + run + sync on the host clock;
  (c) what a caller does without it: copy the coefficients to the host, build the N contexts with create_iir_filter, prepare the batch,
      bind the same device audio, run, sync;
and whether (b)'s and (c)'s renders of the last set are bit-equal.  Prints one JSON line.  Writes nothing."""
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

WORKLOADS = {"order2": (3, 3), "coef8": (8, 8)}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # (reported, not fatal)
        return "unknown (%s)" % e


def graph(pkg, be, length, sr, nff, nfb, coefs=None):
    """coefs None: the coefficients bound from device memory; else the (feedforward, feedback) given to create_iir_filter"""
    c = pkg.OfflineAudioContext(2, length, sr, be)
    src = c.create_buffer_source()
    src.set_device_input(2, length, sr)
    if coefs is None:
        f = c.create_iir_filter([1.0] + [0.0] * (nff - 1), [1.0] + [0.0] * (nfb - 1))
        f.set_device_coefficients()
    else:
        f = c.create_iir_filter(coefs[0], coefs[1])
    src.connect(f)
    f.connect(c.destination())
    src.start()
    return c, src, f


def median(xs):
    return float(np.median(np.asarray(xs, np.float64)))


def bench(pkg, eng, torch, workload, n, L, sr, runs, warmup, seed):
    from scipy import signal
    nff, nfb = WORKLOADS[workload]
    be = eng.backend
    rng = np.random.default_rng(seed)
    base = [signal.butter(nfb - 1, rng.uniform(0.05, 0.8)) for _ in range(n)]
    ff0 = torch.from_numpy(np.stack([b for b, _ in base])).cuda()
    fb0 = torch.from_numpy(np.stack([a for _, a in base])).cuda()
    gen = torch.Generator(device="cuda").manual_seed(seed)
    pcm = torch.rand((n, 2, L), generator=gen, device="cuda") * 2.0 - 1.0

    def draw():  # a new set: the same filters, each scaled by its own factor (normalised away, except in the feedforward)
        s = 0.5 + torch.rand((n, 1), generator=gen, device="cuda", dtype=torch.float64)
        return ff0 * s * 0.75, fb0 * s

    made = [graph(pkg, be, L, sr, nff, nfb) for _ in range(n)]
    batch = pkg.Batch([c for c, _, _ in made])
    src_node, iir_node = made[0][1], made[0][2]
    batch.bind_sources(src_node, pcm)
    es = batch._engine_stream()
    res = {"graphs": n, "frames": L, "feedforward": nff, "feedback": nfb, "channels": 2, "sample_rate": sr, "runs": runs,
           "kernels": sorted({k for k, _t, _n in batch.stage_times()})}

    # (a) the bind alone: the caller's stream sleeps while the host validates, so e0 -> e1 spans the item-table copy and the kernel
    side = torch.cuda.Stream()
    bind_ms, host_ms = [], []
    for r in range(warmup + runs):
        ff, fb = draw()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        with torch.cuda.stream(side):
            torch.cuda._sleep(40_000_000)
            e0.record(side)
            t0 = time.perf_counter()
            batch.bind_iir_coefficients(iir_node, ff, fb)
            t1 = time.perf_counter()
        e1.record(es)
        e1.synchronize()
        if r >= warmup:
            bind_ms.append(e0.elapsed_time(e1))
            host_ms.append((t1 - t0) * 1e3)
    res.update({"bind_ms": round(median(bind_ms), 4), "bind_call_host_ms": round(median(host_ms), 3)})

    # the kernel on its own (device time per launch, averaged over --runs binds)
    from torch.profiler import ProfilerActivity, profile
    ff, fb = draw()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(runs):
            batch.bind_iir_coefficients(iir_node, ff, fb)
        torch.cuda.synchronize()
    for ev in prof.key_averages():
        if "k_bind_iir" in ev.key and ev.count:
            t = getattr(ev, "device_time_total", None)
            if t is None:
                t = ev.cuda_time_total
            res["k_bind_iir_ms"] = round(t / ev.count / 1e3, 4)

    # (b) bind_iir_coefficients + run + sync
    e2e = []
    for r in range(warmup + runs):
        ff, fb = draw()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        batch.bind_iir_coefficients(iir_node, ff, fb)
        batch.run()
        batch.sync()
        t1 = time.perf_counter()
        if r >= warmup:
            e2e.append((t1 - t0) * 1e3)
    res["b_bind_run_sync_ms"] = round(median(e2e), 2)
    last = (ff, fb)
    bound_out = batch.output_tensor().clone()
    torch.cuda.synchronize()
    batch.destroy()
    del made, batch
    gc.collect()

    # (c) coefficients to the host + build + prepare + bind_sources + run + sync per set
    rebuild = []
    for r in range(warmup + runs):
        ff, fb = last if r == warmup + runs - 1 else draw()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        hff, hfb = ff.cpu().numpy(), fb.cpu().numpy()
        ctxs = [graph(pkg, be, L, sr, nff, nfb, (hff[g], hfb[g])) for g in range(n)]
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
    ap.add_argument("--graphs", type=int, default=1000)
    ap.add_argument("--frames", type=int, default=48000)
    ap.add_argument("--sr", type=float, default=48000.0)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=5)
    a = ap.parse_args()
    import torch
    import conftest
    if not torch.cuda.is_available():
        raise SystemExit("iir_bind_bench: no CUDA device")
    pkg = conftest.load_package()
    eng = pkg.Engine(0)
    out = {}
    for workload in WORKLOADS:
        out[workload] = bench(pkg, eng, torch, workload, a.graphs, a.frames, a.sr, a.runs, a.warmup, a.seed)
    out["card"] = card()
    print(json.dumps(out))
    eng.close()


if __name__ == "__main__":
    main()
