#!/usr/bin/env python
"""Rendering a prepared batch into caller memory (wae_batch_bind_output) versus copying its own buffer (GPU).  The C2 shape of BASELINE
configs[1]: N graphs of AudioBufferSource -> lowpass biquad -> gain -> destination, 2 channels x L frames at 48 kHz, each source a device
input bound once.  Per step, on the host clock around work that ends in a device synchronise (medians over --runs timed steps after
--warmup untimed ones, the two variants alternated step by step):
  - ring: bind_output(ys[step % 2]) + run + sync, a two-tensor ring a consumer could read the other half of;
  - clone: run + output_tensor().clone() + sync, the copy a caller makes today to keep a step's output.
Also the clone alone (CUDA events on torch's stream around it, after the stream has waited for the run), the kernel-only time of the
run and whether both variants hold the same PCM to the bit.  The card's name and power limit are read in
the same run.  Prints one JSON line.  Writes nothing."""
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

import graphs as G  # noqa: E402  (tests/graphs.py: the shared graph builders)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # (reported, not fatal)
        return "unknown (%s)" % e


def c2_device(pkg, be, g, length, sr):
    _, f0, q, gain = G.c2_params(g)
    c = pkg.OfflineAudioContext(2, length, sr, be)
    src = c.create_buffer_source()
    src.set_device_input(2, length, sr)
    bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=f0, q=q)
    gn = c.create_gain(gain)
    src.connect(bq)
    bq.connect(gn)
    gn.connect(c.destination())
    src.start()
    return c, src


def median(xs):
    return float(np.median(np.asarray(xs, np.float64)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--graphs", type=int, default=1000)
    ap.add_argument("--frames", type=int, default=480000)
    ap.add_argument("--sr", type=float, default=48000.0)
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=5)
    a = ap.parse_args()
    import torch
    import conftest
    if not torch.cuda.is_available():
        raise SystemExit("output_bind_bench: no CUDA device")
    pkg = conftest.load_package()
    eng = pkg.Engine(0)
    n, L, sr = a.graphs, a.frames, a.sr
    gen = torch.Generator(device="cuda").manual_seed(a.seed)
    pcm = torch.rand((n, 2, L), generator=gen, device="cuda") * 2.0 - 1.0
    made = [c2_device(pkg, eng.backend, g, L, sr) for g in range(n)]
    batch = pkg.Batch([c for c, _ in made])
    batch.bind_sources(made[0][1], pcm)
    ys = [torch.empty((n, 2, L), device="cuda") for _ in range(2)]
    res = {"card": card(), "graphs": n, "frames": L, "channels": 2, "sample_rate": sr, "runs": a.runs,
           "output_bytes": n * 2 * L * 4}

    ring, clone, kern, copy = [], [], [], []
    kept = None
    for r in range(a.warmup + a.runs):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        batch.bind_output(ys[r % 2])
        batch.run()
        batch.sync()
        t1 = time.perf_counter()
        k_ring = batch.stats().last_run_ms
        batch.bind_output(None)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        batch.run()
        view = batch.output_tensor()  # (torch's stream now waits for the run: e0 completes when the run has)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        kept = view.clone()
        e1.record()
        torch.cuda.synchronize()
        t3 = time.perf_counter()
        if r >= a.warmup:
            ring.append((t1 - t0) * 1e3)
            clone.append((t3 - t2) * 1e3)
            kern.append(k_ring)
            copy.append(e0.elapsed_time(e1))
    last = ys[(a.warmup + a.runs - 1) % 2]
    same = bool((last.view(torch.int32) == kept.view(torch.int32)).all())
    res.update({"ring_step_ms": round(median(ring), 2), "clone_step_ms": round(median(clone), 2),
                "ring_step_spread_ms": [round(min(ring), 2), round(max(ring), 2)],
                "clone_step_spread_ms": [round(min(clone), 2), round(max(clone), 2)],
                "clone_alone_ms": round(median(copy), 2), "clone_alone_GBps": round(2 * res["output_bytes"] / (median(copy) * 1e-3) / 1e9, 1),
                "run_kernel_only_ms": round(median(kern), 2), "bit_equal": same})
    print(json.dumps(res))
    batch.destroy()
    eng.close()


if __name__ == "__main__":
    main()
