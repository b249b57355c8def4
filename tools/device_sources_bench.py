#!/usr/bin/env python
"""New input audio for a prepared batch, from device memory versus from the host (GPU).  The C2 shape of BASELINE configs[1]: N graphs of
AudioBufferSource -> lowpass biquad -> gain -> destination, 2 channels x L frames at 48 kHz (G.c2_buffer_biquad_gain's filters), each
graph's source declared as a device input (wae_buffer_source_set_device_input).  Reports, with the card's name and power limit read in
the same run (medians over --runs timed runs after --warmup untimed ones):
  - wae_batch_bind_sources alone: CUDA events on the engine stream around the call (k_bind_sources plus its item-table copy), its
    algorithmic bytes (sum ch * len * 4 read + sum ch * stride * 4 written), their rate, and that rate against the H100 SXM's 3.35 TB/s;
  - a new input set: bind + run + sync on the host clock, and the run's kernel-only time;
  - the host paths on the same PCM: wae_batch_upload + run + sync from page-locked host PCM (the same graphs with AudioBuffers), and the
    one-shot wae_render_batch into page-locked memory on freshly built graphs;
  - whether the bound render equals the AudioBuffer render bit for bit (seeded PCM).
Prints one JSON line.  Writes nothing."""
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
HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet

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
    ap.add_argument("--runs", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=5)
    a = ap.parse_args()
    import torch
    import conftest
    if not torch.cuda.is_available():
        raise SystemExit("device_sources_bench: no CUDA device")
    pkg = conftest.load_package()
    eng = pkg.Engine(0)
    be = eng.backend
    n, L, sr = a.graphs, a.frames, a.sr
    stride = (L + 3) // 4 * 4
    gen = torch.Generator(device="cuda").manual_seed(a.seed)
    pcm = torch.rand((n, 2, L), generator=gen, device="cuda") * 2.0 - 1.0

    made = [c2_device(pkg, be, g, L, sr) for g in range(n)]
    batch = pkg.Batch([c for c, _ in made])
    node = made[0][1]
    es = batch._engine_stream()
    res = {"graphs": n, "frames": L, "channels": 2, "sample_rate": sr, "runs": a.runs}

    # bind alone.  The bind waits for the caller's stream, which sleeps on the device while the host validates the items: e0 (recorded
    # on the caller's stream after the sleep) -> e1 (engine stream, after the kernel) then spans the item-table copy and k_bind_sources,
    # not the host-side checks, which are timed on their own (host clock around the call)
    side = torch.cuda.Stream()
    bind_ms, check_ms = [], []
    for r in range(a.warmup + a.runs):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        with torch.cuda.stream(side):
            torch.cuda._sleep(40_000_000)  # about 20 ms at 2 GHz, longer than the host-side checks
            e0.record(side)
            t0 = time.perf_counter()
            batch.bind_sources(node, pcm)
            t1 = time.perf_counter()
        e1.record(es)
        e1.synchronize()
        if r >= a.warmup:
            bind_ms.append(e0.elapsed_time(e1))
            check_ms.append((t1 - t0) * 1e3)
    bytes_bind = n * 2 * L * 4 + n * 2 * stride * 4
    ms = median(bind_ms)
    res.update({"bind_ms": round(ms, 3), "bind_bytes": bytes_bind, "bind_GBps": round(bytes_bind / (ms * 1e-3) / 1e9, 1),
                "bind_share_of_3.35TBps": round(bytes_bind / (ms * 1e-3) / HBM_BYTES_PER_S, 3),
                "bind_call_host_ms": round(median(check_ms), 3)})

    # a new input set: bind + run + sync
    e2e, kern = [], []
    for r in range(a.warmup + a.runs):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        batch.bind_sources(node, pcm)
        batch.run()
        batch.sync()
        t1 = time.perf_counter()
        if r >= a.warmup:
            e2e.append((t1 - t0) * 1e3)
            kern.append(batch.stats().last_run_ms)
    res.update({"new_input_set_ms": round(median(e2e), 2), "run_kernel_only_ms": round(median(kern), 2)})
    bound_out = batch.output_tensor().clone()
    torch.cuda.synchronize()

    # the same PCM through AudioBuffers: upload + run + sync from page-locked host PCM
    host = pcm.cpu().numpy()
    batch.destroy()
    del made, batch, node
    gc.collect()
    bctx = [G.c2_buffer_biquad_gain(pkg, be, g, L, sr, pcm=host[g]) for g in range(n)]
    bb = pkg.Batch(bctx)
    up = []
    for r in range(a.warmup + a.runs):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        bb.upload()
        bb.run()
        bb.sync()
        t1 = time.perf_counter()
        if r >= a.warmup:
            up.append((t1 - t0) * 1e3)
    res["upload_run_sync_pinned_ms"] = round(median(up), 2)
    buf_out = bb.output_tensor()
    res["bound_equals_buffer_render"] = bool(torch.equal(bound_out, buf_out))
    del buf_out, bound_out
    bb.destroy()
    del bb, bctx
    gc.collect()

    # one-shot wae_render_batch into page-locked memory, fresh graphs every call (built outside the timed window)
    out = torch.empty((n, 2, L), dtype=torch.float32, pin_memory=True).numpy()
    one = []
    for r in range(a.warmup + a.runs):
        ctxs = [G.c2_buffer_biquad_gain(pkg, be, g, L, sr, pcm=host[g]) for g in range(n)]
        t0 = time.perf_counter()
        pkg.render_batch_oneshot(ctxs, out)
        t1 = time.perf_counter()
        if r >= a.warmup:
            one.append((t1 - t0) * 1e3)
        del ctxs
        gc.collect()
    res["oneshot_pinned_ms"] = round(median(one), 2)
    res["card"] = card()
    print(json.dumps(res))
    eng.close()


if __name__ == "__main__":
    main()
