#!/usr/bin/env python
"""New input audio for a prepared batch, copied into its slab versus read by reference (GPU).  The C2 shape of BASELINE configs[1]: N graphs
of AudioBufferSource -> lowpass biquad -> gain -> destination, 2 channels x L frames at 48 kHz (G.c2_buffer_biquad_gain's filters), each
graph's source a device input declared for a copy (wae_buffer_source_set_device_input) in one batch and by reference
(wae_buffer_source_set_device_input_by_reference) in the other.  Reports, with the card's name and power limit read in the same run
(medians over --runs timed runs after --warmup untimed ones, the two modes alternated):
  - a new input set: bind + run + sync on the host clock, and the run's kernel-only time, per mode;
  - the bind alone by CUDA events on the engine stream (k_bind_sources with its item-table copy, against k_bind_source_refs with its own),
    the bind call's host time, and bind + run by CUDA events with the host side hidden behind a device sleep (the device time of a
    new input set);
  - the prepared batch's device memory: its asset_bytes and the cudaMemGetInfo delta of prepare, per mode;
  - the by-reference mode from a tensor whose channel stride is L + 1 (not a multiple of 4: k_chain gathers frame by frame);
  - whether the renders of the three are bit-equal (seeded PCM).
Prints one JSON line.  Writes nothing."""
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


def c2_device(pkg, be, g, length, sr, by_reference):
    _, f0, q, gain = G.c2_params(g)
    c = pkg.OfflineAudioContext(2, length, sr, be)
    src = c.create_buffer_source()
    src.set_device_input(2, length, sr, by_reference=by_reference)
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
        raise SystemExit("source_ref_bench: no CUDA device")
    pkg = conftest.load_package()
    eng = pkg.Engine(0)
    be = eng.backend
    n, L, sr = a.graphs, a.frames, a.sr
    gen = torch.Generator(device="cuda").manual_seed(a.seed)
    pcm = torch.rand((n, 2, L), generator=gen, device="cuda") * 2.0 - 1.0
    odd = torch.empty((n, 2, L + 1), device="cuda")  # channel stride L + 1
    odd[:, :, :L] = pcm
    odd = odd[:, :, :L]
    res = {"card": card(), "graphs": n, "frames": L, "channels": 2, "sample_rate": sr, "runs": a.runs, "warmup": a.warmup}

    batches = {}
    for mode in ("copy", "ref"):
        made = [c2_device(pkg, be, g, L, sr, mode == "ref") for g in range(n)]
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        b = pkg.Batch([c for c, _ in made])
        torch.cuda.synchronize()
        free1 = torch.cuda.mem_get_info()[0]
        batches[mode] = (b, made[0][1])
        res[f"{mode}_asset_bytes"] = int(b.stats().asset_bytes)
        res[f"{mode}_prepare_device_bytes"] = int(free0 - free1)

    # a new input set, the two modes alternated (and the by-reference mode from the stride-(L + 1) tensor)
    cases = [("copy", pcm), ("ref", pcm), ("ref_odd_stride", odd)]
    e2e = {k: [] for k, _ in cases}
    kern = {k: [] for k, _ in cases}
    for r in range(a.warmup + a.runs):
        for key, t in cases:
            b, node = batches[key.split("_")[0]]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            b.bind_sources(node, t)
            b.run()
            b.sync()
            t1 = time.perf_counter()
            if r >= a.warmup:
                e2e[key].append((t1 - t0) * 1e3)
                kern[key].append(b.stats().last_run_ms)
    for key, _ in cases:
        res[f"{key}_new_input_set_ms"] = round(median(e2e[key]), 3)
        res[f"{key}_run_kernel_only_ms"] = round(median(kern[key]), 3)

    # the bind alone.  The bind waits for the caller's stream, which sleeps on the device while the host validates the items: e0
    # (recorded on the caller's stream after the sleep) -> e1 (engine stream, after the kernel) spans the item-table copy and the bind
    # kernel, not the host-side checks
    side = torch.cuda.Stream()
    bind = {"copy": [], "ref": []}
    host = {"copy": [], "ref": []}
    dev = {"copy": [], "ref": []}
    for r in range(a.warmup + a.runs):
        for mode in ("copy", "ref"):
            b, node = batches[mode]
            es = b._engine_stream()
            for with_run in (False, True):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                with torch.cuda.stream(side):
                    torch.cuda._sleep(60_000_000)  # about 30 ms at 2 GHz, longer than the host side of bind (+ run)
                    e0.record(side)
                    t0 = time.perf_counter()
                    b.bind_sources(node, pcm)
                    t1 = time.perf_counter()
                    if with_run:
                        b.run()
                e1.record(es)
                e1.synchronize()
                if r >= a.warmup:
                    (dev if with_run else bind)[mode].append(e0.elapsed_time(e1))
                    if not with_run:
                        host[mode].append((t1 - t0) * 1e3)
    res["k_bind_sources_ms"] = round(median(bind["copy"]), 4)
    res["k_bind_source_refs_ms"] = round(median(bind["ref"]), 4)
    for mode in ("copy", "ref"):
        res[f"{mode}_bind_call_host_ms"] = round(median(host[mode]), 3)
        res[f"{mode}_bind_run_device_ms"] = round(median(dev[mode]), 3)

    outs = {}
    for key, t in cases:
        b, node = batches[key.split("_")[0]]
        b.bind_sources(node, t)
        b.run()
        outs[key] = b.output_tensor().clone()
    torch.cuda.synchronize()
    res["ref_equals_copy_render"] = bool(torch.equal(outs["ref"].view(torch.int32), outs["copy"].view(torch.int32)))
    res["ref_odd_stride_equals_copy_render"] = bool(torch.equal(outs["ref_odd_stride"].view(torch.int32), outs["copy"].view(torch.int32)))
    for b, _ in batches.values():
        b.destroy()
    eng.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
