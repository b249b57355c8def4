#!/usr/bin/env python
"""A new set of convolver responses for a prepared batch, bound from device memory versus built again (GPU).  The C4 shape of BASELINE
configs[3]: N graphs of stereo AudioBufferSource -> ConvolverNode (normalised) -> destination, 2 channels x L frames at 48 kHz, each
source a device input (wae_buffer_source_set_device_input) and each response a stereo R-frame response declared bound from device memory
(wae_convolver_set_device_response).  Per new response set (a [N][2][R] tensor of decaying noise drawn on the GPU) it times, with the
card's name and power limit read in the same run (medians over --runs timed runs after --warmup untimed ones):
  (a) wae_batch_bind_responses alone (CUDA events on the engine stream around the item-table copy and the three kernels), the host
      side of the bind call, and the device time of each kernel (power / trim / transform, torch.profiler in a pass of its own);
  (b) bind_responses + run + sync on the host clock;
  (c) what a caller does without it: copy the responses to the host, build the N contexts with them as AudioBuffers, prepare the batch,
      bind the same device audio, run, sync;
and whether (a)'s and (c)'s renders of the last response set are bit-equal (with their largest difference).  Prints one JSON line.
Writes nothing."""
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

KERNELS = ("k_resp_power", "k_resp_trim", "k_resp_fft")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # (reported, not fatal)
        return "unknown (%s)" % e


def c4(pkg, be, length, ir_len, sr, ir=None):
    """ir None: the response bound from device memory; else a [2][ir_len] float32 array given to set_buffer"""
    c = pkg.OfflineAudioContext(2, length, sr, be)
    src = c.create_buffer_source()
    src.set_device_input(2, length, sr)
    cv = c.create_convolver()
    if ir is None:
        cv.set_device_response(2, ir_len, sr)
    else:
        cv.set_buffer(pkg.AudioBuffer([ir[0], ir[1]], sr))
    src.connect(cv)
    cv.connect(c.destination())
    src.start()
    return c, src, cv


def median(xs):
    return float(np.median(np.asarray(xs, np.float64)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--graphs", type=int, default=128)
    ap.add_argument("--frames", type=int, default=480000)
    ap.add_argument("--ir-frames", type=int, default=178899)
    ap.add_argument("--sr", type=float, default=48000.0)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=5)
    a = ap.parse_args()
    import torch
    import conftest
    if not torch.cuda.is_available():
        raise SystemExit("response_bind_bench: no CUDA device")
    pkg = conftest.load_package()
    eng = pkg.Engine(0)
    be = eng.backend
    n, L, R, sr = a.graphs, a.frames, a.ir_frames, a.sr
    gen = torch.Generator(device="cuda").manual_seed(a.seed)
    pcm = (torch.rand((n, 2, L), generator=gen, device="cuda") * 2.0 - 1.0) * 0.05
    env = torch.exp(-torch.arange(R, device="cuda", dtype=torch.float32) / (0.25 * sr))

    def draw():  # decaying noise, G.synthetic_ir's shape
        return torch.randn((n, 2, R), generator=gen, device="cuda") * env

    made = [c4(pkg, be, L, R, sr) for _ in range(n)]
    batch = pkg.Batch([c for c, _, _ in made])
    src_node, cv_node = made[0][1], made[0][2]
    batch.bind_sources(src_node, pcm)
    es = batch._engine_stream()
    res = {"graphs": n, "frames": L, "ir_frames": R, "channels": 2, "sample_rate": sr, "runs": a.runs}

    # (a) the bind alone: the caller's stream sleeps while the host validates, so e0 -> e1 spans the item-table copy and the kernels
    side = torch.cuda.Stream()
    bind_ms, host_ms = [], []
    for r in range(a.warmup + a.runs):
        irs = draw()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        with torch.cuda.stream(side):
            torch.cuda._sleep(40_000_000)
            e0.record(side)
            t0 = time.perf_counter()
            batch.bind_responses(cv_node, irs)
            t1 = time.perf_counter()
        e1.record(es)
        e1.synchronize()
        if r >= a.warmup:
            bind_ms.append(e0.elapsed_time(e1))
            host_ms.append((t1 - t0) * 1e3)
    res.update({"bind_ms": round(median(bind_ms), 4), "bind_call_host_ms": round(median(host_ms), 3)})

    # the kernels of the bind, each on its own (device time per launch, averaged over --runs binds)
    from torch.profiler import ProfilerActivity, profile
    irs = draw()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.runs):
            batch.bind_responses(cv_node, irs)
        torch.cuda.synchronize()
    for ev in prof.key_averages():
        for k in KERNELS:
            if k in ev.key and ev.count:
                t = getattr(ev, "device_time_total", None)
                if t is None:
                    t = ev.cuda_time_total
                res[k + "_ms"] = round(t / ev.count / 1e3, 4)

    # (b) bind_responses + run + sync
    e2e = []
    for r in range(a.warmup + a.runs):
        irs = draw()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        batch.bind_responses(cv_node, irs)
        batch.run()
        batch.sync()
        t1 = time.perf_counter()
        if r >= a.warmup:
            e2e.append((t1 - t0) * 1e3)
    res["b_bind_run_sync_ms"] = round(median(e2e), 2)
    last = irs
    bound_out = batch.output_tensor().clone()
    torch.cuda.synchronize()
    batch.destroy()
    del made, batch
    gc.collect()

    # (c) responses to the host + build + prepare + bind_sources + run + sync per response set
    rebuild = []
    for r in range(a.warmup + a.runs):
        irs = last if r == a.warmup + a.runs - 1 else draw()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        host = irs.cpu().numpy()
        ctxs = [c4(pkg, be, L, R, sr, host[i]) for i in range(n)]
        b = pkg.Batch([c for c, _, _ in ctxs])
        b.bind_sources(ctxs[0][1], pcm)
        b.run()
        b.sync()
        t1 = time.perf_counter()
        if r >= a.warmup:
            rebuild.append((t1 - t0) * 1e3)
        if r == a.warmup + a.runs - 1:
            rebuilt = b.output_tensor()
            res["bit_equal"] = bool(torch.equal(rebuilt, bound_out))
            res["max_abs_diff_b_vs_c"] = float((rebuilt - bound_out).abs().max().item())
            torch.cuda.synchronize()
        b.destroy()
        del ctxs, b
        gc.collect()
    res["c_host_build_prepare_run_sync_ms"] = round(median(rebuild), 2)
    res["card"] = card()
    print(json.dumps(res))
    eng.close()


if __name__ == "__main__":
    main()
