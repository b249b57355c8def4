#!/usr/bin/env python
"""AudioParam value curves bound from device memory versus the other ways to give every run its own automation (GPU).  N graphs of
sawtooth oscillator -> lowpass biquad -> gain -> destination, 2 channels x L frames at 48 kHz, with a pitch contour on the oscillator's
frequency, a cutoff sweep on the lowpass frequency and a loudness envelope on the gain: curves of P points over the whole render (P = 1000
over 10 s is a 100 Hz control rate).  With the card's name and power limit read in the same run, medians over --runs timed runs after
--warmup untimed ones.  The variants run one after the other, each batch destroyed before the next is prepared: a prepared batch sizes
its chunk to the device memory it finds, so batches of automated graphs of this size do not fit side by side.
  (a) wae_batch_bind_value_curves + run + sync per new curve set (host clock);
  (b) the same graphs built with host curves (set_value_curve_at_time) and prepared, per new curve set (host clock; and + run + sync);
  (c) the per-frame route: each of the three params fed by a device-input AudioBufferSourceNode whose clip is the curve sampled at
      every frame, wae_batch_bind_sources + run + sync per run (the per-frame tensors of the last curve set, made once before any batch
      is prepared); when the batch does not fit in device memory, the graph count is
      halved until it does and reported ("c_graphs");
  (d) for comparison, the host-built chain with constant pitch, cutoff and gain, which k_chain renders fused;
the per-stage kernel times of (a) and (d) in a run of their own, and the largest difference between the bound renders and the host-built
renders of the same curves.  Prints one JSON line.  Writes nothing."""
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


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # (reported, not fatal)
        return "unknown (%s)" % e


def graph(pkg, be, length, sr, points, curves=None, route="bound"):
    """route "bound": the three curves declared (curves None); "host": curves = (f0, cutoff, gain) host arrays; "frames": the three
    params at 0 fed by device-input sources; "constant": 220 Hz, 2 kHz, 0.5.  Returns (context, params or sources)."""
    c = pkg.OfflineAudioContext(2, length, sr, be)
    zero = route == "frames"
    o = c.create_oscillator(type_=pkg.context.SAWTOOTH, frequency=0.0 if zero else 220.0)
    bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=0.0 if zero else 2000.0)
    gn = c.create_gain(0.0 if zero else 0.5)
    o.connect(bq)
    bq.connect(gn)
    gn.connect(c.destination())
    o.start()
    params = [o.frequency, bq.frequency, gn.gain]
    dur = length / sr
    if route == "bound":
        for p in params:
            p.set_device_value_curve(points, 0.0, dur)
    elif route == "host":
        for p, v in zip(params, curves):
            p.set_value_curve_at_time(v, 0.0, dur)
    elif route == "frames":
        srcs = []
        for p in params:
            s = c.create_buffer_source()
            s.set_device_input(1, length, sr)
            s.connect(p)
            s.start()
            srcs.append(s)
        return c, srcs
    return c, params


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
    ap.add_argument("--points", type=int, default=1000)
    ap.add_argument("--sr", type=float, default=48000.0)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--seed", type=int, default=5)
    a = ap.parse_args()
    import torch
    import conftest
    if not torch.cuda.is_available():
        raise SystemExit("value_curve_bind_bench: no CUDA device")
    pkg = conftest.load_package()
    eng = pkg.Engine(0)
    be = eng.backend
    n, L, sr, P = a.graphs, a.frames, a.sr, a.points
    gen = torch.Generator(device="cuda").manual_seed(a.seed)

    def draw():
        """a new curve set: f0 in [110, 440] Hz, cutoff in [300, 6000] Hz, gain in [0.1, 0.9], [n][P] each"""
        r = lambda: torch.rand((n, P), generator=gen, device="cuda")
        return [110.0 + 330.0 * r(), 300.0 + 5700.0 * r(), 0.1 + 0.8 * r()]

    def per_frame(curves):
        """each curve at every frame, as the curve interpolation gives it ([n][1][L] each): the clips of route (c)"""
        pos = torch.clamp(torch.arange(L, device="cuda", dtype=torch.float64) * ((P - 1) / L), max=P - 1)
        k = torch.clamp(pos.floor().long(), max=P - 2)
        frac = (pos - k).float()
        return [(v[:, k] + (v[:, k + 1] - v[:, k]) * frac).unsqueeze(1).contiguous() for v in curves]

    res = {"graphs": n, "frames": L, "channels": 2, "sample_rate": sr, "points": P, "runs": a.runs}
    res["caller_tensor_bytes"] = {"a_curves": 3 * n * P * 4, "c_per_frame": 3 * n * L * 4}
    sets = [draw() for _ in range(a.warmup + a.runs)]
    last = sets[-1]
    clips = per_frame(last)  # (made first: the batches below size their chunks to the device memory they find)

    # (a)
    bound_ctx = [graph(pkg, be, L, sr, P) for _ in range(n)]
    bound = pkg.Batch([c for c, _ in bound_ctx])
    params = bound_ctx[0][1]
    t_a = []
    for r, curves in enumerate(sets):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        bound.bind_value_curves(params, curves)
        bound.run()
        bound.sync()
        if r >= a.warmup:
            t_a.append((time.perf_counter() - t0) * 1e3)
    res["a_bind_run_sync_ms"] = round(median(t_a), 2)
    res["stages_ms_bound"] = {k: round(v, 3) for k, v in stage_times(bound).items()}
    out_a = bound.output_tensor().cpu()
    bound.destroy()

    # (b)
    t_b, t_b_run = [], []
    for r, curves in enumerate(sets):
        host_curves = [v.cpu().numpy() for v in curves]
        t1 = time.perf_counter()
        host = pkg.Batch([graph(pkg, be, L, sr, P, [h[g] for h in host_curves], route="host")[0] for g in range(n)])
        t2 = time.perf_counter()
        host.run()
        host.sync()
        t3 = time.perf_counter()
        if r >= a.warmup:
            t_b.append((t2 - t1) * 1e3)
            t_b_run.append((t3 - t1) * 1e3)
        if r < len(sets) - 1:
            host.destroy()
    res["b_build_prepare_ms"] = round(median(t_b), 1)
    res["b_build_prepare_run_sync_ms"] = round(median(t_b_run), 1)
    res["max_abs_diff_bound_vs_host_built"] = float((out_a - host.output_tensor().cpu()).abs().max().item())
    host.destroy()

    # (d)
    constant = pkg.Batch([graph(pkg, be, L, sr, P, route="constant")[0] for _ in range(n)])
    t_d = []
    for r in range(a.warmup + a.runs):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        constant.run()
        constant.sync()
        if r >= a.warmup:
            t_d.append((time.perf_counter() - t0) * 1e3)
    res["d_constant_chain_run_sync_ms"] = round(median(t_d), 2)
    res["stages_ms_constant"] = {k: round(v, 3) for k, v in stage_times(constant).items()}
    constant.destroy()

    # (c)
    nc = n
    while True:
        try:
            frames_ctx = [graph(pkg, be, L, sr, P, route="frames") for _ in range(nc)]
            frames = pkg.Batch([c for c, _ in frames_ctx])
            break
        except pkg.WaeError as e:
            if e.status != 6 or nc == 1:
                raise
            nc //= 2
    res["c_graphs"] = nc
    srcs = frames_ctx[0][1]
    t_c = []
    for r in range(a.warmup + a.runs):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for s, clip in zip(srcs, clips):
            frames.bind_sources(s, clip[:nc])
        frames.run()
        frames.sync()
        if r >= a.warmup:
            t_c.append((time.perf_counter() - t0) * 1e3)
    res["c_per_frame_bind_run_sync_ms"] = round(median(t_c), 2)
    res["max_abs_diff_bound_vs_per_frame"] = float((out_a[:nc] - frames.output_tensor().cpu()).abs().max().item())
    res["stages_ms_per_frame"] = {k: round(v, 3) for k, v in stage_times(frames).items()}
    res["card"] = card()
    print(json.dumps(res))
    frames.destroy()
    eng.close()


if __name__ == "__main__":
    main()
