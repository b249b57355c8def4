"""Start times bound from device memory (wae_batch_bind_schedules) for event-based scenes, against rebuilding the graphs and against
baking the onsets into full-length device inputs in torch.  Needs a GPU.

Workload: N stereo scenes of 10 s at 48 kHz, each 8 device-input event clips of 1 s at onsets drawn in [0, 9] s, each clip followed by a
gain.  Variants, medians of --iters runs after one warm-up:
  (a) bind_sources + bind_schedules + bind_params + run + sync on one prepared batch;
  (b) build the graphs with the onsets and gains as host values + prepare + bind_sources + run + sync;
  (c) the torch workaround: each event zero-padded to a 10 s device input started at 0 (graph count halved until it fits); the caller
      tensor bytes are reported.
Also an oscillator note sequence (16 notes per graph -> lowpass -> gain) bound vs rebuilt, and the largest difference between (a) and
host-built renders of the same scenes.  Prints one JSON line; --out also writes it to a file.

    python tools/schedule_bind_bench.py [--out results.json]
"""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
SR = 48000.0


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True).strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def scene(pkg, be, k, seconds, clip, declare, onsets=None, gains=None, pcm=None, padded=False):
    c = pkg.OfflineAudioContext(2, int(seconds * SR), SR, be)
    srcs, gs = [], []
    for j in range(k):
        s = c.create_buffer_source()
        g = c.create_gain(1.0)
        if pcm is None:
            s.set_device_input(2, int(seconds * SR) if padded else clip, SR)
        else:
            s.set_buffer(pkg.AudioBuffer(list(pcm[j]), SR))
        if declare or padded:
            g.gain.set_device_value(0.0, 2.0)
        else:
            g.gain.set_value(float(gains[j]))
        s.connect(g)
        g.connect(c.destination())
        s.start_at(0.0 if (declare or padded) else float(onsets[j]))
        if declare:
            s.set_device_schedule((0.0, seconds))
        srcs.append(s)
        gs.append(g)
    return c, srcs, gs


def timed(fn, iters):
    fn()
    ts = []
    for _ in range(iters):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return statistics.median(ts) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--graphs", type=int, default=1000)
    ap.add_argument("--events", type=int, default=8)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    import torch
    from conftest import load_package
    pkg = load_package()
    if not torch.cuda.is_available():
        raise SystemExit("schedule_bind_bench needs a GPU")
    eng = pkg.Engine(0)
    n, k, clip = a.graphs, a.events, int(SR)
    res = {"card": card(), "graphs": n, "events": k, "seconds": a.seconds}
    gen = torch.Generator().manual_seed(1)
    pcm = (torch.rand((k, n, 2, clip), generator=gen) - 0.5).cuda()
    onsets = (torch.rand((n, k), generator=gen, dtype=torch.float64) * (a.seconds - 1.0)).cuda()
    gains = (torch.rand((n, k), generator=gen) * 1.5).cuda()

    # (a) one prepared batch: sources, onsets and gains bound per run
    made = [scene(pkg, eng.backend, k, a.seconds, clip, True) for _ in range(n)]
    b = pkg.Batch([m[0] for m in made])
    _, srcs, gs = made[0]

    def run_a():
        for j in range(k):
            b.bind_sources(srcs[j], pcm[j])
        b.bind_schedules(srcs, onsets)
        b.bind_params([g.gain for g in gs], gains)
        b.run()
        b.sync()
    res["a_bind3_run_sync_ms"] = timed(run_a, a.iters)
    run_a()
    got = b.fetch()

    def run_plain():
        b.run()
        b.sync()
    res["a_run_sync_only_ms"] = timed(run_plain, a.iters)
    b.destroy()
    del b, made
    gc.collect()

    # (b) rebuild with host start times (device-input clips, host gains and onsets) + prepare + bind + run + sync
    on_h, g_h = onsets.cpu().numpy(), gains.cpu().numpy()

    def run_b(keep=False):
        ms = [scene(pkg, eng.backend, k, a.seconds, clip, False, on_h[i], g_h[i]) for i in range(n)]
        bb = pkg.Batch([m[0] for m in ms])
        for j in range(k):
            bb.bind_sources(ms[0][1][j], pcm[j])
        bb.run()
        bb.sync()
        if not keep:
            bb.destroy()
        return bb
    res["b_rebuild_prepare_run_sync_ms"] = timed(run_b, max(1, a.iters - 1))
    bb = run_b(keep=True)
    ref = bb.fetch()
    bb.destroy()
    res["max_abs_diff_a_vs_host_built"] = float(np.abs(got - ref).max())
    res["bit_equal_scenes_a_vs_host_built"] = int(sum(np.array_equal(got[i], ref[i]) for i in range(n)))
    del bb, ref, got
    gc.collect()
    torch.cuda.empty_cache()

    # (c) torch workaround: every event baked into a zero-padded full-length device input
    m = n
    frames = int(a.seconds * SR)
    while m >= 1:
        try:
            padded = torch.zeros((k, m, 2, frames), device="cuda")
            break
        except torch.cuda.OutOfMemoryError:
            m //= 2
    mc = [scene(pkg, eng.backend, k, a.seconds, clip, False, padded=True) for _ in range(m)]
    bc = pkg.Batch([x[0] for x in mc])
    on_frames = (onsets[:m] * SR).round().long()

    def run_c():
        padded.zero_()
        for j in range(k):
            for i in range(m):
                f0 = int(on_frames[i, j])
                padded[j, i, :, f0:f0 + clip] = pcm[j, i]
            bc.bind_sources(mc[0][1][j], padded[j])
        bc.bind_params([g.gain for g in mc[0][2]], gains[:m])
        bc.run()
        bc.sync()
    res["c_graphs"] = m
    res["c_caller_tensor_bytes"] = int(padded.numel() * 4)
    res["c_pad_bind_run_sync_ms"] = timed(run_c, a.iters)
    bc.destroy()
    del bc, mc, padded
    gc.collect()
    torch.cuda.empty_cache()

    # oscillator note sequence: 16 notes per graph -> lowpass -> gain, onsets bound vs rebuilt
    notes = 16
    secs = 4.0
    starts = torch.sort(torch.rand((n, notes), generator=gen, dtype=torch.float64) * (secs - 0.25), dim=1).values.cuda()

    def seq(declare, st=None):
        c = pkg.OfflineAudioContext(1, int(secs * SR), SR, eng.backend)
        lp = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=3000.0)
        g = c.create_gain(0.2)
        lp.connect(g)
        g.connect(c.destination())
        oscs = []
        for j in range(notes):
            o = c.create_oscillator(type_=2, frequency=220.0 * 2 ** (j / 12))
            o.connect(lp)
            if declare:
                o.start_at(0.0)
                o.set_device_schedule((0.0, secs), stop=(0.0, secs))
            else:
                o.start_at(float(st[j]))
                o.stop_at(float(st[j]) + 0.25)
            oscs.append(o)
        return c, oscs
    ms = [seq(True) for _ in range(n)]
    bs = pkg.Batch([x[0] for x in ms])

    def run_seq():
        bs.bind_schedules(ms[0][1], starts, starts + 0.25)
        bs.run()
        bs.sync()
    res["notes_bind_run_sync_ms"] = timed(run_seq, a.iters)
    st_h = starts.cpu().numpy()

    def run_seq_b():
        bb = pkg.Batch([seq(False, st_h[i])[0] for i in range(n)])
        bb.run()
        bb.sync()
        return bb
    res["notes_rebuild_prepare_run_sync_ms"] = timed(run_seq_b, max(1, a.iters - 1))
    run_seq()
    res["notes_max_abs_diff_vs_host_built"] = float(np.abs(bs.fetch() - run_seq_b().fetch()).max())
    res["card_after"] = card()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
