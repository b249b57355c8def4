"""AudioBufferSourceNode offsets bound from device memory (wae_buffer_source_set_device_offset + wae_batch_bind_schedules) for
excerpt-based augmentation, against gathering the excerpts in torch and binding them as clips, and against rebuilding the graphs.  Needs a
GPU.

Workload: N mono graphs at 48 kHz, each a long recording (--recording s) -> lowpass -> gain, rendering an excerpt of --seconds at an
offset drawn per run.  The recordings are device tensors made once.  Per new excerpt set, medians of --iters after one warm-up:
  (a) bound: the recordings bound once (device inputs of the full length); per set bind_schedules(start 0, offsets) + run + sync;
  (b) gather: device inputs of the excerpt's length; per set a torch gather of the excerpts + bind_sources + run + sync;
  (c) rebuild: graphs built with the offsets as host values + prepare + bind_sources of the recordings + run + sync.
Each route reports its host-side time (the calls up to the return of run, before the sync) and its total (after the sync), and the time
of run + sync alone on its prepared batch.  Offsets are whole frames, so (a) and (b) play the same samples; the largest difference
between their outputs is reported.  Prints one JSON line with the card's name and power limit, read in the same run; --out also writes it.

    python tools/offset_bind_bench.py [--graphs 1000] [--recording 30] [--seconds 4] [--out results.json]
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


def graph(pkg, be, in_len, length, declare_offset, offset=0.0):
    """device input of in_len frames -> lowpass -> gain (both bound) -> destination, length frames"""
    c = pkg.OfflineAudioContext(1, length, SR, be)
    s = c.create_buffer_source()
    s.set_device_input(1, in_len, SR)
    lp = c.create_biquad_filter(type_=pkg.LOWPASS)
    g = c.create_gain()
    lp.frequency.set_device_value(100.0, 8000.0)
    g.gain.set_device_value(0.0, 2.0)
    s.connect(lp)
    lp.connect(g)
    g.connect(c.destination())
    if declare_offset:
        s.start_at(0.0)
        s.set_device_schedule((0.0, 0.0), offset=(0.0, in_len / SR))
    else:
        s.start_at_with_offset(0.0, offset)
    return c, s, lp, g


def timed(fn, iters):
    """fn() returns its host-side time; medians (ms) of the host-side and total times"""
    fn()
    hs, ts = [], []
    for _ in range(iters):
        t0 = time.perf_counter()
        hs.append(fn() - t0)
        ts.append(time.perf_counter() - t0)
    return statistics.median(hs) * 1e3, statistics.median(ts) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--graphs", type=int, default=1000)
    ap.add_argument("--recording", type=float, default=30.0, help="seconds per recording")
    ap.add_argument("--seconds", type=float, default=4.0, help="seconds per excerpt")
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    import torch
    from conftest import load_package
    pkg = load_package()
    if not torch.cuda.is_available():
        raise SystemExit("offset_bind_bench needs a GPU")
    eng = pkg.Engine(0)
    n, rec_len, length = a.graphs, int(a.recording * SR), int(a.seconds * SR)
    res = {"card": card(), "graphs": n, "recording_s": a.recording, "excerpt_s": a.seconds, "iters": a.iters}
    gen = torch.Generator(device="cuda").manual_seed(1)
    recs = torch.rand((n, 1, rec_len), generator=gen, device="cuda").sub_(0.5)
    cutoffs = torch.rand(n, generator=gen, device="cuda") * 4000.0 + 500.0
    gains = torch.rand(n, generator=gen, device="cuda") * 1.5
    params = torch.stack([cutoffs, gains], dim=1)
    sets = [torch.randint(0, rec_len - length + 1, (n,), generator=gen, device="cuda") for _ in range(a.iters + 1)]
    it = {"k": 0}

    def next_frames():
        it["k"] = (it["k"] + 1) % len(sets)
        return sets[it["k"]]

    # (a) the recordings bound once; a new excerpt set is one bind of n offsets
    made = [graph(pkg, eng.backend, rec_len, length, True) for _ in range(n)]
    b = pkg.Batch([m[0] for m in made])
    _, s, lp, g = made[0]
    b.bind_sources(s, recs)
    b.bind_params([lp.frequency, g.gain], params)
    zeros = torch.zeros(n, dtype=torch.float64, device="cuda")

    def run_a():
        b.bind_schedules(s, zeros, offsets=next_frames().double() / SR)
        b.run()
        t = time.perf_counter()
        b.sync()
        return t
    res["a_bound_host_ms"], res["a_bound_total_ms"] = timed(run_a, a.iters)

    def run_only(bb):
        def f():
            bb.run()
            t = time.perf_counter()
            bb.sync()
            return t
        return f
    res["a_run_sync_ms"] = timed(run_only(b), a.iters)[1]
    frames = sets[0]
    b.bind_schedules(s, zeros, offsets=frames.double() / SR)
    b.run()
    b.sync()
    got_a = b.fetch()
    res["a_batch_source_bytes"] = int(n * rec_len * 4)
    b.destroy()
    del b, made
    gc.collect()

    # (b) excerpts gathered in torch and bound as clips
    made = [graph(pkg, eng.backend, length, length, False) for _ in range(n)]
    bg = pkg.Batch([m[0] for m in made])
    _, sg, lpg, gg = made[0]
    bg.bind_params([lpg.frequency, gg.gain], params)
    ar = torch.arange(length, device="cuda")

    def gather(fr):
        return torch.gather(recs, 2, (fr[:, None] + ar[None, :])[:, None, :])

    def run_b():
        bg.bind_sources(sg, gather(next_frames()))
        bg.run()
        t = time.perf_counter()
        bg.sync()
        return t
    res["b_gather_host_ms"], res["b_gather_total_ms"] = timed(run_b, a.iters)
    res["b_run_sync_ms"] = timed(run_only(bg), a.iters)[1]
    bg.bind_sources(sg, gather(frames))
    bg.run()
    bg.sync()
    got_b = bg.fetch()
    res["max_abs_diff_a_vs_b"] = float(np.abs(got_a - got_b).max())
    res["bit_equal_graphs_a_vs_b"] = int(sum(np.array_equal(got_a[i], got_b[i]) for i in range(n)))
    bg.destroy()
    del bg, made, got_b
    gc.collect()

    # (c) rebuild: host offsets, prepare, the recordings bound again
    def run_c():
        fr = next_frames().cpu().numpy()
        ms = [graph(pkg, eng.backend, rec_len, length, False, float(fr[i]) / SR) for i in range(n)]
        bc = pkg.Batch([m[0] for m in ms])
        bc.bind_sources(ms[0][1], recs)
        bc.bind_params([ms[0][2].frequency, ms[0][3].gain], params)
        bc.run()
        t = time.perf_counter()
        bc.sync()
        bc.destroy()
        return t
    res["c_rebuild_host_ms"], res["c_rebuild_total_ms"] = timed(run_c, max(1, a.iters - 2))
    res["card_after"] = card()
    eng.close()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
