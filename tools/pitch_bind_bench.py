#!/usr/bin/env python
"""OscillatorNode pitches bound from device memory versus the other ways to give every run its own pitch (GPU).  With the card's name
and power limit read in the same run, medians over --runs timed runs after --warmup untimed ones, the variants of each part alternated
run by run.
Part 1: N graphs of sawtooth oscillator -> lowpass biquad -> gain -> destination, 2 channels x L frames at 48 kHz (the shapes of
tools/value_curve_bind_bench.py), a new (f0, cutoff, gain) per graph and run:
  (a) wae_batch_bind_params of f0, cutoff and gain (f0 declared with wae_param_set_device_value over [55, 880] Hz) + run + sync: the
      fused chain (k_chain);
  (b) f0 as a two-point device value curve (wae_param_set_device_value_curve, both points the pitch) with cutoff and gain bound as in
      (a): bind_value_curves + bind_params + run + sync, the route before pitches could be bound (k_osc_arate -> k_biquad_arate);
  (c) the host-built graphs with those values: build + prepare + run + sync.
Part 2: N sequences of 16 notes (sawtooth -> gain -> destination each, 2 channels x L2 frames), every note's start, stop and pitch new per
run:
  (d) wae_batch_bind_schedules (start and stop windows) + wae_batch_bind_params (the 16 pitches) + run + sync, against
  (e) rebuilding the host-built sequences: build + prepare + run + sync.
Also the per-stage kernel times of (a), (b) and (d) in runs of their own, and the largest differences between the bound renders and the
host-built renders of the same values.  Prints one JSON line.  Writes nothing."""
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
F0 = (55.0, 880.0)
NOTES = 16


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # (reported, not fatal)
        return "unknown (%s)" % e


def chain(pkg, be, length, sr, route, vals=None):
    """route "bound": f0, cutoff and gain declared; "curve": f0 a declared two-point value curve, cutoff and gain declared; "host": vals =
    (f0, cutoff, gain) built in.  Returns (context, [f0 param, cutoff param, gain param])."""
    c = pkg.OfflineAudioContext(2, length, sr, be)
    f0, cut, gain = vals if vals is not None else (220.0, 2000.0, 0.5)
    o = c.create_oscillator(type_=pkg.context.SAWTOOTH, frequency=f0)
    bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=cut)
    gn = c.create_gain(gain)
    o.connect(bq)
    bq.connect(gn)
    gn.connect(c.destination())
    o.start()
    if route == "bound":
        o.frequency.set_device_value(*F0)
    elif route == "curve":
        o.frequency.set_device_value_curve(2, 0.0, length / sr)
    if route in ("bound", "curve"):
        bq.frequency.set_device_value(20.0, 20000.0)
        gn.gain.set_device_value(0.0, 1.0)
    return c, [o.frequency, bq.frequency, gn.gain]


def sequence(pkg, be, length, sr, notes=None):
    """16 notes; notes = None: starts / stops / pitches declared, else [(start, stop, f0)] built in.  Returns (context, oscillators)."""
    c = pkg.OfflineAudioContext(2, length, sr, be)
    oscs = []
    for k in range(NOTES):
        o = c.create_oscillator(type_=pkg.context.SAWTOOTH, frequency=220.0 if notes is None else notes[k][2])
        g = c.create_gain(0.1)
        o.connect(g)
        g.connect(c.destination())
        slot = length / sr / NOTES
        if notes is None:
            o.start_at(k * slot)
            o.set_device_schedule((k * slot, (k + 1) * slot), stop=(k * slot, (k + 1) * slot))
            o.frequency.set_device_value(*F0)
        else:
            o.start_at(notes[k][0])
            o.stop_at(notes[k][1])
        oscs.append(o)
    return c, oscs


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
    return {k: round(v, 3) for k, v in out.items()}


def timed(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--graphs", type=int, default=1000)
    ap.add_argument("--frames", type=int, default=480000)
    ap.add_argument("--seq-frames", type=int, default=384000, help="frames of a 16-note sequence (8 s at 48 kHz: 0.5 s a note)")
    ap.add_argument("--sr", type=float, default=48000.0)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--seed", type=int, default=5)
    a = ap.parse_args()
    import torch
    import conftest
    if not torch.cuda.is_available():
        raise SystemExit("pitch_bind_bench: no CUDA device")
    pkg = conftest.load_package()
    eng = pkg.Engine(0)
    be = eng.backend
    n, L, L2, sr = a.graphs, a.frames, a.seq_frames, a.sr
    rng = np.random.default_rng(a.seed)
    res = {"graphs": n, "frames": L, "seq_frames": L2, "notes": NOTES, "channels": 2, "sample_rate": sr, "runs": a.runs, "card": card()}
    total = a.warmup + a.runs

    # ---- part 1
    sets = []
    for _ in range(total):
        f0 = rng.uniform(110.0, 440.0, n).astype(np.float32)
        sets.append(np.stack([f0, rng.uniform(300.0, 6000.0, n), rng.uniform(0.1, 0.9, n)], 1).astype(np.float32))
    bound_ctx = [chain(pkg, be, L, sr, "bound") for _ in range(n)]
    bound = pkg.Batch([c for c, _ in bound_ctx])
    curve_ctx = [chain(pkg, be, L, sr, "curve") for _ in range(n)]
    curve = pkg.Batch([c for c, _ in curve_ctx])
    bp, cp = bound_ctx[0][1], curve_ctx[0][1]
    t_a, t_b, t_c = [], [], []
    host = None
    for r, vals in enumerate(sets):
        dv = torch.from_numpy(vals).cuda()
        f0_curve = dv[:, :1].repeat(1, 2).contiguous()

        def run_a():
            bound.bind_params(bp, dv)
            bound.run()
            bound.sync()

        def run_b():
            curve.bind_value_curves(cp[0], f0_curve)
            curve.bind_params(cp[1:], dv[:, 1:].contiguous())
            curve.run()
            curve.sync()

        def run_c():
            nonlocal host
            if host is not None:
                host.destroy()
            host = pkg.Batch([chain(pkg, be, L, sr, "host", tuple(float(x) for x in vals[g]))[0] for g in range(n)])
            host.run()
            host.sync()
        ta, tb, tc = timed(run_a), timed(run_b), timed(run_c)
        if r >= a.warmup:
            t_a.append(ta)
            t_b.append(tb)
            t_c.append(tc)
    res["a_bind_params_run_sync_ms"] = round(median(t_a), 2)
    res["b_value_curve_bind_run_sync_ms"] = round(median(t_b), 2)
    res["c_host_build_prepare_run_sync_ms"] = round(median(t_c), 1)
    out_a, out_b, out_c = bound.output_tensor().cpu(), curve.output_tensor().cpu(), host.output_tensor().cpu()
    res["max_abs_diff_a_vs_host_built"] = float((out_a - out_c).abs().max().item())
    res["max_abs_diff_b_vs_host_built"] = float((out_b - out_c).abs().max().item())
    host.destroy()
    res["stages_ms_a"] = stage_times(bound)
    res["stages_ms_b"] = stage_times(curve)
    bound.destroy()
    curve.destroy()

    # ---- part 2
    slot = L2 / sr / NOTES
    seqs = []
    for _ in range(total):
        starts = (np.arange(NOTES)[None, :] + rng.uniform(0.0, 0.25, (n, NOTES))) * slot
        stops = starts + rng.uniform(0.3, 0.7, (n, NOTES)) * slot
        pitches = (110.0 * 2.0 ** (rng.integers(0, 36, (n, NOTES)) / 12.0)).astype(np.float32)
        seqs.append((starts, stops, pitches))
    seq_ctx = [sequence(pkg, be, L2, sr) for _ in range(n)]
    seq = pkg.Batch([c for c, _ in seq_ctx])
    nodes = seq_ctx[0][1]
    freqs = [o.frequency for o in nodes]
    t_d, t_e = [], []
    rebuilt = None
    for r, (starts, stops, pitches) in enumerate(seqs):
        st, sp, pv = (torch.from_numpy(starts).cuda(), torch.from_numpy(stops).cuda(), torch.from_numpy(pitches).cuda())

        def run_d():
            seq.bind_schedules(nodes, st, sp)
            seq.bind_params(freqs, pv)
            seq.run()
            seq.sync()

        def run_e():
            nonlocal rebuilt
            if rebuilt is not None:
                rebuilt.destroy()
            rebuilt = pkg.Batch([sequence(pkg, be, L2, sr, [(float(starts[g, k]), float(stops[g, k]), float(pitches[g, k]))
                                                             for k in range(NOTES)])[0] for g in range(n)])
            rebuilt.run()
            rebuilt.sync()
        td, te = timed(run_d), timed(run_e)
        if r >= a.warmup:
            t_d.append(td)
            t_e.append(te)
    res["d_bind_schedules_params_run_sync_ms"] = round(median(t_d), 2)
    res["e_host_build_prepare_run_sync_ms"] = round(median(t_e), 1)
    res["max_abs_diff_d_vs_host_built"] = float((seq.output_tensor().cpu() - rebuilt.output_tensor().cpu()).abs().max().item())
    rebuilt.destroy()
    res["stages_ms_d"] = stage_times(seq)
    seq.destroy()
    print(json.dumps(res))
    eng.close()


if __name__ == "__main__":
    main()
