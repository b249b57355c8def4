#!/usr/bin/env python
"""PannerNode positions and the AudioListener's pose bound from device memory versus the other ways to give every run its own source
direction (GPU).  With the card's name and power limit read in the same run, medians over --runs timed runs after --warmup untimed ones,
the variants alternated run by run.
Workload: N graphs of a mono device-input clip (wae_buffer_source_set_device_input) -> PannerNode -> stereo destination, L frames at
48 kHz, once with an HRTF panner (synthetic sphere of tests/graphs.py, 256 taps) and once equal-power.  Every run takes a new source
azimuth, distance and listener forward vector per graph:
  (a) wae_batch_bind_params of source x, y, z and listener forward x, y, z + run + sync (the static lowering: HRTF as a convolver,
      k_panner_eq);
  (b) the source position as three two-point device value curves (wae_param_set_device_value_curve; listener params are not bound as
      curves, so the source is given in the listener's frame, the same relative direction) + run + sync: the moving panner
      (k_hrtf_sel + k_hrtf_fir, k_panner_dyn);
  (c) the host-built graphs with those values: build + prepare + run + sync.
Also the render's per-stage kernel times of (a) and (b) in runs of their own, the bind's kernels (k_derive_spatial, k_spatial_blend,
k_resp_fft) from torch.profiler over one bind, and the largest differences of (a) and (b) from (c).  Prints one JSON line.  Writes nothing."""
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
HRTF, EQ = 1, 0


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # (reported, not fatal)
        return "unknown (%s)" % e


def scene(pkg, be, length, sr, model, route, vals=None):
    """route "bound": source position and listener forward declared; "curve": source position as device value curves; "host": vals =
    (x, y, z, fx, fy, fz) built in.  Returns (context, source node, [bound params])."""
    c = pkg.OfflineAudioContext(2, length, sr, be)
    src = c.create_buffer_source()
    src.set_device_input(1, length, sr)
    pos = tuple(vals[:3]) if vals is not None else (1.0, 0.0, -1.0)
    pn = c.create_panner(panning_model=model, distance_model=1, position=pos)
    src.connect(pn)
    pn.connect(c.destination())
    src.start()
    lis = c.listener()
    params = [pn.position_x, pn.position_y, pn.position_z]
    if route == "bound":
        for p in params:
            p.set_device_value(-100.0, 100.0)
        params += [lis.forward_x, lis.forward_y, lis.forward_z]
        for p in params[3:]:
            p.set_device_value(-1.0, 1.0)
    elif route == "curve":
        for p in params:
            p.set_device_value_curve(2, 0.0, length / sr)
    else:
        lis.forward_x.set_value(vals[3])
        lis.forward_y.set_value(vals[4])
        lis.forward_z.set_value(vals[5])
    return c, src, params


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


def bind_kernels(batch, params, values):
    """device time per kernel of one bind, from torch.profiler (a run of its own)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        batch.bind_params(params, values)
        batch.sync()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        if ev.key.startswith(("k_", "void wae::k_", "wae::k_")):
            t = getattr(ev, "device_time_total", None)
            if t is None:
                t = ev.cuda_time_total
            out[ev.key.split("(")[0].replace("void ", "")] = round(t / 1e3, 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--graphs", type=int, default=1000)
    ap.add_argument("--frames", type=int, default=480000)
    ap.add_argument("--sr", type=float, default=48000.0)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--seed", type=int, default=5)
    a = ap.parse_args()
    import torch
    import conftest
    import graphs as G
    if not torch.cuda.is_available():
        raise SystemExit("spatial_bind_bench: no CUDA device")
    pkg = conftest.load_package()
    eng = pkg.Engine(0)
    be = eng.backend
    be.set_hrir_sphere(G.synthetic_hrir_sphere(int(a.sr), 256))
    n, L, sr = a.graphs, a.frames, a.sr
    rng = np.random.default_rng(a.seed)
    res = {"graphs": n, "frames": L, "channels": 2, "sample_rate": sr, "runs": a.runs, "card": card()}
    total = a.warmup + a.runs
    clip = torch.from_numpy(rng.uniform(-0.5, 0.5, (n, 1, L)).astype(np.float32)).cuda()
    for name, model in (("hrtf", HRTF), ("equal_power", EQ)):
        sets, rel = [], []
        for _ in range(total):
            az, d, fa = rng.uniform(0, 2 * np.pi, n), rng.uniform(0.5, 10.0, n), rng.uniform(-np.pi, np.pi, n)
            pos = np.stack([d * np.sin(az), np.zeros(n), -d * np.cos(az)], 1)
            fwd = np.stack([np.sin(fa), np.zeros(n), -np.cos(fa)], 1)
            sets.append(np.concatenate([pos, fwd], 1).astype(np.float32))
            # the same source in the frame of a listener facing -z (rotated by -fa about y): the value-curve route's positions
            c_, s_ = np.cos(fa), np.sin(fa)
            rel.append(np.stack([c_ * pos[:, 0] + s_ * pos[:, 2], pos[:, 1], -s_ * pos[:, 0] + c_ * pos[:, 2]], 1).astype(np.float32))
        bound_ctx = [scene(pkg, be, L, sr, model, "bound") for _ in range(n)]
        bound = pkg.Batch([c for c, _, _ in bound_ctx])
        curve_ctx = [scene(pkg, be, L, sr, model, "curve") for _ in range(n)]
        curve = pkg.Batch([c for c, _, _ in curve_ctx])
        bp, cp = bound_ctx[0][2], curve_ctx[0][2]
        bound.bind_sources(bound_ctx[0][1], clip)
        curve.bind_sources(curve_ctx[0][1], clip)
        t_a, t_b, t_c = [], [], []
        host = None
        for r in range(total):
            dv = torch.from_numpy(sets[r]).cuda()
            rv = torch.from_numpy(rel[r]).cuda()
            curves = [rv[:, k:k + 1].repeat(1, 2).contiguous() for k in range(3)]

            def run_a():
                bound.bind_params(bp, dv)
                bound.run()
                bound.sync()

            def run_b():
                curve.bind_value_curves(cp, curves)
                curve.run()
                curve.sync()

            def run_c():
                nonlocal host
                if host is not None:
                    host.destroy()
                made = [scene(pkg, be, L, sr, model, "host", [float(x) for x in sets[r][g]]) for g in range(n)]
                host = pkg.Batch([c for c, _, _ in made])
                host.bind_sources(made[0][1], clip)
                host.run()
                host.sync()
            ta, tb, tc = timed(run_a), timed(run_b), timed(run_c)
            if r >= a.warmup:
                t_a.append(ta)
                t_b.append(tb)
                t_c.append(tc)
        res[name + "_a_bind_params_run_sync_ms"] = round(median(t_a), 2)
        res[name + "_b_value_curve_bind_run_sync_ms"] = round(median(t_b), 2)
        res[name + "_c_host_build_prepare_run_sync_ms"] = round(median(t_c), 1)
        out_a, out_b, out_c = bound.output_tensor().cpu(), curve.output_tensor().cpu(), host.output_tensor().cpu()
        res[name + "_max_abs_diff_a_vs_host_built"] = float((out_a - out_c).abs().max().item())
        res[name + "_max_abs_diff_b_vs_host_built"] = float((out_b - out_c).abs().max().item())
        res[name + "_bit_equal_graphs_a_vs_host_built"] = int(sum(bool(torch.equal(out_a[g], out_c[g])) for g in range(n)))
        host.destroy()
        res[name + "_stages_ms_a"] = stage_times(bound)
        res[name + "_stages_ms_b"] = stage_times(curve)
        res[name + "_bind_kernels_ms_a"] = bind_kernels(bound, bp, torch.from_numpy(sets[-1]).cuda())
        bound.destroy()
        curve.destroy()
    eng.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
