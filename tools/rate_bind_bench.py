#!/usr/bin/env python
"""Playback rates bound from device memory versus host-built rates (GPU).  N graphs of device-input clip -> AudioBufferSource -> lowpass
biquad -> gain -> destination, 2 channels x L frames at 48 kHz, the clips bound with wae_batch_bind_sources; the source's playbackRate,
the lowpass frequency and the gain bound from device memory, rates drawn per run from {0.9, 1.0, 1.1}.  With the card's name and power
limit read in the same run, medians over --runs timed runs after --warmup untimed ones, the variants alternated run by run:
  (a) wae_batch_bind_params + run + sync per new rate set (host clock);
  (b) the kernel time of the bound source stage (k_buffer_source_slow<true>) next to k_buffer_source_slow in host-built graphs with
      the same rates (per-stage CUDA events, a run of their own), and bytes moved from the shapes over that time against 3.35 TB/s;
  (c) the whole step next to host-built C2 at rate 1, where the source is fused into k_chain: the cost of the arena round trip;
  (d) the same graphs declared with a rate range that includes 0, which the serial kernel renders;
and the largest difference between the bound renders and the host-built renders of the same rates.  Prints one JSON line.  Writes
nothing."""
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
HBM_TBS = 3.35  # H100 SXM data sheet


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # (reported, not fatal)
        return "unknown (%s)" % e


def graph(pkg, be, length, sr, vals=None, rng=(0.9, 1.1)):
    """vals None: playbackRate, lowpass frequency and gain bound from device memory (playbackRate over `rng`); else (rate, frequency,
    gain) as host-built constants"""
    rate, freq, gain = vals if vals is not None else (1.0, 2000.0, 0.5)
    c = pkg.OfflineAudioContext(2, length, sr, be)
    src = c.create_buffer_source(playback_rate=rate)
    src.set_device_input(2, length, sr)
    bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=freq)
    gn = c.create_gain(gain)
    src.connect(bq)
    bq.connect(gn)
    gn.connect(c.destination())
    src.start()
    params = []
    if vals is None:
        src.playback_rate.set_device_value(*rng)
        bq.frequency.set_device_value()
        gn.gain.set_device_value(0.05, 2.0)
        params = [src.playback_rate, bq.frequency, gn.gain]
    return c, src, params


def median(xs):
    return float(np.median(np.asarray(xs, np.float64)))


def stage_ms(batch, name):
    batch.set_timing(True)
    batch.run()
    batch.sync()
    ms = n = 0
    for k, t, inst in batch.stage_times():
        if k == name:
            ms += t
            n = max(n, inst)
    batch.set_timing(False)
    return ms, n


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
        raise SystemExit("rate_bind_bench: no CUDA device")
    pkg = conftest.load_package()
    eng = pkg.Engine(0)
    be = eng.backend
    n, L, sr = a.graphs, a.frames, a.sr
    gen = torch.Generator(device="cuda").manual_seed(a.seed)
    pcm = torch.rand((n, 2, L), generator=gen, device="cuda") * 2.0 - 1.0
    choices = torch.tensor([0.9, 1.0, 1.1], device="cuda")

    def draw():
        return torch.stack([choices[torch.randint(3, (n,), generator=gen, device="cuda")],
                            torch.exp(torch.rand(n, generator=gen, device="cuda") * (np.log(8000.0) - np.log(200.0)) + np.log(200.0)),
                            torch.rand(n, generator=gen, device="cuda") * 0.8 + 0.1], dim=1)

    def prepared(ctxs):
        b = pkg.Batch([c for c, _, _ in ctxs])
        b.bind_sources(ctxs[0][1], pcm)
        return b, ctxs[0][2]

    bound, bparams = prepared([graph(pkg, be, L, sr) for _ in range(n)])
    serial, sparams = prepared([graph(pkg, be, L, sr, rng=(0.0, 1.1)) for _ in range(n)])
    unit, _ = prepared([graph(pkg, be, L, sr, (1.0, 2000.0, 0.5)) for _ in range(n)])
    res = {"graphs": n, "frames": L, "channels": 2, "sample_rate": sr, "runs": a.runs, "rates": [0.9, 1.0, 1.1]}

    # (a), (c), (d) alternated run by run: a new rate set bound to the time-parallel and the serial batch, and the fused rate-1 batch
    t_bound, t_serial, t_unit = [], [], []
    for r in range(a.warmup + a.runs):
        vals = draw()
        for b, p, acc in ((bound, bparams, t_bound), (serial, sparams, t_serial), (unit, None, t_unit)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            if p is not None:
                b.bind_params(p, vals)
            b.run()
            b.sync()
            if r >= a.warmup:
                acc.append((time.perf_counter() - t0) * 1e3)
    res["a_bind_run_sync_ms"] = round(median(t_bound), 2)
    res["c_c2_rate1_fused_run_sync_ms"] = round(median(t_unit), 2)
    res["d_serial_bind_run_sync_ms"] = round(median(t_serial), 2)

    # (b) kernel times and the renders of the last rate set against host-built graphs with the same values
    v = vals.cpu().numpy()
    host, _ = prepared([graph(pkg, be, L, sr, tuple(float(x) for x in v[i])) for i in range(n)])
    bound.run()
    bound.sync()
    host.run()
    host.sync()
    res["max_abs_diff_bound_vs_host_built"] = float((bound.output_tensor() - host.output_tensor()).abs().max().item())
    torch.cuda.synchronize()
    kb, kh, ks = [], [], []
    for r in range(a.warmup + a.runs):
        for b, name, acc in ((bound, "k_buffer_source_slow(bound)", kb), (host, "k_buffer_source_slow", kh), (serial, "k_buffer_source_serial", ks)):
            ms, inst = stage_ms(b, name)
            if r >= a.warmup:
                acc.append((ms, inst))
    rates = v[:, 0].astype(np.float64)
    played = np.minimum(L * rates, L)  # clip frames each source reads
    def traffic(mask):  # bytes: the clip frames read and the output written, 2 channels of f32
        return float(2 * 4 * (played[mask].sum() + L * mask.sum()))
    slow_mask = rates != 1.0  # the host-built rate-1 sources take the fast track inside k_chain
    for key, acc, mask in (("bound_source", kb, np.ones(n, bool)), ("host_slow_source", kh, slow_mask), ("serial_source", ks, np.ones(n, bool))):
        ms = median([x[0] for x in acc])
        by = traffic(mask)
        res[f"b_{key}_kernel_ms"] = round(ms, 3)
        res[f"b_{key}_instances"] = int(acc[-1][1])
        res[f"b_{key}_gb"] = round(by / 1e9, 3)
        res[f"b_{key}_tb_s"] = round(by / (ms * 1e-3) / 1e12, 3) if ms > 0 else None
        res[f"b_{key}_share_of_hbm"] = round(by / (ms * 1e-3) / (HBM_TBS * 1e12), 3) if ms > 0 else None
    res["card"] = card()
    print(json.dumps(res))
    for b in (bound, serial, unit, host):
        b.destroy()
    eng.close()


if __name__ == "__main__":
    main()
