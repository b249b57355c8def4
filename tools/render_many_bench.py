#!/usr/bin/env python
"""Contexts of different lengths, three ways (GPU): N C2-shaped graphs (buffer source -> biquad -> gain -> destination, stereo, 48 kHz)
whose lengths are drawn seeded from U[1 s, 10 s]:
  1. one wae_render_many call;
  2. one call per graph;
  3. every graph padded to the longest length, one wae_render_batch call (render_batch_oneshot).
Prints one JSON line: the call times (host clock around each synchronous call, after one untimed call of each way), rendered / needed
quanta of (1), whether (1) equals (3) truncated to each graph's length within 1e-5, and the card's name and power limit read in the same
run.  Writes nothing."""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--graphs", type=int, default=1000)
    ap.add_argument("--seed", type=int, default=11)
    ap.add_argument("--sr", type=float, default=48000.0)
    a = ap.parse_args()
    import conftest
    import graphs as G
    pkg = conftest.load_package()
    eng = pkg.Engine(0)
    be = eng.backend
    sr = a.sr
    lengths = [int(x) for x in np.random.default_rng(a.seed).uniform(1.0, 10.0, a.graphs) * sr]
    longest = max(lengths)
    pcms = [G.c2_source(g, n) for g, n in enumerate(lengths)]

    def own():
        return [G.c2_buffer_biquad_gain(pkg, be, g, n, sr, pcm=pcms[g]) for g, n in enumerate(lengths)]

    def padded():  # the same graphs in contexts of the longest length (each source ends where its graph would)
        return [G.c2_buffer_biquad_gain(pkg, be, g, longest, sr, pcm=pcms[g]) for g in range(len(lengths))]

    def timed(fn):
        t0 = time.perf_counter()
        r = fn()
        return r, (time.perf_counter() - t0) * 1e3

    ctxs = own()
    plan = pkg.context.plan_many(ctxs)
    outs = [np.empty((2, n), np.float32) for n in lengths]
    pkg.render_many(ctxs, outs)  # warm-up: modules, the engine's device-memory cache, staging slots
    _, ms_many = timed(lambda: pkg.render_many(ctxs, outs))
    pkg.render_many(ctxs[:1], outs[:1])
    _, ms_each = timed(lambda: [pkg.render_many([c], [o]) for c, o in zip(ctxs, outs)])
    pctxs = padded()
    pout = np.empty((len(lengths), 2, longest), np.float32)
    pkg.render_batch_oneshot(pctxs, pout)
    _, ms_padded = timed(lambda: pkg.render_batch_oneshot(pctxs, pout))
    err = max(float(np.abs(o.astype(np.float64) - pout[g, :, :lengths[g]]).max()) for g, o in enumerate(outs))
    print(json.dumps({
        "graphs": len(lengths), "sample_rate": sr, "seconds_min": min(lengths) / sr, "seconds_max": longest / sr,
        "ms_render_many": round(ms_many, 1), "ms_one_call_per_graph": round(ms_each, 1), "ms_padded_oneshot": round(ms_padded, 1),
        "groups": plan["groups"], "rendered_quanta": plan["rendered_quanta"], "needed_quanta": plan["needed_quanta"],
        "padded_quanta": len(lengths) * ((longest + 127) // 128),
        "max_abs_diff_vs_padded": err, "matches_padded_1e-5": err <= 1e-5, "card": card()}))
    eng.close()


if __name__ == "__main__":
    main()
