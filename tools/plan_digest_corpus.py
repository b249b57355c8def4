#!/usr/bin/env python
"""Regression harness for refactorings of the planner (CPU, no GPU): prints, for a corpus of graphs (BASELINE configs, the 24 reference
scenarios, fuzz graphs and fuzz batches), the WAE_PLAN_DIGEST hash of every instance record the sizing pass builds.  Run it with the
library before and after a change and diff the outputs:
    python tools/plan_digest_corpus.py /path/to/old/libwae_b200.so 2> before.txt ; python tools/plan_digest_corpus.py 2> after.txt ; diff before.txt after.txt"""
import sys, os, subprocess
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests")); sys.path.insert(0, ROOT)
os.environ["WAE_PLAN_DIGEST"] = "1"
import conftest
pkg = conftest.load_package()
if len(sys.argv) > 1: pkg.LIB_PATH = sys.argv[1]
import graphs as G, benchmark_scenarios as BS, test_gpu_fuzz as F
import numpy as np
be = pkg.context.Backend(pkg.api(), None)
def P(name, ctxs):
    sys.stderr.write("== %s\n" % name); sys.stderr.flush()
    try:
        p = pkg.context.plan_batch(ctxs)
        sys.stderr.write("   %s\n" % {k: p[k] for k in ("groups", "segments", "stages", "chunk_frames", "arena_floats_per_frame", "source_floats")})
    except pkg.WaeError as e:
        sys.stderr.write("   refused: %s\n" % e)
    sys.stderr.flush()
ir = G.synthetic_ir(20000, 2, decay=0.6)
P("c1", [G.c1_osc_biquad(pkg, be, 48000)])
P("c2", [G.c2_buffer_biquad_gain(pkg, be, g, 12800) for g in range(70)])
P("c2 small", [G.c2_buffer_biquad_gain(pkg, be, g, 12800 + 0) for g in range(5)])
P("c3", [G.c3_many_voices(pkg, be, 300, 48000)])
P("c4", [G.c4_convolver(pkg, be, g, 8192 * 3, ir) for g in range(4)])
P("ns", [G.north_star_voices_convolver(pkg, be, 100, 48000, ir, seed=g) for g in range(3)])
for name, fn in BS.SCENARIOS:
    P(name, [fn(pkg, be, 4.0) for _ in range(2)])
for seed in range(4000, 4400):
    P("fuzz %d" % seed, [F.random_graph(pkg, be, seed)])
for seed in range(5000, 5200, 4):
    P("fuzz batch %d" % seed, [F.random_graph(pkg, be, seed + i) for i in range(4)])
