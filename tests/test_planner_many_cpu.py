"""Planner (CPU, wae_batch_plan_many / wae_batch_plan_quanta): batches of OfflineAudioContexts that differ in channel count, length and
sample rate.  Graphs are grouped by sample rate, suspend frames and length; the shortest graph of a group is at least 3/4 of the longest.
A batch of one shape plans exactly as wae_batch_plan plans it."""
import ctypes
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

import graphs as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ["wae_render_many", "wae_batch_prepare_many", "wae_batch_graph_output", "wae_batch_fetch_graph", "wae_batch_plan_many",
               "wae_batch_plan_quanta"]


@pytest.fixture
def be(pkg):
    so = os.path.join(ROOT, "web-audio-api-rs_b200", "libwae_b200.so")
    if not os.path.exists(so):
        pytest.skip("libwae_b200.so is not built (python -c 'import __graft_entry__ as g; g.build()')")
    return pkg.context.Backend(pkg.api(), None)


def padded(length):
    return (length + 127) // 128 * 128


def c2(pkg, be, seed, channels, length, sr, suspend_frames=()):
    """buffer source -> biquad -> gain -> destination with `channels` destination channels; a gain change at each suspend frame"""
    _, f0, q, gain = G.c2_params(seed)
    pcm = np.random.default_rng(seed).uniform(-1, 1, (2, max(length, 1))).astype(np.float32)
    c = pkg.OfflineAudioContext(channels, length, sr, be)
    src = c.create_buffer_source(pkg.AudioBuffer([pcm[0], pcm[1]], sr))
    bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=min(f0, sr / 2 - 1), q=q)
    gn = c.create_gain(gain)
    src.connect(bq)
    bq.connect(gn)
    gn.connect(c.destination())
    src.start()
    for k, f in enumerate(suspend_frames):
        # (a time half a frame before the quantum boundary: it quantises up to exactly `f`)
        c.suspend_sync((f - 0.5) / sr, lambda ctx, k=k: gn.gain.set_value(0.2 + 0.1 * k))
    return c


LENGTHS = [1, 127, 128, 129, 3000, 3 * 8192 + 77, 5 * 8192 - 5, 4000, 20000, 24000, 31000]


def mixed_batch(pkg, be):
    ctxs, seed = [], 0
    for sr in (44100.0, 48000.0):
        for ch in (1, 2, 6):
            for length in LENGTHS:
                ctxs.append(c2(pkg, be, seed, ch, length, sr))
                seed += 1
    # per-graph suspend points: two graphs share theirs, a third has its own
    ctxs.append(c2(pkg, be, 900, 2, 40000, 48000.0, (1280, 8192)))
    ctxs.append(c2(pkg, be, 901, 1, 36000, 48000.0, (1280, 8192)))
    ctxs.append(c2(pkg, be, 902, 2, 30000, 44100.0, (2560,)))
    return ctxs


def test_mixed_batch_is_planned_within_the_padding_bound(pkg, be):
    ctxs = mixed_batch(pkg, be)
    p = pkg.context.plan_many(ctxs)
    assert p["groups"] >= 1 and p["stages"] > 0
    group_of = p["group_of"]
    assert len(group_of) == len(ctxs) and p["groups"] == len(set(group_of))
    cut_of = [()] * (len(ctxs) - 3) + [(1280, 8192), (1280, 8192), (2560,)]
    members = {}
    for i, c in enumerate(ctxs):
        members.setdefault(group_of[i], []).append(i)
    rendered = needed = 0
    for g, idx in members.items():
        lq = [padded(ctxs[i].length()) for i in idx]
        assert 4 * min(lq) >= 3 * max(lq), (g, lq)                       # the documented bound
        assert len({ctxs[i].sample_rate() for i in idx}) == 1               # one rate per group
        assert len({cut_of[i] for i in idx}) == 1                            # one set of suspend frames
        rendered += max(lq) // 128 * len(idx)
        needed += sum(x // 128 for x in lq)
    assert p["rendered_quanta"] == rendered
    assert p["needed_quanta"] == needed == sum(-(-c.length() // 128) for c in ctxs)
    # the suspend points cut render segments: one segment per group without them, 3 and 2 in the two groups with them
    assert p["segments"] == p["groups"] + 2 + 1


def test_grouping_of_lengths_without_suspend_points(pkg, be):
    """the whole grouping computed here: sorted longest first, cut where the 3/4 bound would break"""
    rng = np.random.default_rng(3)
    lengths = [int(x) for x in rng.integers(1, 60000, 40)]
    ctxs = [c2(pkg, be, i, 2, n, 48000.0) for i, n in enumerate(lengths)]
    p = pkg.context.plan_many(ctxs)
    order = sorted(range(len(lengths)), key=lambda i: (-padded(lengths[i]), i))
    groups, cur = [], [order[0]]
    for i in order[1:]:
        if 4 * padded(lengths[i]) < 3 * padded(lengths[cur[0]]):
            groups.append(cur)
            cur = [i]
        else:
            cur.append(i)
    groups.append(cur)
    want_group = {}
    for k, grp in enumerate(groups):
        for i in grp:
            want_group[i] = k
    assert p["group_of"] == [want_group[i] for i in range(len(lengths))]
    assert p["rendered_quanta"] == sum(padded(lengths[g[0]]) // 128 * len(g) for g in groups)
    assert p["needed_quanta"] == sum(padded(n) // 128 for n in lengths)


def plan_digests(code):
    env = dict(os.environ, WAE_PLAN_DIGEST="1")
    r = subprocess.run([sys.executable, "-s", "-c", code], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr
    return [line for line in r.stderr.splitlines() if line.startswith("[wae plan digest]")]


UNIFORM = """
import sys, os
sys.path.insert(0, "tests"); sys.path.insert(0, ".")
import conftest, graphs as G
pkg = conftest.load_package()
be = pkg.context.Backend(pkg.api(), None)
ir = G.synthetic_ir(20000, 2, decay=0.6)
batches = [
    [G.c2_buffer_biquad_gain(pkg, be, g, 12800) for g in range(70)],
    [G.c4_convolver(pkg, be, g, 8192 * 3, ir) for g in range(4)],
    [G.north_star_voices_convolver(pkg, be, 40, 48000, ir, seed=g) for g in range(3)],
]
for ctxs in batches:
    p = pkg.context.%s(ctxs)
    print({k: p[k] for k in ("groups", "segments", "stages", "chunk_frames", "chunks", "arena_floats_per_frame", "source_floats", "kinds")})
"""


def test_uniform_batch_plans_as_before(pkg, be):
    ir = G.synthetic_ir(20000, 2, decay=0.6)
    batches = [
        [G.c2_buffer_biquad_gain(pkg, be, g, 12800) for g in range(70)],
        [G.c4_convolver(pkg, be, g, 8192 * 3, ir) for g in range(4)],
        [c2(pkg, be, g, 2, 30000, 48000.0, (1280,) if g % 2 else ()) for g in range(6)],
    ]
    for ctxs in batches:
        a, b = pkg.context.plan_batch(ctxs), pkg.context.plan_many(ctxs)
        for k in a:
            assert a[k] == b[k], k
        assert b["rendered_quanta"] == b["needed_quanta"]
    # same instance records, group by group (the planner's digest of every stage build)
    before, after = plan_digests(UNIFORM % "plan_batch"), plan_digests(UNIFORM % "plan_many")
    assert before and before == after


def test_refusal_refuses_the_whole_call(pkg, be):
    """an HRTF panner without an HRIR sphere (the host-only planner has none): the same status and text as wae_batch_plan"""
    bad = pkg.OfflineAudioContext(2, 5000, 48000.0, be)
    o = bad.create_oscillator()
    pn = bad.create_panner(panning_model=pkg.context.HRTF)
    o.connect(pn)
    pn.connect(bad.destination())
    o.start()
    with pytest.raises(pkg.WaeError) as one:
        pkg.context.plan_batch([bad])
    ctxs = [c2(pkg, be, 1, 1, 3000, 44100.0), bad, c2(pkg, be, 2, 2, 12000, 48000.0)]
    with pytest.raises(pkg.WaeError) as many:
        pkg.context.plan_many(ctxs)
    assert (many.value.args, str(many.value)) == (one.value.args, str(one.value))


def test_convolver_suspend_rule_holds_per_group(pkg, be):
    """a group with a ConvolverNode still needs its suspend points on the 8192-frame partition grid"""
    ir = G.synthetic_ir(4000, 2)
    def conv(length, frame):
        c = G.c4_convolver(pkg, be, 0, length, ir)
        c.suspend_sync((frame - 0.5) / 48000.0, lambda ctx: None)
        return c
    ok = [conv(40000, 16384), G.c2_buffer_biquad_gain(pkg, be, 1, 5000)]
    assert pkg.context.plan_many(ok)["groups"] == 2
    with pytest.raises(pkg.WaeError) as e:
        pkg.context.plan_many([conv(40000, 1280), G.c2_buffer_biquad_gain(pkg, be, 1, 5000)])
    assert "multiple of the convolver partition" in str(e.value)


def test_new_symbols_declared_exported_and_c99(pkg, be):
    header = open(os.path.join(ROOT, "include", "wae.h")).read()
    lib = ctypes.CDLL(os.path.join(ROOT, "web-audio-api-rs_b200", "libwae_b200.so"))
    for s in NEW_SYMBOLS:
        assert "WAE_API wae_status %s(" % s in header, s
        assert hasattr(lib, s), s
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    src = "#include \"wae.h\"\nint main(void) { wae_status (*f[])() = {%s}; return (int)sizeof f; }\n" % ", ".join(
        "(wae_status (*)())" + s for s in NEW_SYMBOLS)
    r = subprocess.run([cc, "-std=c99", "-pedantic", "-Wall", "-Werror", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), "-x", "c", "-"],
                       input=src, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
