"""WaveShaperNode curves bound from device memory, on the host (no GPU): the declaration rules of wae_wave_shaper_set_device_curve, the
one-shot refusals, the wae_curve_binding layout of include/wae.h, and plans of graphs with declared curves on every lowering path
wae_batch_plan takes (its default options fuse the shaper into k_chain unless it is over-sampled; the unfused k_shaper is planned by
an engine with fusion off, tests/test_gpu_device_curves.py).  Behind an input that is never silent a declared curve plans exactly as a
host curve of its length that maps 0 to 0: the same stages and the same WAE_PLAN_DIGEST."""
import ctypes
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "web-audio-api-rs_b200", "libwae_b200.so")
SR = 48000.0

INPUTS = ["const", "late", "stop", "switch", "gap"]
NEVER_SILENT = ["const", "switch"]  # (the inputs whose layout never has a silent quantum)


@pytest.fixture
def host(pkg):
    if not os.path.exists(LIB):
        pytest.skip("libwae_b200.so is not built (python -c 'import __graft_entry__ as g; g.build()')")
    return pkg.context.Backend(pkg.api(), None)


def status_and_text(pkg, fn):
    with pytest.raises(pkg._binding.WaeError) as e:
        fn()
    return e.value.status, e.value.message


def make_curve(kind, n):
    """A curve of n points.  kind: "zero" maps 0 to 0 (odd n: centre point 0; even n: the centre pair averages to exactly 0);
    "offset" does not (a tanh lifted by 0.1)."""
    x = np.linspace(-1.0, 1.0, n, dtype=np.float64)
    c = np.tanh(2.5 * x).astype(np.float32)
    if n % 2 == 1:
        c[n // 2] = 0.0
    else:
        c[n // 2] = -c[n // 2 - 1]
    if kind == "offset":
        c = c + np.float32(0.1)
    return c.astype(np.float32)


def noise(seed, ch, frames, amp=0.8):
    return (np.random.default_rng(seed).uniform(-amp, amp, (ch, frames))).astype(np.float32)


def shaper_graph(pkg, be, g, length, n, curve=None, oversample=0, inp="const", ch=2, suspends=(), feedback=False, tail_gain=True):
    """source(s) -> WaveShaperNode -> gain -> destination.  curve: the points given to set_curve, or None: n points declared bound from
    device memory.  inp: "const" (a source covering the render), "late" (starts at frame 3000), "stop" (stops at frame 5000), "switch"
    (a mono tone plus a stereo burst: one and two channels, never silent), "gap" (a burst, silence, another burst).  feedback: the
    shaper sits in a DelayNode feedback cycle.  tail_gain False: the shaper feeds the destination directly.  Returns (context, shaper)."""
    c = pkg.OfflineAudioContext(2, length, SR, be)
    sh = c.create_wave_shaper(oversample=oversample)
    if curve is None:
        sh.set_device_curve(n)
    else:
        sh.set_curve(curve)
    if inp == "switch":
        o = c.create_oscillator(frequency=220.0 + 30 * g)
        o.start()
        o.connect(sh)
        st = c.create_buffer_source(pkg.AudioBuffer(list(noise(g, 2, 4000, 0.5)), SR))
        st.start_at(2000 / SR)
        st.connect(sh)
    elif inp == "gap":
        for k, (f0, frames) in enumerate([(0, 2500), (7000, 3000)]):
            s = c.create_buffer_source(pkg.AudioBuffer(list(noise(10 * g + k, ch, frames)), SR))
            s.start_at(f0 / SR)
            s.connect(sh)
    else:
        s = c.create_buffer_source(pkg.AudioBuffer(list(noise(g, ch, length)), SR))
        s.start_at(3000 / SR if inp == "late" else 0.0)
        if inp == "stop":
            s.stop_at(5000 / SR)
        s.connect(sh)
    if tail_gain:
        gn = c.create_gain(0.8)
        sh.connect(gn)
        gn.connect(c.destination())
    else:
        sh.connect(c.destination())
    if feedback:
        d = c.create_delay(1.0, delay_time=0.005)
        fb = c.create_gain(0.4)
        sh.connect(d)
        d.connect(fb)
        fb.connect(sh)
    for f in suspends:
        c.suspend_sync(f / SR, lambda ctx: None)
    return c, sh


# ---------------------------------------------------------------------------------------------------------- declaration rules
def test_length_zero_refused(pkg, host):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    sh = c.create_wave_shaper()
    assert status_and_text(pkg, lambda: sh.set_device_curve(0)) == (1, "a curve bound from device memory has at least one point")
    sh.set_device_curve(1)  # (the failed call declared nothing; one point is a curve)


def test_declared_twice(pkg, host):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    sh = c.create_wave_shaper()
    sh.set_device_curve(1024)
    assert status_and_text(pkg, lambda: sh.set_device_curve(1024)) == (
        2, "InvalidStateError - the curve is already bound from device memory (wae_wave_shaper_set_device_curve)")


def test_set_curve_after_declaration(pkg, host):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    sh = c.create_wave_shaper()
    sh.set_device_curve(1024)
    assert status_and_text(pkg, lambda: sh.set_curve(make_curve("zero", 1024))) == (
        2, "InvalidStateError - the curve is bound from device memory (wae_wave_shaper_set_device_curve)")


@pytest.mark.parametrize("via_options", [False, True])
def test_declaration_after_set_curve(pkg, host, via_options):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    if via_options:
        sh = c.create_wave_shaper(curve=make_curve("zero", 5))
    else:
        sh = c.create_wave_shaper()
        sh.set_curve(make_curve("zero", 5))
    assert status_and_text(pkg, lambda: sh.set_device_curve(5)) == (
        2, "InvalidStateError - the WaveShaperNode already has a curve (set_curve)")


def test_empty_set_curve_counts(pkg, host):
    """set_curve with no points still gives the node its curve"""
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    sh = c.create_wave_shaper()
    sh.set_curve(np.zeros(0, np.float32))
    assert status_and_text(pkg, lambda: sh.set_device_curve(5))[0] == 2


def test_declaration_after_suspend_point(pkg, host):
    c = pkg.OfflineAudioContext(2, 4096, SR, host)
    sh = c.create_wave_shaper()
    sh.connect(c.destination())
    c.suspend_sync(1024 / SR, lambda ctx: sh.set_device_curve(64))
    st, text = status_and_text(pkg, lambda: pkg.plan_batch([c]))
    assert (st, text) == (2, "InvalidStateError - a curve is bound from device memory before the first suspend point")


def test_oversample_stays_settable(pkg, host):
    c, sh = shaper_graph(pkg, host, 0, 8192, 1024)
    fused = pkg.plan_batch([c])
    sh.set_oversample(pkg.context.OVERSAMPLE_X4)
    assert "k_shaper_os" in pkg.plan_batch([c])["kinds"] and "k_shaper_os" not in fused["kinds"]


def test_not_a_shaper(pkg, host):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    api = pkg.api()
    assert api.wave_shaper_set_device_curve(c._g, c.create_gain().id, 16) == 1
    assert api.wave_shaper_set_device_curve(c._g, 9999, 16) == 1


def test_oracle_refuses(pkg, oracle):
    c = pkg.OfflineAudioContext(2, 1024, SR, oracle)
    with pytest.raises(pkg._binding.WaeError):
        c.create_wave_shaper().set_device_curve(16)


def test_oneshot_refusals(pkg, host):
    api = pkg.api()
    cs = [shaper_graph(pkg, host, g, 4096, 64)[0] for g in range(2)]
    arr = (ctypes.c_void_p * 2)(*[c._g for c in cs])
    out = np.zeros((2, 2, 4096), np.float32)
    assert api.render_batch(None, arr, 2, out.ctypes.data_as(ctypes.c_void_p), 0) == 2
    assert b"wae_batch_bind_curves" in api.last_error()
    outs = (pkg._binding.c_float_p * 2)(*[pkg._binding.fptr(out[i]) for i in range(2)])
    assert api.render_many(None, arr, 2, outs) == 2
    assert b"wae_batch_bind_curves" in api.last_error()
    assert api.batch_bind_curves(None, None, 0, None) == 1


def test_curve_binding_layout(pkg, tmp_path):
    B = pkg._binding
    assert "wae_wave_shaper_set_device_curve" in B.WAE_SYMBOLS and "wae_batch_bind_curves" in B.WAE_SYMBOLS
    src = tmp_path / "binding.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "wae.h"\nint main(void) {\n'
                   '  printf("%zu %zu %zu %zu\\n", sizeof(wae_curve_binding), offsetof(wae_curve_binding, graph_index),\n'
                   '         offsetof(wae_curve_binding, node), offsetof(wae_curve_binding, curve));\n'
                   "  return 0;\n}\n")
    exe = tmp_path / "binding"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = tuple(map(int, subprocess.check_output([str(exe)], text=True).split()))
    S = B.CurveBinding
    assert got == (ctypes.sizeof(S), S.graph_index.offset, S.node.offset, S.curve.offset)
    if not os.path.exists(LIB):
        pytest.skip("libwae_b200.so is not built")
    lib = ctypes.CDLL(LIB)
    assert hasattr(lib, "wae_wave_shaper_set_device_curve") and hasattr(lib, "wae_batch_bind_curves")


# ---------------------------------------------------------------------------------------------------------- plans
# (path, input): oversample 0 = fused into k_chain; X2 / X4 = k_shaper_os
PLAN_CASES = [(os_, inp) for os_ in (0, 1, 2) for inp in INPUTS]


def case_graphs(pkg, be, oversample, inp, declared, n=1024, graphs=3, length=12000, feedback=False):
    return [shaper_graph(pkg, be, g, length, n, None if declared else make_curve("zero", n), oversample=oversample, inp=inp,
                         feedback=feedback)[0] for g in range(graphs)]


@pytest.mark.parametrize("oversample,inp", PLAN_CASES)
def test_declared_shaper_is_planned(pkg, host, oversample, inp):
    p = pkg.plan_batch(case_graphs(pkg, host, oversample, inp, True))
    if oversample:
        assert p["kinds"].get("k_shaper_os", 0) >= 1
    else:
        assert "k_chain" in p["kinds"] and "k_shaper" not in p["kinds"]


@pytest.mark.parametrize("oversample,inp", [c for c in PLAN_CASES if c[1] in NEVER_SILENT])
def test_plan_equals_host_curve_behind_a_never_silent_input(pkg, host, oversample, inp):
    assert pkg.plan_batch(case_graphs(pkg, host, oversample, inp, True)) == pkg.plan_batch(case_graphs(pkg, host, oversample, inp, False))


@pytest.mark.parametrize("inp", ["late", "stop", "gap"])
@pytest.mark.parametrize("oversample", [1, 2])
def test_over_sampled_output_gets_a_track_of_its_own(pkg, host, oversample, inp):
    """behind an input that may be silent the plan covers both answers: the over-sampled shaper's output has a layout track of its own,
    written by a k_meta stage of its own (the bind sets its mode), where a host curve through 0 shares its input's track and a host curve
    that is not through 0 has such a stage too"""
    def plan(declared, kind="zero"):
        return pkg.plan_batch([shaper_graph(pkg, host, g, 12000, 1024, None if declared else make_curve(kind, 1024), oversample=oversample,
                                            inp=inp)[0] for g in range(3)])
    declared, zero, offset = plan(True), plan(False, "zero"), plan(False, "offset")
    assert declared["kinds"]["k_meta"] == zero["kinds"]["k_meta"] + 1 and declared["stages"] == zero["stages"] + 1
    assert declared["kinds"] == offset["kinds"] and declared["stages"] == offset["stages"]


def test_x2_shaper_in_a_feedback_cycle(pkg, host):
    p = pkg.plan_batch(case_graphs(pkg, host, 1, "const", True, feedback=True))
    assert p["has_feedback"] and "k_shaper_os" in p["kinds"]
    assert p == pkg.plan_batch(case_graphs(pkg, host, 1, "const", False, feedback=True))


def test_suspend_points_after_declaration(pkg, host):
    c, _ = shaper_graph(pkg, host, 0, 12000, 1024, suspends=(3072, 8192))
    assert pkg.plan_batch([c])["segments"] == 3


def test_unconnected_declared_shaper_is_planned(pkg, host):
    c, _ = shaper_graph(pkg, host, 0, 4096, 64, curve=make_curve("zero", 64))
    c.create_wave_shaper().set_device_curve(64)
    pkg.plan_batch([c])


DIGEST_SCRIPT = textwrap.dedent("""
    import sys
    sys.path.insert(0, {tests!r}); sys.path.insert(0, {root!r})
    from conftest import load_package
    import test_device_curves_cpu as T
    pkg = load_package()
    be = pkg.context.Backend(pkg.api(), None)
    for os_, inp in T.PLAN_CASES:
        if inp in T.NEVER_SILENT:
            pkg.plan_batch(T.case_graphs(pkg, be, os_, inp, sys.argv[1] == "declared"))
    pkg.plan_batch(T.case_graphs(pkg, be, 1, "const", sys.argv[1] == "declared", feedback=True))
""")


def test_plan_digest_equals_host_curve_behind_a_never_silent_input(pkg, host):
    script = DIGEST_SCRIPT.format(tests=os.path.join(ROOT, "tests"), root=ROOT)
    env = dict(os.environ, WAE_PLAN_DIGEST="1")
    out = {}
    for mode in ("declared", "plain"):
        r = subprocess.run([sys.executable, "-c", script, mode], env=env, capture_output=True, text=True, check=True)
        out[mode] = [line for line in r.stderr.splitlines() if "[wae plan digest]" in line]
    n_cases = sum(1 for _, inp in PLAN_CASES if inp in NEVER_SILENT) + 1
    assert len(out["declared"]) >= n_cases and out["declared"] == out["plain"]
