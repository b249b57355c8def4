"""AudioParam value curves bound from device memory, on the host (no GPU): the declaration rules of wae_param_set_device_value_curve,
the one-shot refusals, the oracle's refusal, the wae_value_curve_binding layout of include/wae.h, and plans of graphs with declared
curves.  No planning decision reads the values of an automated param, so a declared curve plans exactly as its host twin (the same
setValueCurveAtTime given host values): the same plan_batch dicts and the same WAE_PLAN_DIGEST lines, whatever values the twin holds,
through every kind of param the declaration serves.  (tests/test_gpu_device_value_curves.py renders the same graphs.)"""
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

# (case name) -> the value range its curves are drawn from
RANGES = {
    "gain": (0.0, 1.0), "biquad_frequency": (200.0, 4000.0), "osc_frequency": (110.0, 880.0), "osc_detune": (-1200.0, 1200.0),
    "delay_time": (0.0005, 0.02), "delay_cycle": (0.003, 0.02), "constant_offset": (-1.0, 1.0), "stereo_pan": (-1.0, 1.0),
    "panner_x": (-5.0, 5.0), "panner_hrtf_x": (-5.0, 5.0), "buffer_rate": (0.5, 2.0), "compressor_threshold": (-50.0, -5.0),
    "earlier_set": (110.0, 880.0), "earlier_curve": (110.0, 880.0), "audio_rate_input": (0.0, 1.0), "suspend": (110.0, 880.0),
}
CASES = list(RANGES)
PLANNED = [c for c in CASES if c != "panner_hrtf_x"]  # (an HRTF panner is planned by an engine with a sphere: GPU test)


@pytest.fixture
def host(pkg):
    if not os.path.exists(LIB):
        pytest.skip("libwae_b200.so is not built (python -c 'import __graft_entry__ as g; g.build()')")
    return pkg.context.Backend(pkg.api(), None)


def status_and_text(pkg, fn):
    with pytest.raises(pkg._binding.WaeError) as e:
        fn()
    return e.value.status, e.value.message


def curve_values(case, seed, length):
    """`length` values in the case's range"""
    lo, hi = RANGES[case]
    return np.random.default_rng(seed).uniform(lo, hi, length).astype(np.float32)


def noise(seed, frames, amp=0.5):
    return np.random.default_rng(seed).uniform(-amp, amp, (1, frames)).astype(np.float32)


def build(pkg, be, case, values, length=2, start=0.0, duration=None, frames=8192, suspends=(3072,), g=0):
    """One graph of `case` whose curve param gets a setValueCurveAtTime of `length` points at [start, start + duration) (duration
    default: the render's): `values` None declares it bound from device memory, else the host twin with these values.
    Returns (context, the curve's AudioParam)."""
    c = pkg.OfflineAudioContext(2, frames, SR, be)
    duration = frames / SR if duration is None else duration
    dest = c.destination()
    osc = c.create_oscillator(type_=pkg.context.SAWTOOTH, frequency=220.0 + 10 * g)
    src = osc
    if case in ("gain", "audio_rate_input"):
        node = c.create_gain(0.5)
        prm = node.gain
    elif case == "biquad_frequency":
        node = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=1000.0, q=2.0)
        prm = node.frequency
    elif case in ("osc_frequency", "earlier_set", "earlier_curve", "suspend"):
        node = c.create_gain(0.5)
        prm = osc.frequency
    elif case == "osc_detune":
        node = c.create_gain(0.5)
        prm = osc.detune
    elif case == "delay_time":
        node = c.create_delay(max_delay_time=0.05, delay_time=0.001)
        prm = node.delay_time
    elif case == "delay_cycle":  # delay -> feedback gain -> delay: the delay time is read by the cycle's reader
        node = c.create_delay(max_delay_time=0.05, delay_time=0.01)
        fb = c.create_gain(0.5)
        node.connect(fb)
        fb.connect(node)
        prm = node.delay_time
    elif case == "constant_offset":
        src = c.create_constant_source(0.25)
        node = c.create_gain(1.0)
        prm = src.offset
    elif case == "stereo_pan":
        node = c.create_stereo_panner(0.0)
        prm = node.pan
    elif case in ("panner_x", "panner_hrtf_x"):
        model = pkg.context.HRTF if case == "panner_hrtf_x" else pkg.context.EQUALPOWER
        node = c.create_panner(panning_model=model, position=(1.0, 0.0, -1.0))
        prm = node.position_x
    elif case == "buffer_rate":
        src = c.create_buffer_source(pkg.AudioBuffer(list(noise(7 + g, frames)), SR))
        node = c.create_gain(1.0)
        prm = src.playback_rate
    elif case == "compressor_threshold":
        node = c.create_dynamics_compressor()
        prm = node.threshold
    else:
        raise ValueError(case)
    src.connect(node)
    node.connect(dest)
    if case == "earlier_set":  # an earlier event on the same param, before the curve
        prm.set_value_at_time(330.0, 0.0)
        start = max(start, 256 / SR)
    if case == "earlier_curve":  # a host curve before the declared one: the pool holds both, the host one copied in at prepare
        prm.set_value_curve_at_time(np.array([300.0, 500.0, 400.0], np.float32), 0.0, 200 / SR)
        start = max(start, 256 / SR)
    if case == "audio_rate_input":  # a second oscillator into the same param
        lfo = c.create_oscillator(frequency=3.0)
        lfo.connect(prm)
        lfo.start()
    if values is None:
        prm.set_device_value_curve(length, start, duration)
    else:
        prm.set_value_curve_at_time(np.asarray(values, np.float32), start, duration)
    src.start()
    if case == "suspend":
        for fr in suspends:
            c.suspend_sync(fr / SR, lambda ctx: None)
    return c, prm


# ---------------------------------------------------------------------------------------------------------- declaration rules
def one_param(pkg, be):
    c = pkg.OfflineAudioContext(2, 4096, SR, be)
    g = c.create_gain()
    g.connect(c.destination())
    return c, g


def test_short_curve_refused(pkg, host):
    c, g = one_param(pkg, host)
    for n in (0, 1):
        assert status_and_text(pkg, lambda: g.gain.set_device_value_curve(n, 0.0, 1.0)) == (
            2, "InvalidStateError - sequence length should not be less than 2")
    g.gain.set_device_value_curve(2, 0.0, 1.0)  # (the failed calls declared nothing)


@pytest.mark.parametrize("start", [-1.0, float("nan"), float("inf")])
def test_invalid_start_time_refused(pkg, host, start):
    c, g = one_param(pkg, host)
    assert status_and_text(pkg, lambda: g.gain.set_device_value_curve(4, start, 1.0)) == (1, "RangeError - time should be positive")


@pytest.mark.parametrize("duration", [0.0, -1.0, float("nan"), float("inf")])
def test_invalid_duration_refused(pkg, host, duration):
    c, g = one_param(pkg, host)
    assert status_and_text(pkg, lambda: g.gain.set_device_value_curve(4, 0.0, duration)) == (
        1, "RangeError - duration should be strictly positive")


def test_unknown_node_or_param(pkg, host):
    c, g = one_param(pkg, host)
    api = pkg.api()
    assert api.param_set_device_value_curve(c._g, 9999, 0, 4, 0.0, 1.0) == 1
    assert api.param_set_device_value_curve(c._g, g.id, 1, 4, 0.0, 1.0) == 1  # a GainNode has one param
    assert b"unknown param" in api.last_error()
    assert api.param_set_device_value_curve(None, g.id, 0, 4, 0.0, 1.0) == 1


def test_listener_params_refused(pkg, host):
    c = pkg.OfflineAudioContext(2, 4096, SR, host)
    c.listener().position_x.set_value(1.0)  # (the listener exists from here on)
    api = pkg.api()
    assert api.param_set_device_value_curve(c._g, 1, 0, 4, 0.0, 1.0) == 1
    assert b"AudioListener" in api.last_error()
    assert status_and_text(pkg, lambda: c.listener().position_x.set_device_value_curve(4, 0.0, 1.0))[0] == 1


def test_declared_twice(pkg, host):
    c, g = one_param(pkg, host)
    g.gain.set_device_value_curve(4, 0.0, 0.01)
    assert status_and_text(pkg, lambda: g.gain.set_device_value_curve(4, 0.05, 0.01)) == (
        2, "InvalidStateError - the param's value curve is already bound from device memory (wae_param_set_device_value_curve)")


NO_EVENTS = ("InvalidStateError - the param's value curve is bound from device memory (wae_param_set_device_value_curve): it takes no "
             "further events")


@pytest.mark.parametrize("event", ["set_value", "set_value_at_time", "ramp", "curve", "cancel", "cancel_and_hold"])
def test_no_events_after_declaration(pkg, host, event):
    c, g = one_param(pkg, host)
    g.gain.set_device_value_curve(4, 0.0, 0.01)
    push = {"set_value": lambda: g.gain.set_value(0.5), "set_value_at_time": lambda: g.gain.set_value_at_time(0.5, 0.5),
            "ramp": lambda: g.gain.linear_ramp_to_value_at_time(0.5, 0.5),
            "curve": lambda: g.gain.set_value_curve_at_time(np.ones(3, np.float32), 0.5, 0.01),
            "cancel": lambda: g.gain.cancel_scheduled_values(0.0), "cancel_and_hold": lambda: g.gain.cancel_and_hold_at_time(0.0)}
    assert status_and_text(pkg, push[event]) == (2, NO_EVENTS)


def test_no_events_after_declaration_from_a_suspend_callback(pkg, host):
    c, g = one_param(pkg, host)
    g.gain.set_device_value_curve(4, 0.0, 0.01)
    c.suspend_sync(1024 / SR, lambda ctx: g.gain.set_value_at_time(0.5, 0.05))
    assert status_and_text(pkg, lambda: pkg.plan_batch([c])) == (2, NO_EVENTS)


def test_declaration_after_suspend_point(pkg, host):
    c, g = one_param(pkg, host)
    c.suspend_sync(1024 / SR, lambda ctx: g.gain.set_device_value_curve(4, 0.05, 0.01))
    assert status_and_text(pkg, lambda: pkg.plan_batch([c])) == (
        2, "InvalidStateError - a value curve is bound from device memory before the first suspend point")


def test_device_value_then_curve(pkg, host):
    c, g = one_param(pkg, host)
    g.gain.set_device_value(0.0, 1.0)
    assert status_and_text(pkg, lambda: g.gain.set_device_value_curve(4, 0.0, 0.01)) == (
        2, "InvalidStateError - the param's value is bound from device memory (wae_param_set_device_value)")


def test_curve_then_device_value(pkg, host):
    c, g = one_param(pkg, host)
    g.gain.set_device_value_curve(4, 0.0, 0.01)
    assert status_and_text(pkg, lambda: g.gain.set_device_value(0.0, 1.0)) == (2, "InvalidStateError - the param has automation events")


def test_audio_rate_input_allowed(pkg, host):
    c, _ = build(pkg, host, "audio_rate_input", None, length=8)
    pkg.plan_batch([c])


def test_params_set_device_value_refuses_are_declarable(pkg, host):
    """wae_param_set_device_value still refuses these params (test_param_binding_cpu.py pins that); a curve declaration takes them"""
    for case in ("osc_frequency", "osc_detune", "delay_time", "constant_offset", "panner_x"):
        c, prm = build(pkg, host, case, None, length=8)
        pkg.plan_batch([c])


def test_overlap_is_the_hosts_error(pkg, host):
    """folding is the host's: a declared curve over an earlier event answers what the host twin answers, at plan time"""
    def make(values):
        c, g = one_param(pkg, host)
        g.gain.set_value_at_time(0.5, 0.02)
        if values is None:
            g.gain.set_device_value_curve(4, 0.01, 0.05)
        else:
            g.gain.set_value_curve_at_time(values, 0.01, 0.05)
        return c
    declared = status_and_text(pkg, lambda: pkg.plan_batch([make(None)]))
    assert declared == status_and_text(pkg, lambda: pkg.plan_batch([make(np.ones(4, np.float32))]))
    assert declared[0] == 3 and "SetValueCurveAtTime" in declared[1]


def test_oracle_refuses(pkg, oracle):
    c = pkg.OfflineAudioContext(2, 1024, SR, oracle)
    with pytest.raises(pkg._binding.WaeError) as e:
        c.create_gain().gain.set_device_value_curve(4, 0.0, 0.01)
    assert e.value.status == 3


def test_oneshot_refusals(pkg, host):
    api = pkg.api()
    cs = [build(pkg, host, "osc_frequency", None, length=8, frames=4096, g=g)[0] for g in range(2)]
    arr = (ctypes.c_void_p * 2)(*[c._g for c in cs])
    out = np.zeros((2, 2, 4096), np.float32)
    assert api.render_batch(None, arr, 2, out.ctypes.data_as(ctypes.c_void_p), 0) == 2
    assert b"wae_batch_bind_value_curves" in api.last_error()
    outs = (pkg._binding.c_float_p * 2)(*[pkg._binding.fptr(out[i]) for i in range(2)])
    assert api.render_many(None, arr, 2, outs) == 2
    assert b"wae_batch_bind_value_curves" in api.last_error()
    assert api.batch_bind_value_curves(None, None, 0, None) == 1


def test_value_curve_binding_layout(pkg, tmp_path):
    B = pkg._binding
    assert "wae_param_set_device_value_curve" in B.WAE_SYMBOLS and "wae_batch_bind_value_curves" in B.WAE_SYMBOLS
    src = tmp_path / "binding.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "wae.h"\nint main(void) {\n'
                   '  printf("%zu %zu %zu %zu %zu\\n", sizeof(wae_value_curve_binding), offsetof(wae_value_curve_binding, graph_index),\n'
                   '         offsetof(wae_value_curve_binding, node), offsetof(wae_value_curve_binding, param_index),\n'
                   '         offsetof(wae_value_curve_binding, values));\n'
                   "  return 0;\n}\n")
    exe = tmp_path / "binding"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = tuple(map(int, subprocess.check_output([str(exe)], text=True).split()))
    S = B.ValueCurveBinding
    assert got == (ctypes.sizeof(S), S.graph_index.offset, S.node.offset, S.param_index.offset, S.values.offset)
    if not os.path.exists(LIB):
        pytest.skip("libwae_b200.so is not built")
    lib = ctypes.CDLL(LIB)
    assert hasattr(lib, "wae_param_set_device_value_curve") and hasattr(lib, "wae_batch_bind_value_curves")


# ---------------------------------------------------------------------------------------------------------- plans
# (length, start, duration in frames): a curve over the whole render, one starting mid-quantum and ending before the end, and a long one
# starting in a later chunk and running past the end
SHAPES = [(2, 0, 8192), (3, 200, 3000), (1000, 5000, 6000)]


def case_graphs(pkg, be, case, shape, mode, graphs=2):
    """`graphs` graphs of `case`: mode "declared", or host twins "a" / "b" holding two different value sets"""
    length, start, dur = shape
    out = []
    for g in range(graphs):
        values = None if mode == "declared" else curve_values(case, 100 * g + (1 if mode == "a" else 2), length)
        out.append(build(pkg, be, case, values, length, start / SR, dur / SR, g=g)[0])
    return out


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("case", PLANNED)
def test_plan_equals_host_twins(pkg, host, case, shape):
    declared = pkg.plan_batch(case_graphs(pkg, host, case, shape, "declared"))
    assert declared == pkg.plan_batch(case_graphs(pkg, host, case, shape, "a"))
    assert declared == pkg.plan_batch(case_graphs(pkg, host, case, shape, "b"))
    if case == "suspend":
        assert declared["segments"] == 2


def test_hrtf_panner_refusal_equals_host_twin(pkg, host):
    """without an engine there is no HRIR sphere: the declared panner stops where its host twin stops"""
    d = status_and_text(pkg, lambda: pkg.plan_batch(case_graphs(pkg, host, "panner_hrtf_x", SHAPES[0], "declared")))
    assert d == status_and_text(pkg, lambda: pkg.plan_batch(case_graphs(pkg, host, "panner_hrtf_x", SHAPES[0], "a")))


def test_pruned_and_unconnected_declarations_are_planned(pkg, host):
    c, _ = build(pkg, host, "gain", None, length=8)
    idle = c.create_oscillator()
    idle.frequency.set_device_value_curve(8, 0.0, 0.1)  # never started, never connected
    pkg.plan_batch([c])


DIGEST_SCRIPT = textwrap.dedent("""
    import sys
    sys.path.insert(0, {tests!r}); sys.path.insert(0, {root!r})
    from conftest import load_package
    import test_device_value_curves_cpu as T
    pkg = load_package()
    be = pkg.context.Backend(pkg.api(), None)
    for case in T.PLANNED:
        for shape in T.SHAPES:
            pkg.plan_batch(T.case_graphs(pkg, be, case, shape, sys.argv[1]))
""")


def test_plan_digest_equals_host_twins(pkg, host):
    script = DIGEST_SCRIPT.format(tests=os.path.join(ROOT, "tests"), root=ROOT)
    env = dict(os.environ, WAE_PLAN_DIGEST="1")
    out = {}
    for mode in ("declared", "a", "b"):
        r = subprocess.run([sys.executable, "-c", script, mode], env=env, capture_output=True, text=True, check=True)
        out[mode] = [line for line in r.stderr.splitlines() if "[wae plan digest]" in line]
    assert len(out["declared"]) >= len(PLANNED) * len(SHAPES)
    assert out["declared"] == out["a"] == out["b"]
