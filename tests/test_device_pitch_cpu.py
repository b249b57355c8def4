"""OscillatorNode frequency and detune bound from device memory, on the host (no GPU): the declaration rule (every computed frequency the
declared ranges allow lies inside (0, sampleRate / 2)), the planner's re-check when the other param changed after the declaration, the
generic rules of wae_param_set_device_value applied to oscillators, and plans (stages and plan digests) equal to host twins planned at
the same value on the paths an oscillator takes under the default options: the fused chain (materialised, destination-direct and
k_voice_sum), and k_osc_arate when the other param is automated."""
import math
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "web-audio-api-rs_b200", "libwae_b200.so")
SR = 48000.0
NYQ = SR / 2


@pytest.fixture
def host(pkg):
    if not os.path.exists(LIB):
        pytest.skip("libwae_b200.so is not built (python -c 'import __graft_entry__ as g; g.build()')")
    return pkg.context.Backend(pkg.api(), None)


def error_of(fn):
    with pytest.raises(Exception) as e:
        fn()
    return e.value.status, str(e.value)


def status_of(fn):
    return error_of(fn)[0]


def osc_ctx(pkg, host, frequency=440.0, detune=0.0):
    c = pkg.OfflineAudioContext(1, 4096, SR, host)
    osc = c.create_oscillator(frequency=frequency, detune=detune)
    osc.connect(c.destination())
    osc.start()
    return c, osc


# ---- the declaration rule -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lo,hi", [
    (0.0, 1000.0),         # touches 0
    (-100.0, 100.0),       # crosses 0
    (-NYQ, NYQ),           # the whole range
    (100.0, NYQ),          # touches Nyquist
    (100.0, 30000.0),      # crosses it (clamped to maxValue = Nyquist, which it touches)
    (NYQ - 1e-3, NYQ),
])
def test_frequency_ranges_outside(pkg, host, lo, hi):
    c, osc = osc_ctx(pkg, host)
    status, msg = error_of(lambda: osc.frequency.set_device_value(lo, hi))
    assert status == 4, msg
    assert "wae_param_set_device_value_curve" in msg, msg
    osc.frequency.set_device_value(100.0, 1000.0)  # (the failed call declared nothing)


@pytest.mark.parametrize("lo,hi", [(1e-3, 1000.0), (20.0, 20000.0), (100.0, 23999.0), (440.0, 440.0)])
def test_frequency_ranges_inside(pkg, host, lo, hi):
    _, osc = osc_ctx(pkg, host)
    osc.frequency.set_device_value(lo, hi)


def test_top_keeps_a_margin_below_nyquist(pkg, host):
    # one float below Nyquist is inside; Nyquist itself is not (f32 ranges: the largest float below 24000 is 24000 - 2^-9)
    below = float(np.nextafter(np.float32(NYQ), np.float32(0)))
    _, osc = osc_ctx(pkg, host)
    osc.frequency.set_device_value(100.0, below)
    _, osc = osc_ctx(pkg, host)
    assert status_of(lambda: osc.frequency.set_device_value(100.0, NYQ)) == 4


def test_detune_ranges_with_a_constant_frequency(pkg, host):
    top = 1200.0 * math.log2(NYQ / 440.0)  # the detune at which 440 Hz reaches Nyquist
    _, osc = osc_ctx(pkg, host)
    osc.detune.set_device_value(-1200.0, 1200.0)
    _, osc = osc_ctx(pkg, host)
    osc.detune.set_device_value(-153600.0, top - 0.01)  # (the low corner is tiny but > 0)
    _, osc = osc_ctx(pkg, host)
    assert status_of(lambda: osc.detune.set_device_value(0.0, top + 0.01)) == 4
    _, osc = osc_ctx(pkg, host)
    assert status_of(lambda: osc.detune.set_device_value()) == 4  # +-153600 cents
    _, osc = osc_ctx(pkg, host, frequency=0.0)  # a constant frequency of 0: no detune range is inside
    assert status_of(lambda: osc.detune.set_device_value(-100.0, 100.0)) == 4
    _, osc = osc_ctx(pkg, host, frequency=-440.0)
    assert status_of(lambda: osc.detune.set_device_value(-100.0, 100.0)) == 4


def test_detune_ranges_with_a_declared_frequency(pkg, host):
    _, osc = osc_ctx(pkg, host)
    osc.frequency.set_device_value(100.0, 6000.0)
    assert status_of(lambda: osc.detune.set_device_value(0.0, 2400.0)) == 4  # 6000 * 4 = 24000
    osc.detune.set_device_value(-1200.0, 2399.0)
    # declared the other way round: the frequency range is checked against the declared detune range
    _, osc = osc_ctx(pkg, host)
    osc.detune.set_device_value(0.0, 1200.0)
    assert status_of(lambda: osc.frequency.set_device_value(100.0, 12000.0)) == 4
    osc.frequency.set_device_value(100.0, 11999.0)


def test_the_rule_is_not_needed_under_an_automated_other_param(pkg, host):
    # the other param automated or driven at audio rate: k_osc_arate takes the bound value raw, for every value
    _, osc = osc_ctx(pkg, host)
    osc.frequency.set_device_value_curve(2, 0.0, 0.05)
    osc.detune.set_device_value()
    c, osc = osc_ctx(pkg, host)
    osc.detune.linear_ramp_to_value_at_time(100.0, 0.05)
    osc.frequency.set_device_value()
    c, osc = osc_ctx(pkg, host)
    lfo = c.create_oscillator(frequency=3.0)
    lfo.connect(osc.detune)
    lfo.start()
    osc.frequency.set_device_value(-NYQ, NYQ)
    assert pkg.plan_batch([c])["kinds"].get("k_osc_arate") == 1


# ---- the planner's re-check ---------------------------------------------------------------------------------------------------------
def test_planner_rechecks_after_the_other_param_changed(pkg, host):
    cs = []
    for g in range(3):
        c, osc = osc_ctx(pkg, host)
        osc.frequency.set_device_value(100.0, 12000.0)
        if g == 2:
            osc.detune.set_value(1200.0)  # 12000 Hz now reaches 24000 Hz
        cs.append((c, osc))
    pkg.plan_batch([c for c, _ in cs[:2]])
    status, msg = error_of(lambda: pkg.plan_batch([c for c, _ in cs]))
    assert status == 4, msg
    assert "graph 2" in msg and f"OscillatorNode {cs[2][1].id}" in msg, msg
    assert "wae_param_set_device_value_curve" in msg, msg


def test_planner_recheck_names_the_callers_graph_in_a_mixed_batch(pkg, host):
    cs = []
    for g, length in enumerate((4096, 2048, 4096)):
        c = pkg.OfflineAudioContext(1, length, SR, host)
        osc = c.create_oscillator()
        osc.connect(c.destination())
        osc.start()
        osc.detune.set_device_value(-1200.0, 1200.0)
        if g == 1:
            osc.frequency.set_value(20000.0)  # 20000 * 2 > Nyquist
        cs.append(c)
    status, msg = error_of(lambda: pkg.context.plan_many(cs))  # (planned in the order of their shapes: the caller's index is named)
    assert status == 4 and "graph 1," in msg, msg


def test_an_automated_other_param_after_the_declaration_plans_a_rate(pkg, host):
    c, osc = osc_ctx(pkg, host)
    osc.frequency.set_device_value(100.0, 12000.0)
    osc.detune.linear_ramp_to_value_at_time(2400.0, 0.05)  # would leave (0, Nyquist) as a constant: k_osc_arate takes every value
    assert pkg.plan_batch([c])["kinds"].get("k_osc_arate") == 1


# ---- the generic rules ----------------------------------------------------------------------------------------------------------------
def test_generic_rules_apply_to_oscillators(pkg, host):
    _, osc = osc_ctx(pkg, host)
    for lo, hi in ((1000.0, 100.0), (float("nan"), 100.0), (100.0, float("inf"))):
        assert status_of(lambda: osc.frequency.set_device_value(lo, hi)) == 1, (lo, hi)
    assert status_of(lambda: osc.frequency.set_device_value(30000.0, 40000.0)) == 1  # outside [minValue, maxValue]
    osc.frequency.set_device_value(100.0, 1000.0)
    assert status_of(lambda: osc.frequency.set_device_value(100.0, 1000.0)) == 2  # declared twice
    assert status_of(lambda: osc.frequency.set_value(200.0)) == 2  # no events after
    assert status_of(lambda: osc.frequency.linear_ramp_to_value_at_time(200.0, 0.01)) == 2
    assert status_of(lambda: osc.frequency.set_device_value_curve(2, 0.0, 0.01)) == 2
    c, osc = osc_ctx(pkg, host)
    osc.detune.set_value_at_time(10.0, 0.01)
    assert status_of(lambda: osc.detune.set_device_value(-10.0, 10.0)) == 2  # events before
    c, osc = osc_ctx(pkg, host)
    lfo = c.create_oscillator(frequency=2.0)
    lfo.connect(osc.frequency)
    assert status_of(lambda: osc.frequency.set_device_value(100.0, 1000.0)) == 2  # an audio-rate input
    osc.detune.set_device_value(-10.0, 10.0)
    c, osc = osc_ctx(pkg, host)
    osc.detune.set_device_value(-10.0, 10.0)
    lfo = c.create_oscillator(frequency=2.0)
    assert status_of(lambda: lfo.connect(osc.detune)) == 2  # no audio-rate input after


def test_declaration_after_a_suspend_point(pkg, host):
    c, osc = osc_ctx(pkg, host)
    c.suspend_sync(1024 / SR, lambda ctx: osc.frequency.set_device_value(100.0, 1000.0))
    assert status_of(lambda: pkg.plan_batch([c])) == 2


def test_suspend_point_after_the_declaration_plans_every_segment(pkg, host):
    def graph(declare):
        c, osc = osc_ctx(pkg, host, frequency=330.0)
        if declare:
            osc.frequency.set_device_value(100.0, 1000.0)
        c.suspend_sync(1024 / SR, lambda ctx: None)
        c.suspend_sync(2048 / SR, lambda ctx: None)
        return c
    a, b = pkg.plan_batch([graph(True)]), pkg.plan_batch([graph(False)])
    assert a["stages"] == b["stages"] and a["segments"] == b["segments"]


# ---- plans equal to host twins ----------------------------------------------------------------------------------------------------
def custom_table():
    """an 8192-point wavetable (a custom wave plays its own table, not the 2048-point sine)"""
    x = np.arange(8192) / 8192.0
    t = np.sin(2 * np.pi * x) + 0.3 * np.sin(6 * np.pi * x) + 0.1 * np.cos(10 * np.pi * x)
    return (t / np.abs(t).max()).astype(np.float32)


def pitch_graph(pkg, backend, case, declare):
    """The graphs of the digest cases: each declares its pitch over a range whose placeholder (the current value clamped to it) is the
    host twin's value; `declare=False` builds that twin."""
    c = pkg.OfflineAudioContext(2, 4800, SR, backend)
    f, d = case.get("f", 220.0), case.get("d", 0.0)
    voices = case.get("voices", 1)
    dest = c.destination()
    mix = c.create_gain(0.25) if voices > 1 else None
    if mix is not None:
        mix.connect(dest)
    oscs = []
    for v in range(voices):
        if case.get("custom"):
            osc = c.create_oscillator(frequency=f * (v + 1), detune=d, periodic_wave=custom_table())
        else:
            osc = c.create_oscillator(type_=case.get("type", pkg.SAWTOOTH), frequency=f * (v + 1), detune=d)
        oscs.append(osc)
        last = osc
        if case.get("lowpass", True):
            bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=1500.0 + 100 * v)
            last.connect(bq)
            last = bq
        if case.get("gain", True):
            gn = c.create_gain(0.5)
            last.connect(gn)
            last = gn
        last.connect(mix if mix is not None else dest)
        if case.get("two_consumers"):
            osc.connect(dest)
        if case.get("lfo"):
            lfo = c.create_oscillator(frequency=5.0)
            lg = c.create_gain(30.0)
            lfo.connect(lg)
            lg.connect(osc.detune)
            lfo.start()
        osc.start_at(case.get("start", 0.0))
        if declare:
            if case.get("bind", "f") in ("f", "fd"):
                osc.frequency.set_device_value(f * (v + 1), 4000.0)
            if case.get("bind", "f") in ("d", "fd"):
                osc.detune.set_device_value(d, 600.0)
    return c


DIGEST_CASES = {
    "fused_chain": dict(),
    "fused_detune": dict(bind="fd", d=-30.0, type=1),
    "destination_direct": dict(gain=False),
    "late_start": dict(start=0.01234, type=3),
    "materialised_custom_two_consumers": dict(custom=True, two_consumers=True),
    "arate_lfo_on_detune": dict(lfo=True),
    "voices": dict(voices=8, bind="fd", d=7.0, gain=True, lowpass=True),
}


def plan_digests(declare, env=None):
    script = textwrap.dedent(f"""
        import sys
        sys.path.insert(0, {os.path.join(ROOT, 'tests')!r}); sys.path.insert(0, {ROOT!r})
        from conftest import load_package
        import test_device_pitch_cpu as T
        pkg = load_package()
        be = pkg.context.Backend(pkg.api(), None)
        for name, case in T.DIGEST_CASES.items():
            sys.stderr.write("case " + name + "\\n")
            p = pkg.plan_batch([T.pitch_graph(pkg, be, case, {declare!r}) for _ in range(2)])
            sys.stderr.write("kinds " + repr(sorted(p["kinds"].items())) + "\\n")
            sys.stderr.write("stages " + repr(p["stages"]) + "\\n")
    """)
    r = subprocess.run([sys.executable, "-c", script], env=dict(os.environ, WAE_PLAN_DIGEST="1", **(env or {})), capture_output=True,
                       text=True, check=True)
    got, name = {}, None
    for line in r.stderr.splitlines():
        if line.startswith("case "):
            name = line[5:]
            got[name] = []
        elif line.startswith(("kinds ", "stages ")):
            got[name].append(line)
        elif "[wae plan digest]" in line:
            got[name].append(line.rsplit(": ", 1)[1])
    return got


@pytest.mark.parametrize("voice_sum", ["0", "2"])
def test_declared_plans_equal_host_twins(pkg, host, voice_sum):
    env = {"WAE_VOICE_SUM": voice_sum}
    declared, twins = plan_digests(True, env), plan_digests(False, env)
    assert set(declared) == set(DIGEST_CASES)
    assert declared == twins
    kinds = {name: dict(eval(next(x for x in lines if x.startswith("kinds "))[6:])) for name, lines in declared.items()}
    assert kinds["fused_chain"].get("k_chain") and "k_oscillator" not in kinds["fused_chain"], kinds["fused_chain"]
    assert "k_osc_arate" not in kinds["fused_chain"] and "k_biquad_arate" not in kinds["fused_chain"]
    # (an oscillator with two consumers is a chain of its own written to the arena; k_oscillator is the path with fusion off, an engine
    # option the host-only planner does not take: tests/test_gpu_device_pitch.py renders it)
    assert kinds["materialised_custom_two_consumers"].get("k_chain") == 2, kinds["materialised_custom_two_consumers"]
    assert kinds["arate_lfo_on_detune"].get("k_osc_arate"), kinds["arate_lfo_on_detune"]
    if voice_sum == "2":
        assert kinds["voices"].get("k_voice_sum"), kinds["voices"]


def test_declared_graph_plans_like_the_twin_at_its_placeholder(pkg, host):
    # a value outside the declared range is planned clamped to it: the twin at the range's low end
    def graph(f, declare):
        c, osc = osc_ctx(pkg, host, frequency=f)
        if declare:
            osc.frequency.set_device_value(500.0, 1000.0)
        return pkg.plan_batch([c])
    assert graph(440.0, True)["stages"] == graph(500.0, False)["stages"]
