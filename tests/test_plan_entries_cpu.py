"""The bind entries of every kind through the split sizing pass, on the host (no GPU).  Batches whose graphs declare bound params, static
panner positions, curves, IIR coefficients, schedules, loop points and sources read by reference plan with WAE_PLAN_PARALLEL=1: the
sizing pass is then repeated in runs of graphs, their stage builds merged with every entry reference rebased, and the plan fails unless
the merged entries digest as the serial ones.  WAE_PLAN_DIGEST prints that digest on a line of its own, with the number of entries.
HRTF panners are not covered here: the engine-less planner has no HRIR sphere and refuses them (test_device_spatial_cpu.py)."""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "web-audio-api-rs_b200", "libwae_b200.so")
SR = 48000.0
LENGTH = 24000
GRAPHS = 3  # per batch: the split sizing pass plans them in three runs


@pytest.fixture
def host(pkg):
    if not os.path.exists(LIB):
        pytest.skip("libwae_b200.so is not built (python -c 'import __graft_entry__ as g; g.build()')")
    return pkg.context.Backend(pkg.api(), None)


def noise(seed, ch, frames):
    return list(np.random.default_rng(seed).uniform(-0.5, 0.5, (ch, frames)).astype(np.float32))


def graph(pkg, be, case, g, declare):
    """graph `g` of `case`; declare False: its twin, with host values where the graph declares device memory"""
    c = pkg.OfflineAudioContext(2, LENGTH if case != "loops" else 96000, SR, be)
    dest = c.destination()
    if case == "gain_and_pitch":  # oscillator -> gain, fused into one k_chain record: a PATCH_OSC entry and a gain slot's entry
        o = c.create_oscillator(frequency=220.0 + 10 * g)
        gn = c.create_gain(0.5)
        if declare:
            o.frequency.set_device_value(100.0, 1000.0)
            gn.gain.set_device_value(0.0, 1.0)
        o.connect(gn)
        gn.connect(dest)
        o.start()
    elif case == "panner":  # a static equal-power panner (k_panner_eq): a spatial entry
        o = c.create_oscillator(frequency=330.0)
        pn = c.create_panner(position=(1.0, 0.5, -2.0 - g))
        if declare:
            for name in ("position_x", "position_y", "position_z"):
                getattr(pn, name).set_device_value(-50.0, 50.0)
        o.connect(pn)
        pn.connect(dest)
        o.start()
    elif case in ("curve_chain", "curve_oversampled"):
        # a shaper fused into a chain, and an over-sampled one behind a source that starts late (its k_meta record's mode and the
        # k_shaper_os record's rebuild field)
        over = case == "curve_oversampled"
        sh = c.create_wave_shaper(oversample=pkg.context.OVERSAMPLE_X4 if over else pkg.context.OVERSAMPLE_NONE)
        if declare:
            sh.set_device_curve(64)
        else:
            sh.set_curve(np.linspace(-1.0, 1.0, 64, dtype=np.float32))
        s = c.create_buffer_source(pkg.AudioBuffer(noise(g, 2, LENGTH), SR))
        s.connect(sh)
        s.start_at(3000 / SR if over else 0.0)
        gn = c.create_gain(0.8)
        sh.connect(gn)
        gn.connect(dest)
    elif case == "iir":  # order 2 (a biquad of k_chain, and its scan constants) and order 4 (k_iir_serial)
        s = c.create_buffer_source(pkg.AudioBuffer(noise(g, 2, LENGTH), SR))
        f2 = c.create_iir_filter([0.2, 0.3, 0.2], [1.0, -0.4, 0.1])
        f4 = c.create_iir_filter([0.1, 0.2, 0.3, 0.2, 0.1], [1.0, -0.5, 0.2, -0.05, 0.01])
        if declare:
            f2.set_device_coefficients()
            f4.set_device_coefficients()
        s.connect(f2)
        f2.connect(f4)
        f4.connect(dest)
        s.start()
    elif case == "schedules":  # an oscillator fused into a chain, and one with two consumers (k_oscillator and its k_meta record)
        a = c.create_oscillator(frequency=200.0)
        b = c.create_oscillator(frequency=300.0)
        a.connect(c.create_gain(0.5)).connect(dest)
        b.connect(c.create_gain(0.25)).connect(dest)
        b.connect(c.create_stereo_panner(0.3)).connect(dest)
        a.start_at(0.01 * g)
        b.start_at(0.02)
        if declare:
            a.set_device_schedule((0.0, 0.1), (0.3, 0.4))
            b.set_device_schedule((0.0, 0.1))
    elif case == "loops":  # looping sources with loop points bound: the bound slow track (its playhead walk) and the serial one
        for k, rate in enumerate((1.0, -1.0)):
            s = c.create_buffer_source(pkg.AudioBuffer(noise(10 * g + k, 2, 72000), SR), playback_rate=rate, loop=True)
            s.set_loop_start(0.1)
            s.set_loop_end(0.8)
            s.connect(dest)
            s.start()
            if declare:
                s.set_device_loop((0.1, 0.3), (0.8, 1.2))
    elif case == "source_refs":  # read by reference in a chain (fast track -> biquad -> gain) and on the slow track
        a = c.create_buffer_source()
        a.set_device_input(2, LENGTH, SR, by_reference=declare)
        a.connect(c.create_biquad_filter(type_=pkg.LOWPASS, frequency=1000.0 + 100 * g)).connect(c.create_gain(0.5)).connect(dest)
        a.start()
        b = c.create_buffer_source(playback_rate=0.75, loop=True, loop_start=0.05, loop_end=0.2)
        b.set_device_input(2, LENGTH, SR * 0.5, by_reference=declare)
        b.connect(dest)
        b.start()
    else:
        raise ValueError(case)
    return c


CASES = ["gain_and_pitch", "panner", "curve_chain", "curve_oversampled", "iir", "schedules", "loops", "source_refs"]


def plan_entries(declare):
    """case -> (entries, digest) of the [wae plan entries] line of a batch of GRAPHS graphs of the case, and "all" for one batch of
    every case's graphs"""
    script = textwrap.dedent(f"""
        import sys
        sys.path.insert(0, {os.path.join(ROOT, 'tests')!r}); sys.path.insert(0, {ROOT!r})
        from conftest import load_package
        import test_plan_entries_cpu as T
        pkg = load_package()
        be = pkg.context.Backend(pkg.api(), None)
        batches = [(case, [T.graph(pkg, be, case, g, {declare!r}) for g in range(T.GRAPHS)]) for case in T.CASES]
        batches.append(("all", [T.graph(pkg, be, case, 0, {declare!r}) for case in T.CASES if case != "loops"]))
        for name, graphs in batches:
            sys.stderr.write("case " + name + "\\n")
            sys.stderr.flush()
            pkg.plan_batch(graphs)
    """)
    r = subprocess.run([sys.executable, "-c", script], env=dict(os.environ, WAE_PLAN_DIGEST="1", WAE_PLAN_PARALLEL="1"),
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    got, name = {}, None
    for line in r.stderr.splitlines():
        if line.startswith("case "):
            name = line[5:]
        elif line.startswith("[wae plan entries] group 0 entries "):
            count, digest = line[len("[wae plan entries] group 0 entries "):].split(": ")
            got[name] = (int(count), digest)
    return got


def test_every_kind_passes_the_split_self_check(pkg, host):
    declared, twins = plan_entries(True), plan_entries(False)
    assert set(declared) == set(twins) == set(CASES) | {"all"}
    for name in declared:
        # the twins' entries are their output entries; every declared kind adds its own to the digest
        assert declared[name][0] > twins[name][0] > 0, (name, declared[name], twins[name])
