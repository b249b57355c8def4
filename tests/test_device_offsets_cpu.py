"""AudioBufferSourceNode offsets and durations bound from device memory (wae_buffer_source_set_device_offset), on the host (no GPU): the
declaration rules, and plans equal to host twins with the same schedule declaration, started with the windows' low ends."""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "web-audio-api-rs_b200", "libwae_b200.so")
SR = 48000.0
F64_MAX = 1.7976931348623157e308
BOUND = "k_buffer_source_slow(bound)"
SERIAL = "k_buffer_source_serial"


@pytest.fixture
def host(pkg):
    if not os.path.exists(LIB):
        pytest.skip("libwae_b200.so is not built (python -c 'import __graft_entry__ as g; g.build()')")
    return pkg.context.Backend(pkg.api(), None)


def status_of(fn):
    with pytest.raises(Exception) as e:
        fn()
    return e.value.status


def test_declaration_rules(pkg, host):
    api = pkg.api()
    c = pkg.OfflineAudioContext(1, 4096, SR, host)
    s = c.create_buffer_source(pkg.AudioBuffer.zeros(1, 512, SR))
    s.connect(c.destination())
    s.start_at_with_offset_and_duration(0.0, 0.001, 0.002)
    assert api.buffer_source_set_device_offset(c._g, s.id, 0.0, 0.01, 0, 0.0, 0.0) == 2  # no schedule declared
    s.set_device_schedule((0.0, 0.0))
    osc = c.create_oscillator()
    osc.start()
    osc.set_device_schedule((0.0, 0.05))
    assert api.buffer_source_set_device_offset(c._g, osc.id, 0.0, 0.01, 0, 0.0, 0.0) == 1  # not a buffer source
    assert api.buffer_source_set_device_offset(c._g, 12345, 0.0, 0.01, 0, 0.0, 0.0) == 1  # unknown node
    for lo, hi in ((0.02, 0.01), (-0.01, 0.05), (0.0, float("inf")), (float("nan"), 1.0)):
        assert api.buffer_source_set_device_offset(c._g, s.id, lo, hi, 0, 0.0, 0.0) == 1, (lo, hi)
        assert api.buffer_source_set_device_offset(c._g, s.id, 0.0, 0.01, 1, lo, hi) == 1, (lo, hi)
    assert api.buffer_source_set_device_offset(c._g, s.id, 0.0, 0.01, 0, -1.0, float("nan")) == 0  # (no duration: its window is unused)
    assert api.buffer_source_set_device_offset(c._g, s.id, 0.0, 0.01, 1, 0.0, 1.0) == 2  # declared twice
    assert status_of(lambda: s.start_at(0.0)) == 2


def test_python_declaration(pkg, host):
    c = pkg.OfflineAudioContext(1, 4096, SR, host)
    s = c.create_buffer_source(pkg.AudioBuffer.zeros(1, 512, SR))
    s.start()
    assert status_of(lambda: s.set_device_schedule((0.0, 0.0), duration=(0.0, 1.0))) == 1  # a duration without an offset
    assert status_of(lambda: s.set_device_schedule((0.0, 0.0), offset=(0.5, 0.1))) == 1
    # the refused calls declared nothing: the start is still free to be declared
    s.set_device_schedule((0.0, 0.0), offset=(0.0, 0.01), duration=(0.0, 1.0))
    assert c._device_schedules[s.id] == (False, True, True)
    assert status_of(lambda: s.set_device_schedule((0.0, 0.0))) == 2
    s2 = c.create_buffer_source(pkg.AudioBuffer.zeros(1, 512, SR))
    s2.start()
    s2.set_device_schedule((0.0, 0.0), stop=(0.0, 1.0), offset=(0.0, 0.01))
    assert c._device_schedules[s2.id] == (True, True, False)


def absn_graph(pkg, backend, declare, offset=0.0, duration=None, rate=1.0, loop=False, rate_range=None, start=0.01, dev=False):
    """buffer source -> lowpass -> destination with its start declared; `declare`: the offset (and duration) declared with windows whose
    low ends are `offset` / `duration`, else the host twin given them to start"""
    c = pkg.OfflineAudioContext(2, 9600, SR, backend)
    s = c.create_buffer_source(playback_rate=rate, loop=loop)
    if dev:
        s.set_device_input(2, 4800, 44100.0)
    else:
        pcm = np.random.default_rng(3).uniform(-0.5, 0.5, (2, 4800)).astype(np.float32)
        s.set_buffer(pkg.AudioBuffer(list(pcm), SR))
    if rate_range is not None:
        s.playback_rate.set_device_value(*rate_range)
    bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=1000.0)
    s.connect(bq)
    bq.connect(c.destination())
    if declare:
        s.start_at(start)
        s.set_device_schedule((start, start + 0.1), offset=(offset, offset + 0.05),
                              duration=None if duration is None else (duration, duration + 0.5))
    else:
        s.start_at_with_offset_and_duration(start, offset, F64_MAX if duration is None else duration)
        s.set_device_schedule((start, start + 0.1))
    return c


PATHS = {
    "rate1": (dict(), BOUND),
    "rate1_aligned": (dict(start=0.0), BOUND),  # an offset of 0 from an aligned start: the 1:1 copy inside the bound kernel
    "rate09": (dict(rate=0.9), BOUND),
    "bound_range": (dict(rate_range=(0.5, 2.0)), BOUND),
    "dev_44k": (dict(dev=True), BOUND),
    "loop": (dict(loop=True), SERIAL),
    "range_to_zero": (dict(rate_range=(0.0, 2.0)), SERIAL),
}
DIGEST_CASES = {f"{p}-{o}-{d}": dict(PATHS[p][0], offset=o, duration=d)
                for p in PATHS for o in (0.0, 0.0123) for d in (None, 0.03)}


@pytest.mark.parametrize("name", list(PATHS))
def test_stage(pkg, host, name):
    case, stage = PATHS[name]
    for duration in (None, 0.03):
        k = pkg.plan_batch([absn_graph(pkg, host, True, 0.0123, duration, **case)])["kinds"]
        assert k.get(stage) == 1, k
        assert "k_buffer_source" not in k and "k_buffer_source_slow" not in k, k


def plan_digests(declare, env):
    script = textwrap.dedent(f"""
        import sys
        sys.path.insert(0, {os.path.join(ROOT, 'tests')!r}); sys.path.insert(0, {ROOT!r})
        from conftest import load_package
        import test_device_offsets_cpu as T
        pkg = load_package()
        be = pkg.context.Backend(pkg.api(), None)
        for name, kw in T.DIGEST_CASES.items():
            sys.stderr.write("case " + name + "\\n")
            c = T.absn_graph(pkg, be, {declare!r}, **kw)
            sys.stderr.write("kinds " + repr(sorted(pkg.plan_batch([c])["kinds"].items())) + "\\n")
    """)
    r = subprocess.run([sys.executable, "-c", script], env=dict(os.environ, WAE_PLAN_DIGEST="1", **env), capture_output=True, text=True,
                       check=True)
    got, name = {}, None
    for line in r.stderr.splitlines():
        if line.startswith("case "):
            name = line[5:]
            got[name] = []
        elif line.startswith("kinds "):
            got[name].append(line[6:])
        elif "[wae plan digest]" in line:
            got[name].append(line.rsplit(": ", 1)[1])
    return got


@pytest.mark.parametrize("env", [{}, {"WAE_PLAN_PARALLEL": "1"}], ids=["default", "parallel"])
def test_declared_plans_equal_host_twins(pkg, host, env):
    """The records of a declared source hold the windows' low ends: the plan (stages and digest) is that of the host twin with the same
    schedule declaration, started with those offsets and durations."""
    declared, twins = plan_digests(True, env), plan_digests(False, env)
    assert set(declared) == set(DIGEST_CASES)
    assert all(len(v) >= 2 for v in declared.values()), declared  # (the stages and at least one digest)
    assert declared == twins
