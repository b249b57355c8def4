"""OscillatorNode periodic waves bound from device memory, on the host (no GPU): the declaration rules of
wae_oscillator_set_device_periodic_wave, the one-shot refusals, the wae_periodic_wave_binding layout of include/wae.h, and plans of graphs
with declared waves.  A declared wave plans exactly as a host wave of the same length (the planner reads a custom oscillator's table
pointer and length only): the same plan_batch dicts and the same WAE_PLAN_DIGEST lines, on the fused chain (k_chain), an
oscillator shared by two chains (materialised by a chain of its own, summed by k_mix), automated frequency (k_osc_arate), a port of custom voices (k_voice_sum under WAE_VOICE_SUM=2) and with
suspend points added after the declaration.  (wae_batch_plan plans with the default options; the unfused path under WAE_OPT_FUSE 0 is
planned by an engine, tests/test_gpu_device_waves.py.)"""
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

PATHS = ["fused", "shared", "arate", "voices", "suspend"]
TABLE_LENGTHS = [2048, 8192]


@pytest.fixture
def host(pkg):
    if not os.path.exists(LIB):
        pytest.skip("libwae_b200.so is not built (python -c 'import __graft_entry__ as g; g.build()')")
    return pkg.context.Backend(pkg.api(), None)


def status_and_text(pkg, fn):
    with pytest.raises(pkg._binding.WaeError) as e:
        fn()
    return e.value.status, e.value.message


def coefficients(seed, n):
    """(real, imag) of n harmonics with 1/k amplitudes and random signs (DC terms included: ignored, as PeriodicWave ignores them)"""
    rng = np.random.default_rng(seed)
    k = np.arange(1, n + 1, dtype=np.float64)
    real = (rng.uniform(-1, 1, n) / k).astype(np.float32)
    imag = (rng.uniform(-1, 1, n) / k).astype(np.float32)
    return real, imag


def host_table(api, real, imag, table_len, normalize=True):
    """wae_periodic_wave_table: the wavetable of these coefficients (either may be None = zeros)"""
    fp = ctypes.POINTER(ctypes.c_float)
    r = None if real is None else np.ascontiguousarray(real, np.float32)
    i = None if imag is None else np.ascontiguousarray(imag, np.float32)
    n = len(r) if r is not None else len(i)
    out = np.zeros(table_len, np.float32)
    api.check(api.periodic_wave_table(None if r is None else r.ctypes.data_as(fp), None if i is None else i.ctypes.data_as(fp), n,
                                      0 if normalize else 1, out.ctypes.data_as(fp), table_len))
    return out


def osc_with_wave(c, n, table_len, table, frequency, normalize=True):
    """an OscillatorNode playing `table` (set_periodic_wave), or, table None, a wave of n coefficients declared bound from device memory"""
    o = c.create_oscillator(frequency=frequency)
    if table is None:
        o.set_device_periodic_wave(n, table_len, disable_normalization=not normalize)
    else:
        o.set_periodic_wave(table)
    return o


def wave_graph(pkg, be, g, length, n, table_len, table=None, path="fused", normalize=True, voices=8, suspends=()):
    """custom oscillator -> lowpass -> gain -> destination, per path:
    fused: as above (one k_chain); shared: the oscillator also feeds a second gain (two consumers: it is materialised on its own);
    arate: the frequency is ramped (k_osc_arate); voices: `voices` such oscillator -> bandpass -> gain chains summed at the destination
    (k_voice_sum under WAE_VOICE_SUM=2); suspend: as fused, with suspend points added after the declaration.
    table: the wavetable given to set_periodic_wave, or None: n coefficients declared.  Returns (context, [oscillators])."""
    c = pkg.OfflineAudioContext(2, length, SR, be)
    oscs = []
    for v in range(voices if path == "voices" else 1):
        f = 110.0 * (1.0 + 0.25 * v) + 7.0 * g
        o = osc_with_wave(c, n, table_len, table, f, normalize)
        bq = c.create_biquad_filter(type_=pkg.BANDPASS if path == "voices" else pkg.LOWPASS, frequency=2000.0 + 100 * g + 50 * v, q=1.0)
        gn = c.create_gain(0.5 / (1 + v))
        o.connect(bq)
        bq.connect(gn)
        gn.connect(c.destination())
        if path == "shared":
            g2 = c.create_gain(0.25)
            o.connect(g2)
            g2.connect(c.destination())
        if path == "arate":
            o.frequency.set_value_at_time(f, 0.0)
            o.frequency.linear_ramp_to_value_at_time(4.0 * f, length / SR)
        o.start()
        oscs.append(o)
    for fr in suspends or ((3072, 8192) if path == "suspend" else ()):
        c.suspend_sync(fr / SR, lambda ctx: None)
    return c, oscs


# ---------------------------------------------------------------------------------------------------------- declaration rules
def test_too_few_coefficients_refused(pkg, host):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    o = c.create_oscillator()
    for n in (0, 1):
        assert status_and_text(pkg, lambda: o.set_device_periodic_wave(n)) == (
            1, "IndexSizeError - `real` and `imag` length should at least 2")
    o.set_device_periodic_wave(2)  # (the failed calls declared nothing)


def test_table_length_zero_refused(pkg, host):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    o = c.create_oscillator()
    assert status_and_text(pkg, lambda: o.set_device_periodic_wave(16, 0)) == (
        1, "a periodic wave bound from device memory has a wavetable of at least one point")
    o.set_device_periodic_wave(16, 1)


def test_not_an_oscillator(pkg, host):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    api = pkg.api()
    assert api.oscillator_set_device_periodic_wave(c._g, c.create_gain().id, 16, 2048, 0) == 1
    assert api.oscillator_set_device_periodic_wave(c._g, 9999, 16, 2048, 0) == 1
    assert b"not an OscillatorNode" in api.last_error()


def test_declared_twice(pkg, host):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    o = c.create_oscillator()
    o.set_device_periodic_wave(16)
    assert status_and_text(pkg, lambda: o.set_device_periodic_wave(16)) == (
        2, "InvalidStateError - the periodic wave is already bound from device memory (wae_oscillator_set_device_periodic_wave)")


def test_set_periodic_wave_after_declaration(pkg, host):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    o = c.create_oscillator()
    o.set_device_periodic_wave(16)
    assert status_and_text(pkg, lambda: o.set_periodic_wave(np.zeros(2048, np.float32))) == (
        2, "InvalidStateError - the periodic wave is bound from device memory (wae_oscillator_set_device_periodic_wave)")


def test_set_periodic_wave_after_declaration_from_a_suspend_callback(pkg, host):
    c = pkg.OfflineAudioContext(2, 4096, SR, host)
    o = c.create_oscillator()
    o.set_device_periodic_wave(16)
    o.connect(c.destination())
    o.start()
    c.suspend_sync(1024 / SR, lambda ctx: o.set_periodic_wave(np.zeros(2048, np.float32)))
    assert status_and_text(pkg, lambda: pkg.plan_batch([c])) == (
        2, "InvalidStateError - the periodic wave is bound from device memory (wae_oscillator_set_device_periodic_wave)")


@pytest.mark.parametrize("via_options", [False, True])
def test_declaration_replaces_a_host_wave(pkg, host, via_options):
    """a declaration over an earlier host wave replaces it, as a second set_periodic_wave would: the plan is that of a declared wave"""
    def build(declare_over):
        c = pkg.OfflineAudioContext(2, 4096, SR, host)
        table = np.ones(2048, np.float32)
        if declare_over and via_options:
            o = c.create_oscillator(frequency=440.0, periodic_wave=table)
        else:
            o = c.create_oscillator(frequency=440.0)
            if declare_over:
                o.set_periodic_wave(table)
        o.set_device_periodic_wave(16, 8192)
        o.connect(c.destination())
        o.start()
        return c
    assert pkg.plan_batch([build(True)]) == pkg.plan_batch([build(False)])


def test_type_stays_custom(pkg, host):
    """the declaration makes the type Custom for good: set_type afterwards changes nothing (as after set_periodic_wave)"""
    def build(set_type):
        c, (o,) = wave_graph(pkg, host, 0, 4096, 16, 8192)
        if set_type:
            o.set_type(pkg.context.SQUARE)
        return c
    assert pkg.plan_batch([build(True)]) == pkg.plan_batch([build(False)])


def test_declaration_after_suspend_point(pkg, host):
    c = pkg.OfflineAudioContext(2, 4096, SR, host)
    o = c.create_oscillator()
    o.connect(c.destination())
    c.suspend_sync(1024 / SR, lambda ctx: o.set_device_periodic_wave(16))
    assert status_and_text(pkg, lambda: pkg.plan_batch([c])) == (
        2, "InvalidStateError - a periodic wave is bound from device memory before the first suspend point")


def test_suspend_points_after_declaration(pkg, host):
    c, _ = wave_graph(pkg, host, 0, 12000, 16, 8192, path="suspend")
    assert pkg.plan_batch([c])["segments"] == 3


def test_oracle_refuses(pkg, oracle):
    c = pkg.OfflineAudioContext(2, 1024, SR, oracle)
    with pytest.raises(pkg._binding.WaeError) as e:
        c.create_oscillator().set_device_periodic_wave(16)
    assert e.value.status == 3


def test_oneshot_refusals(pkg, host):
    api = pkg.api()
    cs = [wave_graph(pkg, host, g, 4096, 16, 2048)[0] for g in range(2)]
    arr = (ctypes.c_void_p * 2)(*[c._g for c in cs])
    out = np.zeros((2, 2, 4096), np.float32)
    assert api.render_batch(None, arr, 2, out.ctypes.data_as(ctypes.c_void_p), 0) == 2
    assert b"wae_batch_bind_periodic_waves" in api.last_error()
    outs = (pkg._binding.c_float_p * 2)(*[pkg._binding.fptr(out[i]) for i in range(2)])
    assert api.render_many(None, arr, 2, outs) == 2
    assert b"wae_batch_bind_periodic_waves" in api.last_error()
    assert api.batch_bind_periodic_waves(None, None, 0, None) == 1


def test_periodic_wave_binding_layout(pkg, tmp_path):
    B = pkg._binding
    assert "wae_oscillator_set_device_periodic_wave" in B.WAE_SYMBOLS and "wae_batch_bind_periodic_waves" in B.WAE_SYMBOLS
    src = tmp_path / "binding.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "wae.h"\nint main(void) {\n'
                   '  printf("%zu %zu %zu %zu %zu\\n", sizeof(wae_periodic_wave_binding), offsetof(wae_periodic_wave_binding, graph_index),\n'
                   '         offsetof(wae_periodic_wave_binding, node), offsetof(wae_periodic_wave_binding, real),\n'
                   '         offsetof(wae_periodic_wave_binding, imag));\n'
                   "  return 0;\n}\n")
    exe = tmp_path / "binding"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = tuple(map(int, subprocess.check_output([str(exe)], text=True).split()))
    S = B.PeriodicWaveBinding
    assert got == (ctypes.sizeof(S), S.graph_index.offset, S.node.offset, S.real.offset, S.imag.offset)
    if not os.path.exists(LIB):
        pytest.skip("libwae_b200.so is not built")
    lib = ctypes.CDLL(LIB)
    assert hasattr(lib, "wae_oscillator_set_device_periodic_wave") and hasattr(lib, "wae_batch_bind_periodic_waves")


# ---------------------------------------------------------------------------------------------------------- plans
KERNEL_OF_PATH = {"fused": "k_chain", "shared": "k_mix", "arate": "k_osc_arate", "voices": "k_voice_sum", "suspend": "k_chain"}


def case_graphs(pkg, be, path, table_len, declared, n=33, graphs=3, length=12000):
    api = pkg.api()
    out = []
    for g in range(graphs):
        table = None if declared else host_table(api, *coefficients(g, n), table_len)
        out.append(wave_graph(pkg, be, g, length, n, table_len, table, path=path)[0])
    return out


@pytest.fixture
def voice_sum_env():
    old = os.environ.get("WAE_VOICE_SUM")
    os.environ["WAE_VOICE_SUM"] = "2"
    yield
    if old is None:
        del os.environ["WAE_VOICE_SUM"]
    else:
        os.environ["WAE_VOICE_SUM"] = old


@pytest.mark.parametrize("table_len", TABLE_LENGTHS)
@pytest.mark.parametrize("path", PATHS)
def test_plan_equals_host_wave(pkg, host, voice_sum_env, path, table_len):
    declared = pkg.plan_batch(case_graphs(pkg, host, path, table_len, True))
    assert KERNEL_OF_PATH[path] in declared["kinds"], declared["kinds"]
    assert declared == pkg.plan_batch(case_graphs(pkg, host, path, table_len, False))


def test_never_started_and_unconnected_declared_oscillators_are_planned(pkg, host):
    c, _ = wave_graph(pkg, host, 0, 4096, 16, 2048)
    idle = c.create_oscillator()
    idle.set_device_periodic_wave(16)
    idle.connect(c.destination())  # never started
    c.create_oscillator().set_device_periodic_wave(8, 64)  # not connected
    pkg.plan_batch([c])


DIGEST_SCRIPT = textwrap.dedent("""
    import sys
    sys.path.insert(0, {tests!r}); sys.path.insert(0, {root!r})
    from conftest import load_package
    import test_device_waves_cpu as T
    pkg = load_package()
    be = pkg.context.Backend(pkg.api(), None)
    for path in T.PATHS:
        for table_len in T.TABLE_LENGTHS:
            pkg.plan_batch(T.case_graphs(pkg, be, path, table_len, sys.argv[1] == "declared"))
""")


def test_plan_digest_equals_host_wave(pkg, host):
    script = DIGEST_SCRIPT.format(tests=os.path.join(ROOT, "tests"), root=ROOT)
    env = dict(os.environ, WAE_PLAN_DIGEST="1", WAE_VOICE_SUM="2")
    out = {}
    for mode in ("declared", "plain"):
        r = subprocess.run([sys.executable, "-c", script, mode], env=env, capture_output=True, text=True, check=True)
        out[mode] = [line for line in r.stderr.splitlines() if "[wae plan digest]" in line]
    assert len(out["declared"]) >= len(PATHS) * len(TABLE_LENGTHS) and out["declared"] == out["plain"]
