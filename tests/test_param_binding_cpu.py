"""Params bound from device memory on the host (no GPU): the declaration rules of wae_param_set_device_value, the one-shot refusals,
the wae_param_binding layout of include/wae.h, and plans of graphs with bound params (the same stages as the same graphs with
constants, and the plans of graphs without declarations unchanged)."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import graphs as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "web-audio-api-rs_b200", "libwae_b200.so")
SR = 48000.0
F32_MAX = 3.4028234663852886e38


@pytest.fixture
def host(pkg):
    if not os.path.exists(LIB):
        pytest.skip("libwae_b200.so is not built (python -c 'import __graft_entry__ as g; g.build()')")
    return pkg.context.Backend(pkg.api(), None)


def status_of(fn):
    with pytest.raises(Exception) as e:
        fn()
    return e.value.status


def test_supported_params(pkg, host):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    bq = c.create_biquad_filter()
    for p in (bq.q, bq.detune, bq.frequency, bq.gain):
        p.set_device_value()
    c.create_gain().gain.set_device_value(0.05, 2.0)
    c.create_stereo_panner().pan.set_device_value()
    comp = c.create_dynamics_compressor()
    for name in ("attack", "knee", "ratio", "release", "threshold"):
        getattr(comp, name).set_device_value()


def test_unsupported_params(pkg, host):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    osc = c.create_oscillator()
    assert status_of(lambda: osc.frequency.set_device_value()) == 4
    assert status_of(lambda: osc.detune.set_device_value()) == 4
    assert status_of(lambda: c.create_delay().delay_time.set_device_value()) == 4
    assert status_of(lambda: c.create_constant_source().offset.set_device_value()) == 4
    assert status_of(lambda: c.create_panner().position_x.set_device_value()) == 4
    assert status_of(lambda: c.listener().position_x.set_device_value()) == 4
    api = pkg.api()
    g = c.create_gain()
    assert api.param_set_device_value(c._g, g.id, 1, 0.0, 1.0) == 1  # param index out of range
    assert api.param_set_device_value(c._g, 9999, 0, 0.0, 1.0) == 1


@pytest.mark.parametrize("lo,hi", [(1.0, 0.0), (float("nan"), 1.0), (0.0, float("inf")), (-F32_MAX * 2, 0.0)])
def test_range_refusals(pkg, host, lo, hi):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    g = c.create_gain()
    assert status_of(lambda: g.gain.set_device_value(lo, hi)) == 1
    g.gain.set_device_value(0.0, 1.0)  # (the failed call declared nothing)


def test_range_outside_min_max(pkg, host):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    p = c.create_stereo_panner()
    assert status_of(lambda: p.pan.set_device_value(2.0, 3.0)) == 1


def test_declared_twice(pkg, host):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    g = c.create_gain()
    g.gain.set_device_value()
    assert status_of(lambda: g.gain.set_device_value()) == 2


def test_events_before_and_after(pkg, host):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    a = c.create_gain()
    a.gain.set_value(0.5)  # a value is no automation: the placeholder
    a.gain.set_device_value()
    assert status_of(lambda: a.gain.set_value(0.25)) == 2
    assert status_of(lambda: a.gain.linear_ramp_to_value_at_time(0.0, 0.01)) == 2
    b = c.create_gain()
    b.gain.set_value_at_time(0.5, 0.01)
    assert status_of(lambda: b.gain.set_device_value()) == 2


def test_connections_before_and_after(pkg, host):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    lfo = c.create_oscillator()
    a = c.create_gain()
    a.gain.set_device_value()
    assert status_of(lambda: lfo.connect(a.gain)) == 2
    b = c.create_biquad_filter()
    lfo.connect(b.frequency)
    assert status_of(lambda: b.frequency.set_device_value()) == 2
    b.q.set_device_value()  # (another param of the node)


def test_set_value_from_suspend_callback(pkg, host):
    c = pkg.OfflineAudioContext(2, 4096, SR, host)
    src = c.create_buffer_source(pkg.AudioBuffer.zeros(2, 4096, SR))
    g = c.create_gain()
    src.connect(g)
    g.connect(c.destination())
    src.start()
    g.gain.set_device_value()
    c.suspend_sync(1024 / SR, lambda ctx: g.gain.set_value(0.5))
    assert status_of(lambda: pkg.plan_batch([c])) == 2


def test_declaration_after_suspend_point(pkg, host):
    c = pkg.OfflineAudioContext(2, 4096, SR, host)
    g = c.create_gain()
    g.connect(c.destination())
    c.suspend_sync(1024 / SR, lambda ctx: g.gain.set_device_value())
    assert status_of(lambda: pkg.plan_batch([c])) == 2


def c2_bound(pkg, backend, g, length, lo=0.05, hi=2.0):
    """G.c2_buffer_biquad_gain with its biquad frequency / Q and its gain bound from device memory."""
    c, (bq, gn) = c2_nodes(pkg, backend, g, length)
    bq.frequency.set_device_value()
    bq.q.set_device_value()
    gn.gain.set_device_value(lo, hi)
    return c


def c2_nodes(pkg, backend, g, length):
    _, f0, q, gain = G.c2_params(g)
    c = pkg.OfflineAudioContext(2, length, SR, backend)
    src = c.create_buffer_source(pkg.AudioBuffer(list(G.c2_source(g, length)), SR))
    bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=f0, q=q)
    gn = c.create_gain(gain)
    src.connect(bq)
    bq.connect(gn)
    gn.connect(c.destination())
    src.start()
    return c, (bq, gn)


def test_c2_plan_unchanged_by_binding(pkg, host):
    bound = pkg.plan_batch([c2_bound(pkg, host, g, 20000) for g in range(8)])
    plain = pkg.plan_batch([G.c2_buffer_biquad_gain(pkg, host, g, 20000) for g in range(8)])
    for key in ("kinds", "chunk_frames", "arena_floats_per_frame", "source_floats", "groups", "stages"):
        assert bound[key] == plain[key], key
    assert bound["kinds"] == {"k_chain": 1}, bound["kinds"]


def test_default_range_gain_plans_as_possibly_silent(pkg, host):
    """A gain whose range includes 0 may answer with silence: it stays fused into the chain, whose output carries a layout track."""
    fused = pkg.plan_batch([c2_bound(pkg, host, g, 20000, -F32_MAX, F32_MAX) for g in range(4)])
    assert fused["kinds"] == {"k_chain": 1}
    assert fused["stages"] == pkg.plan_batch([c2_bound(pkg, host, g, 20000) for g in range(4)])["stages"]


def test_plan_digest_corpus_has_no_declarations(pkg, host):
    """The corpus graphs declare nothing, and a graph without declarations plans as before: the plan of C2 with constants is the plan
    of C2 whose bound params were planned from the same values (tools/plan_digest_corpus.py prints the digests of the whole corpus)."""
    import textwrap, sys
    script = textwrap.dedent(f"""
        import sys
        sys.path.insert(0, {os.path.join(ROOT, 'tests')!r}); sys.path.insert(0, {ROOT!r})
        from conftest import load_package
        import graphs as G
        import test_param_binding_cpu as T
        pkg = load_package()
        be = pkg.context.Backend(pkg.api(), None)
        if sys.argv[1] == "bound":
            cs = [T.c2_bound(pkg, be, g, 30000) for g in range(5)]
        else:
            cs = [G.c2_buffer_biquad_gain(pkg, be, g, 30000) for g in range(5)]
        pkg.plan_batch(cs)
    """)
    env = dict(os.environ, WAE_PLAN_DIGEST="1")
    out = {}
    for mode in ("bound", "plain"):
        r = subprocess.run([sys.executable, "-c", script, mode], env=env, capture_output=True, text=True, check=True)
        out[mode] = [line for line in r.stderr.splitlines() if "[wae plan digest]" in line]
    assert out["bound"] and out["bound"] == out["plain"]


def test_oneshot_refusals(pkg, host):
    api = pkg.api()
    cs = [c2_bound(pkg, host, g, 4096) for g in range(2)]
    arr = (ctypes.c_void_p * 2)(*[c._g for c in cs])
    out = np.zeros((2, 2, 4096), np.float32)
    assert api.render_batch(None, arr, 2, out.ctypes.data_as(ctypes.c_void_p), 0) == 2
    assert b"wae_batch_bind_params" in api.last_error()
    outs = (pkg._binding.c_float_p * 2)(*[pkg._binding.fptr(out[i]) for i in range(2)])
    assert api.render_many(None, arr, 2, outs) == 2
    assert api.batch_bind_params(None, None, 0, None) == 1


def test_param_binding_layout(pkg, tmp_path):
    B = pkg._binding
    assert "wae_param_set_device_value" in B.WAE_SYMBOLS and "wae_batch_bind_params" in B.WAE_SYMBOLS
    src = tmp_path / "binding.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "wae.h"\nint main(void) {\n'
                   '  printf("%zu %zu %zu %zu %zu\\n", sizeof(wae_param_binding), offsetof(wae_param_binding, graph_index),\n'
                   '         offsetof(wae_param_binding, node), offsetof(wae_param_binding, param_index), offsetof(wae_param_binding, value));\n'
                   "  return 0;\n}\n")
    exe = tmp_path / "binding"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = tuple(map(int, subprocess.check_output([str(exe)], text=True).split()))
    S = B.ParamBinding
    assert got == (ctypes.sizeof(S), S.graph_index.offset, S.node.offset, S.param_index.offset, S.value.offset)
    if not os.path.exists(LIB):
        pytest.skip("libwae_b200.so is not built")
    lib = ctypes.CDLL(LIB)
    assert hasattr(lib, "wae_param_set_device_value") and hasattr(lib, "wae_batch_bind_params")
