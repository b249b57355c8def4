"""Device inputs on the host (no GPU): wae_buffer_source_set_device_input validates like AudioBuffer::new and set_buffer, graphs whose
sources are device inputs plan exactly like the same graphs given AudioBuffers, and the wae_source_binding layout of include/wae.h is the
one the ctypes binding declares."""
import ctypes
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

import graphs as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "web-audio-api-rs_b200", "libwae_b200.so")
SR = 48000.0


@pytest.fixture
def host(pkg):
    if not os.path.exists(LIB):
        pytest.skip("libwae_b200.so is not built (python -c 'import __graft_entry__ as g; g.build()')")
    return pkg.context.Backend(pkg.api(), None)


def status_of(fn):
    with pytest.raises(Exception) as e:
        fn()
    return e.value.status, e.value.message


def test_set_device_input_on_other_nodes(pkg, host):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    g = c.create_gain()
    api = pkg.api()
    assert api.buffer_source_set_device_input(c._g, g.id, 2, 1000, SR) == 1  # INVALID_ARGUMENT
    assert b"AudioBufferSourceNode" in api.last_error()
    assert api.buffer_source_set_device_input(c._g, 9999, 2, 1000, SR) == 1


@pytest.mark.parametrize("channels,length,text", [
    (0, 1000, "NotSupportedError - Invalid number of channels: 0 is outside range [1, 32]"),
    (33, 1000, "NotSupportedError - Invalid number of channels: 33 is outside range [1, 32]"),
    (2, 0, "NotSupportedError - Invalid length: 0 is less than or equal to minimum bound (0)"),
])
def test_set_device_input_validates_like_audio_buffer(pkg, host, channels, length, text):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    s = c.create_buffer_source()
    assert status_of(lambda: s.set_device_input(channels, length, SR)) == (3, text)
    s.set_device_input(1, 10, SR)  # (the failed call assigned nothing)


def test_buffer_assigned_twice(pkg, host):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    twice = (2, "InvalidStateError - cannot assign buffer twice")
    a = c.create_buffer_source()
    a.set_device_input(2, 1000, SR)
    assert status_of(lambda: a.set_buffer(pkg.AudioBuffer.zeros(2, 1000, SR))) == twice
    assert status_of(lambda: a.set_device_input(2, 1000, SR)) == twice
    b = c.create_buffer_source()
    b.set_buffer(pkg.AudioBuffer.zeros(1, 10, SR))
    assert status_of(lambda: b.set_device_input(2, 1000, SR)) == twice
    d = c.create_buffer_source(pkg.AudioBuffer.zeros(1, 10, SR))
    assert status_of(lambda: d.set_device_input(1, 10, SR)) == twice


def c2_device(pkg, backend, g, length, frames=None):
    """G.c2_buffer_biquad_gain with its source declared as a device input of `frames` frames."""
    _, f0, q, gain = G.c2_params(g)
    c = pkg.OfflineAudioContext(2, length, SR, backend)
    src = c.create_buffer_source()
    src.set_device_input(2, frames or length, SR)
    bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=f0, q=q)
    gn = c.create_gain(gain)
    src.connect(bq)
    bq.connect(gn)
    gn.connect(c.destination())
    src.start()
    return c


@pytest.mark.parametrize("n,length", [(3, 48000), (70, 20000)])
def test_plan_equals_buffer_plan(pkg, host, n, length):
    dev = pkg.plan_batch([c2_device(pkg, host, g, length) for g in range(n)])
    buf = pkg.plan_batch([G.c2_buffer_biquad_gain(pkg, host, g, length) for g in range(n)])  # distinct random PCM per graph
    for key in ("kinds", "chunk_frames", "arena_floats_per_frame", "source_floats", "groups", "stages"):
        assert dev[key] == buf[key], key
    assert dev["source_floats"] == n * 2 * length


def test_plan_digest_equals_buffer_plan(pkg, host):
    """WAE_PLAN_DIGEST=1 hashes every instance record the sizing pass builds (the slab offsets of the sources included)."""
    script = textwrap.dedent(f"""
        import sys
        sys.path.insert(0, {os.path.join(ROOT, 'tests')!r}); sys.path.insert(0, {ROOT!r})
        from conftest import load_package
        import graphs as G
        import test_device_sources_cpu as T
        pkg = load_package()
        be = pkg.context.Backend(pkg.api(), None)
        if sys.argv[1] == "dev":
            cs = [T.c2_device(pkg, be, g, 30000) for g in range(5)]
        else:
            cs = [G.c2_buffer_biquad_gain(pkg, be, g, 30000) for g in range(5)]
        pkg.plan_batch(cs)
    """)
    env = dict(os.environ, WAE_PLAN_DIGEST="1")
    out = {}
    for mode in ("dev", "buf"):
        r = subprocess.run([sys.executable, "-c", script, mode], env=env, capture_output=True, text=True, check=True)
        out[mode] = [line for line in r.stderr.splitlines() if "[wae plan digest]" in line]
    assert out["dev"] and out["dev"] == out["buf"]


def test_source_binding_layout(pkg, tmp_path):
    B = pkg._binding
    assert "wae_buffer_source_set_device_input" in B.WAE_SYMBOLS and "wae_batch_bind_sources" in B.WAE_SYMBOLS
    src = tmp_path / "binding.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "wae.h"\nint main(void) {\n'
                   '  printf("%zu %zu %zu %zu %zu\\n", sizeof(wae_source_binding), offsetof(wae_source_binding, node),\n'
                   '         offsetof(wae_source_binding, pcm), offsetof(wae_source_binding, channel_stride), offsetof(wae_source_binding, graph_index));\n'
                   "  return 0;\n}\n")
    exe = tmp_path / "binding"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    size, node, pcm, stride, gi = map(int, subprocess.check_output([str(exe)], text=True).split())
    S = B.SourceBinding
    assert (size, node, pcm, stride, gi) == (ctypes.sizeof(S), S.node.offset, S.pcm.offset, S.channel_stride.offset, S.graph_index.offset)
    if not os.path.exists(LIB):
        pytest.skip("libwae_b200.so is not built")
    lib = ctypes.CDLL(LIB)
    assert hasattr(lib, "wae_buffer_source_set_device_input") and hasattr(lib, "wae_batch_bind_sources")


def test_oneshot_and_bind_refusals_without_device(pkg, host):
    """The refusals that need no device: binding into nothing, and the one-shot calls (they answer before touching the engine)."""
    api = pkg.api()
    cs = [c2_device(pkg, host, g, 4096) for g in range(2)]
    arr = (ctypes.c_void_p * 2)(*[c._g for c in cs])
    out = np.zeros((2, 2, 4096), np.float32)
    assert api.render_batch(None, arr, 2, out.ctypes.data_as(ctypes.c_void_p), 0) == 2
    assert b"wae_batch_bind_sources" in api.last_error()
    outs = (pkg._binding.c_float_p * 2)(*[pkg._binding.fptr(out[i]) for i in range(2)])
    assert api.render_many(None, arr, 2, outs) == 2
    assert api.batch_bind_sources(None, None, 0, None) == 1
