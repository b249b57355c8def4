"""Device inputs read by reference on the host (no GPU): wae_buffer_source_set_device_input_by_reference validates like
wae_buffer_source_set_device_input, one-shot renders refuse it, and a graph whose inputs are read by reference plans like its
copy-declared twin (same stages, chunk and arena) with the referenced inputs' slab floats left out."""
import ctypes
import os

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


def test_declaration_on_other_nodes(pkg, host):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    g = c.create_gain()
    api = pkg.api()
    assert api.buffer_source_set_device_input_by_reference(c._g, g.id, 2, 1000, SR) == 1  # INVALID_ARGUMENT
    assert b"AudioBufferSourceNode" in api.last_error()
    assert api.buffer_source_set_device_input_by_reference(c._g, 9999, 2, 1000, SR) == 1


@pytest.mark.parametrize("channels,length,text", [
    (0, 1000, "NotSupportedError - Invalid number of channels: 0 is outside range [1, 32]"),
    (33, 1000, "NotSupportedError - Invalid number of channels: 33 is outside range [1, 32]"),
    (2, 0, "NotSupportedError - Invalid length: 0 is less than or equal to minimum bound (0)"),
])
def test_declaration_validates_like_audio_buffer(pkg, host, channels, length, text):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    s = c.create_buffer_source()
    assert status_of(lambda: s.set_device_input(channels, length, SR, by_reference=True)) == (3, text)
    s.set_device_input(1, 10, SR, by_reference=True)  # (the failed call assigned nothing)
    assert s.id in c._source_refs


def test_buffer_assigned_twice(pkg, host):
    """"cannot assign buffer twice" in both directions against set_buffer, and between the two declarations"""
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    twice = (2, "InvalidStateError - cannot assign buffer twice")
    a = c.create_buffer_source()
    a.set_device_input(2, 1000, SR, by_reference=True)
    assert status_of(lambda: a.set_buffer(pkg.AudioBuffer.zeros(2, 1000, SR))) == twice
    assert status_of(lambda: a.set_device_input(2, 1000, SR, by_reference=True)) == twice
    assert status_of(lambda: a.set_device_input(2, 1000, SR)) == twice
    b = c.create_buffer_source()
    b.set_buffer(pkg.AudioBuffer.zeros(1, 10, SR))
    assert status_of(lambda: b.set_device_input(2, 1000, SR, by_reference=True)) == twice
    d = c.create_buffer_source()
    d.set_device_input(1, 10, SR)
    assert status_of(lambda: d.set_device_input(1, 10, SR, by_reference=True)) == twice


def test_oneshot_refusals(pkg, host):
    api = pkg.api()
    cs = [make(pkg, host, "chain", g, 4096, True) for g in range(2)]
    arr = (ctypes.c_void_p * 2)(*[c._g for c in cs])
    out = np.zeros((2, 2, 4096), np.float32)
    assert api.render_batch(None, arr, 2, out.ctypes.data_as(ctypes.c_void_p), 0) == 2
    assert b"device inputs" in api.last_error() and b"wae_batch_bind_sources" in api.last_error()
    outs = (pkg._binding.c_float_p * 2)(*[pkg._binding.fptr(out[i]) for i in range(2)])
    assert api.render_many(None, arr, 2, outs) == 2
    assert b"wae_batch_bind_sources" in api.last_error()


def test_symbol_bound(pkg):
    assert "wae_buffer_source_set_device_input_by_reference" in pkg._binding.WAE_SYMBOLS
    if not os.path.exists(LIB):
        pytest.skip("libwae_b200.so is not built")
    assert hasattr(ctypes.CDLL(LIB), "wae_buffer_source_set_device_input_by_reference")


def make(pkg, be, shape, g, length, ref, frames=None, channels=2):
    """a graph of `shape` whose sources are device inputs of `frames` frames, declared by reference (ref) or for a copy"""
    frames = frames or length
    c = pkg.OfflineAudioContext(2, length, SR, be)

    def src(**kw):
        s = c.create_buffer_source(**kw)
        s.set_device_input(channels, frames, SR, by_reference=ref)
        return s

    if shape == "chain":  # fused k_chain
        _, f0, q, gain = G.c2_params(g)
        s = src()
        bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=f0, q=q)
        gn = c.create_gain(gain)
        s.connect(bq)
        bq.connect(gn)
        gn.connect(c.destination())
        s.start()
    elif shape == "fast_loop":  # k_buffer_source: two consumers keep it out of a chain
        s = src(loop=True)
        s.connect(c.create_gain(0.5)).connect(c.destination())
        s.connect(c.create_stereo_panner(-0.3)).connect(c.destination())
        s.start()
    elif shape == "slow":  # resampled slow track
        s = c.create_buffer_source(playback_rate=0.75, loop=True, loop_start=0.05 + 0.01 * g, loop_end=0.2)
        s.set_device_input(channels, frames, SR * 0.5, by_reference=ref)
        s.connect(c.destination())
        s.start()
    elif shape == "serial":  # automated detune
        s = src()
        s.detune.linear_ramp_to_value_at_time(300.0 + 50 * g, length / SR)
        s.connect(c.destination())
        s.start()
    elif shape == "two":  # two inputs in one graph
        a, b = src(), src()
        a.connect(c.destination())
        b.connect(c.create_gain(0.25)).connect(c.destination())
        a.start()
        b.start_at_with_offset(0.01, 0.02)
    else:
        raise ValueError(shape)
    return c


SHAPES = ["chain", "fast_loop", "slow", "serial", "two"]


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("n,length,frames", [(3, 48000, 48000), (5, 30001, 29999), (70, 20000, 20003)])
def test_plan_equals_copy_twin(pkg, host, shape, n, length, frames):
    ref = pkg.plan_batch([make(pkg, host, shape, g, length, True, frames) for g in range(n)])
    cp = pkg.plan_batch([make(pkg, host, shape, g, length, False, frames) for g in range(n)])
    for key in ("kinds", "chunk_frames", "arena_floats_per_frame", "groups", "stages"):
        assert ref[key] == cp[key], key
    inputs = 2 if shape == "two" else 1
    assert cp["source_floats"] - ref["source_floats"] == n * inputs * 2 * ((frames + 3) // 4 * 4)
    assert ref["source_floats"] == 0


def test_mixed_declarations_in_one_batch(pkg, host):
    """copy and reference declarations side by side: only the referenced inputs leave the slab"""
    n, length = 6, 24000
    mixed = pkg.plan_batch([make(pkg, host, "chain", g, length, g % 2 == 0) for g in range(n)])
    cp = pkg.plan_batch([make(pkg, host, "chain", g, length, False) for g in range(n)])
    for key in ("kinds", "chunk_frames", "arena_floats_per_frame", "groups", "stages"):
        assert mixed[key] == cp[key], key
    assert mixed["source_floats"] == cp["source_floats"] // 2
