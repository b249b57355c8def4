"""ConvolverNode responses bound from device memory, on the host (no GPU): the declaration rules of wae_convolver_set_device_response,
the one-shot refusals, the wae_response_binding layout of include/wae.h, and plans of graphs with declared responses (the same stages,
sizes and digest as the same graphs given an AudioBuffer of the declared shape whose last partition is not trimmed)."""
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
BLOCK = 8192  # frames per convolver partition


@pytest.fixture
def host(pkg):
    if not os.path.exists(LIB):
        pytest.skip("libwae_b200.so is not built (python -c 'import __graft_entry__ as g; g.build()')")
    return pkg.context.Backend(pkg.api(), None)


def status_and_text(pkg, fn):
    with pytest.raises(pkg._binding.WaeError) as e:
        fn()
    return e.value.status, e.value.message


def full_ir(ch, length, seed=3):
    """A response of this shape whose last sample is far above the trimming threshold: no partition is trimmed, normalised or not."""
    ir = G.synthetic_ir(length, ch, seed=seed, decay=0.2)
    for c in ir:
        c[-1] = 0.5
    return ir


def conv_graph(pkg, be, g, length, ir_ch, ir_len, ir=None, in_ch=2, normalize=True, layout="fixed", stop=None):
    """A source -> ConvolverNode -> destination.  ir: the response given to set_buffer (a list of channels), or None: a response of
    [ir_ch][ir_len] declared bound from device memory.  layout "switch": a tone plus a stereo source that ends (the input changes
    between one and two channels).  stop: the source's stop frame.  Returns (context, convolver)."""
    rng = np.random.default_rng(4000 + g)
    c = pkg.OfflineAudioContext(2, length, SR, be)
    cv = c.create_convolver(disable_normalization=not normalize)
    if ir is None:
        cv.set_device_response(ir_ch, ir_len, SR)
    else:
        cv.set_buffer(pkg.AudioBuffer(ir, SR))
    if layout == "switch":
        o = c.create_oscillator(frequency=220.0 + 30 * g)
        o.start()
        o.connect(cv)
        n_st = 9000 + 500 * g
        st = c.create_buffer_source(pkg.AudioBuffer(list(rng.uniform(-0.5, 0.5, (2, n_st)).astype(np.float32)), SR))
        st.start_at(3000 / SR)
        st.connect(cv)
    else:
        pcm = (rng.uniform(-1.0, 1.0, (in_ch, length)) * 0.05).astype(np.float32)
        pcm[:, :4096] += rng.uniform(-0.5, 0.5, (in_ch, min(4096, length))).astype(np.float32)
        s = c.create_buffer_source(pkg.AudioBuffer(list(pcm), SR))
        s.connect(cv)
        s.start()
        if stop is not None:
            s.stop_at(stop / SR)
    cv.connect(c.destination())
    return c, cv


# ---------------------------------------------------------------------------------------------------------- declaration rules
@pytest.mark.parametrize("ch", [0, 3, 5, 8])
def test_channel_counts_refused(pkg, host, ch):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    cv = c.create_convolver()
    assert status_and_text(pkg, lambda: cv.set_device_response(ch, 1000, SR)) == (
        3, "NotSupportedError - the convolution buffer must consist of 1, 2 or 4 channels")
    cv.set_device_response(2, 1000, SR)  # (the failed call declared nothing)


def test_rate_refused(pkg, host):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    cv = c.create_convolver()
    assert status_and_text(pkg, lambda: cv.set_device_response(2, 1000, 44100.0)) == (
        3, "NotSupportedError - sample rate of the convolution buffer must match the audio context")


def test_length_zero_refused(pkg, host):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    cv = c.create_convolver()
    assert status_and_text(pkg, lambda: cv.set_device_response(1, 0, SR)) == (
        3, "NotSupportedError - Invalid length: 0 is less than or equal to minimum bound (0)")


def test_texts_match_set_buffer(pkg, host):
    """the declaration answers with set_buffer's own texts"""
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    a, b = c.create_convolver(), c.create_convolver()
    s1, t1 = status_and_text(pkg, lambda: a.set_buffer(pkg.AudioBuffer([np.zeros(10, np.float32)] * 3, SR)))
    s2, t2 = status_and_text(pkg, lambda: b.set_device_response(3, 10, SR))
    assert (s1, t1) == (s2, t2)
    s1, t1 = status_and_text(pkg, lambda: a.set_buffer(pkg.AudioBuffer([np.zeros(10, np.float32)], 22050.0)))
    s2, t2 = status_and_text(pkg, lambda: b.set_device_response(1, 10, 22050.0))
    assert (s1, t1) == (s2, t2)


def test_not_a_convolver(pkg, host):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    api = pkg.api()
    assert api.convolver_set_device_response(c._g, c.create_gain().id, 2, 100, SR) == 1
    assert api.convolver_set_device_response(c._g, 9999, 2, 100, SR) == 1


def test_declared_twice(pkg, host):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    cv = c.create_convolver()
    cv.set_device_response(2, 1000, SR)
    st, text = status_and_text(pkg, lambda: cv.set_device_response(2, 1000, SR))
    assert st == 2 and "already bound from device memory" in text


def test_set_buffer_after_declaration(pkg, host):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    cv = c.create_convolver()
    cv.set_device_response(2, 1000, SR)
    st, text = status_and_text(pkg, lambda: cv.set_buffer(pkg.AudioBuffer(full_ir(2, 1000), SR)))
    assert st == 2 and "wae_convolver_set_device_response" in text


@pytest.mark.parametrize("via_options", [False, True])
def test_declaration_after_set_buffer(pkg, host, via_options):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    if via_options:
        cv = c.create_convolver(pkg.AudioBuffer(full_ir(2, 1000), SR))
    else:
        cv = c.create_convolver()
        cv.set_buffer(pkg.AudioBuffer(full_ir(2, 1000), SR))
    st, text = status_and_text(pkg, lambda: cv.set_device_response(2, 1000, SR))
    assert st == 2 and "already has a response" in text


def test_declaration_after_suspend_point(pkg, host):
    c = pkg.OfflineAudioContext(2, 4 * BLOCK, SR, host)
    cv = c.create_convolver()
    cv.connect(c.destination())
    c.suspend_sync(BLOCK / SR, lambda ctx: cv.set_device_response(2, 1000, SR))
    st, text = status_and_text(pkg, lambda: pkg.plan_batch([c]))
    assert st == 2 and "before the first suspend point" in text


def test_suspend_points_after_declaration(pkg, host):
    """allowed at multiples of 8192 frames, as for any ConvolverNode; elsewhere refused by the existing rule"""
    c, _ = conv_graph(pkg, host, 0, 4 * BLOCK, 2, 20000)
    c.suspend_sync(2 * BLOCK / SR, lambda ctx: None)
    assert pkg.plan_batch([c])["segments"] == 2
    d, _ = conv_graph(pkg, host, 0, 4 * BLOCK, 2, 20000)
    d.suspend_sync(100 * 128 / SR, lambda ctx: None)
    with pytest.raises(pkg._binding.WaeError) as e:
        pkg.plan_batch([d])
    assert e.value.status == 4


def test_normalize_fixed_at_declaration(pkg, host):
    """set_normalize after the declaration changes nothing (as after set_buffer): the plan is the same either way"""
    c, cv = conv_graph(pkg, host, 0, 30000, 2, 20000, normalize=True)
    cv.set_normalize(False)
    assert pkg.plan_batch([c]) == pkg.plan_batch([conv_graph(pkg, host, 0, 30000, 2, 20000, normalize=True)[0]])


def test_feedback_cycle_refused(pkg, host):
    c = pkg.OfflineAudioContext(2, 8192, SR, host)
    s = c.create_buffer_source(pkg.AudioBuffer(list(np.ones((2, 100), np.float32)), SR))
    cv = c.create_convolver()
    cv.set_device_response(2, 2000, SR)
    d = c.create_delay(1.0, delay_time=0.01)
    g = c.create_gain(0.5)
    s.connect(cv)
    cv.connect(d)
    d.connect(g)
    g.connect(cv)
    cv.connect(c.destination())
    s.start()
    st, text = status_and_text(pkg, lambda: pkg.plan_batch([c]))
    assert st == 4 and "feedback cycle" in text


def test_oracle_refuses(pkg, oracle):
    c = pkg.OfflineAudioContext(2, 1024, SR, oracle)
    with pytest.raises(pkg._binding.WaeError):
        c.create_convolver().set_device_response(2, 100, SR)


def test_oneshot_refusals(pkg, host):
    api = pkg.api()
    cs = [conv_graph(pkg, host, g, 4096, 2, 3000)[0] for g in range(2)]
    arr = (ctypes.c_void_p * 2)(*[c._g for c in cs])
    out = np.zeros((2, 2, 4096), np.float32)
    assert api.render_batch(None, arr, 2, out.ctypes.data_as(ctypes.c_void_p), 0) == 2
    assert b"wae_batch_bind_responses" in api.last_error()
    outs = (pkg._binding.c_float_p * 2)(*[pkg._binding.fptr(out[i]) for i in range(2)])
    assert api.render_many(None, arr, 2, outs) == 2
    assert b"wae_batch_bind_responses" in api.last_error()
    assert api.batch_bind_responses(None, None, 0, None) == 1


def test_response_binding_layout(pkg, tmp_path):
    B = pkg._binding
    assert "wae_convolver_set_device_response" in B.WAE_SYMBOLS and "wae_batch_bind_responses" in B.WAE_SYMBOLS
    src = tmp_path / "binding.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "wae.h"\nint main(void) {\n'
                   '  printf("%zu %zu %zu %zu %zu\\n", sizeof(wae_response_binding), offsetof(wae_response_binding, graph_index),\n'
                   '         offsetof(wae_response_binding, node), offsetof(wae_response_binding, pcm), offsetof(wae_response_binding, channel_stride));\n'
                   "  return 0;\n}\n")
    exe = tmp_path / "binding"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = tuple(map(int, subprocess.check_output([str(exe)], text=True).split()))
    S = B.ResponseBinding
    assert got == (ctypes.sizeof(S), S.graph_index.offset, S.node.offset, S.pcm.offset, S.channel_stride.offset)
    if not os.path.exists(LIB):
        pytest.skip("libwae_b200.so is not built")
    lib = ctypes.CDLL(LIB)
    assert hasattr(lib, "wae_convolver_set_device_response") and hasattr(lib, "wae_batch_bind_responses")


# ---------------------------------------------------------------------------------------------------------- plans
PLAN_CASES = [(ch, n, 2, "fixed") for ch in (1, 2, 4) for n in (BLOCK * 2 - 300, BLOCK * 2, BLOCK * 2 + 300)] + [
    (1, 5000, 1, "fixed"), (2, 20000, 1, "fixed"), (4, 20000, 1, "fixed"), (1, 17000, 2, "switch"), (1, BLOCK * 3, 2, "switch")]


def case_graphs(pkg, be, ch, n, in_ch, layout, declared, graphs=3, length=BLOCK * 4 + 500):
    return [conv_graph(pkg, be, g, length, ch, n, None if declared else full_ir(ch, n, seed=g), in_ch=in_ch, layout=layout)[0]
            for g in range(graphs)]


@pytest.mark.parametrize("ch,n,in_ch,layout", PLAN_CASES)
def test_plan_equals_host_response_of_declared_shape(pkg, host, ch, n, in_ch, layout):
    declared = pkg.plan_batch(case_graphs(pkg, host, ch, n, in_ch, layout, True))
    plain = pkg.plan_batch(case_graphs(pkg, host, ch, n, in_ch, layout, False))
    assert declared == plain


def test_switching_layout_gets_the_compacted_path(pkg, host):
    plain = pkg.plan_batch(case_graphs(pkg, host, 1, 17000, 2, "switch", False))
    declared = pkg.plan_batch(case_graphs(pkg, host, 1, 17000, 2, "switch", True))
    fixed = pkg.plan_batch(case_graphs(pkg, host, 1, 17000, 2, "fixed", True))
    assert declared == plain and declared["kinds"] != fixed["kinds"]


DIGEST_SCRIPT = textwrap.dedent("""
    import sys
    sys.path.insert(0, {tests!r}); sys.path.insert(0, {root!r})
    from conftest import load_package
    import test_device_responses_cpu as T
    pkg = load_package()
    be = pkg.context.Backend(pkg.api(), None)
    for case in T.PLAN_CASES:
        pkg.plan_batch(T.case_graphs(pkg, be, *case, sys.argv[1] == "declared"))
""")


def test_plan_digest_equals_host_response_of_declared_shape(pkg, host):
    script = DIGEST_SCRIPT.format(tests=os.path.join(ROOT, "tests"), root=ROOT)
    env = dict(os.environ, WAE_PLAN_DIGEST="1")
    out = {}
    for mode in ("declared", "plain"):
        r = subprocess.run([sys.executable, "-c", script, mode], env=env, capture_output=True, text=True, check=True)
        out[mode] = [line for line in r.stderr.splitlines() if "[wae plan digest]" in line]
    assert len(out["declared"]) >= len(PLAN_CASES) and out["declared"] == out["plain"]
