"""IIRFilterNode coefficients bound from device memory, on the host (no GPU): the declaration rules of
wae_iir_filter_set_device_coefficients, the refusals (oracle backend, one-shot calls, get_frequency_response), the wae_iir_binding layout
of include/wae.h, and plans of graphs with declared filters.  The planner picks an IIR filter's path from its coefficient counts only, so a
declared filter plans exactly as the node it was constructed as: the same plan_batch / plan_many dicts and the same WAE_PLAN_DIGEST lines,
on the chain path (order 1 and 2, extended by a biquad and a gain, and destination-direct), on the serial path (behind a late-starting
input, 3 / 8 / 20 coefficients, suspend points) and for a batch of mixed shapes.  (wae_batch_plan plans with the default options; the
serial path under WAE_OPT_SERIAL_FILTERS is planned by an engine, tests/test_gpu_device_iir.py.)"""
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


@pytest.fixture
def host(pkg):
    if not os.path.exists(LIB):
        pytest.skip("libwae_b200.so is not built (python -c 'import __graft_entry__ as g; g.build()')")
    return pkg.context.Backend(pkg.api(), None)


def status_and_text(pkg, fn):
    with pytest.raises(pkg._binding.WaeError) as e:
        fn()
    return e.value.status, e.value.message


def stable_filter(seed, nff, nfb):
    """(feedforward, feedback) of a stable filter: the feedback of a Butterworth or Chebyshev low-pass of order nfb - 1, the feedforward
    that filter's numerator (zero-padded or cut to nff), both scaled so that feedback[0] is not 1 (the coefficients are normalised)"""
    from scipy import signal
    rng = np.random.default_rng(seed)
    order = max(nff, nfb) - 1
    if order == 0:
        b, a = np.array([rng.uniform(0.2, 0.9)]), np.array([1.0])
    elif seed % 2:
        b, a = signal.cheby1(order, 0.5, rng.uniform(0.15, 0.6))
    else:
        b, a = signal.butter(order, rng.uniform(0.1, 0.6))
    ff = np.zeros(nff)
    ff[: min(nff, len(b))] = b[:nff]
    if not ff.any():
        ff[0] = 0.5
    fb = np.array(a[:nfb], np.float64)
    if nfb < len(a):  # (a shorter feedback: a filter of its own, still stable)
        fb = np.array(signal.butter(nfb - 1, 0.3)[1] if nfb > 1 else [1.0])
    scale = rng.uniform(0.5, 3.0)
    return ff * scale, fb * scale


def iir_graph(pkg, be, g, length, nff, nfb, coefs=None, path="chain", channels=2, suspends=(), pcm=None):
    """buffer source -> IIRFilterNode (nff / nfb coefficients) [-> lowpass -> gain] -> destination, per path:
    chain: source -> IIR -> lowpass -> gain -> destination (the IIR opens a k_chain when its order is <= 2);
    dest: source -> IIR -> destination (the chain writes the rendered PCM itself);
    late: the source starts at 0.05 s (an input that may be silent: k_iir_serial);
    stop: the source stops at 0.1 s (k_iir_serial);
    switch: a mono source plays throughout and a stereo one from 0.05 s to 0.1 s (the input switches between one and two channels);
    suspend: chain, with suspend points at 3072 and 8192 frames added after the declaration.
    coefs: the (feedforward, feedback) the node is constructed with and not declared, or None: declared, constructed with the
    identity (1, 0, ...) / (1, 0, ...).  Returns (context, iir node)."""
    c = pkg.OfflineAudioContext(2, length, SR, be)
    rng = np.random.default_rng(1000 + g)
    if pcm is None:
        pcm = (rng.uniform(-1, 1, (channels, length)) * 0.5).astype(np.float32)
    src = c.create_buffer_source(pkg.AudioBuffer(list(pcm), SR))
    if coefs is None:
        f = c.create_iir_filter([1.0] + [0.0] * (nff - 1), [1.0] + [0.0] * (nfb - 1))
        f.set_device_coefficients()
    else:
        f = c.create_iir_filter(list(coefs[0]), list(coefs[1]))
    src.connect(f)
    if path in ("chain", "suspend"):
        bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=3000.0 + 200 * g, q=0.9)
        gn = c.create_gain(0.7)
        f.connect(bq)
        bq.connect(gn)
        gn.connect(c.destination())
    elif path == "dest":
        f.connect(c.destination())
    else:
        gn = c.create_gain(0.8)
        f.connect(gn)
        gn.connect(c.destination())
    if path == "late":
        src.start_at(0.05)
    elif path == "stop":
        src.start()
        src.stop_at(0.1)
    elif path == "switch":
        src.start()
        st = c.create_buffer_source(pkg.AudioBuffer(list((rng.uniform(-1, 1, (2, length)) * 0.5).astype(np.float32)), SR))
        st.connect(f)
        st.start_at(0.05)
        st.stop_at(0.1)
    else:
        src.start()
    for fr in suspends or ((3072, 8192) if path == "suspend" else ()):
        c.suspend_sync(fr / SR, lambda ctx: None)
    return c, f


# ---------------------------------------------------------------------------------------------------------- declaration rules
def test_not_an_iir_filter(pkg, host):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    api = pkg.api()
    assert api.iir_filter_set_device_coefficients(c._g, c.create_gain().id) == 1
    assert b"not an IIRFilterNode" in api.last_error()
    assert api.iir_filter_set_device_coefficients(c._g, c.create_biquad_filter().id) == 1
    assert api.iir_filter_set_device_coefficients(c._g, 9999) == 1


def test_declared_twice(pkg, host):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    f = c.create_iir_filter([1.0, 0.5], [1.0, -0.2])
    f.set_device_coefficients()
    assert status_and_text(pkg, f.set_device_coefficients) == (
        2, "InvalidStateError - the coefficients are already bound from device memory (wae_iir_filter_set_device_coefficients)")


def test_declaration_after_suspend_point(pkg, host):
    c = pkg.OfflineAudioContext(2, 4096, SR, host)
    f = c.create_iir_filter([1.0, 0.5], [1.0, -0.2])
    f.connect(c.destination())
    c.suspend_sync(1024 / SR, lambda ctx: f.set_device_coefficients())
    assert status_and_text(pkg, lambda: pkg.plan_batch([c])) == (
        2, "InvalidStateError - IIR coefficients are bound from device memory before the first suspend point")


def test_suspend_points_after_declaration(pkg, host):
    c, _ = iir_graph(pkg, host, 0, 12000, 3, 3, path="suspend")
    p = pkg.plan_batch([c])
    assert p["segments"] == 3 and "k_iir_serial" in p["kinds"], p


def test_oracle_refuses(pkg, oracle):
    c = pkg.OfflineAudioContext(2, 1024, SR, oracle)
    with pytest.raises(pkg._binding.WaeError) as e:
        c.create_iir_filter([1.0, 0.5], [1.0, -0.2]).set_device_coefficients()
    assert e.value.status == 3


def test_frequency_response_refused(pkg, host):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    plain = c.create_iir_filter([1.0, 0.5], [1.0, -0.2])
    f = c.create_iir_filter([1.0, 0.5], [1.0, -0.2])
    f.set_device_coefficients()
    freqs = np.array([100.0, 1000.0], np.float32)
    mag, _ = plain.get_frequency_response(freqs)
    assert np.isfinite(mag).all()
    with pytest.raises(pkg._binding.WaeError) as e:
        f.get_frequency_response(freqs)
    assert e.value.status == 2 and "device memory" in e.value.message


def test_oneshot_refusals(pkg, host):
    api = pkg.api()
    cs = [iir_graph(pkg, host, g, 4096, 3, 3)[0] for g in range(2)]
    arr = (ctypes.c_void_p * 2)(*[c._g for c in cs])
    out = np.zeros((2, 2, 4096), np.float32)
    assert api.render_batch(None, arr, 2, out.ctypes.data_as(ctypes.c_void_p), 0) == 2
    assert api.last_error() == (b"graph 0 has IIR coefficients bound from device memory: render it with wae_batch_prepare "
                                b"(or _prepare_many), wae_batch_bind_iir_coefficients and wae_batch_run")
    outs = (pkg._binding.c_float_p * 2)(*[pkg._binding.fptr(out[i]) for i in range(2)])
    assert api.render_many(None, arr, 2, outs) == 2
    assert b"wae_batch_bind_iir_coefficients" in api.last_error()
    assert api.batch_bind_iir_coefficients(None, None, 0, None) == 1
    with pytest.raises(pkg._binding.WaeError) as e:
        pkg.render_batch_oneshot(cs)
    assert e.value.status == 2
    with pytest.raises(pkg._binding.WaeError) as e:
        pkg.render_many(cs)
    assert e.value.status == 2


def test_iir_binding_layout(pkg, tmp_path):
    B = pkg._binding
    assert "wae_iir_filter_set_device_coefficients" in B.WAE_SYMBOLS and "wae_batch_bind_iir_coefficients" in B.WAE_SYMBOLS
    src = tmp_path / "binding.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "wae.h"\nint main(void) {\n'
                   '  printf("%zu %zu %zu %zu %zu\\n", sizeof(wae_iir_binding), offsetof(wae_iir_binding, graph_index),\n'
                   '         offsetof(wae_iir_binding, node), offsetof(wae_iir_binding, feedforward),\n'
                   '         offsetof(wae_iir_binding, feedback));\n'
                   "  return 0;\n}\n")
    exe = tmp_path / "binding"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    got = tuple(map(int, subprocess.check_output([str(exe)], text=True).split()))
    S = B.IirBinding
    assert got == (ctypes.sizeof(S), S.graph_index.offset, S.node.offset, S.feedforward.offset, S.feedback.offset)
    if not os.path.exists(LIB):
        pytest.skip("libwae_b200.so is not built")
    lib = ctypes.CDLL(LIB)
    assert hasattr(lib, "wae_iir_filter_set_device_coefficients") and hasattr(lib, "wae_batch_bind_iir_coefficients")


# ---------------------------------------------------------------------------------------------------------- plans
# (name, path, nff, nfb, channels, the kernel the IIR filter lands in)
CASES = [
    ("order1_chain", "chain", 2, 2, 2, "k_chain"),
    ("order2_chain", "chain", 3, 3, 2, "k_chain"),
    ("order2_chain_mono", "chain", 3, 2, 1, "k_chain"),
    ("order2_dest", "dest", 3, 3, 2, "k_chain"),
    ("order2_late", "late", 3, 3, 2, "k_iir_serial"),
    ("order2_stop", "stop", 2, 3, 2, "k_iir_serial"),
    ("order2_switch", "switch", 3, 3, 1, "k_iir_serial"),
    ("coef3", "chain", 3, 1, 2, "k_chain"),
    ("coef8", "chain", 8, 8, 2, "k_iir_serial"),
    ("coef8_ff4", "late", 4, 8, 2, "k_iir_serial"),
    ("coef20", "chain", 20, 20, 2, "k_iir_serial"),
    ("suspend", "suspend", 3, 3, 2, "k_iir_serial"),
]
CASE_NAMES = [c[0] for c in CASES]


def case_graphs(pkg, be, name, declared, graphs=3, length=12000):
    _, path, nff, nfb, channels, _ = dict((c[0], c) for c in CASES)[name]
    out = []
    for g in range(graphs):
        coefs = None if declared else ([1.0] + [0.0] * (nff - 1), [1.0] + [0.0] * (nfb - 1))
        out.append(iir_graph(pkg, be, g, length, nff, nfb, coefs, path, channels)[0])
    return out


def mixed_graphs(pkg, be, declared):
    """graphs of three shapes (length, channel count), each with a chain-path and a serial-path filter"""
    out = []
    for g, (length, channels) in enumerate([(12000, 2), (12000, 1), (30000, 2), (9600, 2), (30000, 1)]):
        nff, nfb = (3, 3) if g % 2 == 0 else (8, 5)
        c = pkg.OfflineAudioContext(channels, length, SR, be)
        src = c.create_buffer_source(pkg.AudioBuffer([np.full(length, 0.25, np.float32)] * 2, SR))
        f = c.create_iir_filter([1.0] + [0.0] * (nff - 1), [1.0] + [0.0] * (nfb - 1))
        if declared:
            f.set_device_coefficients()
        src.connect(f)
        f.connect(c.destination())
        src.start()
        out.append(c)
    return out


@pytest.mark.parametrize("name", CASE_NAMES)
def test_plan_equals_constructed_node(pkg, host, name):
    declared = pkg.plan_batch(case_graphs(pkg, host, name, True))
    kernel = dict((c[0], c[5]) for c in CASES)[name]
    assert kernel in declared["kinds"], declared["kinds"]
    assert declared == pkg.plan_batch(case_graphs(pkg, host, name, False))


def test_plan_many_equals_constructed_nodes(pkg, host):
    declared = pkg.plan_many(mixed_graphs(pkg, host, True))
    assert declared["groups"] >= 2, declared
    assert declared == pkg.plan_many(mixed_graphs(pkg, host, False))


def test_never_started_and_unconnected_declared_filters_are_planned(pkg, host):
    c, _ = iir_graph(pkg, host, 0, 4096, 3, 3)
    idle_src = c.create_buffer_source(pkg.AudioBuffer([np.ones(4096, np.float32)], SR))
    idle = c.create_iir_filter([1.0, 0.0, 0.0], [1.0, 0.0, 0.0])
    idle.set_device_coefficients()
    idle_src.connect(idle)
    idle.connect(c.destination())  # never started
    c.create_iir_filter([1.0] * 8, [1.0] + [0.0] * 7).set_device_coefficients()  # not connected
    pkg.plan_batch([c])


DIGEST_SCRIPT = textwrap.dedent("""
    import sys
    sys.path.insert(0, {tests!r}); sys.path.insert(0, {root!r})
    from conftest import load_package
    import test_device_iir_cpu as T
    pkg = load_package()
    be = pkg.context.Backend(pkg.api(), None)
    declared = sys.argv[1] == "declared"
    for name in T.CASE_NAMES:
        pkg.plan_batch(T.case_graphs(pkg, be, name, declared))
    pkg.plan_many(T.mixed_graphs(pkg, be, declared))
""")


def test_plan_digest_equals_constructed_node(pkg, host):
    script = DIGEST_SCRIPT.format(tests=os.path.join(ROOT, "tests"), root=ROOT)
    env = dict(os.environ, WAE_PLAN_DIGEST="1")
    out = {}
    for mode in ("declared", "plain"):
        r = subprocess.run([sys.executable, "-c", script, mode], env=env, capture_output=True, text=True, check=True)
        out[mode] = [line for line in r.stderr.splitlines() if "[wae plan digest]" in line]
    assert len(out["declared"]) >= len(CASES) + 2 and out["declared"] == out["plain"]
