"""DynamicsCompressorNode reduction read-outs at declared render times (wae_compressor_set_readouts), what needs no GPU: the declaration's
refusals, the header, the planned stages, and the oracle's reduction() in suspend callbacks (what the GPU read-outs are checked against)
against the suite's f64 statement of the compressor (tests/test_gpu_witnesses_dynamics_spatial.py), evaluated up to each read-out's quantum."""
import ctypes
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

import test_gpu_witnesses_dynamics_spatial as W

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RQ = 128
NEW_SYMBOLS = ["wae_compressor_set_readouts", "wae_batch_compressor_readouts_device_ptr", "wae_batch_fetch_compressor_readouts"]


@pytest.fixture
def be(pkg):
    so = os.path.join(ROOT, "web-audio-api-rs_b200", "libwae_b200.so")
    if not os.path.exists(so):
        pytest.skip("libwae_b200.so is not built (python -c 'import __graft_entry__ as g; g.build()')")
    return pkg.context.Backend(pkg.api(), None)


def graph(pkg, be, length=RQ * 40, sr=48000.0):
    c = pkg.OfflineAudioContext(2, length, sr, be)
    osc = c.create_oscillator(frequency=1000.0)
    d = c.create_dynamics_compressor(threshold=-30.0)
    osc.connect(d)
    d.connect(c.destination())
    osc.start()
    return c, d, osc


def declare(be, c, node, times):
    t = np.ascontiguousarray(times, np.float64)
    return be.api.compressor_set_readouts(c._g, node, t.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), len(t))


def times_at(quanta, sr):
    # (half a frame before the quantum's first frame: ceil(t sr / 128) is exactly q, whatever the rounding of q * 128 / sr)
    return [max(q * RQ - 0.5, 0.0) / sr for q in quanta]


def test_refusals(pkg, be):
    c, d, osc = graph(pkg, be)
    end = 40 * RQ / 48000.0
    assert declare(be, c, osc.id, [0.0]) == 1                      # not a compressor
    assert declare(be, c, d.id, []) == 1                           # n == 0
    for bad in ([-1e-3], [float("nan")], [float("inf")], [0.01, 0.005], [end + 1e-4]):
        assert declare(be, c, d.id, bad) == 1, bad
    assert declare(be, c, d.id, [0.0, 0.0, end]) == 0              # quantum 0, a duplicate, the end quantum
    assert declare(be, c, d.id, [0.001]) == 2                      # a second declaration
    assert be.api.graph_suspend(c._g, 0.002) == 2                  # a suspend point after a declaration
    assert b"compressor read-outs" in be.api.last_error()
    c2, d2, _ = graph(pkg, be)
    assert be.api.graph_suspend(c2._g, 0.002) == 0
    assert declare(be, c2, d2.id, [0.001]) == 2                    # a declaration after a suspend point


def test_one_shot_renders_refuse_a_declaration(pkg, be):
    c, d, _ = graph(pkg, be)
    d.set_readouts([0.001])
    arr = (ctypes.c_void_p * 1)(c._g)
    out = np.zeros((1, 2, c._length), np.float32)
    assert be.api.render_batch(None, arr, 1, out.ctypes.data_as(ctypes.c_void_p), 0) == 2
    outs = (ctypes.POINTER(ctypes.c_float) * 1)(out[0].ctypes.data_as(ctypes.POINTER(ctypes.c_float)))
    assert be.api.render_many(None, arr, 1, outs) == 2


def test_new_symbols_declared_exported_and_c99(pkg, be):
    header = open(os.path.join(ROOT, "include", "wae.h")).read()
    lib = ctypes.CDLL(os.path.join(ROOT, "web-audio-api-rs_b200", "libwae_b200.so"))
    for s in NEW_SYMBOLS:
        assert "WAE_API wae_status %s(" % s in header, s
        assert hasattr(lib, s), s
        assert s in pkg._binding.WAE_SYMBOLS, s
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler")
    src = "#include \"wae.h\"\nint main(void) { wae_status (*f[])() = {%s}; return (int)sizeof f; }\n" % \
          ", ".join("(wae_status (*)())" + s for s in NEW_SYMBOLS)
    r = subprocess.run([cc, "-std=c99", "-pedantic", "-Wall", "-Werror", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), "-x", "c", "-"],
                       input=src, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


@pytest.mark.parametrize("declared", [4, 2])
def test_plan_is_the_twin_plus_the_readout_stage(pkg, be, declared):
    # every compressor declared: the same stages (k_compressor<true> runs in the compressor's stage); some declared: the declared ones
    # take a k_compressor stage of their own next to the undeclared ones'
    twin = pkg.context.plan_batch([graph(pkg, be)[0] for _ in range(4)])
    ctxs = []
    for k in range(4):
        c, d, _ = graph(pkg, be)
        if k < declared:
            d.set_readouts([0.0, 0.001, 0.001, 40 * RQ / 48000.0])
        ctxs.append(c)
    got = pkg.context.plan_batch(ctxs)
    want = dict(twin["kinds"])
    if declared < 4:
        want["k_compressor"] += 1
    assert got["kinds"] == want
    for k in ("groups", "segments", "chunk_frames", "arena_floats_per_frame", "source_floats"):
        assert got[k] == twin[k], k


# ---- the oracle's reduction() in suspend callbacks against the f64 statement -----------------------------------------------------------
def oracle_reduction_readouts(pkg, backend, build, times):
    """reduction() at suspend_sync(t) for each declared time (the end quantum: after the render), in time order.  `build(ctx) -> node`."""
    got = []
    c, d = build(backend)
    total = -(-c._length // RQ)
    quanta = [math.ceil(t * c._sample_rate / RQ) for t in times]
    by_q = {}
    for t, q in zip(times, quanta):
        if q < total:
            by_q.setdefault(q, []).append(t)
    for q, ts in sorted(by_q.items()):
        c.suspend_sync(ts[0], lambda ctx, n=len(ts): [got.append(d.reduction()) for _ in range(n)])
    c.start_rendering_sync()
    for q in quanta:
        if q == total:
            got.append(d.reduction())
    return np.array(got, np.float32), quanta


def witness_readouts(comp, quanta):
    """the f64 statement's reduction at the last frame of quantum q - 1 for each read-out quantum q (0 before the first quantum)"""
    cut = sorted({q for q in quanta if q > 0})
    # (the statement of the first q quanta: a source that starts later plays no part in them)
    graphs = [W._Comp(comp.sr, q * RQ, [s for s in comp.srcs if s.a < q * RQ], comp.params, comp.steps) for q in cut]
    red = dict(zip(cut, (r for _, r in W._comp_witness(graphs)))) if cut else {}
    return np.array([red.get(q, 0.0) for q in quanta])


def witness_cases():
    """(name, _Comp): a constant input, an input switching between one and two channels, k-rate threshold / ratio steps"""
    rng = np.random.default_rng(11)
    sr, n = 48000.0, RQ * 96
    return [
        ("constant", W._Comp(sr, n, W._comp_inputs(rng, sr, n, 2, "constant"))),
        ("switch", W._Comp(sr, n, W._comp_inputs(rng, sr, n, 2, "switch"))),
        # (32768 Hz: a quantum is 2^-8 s, so the steps land exactly on quantum boundaries)
        ("steps", W._Comp(32768.0, RQ * 100, W._comp_inputs(rng, 32768.0, RQ * 100, 2, "late"), dict(release=0.05),
                          steps=[("threshold", 30, -50.0), ("ratio", 60, 3.0)])),
    ]


@pytest.mark.parametrize("case", range(3))
def test_oracle_reduction_readouts_vs_f64(pkg, oracle, case):
    name, comp = witness_cases()[case]
    total = comp.n // RQ
    quanta = [0, 1, 5, 5, 17, 31, 32, 61, total - 1, total]

    def build(backend):
        return comp.build(pkg, backend)
    got, q = oracle_reduction_readouts(pkg, oracle, build, times_at(quanta, comp.sr))
    assert q == quanta
    want = witness_readouts(comp, quanta)
    _, budget = W._comp_budget(comp.sr)
    assert got[0] == 0.0
    assert got[2] == got[3]
    assert np.all(np.abs(got - want) <= budget * np.maximum(1.0, np.abs(want) / 4)), (name, got, want)
    assert np.abs(want).max() > 1.0, name  # the compressor engages
