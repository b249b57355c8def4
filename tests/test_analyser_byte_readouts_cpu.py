"""AnalyserNode byte read-outs at declared render times (wae_analyser_set_byte_readouts), what needs no GPU: the declaration's refusals, the
header, the planned stages, and the oracle's get_byte_* in suspend callbacks against the reference's byte formulas (analysis.rs:266-276,
371-401) applied in f32 to the oracle's own float read-outs at the same quanta."""
import ctypes
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

import test_analyser_readouts_cpu as RC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RQ = 128
NEW_SYMBOLS = ["wae_analyser_set_byte_readouts", "wae_batch_analyser_byte_readouts_device_ptr", "wae_batch_fetch_analyser_byte_readouts"]
FREQ, TIME = 1, 2
F32 = np.float32


def byte_frequency(db, min_db, max_db):
    """get_byte_frequency_data (analysis.rs:390-398) of dB rows: (u8) clamp(255 / (max - min) * (dB - min), 0, 255) in f32"""
    db = np.asarray(db, F32)
    with np.errstate(invalid="ignore", over="ignore"):
        scaled = F32(255) / (F32(max_db) - F32(min_db)) * (db - F32(min_db))
    return np.where(np.isnan(scaled), 0, np.clip(scaled, 0, 255)).astype(np.uint8)


def byte_time_domain(x):
    """get_byte_time_domain_data (analysis.rs:266-276): (u8) clamp(128 (1 + x), 0, 255) in f32; `as u8` maps NaN to 0"""
    scaled = F32(128) * (F32(1) + np.asarray(x, F32))
    return np.where(np.isnan(scaled), 0, np.clip(scaled, 0, 255)).astype(np.uint8)


def declare_bytes(be, c, node, kinds):
    return be.api.analyser_set_byte_readouts(c._g, node, kinds)


def test_refusals(pkg, be_product):
    be = be_product
    c, a, osc = RC.graph(pkg, be)
    assert declare_bytes(be, c, a.id, FREQ) == 2                    # before set_readouts
    assert RC.declare(be, c, a.id, [0.0, 0.001], FREQ) == 0
    assert declare_bytes(be, c, osc.id, FREQ) == 1                  # not an analyser
    assert declare_bytes(be, c, a.id, 0) == 1 and declare_bytes(be, c, a.id, 4) == 1
    assert declare_bytes(be, c, a.id, TIME) == 1                    # a kind the read-outs do not declare
    assert declare_bytes(be, c, a.id, FREQ | TIME) == 1
    assert declare_bytes(be, c, a.id, FREQ) == 0
    assert declare_bytes(be, c, a.id, FREQ) == 2                    # a second declaration
    assert be.api.graph_suspend(c._g, 0.002) == 2                   # a suspend point after a declaration
    c2, a2, _ = RC.graph(pkg, be)
    assert be.api.graph_suspend(c2._g, 0.002) == 0
    assert declare_bytes(be, c2, a2.id, FREQ) == 2                  # a graph with a suspend point


def test_new_symbols_declared_exported_and_c99(pkg, be_product):
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


@pytest.mark.parametrize("byte_kinds", [FREQ, TIME, FREQ | TIME])
def test_plan_is_the_float_declaration_plan(pkg, be_product, byte_kinds):
    # byte rows are written by the float read-outs' own kernels: the stages are those of the float declaration
    def ctxs(with_bytes):
        out = []
        for _ in range(4):
            c, a, _ = RC.graph(pkg, be_product)
            a.set_readouts([0.0, 0.001, 0.001, 40 * RQ / 48000.0], frequency=True, time_domain=True)
            if with_bytes:
                a.set_byte_readouts(frequency=bool(byte_kinds & FREQ), time_domain=bool(byte_kinds & TIME))
            out.append(c)
        return out
    assert pkg.context.plan_batch(ctxs(True))["kinds"] == pkg.context.plan_batch(ctxs(False))["kinds"]


@pytest.fixture
def be_product(pkg):
    so = os.path.join(ROOT, "web-audio-api-rs_b200", "libwae_b200.so")
    if not os.path.exists(so):
        pytest.skip("libwae_b200.so is not built (python -c 'import __graft_entry__ as g; g.build()')")
    return pkg.context.Backend(pkg.api(), None)


# ---- the oracle's byte read-outs in suspend callbacks against the formulas ------------------------------------------------------------
def oracle_all_readouts(pkg, backend, build, times):
    """float and byte read-outs the reference's API gives at suspend_sync(t) for each declared time (the end quantum: after the render):
    (freq dB, time, byte freq, byte time) rows in time order.  Per read-out the float frequency call comes first and the byte one reuses
    its smoothing step (the same current_time: last_fft_time, analysis.rs:347-361)."""
    rows = [[], [], [], []]

    def take(a):
        rows[0].append(a.get_float_frequency_data().copy())
        rows[1].append(a.get_float_time_domain_data().copy())
        rows[2].append(a.get_byte_frequency_data().copy())
        rows[3].append(a.get_byte_time_domain_data().copy())

    c, a = build(backend)
    total = -(-c._length // RQ)
    quanta = [math.ceil(t * c._sample_rate / RQ) for t in times]
    by_q = {}
    for t, q in zip(times, quanta):
        if q < total:
            by_q.setdefault(q, []).append(t)
    for q, ts in sorted(by_q.items()):
        c.suspend_sync(ts[0], lambda ctx, n=len(ts): [take(a) for _ in range(n)])
    c.start_rendering_sync()
    for q in quanta:
        if q == total:
            take(a)
    return [np.array(r) for r in rows], quanta


def loud_graph(pkg, length, sr, fft_size, tau, min_db=-100.0, max_db=-30.0, amp=1.5):
    """a buffer source of noise and a sine, loud enough that time-domain bytes clip at both ends and spectra pass max_db"""
    rng = np.random.default_rng(fft_size)
    sig = (amp * np.sin(2 * np.pi * 1500.0 * np.arange(length) / sr) + 0.2 * rng.uniform(-1, 1, length)).astype(np.float32)

    def build(backend):
        c = pkg.OfflineAudioContext(1, length, sr, backend)
        src = c.create_buffer_source(pkg.AudioBuffer([sig], sr))
        a = c.create_analyser(fft_size=fft_size, smoothing_time_constant=tau)
        a.set_min_decibels(min_db)
        a.set_max_decibels(max_db)
        src.connect(a)
        a.connect(c.destination())
        src.start()
        return c, a
    return build


@pytest.mark.parametrize("fft_size,tau,min_db,max_db", [(32, 0.0, -100.0, -30.0), (256, 0.8, -60.0, -20.0), (2048, 0.8, -100.0, -30.0)])
def test_oracle_byte_readouts_are_the_formulas_of_its_float_readouts(pkg, oracle, fft_size, tau, min_db, max_db):
    sr, length = 44100.0, RQ * 60
    times = [q * RQ / sr for q in (0, 3, 3, 17, 40, 59, 60)]
    (f, t, bf, bt), _ = oracle_all_readouts(pkg, oracle, loud_graph(pkg, length, sr, fft_size, tau, min_db, max_db), times)
    assert np.array_equal(bf, byte_frequency(f, min_db, max_db))
    assert np.array_equal(bt, byte_time_domain(t))
    assert (bt == 255).any() and (bt == 0).any() and (bf == 255).any() and (bf[0] == 0).all()
