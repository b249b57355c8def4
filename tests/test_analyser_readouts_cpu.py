"""AnalyserNode read-outs at declared render times (wae_analyser_set_readouts), what needs no GPU: the declaration's refusals, the
header, the planned stages, and the oracle's read-outs in suspend callbacks (what the GPU read-outs are checked against) against an f64
numpy statement of Blackman window -> rfft -> |X| / N with the reference's f32 smoothing recurrence."""
import ctypes
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RQ = 128
NEW_SYMBOLS = ["wae_analyser_set_readouts", "wae_batch_analyser_readouts_device_ptr", "wae_batch_fetch_analyser_readouts"]
FREQ, TIME = 1, 2


@pytest.fixture
def be(pkg):
    so = os.path.join(ROOT, "web-audio-api-rs_b200", "libwae_b200.so")
    if not os.path.exists(so):
        pytest.skip("libwae_b200.so is not built (python -c 'import __graft_entry__ as g; g.build()')")
    return pkg.context.Backend(pkg.api(), None)


def graph(pkg, be, length=RQ * 40, sr=48000.0, fft_size=256):
    c = pkg.OfflineAudioContext(2, length, sr, be)
    osc = c.create_oscillator(frequency=1000.0)
    a = c.create_analyser(fft_size=fft_size)
    osc.connect(a)
    a.connect(c.destination())
    osc.start()
    return c, a, osc


def declare(be, c, node, times, kinds=FREQ):
    t = np.ascontiguousarray(times, np.float64)
    return be.api.analyser_set_readouts(c._g, node, t.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), len(t), kinds)


def test_refusals(pkg, be):
    c, a, osc = graph(pkg, be)
    end = 40 * RQ / 48000.0
    assert declare(be, c, osc.id, [0.0]) == 1                      # not an analyser
    assert declare(be, c, a.id, []) == 1                           # n == 0
    for bad in ([-1e-3], [float("nan")], [float("inf")], [0.01, 0.005], [end + 1e-4]):
        assert declare(be, c, a.id, bad) == 1, bad
    assert declare(be, c, a.id, [0.0], 0) == 1 and declare(be, c, a.id, [0.0], 4) == 1 and declare(be, c, a.id, [0.0], 7) == 1
    assert declare(be, c, a.id, [0.0, 0.0, end], FREQ | TIME) == 0  # quantum 0, a duplicate, the end quantum
    assert declare(be, c, a.id, [0.001]) == 2                      # a second declaration
    assert be.api.graph_suspend(c._g, 0.002) == 2                  # a suspend point after a declaration
    c2, a2, _ = graph(pkg, be)
    assert be.api.graph_suspend(c2._g, 0.002) == 0
    assert declare(be, c2, a2.id, [0.001]) == 2                    # a declaration after a suspend point


def test_one_shot_renders_refuse_a_declaration(pkg, be):
    c, a, _ = graph(pkg, be)
    a.set_readouts([0.001])
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
    src = "#include \"wae.h\"\nint main(void) { wae_status (*f[])() = {%s}; return (int)sizeof f + WAE_READOUT_FREQUENCY + " \
          "WAE_READOUT_TIME_DOMAIN; }\n" % ", ".join("(wae_status (*)())" + s for s in NEW_SYMBOLS)
    r = subprocess.run([cc, "-std=c99", "-pedantic", "-Wall", "-Werror", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), "-x", "c", "-"],
                       input=src, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


@pytest.mark.parametrize("kinds,new", [(FREQ, {"k_readout_fft": 1, "k_readout_smooth": 1}), (TIME, {"k_readout_time": 1}),
                                       (FREQ | TIME, {"k_readout_fft": 1, "k_readout_smooth": 1, "k_readout_time": 1})])
def test_plan_is_the_twin_plus_the_readout_stages(pkg, be, kinds, new):
    twin = pkg.context.plan_batch([graph(pkg, be)[0] for _ in range(4)])
    ctxs = []
    for _ in range(4):
        c, a, _ = graph(pkg, be)
        a.set_readouts([0.0, 0.001, 0.001, 40 * RQ / 48000.0], frequency=bool(kinds & FREQ), time_domain=bool(kinds & TIME))
        ctxs.append(c)
    got = pkg.context.plan_batch(ctxs)
    want = dict(twin["kinds"])
    for k, n in new.items():
        want[k] = want.get(k, 0) + n
    assert got["kinds"] == want


# ---- the oracle's read-outs in suspend callbacks against numpy ----------------------------------------------------------------------
def blackman_rfft_mag(window):
    """|rfft(window x Blackman)| / N, bins 0 .. N/2 - 1, in f64 (analysis.rs:13-24, 278-333)"""
    n = len(window)
    i = np.arange(n)
    w = 0.42 - 0.5 * np.cos(2 * np.pi * i / n) + 0.08 * np.cos(4 * np.pi * i / n)
    return np.abs(np.fft.rfft(np.asarray(window, np.float64) * w))[:n // 2] / n


def numpy_readouts(signal, quanta, fft_size, tau):
    """frequency (dB) and time-domain rows of read-outs at the given quanta of a mono signal: the window is the fft_size frames before
    q * 128 (zeros before the start); the smoothing recurrence in f32, a repeated quantum repeats the row"""
    padded = np.concatenate([np.zeros(fft_size, np.float32), np.asarray(signal, np.float32)])
    last = np.zeros(fft_size // 2, np.float32)
    tau32 = np.float32(tau)
    freq, time, prev_q, row = [], [], None, None
    for q in quanta:
        win = padded[q * RQ:q * RQ + fft_size]
        time.append(win.copy())
        if q != prev_q:
            mag = blackman_rfft_mag(win).astype(np.float32)
            with np.errstate(divide="ignore"):
                last = tau32 * last + (np.float32(1) - tau32) * mag
                row = (20 * np.log10(last.astype(np.float64))).astype(np.float32)
            prev_q = q
        freq.append(row)
    return np.array(freq), np.array(time)


def oracle_readouts(pkg, backend, build, times):
    """Read-outs the reference's API gives at suspend_sync(t) for each declared time (the end quantum: after the render): frequency and
    time-domain rows, in time order.  `build(ctx) -> analyser`."""
    rows_f, rows_t = [], []

    def take(a):
        rows_f.append(a.get_float_frequency_data().copy())
        rows_t.append(a.get_float_time_domain_data().copy())

    c, a = build(backend)
    total = -(-c._length // RQ)
    quanta = [math.ceil(t * c._sample_rate / RQ) for t in times]
    at_end = [t for t, q in zip(times, quanta) if q == total]
    by_q = {}
    for t, q in zip(times, quanta):
        if q < total:
            by_q.setdefault(q, []).append(t)
    for q, ts in sorted(by_q.items()):
        c.suspend_sync(ts[0], lambda ctx, n=len(ts): [take(a) for _ in range(n)])
    c.start_rendering_sync()
    for _ in at_end:
        take(a)
    return np.array(rows_f), np.array(rows_t), quanta


@pytest.mark.parametrize("fft_size,tau", [(32, 0.0), (256, 0.8), (2048, 0.8)])
def test_oracle_readouts_vs_numpy(pkg, oracle, fft_size, tau):
    sr, length = 44100.0, RQ * 60
    rng = np.random.default_rng(fft_size)
    sig = (0.5 * np.sin(2 * np.pi * 1500.0 * np.arange(length) / sr) + 0.2 * rng.uniform(-1, 1, length)).astype(np.float32)

    def build(backend):
        c = pkg.OfflineAudioContext(1, length, sr, backend)
        src = c.create_buffer_source(pkg.AudioBuffer([sig], sr))
        a = c.create_analyser(fft_size=fft_size, smoothing_time_constant=tau)
        src.connect(a)
        a.connect(c.destination())
        src.start()
        return c, a

    times = [q * RQ / sr for q in (0, 3, 3, 17, 40, 59, 60)]
    got_f, got_t, quanta = oracle_readouts(pkg, oracle, build, times)
    want_f, want_t = numpy_readouts(sig, quanta, fft_size, tau)
    assert np.array_equal(got_t, want_t)
    loud = want_f > -90.0
    assert loud.sum() > 0
    assert np.abs(got_f[loud] - want_f[loud]).max() <= 2e-2
    assert np.array_equal(got_f[1], got_f[2])  # the same quantum: the same row, not smoothed again
    assert np.all(np.isneginf(got_f[0]))        # quantum 0: an all-zero window
