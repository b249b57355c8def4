"""OscillatorNode periodic waves bound from device memory (wae_oscillator_set_device_periodic_wave + wae_batch_bind_periodic_waves) on the
GPU.  A batch is planned once and run with coefficients bound from torch tensors.

The synthesised wavetable itself is read out through the oscillator: at frequency = sample_rate / table_len, started at 0, an
oscillator steps exactly one table entry per frame with interpolation weight 0, on both the 2048-point fixed-point path and the f64 path
of other lengths, so its render is the bound table.  That table is compared with wae_periodic_wave_table's (the host's f32 expression)
and with numpy's inverse FFT.  Renders are compared with the engine's render of twins given the read-out table through set_periodic_wave
(bit-equal: same plan, same table) and with the oracle given the host table (1e-5)."""
import contextlib
import ctypes as C

import numpy as np
import pytest

import graphs as G
from test_device_waves_cpu import coefficients, host_table, wave_graph

pytestmark = pytest.mark.gpu
TOL = 1e-5
SR = G.SR
PATHS = {"fused": dict(), "unfused": dict(fuse=0), "arate": dict(), "voices": dict(voice_sum=2), "suspend": dict()}


@contextlib.contextmanager
def options(pkg, engine, fuse=1, chunk=0, voice_sum=0):
    engine.set_option(pkg.OPT_FUSE, fuse)
    engine.set_option(pkg.OPT_CHUNK_FRAMES, chunk)
    engine.set_option(pkg.OPT_VOICE_SUM, voice_sum)
    try:
        yield
    finally:
        engine.set_option(pkg.OPT_FUSE, 1)
        engine.set_option(pkg.OPT_CHUNK_FRAMES, 0)
        engine.set_option(pkg.OPT_VOICE_SUM, 0)


def tensor(torch, arrays):
    return torch.from_numpy(np.ascontiguousarray(np.stack(arrays).astype(np.float32))).cuda()


def maxdiff(a, b):
    return float(np.abs(a.astype(np.float64) - b.astype(np.float64)).max())


def run(batch):
    batch.run()
    batch.sync()
    return batch.fetch()


def readout_graph(pkg, be, n, table_len, table=None, normalize=True):
    """a custom oscillator at sample_rate / table_len started at 0 -> destination: its render is its wavetable"""
    c = pkg.OfflineAudioContext(2, table_len, SR, be)
    o = c.create_oscillator(frequency=SR / table_len)
    if table is None:
        o.set_device_periodic_wave(n, table_len, disable_normalization=not normalize)
    else:
        o.set_periodic_wave(table)
    o.connect(c.destination())
    o.start()
    return c, o


def read_out(pkg, engine, torch, reals, imags, table_len, normalize=True):
    """the wavetables the bind synthesises from reals[g] / imags[g] (either list may be None), [graphs][table_len]"""
    given = reals if reals is not None else imags
    n = len(given[0])
    made = [readout_graph(pkg, engine.backend, n, table_len, normalize=normalize) for _ in given]
    b = pkg.Batch([c for c, _ in made])
    b.bind_periodic_waves(made[0][1], None if reals is None else tensor(torch, reals), None if imags is None else tensor(torch, imags))
    out = run(b)
    b.destroy()
    return out[:, 0, :]


# ---------------------------------------------------------------------------------------------------------- the wavetable itself
@pytest.mark.parametrize("normalize", [True, False])
@pytest.mark.parametrize("harmonics", [2, 5, 33, 200])
@pytest.mark.parametrize("table_len", [2048, 8192])
def test_table_read_out(pkg, engine, table_len, harmonics, normalize):
    torch = pytest.importorskip("torch")
    api = pkg.api()
    rng = np.random.default_rng(77 + harmonics)
    reals = [rng.uniform(-1, 1, harmonics).astype(np.float32) for _ in range(3)]
    imags = [rng.uniform(-1, 1, harmonics).astype(np.float32) for _ in range(3)]
    got = read_out(pkg, engine, torch, reals, imags, table_len, normalize)
    # the read-out is exact: a host table played the same way renders that table bit for bit
    hosts = [host_table(api, reals[g], imags[g], table_len, normalize) for g in range(3)]
    twin = run(pkg.Batch([readout_graph(pkg, engine.backend, harmonics, table_len, hosts[g])[0] for g in range(3)]))[:, 0, :]
    assert np.array_equal(twin, np.stack(hosts))
    # the host's f32 expression: equal but for the last bits of the sin / cos of a few arguments
    diff = maxdiff(got, np.stack(hosts))
    unequal = int((got != np.stack(hosts)).sum())
    print(f"[wave table] len {table_len} harmonics {harmonics} normalize {normalize}: max |diff| {diff:.3g}, "
          f"unequal {unequal} of {got.size}")
    assert diff <= 2e-7 * harmonics + 1e-6 and unequal <= got.size // 4
    # the Fourier series (tests/test_independent_witnesses.py: the reference's f32 accumulation error bound)
    tol = 2e-5 + 2e-7 * harmonics * harmonics
    for g in range(3):
        spec = np.zeros(table_len // 2 + 1, np.complex128)
        spec[1:harmonics] = (reals[g][1:].astype(np.float64) - 1j * imags[g][1:].astype(np.float64)) * table_len / 2
        want = np.fft.irfft(spec, table_len)
        if normalize:
            want = want / np.abs(want).max()
        assert maxdiff(got[g], want) <= tol, (g, maxdiff(got[g], want))


@pytest.mark.parametrize("which", ["real", "imag"])
def test_one_side_null(pkg, engine, which):
    """a NULL real or imag is zeros, as in wae_periodic_wave_table"""
    torch = pytest.importorskip("torch")
    api = pkg.api()
    rows = [coefficients(5 + g, 16)[0] for g in range(2)]
    got = read_out(pkg, engine, torch, rows if which == "real" else None, rows if which == "imag" else None, 2048)
    want = np.stack([host_table(api, r if which == "real" else None, r if which == "imag" else None, 2048) for r in rows])
    assert maxdiff(got, want) <= 1e-6


def test_non_finite_coefficients(pkg, engine):
    """NaN and infinite coefficients go through as the host takes them: the render has NaN and infinity where the render of the
    host-table twin has them (no read-out: a neighbouring infinity times interpolation weight 0 is NaN)"""
    torch = pytest.importorskip("torch")
    api = pkg.api()
    n, table_len = 9, 2048
    reals = [coefficients(g, n)[0] for g in range(3)]
    imags = [coefficients(g, n)[1] for g in range(3)]
    reals[0][3] = np.nan
    imags[1][2] = np.inf
    reals[2][4], imags[2][5] = -np.inf, np.inf
    for normalize in (True, False):
        def build(be, g, table):
            return wave_graph(pkg, be, g, 4096, n, table_len, table, normalize=normalize)
        made = [build(engine.backend, g, None) for g in range(3)]
        b = pkg.Batch([c for c, _ in made])
        b.bind_periodic_waves(made[0][1][0], tensor(torch, reals), tensor(torch, imags))
        got = run(b)
        twin = run(pkg.Batch([build(engine.backend, g, host_table(api, reals[g], imags[g], table_len, normalize))[0] for g in range(3)]))
        assert np.array_equal(np.isnan(got), np.isnan(twin)) and np.array_equal(np.isinf(got), np.isinf(twin))
        assert np.array_equal(got[np.isinf(got)], twin[np.isinf(twin)])
        assert not np.isfinite(got).all()


# ---------------------------------------------------------------------------------------------------------- renders
def check(pkg, engine, oracle, torch, build, n, table_len, reals, imags, batch=None, normalize=True):
    """binds (reals[g], imags[g]) to every oscillator of graph g of a prepared batch of declared graphs (or `batch`), runs it, and compares
    with the engine's render of twins given the read-out wavetables (bit-equal) and with the oracle given the host wavetables (1e-5)
    -> (render, batch)"""
    api = pkg.api()
    if batch is None:
        made = [build(engine.backend, g, None) for g in range(len(reals))]
        batch = (pkg.Batch([c for c, _ in made]), made[0][1])
    b, oscs = batch
    for osc in oscs:
        b.bind_periodic_waves(osc, tensor(torch, reals), tensor(torch, imags))
    got = run(b)
    tables = read_out(pkg, engine, torch, reals, imags, table_len, normalize)
    twin = run(pkg.Batch([build(engine.backend, g, tables[g])[0] for g in range(len(reals))]))
    assert np.array_equal(got, twin), maxdiff(got, twin)
    want = G.render(pkg, [build(oracle, g, host_table(api, reals[g], imags[g], table_len, normalize))[0] for g in range(len(reals))])
    assert np.isfinite(want).all() and float(np.abs(want).max()) > 1e-3
    assert maxdiff(got, want) <= TOL, maxdiff(got, want)
    return got, batch


@pytest.mark.parametrize("chunk", [8192, 0])
@pytest.mark.parametrize("table_len", [2048, 8192])
@pytest.mark.parametrize("path", list(PATHS))
def test_paths(pkg, engine, oracle, path, table_len, chunk):
    torch = pytest.importorskip("torch")
    n = 48
    coeffs = [coefficients(100 + g, n) for g in range(2)]

    def build(be, g, table):
        return wave_graph(pkg, be, g, 20000, n, table_len, table, path=path)
    with options(pkg, engine, chunk=chunk, **PATHS[path]):
        if path in ("unfused", "voices"):
            names = {name for name, _t, _k in pkg.Batch([build(engine.backend, g, None)[0] for g in range(2)]).stage_times()}
            assert ("k_oscillator" if path == "unfused" else "k_voice_sum") in names, names
        check(pkg, engine, oracle, torch, build, n, table_len, [c[0] for c in coeffs], [c[1] for c in coeffs])


@pytest.mark.parametrize("path", ["fused", "voices"])
def test_rebinding(pkg, engine, oracle, path):
    """one prepared batch: coefficient set A, then B (normalised to another peak), then A again; each run equals its twin, and the
    third run repeats the first bit for bit"""
    torch = pytest.importorskip("torch")
    n, table_len = 64, 8192
    a = [coefficients(200 + g, n) for g in range(2)]
    bb = [coefficients(300 + g, n) for g in range(2)]

    def build(be, g, table):
        return wave_graph(pkg, be, g, 12000, n, table_len, table, path=path)
    with options(pkg, engine, **PATHS[path]):
        first, batch = check(pkg, engine, oracle, torch, build, n, table_len, [c[0] for c in a], [c[1] for c in a])
        second, _ = check(pkg, engine, oracle, torch, build, n, table_len, [c[0] for c in bb], [c[1] for c in bb], batch=batch)
        third, _ = check(pkg, engine, oracle, torch, build, n, table_len, [c[0] for c in a], [c[1] for c in a], batch=batch)
    assert np.array_equal(first, third) and not np.array_equal(first, second)


def test_without_normalization(pkg, engine, oracle):
    torch = pytest.importorskip("torch")
    n, table_len = 20, 2048
    coeffs = [coefficients(400 + g, n) for g in range(2)]

    def build(be, g, table):
        return wave_graph(pkg, be, g, 12000, n, table_len, table, normalize=False)
    check(pkg, engine, oracle, torch, build, n, table_len, [c[0] for c in coeffs], [c[1] for c in coeffs], normalize=False)


# ---------------------------------------------------------------------------------------------------------- runs and binds
def test_template_bind_with_oscillators_that_never_start(pkg, engine, oracle):
    """one tensor for every graph of a template, where the oscillator of the odd graphs is never started: those items are validated and
    write nothing, and the odd graphs render silence"""
    torch = pytest.importorskip("torch")
    api = pkg.api()
    n, table_len, n_g = 16, 2048, 4
    coeffs = [coefficients(500 + g, n) for g in range(n_g)]

    def build(be, g, table):
        c = pkg.OfflineAudioContext(2, 6000, SR, be)
        o = c.create_oscillator(frequency=300.0 + 20 * g)
        if table is None:
            o.set_device_periodic_wave(n, table_len)
        else:
            o.set_periodic_wave(table)
        gn = c.create_gain(0.5)
        o.connect(gn)
        gn.connect(c.destination())
        if g % 2 == 0:
            o.start()
        return c, o
    made = [build(engine.backend, g, None) for g in range(n_g)]
    b = pkg.Batch([c for c, _ in made])
    with pytest.raises(pkg.WaeError) as e:
        b.run()
    assert e.value.status == 2 and "wae_batch_bind_periodic_waves" in e.value.message
    b.bind_periodic_waves(made[0][1], tensor(torch, [c[0] for c in coeffs]), tensor(torch, [c[1] for c in coeffs]))
    got = run(b)
    want = G.render(pkg, [build(oracle, g, host_table(api, *coeffs[g], table_len))[0] for g in range(n_g)])
    assert maxdiff(got, want) <= TOL
    assert not got[1::2].any() and got[0::2].any()


def test_ordering_after_a_torch_kernel(pkg, engine, oracle):
    """the coefficients are written by a torch kernel on torch's current stream right before the bind, without a synchronisation"""
    torch = pytest.importorskip("torch")
    api = pkg.api()
    n, table_len = 32, 8192
    coeffs = [coefficients(600 + g, n) for g in range(3)]

    def build(be, g, table):
        return wave_graph(pkg, be, g, 8000, n, table_len, table)
    made = [build(engine.backend, g, None) for g in range(3)]
    b = pkg.Batch([c for c, _ in made])
    re, im = tensor(torch, [c[0] for c in coeffs]), tensor(torch, [c[1] for c in coeffs])
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)  # the write lands long after the host has bound and launched
        x, y = re * 0.5, im * 2.0
        b.bind_periodic_waves(made[0][1][0], x, y)
        del x, y  # (kept from reuse until the bind has read them: record_stream)
        b.run()
    b.sync()
    got = b.fetch()
    want = G.render(pkg, [build(oracle, g, host_table(api, coeffs[g][0] * np.float32(0.5), coeffs[g][1] * np.float32(2.0),
                                                        table_len))[0] for g in range(3)])
    assert maxdiff(got, want) <= TOL


def test_errors_before_launch(pkg, engine):
    torch = pytest.importorskip("torch")
    B = pkg._binding
    api = pkg.api()
    n_g, n, table_len = 3, 32, 2048
    coeffs = [coefficients(700 + g, n) for g in range(n_g)]

    def build(be, g, table):
        return wave_graph(pkg, be, g, 8000, n, table_len, table)
    made = [build(engine.backend, g, None) for g in range(n_g)]
    b = pkg.Batch([c for c, _ in made])
    node = made[0][1][0].id
    with pytest.raises(pkg.WaeError) as e:
        b.run()
    assert e.value.status == 2 and "graph 0" in e.value.message and f"node {node}" in e.value.message
    good = tensor(torch, [c[0] for c in coeffs])

    def raw(items):
        def ptr(p):
            return None if p is None else C.cast(C.c_void_p(p), B.c_float_p)
        arr = (B.PeriodicWaveBinding * len(items))(*[B.PeriodicWaveBinding(g, nd, ptr(r), ptr(i)) for g, nd, r, i in items])
        return api.batch_bind_periodic_waves(b.handle, arr, len(items), None)

    host = np.stack([c[0] for c in coeffs])
    seg = next(x for x in torch.cuda.memory_snapshot() if x["address"] <= good.data_ptr() < x["address"] + x["total_size"])
    assert raw([(0, node, host.ctypes.data, None)]) == 1                                        # host (numpy) memory
    assert raw([(0, node, None, None)]) == 1                                                    # both null
    assert raw([(0, node, good.data_ptr(), seg["address"] + seg["total_size"] - 4 * (n - 1))]) == 1  # imag past its allocation
    assert raw([(0, node + 1, good.data_ptr(), None)]) == 2                                     # not a declared wave
    assert raw([(0, 9999, good.data_ptr(), None)]) == 2                                         # unknown node
    assert raw([(n_g, node, good.data_ptr(), None)]) == 2                                       # graph index out of range
    assert raw([(1, node, good.data_ptr(), None), (1, node, good.data_ptr(), None)]) == 1       # named twice
    assert raw([(0, node, good.data_ptr(), None), (0, node, host.ctypes.data, None)]) == 1       # a bad second item: nothing is bound
    with pytest.raises(pkg.WaeError) as e:
        b.bind_periodic_waves(node, good[:, : n - 1])                                           # fewer coefficients than declared
    assert e.value.status == 1
    with pytest.raises(pkg.WaeError) as e:
        b.bind_periodic_waves(node, good, good[:, :8])                                          # real and imag differ in shape
    assert e.value.status == 1
    with pytest.raises(pkg.WaeError) as e:
        b.run()
    assert e.value.status == 2  # nothing was bound by the failed calls
    b.bind_periodic_waves(node, good)
    got = run(b)
    twin = run(pkg.Batch([build(engine.backend, g, host_table(api, coeffs[g][0], None, table_len))[0] for g in range(n_g)]))
    assert maxdiff(got, twin) <= TOL


# ---------------------------------------------------------------------------------------------------------- with the other binds
def synth_graph(pkg, be, g, length, n, table_len, table=None, curve=None, pcm=None, ir=None, vals=None):
    """custom oscillator (declared) -> lowpass (frequency declared) -> gain (declared) \\
                                                                                     convolver (declared) -> destination
       device source -> WaveShaper (declared) ---------------------------------------/"""
    c = pkg.OfflineAudioContext(2, length, SR, be)
    o = c.create_oscillator(frequency=180.0 + 40 * g)
    if table is None:
        o.set_device_periodic_wave(n, table_len)
    else:
        o.set_periodic_wave(table)
    bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=3000.0 if vals is None else float(vals[0]), q=1.0)
    gn = c.create_gain(0.5 if vals is None else float(vals[1]))
    if vals is None:
        bq.frequency.set_device_value()
        gn.gain.set_device_value()
    src = c.create_buffer_source()
    if pcm is None:
        src.set_device_input(2, length, SR)
    else:
        src.set_buffer(pkg.AudioBuffer(list(pcm), SR))
    sh = c.create_wave_shaper()
    if curve is None:
        sh.set_device_curve(257)
    else:
        sh.set_curve(curve)
    cv = c.create_convolver()
    if ir is None:
        cv.set_device_response(2, 9000, SR)
    else:
        cv.set_buffer(pkg.AudioBuffer(list(ir), SR))
    o.connect(bq)
    bq.connect(gn)
    gn.connect(cv)
    src.connect(sh)
    sh.connect(cv)
    cv.connect(c.destination())
    o.start()
    src.start()
    return c, o, bq, gn, src, sh, cv


def test_sources_params_responses_curves_and_waves_together(pkg, engine, oracle):
    torch = pytest.importorskip("torch")
    api = pkg.api()
    n_g, length, n, table_len = 4, 20000, 40, 8192
    coeffs = [coefficients(800 + g, n) for g in range(n_g)]
    pcms = [G.c2_source(g, length) * np.float32(0.3) for g in range(n_g)]
    curves = [np.tanh(np.linspace(-2.0, 2.0, 257) * (1 + g)).astype(np.float32) for g in range(n_g)]
    irs = [np.stack(G.synthetic_ir(9000, 2, seed=810 + g)) for g in range(n_g)]
    vals = np.array([[700.0 + 800 * g, 0.3 + 0.1 * g] for g in range(n_g)], np.float32)
    made = [synth_graph(pkg, engine.backend, g, length, n, table_len) for g in range(n_g)]
    b = pkg.Batch([m[0] for m in made])
    _, o, bq, gn, src, sh, cv = made[0]
    b.bind_periodic_waves(o, tensor(torch, [c[0] for c in coeffs]), tensor(torch, [c[1] for c in coeffs]))
    b.bind_params([bq.frequency, gn.gain], torch.from_numpy(vals).cuda())
    b.bind_sources(src, tensor(torch, pcms))
    b.bind_curves(sh, tensor(torch, curves))
    b.bind_responses(cv, tensor(torch, irs))
    got = run(b)
    want = G.render(pkg, [synth_graph(pkg, oracle, g, length, n, table_len, host_table(api, *coeffs[g], table_len), curves[g], pcms[g],
                                      irs[g], vals[g])[0] for g in range(n_g)])
    assert maxdiff(got, want) <= TOL, maxdiff(got, want)
