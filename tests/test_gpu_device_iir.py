"""IIRFilterNode coefficients bound from device memory (wae_iir_filter_set_device_coefficients + wae_batch_bind_iir_coefficients) on the
GPU.  A batch is planned once with placeholder coefficients and run with coefficients bound from float64 torch tensors.

Bound coefficients are normalised on the device with the host's IEEE f64 division, so a render is compared bit for bit with the engine's
render of twins constructed with the same coefficients (create_iir_filter), on every path of tests/test_device_iir_cpu.py at two chunk
sizes and under WAE_OPT_SERIAL_FILTERS, and with the oracle at 1e-5.  A batch of 256 graphs, each bound to its own stable filter of order
1 to 19, is checked against scipy.signal.lfilter in f64."""
import contextlib
import ctypes as C

import numpy as np
import pytest

import graphs as G
from test_device_iir_cpu import CASES, iir_graph, stable_filter

pytestmark = pytest.mark.gpu
TOL = 1e-5
SR = G.SR
LENGTH = 12000
CASE = {c[0]: c for c in CASES}


@contextlib.contextmanager
def options(pkg, engine, chunk=0, serial=0):
    engine.set_option(pkg.OPT_CHUNK_FRAMES, chunk)
    engine.set_option(pkg.OPT_SERIAL_FILTERS, serial)
    try:
        yield
    finally:
        engine.set_option(pkg.OPT_CHUNK_FRAMES, 0)
        engine.set_option(pkg.OPT_SERIAL_FILTERS, 0)


def t64(torch, rows):
    return torch.from_numpy(np.ascontiguousarray(np.stack(rows), np.float64)).cuda()


def maxdiff(a, b):
    return float(np.abs(a.astype(np.float64) - b.astype(np.float64)).max())


def run(batch):
    batch.run()
    batch.sync()
    return batch.fetch()


def filters(seed, n_g, nff, nfb):
    return [stable_filter(seed + g, nff, nfb) for g in range(n_g)]


def check(pkg, engine, oracle, torch, name, coefs, batch=None, length=LENGTH):
    """binds coefs[g] to the declared filter of graph g of a prepared batch of case `name` (or `batch`), runs it, and compares with the
    engine's render of twins constructed with coefs[g] (bit-equal) and with the oracle (1e-5) -> (render, batch)"""
    _, path, nff, nfb, channels, _ = CASE[name]

    def build(be, g, cf):
        return iir_graph(pkg, be, g, length, nff, nfb, cf, path, channels)
    if batch is None:
        made = [build(engine.backend, g, None) for g in range(len(coefs))]
        batch = (pkg.Batch([c for c, _ in made]), made[0][1])
    b, node = batch
    b.bind_iir_coefficients(node, t64(torch, [c[0] for c in coefs]), t64(torch, [c[1] for c in coefs]))
    got = run(b)
    twin = run(pkg.Batch([build(engine.backend, g, coefs[g])[0] for g in range(len(coefs))]))
    assert np.array_equal(got, twin, equal_nan=True), maxdiff(got, twin)
    if path == "switch":  # (the engine renders channel 1 of this graph silent where the oracle up-mixes, with or without a bind: NEXT.md)
        return got, batch
    want = G.render(pkg, [build(oracle, g, coefs[g])[0] for g in range(len(coefs))])
    assert np.isfinite(want).all() and float(np.abs(want).max()) > 1e-3
    assert maxdiff(got, want) <= TOL, maxdiff(got, want)
    return got, batch


# ---------------------------------------------------------------------------------------------------------- renders
@pytest.mark.parametrize("chunk", [4096, 0])
@pytest.mark.parametrize("name", [c[0] for c in CASES])
def test_paths(pkg, engine, oracle, name, chunk):
    torch = pytest.importorskip("torch")
    _, path, nff, nfb, channels, kernel = CASE[name]
    with options(pkg, engine, chunk=chunk):
        made = [iir_graph(pkg, engine.backend, g, LENGTH, nff, nfb, None, path, channels) for g in range(3)]
        names = {k for k, _t, _n in pkg.Batch([c for c, _ in made]).stage_times()}
        assert kernel in names, names
        check(pkg, engine, oracle, torch, name, filters(10 * nff + nfb, 3, nff, nfb))


@pytest.mark.parametrize("name", ["order1_chain", "order2_chain", "order2_dest", "coef3"])
def test_serial_filters_option(pkg, engine, oracle, name):
    """WAE_OPT_SERIAL_FILTERS: the chain-path cases on k_iir_serial (the source and gain keep their own k_chain)"""
    torch = pytest.importorskip("torch")
    _, path, nff, nfb, channels, _ = CASE[name]
    with options(pkg, engine, serial=1):
        made = [iir_graph(pkg, engine.backend, g, LENGTH, nff, nfb, None, path, channels) for g in range(3)]
        names = {k for k, _t, _n in pkg.Batch([c for c, _ in made]).stage_times()}
        assert "k_iir_serial" in names, names
        check(pkg, engine, oracle, torch, name, filters(50 + nff, 3, nff, nfb))


def test_f64_witness(pkg, engine):
    """256 graphs, each bound to its own Butterworth or Chebyshev filter of order 1 to 19 (one bind per order), against scipy's lfilter
    in f64 at the tolerance of tests/test_gpu_witnesses.py::test_iir_high_orders_vs_scipy"""
    torch = pytest.importorskip("torch")
    from scipy import signal
    n_g, rq = 256, 128
    n = rq * 100 + 45
    xs, coefs = [], []
    for k in range(n_g):
        order = 1 + k % 19
        frac = ((k * 37) % 100) / 100
        wc = (0.25 + 0.5 * frac) if order < 10 else (0.5 + 0.25 * frac)
        b, a = signal.butter(order, wc) if k % 2 == 0 else signal.cheby1(order, 0.5, wc)
        x = np.random.default_rng(k).uniform(-1, 1, n).astype(np.float32)
        x[n // 2:] = 0.0  # the input falls silent: the filter rings out
        xs.append(x)
        coefs.append((b * 1.75, a * 1.75))
    made = []
    for k in range(n_g):
        order = 1 + k % 19
        c = pkg.OfflineAudioContext(1, n, SR, engine.backend)
        s = c.create_buffer_source(pkg.AudioBuffer([xs[k]], SR))
        f = c.create_iir_filter([1.0] + [0.0] * order, [1.0] + [0.0] * order)
        f.set_device_coefficients()
        s.connect(f)
        f.connect(c.destination())
        s.start()
        made.append((c, f))
    batch = pkg.Batch([c for c, _ in made])
    for order in range(1, 20):
        ks = [k for k in range(n_g) if 1 + k % 19 == order]
        batch.bind_iir_coefficients([made[k][1] for k in ks], t64(torch, [coefs[k][0] for k in ks]), t64(torch, [coefs[k][1] for k in ks]),
                                    graphs=ks)
    got = run(batch)
    worst = 0.0
    for k in range(n_g):
        b, a = coefs[k]
        want = signal.lfilter(b, a, xs[k].astype(np.float64))
        want = np.where(np.abs(want) < np.finfo(np.float64).tiny, 0.0, want)
        sos = signal.tf2sos(b, a)  # (the direct form is a witness while it agrees with the cascade of sections)
        assert np.abs(signal.sosfilt(sos, xs[k].astype(np.float64)) - want).max() <= 1e-8 * max(1.0, np.abs(want).max()), k
        err = float(np.abs(got[k, 0].astype(np.float64) - want).max())
        assert err <= 4e-7 * max(1.0, float(np.abs(want).max())), (k, err)
        worst = max(worst, err)
    print(f"[iir witness] {n_g} filters, orders 1..19: max |gpu - lfilter| {worst:.3g}")


# ---------------------------------------------------------------------------------------------------------- rebinds and ordering
@pytest.mark.parametrize("name", ["order2_chain", "coef8", "suspend"])
def test_rebinding(pkg, engine, oracle, name):
    """one prepared batch: coefficient set A, then B, then A again; each run equals its twin, and the third repeats the first bit for bit"""
    torch = pytest.importorskip("torch")
    _, _, nff, nfb, _, _ = CASE[name]
    a, bb = filters(200, 3, nff, nfb), filters(300, 3, nff, nfb)
    first, batch = check(pkg, engine, oracle, torch, name, a)
    second, _ = check(pkg, engine, oracle, torch, name, bb, batch=batch)
    third, _ = check(pkg, engine, oracle, torch, name, a, batch=batch)
    assert np.array_equal(first, third) and not np.array_equal(first, second)


@pytest.mark.parametrize("name", ["order2_chain", "coef8"])
def test_ordering_after_a_torch_kernel(pkg, engine, oracle, name):
    """the coefficients are written by a torch kernel on torch's current stream right before the bind, without a synchronisation"""
    torch = pytest.importorskip("torch")
    _, path, nff, nfb, channels, _ = CASE[name]
    coefs = filters(600, 3, nff, nfb)
    made = [iir_graph(pkg, engine.backend, g, LENGTH, nff, nfb, None, path, channels) for g in range(3)]
    b = pkg.Batch([c for c, _ in made])
    ff, fb = t64(torch, [c[0] for c in coefs]), t64(torch, [c[1] for c in coefs])
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)  # the write lands long after the host has bound and launched
        x = ff * 0.5
        b.bind_iir_coefficients(made[0][1], x, fb)
        del x  # (kept from reuse until the bind has read it: record_stream)
        b.run()
    b.sync()
    got = b.fetch()
    twin = run(pkg.Batch([iir_graph(pkg, engine.backend, g, LENGTH, nff, nfb, (coefs[g][0] * 0.5, coefs[g][1]), path, channels)[0]
                          for g in range(3)]))
    assert np.array_equal(got, twin)


# ---------------------------------------------------------------------------------------------------------- edge cases
def test_non_finite_coefficients(pkg, engine):
    """NaN and infinite coefficients are used as the host constructor takes them: bit-equal to the twins, NaN positions included"""
    torch = pytest.importorskip("torch")
    for name in ("order2_chain", "coef8"):
        _, path, nff, nfb, channels, _ = CASE[name]
        coefs = [tuple(np.array(x) for x in c) for c in filters(700, 3, nff, nfb)]
        coefs[0][0][1] = np.nan
        coefs[1][1][1] = np.inf
        coefs[2][1][0] = -np.inf
        made = [iir_graph(pkg, engine.backend, g, 4096, nff, nfb, None, path, channels) for g in range(3)]
        b = pkg.Batch([c for c, _ in made])
        b.bind_iir_coefficients(made[0][1], t64(torch, [c[0] for c in coefs]), t64(torch, [c[1] for c in coefs]))
        got = run(b)
        twin = run(pkg.Batch([iir_graph(pkg, engine.backend, g, 4096, nff, nfb, coefs[g], path, channels)[0] for g in range(3)]))
        assert np.array_equal(got, twin, equal_nan=True), name


@pytest.mark.parametrize("name", ["order2_chain", "coef8", "suspend"])
def test_zero_first_feedback_renders_zeros(pkg, engine, name):
    """the deviation: feedback[0] == 0 (refused by the reference's constructor) writes all-zero coefficients, and that graph's filter
    outputs zeros; the other items of the bind render as their twins"""
    torch = pytest.importorskip("torch")
    _, path, nff, nfb, channels, _ = CASE[name]
    coefs = [tuple(np.array(x) for x in c) for c in filters(800, 3, nff, nfb)]
    bad = (coefs[1][0].copy(), coefs[1][1].copy())
    bad[1][0] = 0.0
    made = [iir_graph(pkg, engine.backend, g, LENGTH, nff, nfb, None, path, channels) for g in range(3)]
    b = pkg.Batch([c for c, _ in made])
    b.bind_iir_coefficients(made[0][1], t64(torch, [coefs[0][0], bad[0], coefs[2][0]]), t64(torch, [coefs[0][1], bad[1], coefs[2][1]]))
    got = run(b)
    twin = run(pkg.Batch([iir_graph(pkg, engine.backend, g, LENGTH, nff, nfb, coefs[g], path, channels)[0] for g in range(3)]))
    assert not got[1].any()
    assert np.array_equal(got[0::2], twin[0::2]) and got[0].any()


def test_template_bind_with_silent_and_unconnected_filters(pkg, engine, oracle):
    """one tensor for every graph of a template, where the source of the odd graphs never starts: those items bind like the others and
    the odd graphs render silence.  A second declared filter connected to nothing is still lowered: runs wait for its bind, and what it
    is bound to changes no output"""
    torch = pytest.importorskip("torch")
    n_g, nff, nfb = 4, 3, 3
    coefs = filters(900, n_g, nff, nfb)

    def build(be, g, cf):
        c = pkg.OfflineAudioContext(2, 6000, SR, be)
        s = c.create_buffer_source(pkg.AudioBuffer(list(G.c2_source(g, 6000) * np.float32(0.5)), SR))
        f = c.create_iir_filter(*(cf or ([1.0, 0.0, 0.0], [1.0, 0.0, 0.0])))
        lone = c.create_iir_filter([1.0] * 8, [1.0] + [0.0] * 7)
        if cf is None:
            f.set_device_coefficients()
            lone.set_device_coefficients()
        s.connect(f)
        f.connect(c.destination())
        if g % 2 == 0:
            s.start()
        return c, f, lone
    made = [build(engine.backend, g, None) for g in range(n_g)]
    b = pkg.Batch([m[0] for m in made])
    b.bind_iir_coefficients(made[0][1], t64(torch, [c[0] for c in coefs]), t64(torch, [c[1] for c in coefs]))
    with pytest.raises(pkg.WaeError) as e:
        b.run()
    assert e.value.status == 2 and f"node {made[0][2].id}" in e.value.message
    b.bind_iir_coefficients(made[0][2], t64(torch, [np.ones(8)] * n_g), t64(torch, [np.ones(8)] * n_g))
    got = run(b)
    want = G.render(pkg, [build(oracle, g, coefs[g])[0] for g in range(n_g)])
    assert maxdiff(got, want) <= TOL
    assert not got[1::2].any() and got[0::2].any()
    b.bind_iir_coefficients(made[0][2], t64(torch, [np.full(8, 0.5)] * n_g), t64(torch, [np.full(8, 2.0)] * n_g))
    assert np.array_equal(run(b), got)


def test_errors_before_launch(pkg, engine):
    torch = pytest.importorskip("torch")
    B = pkg._binding
    api = pkg.api()
    n_g, nff, nfb = 3, 8, 8
    _, path, _, _, channels, _ = CASE["coef8"]
    coefs = filters(1000, n_g, nff, nfb)
    made = [iir_graph(pkg, engine.backend, g, 4096, nff, nfb, None, path, channels) for g in range(n_g)]
    b = pkg.Batch([c for c, _ in made])
    node = made[0][1].id
    with pytest.raises(pkg.WaeError) as e:
        b.run()
    assert e.value.status == 2 and "graph 0" in e.value.message and f"node {node}" in e.value.message
    ff, fb = t64(torch, [c[0] for c in coefs]), t64(torch, [c[1] for c in coefs])

    def raw(items):
        def ptr(p):
            return C.cast(C.c_void_p(p), B.c_double_p)
        arr = (B.IirBinding * len(items))(*[B.IirBinding(g, nd, ptr(f0), ptr(f1)) for g, nd, f0, f1 in items])
        return api.batch_bind_iir_coefficients(b.handle, arr, len(items), None)

    host = np.stack([c[0] for c in coefs])
    seg = next(x for x in torch.cuda.memory_snapshot() if x["address"] <= fb.data_ptr() < x["address"] + x["total_size"])
    ok = (1, node, ff.data_ptr() + 64 * 1, fb.data_ptr() + 64 * 1)
    assert raw([(0, node, host.ctypes.data, fb.data_ptr())]) == 1                                      # host (numpy) memory
    assert raw([(0, node, ff.data_ptr(), seg["address"] + seg["total_size"] - 8 * (nfb - 1))]) == 1   # past its allocation
    assert raw([(0, node, ff.data_ptr() + 4, fb.data_ptr())]) == 1                                    # not 8-byte aligned
    assert raw([(0, node + 1, ff.data_ptr(), fb.data_ptr())]) == 2                                    # not a declared filter
    assert raw([(n_g, node, ff.data_ptr(), fb.data_ptr())]) == 2                                      # graph index out of range
    assert raw([ok, ok]) == 1                                                                         # named twice
    assert raw([ok, (0, node, host.ctypes.data, fb.data_ptr())]) == 1                                 # a bad second item: nothing bound
    assert raw([ok, (0, node + 1, ff.data_ptr(), fb.data_ptr())]) == 2
    with pytest.raises(pkg.WaeError) as e:
        b.bind_iir_coefficients(node, ff.float(), fb.float())                                         # float32
    assert e.value.status == 1
    with pytest.raises(pkg.WaeError) as e:
        b.bind_iir_coefficients(node, ff[:, : nff - 1], fb)                                           # fewer columns than declared
    assert e.value.status == 1
    with pytest.raises(pkg.WaeError) as e:
        b.run()
    assert e.value.status == 2  # nothing was bound by the failed calls
    b.bind_iir_coefficients(node, ff, fb)
    got = run(b)
    twin = run(pkg.Batch([iir_graph(pkg, engine.backend, g, 4096, nff, nfb, coefs[g], path, channels)[0] for g in range(n_g)]))
    assert np.array_equal(got, twin)


# ---------------------------------------------------------------------------------------------------------- with the other binds
def six_graph(pkg, be, g, length, n, table_len, iir=None, table=None, curve=None, pcm=None, ir=None, vals=None):
    """custom oscillator (declared) -> lowpass (frequency declared) -> gain (declared) -> IIR (declared) \\
                                                                                                     convolver (declared) -> destination
       device source -> WaveShaper (declared) -----------------------------------------------------/"""
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
    f = c.create_iir_filter(*(iir or ([1.0] * 5, [1.0] + [0.0] * 4)))
    if iir is None:
        f.set_device_coefficients()
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
    gn.connect(f)
    f.connect(cv)
    src.connect(sh)
    sh.connect(cv)
    cv.connect(c.destination())
    o.start()
    src.start()
    return c, o, bq, gn, f, src, sh, cv


def test_all_six_binds_together(pkg, engine, oracle):
    torch = pytest.importorskip("torch")
    from test_device_waves_cpu import coefficients, host_table
    api = pkg.api()
    n_g, length, n, table_len = 4, 20000, 40, 8192
    waves = [coefficients(800 + g, n) for g in range(n_g)]
    iirs = filters(1100, n_g, 5, 5)
    pcms = [G.c2_source(g, length) * np.float32(0.3) for g in range(n_g)]
    curves = [np.tanh(np.linspace(-2.0, 2.0, 257) * (1 + g)).astype(np.float32) for g in range(n_g)]
    irs = [np.stack(G.synthetic_ir(9000, 2, seed=810 + g)) for g in range(n_g)]
    vals = np.array([[700.0 + 800 * g, 0.3 + 0.1 * g] for g in range(n_g)], np.float32)
    made = [six_graph(pkg, engine.backend, g, length, n, table_len) for g in range(n_g)]
    b = pkg.Batch([m[0] for m in made])
    _, o, bq, gn, f, src, sh, cv = made[0]
    f32 = lambda rows: torch.from_numpy(np.ascontiguousarray(np.stack(rows), np.float32)).cuda()
    b.bind_periodic_waves(o, f32([w[0] for w in waves]), f32([w[1] for w in waves]))
    b.bind_params([bq.frequency, gn.gain], torch.from_numpy(vals).cuda())
    b.bind_iir_coefficients(f, t64(torch, [c[0] for c in iirs]), t64(torch, [c[1] for c in iirs]))
    b.bind_sources(src, f32(pcms))
    b.bind_curves(sh, f32(curves))
    b.bind_responses(cv, f32(irs))
    got = run(b)
    want = G.render(pkg, [six_graph(pkg, oracle, g, length, n, table_len, iirs[g], host_table(api, *waves[g], table_len), curves[g], pcms[g],
                                    irs[g], vals[g])[0] for g in range(n_g)])
    assert maxdiff(got, want) <= TOL, maxdiff(got, want)
