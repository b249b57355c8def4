"""AudioParam value curves bound from device memory (wae_param_set_device_value_curve + wae_batch_bind_value_curves) on the GPU.
Every graph is built three ways: with the curve declared and its values bound from a torch tensor, on the engine with the same values
given to set_value_curve_at_time (the host twin: same plan, same values, so bit-equal), and on the oracle (1e-5).  A third statement
checks the bound curve against numpy's f64 evaluation of the specification's interpolation."""
import contextlib

import numpy as np
import pytest

import graphs as G
from test_device_value_curves_cpu import CASES, build, curve_values

pytestmark = pytest.mark.gpu
TOL = 1e-5
SR = 48000.0
FRAMES = 8192
# (length, start frame, duration in frames): from 0 over the whole render, mid-quantum and ending before the end, inside a later chunk
# (of 1024 frames) and running past the end
SHAPES = [(2, 0, FRAMES), (3, 200, 3000), (1000, 5000.5, 6000)]


@contextlib.contextmanager
def options(pkg, engine, chunk=0, param_parallel=2):
    engine.set_option(pkg.OPT_CHUNK_FRAMES, chunk)
    engine.set_option(pkg.OPT_PARAM_PARALLEL, param_parallel)
    try:
        yield
    finally:
        engine.set_option(pkg.OPT_CHUNK_FRAMES, 0)
        engine.set_option(pkg.OPT_PARAM_PARALLEL, 2)


@pytest.fixture(scope="module")
def sphere(engine, oracle):
    """the HRIR sphere of the HRTF panner case, on both backends"""
    data = G.synthetic_hrir_sphere(int(SR), 256)
    oracle.set_hrir_sphere(data)
    engine.backend.set_hrir_sphere(data)


def tensor(torch, rows):
    return torch.from_numpy(np.ascontiguousarray(np.stack(rows), np.float32)).cuda()


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def maxdiff(a, b):
    return float(np.abs(a.astype(np.float64) - b.astype(np.float64)).max())


def run(batch):
    batch.run()
    batch.sync()
    return batch.fetch()


def check(pkg, engine, oracle, case, shape, vals, chunk=0, param_parallel=2, frames=FRAMES, oracle_tol=TOL):
    """binds vals[g] to the declared curve of graph g of `case`, runs it, and compares it with the host twins (bit-equal) and the oracle
    -> the bound render"""
    torch = pytest.importorskip("torch")
    length, start, dur = shape
    n = len(vals)
    kw = dict(length=length, start=start / SR, duration=dur / SR, frames=frames)
    with options(pkg, engine, chunk, param_parallel):
        made = [build(pkg, engine.backend, case, None, g=g, **kw) for g in range(n)]
        b = pkg.Batch([c for c, _ in made])
        b.bind_value_curves(made[0][1], tensor(torch, vals))
        got = run(b)
        twin = run(pkg.Batch([build(pkg, engine.backend, case, vals[g], g=g, **kw)[0] for g in range(n)]))
    assert np.array_equal(bits(got), bits(twin)), (case, shape, maxdiff(got, twin))
    if oracle_tol is not None:
        want = G.render(pkg, [build(pkg, oracle, case, vals[g], g=g, **kw)[0] for g in range(n)])
        assert maxdiff(got, want) <= oracle_tol, (case, shape, maxdiff(got, want))
    b.destroy()
    return got


@pytest.mark.parametrize("shape", SHAPES, ids=["len2_whole", "len3_mid_quantum", "len1000_past_end"])
@pytest.mark.parametrize("case", CASES)
def test_bound_equals_host_twin_and_oracle(pkg, engine, oracle, sphere, case, shape):
    vals = [curve_values(case, 100 * g + 1, shape[0]) for g in range(3)]
    check(pkg, engine, oracle, case, shape, vals)


@pytest.mark.parametrize("param_parallel", [0, 1, 2])
@pytest.mark.parametrize("chunk", [128, 1024, 0])
@pytest.mark.parametrize("case", ["osc_frequency", "gain", "delay_time", "panner_x", "suspend"])
def test_chunk_sizes_and_param_kernels(pkg, engine, oracle, case, chunk, param_parallel):
    shape = SHAPES[2]
    vals = [curve_values(case, 200 * g + 3, shape[0]) for g in range(2)]
    check(pkg, engine, oracle, case, shape, vals, chunk, param_parallel)


def test_against_f64_interpolation(pkg, engine):
    """third statement: ConstantSource(1) -> gain whose gain is the curve renders the curve itself, which the specification states as
    v[k] + (v[k+1] - v[k]) * frac with k + frac = (t - start) / duration * (length - 1), and the last value after the end.  (Compared from
    the curve's start on: before it, after the first quantum, the reference holds the curve evaluated at a time before its start, which
    the host twin and the oracle share.)"""
    torch = pytest.importorskip("torch")
    for length, start, dur in [(2, 0, FRAMES), (5, 333, 4000), (1000, 1000, 6000), (1000, 0, 3 * FRAMES)]:
        vals = [np.random.default_rng(31 + g).uniform(-1, 1, length).astype(np.float32) for g in range(2)]
        made = []
        for g in range(2):
            c = pkg.OfflineAudioContext(1, FRAMES, SR, engine.backend)
            src = c.create_constant_source(1.0)
            gn = c.create_gain(1.0)
            gn.gain.set_device_value_curve(length, start / SR, dur / SR)
            src.connect(gn)
            gn.connect(c.destination())
            src.start()
            made.append((c, gn.gain))
        b = pkg.Batch([c for c, _ in made])
        b.bind_value_curves(made[0][1], tensor(torch, vals))
        got = run(b)
        t = np.arange(FRAMES, dtype=np.float64) / SR
        for g in range(2):
            v = vals[g].astype(np.float64)
            pos = np.clip((t - start / SR) / (dur / SR) * (length - 1), 0.0, length - 1)
            k = np.minimum(np.floor(pos).astype(np.int64), length - 2)
            want = v[k] + (v[k + 1] - v[k]) * (pos - k)
            want[t >= (start + dur) / SR] = v[-1]
            on = t >= start / SR
            assert maxdiff(got[g, 0][on], want[on]) <= 1e-6, (length, start, dur, maxdiff(got[g, 0][on], want[on]))
        b.destroy()


def test_rebind_and_non_finite_values(pkg, engine, oracle):
    """a second bind replaces the first; NaN and infinite values are used as they are, bit-equal to the host twin"""
    torch = pytest.importorskip("torch")
    case, shape = "gain", (8, 0, FRAMES)
    kw = dict(length=8, start=0.0, duration=FRAMES / SR)
    made = [build(pkg, engine.backend, case, None, g=g, **kw) for g in range(2)]
    b = pkg.Batch([c for c, _ in made])
    sets = [[curve_values(case, 7 + g, 8) for g in range(2)], [curve_values(case, 17 + g, 8) for g in range(2)]]
    odd = [curve_values(case, 27 + g, 8) for g in range(2)]
    odd[0][2], odd[1][5], odd[1][6] = np.nan, np.inf, -np.inf
    last = None
    for vals in sets + [odd, sets[0]]:
        b.bind_value_curves(made[0][1], tensor(torch, vals))
        got = run(b)
        twin = run(pkg.Batch([build(pkg, engine.backend, case, vals[g], g=g, **kw)[0] for g in range(2)]))
        assert np.array_equal(bits(got), bits(twin))
        if vals is not odd:
            want = G.render(pkg, [build(pkg, oracle, case, vals[g], g=g, **kw)[0] for g in range(2)])
            assert maxdiff(got, want) <= TOL
        else:  # (bit-equal to the twin above; and the values did reach the render)
            assert not np.array_equal(bits(got), bits(last))
        last = got


def test_ordered_after_torch_stream(pkg, engine):
    """values written by a kernel on a torch side stream and bound from that stream are the ones the run reads"""
    torch = pytest.importorskip("torch")
    case, length = "osc_frequency", 1000
    kw = dict(length=length, start=0.0, duration=FRAMES / SR)
    made = [build(pkg, engine.backend, case, None, g=g, **kw) for g in range(4)]
    b = pkg.Batch([c for c, _ in made])
    vals = [curve_values(case, 50 + g, length) for g in range(4)]
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        t = torch.zeros((4, length), device="cuda")
        torch.cuda._sleep(20_000_000)  # (a late writer: without the ordering the bind would read zeros)
        t.copy_(tensor(torch, vals))
        b.bind_value_curves(made[0][1], t)
    got = run(b)
    twin = run(pkg.Batch([build(pkg, engine.backend, case, vals[g], g=g, **kw)[0] for g in range(4)]))
    assert np.array_equal(bits(got), bits(twin))


def test_errors_and_runs_before_the_bind(pkg, engine):
    torch = pytest.importorskip("torch")
    api = pkg.api()
    made = [build(pkg, engine.backend, "osc_detune", None, length=8) for _ in range(2)]
    b = pkg.Batch([c for c, _ in made])
    prm = made[0][1]
    with pytest.raises(pkg.WaeError) as e:
        b.run()
    assert e.value.status == 2 and f"graph 0, node {prm._node}, param {prm._index} (wae_batch_bind_value_curves)" in e.value.message
    good = torch.zeros((2, 8), device="cuda")
    with pytest.raises(pkg.WaeError) as e:  # a shape that is not the declaration's
        b.bind_value_curves(prm, torch.zeros((2, 9), device="cuda"))
    assert e.value.status == 1
    B = pkg._binding
    import ctypes as C

    def item(g, node, index, ptr):
        return B.ValueCurveBinding(g, node, index, C.cast(C.c_void_p(ptr), B.c_float_p))
    one = lambda *its: (B.ValueCurveBinding * len(its))(*its)
    p = good.data_ptr()
    assert api.batch_bind_value_curves(b.handle, one(item(2, prm._node, prm._index, p)), 1, None) == 2  # graph out of range
    assert api.batch_bind_value_curves(b.handle, one(item(0, prm._node, 0, p)), 1, None) == 2  # no declaration (frequency)
    assert api.batch_bind_value_curves(b.handle, one(item(0, prm._node, prm._index, 0)), 1, None) == 1  # null
    assert api.batch_bind_value_curves(b.handle, one(item(0, prm._node, prm._index, p + 2)), 1, None) == 1  # not 4-byte aligned
    host = np.zeros(8, np.float32)
    assert api.batch_bind_value_curves(b.handle, one(item(0, prm._node, prm._index, host.ctypes.data)), 1, None) == 1  # host memory
    assert api.batch_bind_value_curves(b.handle, one(item(0, prm._node, prm._index, p), item(0, prm._node, prm._index, p)), 2, None) == 1
    # all-or-nothing: graph 0 was not bound by the refused calls
    assert api.batch_bind_value_curves(b.handle, one(item(1, prm._node, prm._index, p)), 1, None) == 0
    with pytest.raises(pkg.WaeError) as e:
        b.run()
    assert "graph 0," in e.value.message
    b.bind_value_curves(prm, good)
    b.run()
    b.sync()


def test_pruned_declaration_needs_no_bind(pkg, engine, oracle):
    """a declared param the planner never lowers needs no bind, and binding it is accepted and writes nothing: the gain of a node in a
    cycle without a DelayNode (the param is in the cycle, whose nodes are muted)"""
    torch = pytest.importorskip("torch")

    def make(be, vals, declare_muted):
        c, prm = build(pkg, be, "gain", vals, length=4)
        a, b = c.create_gain(), c.create_gain()
        a.connect(b)
        b.connect(a.gain)
        a.connect(c.destination())
        if declare_muted:
            a.gain.set_device_value_curve(16, 0.0, 0.1)
        return c, prm, a
    vals = [curve_values("gain", 3, 4)]
    c, prm, a = make(engine.backend, None, True)
    b = pkg.Batch([c])
    b.bind_value_curves(prm, tensor(torch, vals))
    got = run(b)
    b.bind_value_curves(a.gain, torch.ones((1, 16), device="cuda"))
    assert np.array_equal(bits(run(b)), bits(got))
    twin = run(pkg.Batch([make(engine.backend, vals[0], False)[0]]))
    assert np.array_equal(bits(got), bits(twin))


def test_suspend_with_the_node_living_across(pkg, engine, oracle):
    """two suspend points after the declaration, one of them inside the curve, at three chunk sizes"""
    torch = pytest.importorskip("torch")
    length, start, dur = 1000, 1000, 6000
    kw = dict(length=length, start=start / SR, duration=dur / SR, suspends=(2048, 4480))
    vals = [curve_values("suspend", 60 + g, length) for g in range(2)]
    for chunk in (128, 1024, 0):
        with options(pkg, engine, chunk):
            made = [build(pkg, engine.backend, "suspend", None, g=g, **kw) for g in range(2)]
            assert pkg.plan_batch([made[0][0]])["segments"] == 3
            b = pkg.Batch([c for c, _ in made])
            b.bind_value_curves(made[0][1], tensor(torch, vals))
            got = run(b)
            twin = run(pkg.Batch([build(pkg, engine.backend, "suspend", vals[g], g=g, **kw)[0] for g in range(2)]))
        assert np.array_equal(bits(got), bits(twin))
        want = G.render(pkg, [build(pkg, oracle, "suspend", vals[g], g=g, **kw)[0] for g in range(2)])
        assert maxdiff(got, want) <= TOL


def test_all_binds_in_one_batch(pkg, engine, oracle):
    torch = pytest.importorskip("torch")
    from test_device_waves_cpu import coefficients, host_table
    from test_gpu_device_iir import filters, six_graph, t64
    api = pkg.api()
    n_g, length, n, table_len, cl = 3, 20000, 40, 8192, 100
    waves = [coefficients(900 + g, n) for g in range(n_g)]
    iirs = filters(1200, n_g, 5, 5)
    pcms = [G.c2_source(g, length) * np.float32(0.3) for g in range(n_g)]
    curves = [np.tanh(np.linspace(-2.0, 2.0, 257) * (1 + g)).astype(np.float32) for g in range(n_g)]
    irs = [np.stack(G.synthetic_ir(9000, 2, seed=910 + g)) for g in range(n_g)]
    vals = np.array([[700.0 + 800 * g, 0.3 + 0.1 * g] for g in range(n_g)], np.float32)
    contour = [curve_values("osc_frequency", 70 + g, cl) for g in range(n_g)]

    def seven(be, g, host):
        m = six_graph(pkg, be, g, length, n, table_len, *((iirs[g], host_table(api, *waves[g], table_len), curves[g], pcms[g], irs[g],
                                                            vals[g]) if host else ()))
        c = m[0]
        o2 = c.create_oscillator(frequency=300.0)
        if host:
            o2.frequency.set_value_curve_at_time(contour[g], 0.01, 0.3)
        else:
            o2.frequency.set_device_value_curve(cl, 0.01, 0.3)
        g2 = c.create_gain(0.2)
        o2.connect(g2)
        g2.connect(c.destination())
        o2.start()
        return m, o2
    made = [seven(engine.backend, g, False) for g in range(n_g)]
    b = pkg.Batch([m[0][0] for m in made])
    (_, o, bq, gn, f, src, sh, cv), o2 = made[0]
    f32 = lambda rows: tensor(torch, rows)
    b.bind_periodic_waves(o, f32([w[0] for w in waves]), f32([w[1] for w in waves]))
    b.bind_params([bq.frequency, gn.gain], torch.from_numpy(vals).cuda())
    b.bind_iir_coefficients(f, t64(torch, [c[0] for c in iirs]), t64(torch, [c[1] for c in iirs]))
    b.bind_sources(src, f32(pcms))
    b.bind_curves(sh, f32(curves))
    b.bind_responses(cv, f32(irs))
    b.bind_value_curves([o2.frequency], [f32(contour)])
    got = run(b)
    want = G.render(pkg, [seven(oracle, g, True)[0][0] for g in range(n_g)])
    assert maxdiff(got, want) <= TOL, maxdiff(got, want)


def test_thousand_graphs(pkg, engine, oracle):
    """1000 graphs of three bound curves (pitch, cutoff, loudness), rendered by run and run_pipelined"""
    torch = pytest.importorskip("torch")
    n, frames, cl = 1000, 4096, 64

    def make(be, g, vals):
        c = pkg.OfflineAudioContext(2, frames, SR, be)
        o = c.create_oscillator(type_=pkg.context.SAWTOOTH)
        bq = c.create_biquad_filter(type_=pkg.LOWPASS, q=1.0)
        gn = c.create_gain()
        prms = [o.frequency, bq.frequency, gn.gain]
        for p, v in zip(prms, vals or [None] * 3):
            if v is None:
                p.set_device_value_curve(cl, 0.0, frames / SR)
            else:
                p.set_value_curve_at_time(v, 0.0, frames / SR)
        o.connect(bq)
        bq.connect(gn)
        gn.connect(c.destination())
        o.start()
        return c, prms
    gen = torch.Generator().manual_seed(9)
    f0 = (110.0 + 440.0 * torch.rand((n, cl), generator=gen)).cuda()
    cut = (500.0 + 4000.0 * torch.rand((n, cl), generator=gen)).cuda()
    loud = torch.rand((n, cl), generator=gen).cuda()
    made = [make(engine.backend, g, None) for g in range(n)]
    b = pkg.Batch([c for c, _ in made])
    assert len(b.groups()) > 1
    b.bind_value_curves(made[0][1], [f0, cut, loud])
    got = run(b)
    host = [t.cpu().numpy() for t in (f0, cut, loud)]
    tw = run(pkg.Batch([make(engine.backend, g, [h[g] for h in host])[0] for g in range(n)]))
    assert np.array_equal(bits(got), bits(tw))
    ids = [0, 1, 511, 999]
    want = G.render(pkg, [make(oracle, g, [h[g] for h in host])[0] for g in ids])
    assert max(maxdiff(got[i], w) for i, w in zip(ids, want)) <= TOL
    out = torch.empty((n, 2, frames), dtype=torch.float32, pin_memory=True)
    b.run_pipelined(out.data_ptr())
    assert np.array_equal(bits(out.numpy()), bits(got))
