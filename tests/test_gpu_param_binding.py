"""Params bound from device memory (wae_param_set_device_value + wae_batch_bind_params) on the GPU.  A batch is planned once and run
with several parameter sets bound from torch tensors; each render is compared with the oracle's render of graphs built with those values
as constants (1e-5), and, where no transcendental function is involved, with the engine's own render of such graphs (bit-equal)."""
import ctypes as C

import numpy as np
import pytest

import graphs as G

pytestmark = pytest.mark.gpu
TOL = 1e-5
SR = 48000.0


def noise(seed, ch, frames, amp=0.5):
    return np.random.default_rng(seed).uniform(-amp, amp, (ch, frames)).astype(np.float32)


def run_bound(pkg, engine, oracle, build, values, length, n_params, bit_equal=False, batch=None, tol=TOL):
    """build(pkg, backend, i, vals, bound) -> (ctx, [params]).  Binds values[i] to graph i, runs, and compares every graph with the
    oracle (and with the engine's render of constant-valued twins when bit_equal).  Returns the batch for further rounds."""
    torch = pytest.importorskip("torch")
    n = len(values)
    if batch is None:
        made = [build(pkg, engine.backend, i, values[i], True) for i in range(n)]
        batch = (pkg.Batch([c for c, _ in made]), made[0][1])
    b, params = batch
    assert len(params) == n_params
    b.bind_params(params, torch.tensor(np.asarray(values, np.float32)).cuda())
    b.run()
    b.sync()
    got = [b.fetch_graph(i) for i in range(n)]
    want = [np.stack(x.channels) for x in pkg.render_batch([build(pkg, oracle, i, values[i], False)[0] for i in range(n)])]
    if bit_equal:
        twin = pkg.Batch([build(pkg, engine.backend, i, values[i], False)[0] for i in range(n)])
        twin.run()
        twin.sync()
        for i in range(n):
            assert np.array_equal(got[i], twin.fetch_graph(i)), (i, values[i])
    for i in range(n):
        assert tol is None or float(np.abs(got[i] - want[i]).max()) <= tol, (i, values[i])
    return batch


def declare(params, bound, ranges=None):
    if bound:
        for k, p in enumerate(params):
            lo, hi = (ranges or {}).get(k, (None, None))
            p.set_device_value(lo, hi)
    return params


def b_c2(length, btype=None):
    def build(pkg, be, i, v, bound):
        f, q, g, det, gain = v
        c = pkg.OfflineAudioContext(2, length, SR, be)
        s = c.create_buffer_source(pkg.AudioBuffer(list(noise(i, 2, length)), SR))
        bq = c.create_biquad_filter(type_=pkg.LOWPASS if btype is None else btype, frequency=f, q=q, gain=g, detune=det)
        gn = c.create_gain(gain)
        s.connect(bq)
        bq.connect(gn)
        gn.connect(c.destination())
        s.start()
        return c, declare([bq.frequency, bq.q, bq.gain, bq.detune, gn.gain], bound, {4: (0.05, 2.0)})
    return build


def c2_values(rng, n):
    return [[float(np.exp(rng.uniform(np.log(100.0), np.log(8000.0)))), float(rng.uniform(0.5, 4.0)), float(rng.uniform(-12, 12)),
             float(rng.uniform(-600, 600)), float(rng.uniform(0.1, 0.9))] for _ in range(n)]


def test_c2_rebind_three_times(pkg, engine, oracle):
    rng = np.random.default_rng(7)
    batch = None
    for _ in range(3):
        batch = run_bound(pkg, engine, oracle, b_c2(20000), c2_values(rng, 64), 20000, 5, batch=batch)


def test_gains_only_bit_equal(pkg, engine, oracle):
    def build(pkg, be, i, v, bound):
        c = pkg.OfflineAudioContext(2, 12000, SR, be)
        s = c.create_buffer_source(pkg.AudioBuffer(list(noise(i, 2, 12000)), SR))
        bq = c.create_biquad_filter(frequency=1200.0 + 100 * i)
        g1, g2 = c.create_gain(v[0]), c.create_gain(v[1])
        s.connect(g1)
        g1.connect(bq)
        bq.connect(g2)
        g2.connect(c.destination())
        s.start()
        return c, declare([g1.gain, g2.gain], bound, {0: (0.05, 4.0)})
    rng = np.random.default_rng(3)
    vals = [[float(rng.uniform(0.05, 4.0)), float(rng.uniform(-2, 2))] for _ in range(12)] + [[1.0, 1.0 + 1e-7], [0.5, 0.0]]
    run_bound(pkg, engine, oracle, build, vals, 12000, 2, bit_equal=True)


def test_compressor_only_bit_equal(pkg, engine, oracle):
    def build(pkg, be, i, v, bound):
        c = pkg.OfflineAudioContext(2, 12000, SR, be)
        s = c.create_buffer_source(pkg.AudioBuffer(list(noise(i, 2, 12000, 0.9)), SR))
        comp = c.create_dynamics_compressor(*v)
        s.connect(comp)
        comp.connect(c.destination())
        s.start()
        return c, declare([comp.attack, comp.knee, comp.ratio, comp.release, comp.threshold], bound)
    rng = np.random.default_rng(4)
    vals = [[float(rng.uniform(0, 0.1)), float(rng.uniform(0, 40)), float(rng.uniform(1, 20)), float(rng.uniform(0, 1)),
             float(rng.uniform(-60, 0))] for _ in range(8)]
    # Bit-equal to the same graphs built with constants.  Not compared with the oracle: with settings away from the defaults the
    # compressor's f32 log10 / pow chains (CUDA libm against glibc) put the engine's render of the constant graphs up to 3e-4 from it.
    run_bound(pkg, engine, oracle, build, vals, 12000, 5, bit_equal=True, tol=None)


@pytest.mark.parametrize("serial", [0, 1], ids=["scan", "serial"])
def test_every_biquad_type_and_edges(pkg, engine, oracle, serial):
    edges = [[0.0, 1.0, 6.0, 0.0, 1.0], [24000.0, 1.0, 6.0, 0.0, 1.0], [20000.0, 1.0, 6.0, 1200.0, 1.0], [1000.0, 0.0, 6.0, 0.0, 1.0],
             [1000.0, -3.0, -6.0, 0.0, 1.0], [700.0, 2.0, 9.0, -350.0, 1.0], [300.0, 0.7, -9.0, 35.0, 1.0]]
    engine.set_option(pkg.OPT_SERIAL_FILTERS, serial)
    try:
        for t in range(8):
            run_bound(pkg, engine, oracle, b_c2(6000, btype=t), edges, 6000, 5)
    finally:
        engine.set_option(pkg.OPT_SERIAL_FILTERS, 0)


def test_long_few_graphs(pkg, engine, oracle):
    rng = np.random.default_rng(5)
    run_bound(pkg, engine, oracle, b_c2(480000), c2_values(rng, 2), 480000, 5)


def test_voice_sum_into_bound_biquads(pkg, engine, oracle):
    def build(pkg, be, i, v, bound):
        c = pkg.OfflineAudioContext(2, 24000, SR, be)
        out = c.create_gain(0.1)
        ps = []
        for k in range(8):
            o = c.create_oscillator(type_=pkg.SAWTOOTH, frequency=110.0 * (k + 1) + i)
            bq = c.create_biquad_filter(frequency=v[k])
            g = c.create_gain(0.5)
            o.connect(bq)
            bq.connect(g)
            g.connect(out)
            o.start()
            ps.append(bq.frequency)
        out.connect(c.destination())
        return c, declare(ps, bound)
    rng = np.random.default_rng(6)
    engine.set_option(pkg.OPT_VOICE_SUM, 2)
    try:
        run_bound(pkg, engine, oracle, build, [[float(rng.uniform(200, 5000)) for _ in range(8)] for _ in range(3)], 24000, 8)
    finally:
        engine.set_option(pkg.OPT_VOICE_SUM, -1)


@pytest.mark.parametrize("ch", [1, 2])
def test_stereo_panner(pkg, engine, oracle, ch):
    def build(pkg, be, i, v, bound):
        c = pkg.OfflineAudioContext(2, 8000, SR, be)
        s = c.create_buffer_source(pkg.AudioBuffer(list(noise(i, ch, 8000)), SR))
        p = c.create_stereo_panner(v[0])
        s.connect(p)
        p.connect(c.destination())
        s.start()
        return c, declare([p.pan], bound)
    run_bound(pkg, engine, oracle, build, [[-1.0], [-0.3], [0.0], [0.4], [1.0], [0.77]], 8000, 1)


@pytest.mark.parametrize("fuse", [1, 0], ids=["fused", "unfused"])
def test_gain_about_zero(pkg, engine, oracle, fuse):
    def build(pkg, be, i, v, bound, lo=None):
        c = pkg.OfflineAudioContext(2, 8000, SR, be)
        s = c.create_buffer_source(pkg.AudioBuffer(list(noise(i, 2, 8000)), SR))
        g = c.create_gain(v[0])
        sh = c.create_wave_shaper(curve=np.array([0.25, 0.5, 0.75], np.float32))
        bq = c.create_biquad_filter(frequency=900.0)
        s.connect(g)
        g.connect(sh)
        sh.connect(bq)
        bq.connect(c.destination())
        s.start()
        return c, declare([g.gain], bound, {0: (lo, None)} if lo is not None else None)
    engine.set_option(pkg.OPT_FUSE, fuse)
    try:
        batch = run_bound(pkg, engine, oracle, build, [[0.0], [1e-7], [0.5], [-1e-7]], 8000, 1)
        run_bound(pkg, engine, oracle, build, [[0.3], [0.0], [2.0], [1e-7]], 8000, 1, batch=batch)  # (rebound both ways)
        excl = lambda pkg, be, i, v, bound: build(pkg, be, i, v, bound, lo=0.01)
        run_bound(pkg, engine, oracle, excl, [[0.3], [1.5]], 8000, 1, bit_equal=True)
    finally:
        engine.set_option(pkg.OPT_FUSE, 1)


def test_across_suspend_points(pkg, engine, oracle):
    def build(pkg, be, i, v, bound):
        c = pkg.OfflineAudioContext(2, 12000, SR, be)
        s = c.create_buffer_source(pkg.AudioBuffer(list(noise(i, 2, 12000)), SR))
        bq = c.create_biquad_filter(frequency=v[0])
        g = c.create_gain(v[1])
        s.connect(bq)
        bq.connect(g)
        g.connect(c.destination())
        s.start()
        ps = declare([bq.frequency, g.gain], bound)

        def cb(ctx):  # a second source joins at the suspend point
            s2 = ctx.create_buffer_source(pkg.AudioBuffer(list(noise(50 + i, 2, 4000)), SR))
            s2.connect(bq)
            s2.start()
        c.suspend_sync(5000 / SR, cb)
        return c, ps
    run_bound(pkg, engine, oracle, build, [[500.0, 0.3], [3000.0, 1.7], [9000.0, 0.0]], 12000, 2)


def test_combined_binds_in_a_loop(pkg, engine, oracle):
    torch = pytest.importorskip("torch")
    n, length = 16, 10000

    def build(pkg, be, i, v, pcm):
        c = pkg.OfflineAudioContext(2, length, SR, be)
        if pcm is None:
            s = c.create_buffer_source()
            s.set_device_input(2, length, SR)
        else:
            s = c.create_buffer_source(pkg.AudioBuffer(list(pcm), SR))
        bq = c.create_biquad_filter(frequency=v[0], q=v[1])
        g = c.create_gain(v[2])
        s.connect(bq)
        bq.connect(g)
        g.connect(c.destination())
        s.start()
        if pcm is None:
            declare([bq.frequency, bq.q, g.gain], True)
        return c, (s, [bq.frequency, bq.q, g.gain])
    made = [build(pkg, engine.backend, i, [1000.0, 1.0, 0.5], None) for i in range(n)]
    b = pkg.Batch([c for c, _ in made])
    src, params = made[0][1]
    gen = torch.Generator(device="cuda").manual_seed(11)
    for _ in range(3):
        pcm = torch.rand((n, 2, length), device="cuda", generator=gen) - 0.5  # (queued on torch's default stream)
        vals = torch.stack([torch.rand(n, device="cuda", generator=gen) * 5000 + 100, torch.rand(n, device="cuda", generator=gen) * 3 + 0.3,
                            torch.rand(n, device="cuda", generator=gen)], dim=1)
        b.bind_sources(src, pcm)
        b.bind_params(params, vals)
        b.run()
        out = b.output_tensor().clone()
        v, p = vals.cpu().numpy(), pcm.cpu().numpy()
        want = pkg.render_batch([build(pkg, oracle, i, [float(x) for x in v[i]], p[i])[0] for i in range(n)])
        got = out.cpu().numpy()
        for i in range(n):
            assert float(np.abs(got[i] - np.stack(want[i].channels)).max()) <= TOL, i


def test_errors(pkg, engine, oracle):
    torch = pytest.importorskip("torch")
    build = b_c2(4000)
    made = [build(pkg, engine.backend, i, [1000.0, 1.0, 0.0, 0.0, 0.5], True) for i in range(3)]
    b = pkg.Batch([c for c, _ in made])
    params = made[0][1]
    with pytest.raises(pkg.WaeError) as e:  # never bound
        b.run()
    assert e.value.status == 2 and "wae_batch_bind_params" in e.value.message
    api = pkg.api()
    host = np.ones(1, np.float32)
    item = pkg._binding.ParamBinding(0, params[0]._node, params[0]._index, pkg._binding.fptr(host))
    assert api.batch_bind_params(b.handle, C.byref(item), 1, None) == 1  # host memory
    dev = torch.ones(2, device="cuda")
    ptr = C.cast(C.c_void_p(dev.data_ptr()), pkg._binding.c_float_p)
    twice = (pkg._binding.ParamBinding * 2)(*[pkg._binding.ParamBinding(0, params[0]._node, params[0]._index, ptr)] * 2)
    assert api.batch_bind_params(b.handle, twice, 2, None) == 1
    undeclared = pkg._binding.ParamBinding(0, params[0]._node, 9, ptr)
    assert api.batch_bind_params(b.handle, C.byref(undeclared), 1, None) == 2
    out_of_range = pkg._binding.ParamBinding(7, params[0]._node, params[0]._index, ptr)
    assert api.batch_bind_params(b.handle, C.byref(out_of_range), 1, None) == 2
    torch.cuda.synchronize()
    # a non-finite value renders the param's default value (frequency 350, Q 1, gain 0, detune 0; the gain node's 1)
    nan = float("nan")
    vals = [[nan, 1.0, 0.0, 0.0, 0.5], [1000.0, float("inf"), 0.0, 0.0, 0.5], [1000.0, 1.0, 0.0, 0.0, nan]]
    b.bind_params(params, torch.tensor(vals, dtype=torch.float32).cuda())
    b.run()
    b.sync()
    want_vals = [[350.0, 1.0, 0.0, 0.0, 0.5], [1000.0, 1.0, 0.0, 0.0, 0.5], [1000.0, 1.0, 0.0, 0.0, 1.0]]
    want = pkg.render_batch([build(pkg, oracle, i, want_vals[i], False)[0] for i in range(3)])
    for i in range(3):
        assert float(np.abs(b.fetch_graph(i) - np.stack(want[i].channels)).max()) <= TOL, i
