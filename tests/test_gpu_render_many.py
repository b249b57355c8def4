"""wae_render_many / wae_batch_prepare_many on the GPU: one call for OfflineAudioContexts of different lengths, channel counts and sample
rates.  Every graph matches the oracle (1e-5) and is bit-equal to its render alone; a graph shorter than its group reads out (analyser,
compressor) what it reads out alone — the kernels stop its state at its own end — and the work items of k_chain and the convolver
kernels past its end exit without changing what it renders."""
import numpy as np
import pytest

import graphs as G

pytestmark = pytest.mark.gpu
TOL = 1e-5
CHUNK = 8 * 8192  # one chunk size for every render compared bit for bit (a lone graph would otherwise get its own automatic chunk)
FED = 110000      # frames of the sources that run past the end of the shorter graphs


def noise(seed, ch, frames, amp=0.5):
    return np.random.default_rng(seed).uniform(-amp, amp, (ch, frames)).astype(np.float32)


def source(pkg, c, seed, ch, frames, start=0.0):
    s = c.create_buffer_source(pkg.AudioBuffer(list(noise(seed, ch, frames)), c.sample_rate()))
    s.start_at(start)
    return s


def build(pkg, be, kind, i, ch, length, sr):
    c = pkg.OfflineAudioContext(ch, length, sr, be)
    d = c.destination()
    if kind == "c2":
        return G.c2_buffer_biquad_gain(pkg, be, i, length, sr) if ch == 2 else _c2_other(pkg, be, c, i, length, sr)
    if kind in ("conv2", "conv1", "conv4", "conv_fed"):
        n_ir = {"conv2": 2, "conv1": 1, "conv4": 4, "conv_fed": 2}[kind]
        cv = c.create_convolver(pkg.AudioBuffer(G.synthetic_ir(9000, n_ir, seed=i), sr))
        # (conv_fed: the source runs past the graph's end, so the group feeds the convolver there)
        source(pkg, c, i, 2, FED if kind == "conv_fed" else min(length, 30000)).connect(cv)
        cv.connect(d)
    elif kind == "chain_fed":  # buffer source -> biquad -> gain, the source longer than the graph
        bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=700.0 + 50 * i, q=2.0)
        gn = c.create_gain(0.8)
        source(pkg, c, 500 + i, 2, FED).connect(bq)
        bq.connect(gn)
        gn.connect(d)
    elif kind == "hrtf":
        o = c.create_oscillator(type_=pkg.SAWTOOTH, frequency=200.0 + 10 * i)
        p = c.create_panner(panning_model=pkg.context.HRTF, position=(1.0, 0.3, -0.5))
        o.connect(p)
        p.connect(d)
        o.start()
    elif kind == "feedback":
        s = source(pkg, c, i, 1, 6000)
        g = c.create_gain(1.0)
        dl = c.create_delay(0.5, 0.0123 + 0.001 * (i % 5))
        fb = c.create_gain(0.6)
        s.connect(g)
        g.connect(dl)
        dl.connect(fb)
        fb.connect(g)
        g.connect(d)
    elif kind in ("os2", "os4"):
        o = c.create_oscillator(frequency=330.0 + 7 * i)
        sh = c.create_wave_shaper(curve=np.tanh(np.linspace(-3, 3, 129)).astype(np.float32), oversample=1 if kind == "os2" else 2)
        o.connect(sh)
        sh.connect(d)
        o.start()
    elif kind == "analyser":
        o = c.create_oscillator(type_=pkg.SAWTOOTH, frequency=97.0 + 13 * i)
        g = c.create_gain(0.2)
        g.gain.linear_ramp_to_value_at_time(1.0, length / sr)  # keeps changing past any shorter graph's end
        an = c.create_analyser(fft_size=32768)  # (the read-out spans almost the whole ring: frames past the end would land in it)
        o.connect(g)
        g.connect(an)
        an.connect(d)
        o.start()
        c._an = an
    elif kind == "compressor":
        s = source(pkg, c, i, 2, length)
        g = c.create_gain(0.1)
        g.gain.exponential_ramp_to_value_at_time(2.0, length / sr)
        cp = c.create_dynamics_compressor(threshold=-30.0, release=0.05)
        s.connect(g)
        g.connect(cp)
        cp.connect(d)
        c._cp = cp
    elif kind == "suspend":
        s = source(pkg, c, i, 2, length)
        g = c.create_gain(0.7)
        s.connect(g)
        g.connect(d)
        c.suspend_sync((1280 - 0.5) / sr, lambda ctx: g.gain.set_value(0.25))
        c.suspend_sync((4096 - 0.5) / sr, lambda ctx: (lambda o: (o.connect(d), o.start()))(ctx.create_oscillator(frequency=500.0)))
    return c


def _c2_other(pkg, be, c, i, length, sr):
    _, f0, q, gain = G.c2_params(i)
    s = source(pkg, c, 1000 + i, 2, length)
    bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=f0, q=q)
    gn = c.create_gain(gain)
    s.connect(bq)
    bq.connect(gn)
    gn.connect(c.destination())
    return c


KINDS = ["c2"] * 14 + ["conv2", "conv1", "conv4"] * 3 + ["hrtf"] * 4 + ["feedback"] * 4 + ["os2", "os4"] * 3 + ["analyser"] * 5 + \
        ["compressor"] * 5 + ["suspend"] * 4


def specs():
    rng = np.random.default_rng(2024)
    out = []
    for i, kind in enumerate(KINDS):
        sr = [44100.0, 48000.0][i % 2] if kind != "conv1" else 48000.0
        ch = int(rng.choice([1, 2, 6])) if kind in ("c2", "feedback", "os2") else 2
        length = int(rng.integers(2000, 70000))
        if kind in ("analyser", "compressor"):
            length = [40000, 37000, 33000, 31000, 30500][i % 5]  # several lengths inside one group
        out.append((kind, i, ch, length, sr))
    return out


@pytest.fixture(scope="module")
def spheres(engine, oracle):
    sphere = G.synthetic_hrir_sphere(44100, 256)  # contexts at 48 kHz resample it
    engine.backend.set_hrir_sphere(sphere)
    oracle.set_hrir_sphere(sphere)


@pytest.fixture(scope="module")
def chunked(pkg, engine):
    engine.set_option(pkg.OPT_CHUNK_FRAMES, CHUNK)
    yield
    engine.set_option(pkg.OPT_CHUNK_FRAMES, 0)


def guarded(ctxs, alloc=None):
    """one NaN-filled array per context with 64 floats of guard tail"""
    out = []
    for k, c in enumerate(ctxs):
        n = c._channels * c.length() + 64
        a = alloc(k, n) if alloc else np.empty(n, np.float32)
        a[:] = np.nan
        out.append(a)
    return out


def pcm(buf):
    return np.stack(buf.channels) if buf.channels else np.zeros((0, 0), np.float32)


def test_mixed_batch_matches_oracle_and_alone_renders(pkg, engine, oracle, spheres, chunked):
    import torch
    sp = specs()
    ctxs = [build(pkg, engine.backend, *s) for s in sp]
    # (the host-only planner has no HRIR sphere: the grouping of the other graphs)
    plan = pkg.context.plan_many([c for s, c in zip(sp, ctxs) if s[0] != "hrtf"])
    assert plan["groups"] > 1 and plan["rendered_quanta"] > plan["needed_quanta"]
    outs = guarded(ctxs)
    got = [pcm(b) for b in pkg.render_many(ctxs, outs)]
    for c, o in zip(ctxs, outs):
        assert np.isnan(o[c._channels * c.length():]).all()
    for (kind, i, ch, length, sr), g in zip(sp, got):
        assert g.shape == (ch, length) and np.isfinite(g).all(), kind
    # the oracle, context by context
    want = [pcm(b) for b in pkg.render_many([build(pkg, oracle, *s) for s in sp])]
    for s, g, w in zip(sp, got, want):
        err = float(np.abs(g.astype(np.float64) - w).max()) if g.size else 0.0
        assert err <= TOL, (s, err)
    # page-locked and pageable buffers in one call (every other one pinned): the same bits
    keep = []

    def alloc(k, n):
        if k % 2:
            return np.empty(n, np.float32)
        t = torch.empty(n, dtype=torch.float32, pin_memory=True)
        keep.append(t)
        return t.numpy()
    outs2 = guarded(ctxs, alloc)
    again = [pcm(b) for b in pkg.render_many(ctxs, outs2)]
    for c, o in zip(ctxs, outs2):
        assert np.isnan(o[c._channels * c.length():]).all()
    for g, a in zip(got, again):
        assert np.array_equal(g, a)
    # each graph alone, in a batch of one shape: bit-equal
    for s, c, g in zip(sp, ctxs, got):
        assert np.array_equal(pkg.render_batch_oneshot([c])[0], g), s


@pytest.mark.parametrize("chunk", [CHUNK, 8192])
def test_shorter_graphs_read_out_their_own_end(pkg, engine, oracle, chunk):
    """analyser and compressor graphs of several lengths in one group (plus a longer c2 graph so that every one of them is shorter than
    its group): time-domain and frequency data, float and byte, and the compressor's reduction equal the oracle's.  The analysers read
    32768 frames of a 32896-frame ring, so a few hundred frames recorded past a graph's end would show; with 8192-frame chunks the
    shorter graphs end chunks before their group does."""
    engine.set_option(pkg.OPT_CHUNK_FRAMES, chunk)
    sp = [("analyser", i, 2, n, 48000.0) for i, n in enumerate([40000, 37000, 33000, 31000])] + \
         [("compressor", 10 + i, 2, n, 48000.0) for i, n in enumerate([40000, 36000, 32000, 30500])] + \
         [("c2", 20, 2, 40500, 48000.0)]
    ctxs = [build(pkg, engine.backend, *s) for s in sp]
    ref = [build(pkg, oracle, *s) for s in sp]
    group_of = pkg.context.plan_many(ctxs)["group_of"]
    assert len(set(group_of)) == 1
    b = pkg.context.Batch(ctxs, many=True)
    b.run()
    b.sync()
    pkg.render_many(ref)
    for k, (s, c, r) in enumerate(zip(sp, ctxs, ref)):
        got = b.fetch_graph(k)
        if s[0] == "analyser":
            x, y = c._an.get_float_time_domain_data(), r._an.get_float_time_domain_data()
            assert float(np.abs(x.astype(np.float64) - y).max()) <= TOL, s
            # frequency data as tests/test_gpu_parity.py holds it: magnitudes, and dB where the bin is above the noise floor
            fg, fc = c._an.get_float_frequency_data(), r._an.get_float_frequency_data()
            lin_g, lin_c = 10.0 ** (fg.astype(np.float64) / 20), 10.0 ** (fc.astype(np.float64) / 20)
            assert np.abs(lin_g - lin_c).max() <= 1e-6, s
            loud = lin_c > 1e-4
            assert loud.any() and np.abs(fg[loud] - fc[loud]).max() <= 1e-2, s
            for name in ("get_byte_time_domain_data", "get_byte_frequency_data"):
                x, y = getattr(c._an, name)(), getattr(r._an, name)()
                assert np.abs(x.astype(int) - y.astype(int)).max() <= 1, (s, name)
        if s[0] == "compressor":
            assert abs(c._cp.reduction() - r._cp.reduction()) <= 1e-4, s
        assert got.shape == (2, s[3])
    engine.set_option(pkg.OPT_CHUNK_FRAMES, 0)


@pytest.mark.parametrize("chunk", [CHUNK, 8192])
def test_padding_spans_slabs_and_partitions(pkg, engine, oracle, chunk):
    """graphs fed past their end in a group up to 3 convolver partitions (24k frames) longer: the k_chain slabs (filtered chains in few
    instances: time slabs, early-published hand-offs) and the convolver blocks past each graph's end exit, and every graph still matches
    the oracle and its lone render bit for bit.  With 8192-frame chunks whole chunks of the shorter graphs are past their end."""
    engine.set_option(pkg.OPT_CHUNK_FRAMES, chunk)
    try:
        sp = [(kind, i, 2, n, 48000.0) for i, (kind, n) in enumerate(
            [("chain_fed", 100000), ("chain_fed", 76000), ("chain_fed", 88888), ("conv_fed", 100000), ("conv_fed", 75500), ("conv_fed", 90001)])]
        ctxs = [build(pkg, engine.backend, *s) for s in sp]
        plan = pkg.context.plan_many(ctxs)
        assert len(set(plan["group_of"])) == 1 and "k_chain" in plan["kinds"] and "k_conv_fft_in" in plan["kinds"]
        got = [pcm(b) for b in pkg.render_many(ctxs)]
        want = [pcm(b) for b in pkg.render_many([build(pkg, oracle, *s) for s in sp])]
        for s, c, g, w in zip(sp, ctxs, got, want):
            assert float(np.abs(g.astype(np.float64) - w).max()) <= TOL, s
            assert np.array_equal(pkg.render_batch_oneshot([c])[0], g), s
    finally:
        engine.set_option(pkg.OPT_CHUNK_FRAMES, 0)


def test_prepared_mixed_batch_outputs(pkg, engine, chunked):
    """fetch_graph(i) and the packed device output at graph_output(i) equal wae_render_many's PCM; the packed host calls refuse"""
    import torch
    sp = [("c2", i, [1, 2, 6][i % 3], 5000 + 3777 * i, [44100.0, 48000.0][i % 2]) for i in range(9)]
    ctxs = [build(pkg, engine.backend, *s) for s in sp]
    want = [pcm(x) for x in pkg.render_many(ctxs)]
    b = pkg.context.Batch(ctxs, many=True)
    b.run()
    b.sync()
    p, n_floats = b.device_ptr()
    assert n_floats == sum(c._channels * c.length() for c in ctxs)

    class _W:
        __cuda_array_interface__ = {"shape": (n_floats,), "typestr": "<f4", "data": (p, False), "version": 2}
    packed = torch.as_tensor(_W(), device="cuda").cpu().numpy()
    for k, (c, w) in enumerate(zip(ctxs, want)):
        assert np.array_equal(b.fetch_graph(k), w)
        off, ch, length = b.graph_output(k)
        assert (ch, length) == (c._channels, c.length())
        assert np.array_equal(packed[off:off + ch * length].reshape(ch, length), w)
    with pytest.raises(pkg.WaeError) as e:
        b.fetch()
    assert e.value.status == 2 and "wae_batch_fetch_graph" in str(e.value)
    b.destroy()


def test_uniform_batch_through_render_many_is_the_oneshot_render(pkg, engine):
    ctxs = [G.c2_buffer_biquad_gain(pkg, engine.backend, g, 12800) for g in range(70)]
    one = pkg.render_batch_oneshot(ctxs)
    many = pkg.render_many(ctxs)
    for k in range(len(ctxs)):
        assert np.array_equal(one[k], pcm(many[k]))
