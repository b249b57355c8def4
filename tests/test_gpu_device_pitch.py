"""OscillatorNode frequency and detune bound from device memory (wae_param_set_device_value + wae_batch_bind_params) on the GPU.  Every
case is rendered three ways: bound from a torch tensor, host-built with the same values, and on the oracle.  Every render is within 1e-5
of the oracle, and bit-equal to the host-built render when the detune is 0 and both plans take the same stages (a nonzero detune may
move the last bit of the phase increment: CUDA's exp2 against glibc's)."""
import contextlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
TOL = 1e-5
SR = 48000.0
LENGTH = 9600
F_RANGE = (20.0, 16000.0)
D_RANGE = (-1200.0, 600.0)
# pitches of the graphs of a batch: low, fractional, around the lowpass, high (16000 * 2^(600/1200) < Nyquist)
FREQS = [55.0, 220.5, 1000.0, 3333.3, 12000.0]
TYPES = {"sine": 0, "square": 1, "sawtooth": 2, "triangle": 3}


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


def custom_table():
    x = 2.0 * np.pi * np.arange(8192) / 8192.0
    return ((np.sin(x) + 0.3 * np.sin(3.0 * x) + 0.1 * np.cos(5.0 * x)) / 1.4).astype(np.float32)


def run(batch):
    batch.run()
    batch.sync()
    return batch.fetch()


def maxdiff(a, b):
    return float(np.abs(a.astype(np.float64) - b.astype(np.float64)).max())


def stage_names(batch):
    return sorted((name, k) for name, _t, k in batch.stage_times())


def clamp(v, lo, hi, default):
    return default if not np.isfinite(v) else min(max(float(np.float32(v)), lo), hi)


def make(pkg, be, spec, pitch, declare):
    """spec["type"] oscillator -> spec["tail"] -> destination, at pitch = (frequency, detune) for each of spec["voices"] voices (a list
    of pitches then).  `declare`: frequency and detune (spec["bind"]: "f", "d" or "fd") declared with F_RANGE / D_RANGE, planned with
    placeholders of their own; the host twin sets the pitch."""
    c = pkg.OfflineAudioContext(2, LENGTH, SR, be)
    voices = spec.get("voices", 0)
    pitches = pitch if voices else [pitch]
    port = c.destination()
    if voices:
        port = c.create_gain(1.0 / voices)
        port.connect(c.destination())
    oscs = []
    for v, (f, d) in enumerate(pitches):
        osc = c.create_oscillator()
        if spec.get("type", "sawtooth") == "custom":
            osc.set_periodic_wave(custom_table())
        elif spec.get("type") == "device_wave":  # (the oracle plays the wavetable the bind synthesises)
            if c._api.is_product:
                osc.set_device_periodic_wave(8, 8192)
            else:
                osc.set_periodic_wave(spec["wave_table"])
        else:
            osc.set_type(TYPES[spec.get("type", "sawtooth")])
        bind = spec.get("bind", "f")
        if declare and "f" in bind:
            osc.frequency.set_value(700.0)  # (the placeholder: any value, the bound one replaces it)
            osc.frequency.set_device_value(*F_RANGE)
        else:
            osc.frequency.set_value(f)
        if declare and "d" in bind:
            osc.detune.set_device_value(*D_RANGE)
        elif not spec.get("lfo"):
            osc.detune.set_value(d)
        if spec.get("lfo"):  # an LFO on the detune: k_osc_arate
            lfo = c.create_oscillator(frequency=6.0)
            depth = c.create_gain(25.0)
            lfo.connect(depth)
            depth.connect(osc.detune)
            lfo.start()
        if spec.get("curve"):  # a device value curve on the frequency (its host twin: the same values as a host curve)
            if declare:
                osc.frequency.set_device_value_curve(2, 0.01, 0.1)
            else:
                osc.frequency.set_value_curve_at_time(np.array(spec["curve"], np.float32), 0.01, 0.1)
        last = osc
        tail = spec.get("tail", "chain")
        if tail in ("chain", "direct"):
            bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=1800.0 + 50.0 * v, q=2.0)
            last.connect(bq)
            last = bq
        if tail == "chain":
            gn = c.create_gain(0.6)
            last.connect(gn)
            last = gn
        if tail == "split":  # two consumers
            g2 = c.create_gain(0.3)
            osc.connect(g2)
            g2.connect(port)
        last.connect(port)
        start = spec.get("start", 0.0)
        if spec.get("schedule"):
            osc.start_at(0.0 if declare else start)
            if declare:
                osc.set_device_schedule((0.0, 0.2))
        else:
            osc.start_at(start)
        oscs.append(osc)
    return c, oscs


def bound_values(rows, spec):
    """the [graphs][params] tensor of bind_params for rows of (f, d) per voice"""
    cols = []
    for row in rows:
        pitches = row if spec.get("voices") else [row]
        vals = []
        for f, d in pitches:
            if "f" in spec.get("bind", "f"):
                vals.append(f)
            if "d" in spec.get("bind", "f"):
                vals.append(d)
        cols.append(vals)
    return np.array(cols, np.float32)


def bound_params(spec, oscs):
    ps = []
    for o in oscs:
        if "f" in spec.get("bind", "f"):
            ps.append(o.frequency)
        if "d" in spec.get("bind", "f"):
            ps.append(o.detune)
    return ps


def host_pitch(row, spec):
    """the pitch the bind gives the host twin: clamped to the ranges, a non-finite value -> the default clamped to the range"""
    def one(p):
        f, d = p
        if "f" in spec.get("bind", "f"):
            f = clamp(f, *F_RANGE, default=min(max(440.0, F_RANGE[0]), F_RANGE[1]))
        if "d" in spec.get("bind", "f"):
            d = clamp(d, *D_RANGE, default=0.0)
        return (f, d)
    return [one(p) for p in row] if spec.get("voices") else one(row)


def render_three(pkg, engine, oracle, spec, rows, opts=None, exact=None, extra_bind=None):
    """bound / host-built / oracle renders of one graph per row; returns (bound, twin, oracle)"""
    torch = pytest.importorskip("torch")
    opts = opts or {}
    n = len(rows)
    with options(pkg, engine, **opts):
        made = [make(pkg, engine.backend, spec, rows[i], True) for i in range(n)]
        b = pkg.Batch([c for c, _ in made])
        twins = [make(pkg, engine.backend, spec, host_pitch(rows[i], spec), False)[0] for i in range(n)]
        tw = pkg.Batch(twins)
    try:
        if extra_bind:
            extra_bind(b, made, tw)
        b.bind_params(bound_params(spec, made[0][1]), torch.from_numpy(bound_values(rows, spec)).cuda())
        got = run(b)
        twin = run(tw)
        stages = (stage_names(b), stage_names(tw))
    finally:
        b.destroy()
        tw.destroy()
    want = np.stack([np.stack(x.channels) for x in
                     pkg.render_batch([make(pkg, oracle, spec, host_pitch(rows[i], spec), False)[0] for i in range(n)])])
    assert np.isfinite(got).all()
    assert maxdiff(got, want) <= TOL, (spec, maxdiff(got, want))
    assert maxdiff(twin, want) <= TOL
    if exact is None:
        exact = not spec.get("voices") and all(host_pitch(r, spec)[1] == 0.0 for r in rows)
    if exact:
        assert stages[0] == stages[1], stages
        assert np.array_equal(got, twin), (spec, maxdiff(got, twin))
    print(f"{spec}: max |bound - twin| = {maxdiff(got, twin):.3e}, max |bound - oracle| = {maxdiff(got, want):.3e}")
    return got, twin, want


# ---- the fused chain, every oscillator type -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("type_", ["sine", "square", "sawtooth", "triangle", "custom"])
def test_fused_chain(pkg, engine, oracle, type_):
    got, _, want = render_three(pkg, engine, oracle, dict(type=type_), [(f, 0.0) for f in FREQS])
    assert float(np.abs(want).max()) > 1e-2


@pytest.mark.parametrize("type_", ["sine", "sawtooth", "custom"])
def test_fused_chain_with_detune(pkg, engine, oracle, type_):
    rows = [(f, d) for f, d in zip(FREQS, (-1100.0, -7.5, 0.0, 13.25, 550.0))]
    render_three(pkg, engine, oracle, dict(type=type_, bind="fd"), rows)
    render_three(pkg, engine, oracle, dict(type=type_, bind="d"), [(440.0, d) for _, d in rows])


def test_destination_direct(pkg, engine, oracle):
    render_three(pkg, engine, oracle, dict(type="square", tail="direct"), [(f, 0.0) for f in FREQS])


@pytest.mark.parametrize("type_", ["sine", "square", "custom"])
def test_unfused_oscillator(pkg, engine, oracle, type_):
    """fusion off: k_oscillator, its output read by two consumers"""
    with options(pkg, engine, fuse=0):
        c, _ = make(pkg, engine.backend, dict(type=type_, tail="split"), (440.0, 0.0), True)
        b = pkg.Batch([c])
        assert "k_oscillator" in {name for name, _ in stage_names(b)}
        b.destroy()
    render_three(pkg, engine, oracle, dict(type=type_, tail="split"), [(f, 0.0) for f in FREQS], opts=dict(fuse=0))
    render_three(pkg, engine, oracle, dict(type=type_, tail="split", bind="fd"), [(f, 25.0) for f in FREQS], opts=dict(fuse=0))


def test_voice_sum_ports(pkg, engine, oracle):
    """k_voice_sum: eight voices per port, each with its own bound frequency and a nonzero bound detune"""
    rng = np.random.default_rng(11)
    rows = [[(float(rng.uniform(60, 2000)), float(rng.uniform(-50, 50))) for _ in range(8)] for _ in range(3)]
    spec = dict(voices=8, bind="fd", type="sawtooth")
    with options(pkg, engine, voice_sum=2):
        c, _ = make(pkg, engine.backend, spec, rows[0], True)
        b = pkg.Batch([c])
        assert "k_voice_sum" in {name for name, _ in stage_names(b)}
        b.destroy()
    render_three(pkg, engine, oracle, spec, rows, opts=dict(voice_sum=2))
    # the same voices with detune 0: bit-equal to the host twin
    rows0 = [[(f, 0.0) for f, _ in r] for r in rows]
    render_three(pkg, engine, oracle, spec, rows0, opts=dict(voice_sum=2), exact=True)


# ---- k_osc_arate -------------------------------------------------------------------------------------------------------------------
def test_arate_bound_frequency_with_an_lfo_on_detune(pkg, engine, oracle):
    render_three(pkg, engine, oracle, dict(type="sine", lfo=True), [(f, 0.0) for f in FREQS], exact=True)


def test_arate_bound_detune_under_a_device_value_curve(pkg, engine, oracle):
    torch = pytest.importorskip("torch")
    curve = [300.0, 900.0]
    spec = dict(type="triangle", bind="d", curve=curve)

    def bind_curve(b, made, tw):
        b.bind_value_curves(made[0][1][0].frequency, torch.tensor([curve] * len(made), dtype=torch.float32).cuda())
    render_three(pkg, engine, oracle, spec, [(440.0, d) for d in (-1200.0, -5.0, 0.0, 31.0, 600.0)], extra_bind=bind_curve, exact=False)
    render_three(pkg, engine, oracle, spec, [(440.0, 0.0)] * 3, extra_bind=bind_curve, exact=True)


# ---- starts, waves, schedules ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("start", [0.01234, 2560 / SR + 0.3 / SR, 0.15])
def test_late_sub_sample_starts(pkg, engine, oracle, start):
    render_three(pkg, engine, oracle, dict(type="square", start=start), [(f, 0.0) for f in FREQS])
    render_three(pkg, engine, oracle, dict(type="sawtooth", start=start, tail="split"), [(f, 0.0) for f in FREQS], opts=dict(fuse=0))


def test_declared_periodic_wave_and_pitch(pkg, engine, oracle):
    torch = pytest.importorskip("torch")
    from test_gpu_device_waves import read_out
    rng = np.random.default_rng(5)
    re, im = rng.uniform(-1, 1, 8).astype(np.float32), rng.uniform(-1, 1, 8).astype(np.float32)
    re[0] = im[0] = 0.0
    table = read_out(pkg, engine, torch, [re], [im], 8192)[0]
    spec = dict(type="device_wave", wave_table=table)

    def bind_waves(b, made, tw):  # (the host twin declares and binds the same wave)
        n = len(made)
        for batch in (b, tw):
            batch.bind_periodic_waves(made[0][1][0], torch.from_numpy(np.stack([re] * n)).cuda(), torch.from_numpy(np.stack([im] * n)).cuda())
    render_three(pkg, engine, oracle, spec, [(f, 0.0) for f in FREQS], extra_bind=bind_waves)
    render_three(pkg, engine, oracle, dict(spec, tail="split"), [(f, 0.0) for f in FREQS], extra_bind=bind_waves, opts=dict(fuse=0))


@pytest.mark.parametrize("order", ["schedule_first", "pitch_first"])
def test_declared_schedule_and_pitch(pkg, engine, oracle, order):
    """a melody note: its start and its pitch bound, in either order, then each rebound alone"""
    torch = pytest.importorskip("torch")
    starts = [0.0, 0.0123, 2560 / SR, 0.0377 + 0.25 / SR, 0.1]
    for tail, opts in (("chain", {}), ("split", dict(fuse=0))):
        for bind in ("f", "fd"):
            spec = dict(type="sawtooth", tail=tail, bind=bind, schedule=True)
            rows = [(f, 0.0 if bind == "f" else 17.0) for f in FREQS]
            n = len(rows)
            with options(pkg, engine, **opts):
                made = [make(pkg, engine.backend, spec, rows[i], True) for i in range(n)]
                b = pkg.Batch([c for c, _ in made])
                tw = pkg.Batch([make(pkg, engine.backend, dict(spec, start=starts[i]), rows[i], False)[0] for i in range(n)])
            node = made[0][1][0]
            values = torch.from_numpy(bound_values(rows, spec)).cuda()
            wrong = torch.from_numpy(bound_values([(f * 1.5, 0.0) for f, _ in rows], spec)).cuda()
            st = torch.tensor(starts, dtype=torch.float64).cuda()
            st_wrong = torch.tensor([s + 0.01 for s in starts], dtype=torch.float64).cuda()
            try:
                if order == "schedule_first":
                    b.bind_schedules(node, st)
                    b.bind_params(bound_params(spec, made[0][1]), values)
                else:
                    b.bind_params(bound_params(spec, made[0][1]), values)
                    b.bind_schedules(node, st)
                got = run(b)
                twin = run(tw)
                # each rebound alone: a wrong value, then the right one again
                b.bind_params(bound_params(spec, made[0][1]), wrong)
                b.bind_params(bound_params(spec, made[0][1]), values)
                again = run(b)
                b.bind_schedules(node, st_wrong)
                b.bind_schedules(node, st)
                again2 = run(b)
            finally:
                b.destroy()
                tw.destroy()
            want = np.stack([np.stack(x.channels) for x in pkg.render_batch(
                [make(pkg, oracle, dict(spec, start=starts[i]), rows[i], False)[0] for i in range(n)])])
            assert maxdiff(got, want) <= TOL, (spec, maxdiff(got, want))
            if bind == "f":  # (a twin started at 0 plays ungated, a declared source is always gated: compared where both are)
                late = [i for i in range(n) if starts[i] > 0.0]
                assert np.array_equal(got[late], twin[late]), (spec, order, maxdiff(got[late], twin[late]))
            assert np.array_equal(got, again) and np.array_equal(got, again2), spec


# ---- chunks, rebinding, clamping, refusals ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("chunk", [128, 1024, 0])
def test_chunks(pkg, engine, oracle, chunk):
    render_three(pkg, engine, oracle, dict(type="sawtooth", start=0.0123), [(f, 0.0) for f in FREQS], opts=dict(chunk=chunk))


def test_rebinding_a_b_a(pkg, engine, oracle):
    torch = pytest.importorskip("torch")
    spec = dict(type="sawtooth", bind="fd", start=0.0071)
    a = [(f, 0.0) for f in FREQS]
    bb = [(f * 0.75, -3.0) for f in FREQS]
    made = [make(pkg, engine.backend, spec, a[i], True) for i in range(len(a))]
    b = pkg.Batch([c for c, _ in made])
    params = bound_params(spec, made[0][1])
    outs = []
    try:
        for rows in (a, bb, a):
            b.bind_params(params, torch.from_numpy(bound_values(rows, spec)).cuda())
            outs.append(run(b).copy())
    finally:
        b.destroy()
    assert np.array_equal(outs[0], outs[2])
    assert not np.array_equal(outs[0], outs[1])
    _, twin, _ = render_three(pkg, engine, oracle, spec, bb, exact=False)
    assert maxdiff(outs[1], twin) <= TOL


def test_clamped_and_non_finite_values(pkg, engine, oracle):
    # below / above the ranges -> clamped; NaN / inf -> the default (440 Hz, 0 cents) clamped to the range
    rows = [(1.0, 0.0), (50000.0, 0.0), (float("nan"), 0.0), (float("inf"), 0.0), (-float("inf"), 0.0)]
    render_three(pkg, engine, oracle, dict(type="square", bind="fd"), rows)
    rows = [(300.0, -5000.0), (300.0, 9000.0), (300.0, float("nan"))]
    render_three(pkg, engine, oracle, dict(type="square", bind="fd"), rows, exact=False)


def test_default_clamped_into_a_range_without_it(pkg, engine, oracle):
    """a non-finite frequency in a range that does not hold the default (440 Hz) takes the range's nearest end"""
    torch = pytest.importorskip("torch")
    c = pkg.OfflineAudioContext(2, LENGTH, SR, engine.backend)
    osc = c.create_oscillator()
    osc.frequency.set_device_value(1000.0, 2000.0)
    osc.connect(c.destination())
    osc.start()
    b = pkg.Batch([c])
    try:
        b.bind_params([osc.frequency], torch.tensor([float("nan")], dtype=torch.float32).cuda())
        got = run(b)
    finally:
        b.destroy()
    t = pkg.OfflineAudioContext(2, LENGTH, SR, oracle)
    o = t.create_oscillator(frequency=1000.0)
    o.connect(t.destination())
    o.start()
    want = np.stack(pkg.render_batch([t])[0].channels)
    assert maxdiff(got[0], want) <= TOL


def test_runs_refused_until_the_bind(pkg, engine):
    torch = pytest.importorskip("torch")
    spec = dict(type="sine", bind="fd")
    made = [make(pkg, engine.backend, spec, (440.0, 0.0), True) for _ in range(2)]
    b = pkg.Batch([c for c, _ in made])
    try:
        with pytest.raises(Exception) as e:
            b.run()
        assert e.value.status == 2 and "wae_batch_bind_params" in str(e.value)
        b.bind_params(bound_params(spec, made[0][1]), torch.tensor([[440.0, 0.0]] * 2, dtype=torch.float32).cuda())
        run(b)
    finally:
        b.destroy()
