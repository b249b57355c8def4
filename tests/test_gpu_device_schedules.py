"""Start / stop times of scheduled sources bound from device memory (wae_source_set_device_schedule + wae_batch_bind_schedules) on the
GPU.  Every case is rendered three ways: bound from a torch tensor, host-built with the same times, and on the oracle.  Every render is
within 1e-5 of the oracle, and bit-equal to the host-built render wherever both plans take the same stages."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
TOL = 1e-5
SR = 48000.0
LENGTH = 9600
END = LENGTH / SR
# starts at 0, mid-quantum, on a block boundary, one rounding below one, and after the render ends
STARTS = [0.0, 0.0123, 2560 / SR, float(np.nextafter(3840 / SR, 0.0)), END + 0.5]
# stops before the start, inside the first quantum, and at the render end
STOPS = [lambda s: max(0.0, s - 0.001), lambda s: s + 50 / SR, lambda s: END]
WIN = (0.0, END + 1.0)


def times_grid(with_stop):
    if not with_stop:
        return [(s, None) for s in STARTS]
    return [(s, f(s)) for s in STARTS for f in STOPS]


def noise(seed, ch, frames, amp=0.5):
    return np.random.default_rng(seed).uniform(-amp, amp, (ch, frames)).astype(np.float32)


def make(pkg, be, spec, t, declare, pcm=None):
    """spec['src'] (osc type / 'const' / 'absn') -> spec['tail'] -> destination, started at t = (start, stop); `declare`: the times
    declared with windows WIN and a placeholder start of 0"""
    c = pkg.OfflineAudioContext(2 if spec["src"] == "absn" else 1, LENGTH, SR, be)
    src = spec["src"]
    if src == "const":
        s = c.create_constant_source()
        s.offset.set_value(0.7)
    elif src == "absn":
        s = c.create_buffer_source(playback_rate=spec.get("rate", 1.0), loop=spec.get("loop", False))
        if spec.get("dev") and declare:
            s.set_device_input(pcm.shape[0], pcm.shape[1], SR)
        else:
            s.set_buffer(pkg.AudioBuffer(list(pcm), SR))
    else:
        s = c.create_oscillator()
        s.frequency.set_value(spec.get("freq", 440.0))
        if src == "custom":
            x = 2.0 * np.pi * np.arange(2048) / 2048.0
            s.set_periodic_wave(((np.sin(x) + 0.3 * np.sin(3.0 * x)) / 1.3).astype(np.float32))
        else:
            s.set_type({"sine": 0, "square": 1, "sawtooth": 2}[src])
    tail = spec.get("tail")
    last = s
    if tail == "lowpass":  # fused into k_chain
        bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=2000.0)
        s.connect(bq)
        last = bq
    elif tail == "shaper":  # a curve that does not map 0 to 0: every silent quantum of the source shows
        sh = c.create_wave_shaper(np.array([0.25, 0.5, 0.0], np.float32))
        s.connect(sh)
        last = sh
    elif tail == "split":  # two consumers: the source is rendered on its own (S_OSC / S_CONST) with a layout track
        g = c.create_gain(0.5)
        s.connect(g)
        g.connect(c.destination())
    last.connect(c.destination())
    start, stop = t
    if declare:
        s.start_at(0.0)
        s.set_device_schedule(WIN, stop=None if stop is None else WIN)
    else:
        s.start_at(start)
        if stop is not None:
            s.stop_at(stop)
    return c, s


def render_three(pkg, engine, oracle, spec, ts, chunk=None, pcms=None):
    """bound / host-built / oracle renders of one graph per t in ts; returns (bound renders, bit-equal count)"""
    torch = pytest.importorskip("torch")
    n = len(ts)
    pcms = pcms or [None] * n
    made = [make(pkg, engine.backend, spec, ts[i], True, pcms[i]) for i in range(n)]
    if chunk:
        engine.set_option(pkg.OPT_CHUNK_FRAMES, chunk)
    try:
        b = pkg.Batch([c for c, _ in made])
    finally:
        if chunk:
            engine.set_option(pkg.OPT_CHUNK_FRAMES, 0)
    node = made[0][1]
    if spec.get("dev"):
        b.bind_sources(node, torch.from_numpy(np.stack(pcms)).cuda())
    starts = torch.tensor([t[0] for t in ts], dtype=torch.float64).cuda()
    stops = None if ts[0][1] is None else torch.tensor([t[1] for t in ts], dtype=torch.float64).cuda()
    b.bind_schedules(node, starts, stops)
    b.run()
    b.sync()
    got = [b.fetch_graph(i) for i in range(n)]
    twins = [make(pkg, engine.backend, spec, ts[i], False, pcms[i])[0] for i in range(n)]
    tw = pkg.Batch(twins)
    tw.run()
    tw.sync()
    want = [np.stack(x.channels) for x in pkg.render_batch([make(pkg, oracle, spec, ts[i], False, pcms[i])[0] for i in range(n)])]
    bound_kinds = pkg.plan_batch([made[0][0]])["kinds"]
    equal = 0
    for i in range(n):
        ref = tw.fetch_graph(i)
        same = np.array_equal(got[i], ref)
        equal += same
        if pkg.plan_batch([twins[i]])["kinds"] == bound_kinds:
            assert same, (spec, ts[i], float(np.abs(got[i] - ref).max()))
        assert float(np.abs(got[i] - want[i]).max()) <= TOL, (spec, ts[i], float(np.abs(got[i] - want[i]).max()))
    return got, equal


OSC_SPECS = [dict(src=s, tail=t) for s in ("sine", "square", "sawtooth", "custom") for t in ("lowpass", "split", "shaper", None)]


@pytest.mark.parametrize("with_stop", [False, True], ids=["start", "start_stop"])
@pytest.mark.parametrize("spec", OSC_SPECS, ids=[f"{s['src']}-{s['tail']}" for s in OSC_SPECS])
def test_oscillator(pkg, engine, oracle, spec, with_stop):
    _, equal = render_three(pkg, engine, oracle, spec, times_grid(with_stop))
    print(f"{spec}: {equal} bit-equal")


def test_oscillator_high_frequency_polyblep(pkg, engine, oracle):
    """polyBLEP near a sub-sample start, and a frequency outside Nyquist"""
    for freq in (9000.0, 30000.0):
        render_three(pkg, engine, oracle, dict(src="square", tail="split", freq=freq), times_grid(True))


@pytest.mark.parametrize("tail", ["lowpass", "split", "shaper", None])
def test_constant_source(pkg, engine, oracle, tail):
    for with_stop in (False, True):
        render_three(pkg, engine, oracle, dict(src="const", tail=tail), times_grid(with_stop))


ABSN_SPECS = {
    "rate1": dict(src="absn", tail="shaper"),          # the fast-track copy inside the bound kernel where the start is aligned
    "rate09": dict(src="absn", tail="lowpass", rate=0.9),
    "loop": dict(src="absn", tail="shaper", loop=True),  # serial
    "dev": dict(src="absn", tail="shaper", dev=True),
    "dev_rate11": dict(src="absn", tail=None, dev=True, rate=1.1),
}


@pytest.mark.parametrize("with_stop", [False, True], ids=["start", "start_stop"])
@pytest.mark.parametrize("name", list(ABSN_SPECS))
def test_buffer_source(pkg, engine, oracle, name, with_stop):
    ts = times_grid(with_stop)
    pcms = [noise(10 + i, 2, 3000) for i in range(len(ts))]
    _, equal = render_three(pkg, engine, oracle, ABSN_SPECS[name], ts, pcms=pcms)
    print(f"{name}: {equal} of {len(ts)} bit-equal")


def test_voice_sum_mode(pkg, engine, oracle, monkeypatch):
    monkeypatch.setenv("WAE_VOICE_SUM", "2")
    render_three(pkg, engine, oracle, dict(src="sine", tail="lowpass"), times_grid(True))


@pytest.mark.parametrize("chunk", [128, 1024, None], ids=["128", "1024", "default"])
def test_chunk_sizes(pkg, engine, oracle, chunk):
    got, _ = render_three(pkg, engine, oracle, dict(src="sawtooth", tail="shaper"), times_grid(True), chunk=chunk)
    ts = times_grid(True)
    pcms = [noise(30 + i, 2, 3000) for i in range(len(ts))]
    render_three(pkg, engine, oracle, ABSN_SPECS["rate09"], ts, chunk=chunk, pcms=pcms)


def test_rebind_a_b_a(pkg, engine):
    torch = pytest.importorskip("torch")
    spec = dict(src="square", tail="shaper")
    n = 6
    made = [make(pkg, engine.backend, spec, (0.0, None), True) for _ in range(n)]
    b = pkg.Batch([c for c, _ in made])
    a = torch.tensor([0.0, 0.0123, 0.05, 0.1, 0.15, 0.3], dtype=torch.float64).cuda()
    bb = torch.tensor([0.02, 0.0, 0.19, 0.0071, 2.0, 0.04], dtype=torch.float64).cuda()
    outs = []
    for t in (a, bb, a):
        b.bind_schedules(made[0][1], t)
        b.run()
        b.sync()
        outs.append(b.fetch())
    assert np.array_equal(outs[0], outs[2])
    assert not np.array_equal(outs[0], outs[1])


def test_clamped_and_non_finite_times(pkg, engine, oracle):
    torch = pytest.importorskip("torch")
    spec = dict(src="sine", tail="split")
    n = 4
    made = [make(pkg, engine.backend, spec, (0.0, None), True) for _ in range(n)]
    b = pkg.Batch([c for c, _ in made])
    b.bind_schedules(made[0][1], torch.tensor([float("nan"), -1.0, float("inf"), 0.01], dtype=torch.float64).cuda())
    b.run()
    b.sync()
    as_rendered = [0.0, 0.0, WIN[1], 0.01]
    want = [np.stack(x.channels) for x in pkg.render_batch([make(pkg, oracle, spec, (t, None), False)[0] for t in as_rendered])]
    for i in range(n):
        assert float(np.abs(b.fetch_graph(i) - want[i]).max()) <= TOL, i


def test_runs_wait_for_the_bind(pkg, engine):
    made = make(pkg, engine.backend, dict(src="sine", tail=None), (0.0, None), True)
    b = pkg.Batch([made[0]])
    with pytest.raises(Exception) as e:
        b.run()
    assert e.value.status == 2


def soundscape(pkg, be, pcm, onsets, gains, declare, n_events, length):
    """n_events clips (device inputs when declared) at onsets, each followed by a gain, summed at the destination"""
    c = pkg.OfflineAudioContext(2, length, SR, be)
    srcs, gs = [], []
    for k in range(n_events):
        s = c.create_buffer_source()
        g = c.create_gain(1.0 if declare else float(gains[k]))
        if declare:
            s.set_device_input(2, pcm.shape[-1], SR)
            g.gain.set_device_value(0.0, 2.0)
        else:
            s.set_buffer(pkg.AudioBuffer(list(pcm[k]), SR))
        s.connect(g)
        g.connect(c.destination())
        if declare:
            s.start_at(0.0)
            s.set_device_schedule((0.0, length / SR))
        else:
            s.start_at(float(onsets[k]))
        srcs.append(s)
        gs.append(g)
    return c, srcs, gs


def test_thousand_soundscapes(pkg, engine, oracle):
    """1000 graphs x 8 device-input events: sources, gains and onsets bound in one run, rendered by run and run_pipelined"""
    torch = pytest.importorskip("torch")
    n, k, length, clip = 1000, 8, 9600, 2400
    gen = torch.Generator().manual_seed(11)
    pcm = torch.rand((n, k, 2, clip), generator=gen).sub_(0.5)
    onsets = torch.rand((n, k), generator=gen, dtype=torch.float64) * ((length - clip) / SR)
    onsets[:, 0] = torch.floor(onsets[:, 0] * SR / 128) * 128 / SR  # some aligned starts: the 1:1 copy
    gains = torch.rand((n, k), generator=gen) * 1.5
    made = [soundscape(pkg, engine.backend, pcm[0].numpy(), None, None, True, k, length) for _ in range(n)]
    b = pkg.Batch([m[0] for m in made])
    _, srcs, gs = made[0]
    for j in range(k):
        b.bind_sources(srcs[j], pcm[:, j].contiguous().cuda())
    b.bind_params([g.gain for g in gs], gains.cuda())
    b.bind_schedules(srcs, onsets.cuda())
    b.run()
    b.sync()
    got = b.fetch()
    ids = [0, 1, 2, 499, 500, 998, 999]
    twins = [soundscape(pkg, engine.backend, pcm[i].numpy(), onsets[i].numpy(), gains[i].numpy(), False, k, length)[0] for i in ids]
    tw = pkg.Batch(twins)
    tw.run()
    tw.sync()
    want = [np.stack(x.channels) for x in pkg.render_batch(
        [soundscape(pkg, oracle, pcm[i].numpy(), onsets[i].numpy(), gains[i].numpy(), False, k, length)[0] for i in ids])]
    for j, i in enumerate(ids):
        assert float(np.abs(got[i] - tw.fetch_graph(j)).max()) <= 1e-6, i
        assert float(np.abs(got[i] - want[j]).max()) <= TOL, i
    out = torch.empty((n, 2, length), dtype=torch.float32, pin_memory=True)
    b.run_pipelined(out.data_ptr())
    assert np.array_equal(out.numpy(), got)
