"""AudioBufferSourceNode playbackRate / detune bound from device memory (wae_param_set_device_value + wae_batch_bind_params) on the GPU.
Every graph is built three ways: with the rate params declared and bound from a torch tensor, on the engine with the same values as
constants (host-built), and on the oracle.  Every render is within 1e-5 of the oracle.  With detune 0 it is bit-equal to the host-built
render wherever both plans give the source the same layout (constant or gated); with detune != 0 the device's exp2 may differ from
glibc's in the last bit of the computed rate, and the number of bit-equal renders is reported."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
TOL = 1e-5
SR = 48000.0
F64_MAX = 1.7976931348623157e308
RATES = [1.0 / 3.0, 0.5, 0.9, 1.0, 1.1, 2.0]
DETUNES = [0.0, 100.0, -100.0]


def noise(seed, ch, frames, amp=0.5):
    return np.random.default_rng(seed).uniform(-amp, amp, (ch, frames)).astype(np.float32)


def make(pkg, be, pcm, vals, bound, dev=False, length=24000, sched=None, loop=False, rng=(1.0 / 3.0, 2.0), det=(-100.0, 100.0),
         buf_sr=SR, tail=None, suspend=None):
    """clip (AudioBuffer or device input) -> source -> [tail] -> destination; vals = (playbackRate, detune)"""
    c = pkg.OfflineAudioContext(2, length, SR, be)
    rate, detune = (1.0, 0.0) if bound else vals
    if dev:
        s = c.create_buffer_source(playback_rate=rate, detune=detune, loop=loop)
        s.set_device_input(pcm.shape[0], pcm.shape[1], buf_sr)
    else:
        s = c.create_buffer_source(pkg.AudioBuffer(list(pcm), buf_sr), playback_rate=rate, detune=detune, loop=loop)
    params = []
    if bound:
        s.playback_rate.set_device_value(*rng)
        s.detune.set_device_value(*det)
        params = [s.playback_rate, s.detune]
    last = s
    if tail == "shaper":  # a curve that does not map 0 to 0: every silent quantum of the source shows
        sh = c.create_wave_shaper(np.array([0.25, 0.5, 0.0], np.float32))
        s.connect(sh)
        last = sh
    elif tail == "gain":
        gn = c.create_gain(0.8)
        s.connect(gn)
        last = gn
        if suspend is not None:
            c.suspend_sync(suspend / SR, lambda ctx: gn.gain.set_value(0.5))
    last.connect(c.destination())
    kind, *a = sched or ("aligned",)
    if kind == "aligned":
        s.start()
    elif kind == "at":  # start(when, offset, duration)
        s.start_at_with_offset_and_duration(a[0], a[1], a[2] if len(a) > 2 else F64_MAX)
    elif kind == "stop":
        s.start()
        s.stop_at(a[0])
    return c, {"node": s, "params": params}


def mixes_dyn(pkg, ctx):
    """the destination mixes a source output with a layout track"""
    return "k_mix_dyn" in pkg.plan_batch([ctx])["kinds"]


def render_three(pkg, engine, oracle, pcms, vals, dev=False, bit=None, run=None, chunk=None, **kw):
    """bound / host-built / oracle renders of graphs i = make(pcms[i], vals[i]).  bit: None -> bit-equality required where detune is 0 and
    both plans give the source the same layout; True / False: always / never required.  Returns (bound renders, bit-equal count)."""
    torch = pytest.importorskip("torch")
    n = len(vals)
    made = [make(pkg, engine.backend, pcms[i], vals[i], True, dev=dev, **kw) for i in range(n)]
    if chunk:
        engine.set_option(pkg.OPT_CHUNK_FRAMES, chunk)
    try:
        b = pkg.Batch([c for c, _ in made])
    finally:
        if chunk:
            engine.set_option(pkg.OPT_CHUNK_FRAMES, 0)
    h = made[0][1]
    if dev:
        b.bind_sources(h["node"], torch.from_numpy(np.stack(pcms)).cuda())
    b.bind_params(h["params"], torch.tensor(np.asarray(vals, np.float32)).cuda())
    (run or (lambda x: (x.run(), x.sync())))(b)
    got = [b.fetch_graph(i) for i in range(n)]
    equal = check(pkg, engine, oracle, got, pcms, vals, bit, **kw)
    return b, got, equal


def check(pkg, engine, oracle, got, pcms, vals, bit=None, **kw):
    """got[i] against the host-built and oracle renders of make(pcms[i], vals[i]) (see render_three); returns the bit-equal count"""
    n = len(vals)
    tw = pkg.Batch([make(pkg, engine.backend, pcms[i], vals[i], False, **kw)[0] for i in range(n)])
    tw.run()
    tw.sync()
    ref = [tw.fetch_graph(i) for i in range(n)]
    want = [np.stack(x.channels) for x in pkg.render_batch([make(pkg, oracle, pcms[i], vals[i], False, **kw)[0] for i in range(n)])]
    bound_dyn = mixes_dyn(pkg, make(pkg, engine.backend, pcms[0], vals[0], True, **kw)[0]) if bit is None else None
    equal = 0
    for i in range(n):
        same = np.array_equal(got[i], ref[i])
        equal += same
        need = bit if bit is not None else (vals[i][1] == 0.0 and mixes_dyn(pkg, make(pkg, engine.backend, pcms[i], vals[i], False, **kw)[0]) == bound_dyn)
        assert same or not need, (i, vals[i], float(np.abs(got[i] - ref[i]).max()))
        assert float(np.abs(got[i] - want[i]).max()) <= TOL, (i, vals[i])
    return equal


GRID = [(r, d) for r in RATES for d in DETUNES]
# clips long enough to cover the render at every rate of the range (2 * 2^(1/12) at most), clips that end inside it at every rate, and
# schedules that start late, skip into the clip, stop or last a given time
SCHEDULES = {
    "aligned_long": dict(clip=60000),
    "aligned_short": dict(clip=7000),
    "late": dict(clip=20000, sched=("at", 0.0123, 0.0)),
    "block_start": dict(clip=20000, sched=("at", 2560 / SR, 0.0)),
    "offset": dict(clip=60000, sched=("at", 0.0, 0.05)),
    "late_offset": dict(clip=20000, sched=("at", 0.0071, 0.031)),
    "stop": dict(clip=60000, sched=("stop", 0.3)),
    "duration": dict(clip=60000, sched=("at", 0.002, 0.01, 0.21)),
}


@pytest.mark.parametrize("dev", [False, True], ids=["audiobuffer", "device_input"])
@pytest.mark.parametrize("name", list(SCHEDULES))
def test_rate_detune_grid(pkg, engine, oracle, name, dev):
    s = SCHEDULES[name]
    pcms = [noise(100 + i, 2, s["clip"]) for i in range(len(GRID))]
    _, _, equal = render_three(pkg, engine, oracle, pcms, GRID, dev=dev, sched=s.get("sched"))
    print(f"{name}: {equal} of {len(GRID)} renders bit-equal to the host-built graphs")


def test_buffer_at_44k1(pkg, engine, oracle):
    pcms = [noise(200 + i, 2, 40000) for i in range(len(GRID))]
    _, _, equal = render_three(pkg, engine, oracle, pcms, GRID, buf_sr=44100.0, sched=("at", 0.004, 0.02))
    print(f"44.1 kHz buffer: {equal} of {len(GRID)} bit-equal")


@pytest.mark.parametrize("sched", [("aligned",), ("at", 2560 / SR, 0.0)], ids=["frame0", "block2560"])
def test_rate_one_is_the_fast_track(pkg, engine, oracle, sched):
    """rate exactly 1, aligned: bit-equal to the host-built fast track (fused with the shaper there), the layout included — the shaper's
    curve maps a silent quantum to 0.5 on one channel"""
    pcms = [noise(300 + i, 2, 9000 + 1000 * i) for i in range(4)]
    render_three(pkg, engine, oracle, pcms, [(1.0, 0.0)] * 4, bit=True, sched=sched, tail="shaper")
    pcms = [noise(310 + i, 2, 9000) for i in range(4)]  # (device inputs of one shape)
    render_three(pkg, engine, oracle, pcms, [(1.0, 0.0)] * 4, dev=True, bit=True, sched=sched, tail="shaper")


def test_rebind(pkg, engine, oracle):
    """one batch bound with 1.0, 1.1, 1.0 and a set that crosses the layout boundary: each run is its own host-built render"""
    torch = pytest.importorskip("torch")
    n, clip = 6, 30000  # the clip covers the render at rates up to 1.25
    pcms = [noise(400 + i, 2, clip) for i in range(n)]
    made = [make(pkg, engine.backend, pcms[i], None, True, tail="shaper") for i in range(n)]
    b = pkg.Batch([c for c, _ in made])
    for vals in ([(1.0, 0.0)] * n, [(1.1, 0.0)] * n, [(1.0, 0.0)] * n, [(0.5, 0.0), (1.2, 0.0), (1.3, 0.0), (2.0, 0.0), (1.0, 0.0), (1.0 / 3.0, 0.0)]):
        b.bind_params(made[0][1]["params"], torch.tensor(np.asarray(vals, np.float32)).cuda())
        b.run()
        b.sync()
        check(pkg, engine, oracle, [b.fetch_graph(i) for i in range(n)], pcms, vals, tail="shaper")


def test_serial_paths(pkg, engine, oracle):
    """a looping source and a range that allows negative rates take the serial kernel: 1e-5 of the oracle always, bit-equal to the
    host-built graph where that takes the serial kernel too (a negative rate)"""
    pcms = [noise(500 + i, 2, 12000) for i in range(4)]
    render_three(pkg, engine, oracle, pcms, [(0.75, 0.0), (1.3, 50.0), (1.0, 0.0), (0.5, -100.0)], bit=False, loop=True)
    render_three(pkg, engine, oracle, pcms, [(-0.5, 0.0), (-1.0, 0.0), (-0.5, 30.0), (-0.75, 0.0)], bit=True, rng=(-1.0, 1.0),
                 sched=("at", 0.0, 0.2))
    render_three(pkg, engine, oracle, pcms, [(0.5, 0.0), (0.9, 0.0), (1.0, 0.0), (0.25, 0.0)], bit=False, rng=(-1.0, 1.0))


def test_non_finite_and_clamped_values(pkg, engine, oracle):
    torch = pytest.importorskip("torch")
    n = 5
    pcms = [noise(600 + i, 2, 20000) for i in range(n)]
    made = [make(pkg, engine.backend, pcms[i], None, True, rng=(0.5, 2.0)) for i in range(n)]
    b = pkg.Batch([c for c, _ in made])
    vals = [(float("nan"), 0.0), (float("inf"), float("-inf")), (5.0, 300.0), (0.1, -300.0), (1.5, float("nan"))]
    as_rendered = [(1.0, 0.0), (1.0, 0.0), (2.0, 100.0), (0.5, -100.0), (1.5, 0.0)]
    b.bind_params(made[0][1]["params"], torch.tensor(np.asarray(vals, np.float32)).cuda())
    b.run()
    b.sync()
    want = [np.stack(x.channels) for x in pkg.render_batch([make(pkg, oracle, pcms[i], as_rendered[i], False)[0] for i in range(n)])]
    for i in range(n):
        assert float(np.abs(b.fetch_graph(i) - want[i]).max()) <= TOL, i


def test_chunk_size_invariance(pkg, engine, oracle):
    vals = [(r, d) for r in (1.0 / 3.0, 1.0, 1.1, 2.0) for d in (0.0, 100.0)]
    for name in ("aligned_short", "late_offset", "duration", "block_start"):
        s = SCHEDULES[name]
        pcms = [noise(700 + i, 2, s["clip"]) for i in range(len(vals))]
        _, a, _ = render_three(pkg, engine, oracle, pcms, vals, sched=s.get("sched"), length=40000)
        _, c, _ = render_three(pkg, engine, oracle, pcms, vals, sched=s.get("sched"), length=40000, chunk=8192)
        for x, y in zip(a, c):
            assert np.array_equal(x, y), name


def test_source_across_a_suspend_point(pkg, engine, oracle):
    vals = [(0.9, 0.0), (1.0, 0.0), (1.1, 100.0), (2.0, -100.0)]
    pcms = [noise(800 + i, 2, 20000) for i in range(len(vals))]
    render_three(pkg, engine, oracle, pcms, vals, tail="gain", suspend=6000.5, sched=("at", 0.0123, 0.0))
    render_three(pkg, engine, oracle, pcms, vals, tail="gain", suspend=9000.0)


def test_thousand_graphs_in_groups(pkg, engine, oracle):
    """1000 device-input clips and their rates bound from one tensor each; rendered by run and run_pipelined"""
    torch = pytest.importorskip("torch")
    n, length, clip = 1000, 4096, 1024  # the clip ends inside the render at every rate: both plans gated
    pcms = torch.rand((n, 2, clip), generator=torch.Generator().manual_seed(5)).sub_(0.5).cuda()
    vals = torch.tensor([0.9, 1.0, 1.1])[torch.randint(3, (n,), generator=torch.Generator().manual_seed(6))]
    vals = torch.stack([vals, torch.zeros(n)], 1).cuda()
    host_pcm, host_vals = pcms.cpu().numpy(), [tuple(map(float, v)) for v in vals.cpu().numpy()]
    made = [make(pkg, engine.backend, host_pcm[i], None, True, dev=True, length=length) for i in range(n)]
    b = pkg.Batch([c for c, _ in made])
    assert len(b.groups()) > 1
    b.bind_sources(made[0][1]["node"], pcms)
    b.bind_params(made[0][1]["params"], vals)
    b.run()
    b.sync()
    got = b.fetch()
    tw = pkg.Batch([make(pkg, engine.backend, host_pcm[i], host_vals[i], False, length=length)[0] for i in range(n)])
    tw.run()
    tw.sync()
    assert np.array_equal(got, tw.fetch())
    ids = [0, 1, 2, 511, 512, 999]
    want = [np.stack(x.channels) for x in pkg.render_batch([make(pkg, oracle, host_pcm[i], host_vals[i], False, length=length)[0] for i in ids])]
    assert max(float(np.abs(got[i] - w).max()) for i, w in zip(ids, want)) <= TOL
    out = torch.empty((n, 2, length), dtype=torch.float32, pin_memory=True)
    b.run_pipelined(out.data_ptr())
    assert np.array_equal(out.numpy(), got)


@pytest.mark.parametrize("rate", [1.0 / 3.0, 0.9, 1.1, 2.0])
def test_against_linear_interpolation(pkg, engine, oracle, rate):
    """third statement: output frame m is the clip linearly interpolated at offset + m * rate (numpy.interp, f64)"""
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(int(rate * 100))
    clip = np.cumsum(rng.uniform(-0.05, 0.05, (2, 30000)), axis=1).astype(np.float32)
    offset = 0.0125  # seconds: 600 frames into the clip
    c, h = make(pkg, engine.backend, clip, None, True, sched=("at", 0.0, offset))
    b = pkg.Batch([c])
    b.bind_params(h["params"], torch.tensor([[rate, 0.0]], dtype=torch.float32).cuda())
    b.run()
    b.sync()
    got = b.fetch_graph(0).astype(np.float64)
    pos = offset * SR + np.arange(got.shape[1]) * float(np.float32(rate))  # (the rate as bound: float32)
    inside = pos < clip.shape[1] - 1
    for ch in range(2):
        want = np.interp(pos[inside], np.arange(clip.shape[1]), clip[ch].astype(np.float64))
        assert inside.sum() > 5000 and np.abs(got[ch][inside] - want).max() <= TOL
