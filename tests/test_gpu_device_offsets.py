"""AudioBufferSourceNode offsets and durations bound from device memory (wae_buffer_source_set_device_offset + wae_batch_bind_schedules)
on the GPU.  Every case is rendered three ways: bound from a torch tensor, as the host twin (the same schedule declaration, the offset and
duration given to start), and on the oracle.  Every bound render is bit-equal to its twin and within 1e-5 of the oracle."""
import ctypes as C
import math
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
TOL = 1e-5
SR = 48000.0
LENGTH = 9600
END = LENGTH / SR
F64_MAX = 1.7976931348623157e308
CLIP = 4800
WIN = (0.0, END)   # the start window
DWIN = (0.0, 1.0)  # the duration window
STARTS = [0.0, 2560 / SR, 0.0123]  # aligned at 0, aligned later, mid-quantum
# durations: none, 4.5 frames (the reference's test_with_duration_0/1), ending mid-quantum, longer than the rest of the buffer
DURATIONS = [None, 4.5 / SR, 700 / SR, 0.5]


def noise(seed, ch, frames):
    return np.random.default_rng(seed).uniform(-0.5, 0.5, (ch, frames)).astype(np.float32)


def clamp(v, lo, hi):
    return lo if math.isnan(v) else min(max(v, lo), hi)


def buffer_duration(spec):
    return CLIP / spec.get("buf_sr", SR)


def offsets_for(spec):
    """0, whole and fractional frames, exactly the buffer's duration (plays nothing), above the window (clamped to it) and NaN (lo)"""
    if spec.get("loop"):  # inside and past the loop end [0.02, 0.05)
        return [0.0, 0.03, 0.07, float("nan")]
    return [0.0, 100 / SR, 100.37 / SR, buffer_duration(spec), 0.5, float("nan")]


def make(pkg, be, spec, t, mode, pcm):
    """buffer source -> spec['tail'] -> destination playing `pcm`; t = (start, offset, duration or None) as rendered.  mode 'bound': start,
    offset (and duration) declared; 'twin': the start declared, the offset and duration given to start; 'oracle': all host values."""
    c = pkg.OfflineAudioContext(2, LENGTH, SR, be)
    s = c.create_buffer_source(playback_rate=spec.get("rate", 1.0), loop=spec.get("loop", False))
    if spec.get("loop"):
        s.set_loop_start(0.02)
        s.set_loop_end(0.05)
    buf_sr = spec.get("buf_sr", SR)
    if spec.get("dev") and mode != "oracle":
        s.set_device_input(pcm.shape[0], pcm.shape[1], buf_sr)
    else:
        s.set_buffer(pkg.AudioBuffer(list(pcm), buf_sr))
    last = s
    if spec.get("tail") == "lowpass":
        last = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=2000.0)
        s.connect(last)
    elif spec.get("tail") == "shaper":  # a curve that does not map 0 to 0: every silent quantum of the source shows
        last = c.create_wave_shaper(np.array([0.25, 0.5, 0.0], np.float32))
        s.connect(last)
    last.connect(c.destination())
    start, offset, duration = t
    if mode == "bound":
        s.start_at(0.0)
        s.set_device_schedule(WIN, offset=(0.0, buffer_duration(spec)), duration=None if duration is None else DWIN)
    else:
        s.start_at_with_offset_and_duration(0.0 if mode == "twin" else start, offset, F64_MAX if duration is None else duration)
        if mode == "twin":
            s.set_device_schedule(WIN)
    return c, s


def render_three(pkg, engine, oracle, spec, raw, chunk=None):
    """raw: (start, offset, duration or None) per graph as bound; returns the bound renders"""
    torch = pytest.importorskip("torch")
    owin = (0.0, buffer_duration(spec))
    ts = [(s, clamp(o, *owin), None if d is None else clamp(d, *DWIN)) for s, o, d in raw]
    n = len(ts)
    pcms = [noise(50 + i, 2, CLIP) for i in range(n)]
    pcm_dev = torch.from_numpy(np.stack(pcms)).cuda()
    starts = torch.tensor([t[0] for t in ts], dtype=torch.float64).cuda()

    def batch(mode):
        made = [make(pkg, engine.backend, spec, ts[i], mode, pcms[i]) for i in range(n)]
        if chunk:
            engine.set_option(pkg.OPT_CHUNK_FRAMES, chunk)
        try:
            b = pkg.Batch([c for c, _ in made])
        finally:
            if chunk:
                engine.set_option(pkg.OPT_CHUNK_FRAMES, 0)
        if spec.get("dev"):
            b.bind_sources(made[0][1], pcm_dev)
        return b, made[0][1]

    b, node = batch("bound")
    offsets = torch.tensor([r[1] for r in raw], dtype=torch.float64).cuda()
    durations = None if raw[0][2] is None else torch.tensor([r[2] for r in raw], dtype=torch.float64).cuda()
    b.bind_schedules(node, starts, offsets=offsets, durations=durations)
    b.run()
    b.sync()
    got = b.fetch()
    tw, tnode = batch("twin")
    tw.bind_schedules(tnode, starts)
    tw.run()
    tw.sync()
    twin = tw.fetch()
    want = [np.stack(x.channels) for x in pkg.render_batch([make(pkg, oracle, spec, ts[i], "oracle", pcms[i])[0] for i in range(n)])]
    for i in range(n):
        assert np.array_equal(got[i], twin[i]), (spec, raw[i], float(np.abs(got[i] - twin[i]).max()))
        assert float(np.abs(got[i] - want[i]).max()) <= TOL, (spec, raw[i], float(np.abs(got[i] - want[i]).max()))
    return got


SPECS = {
    "rate1": dict(tail="shaper"),                     # the 1:1 copy inside the bound kernel for an offset of 0 from an aligned start
    "rate09": dict(tail="lowpass", rate=0.9),
    "host_44k": dict(tail=None, buf_sr=44100.0),
    "dev": dict(tail="shaper", dev=True),
    "dev_44k_rate11": dict(tail=None, dev=True, buf_sr=44100.0, rate=1.1),
    "loop": dict(tail="shaper", loop=True),           # the serial kernel
}


@pytest.mark.parametrize("with_duration", [False, True], ids=["offset", "offset_duration"])
@pytest.mark.parametrize("name", list(SPECS))
def test_buffer_source(pkg, engine, oracle, name, with_duration):
    spec = SPECS[name]
    raw = [(s, o, d) for s in STARTS for o in offsets_for(spec) for d in (DURATIONS[1:] if with_duration else [None])]
    render_three(pkg, engine, oracle, spec, raw)


@pytest.mark.parametrize("chunk", [128, 1024, None], ids=["128", "1024", "default"])
def test_chunk_sizes(pkg, engine, oracle, chunk):
    for name, duration in (("rate09", None), ("dev", 700 / SR)):
        spec = SPECS[name]
        raw = [(s, o, duration) for s in STARTS for o in offsets_for(spec)[:4]]
        render_three(pkg, engine, oracle, spec, raw, chunk=chunk)


def test_clamped_and_non_finite(pkg, engine, oracle):
    """offsets and durations outside their windows land on the window's ends, NaN on lo"""
    spec = dict(tail="lowpass")
    raw = [(0.0, o, d) for o in (float("nan"), -1.0, float("inf"), 0.5, 0.02)
           for d in (float("nan"), -1.0, float("inf"), 5.0, 0.01)]
    render_three(pkg, engine, oracle, spec, raw)


def test_closed_form(pkg, engine):
    """rate 1, an integer-frame offset o and an aligned start s: the output is pcm[n - s + o] over the played span and zero elsewhere"""
    torch = pytest.importorskip("torch")
    cases = [(s, o) for s in (0, 256, 1280) for o in (0, 37, 128, 1000, CLIP - 1)]
    pcm = noise(7, 1, CLIP)
    made = []
    for _ in cases:
        c = pkg.OfflineAudioContext(1, LENGTH, SR, engine.backend)
        s = c.create_buffer_source(pkg.AudioBuffer(list(pcm), SR))
        s.connect(c.destination())
        s.start_at(0.0)
        s.set_device_schedule(WIN, offset=(0.0, CLIP / SR))
        made.append((c, s))
    b = pkg.Batch([c for c, _ in made])
    b.bind_schedules(made[0][1], torch.tensor([s / SR for s, _ in cases], dtype=torch.float64).cuda(),
                     offsets=torch.tensor([o / SR for _, o in cases], dtype=torch.float64).cuda())
    b.run()
    b.sync()
    got = b.fetch()
    for i, (s, o) in enumerate(cases):
        want = np.zeros(LENGTH, np.float32)
        e = min(LENGTH, s + CLIP - o)
        want[s:e] = pcm[0, o:o + e - s]
        assert float(np.abs(got[i][0] - want).max()) <= 1e-6, (s, o)
        if o == 0:
            assert np.array_equal(got[i][0], want), s  # the 1:1 copy


def declared_batch(pkg, engine, n, spec=None, with_buffer=lambda i: True):
    spec = spec or dict(tail="shaper")
    made = []
    for i in range(n):
        c = pkg.OfflineAudioContext(2, LENGTH, SR, engine.backend)
        s = c.create_buffer_source()
        if with_buffer(i):
            s.set_buffer(pkg.AudioBuffer(list(noise(90 + i, 2, CLIP)), SR))
        sh = c.create_wave_shaper(np.array([0.25, 0.5, 0.0], np.float32))
        s.connect(sh)
        sh.connect(c.destination())
        s.start_at(0.0)
        s.set_device_schedule(WIN, offset=(0.0, 1.0), duration=DWIN)
        made.append((c, s))
    return pkg.Batch([c for c, _ in made]), made


def test_rebind_a_b_a(pkg, engine):
    torch = pytest.importorskip("torch")
    n = 6
    b, made = declared_batch(pkg, engine, n)
    starts = torch.tensor([0.0, 0.0123, 0.05, 0.0, 0.02, 0.1], dtype=torch.float64).cuda()
    a = (torch.tensor([0.0, 0.01, 0.02, 0.0373, 0.05, 0.0], dtype=torch.float64).cuda(),
         torch.tensor([0.5, 0.02, 0.001, 0.04, 0.5, 0.03], dtype=torch.float64).cuda())
    bb = (torch.tensor([0.03, 0.0, 0.0011, 0.09, 0.0, 0.002], dtype=torch.float64).cuda(),
          torch.tensor([0.01, 0.5, 0.06, 0.0001, 0.03, 0.5], dtype=torch.float64).cuda())
    outs = []
    for o, d in (a, bb, a):
        b.bind_schedules(made[0][1], starts, offsets=o, durations=d)
        b.run()
        b.sync()
        outs.append(b.fetch())
    assert np.array_equal(outs[0], outs[2])
    assert all(not np.array_equal(outs[0][i], outs[1][i]) for i in range(n))


def test_runs_wait_for_the_bind(pkg, engine):
    b, _ = declared_batch(pkg, engine, 2)
    with pytest.raises(Exception) as e:
        b.run()
    assert e.value.status == 2


def test_template_bind_over_sources_that_never_play(pkg, engine):
    """one bind over graphs of which every other one's source has no buffer (never plays, the planner gives it no patch entries): the
    bind writes nothing there, the others render as bound, and a batch of only such graphs runs without a bind"""
    torch = pytest.importorskip("torch")
    n = 4
    b, made = declared_batch(pkg, engine, n, with_buffer=lambda i: i % 2 == 0)
    silent = declared_batch(pkg, engine, 1, with_buffer=lambda i: False)[0]
    silent.run()
    silent.sync()
    idle = silent.fetch()[0]
    starts = torch.full((n,), 0.0123, dtype=torch.float64).cuda()
    offs = torch.full((n,), 0.01, dtype=torch.float64).cuda()
    durs = torch.full((n,), 0.05, dtype=torch.float64).cuda()
    b.bind_schedules(made[0][1], starts, offsets=offs, durations=durs)
    b.run()
    b.sync()
    got = b.fetch()
    for i in range(1, n, 2):
        assert np.array_equal(got[i], idle), i
    for i in range(0, n, 2):
        assert not np.array_equal(got[i], idle), i


def test_row_extent(pkg, engine):
    """the row an item reads is start, [stop], [offset], [duration]: its declared width must lie in one allocation"""
    torch = pytest.importorskip("torch")
    B = pkg._binding if hasattr(pkg, "_binding") else sys.modules[pkg.__name__ + "._binding"]
    rows = torch.zeros((1, 3), dtype=torch.float64, device="cuda")
    seg = next(x for x in torch.cuda.memory_snapshot() if x["address"] <= rows.data_ptr() < x["address"] + x["total_size"])
    end = seg["address"] + seg["total_size"]

    def bind(b, node, p):
        items = (B.ScheduleBinding * 1)(B.ScheduleBinding(0, node, C.cast(C.c_void_p(p), B.c_double_p)))
        return pkg.api().batch_bind_schedules(b.handle, items, 1, None)
    b3, m3 = declared_batch(pkg, engine, 1)  # start, offset, duration
    assert bind(b3, m3[0][1].id, end - 16) == 1
    assert bind(b3, m3[0][1].id, end - 24) == 0
    c = pkg.OfflineAudioContext(2, LENGTH, SR, engine.backend)
    s = c.create_buffer_source(pkg.AudioBuffer(list(noise(3, 2, CLIP)), SR))
    s.connect(c.destination())
    s.start_at(0.0)
    s.set_device_schedule(WIN, offset=(0.0, 0.1))  # start, offset
    b2 = pkg.Batch([c])
    assert bind(b2, s.id, end - 8) == 1
    assert bind(b2, s.id, end - 16) == 0


def excerpt_graph(pkg, be, rec_len, length, declare, rec=None, offset=0.0, cutoff=1000.0, gain=1.0):
    """the README scenario: a long recording (a device input when declared), an excerpt of `length` frames at `offset`, a lowpass and a
    gain whose values are bound when declared"""
    c = pkg.OfflineAudioContext(1, length, SR, be)
    s = c.create_buffer_source()
    lp = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=cutoff)
    g = c.create_gain(gain)
    s.connect(lp)
    lp.connect(g)
    g.connect(c.destination())
    if declare:
        s.set_device_input(1, rec_len, SR)
        lp.frequency.set_device_value(100.0, 8000.0)
        g.gain.set_device_value(0.0, 2.0)
        s.start_at(0.0)
        s.set_device_schedule((0.0, 0.0), offset=(0.0, rec_len / SR))
    else:
        s.set_buffer(pkg.AudioBuffer([rec], SR))
        s.start_at_with_offset(0.0, offset)
    return c, s, lp, g


def test_thousand_excerpts(pkg, engine, oracle):
    """1000 graphs, each a long device-input recording bound once and an excerpt at a bound offset through a bound lowpass and gain,
    rendered by run and run_pipelined"""
    torch = pytest.importorskip("torch")
    n, rec_len, length = 1000, 24000, 4800
    gen = torch.Generator().manual_seed(5)
    recs = torch.rand((n, 1, rec_len), generator=gen).sub_(0.5)
    offsets = torch.rand(n, generator=gen, dtype=torch.float64) * ((rec_len - length) / SR)
    offsets[:4] = torch.tensor([0.0, 0.0, 1.0 / SR, (rec_len - length) / SR], dtype=torch.float64)
    cutoffs = torch.rand(n, generator=gen) * 4000.0 + 500.0
    gains = torch.rand(n, generator=gen) * 1.5
    made = [excerpt_graph(pkg, engine.backend, rec_len, length, True) for _ in range(n)]
    b = pkg.Batch([m[0] for m in made])
    _, s, lp, g = made[0]
    b.bind_sources(s, recs.cuda())
    b.bind_params([lp.frequency, g.gain], torch.stack([cutoffs, gains], dim=1).cuda())
    b.bind_schedules(s, torch.zeros(n, dtype=torch.float64).cuda(), offsets=offsets.cuda())
    b.run()
    b.sync()
    got = b.fetch()
    ids = [0, 1, 2, 3, 499, 500, 998, 999]

    def host(be, i):
        return excerpt_graph(pkg, be, rec_len, length, False, recs[i, 0].numpy(), float(offsets[i]), float(cutoffs[i]), float(gains[i]))[0]
    tw = pkg.Batch([host(engine.backend, i) for i in ids])
    tw.run()
    tw.sync()
    want = [np.stack(x.channels) for x in pkg.render_batch([host(oracle, i) for i in ids])]
    for j, i in enumerate(ids):
        assert float(np.abs(got[i] - tw.fetch_graph(j)).max()) <= 1e-6, i
        assert float(np.abs(got[i] - want[j]).max()) <= TOL, i
    out = torch.empty((n, 1, length), dtype=torch.float32, pin_memory=True)
    b.run_pipelined(out.data_ptr())
    assert np.array_equal(out.numpy(), got)
