"""AudioBufferSourceNode loop points bound from device memory (wae_buffer_source_set_device_loop + wae_batch_bind_loops) on the GPU.  A
bound render on the bound slow track is bit-equal to the host-built graph with the same loop points and rate (both play
k_buffer_source_slow over equal playhead tables), and every render is within 1e-5 of the oracle."""
import ctypes as C
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
TOL = 1e-5
SR = 48000.0
LENGTH = 9600
F64_MAX = 1.7976931348623157e308
CLIP = 4800
SWIN = (0.0, 0.03)    # loop start window
EWIN = (0.0413, 0.1)  # loop end window (past the 0.1 s clip at 48 kHz: clamped to the buffer's end)
BOUND = "k_buffer_source_slow(bound)"
SERIAL = "k_buffer_source_serial"


def noise(seed, ch, frames):
    return np.random.default_rng(seed).uniform(-0.5, 0.5, (ch, frames)).astype(np.float32)


def clamp(v, lo, hi):
    return lo if math.isnan(v) else min(max(v, lo), hi)


def make(pkg, be, spec, t, mode, pcm):
    """clip -> looping source -> spec['tail'] -> destination.  t = (loop_start, loop_end, offset, rate) as rendered.  mode 'bound': loop
    points declared (and the rate when spec['bind_rate']); 'twin' / 'oracle': all host values."""
    ls, le, offset, rate = t
    c = pkg.OfflineAudioContext(pcm.shape[0], spec.get("length", LENGTH), SR, be)
    s = c.create_buffer_source(playback_rate=rate if mode != "bound" or not spec.get("bind_rate") else 1.0, loop=True)
    buf_sr = spec.get("buf_sr", SR)
    if spec.get("dev") and mode != "oracle":
        s.set_device_input(pcm.shape[0], pcm.shape[1], buf_sr)
    else:
        s.set_buffer(pkg.AudioBuffer(list(pcm), buf_sr))
    last = s
    if spec.get("tail") == "lowpass":
        last = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=2000.0)
        s.connect(last)
    last.connect(c.destination())
    sched = spec.get("sched")  # (start, stop, offset window, duration) as rendered
    if mode == "bound":
        s.set_loop_start(0.0)
        s.set_loop_end(0.0)
        if spec.get("bind_rate"):
            s.playback_rate.set_device_value(*spec["bind_rate"])
        if sched is not None:
            s.start_at(0.0)
            s.set_device_schedule((0.0, 0.1), stop=(0.0, 0.2), offset=(0.0, 0.2), duration=(0.0, 1.0))
        else:
            s.start_at_with_offset(0.0, offset)
        s.set_device_loop(spec.get("swin", SWIN), spec.get("ewin", EWIN))
    else:
        s.set_loop_start(ls)
        s.set_loop_end(le)
        if sched is not None:
            s.start_at_with_offset_and_duration(sched[0], offset, sched[3])
            s.stop_at(sched[1])
        else:
            s.start_at_with_offset(0.0, offset)
    return c, s


def render(pkg, engine, oracle, spec, raw, chunk=None, twin=True):
    """raw: (loop_start, loop_end, offset, rate) per graph as bound; the bound render is checked against the twin (bit for bit) and the
    oracle (1e-5); returns it"""
    torch = pytest.importorskip("torch")
    swin, ewin = spec.get("swin", SWIN), spec.get("ewin", EWIN)
    if spec.get("bind_rate"):
        raw = [(a, b, o, float(np.float32(clamp(r, *spec["bind_rate"])))) for a, b, o, r in raw]
    ts = [(clamp(a, *swin), clamp(b, *ewin), o, r) for a, b, o, r in raw]
    n = len(ts)
    ch = spec.get("ch", 2)
    pcms = [noise(70 + i, ch, CLIP) for i in range(n)]

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
            b.bind_sources(made[0][1], torch.from_numpy(np.stack(pcms)).cuda())
        return b, made[0][1]

    b, node = batch("bound")
    b.bind_loops(node, torch.tensor([r[0] for r in raw], dtype=torch.float64).cuda(), torch.tensor([r[1] for r in raw], dtype=torch.float64).cuda())
    if spec.get("bind_rate"):
        b.bind_params(node.playback_rate, torch.tensor([[r[3]] for r in raw], dtype=torch.float32).cuda())
    if spec.get("sched") is not None:
        st, sp, _, du = spec["sched"]
        rows = [[st, sp, r[2], du] for r in raw]
        cols = torch.tensor(rows, dtype=torch.float64).cuda()
        b.bind_schedules(node, cols[:, 0].contiguous(), stops=cols[:, 1].contiguous(), offsets=cols[:, 2].contiguous(),
                         durations=cols[:, 3].contiguous())
    b.run()
    b.sync()
    got = b.fetch()
    want = [np.stack(x.channels) for x in pkg.render_batch([make(pkg, oracle, spec, ts[i], "oracle", pcms[i])[0] for i in range(n)])]
    if twin:
        tw, _ = batch("twin")
        tw.run()
        tw.sync()
        tg = tw.fetch()
    for i in range(n):
        if twin:
            assert np.array_equal(got[i], tg[i]), (spec, raw[i], float(np.abs(got[i] - tg[i]).max()))
        assert float(np.abs(got[i] - want[i]).max()) <= TOL, (spec, raw[i], float(np.abs(got[i] - want[i]).max()))
    return b, node, got


def cases(rate):
    """loop regions inside, at 0, to the buffer's end, clamped to the windows and NaN; offsets before, inside and past the loop end"""
    # (a source started past its loop end plays on to the buffer's end; the loop ends are chosen so that no rate here reaches the
    # buffer's end exactly on a frame, where the reference's accumulated playhead and the closed form may fall on either side of it)
    pts = [(0.01, 0.0497), (0.0, 0.1), (0.025, 0.0451), (-1.0, 5.0), (float("nan"), float("nan"))]
    return [(a, b, o, rate) for a, b in pts for o in (0.0, 0.03, 0.08)]


SPECS = {
    "rate05": dict(tail="lowpass"),
    "rate09_mono": dict(tail=None, ch=1),
    "rate11": dict(tail="lowpass"),
    "rate2": dict(tail=None),
    "dev_44k": dict(tail="lowpass", dev=True, buf_sr=44100.0),
    "bound_rate": dict(tail="lowpass", bind_rate=(0.5, 2.0)),
}
RATES = {"rate05": 0.5, "rate09_mono": 0.9, "rate11": 1.1, "rate2": 2.0, "dev_44k": 1.0, "bound_rate": 0.9}


@pytest.mark.parametrize("name", list(SPECS))
def test_bound_slow_track(pkg, engine, oracle, name):
    spec = SPECS[name]
    raw = cases(RATES[name])
    if name == "bound_rate":
        raw = [(a, b, o, r) for (a, b, o, _), r in zip(raw, [0.5, 0.9, 1.1, 2.0, 1.37] * 3)]
    render(pkg, engine, oracle, spec, raw)


@pytest.mark.parametrize("chunk", [128, 1024, None], ids=["128", "1024", "default"])
def test_chunk_sizes(pkg, engine, oracle, chunk):
    render(pkg, engine, oracle, SPECS["rate11"], cases(1.1)[:9], chunk=chunk)
    render(pkg, engine, oracle, SPECS["bound_rate"], [(0.012, 0.047, 0.0, 1.9), (0.0, 0.06, 0.02, 0.6)], chunk=chunk)


def test_with_bound_schedule(pkg, engine, oracle):
    """bound start, stop, offset and duration together with bound loop points and rate: against the oracle"""
    for sched in ((0.0123, 0.15, None, 0.07), (0.0, 0.19, None, 1.0)):
        spec = dict(tail="lowpass", bind_rate=(0.5, 2.0), sched=sched)
        render(pkg, engine, oracle, spec, [(0.01, 0.0497, o, r) for o in (0.0, 0.03, 0.09) for r in (0.7, 1.6)], twin=False)


def test_thousand_graphs(pkg, engine, oracle):
    rng = np.random.default_rng(7)
    raw = [(float(rng.uniform(*SWIN)), float(rng.uniform(*EWIN)), float(rng.uniform(0.0, 0.1)), 1.1) for _ in range(1000)]
    render(pkg, engine, oracle, dict(tail="lowpass", length=4800), raw)


def test_capacity_edge(pkg, engine, oracle):
    """the shortest loop the windows allow, at the top rate, over the whole render"""
    spec = dict(tail=None, swin=(0.0, 0.002), ewin=(0.0025, 0.003), bind_rate=(0.5, 2.0), length=48000)
    render(pkg, engine, oracle, spec, [(0.002, 0.0025, 0.0, 2.0), (0.0, 0.003, 0.001, 2.0), (0.002, 0.0025, 0.0, 1.3)])


def test_serial_path_with_bound_points(pkg, engine, oracle):
    """overlapping windows and a rate range reaching 0 take the serial kernel, which reads the bound points raw"""
    for spec in (dict(tail="lowpass", swin=(0.0, 0.06), ewin=(0.04, 0.1)), dict(tail=None, bind_rate=(0.0, 2.0))):
        render(pkg, engine, oracle, spec, [(0.01, 0.05, 0.0, 0.8), (0.05, 0.045, 0.02, 1.2), (0.0, 0.1, 0.0, 0.0)][:2 if "swin" in spec else 3],
                         twin=False)
        assert SERIAL in pkg.plan_batch([make(pkg, engine.backend, spec, (0.0, 0.04, 0.0, 1.0), "bound", noise(1, 2, CLIP))[0]])["kinds"]


def test_rebind_between_runs(pkg, engine, oracle):
    torch = pytest.importorskip("torch")
    spec = SPECS["rate11"]
    b, node, _ = render(pkg, engine, oracle, spec, [(0.01, 0.05, 0.0, 1.1)])
    for pts in ((0.02, 0.06), (0.0, 0.1), (0.01, 0.05)):
        b.bind_loops(node, torch.tensor([pts[0]], dtype=torch.float64).cuda(), torch.tensor([pts[1]], dtype=torch.float64).cuda())
        b.run()
        b.sync()
        got = b.fetch()[0]
        want = np.stack(pkg.render_batch([make(pkg, oracle, spec, (pts[0], pts[1], 0.0, 1.1), "oracle", noise(70, 2, CLIP))[0]])[0].channels)
        assert float(np.abs(got - want).max()) <= TOL, pts


def test_run_before_bind(pkg, engine):
    c, s = make(pkg, engine.backend, SPECS["rate11"], (0.01, 0.05, 0.0, 1.1), "bound", noise(1, 2, CLIP))
    b = pkg.Batch([c])
    with pytest.raises(pkg.WaeError) as e:
        b.run()
    assert e.value.status == 2 and "wae_batch_bind_loops" in e.value.message


def test_bind_contract(pkg, engine):
    torch = pytest.importorskip("torch")
    api = pkg.api()
    made = [make(pkg, engine.backend, SPECS["rate11"], (0.01, 0.05, 0.0, 1.1), "bound", noise(1, 2, CLIP)) for _ in range(2)]
    b = pkg.Batch([c for c, _ in made])
    node = made[0][1].id
    pts = torch.tensor([[0.01, 0.05], [0.02, 0.06]], dtype=torch.float64).cuda()
    B = pkg._binding

    def items(*rows):
        arr = (B.LoopBinding * len(rows))()
        for k, (g, nid, p) in enumerate(rows):
            arr[k] = B.LoopBinding(g, nid, C.cast(C.c_void_p(p), B.c_double_p))
        return arr

    def call(*rows):
        return api.batch_bind_loops(b.handle, items(*rows), len(rows), None)

    base = pts.data_ptr()
    host = np.zeros(2)
    assert call((0, node, 0)) == 1                                   # null pointer
    assert call((0, node, base + 4)) == 1                            # misaligned
    assert call((0, node, host.ctypes.data)) == 1                    # not device memory
    assert call((0, node, base), (0, node, base + 16)) == 1          # a node named twice
    assert call((0, node + 1000, base)) == 2                         # no declaration
    assert call((5, node, base)) == 2                                # graph index out of range
    # all-or-nothing: a bad second item leaves the batch unbound
    assert call((0, node, base), (1, node, 0)) == 1
    with pytest.raises(pkg.WaeError):
        b.run()
    assert call((0, node, base), (1, node, base + 16)) == 0
    b.run()
    b.sync()
