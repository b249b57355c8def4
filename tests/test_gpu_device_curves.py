"""WaveShaperNode curves bound from device memory (wae_wave_shaper_set_device_curve + wae_batch_bind_curves) on the GPU.  A batch is
planned once and run with curves bound from torch tensors; each render is compared with the oracle's render of the same graphs given the
same curves through set_curve (1e-5) and with the engine's own render of such graphs (bit-equal where the plan is the same, i.e. behind
an input that is never silent; within 1e-5 elsewhere, where the declared plan covers both answers of can_propagate_silence and an
over-sampled shaper behind a dynamic input always takes the `rebuild` path).

The over-sampled path is checked behind inputs that keep their channel count, with curves through 0 or not.  Curves that are not
through 0 are checked with the shaper feeding the destination directly: a fused gain after an over-sampled shaper copies out channels
the layout track calls unspecified (NEXT.md).  Behind a mono input that may fall silent a host curve that is not through 0 takes
`as_static`, whose first quantum carries the down-sampled curve(0) of the zero history where the reference's fresh resamplers start
from zero; the declared curve takes `rebuild = 1`, which matches the oracle there, and equals the host-curve render bit for bit from
the second quantum on."""
import contextlib
import ctypes as C

import numpy as np
import pytest

import graphs as G
from test_device_curves_cpu import INPUTS, NEVER_SILENT, make_curve, noise, shaper_graph

pytestmark = pytest.mark.gpu
TOL = 1e-5
SR = G.SR
PATHS = {"fused": (1, 0), "unfused": (0, 0), "x2": (1, 1), "x4": (1, 2)}  # path -> (fuse option, oversample)
CURVES = {"zero_odd": ("zero", 257), "offset_odd": ("offset", 257), "zero_even": ("zero", 1024), "offset_even": ("offset", 1024)}


@contextlib.contextmanager
def options(pkg, engine, fuse=1, chunk=0):
    engine.set_option(pkg.OPT_FUSE, fuse)
    engine.set_option(pkg.OPT_CHUNK_FRAMES, chunk)
    try:
        yield
    finally:
        engine.set_option(pkg.OPT_FUSE, 1)
        engine.set_option(pkg.OPT_CHUNK_FRAMES, 0)


def tensor(torch, arrays):
    return torch.from_numpy(np.ascontiguousarray(np.stack(arrays).astype(np.float32))).cuda()


def maxdiff(a, b):
    return float(np.abs(a.astype(np.float64) - b.astype(np.float64)).max())


def declared_batch(pkg, engine, build, n):
    made = [build(engine.backend, g, None) for g in range(n)]
    return pkg.Batch([c for c, _ in made]), made[0][1]


def bind_run(torch, batch, curves):
    b, sh = batch
    b.bind_curves(sh, tensor(torch, curves))
    b.run()
    b.sync()
    return b.fetch()


def host_renders(pkg, engine, oracle, build, curves):
    want = G.render(pkg, [build(oracle, g, curves[g])[0] for g in range(len(curves))])
    twin = pkg.Batch([build(engine.backend, g, curves[g])[0] for g in range(len(curves))])
    twin.run()
    twin.sync()
    return want, twin.fetch()


def check(pkg, engine, oracle, build, curves, bit_equal=False, batch=None):
    """binds curves[g] to graph g of a prepared batch of declared graphs (or `batch`), runs it, and compares with the oracle and with the
    engine's host-curve render -> (render, batch)"""
    torch = pytest.importorskip("torch")
    batch = batch or declared_batch(pkg, engine, build, len(curves))
    got = bind_run(torch, batch, curves)
    want, twin = host_renders(pkg, engine, oracle, build, curves)
    assert np.isfinite(want).all()
    assert maxdiff(got, want) <= TOL, maxdiff(got, want)
    assert maxdiff(got, twin) <= TOL, maxdiff(got, twin)
    if bit_equal:
        assert np.array_equal(got, twin)
    return got, batch


# ---------------------------------------------------------------------------------------------------------- paths x curves x inputs
OS_INPUTS = [i for i in INPUTS if i != "switch"]
CASES = ([(p, c, i) for p in ("fused", "unfused") for c in CURVES for i in INPUTS] +
         [(p, c, i) for p in ("x2", "x4") for c in CURVES if c.startswith("zero") for i in OS_INPUTS])


@pytest.mark.parametrize("path,curve,inp", CASES)
def test_paths_curves_inputs(pkg, engine, oracle, path, curve, inp):
    fuse, oversample = PATHS[path]
    kind, n = CURVES[curve]
    curves = [make_curve(kind, n) * np.float32(1.0 - 0.1 * g) for g in range(2)]

    def build(be, g, c):
        return shaper_graph(pkg, be, g, 12000, n, c, oversample=oversample, inp=inp)
    with options(pkg, engine, fuse=fuse):
        check(pkg, engine, oracle, build, curves, bit_equal=inp in NEVER_SILENT or oversample > 0)


@pytest.mark.parametrize("inp", ["late", "stop", "gap"])
@pytest.mark.parametrize("curve", ["offset_odd", "offset_even"])
@pytest.mark.parametrize("path", ["x2", "x4"])
def test_over_sampled_curves_not_through_zero(pkg, engine, oracle, path, curve, inp):
    """`rebuild` patched to 1 and the output track's k_meta patched to META_SHAPER: the same plan a host curve of these points gets"""
    _, oversample = PATHS[path]
    kind, n = CURVES[curve]
    curves = [make_curve(kind, n) * np.float32(1.0 - 0.1 * g) for g in range(2)]

    def build(be, g, c):
        return shaper_graph(pkg, be, g, 12000, n, c, oversample=oversample, inp=inp, tail_gain=False)
    check(pkg, engine, oracle, build, curves, bit_equal=True)


@pytest.mark.parametrize("inp", ["late", "gap"])
@pytest.mark.parametrize("kind", ["zero", "offset"])
@pytest.mark.parametrize("path", ["x2", "x4"])
def test_over_sampled_mono_input_that_may_fall_silent(pkg, engine, oracle, path, kind, inp):
    """the host curve takes `freeze` (through 0) or `as_static` (not), the declared one `rebuild` 2 or 1.  Through 0 the renders are
    bit-equal.  Not through 0 the declared render matches the oracle from frame 0, while the host curve's `as_static` adds the
    down-sampled curve(0) of the zero history to the first quantum; from the second quantum on the two renders are bit-equal."""
    torch = pytest.importorskip("torch")
    _, oversample = PATHS[path]
    n = 1024
    curves = [make_curve(kind, n) * np.float32(1.0 - 0.1 * g) for g in range(2)]

    def build(be, g, c):
        return shaper_graph(pkg, be, g, 12000, n, c, oversample=oversample, inp=inp, ch=1, tail_gain=False)
    got = bind_run(torch, declared_batch(pkg, engine, build, 2), curves)
    want, twin = host_renders(pkg, engine, oracle, build, curves)
    assert maxdiff(got, want) <= TOL, maxdiff(got, want)
    if kind == "zero":
        assert np.array_equal(got, twin)
    else:
        assert np.array_equal(got[..., 128:], twin[..., 128:])
        assert maxdiff(twin[..., :128], want[..., :128]) > 1e-3  # (the host curve's first quantum, NEXT.md)


REBIND = [("fused", i, True) for i in ("late", "gap", "switch")] + [("unfused", i, True) for i in ("late", "gap", "switch")] + \
         [(p, i, False) for p in ("x2", "x4") for i in ("late", "stop", "gap")]


@pytest.mark.parametrize("path,inp,tail_gain", REBIND)
def test_rebinding_switches_the_patched_decisions(pkg, engine, oracle, path, inp, tail_gain):
    """one prepared batch: a curve through 0, one that is not, the first again; each run equals its host-curve build (the patched
    shaper_keeps_silence, k_meta mode and rebuild fields follow the curve), and the third run repeats the first bit for bit"""
    fuse, oversample = PATHS[path]
    n = 1024
    zero = [make_curve("zero", n) for _ in range(2)]
    off = [make_curve("offset", n) for _ in range(2)]

    def build(be, g, c):
        return shaper_graph(pkg, be, g, 12000, n, c, oversample=oversample, inp=inp, tail_gain=tail_gain)
    with options(pkg, engine, fuse=fuse):
        first, batch = check(pkg, engine, oracle, build, zero)
        second, _ = check(pkg, engine, oracle, build, off, batch=batch)
        third, _ = check(pkg, engine, oracle, build, zero, batch=batch)
    assert np.array_equal(first, third) and not np.array_equal(first, second)


@pytest.mark.parametrize("chunk", [128, 1024, 0])
@pytest.mark.parametrize("oversample", [0, 2])
def test_suspend_points_and_chunks(pkg, engine, oracle, chunk, oversample):
    n = 1024
    curves = [make_curve("zero" if oversample else "offset", n) * np.float32(1.0 + 0.2 * g) for g in range(2)]

    def build(be, g, c):
        return shaper_graph(pkg, be, g, 12000, n, c, oversample=oversample, inp="gap", suspends=(3072, 8192))
    with options(pkg, engine, chunk=chunk):
        check(pkg, engine, oracle, build, curves)


@pytest.mark.parametrize("curve", ["zero_even", "zero_odd"])
def test_feedback_cycle(pkg, engine, oracle, curve):
    kind, n = CURVES[curve]
    curves = [make_curve(kind, n) for _ in range(2)]

    def build(be, g, c):
        return shaper_graph(pkg, be, g, 12000, n, c, oversample=1, inp="const", feedback=True)
    check(pkg, engine, oracle, build, curves, bit_equal=True)


@pytest.mark.parametrize("oversample", [0, 2])
@pytest.mark.parametrize("n", [1, 65536])
def test_extreme_lengths(pkg, engine, oracle, n, oversample):
    if n == 1:
        curves = [np.array([0.0 if oversample else 0.3], np.float32), np.array([-0.0], np.float32)]
    else:
        curves = [make_curve("zero" if oversample else "offset", n), make_curve("zero", n)]

    def build(be, g, c):
        return shaper_graph(pkg, be, g, 12000, n, c, oversample=oversample, inp="late")
    check(pkg, engine, oracle, build, curves)


@pytest.mark.parametrize("oversample", [0])
def test_non_finite_points(pkg, engine, oversample):
    """NaN at the centre (the curve does not map 0 to 0) and infinities elsewhere are used as given: the render equals the engine's
    render of the same curves given to set_curve"""
    torch = pytest.importorskip("torch")
    n = 257
    curves = [make_curve("zero", n) for _ in range(2)]
    curves[0][n // 2] = np.nan
    curves[0][0], curves[0][-1] = -np.inf, np.inf
    curves[1][10] = np.inf

    def build(be, g, c):
        return shaper_graph(pkg, be, g, 8000, n, c, oversample=oversample, inp="late")
    got = bind_run(torch, declared_batch(pkg, engine, build, 2), curves)
    twin = pkg.Batch([build(engine.backend, g, curves[g])[0] for g in range(2)])
    twin.run()
    twin.sync()
    assert np.array_equal(got, twin.fetch(), equal_nan=True)


# ---------------------------------------------------------------------------------------------------------- with the other binds
def augmentation_graph(pkg, be, g, length, n, curve=None, pcm=None, ir=None, gain=None):
    """device source -> shaper (declared) -> lowpass (frequency declared) -> gain (declared) -> convolver (declared) -> destination"""
    c = pkg.OfflineAudioContext(2, length, SR, be)
    src = c.create_buffer_source()
    if pcm is None:
        src.set_device_input(2, length, SR)
    else:
        src.set_buffer(pkg.AudioBuffer(list(pcm), SR))
    sh = c.create_wave_shaper()
    if curve is None:
        sh.set_device_curve(n)
    else:
        sh.set_curve(curve)
    bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=3000.0 if gain is None else gain[0], q=1.0)
    gn = c.create_gain(0.5 if gain is None else gain[1])
    if gain is None:
        bq.frequency.set_device_value()
        gn.gain.set_device_value()
    cv = c.create_convolver()
    if ir is None:
        cv.set_device_response(2, 9000, SR)
    else:
        cv.set_buffer(pkg.AudioBuffer(list(ir), SR))
    src.connect(sh)
    sh.connect(bq)
    bq.connect(gn)
    gn.connect(cv)
    cv.connect(c.destination())
    src.start()
    return c, src, sh, bq, gn, cv


def test_sources_curves_params_and_responses_together(pkg, engine, oracle):
    torch = pytest.importorskip("torch")
    n_g, length, n = 4, 20000, 1024
    pcms = [noise(700 + g, 2, length) for g in range(n_g)]
    curves = [make_curve("offset" if g % 2 else "zero", n) for g in range(n_g)]
    irs = [np.stack(G.synthetic_ir(9000, 2, seed=710 + g)) for g in range(n_g)]
    vals = np.array([[800.0 + 900 * g, 0.3 + 0.1 * g] for g in range(n_g)], np.float32)
    made = [augmentation_graph(pkg, engine.backend, g, length, n) for g in range(n_g)]
    b = pkg.Batch([m[0] for m in made])
    _, src, sh, bq, gn, cv = made[0]
    b.bind_sources(src, tensor(torch, pcms))
    b.bind_curves(sh, tensor(torch, curves))
    b.bind_params([bq.frequency, gn.gain], torch.from_numpy(vals).cuda())
    b.bind_responses(cv, tensor(torch, irs))
    b.run()
    b.sync()
    got = b.fetch()
    want = G.render(pkg, [augmentation_graph(pkg, oracle, g, length, n, curves[g], pcms[g], irs[g], vals[g])[0] for g in range(n_g)])
    assert maxdiff(got, want) <= TOL


def c2_curve_graph(pkg, be, g, length, n, curve=None, pcm=None):
    """C2's shape with a distortion stage: device source -> 1024-point shaper (fused) -> lowpass -> gain -> destination"""
    _, f0, q, gain = G.c2_params(g)
    c = pkg.OfflineAudioContext(2, length, SR, be)
    src = c.create_buffer_source()
    if pcm is None:
        src.set_device_input(2, length, SR)
    else:
        src.set_buffer(pkg.AudioBuffer(list(pcm), SR))
    sh = c.create_wave_shaper()
    if curve is None:
        sh.set_device_curve(n)
    else:
        sh.set_curve(curve)
    bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=f0, q=q)
    gn = c.create_gain(gain)
    src.connect(sh)
    sh.connect(bq)
    bq.connect(gn)
    gn.connect(c.destination())
    src.start()
    return c, src, sh


def test_thousand_graphs_from_one_tensor(pkg, engine, oracle):
    """1000 graphs from one [1000][1024] tensor, the sources bound too; rendered by run, run_group and run_pipelined"""
    torch = pytest.importorskip("torch")
    n_g, length, n = 1000, 4096, 1024
    pcms = torch.from_numpy(np.stack([G.c2_source(g, length) for g in range(n_g)])).cuda()
    x = torch.linspace(-1.0, 1.0, n, device="cuda")
    drive = torch.linspace(0.5, 4.0, n_g, device="cuda")[:, None]
    curves = torch.tanh(drive * x[None, :]) + (torch.arange(n_g, device="cuda")[:, None] % 3 == 0).float() * 0.05
    made = [c2_curve_graph(pkg, engine.backend, g, length, n) for g in range(n_g)]
    b = pkg.Batch([m[0] for m in made])
    b.bind_sources(made[0][1], pcms)
    b.bind_curves(made[0][2], curves)
    b.run()
    b.sync()
    got = b.fetch()
    host_curves, host_pcm = curves.cpu().numpy(), pcms.cpu().numpy()
    check_ids = [0, 1, 3, 500, 999]
    want = G.render(pkg, [c2_curve_graph(pkg, oracle, g, length, n, host_curves[g], host_pcm[g])[0] for g in check_ids])
    assert maxdiff(got[check_ids], want) <= TOL
    twin = pkg.Batch([c2_curve_graph(pkg, engine.backend, g, length, n, host_curves[g], host_pcm[g])[0] for g in range(n_g)])
    twin.run()
    twin.sync()
    assert np.array_equal(got, twin.fetch())
    for k in range(len(b.groups())):
        b.run_group(k)
    b.sync()
    assert np.array_equal(b.fetch(), got)
    out = torch.empty((n_g, 2, length), dtype=torch.float32, pin_memory=True)
    b.run_pipelined(out.data_ptr())
    assert np.array_equal(out.numpy(), got)


def test_ordering_after_a_torch_kernel(pkg, engine, oracle):
    """the curves are written by a torch kernel on torch's current stream right before the bind, without a synchronisation"""
    torch = pytest.importorskip("torch")
    n = 1024
    base = [make_curve("offset", n) for _ in range(3)]

    def build(be, g, c):
        return shaper_graph(pkg, be, g, 8000, n, c, inp="late")
    b, sh = declared_batch(pkg, engine, build, 3)
    src = tensor(torch, base)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)  # the write lands long after the host has bound and launched
        x = src * 0.5
        b.bind_curves(sh, x)
        del x  # (kept from reuse until the bind has read it: record_stream)
        b.run()
    b.sync()
    got = b.fetch()
    want = G.render(pkg, [build(oracle, g, base[g] * np.float32(0.5))[0] for g in range(3)])
    assert maxdiff(got, want) <= TOL


def test_errors_before_launch(pkg, engine):
    torch = pytest.importorskip("torch")
    B = pkg._binding
    api = pkg.api()
    n_g, n = 3, 1024
    curves = [make_curve("offset", n) for _ in range(n_g)]

    def build(be, g, c):
        ctx, sh = shaper_graph(pkg, be, g, 8000, n, c, inp="late")
        if c is None:
            ctx._unconnected = ctx.create_wave_shaper()
            ctx._unconnected.set_device_curve(16)  # declared, not connected: planned, so bound like any other
        return ctx, sh
    b, sh = declared_batch(pkg, engine, build, n_g)
    node = sh.id
    with pytest.raises(pkg.WaeError) as e:
        b.run()
    assert e.value.status == 2 and "graph 0" in e.value.message and f"node {node}" in e.value.message
    good = tensor(torch, curves)

    def raw(items):
        arr = (B.CurveBinding * len(items))(*[B.CurveBinding(g, nd, C.cast(C.c_void_p(p), B.c_float_p)) for g, nd, p in items])
        return api.batch_bind_curves(b.handle, arr, len(items), None)

    host = np.stack(curves)
    assert raw([(0, node, host.ctypes.data)]) == 1                                   # host (numpy) memory
    assert raw([(0, node, 0)]) == 1                                                  # null
    seg = next(x for x in torch.cuda.memory_snapshot() if x["address"] <= good.data_ptr() < x["address"] + x["total_size"])
    assert raw([(0, node, seg["address"] + seg["total_size"] - 4 * (n - 1))]) == 1  # extent past the end of the allocation
    assert raw([(0, node - 1, good.data_ptr())]) == 2                                # not a declared curve
    assert raw([(n_g, node, good.data_ptr())]) == 2                                  # graph index out of range
    assert raw([(1, node, good.data_ptr()), (1, node, good.data_ptr())]) == 1        # named twice
    with pytest.raises(pkg.WaeError) as e:
        b.bind_curves(node, good[:, : n - 1])                                        # shorter than the declared length
    assert e.value.status == 1
    with pytest.raises(pkg.WaeError) as e:
        b.bind_curves(node, good.unsqueeze(1))                                       # not [n][length]
    assert e.value.status == 1
    with pytest.raises(pkg.WaeError) as e:
        b.run()
    assert e.value.status == 2  # nothing was bound by the failed calls
    b.bind_curves(node, good)
    with pytest.raises(pkg.WaeError) as e:
        b.run()
    other = b.contexts[0]._unconnected.id
    assert e.value.status == 2 and f"node {other}" in e.value.message  # the shaper that is not connected
    b.bind_curves(other, torch.zeros((n_g, 16), device="cuda"))
    b.run()
    b.sync()
    twin = pkg.Batch([build(engine.backend, g, curves[g])[0] for g in range(n_g)])
    twin.run()
    twin.sync()
    assert maxdiff(b.fetch(), twin.fetch()) <= TOL
