"""AudioBufferSourceNodes read by reference from device memory (wae_buffer_source_set_device_input_by_reference + wae_batch_bind_sources)
on the GPU.  Every graph is built three ways: with its sources read by reference, with the same sources declared for a copy and bound
from the same tensor, and on the oracle with AudioBuffers.  Every by-reference render is bit-equal to the copy-bound one and within 1e-5
of the oracle.  Each bound channel is a slice of a NaN-filled allocation, NaN between the channels and after the last one: a read outside
[0, length) would show as NaN in the output without faulting."""
import ctypes as C

import numpy as np
import pytest

import graphs as G

pytestmark = pytest.mark.gpu
TOL = 1e-5
SR = 48000.0
HOLD = 50_000_000  # torch.cuda._sleep cycles, about 25 ms: far longer than a run of these batches


@pytest.fixture
def torch():
    return pytest.importorskip("torch")


@pytest.fixture
def options(pkg, engine):
    """engine options set by a case, reset to their defaults afterwards"""
    touched = []

    def set_(opt, value):
        touched.append(opt)
        engine.set_option(opt, value)
    yield set_
    for opt in touched:
        engine.set_option(opt, 0)


def noise(seed, ch, frames, amp=0.5):
    return np.random.default_rng(seed).uniform(-amp, amp, (ch, frames)).astype(np.float32)


def bits(t):
    import torch
    return t.contiguous().view(torch.int32)


def same_bits(a, b):
    return a.shape == b.shape and bool((bits(a) == bits(b)).all())


def source(pkg, c, pcm, mode, sample_rate=None, **kw):
    """mode 'ref': a device input read by reference, 'copy': one copied by its bind, 'oracle': an AudioBuffer"""
    sr = sample_rate or c.sample_rate()
    if mode == "oracle":
        return c.create_buffer_source(pkg.AudioBuffer(list(pcm), sr), **kw)
    s = c.create_buffer_source(**kw)
    s.set_device_input(pcm.shape[0], pcm.shape[1], sr, by_reference=mode == "ref")
    return s


def b_chain(pkg, be, i, pcm, mode, length):  # the fused k_chain
    _, f0, q, gain = G.c2_params(i)
    c = pkg.OfflineAudioContext(2, length, SR, be)
    s = source(pkg, c, pcm, mode)
    bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=f0, q=q)
    gn = c.create_gain(gain)
    s.connect(bq)
    bq.connect(gn)
    gn.connect(c.destination())
    s.start()
    return c, {"node": s}


def b_fast_loop(pkg, be, i, pcm, mode, length):  # k_buffer_source, looping (two consumers keep it out of a chain)
    c = pkg.OfflineAudioContext(2, length, SR, be)
    s = source(pkg, c, pcm, mode, loop=True)
    s.connect(c.create_gain(0.5)).connect(c.destination())
    s.connect(c.create_stereo_panner(-0.3 + 0.1 * i)).connect(c.destination())
    s.start()
    return c, {"node": s}


def b_slow(pkg, be, i, pcm, mode, length):  # the slow track, resampled
    c = pkg.OfflineAudioContext(2, length, SR, be)
    s = source(pkg, c, pcm, mode, sample_rate=SR / 2, playback_rate=0.75, loop=True, loop_start=0.05 + 0.01 * i, loop_end=0.2)
    s.connect(c.destination())
    s.start()
    return c, {"node": s}


def b_serial(pkg, be, i, pcm, mode, length):  # k_buffer_source_serial (automated detune)
    c = pkg.OfflineAudioContext(2, length, SR, be)
    s = source(pkg, c, pcm, mode)
    s.detune.linear_ramp_to_value_at_time(300.0 + 50 * i, length / SR)
    s.connect(c.destination())
    s.start()
    return c, {"node": s}


def b_conv(pkg, be, i, pcm, mode, length):  # a source a convolver consumes: the copy twin's arena buffer aliases the slab
    c = pkg.OfflineAudioContext(2, length, SR, be)
    cv = c.create_convolver(pkg.AudioBuffer(G.synthetic_ir(9000, 2, seed=i), SR))
    s = source(pkg, c, pcm, mode)
    s.connect(cv)
    cv.connect(c.destination())
    s.start()
    return c, {"node": s}


# the bound slow track: playback rate, start time, offset and loop points bound from device memory (host values on the oracle)
BOUND = [dict(rate=0.9 + 0.05 * i, start=0.0007 * i, offset=0.01 * i, ls=0.02 + 0.005 * i, le=0.15 + 0.01 * i) for i in range(8)]


def b_bound(pkg, be, i, pcm, mode, length):
    c = pkg.OfflineAudioContext(2, length, SR, be)
    v = BOUND[i]
    dur = pcm.shape[1] / SR
    if mode == "oracle":
        s = source(pkg, c, pcm, mode, playback_rate=v["rate"], loop=True, loop_start=v["ls"], loop_end=v["le"])
        s.start_at_with_offset(v["start"], v["offset"])
    else:
        s = source(pkg, c, pcm, mode, loop=True)
        s.playback_rate.set_device_value(0.5, 1.5)
        s.start_at(0.0)
        s.set_device_schedule((0.0, length / SR), offset=(0.0, dur))
        s.set_device_loop((0.0, 0.06), (0.1, dur))
    s.connect(c.destination())
    return c, {"node": s}


def bind_bound(torch, b, hs, n):
    s = hs[0]["node"]
    f64 = dict(dtype=torch.float64, device="cuda")
    b.bind_params([s.playback_rate], torch.tensor([BOUND[i]["rate"] for i in range(n)], dtype=torch.float32, device="cuda"))
    b.bind_schedules(s, torch.tensor([BOUND[i]["start"] for i in range(n)], **f64),
                     offsets=torch.tensor([BOUND[i]["offset"] for i in range(n)], **f64))
    b.bind_loops(s, torch.tensor([BOUND[i]["ls"] for i in range(n)], **f64), torch.tensor([BOUND[i]["le"] for i in range(n)], **f64))


def b_suspend(pkg, be, i, pcm, mode, length):
    """one source started at a suspend point, another declared and started in the callback"""
    c = pkg.OfflineAudioContext(2, length, SR, be)
    s = source(pkg, c, pcm, mode)
    s.connect(c.destination())
    h = {"node": s}

    def cb(ctx):
        s.start()
        late = source(pkg, ctx, pcm[:, ::-1].copy(), mode)
        late.connect(ctx.destination())
        late.start()
        h["late"] = late

    c.suspend_sync((2560 - 0.5) / SR, cb)
    return c, h


def nan_padded(torch, pcms, pad):
    """[n][channels][length] of the PCM, a view of a NaN-filled [n + 1][channels][length + pad] allocation"""
    host = np.stack(pcms)
    n, ch, length = host.shape
    t = torch.full((n + 1, ch, length + pad), float("nan"), dtype=torch.float32, device="cuda")
    t[:n, :, :length] = torch.from_numpy(host).cuda()
    return t[:n, :, :length]


def bind_all(torch, b, hs, pcms, pad, key="node", flip=False):
    """one bind_sources call per distinct PCM shape (node ids of template graphs agree); returns the tensors bound"""
    out = []
    for shp in sorted({p.shape for p in pcms}):
        idx = [i for i, p in enumerate(pcms) if p.shape == shp]
        t = nan_padded(torch, [pcms[i][:, ::-1].copy() if flip else pcms[i] for i in idx], pad)
        b.bind_sources([hs[i][key] for i in idx], t, graphs=idx)
        out.append(t)
    return out


def render_three(pkg, engine, oracle, build, pcms, length, pad=4, many=False, groups=False, extra=None):
    torch = pytest.importorskip("torch")
    n = len(pcms)
    lens = length if isinstance(length, list) else [length] * n
    made = {m: [build(pkg, engine.backend if m != "oracle" else oracle, i, pcms[i], m, lens[i]) for i in range(n)]
            for m in ("ref", "copy", "oracle")}
    got = {}
    for m in ("ref", "copy"):
        b = pkg.Batch([c for c, _ in made[m]], many=many)
        hs = [h for _, h in made[m]]
        bind_all(torch, b, hs, pcms, pad)
        if "late" in hs[0]:
            bind_all(torch, b, hs, pcms, pad, key="late", flip=True)
        if extra:
            extra(torch, b, hs, n)
        if groups:
            assert len(b.groups()) > 1
            for k in range(len(b.groups())):
                b.run_group(k)
        else:
            b.run()
        b.sync()
        got[m] = [b.fetch_graph(i) for i in range(n)]
        if m == "ref":
            keep = b
    bufs = pkg.render_many([c for c, _ in made["oracle"]]) if many else pkg.render_batch([c for c, _ in made["oracle"]])
    for i in range(n):
        assert np.array_equal(got["ref"][i], got["copy"][i]), i
        assert float(np.abs(got["ref"][i] - np.stack(bufs[i].channels)).max()) <= TOL, i
    return keep


@pytest.mark.parametrize("tma,frames,pad", [(1, 60000, 4), (0, 60000, 4), (0, 60001, 3), (1, 59999, 1)],
                         ids=["tma", "cp_async", "gather_odd_length", "tma_gather_odd_stride"])
def test_fused_chain(pkg, engine, oracle, options, tma, frames, pad):
    options(pkg.OPT_CHAIN_TMA, tma)
    render_three(pkg, engine, oracle, b_chain, [noise(i, 2, frames) for i in range(4)], 60000, pad=pad)


@pytest.mark.parametrize("build,frames,length", [(b_fast_loop, 7001, 40000), (b_slow, 30000, 40000), (b_serial, 30001, 40000),
                                                 (b_conv, 40064 + 5, 40000)],
                         ids=["k_buffer_source_loop", "slow_resampled", "serial", "convolver_alias"])
def test_playback_paths(pkg, engine, oracle, build, frames, length):
    render_three(pkg, engine, oracle, build, [noise(10 + i, 2, frames) for i in range(3)], length, pad=5)


def test_bound_slow_track(pkg, engine, oracle):
    render_three(pkg, engine, oracle, b_bound, [noise(40 + i, 2, 12001) for i in range(4)], 24000, pad=3, extra=bind_bound)


def test_voice_sum_option(pkg, engine, oracle, options):
    options(pkg.OPT_VOICE_SUM, 2)
    render_three(pkg, engine, oracle, b_chain, [noise(50 + i, 2, 20000) for i in range(3)], 20000)


def test_suspend_point(pkg, engine, oracle):
    render_three(pkg, engine, oracle, b_suspend, [noise(30 + i, 2, 9000) for i in range(3)], 12000, pad=1)


def test_prepare_many_mixed_shapes(pkg, engine, oracle):
    lens = [30000, 30000, 12000, 20000, 12000]
    pcms = [noise(200 + i, 2, lens[i] - 1000 * (i % 2)) for i in range(len(lens))]
    render_three(pkg, engine, oracle, b_chain, pcms, lens, pad=7, many=True)


def test_run_group_over_split_groups(pkg, engine, oracle, options):
    options(pkg.OPT_PIPELINE_GROUPS, 3)
    render_three(pkg, engine, oracle, b_chain, [noise(300 + i, 2, 6001) for i in range(9)], 6000, groups=True)


@pytest.mark.parametrize("chunk", [128, 1024, 0])
def test_chunk_sizes(pkg, engine, oracle, options, chunk):
    options(pkg.OPT_CHUNK_FRAMES, chunk)
    render_three(pkg, engine, oracle, b_chain, [noise(400 + i, 2, 5000 + 3 * i) for i in range(3)], 5000 + 128 * 3, pad=2)


# ---- binding: rebinding, sharing, ordering, lifetime, refusals --------------------------------------------------------------------
def ref_batch(pkg, engine, n, length, mode="ref", build=b_chain, frames=None):
    made = [build(pkg, engine.backend, i, np.zeros((2, frames or length), np.float32), mode, length) for i in range(n)]
    return pkg.Batch([c for c, _ in made]), made[0][1]["node"]


def copy_render(torch, pkg, engine, t, length, build=b_chain):
    """the render of the copy-declared twin with `t` bound"""
    b, node = ref_batch(pkg, engine, t.shape[0], length, "copy", build, t.shape[2])
    b.bind_sources(node, t)
    b.run()
    b.sync()
    return torch.from_numpy(b.fetch()).cuda()


def test_rebind_to_another_stride_and_share_one_tensor(pkg, engine, torch):
    n, length = 4, 30000
    b, node = ref_batch(pkg, engine, n, length)
    a = nan_padded(torch, [noise(500 + i, 2, length) for i in range(n)], 4)
    c = nan_padded(torch, [noise(600 + i, 2, length) for i in range(n)], 9)
    shared = nan_padded(torch, [noise(700, 2, length)], 3).expand(n, 2, length)  # one tensor named by every graph
    for t in (a, c, shared, a):
        b.bind_sources(node, t)
        b.run()
        b.sync()
        assert same_bits(torch.from_numpy(b.fetch()).cuda(), copy_render(torch, pkg, engine, t, length))


def test_mixed_copy_and_reference_items_in_one_call(pkg, engine, torch):
    n, length = 6, 8000
    made = [b_chain(pkg, engine.backend, i, np.zeros((2, length), np.float32), "ref" if i % 2 else "copy", length) for i in range(n)]
    b = pkg.Batch([c for c, _ in made])
    t = nan_padded(torch, [noise(800 + i, 2, length) for i in range(n)], 5)
    b.bind_sources(made[0][1]["node"], t)
    b.run()
    b.sync()
    assert same_bits(torch.from_numpy(b.fetch()).cuda(), copy_render(torch, pkg, engine, t, length))


def test_in_place_write_after_bind_is_seen(pkg, engine, torch):
    n, length = 4, 100000
    b, node = ref_batch(pkg, engine, n, length)
    t = nan_padded(torch, [noise(900 + i, 2, length) for i in range(n)], 4)
    new = torch.from_numpy(np.stack([noise(950 + i, 2, length) for i in range(n)])).cuda()
    want = copy_render(torch, pkg, engine, new, length)
    b.bind_sources(node, t)
    torch.cuda._sleep(HOLD)  # the write lands long after the host has queued the run
    t.copy_(new)
    b.run()
    y = b.output_tensor().clone()
    torch.cuda.synchronize()
    assert same_bits(y, want)


def test_ring_feeds_each_output_back(pkg, engine, torch):
    """step k renders from step k - 1's output, through a ring of three tensors (the output is bound first: a referenced input may not
    overlap it), the engine stream held back before each run; the copy twin, synchronised step by step, gives the expected steps"""
    n, length, steps = 4, 8192 + 77, 5
    x0 = torch.from_numpy(np.stack([noise(1000 + i, 2, length) for i in range(n)])).cuda()
    want, cur = [], x0
    for _ in range(steps):
        cur = copy_render(torch, pkg, engine, cur, length)
        want.append(cur)
    b, node = ref_batch(pkg, engine, n, length)
    ring = [torch.full((n, 2, length), float("nan"), device="cuda") for _ in range(3)]
    ring[2].copy_(x0)
    got = []
    for k in range(steps):
        b.bind_output(ring[k % 3])
        b.bind_sources(node, ring[(k - 1) % 3])
        with torch.cuda.stream(b._engine_stream()):
            torch.cuda._sleep(HOLD)
        b.run()
        got.append(b.output_tensor().clone())  # (orders torch after the run: the next write into this tensor may follow)
    torch.cuda.synchronize()
    for k in range(steps):
        assert same_bits(got[k], want[k]), f"step {k}"


def test_caller_drops_the_tensor_before_run(pkg, engine, torch):
    n, length = 4, 50000
    b, node = ref_batch(pkg, engine, n, length)
    host = [noise(1100 + i, 2, length) for i in range(n)]
    want = copy_render(torch, pkg, engine, torch.from_numpy(np.stack(host)).cuda(), length)
    t = nan_padded(torch, host, 4)
    b.bind_sources(node, t)
    del t
    junk = [torch.full((n + 1, 2, length + 4), 7.0, device="cuda") for _ in range(4)]  # would take the freed memory
    b.run()
    b.sync()
    assert same_bits(torch.from_numpy(b.fetch()).cuda(), want)
    del junk


def test_refusals(pkg, engine, torch):
    B = pkg._binding
    api = pkg.api()
    n, length = 3, 8000
    b, node = ref_batch(pkg, engine, n, length)
    with pytest.raises(pkg.WaeError) as e:
        b.run()  # a run before the bind
    assert e.value.status == 2 and f"node {node.id}" in e.value.message
    good = nan_padded(torch, [noise(1200 + i, 2, length) for i in range(n)], 4)

    def raw(graph, nd, ptr, stride):
        item = B.SourceBinding(graph, nd, C.cast(C.c_void_p(ptr), B.c_float_p), stride)
        return api.batch_bind_sources(b.handle, C.byref(item), 1, None)

    host = np.stack([noise(0, 2, length)])
    assert raw(0, node.id, host.ctypes.data, length) == 1               # host (numpy) memory
    assert raw(0, node.id, good.data_ptr() + 2, length) == 1            # not 4-byte aligned
    assert raw(0, node.id, good.data_ptr(), 1 << 40) == 1               # extent outside any allocation
    assert raw(0, node.id, good.data_ptr(), length - 1) == 1            # channel stride below the declared length
    assert raw(0, node.id + 3, good.data_ptr(), length) == 2            # not a device input
    assert raw(n, node.id, good.data_ptr(), length) == 2                # graph index out of range
    with pytest.raises(pkg.WaeError) as e:
        b.bind_sources(node, good[[0, 0]], graphs=[1, 1])
    assert e.value.status == 1 and "twice" in e.value.message
    own = b.output_tensor()  # the batch's own output: [n][2][length], the inputs' shape
    with pytest.raises(pkg.WaeError) as e:
        b.bind_sources(node, own)
    assert e.value.status == 1 and "overlaps" in e.value.message
    with pytest.raises(pkg.WaeError) as e:
        b.run()
    assert e.value.status == 2  # nothing was bound by the failed calls
    y = torch.zeros((n, 2, length), device="cuda")
    b.bind_output(y)
    with pytest.raises(pkg.WaeError) as e:
        b.bind_sources(node, y)
    assert e.value.status == 1 and "overlaps" in e.value.message
    b.bind_output(None)
    b.bind_sources(node, good)
    over = torch.as_strided(good, (n, 2, length), (2 * length, length, 1), good.storage_offset())  # contiguous, in good's allocation
    with pytest.raises(pkg.WaeError) as e:
        b.bind_output(over)
    assert e.value.status == 1 and "reads by reference" in e.value.message
    b.run()
    b.sync()
    assert same_bits(torch.from_numpy(b.fetch()).cuda(), copy_render(torch, pkg, engine, good, length))
