"""AudioBufferSourceNodes bound from device memory (wae_buffer_source_set_device_input + wae_batch_bind_sources) on the GPU.  Every graph
is built twice on the engine, once with device inputs bound from torch tensors and once with AudioBuffers holding the same PCM: the two
renders are bit-equal, and both are within 1e-5 of the oracle (which builds the AudioBuffer twin)."""
import ctypes as C

import numpy as np
import pytest

import graphs as G

pytestmark = pytest.mark.gpu
TOL = 1e-5
SR = 48000.0


def noise(seed, ch, frames, amp=0.5):
    return np.random.default_rng(seed).uniform(-amp, amp, (ch, frames)).astype(np.float32)


def source(pkg, c, pcm, dev, **kw):
    if dev:
        s = c.create_buffer_source(**kw)
        s.set_device_input(pcm.shape[0], pcm.shape[1], c.sample_rate())
    else:
        s = c.create_buffer_source(pkg.AudioBuffer(list(pcm), c.sample_rate()), **kw)
    return s


def b_chain(pkg, be, i, pcm, dev, length):
    _, f0, q, gain = G.c2_params(i)
    c = pkg.OfflineAudioContext(2, length, SR, be)
    s = source(pkg, c, pcm, dev)
    bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=f0, q=q)
    gn = c.create_gain(gain)
    s.connect(bq)
    bq.connect(gn)
    gn.connect(c.destination())
    s.start()
    return c, {"node": s}


def b_slow(pkg, be, i, pcm, dev, length):
    c = pkg.OfflineAudioContext(2, length, SR, be)
    s = source(pkg, c, pcm, dev, playback_rate=0.75, loop=True, loop_start=0.05 + 0.01 * i, loop_end=0.2)
    s.connect(c.destination())
    s.start()
    return c, {"node": s}


def b_serial(pkg, be, i, pcm, dev, length):
    c = pkg.OfflineAudioContext(2, length, SR, be)
    s = source(pkg, c, pcm, dev)
    s.detune.linear_ramp_to_value_at_time(300.0 + 50 * i, length / SR)
    s.connect(c.destination())
    s.start()
    return c, {"node": s}


def b_late(pkg, be, i, pcm, dev, length):
    c = pkg.OfflineAudioContext(2, length, SR, be)
    s = source(pkg, c, pcm, dev)
    s.connect(c.destination())
    s.start_at_with_offset(0.0123 + 0.001 * i, 0.05)
    return c, {"node": s}


def b_six(pkg, be, i, pcm, dev, length):
    c = pkg.OfflineAudioContext(2, length, SR, be)
    s = source(pkg, c, pcm, dev)
    g = c.create_gain(0.5)
    s.connect(g)
    g.connect(c.destination())
    s.start()
    return c, {"node": s}


def b_suspend(pkg, be, i, pcm, dev, length):
    """one source started at a suspend point, another declared (device input or buffer) and started in the callback"""
    c = pkg.OfflineAudioContext(2, length, SR, be)
    s = source(pkg, c, pcm, dev)
    s.connect(c.destination())
    h = {"node": s}

    def cb(ctx):
        s.start()
        late = source(pkg, ctx, pcm[:, ::-1].copy(), dev)
        late.connect(ctx.destination())
        late.start()
        h["late"] = late

    c.suspend_sync((2560 - 0.5) / SR, cb)
    return c, h


def b_conv(pkg, be, i, pcm, dev, length):
    c = pkg.OfflineAudioContext(2, length, SR, be)
    cv = c.create_convolver(pkg.AudioBuffer(G.synthetic_ir(9000, 2, seed=i), SR))
    s = source(pkg, c, pcm, dev)
    s.connect(cv)
    cv.connect(c.destination())
    s.start()
    return c, {"node": s}


def tensor(torch, pcms):
    return torch.from_numpy(np.stack(pcms)).cuda()


def bind_all(torch, b, hs, pcms, key="node", flip=False):
    """one bind_sources call per distinct PCM shape (node ids of template graphs agree)"""
    shapes = sorted({p.shape for p in pcms})
    for shp in shapes:
        idx = [i for i, p in enumerate(pcms) if p.shape == shp]
        data = [pcms[i][:, ::-1].copy() if flip else pcms[i] for i in idx]
        b.bind_sources([hs[i][key] for i in idx], tensor(torch, data), graphs=idx)


def oracle_pcm(pkg, ctxs, many):
    bufs = pkg.render_many(ctxs) if many else pkg.render_batch(ctxs)
    return [np.stack(b.channels) for b in bufs]


def render_three(pkg, engine, oracle, build, pcms, length, many=False, run=None):
    torch = pytest.importorskip("torch")
    n = len(pcms)
    lens = length if isinstance(length, list) else [length] * n
    dev = [build(pkg, engine.backend, i, pcms[i], True, lens[i]) for i in range(n)]
    buf = [build(pkg, engine.backend, i, pcms[i], False, lens[i]) for i in range(n)]
    ora = [build(pkg, oracle, i, pcms[i], False, lens[i]) for i in range(n)]
    bd = pkg.Batch([c for c, _ in dev], many=many)
    hs = [h for _, h in dev]
    bind_all(torch, bd, hs, pcms)
    if "late" in hs[0]:
        bind_all(torch, bd, hs, pcms, key="late", flip=True)
    (run or (lambda b: (b.run(), b.sync())))(bd)
    got = [bd.fetch_graph(i) for i in range(n)]
    bb = pkg.Batch([c for c, _ in buf], many=many)
    bb.run()
    bb.sync()
    ref = [bb.fetch_graph(i) for i in range(n)]
    want = oracle_pcm(pkg, [c for c, _ in ora], many)
    for i in range(n):
        assert np.array_equal(got[i], ref[i]), i
        assert float(np.abs(got[i] - want[i]).max()) <= TOL, i
    return bd, hs, got


@pytest.mark.parametrize("tma", [1, 0])
def test_fused_chain(pkg, engine, oracle, tma):
    engine.set_option(pkg.OPT_CHAIN_TMA, tma)
    try:
        render_three(pkg, engine, oracle, b_chain, [noise(i, 2, 60000) for i in range(4)], 60000)
    finally:
        engine.set_option(pkg.OPT_CHAIN_TMA, 0)


@pytest.mark.parametrize("build", [b_slow, b_serial, b_late, b_conv], ids=["slow_loop", "serial_detune", "late_offset", "convolver"])
def test_playback_paths(pkg, engine, oracle, build):
    render_three(pkg, engine, oracle, build, [noise(10 + i, 2, 30000) for i in range(3)], 40000)


def test_six_channel_source(pkg, engine, oracle):
    render_three(pkg, engine, oracle, b_six, [noise(20 + i, 6, 25000) for i in range(2)], 25000)


def test_suspend_start_and_declare_in_callback(pkg, engine, oracle):
    render_three(pkg, engine, oracle, b_suspend, [noise(30 + i, 2, 9000) for i in range(3)], 12000)


def test_many_graphs_run_and_pipelined(pkg, engine, oracle):
    torch = pytest.importorskip("torch")
    n, length = 64, 20000
    pcms = [noise(100 + i, 2, length) for i in range(n)]
    bd, hs, got = render_three(pkg, engine, oracle, b_chain, pcms, length)
    assert len(bd.groups()) > 1
    out = torch.empty((n, 2, length), dtype=torch.float32, pin_memory=True)
    bd.run_pipelined(out.data_ptr())
    assert np.array_equal(out.numpy(), np.stack(got))


def test_prepare_many_mixed_shapes(pkg, engine, oracle):
    lens = [30000, 30000, 12000, 20000, 12000]
    pcms = [noise(200 + i, 2, lens[i] - 1000 * (i % 2)) for i in range(len(lens))]
    render_three(pkg, engine, oracle, b_chain, pcms, lens, many=True)


def dev_batch(pkg, engine, n, length, build=b_chain, frames=None, channels=2):
    made = [build(pkg, engine.backend, i, np.zeros((channels, frames or length), np.float32), True, length) for i in range(n)]
    return pkg.Batch([c for c, _ in made]), made[0][1]["node"]


def buf_render(pkg, engine, pcms, length, build=b_chain):
    b = pkg.Batch([build(pkg, engine.backend, i, pcms[i], False, length)[0] for i in range(len(pcms))])
    b.run()
    b.sync()
    return b.fetch()


def test_rebinding(pkg, engine):
    torch = pytest.importorskip("torch")
    n, length = 4, 30000
    A = [noise(300 + i, 2, length) for i in range(n)]
    Bp = [noise(400 + i, 2, length) for i in range(n)]
    b, node = dev_batch(pkg, engine, n, length)
    b.bind_sources(node, tensor(torch, A))
    b.run()
    b.sync()
    assert np.array_equal(b.fetch(), buf_render(pkg, engine, A, length))
    b.bind_sources(node, tensor(torch, Bp))
    b.run()
    b.sync()
    out_b = b.fetch()
    assert np.array_equal(out_b, buf_render(pkg, engine, Bp, length))
    b.run()
    b.sync()
    assert np.array_equal(b.fetch(), out_b)  # runs never alter bound audio
    b.bind_sources(node, tensor(torch, [A[1], A[3]]), graphs=[1, 3])
    b.run()
    b.sync()
    mixed = [Bp[0], A[1], Bp[2], A[3]]
    assert np.array_equal(b.fetch(), buf_render(pkg, engine, mixed, length))


def test_alignment_and_strides(pkg, engine):
    torch = pytest.importorskip("torch")
    n, length = 2, 480001
    pcms = [noise(500 + i, 2, length) for i in range(n)]
    want = buf_render(pkg, engine, pcms, length)
    b, node = dev_batch(pkg, engine, n, length)
    host = np.stack(pcms)
    padded = torch.zeros((n, 2, length + 7), dtype=torch.float32, device="cuda")
    padded[:, :, :length] = torch.from_numpy(host).cuda()
    flat = torch.zeros(n * 2 * length + 1, dtype=torch.float32, device="cuda")
    flat[1:] = torch.from_numpy(host.reshape(-1)).cuda()
    for t in (torch.from_numpy(host).cuda(), padded[:, :, :length], flat[1:].view(n, 2, length)):
        b.bind_sources(node, t)
        b.run()
        b.sync()
        assert np.array_equal(b.fetch(), want)


def test_slots_kept_through_upload_and_pipelined(pkg, engine):
    """graphs with device inputs and graphs with (small, possibly pageable) AudioBuffers in the same groups"""
    torch = pytest.importorskip("torch")
    n, length = 16, 6000
    pcms = [noise(600 + i, 2, length) for i in range(n)]
    made = [b_chain(pkg, engine.backend, i, pcms[i], i % 2 == 0, length) for i in range(n)]
    b = pkg.Batch([c for c, _ in made])
    ev = list(range(0, n, 2))
    b.bind_sources(made[0][1]["node"], tensor(torch, [pcms[i] for i in ev]), graphs=ev)
    want = buf_render(pkg, engine, pcms, length)
    b.upload()
    b.run()
    b.sync()
    assert np.array_equal(b.fetch(), want)
    out = torch.empty((n, 2, length), dtype=torch.float32, pin_memory=True)
    b.run_pipelined(out.data_ptr())
    assert np.array_equal(out.numpy(), want)
    b.upload()
    b.run_pipelined(out.data_ptr())
    assert np.array_equal(out.numpy(), want)


def test_stream_ordering_with_torch(pkg, engine):
    torch = pytest.importorskip("torch")
    n, length = 8, 200000
    b, node = dev_batch(pkg, engine, n, length)
    base = tensor(torch, [noise(700 + i, 2, length) for i in range(n)])
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        x = torch.sin(base * 3.0) * 0.5  # queued on s right before the bind
        b.bind_sources(node, x)
        del x  # (the engine stream holds the memory until the copy has run: record_stream)
        b.run()
        y = b.output_tensor() * 2.0  # consumed on s right after the run
        z = b.output_tensor(3)[1].clone()
    s.synchronize()
    b.sync()
    got = b.fetch()
    assert np.array_equal(y.cpu().numpy(), got * 2.0)
    assert np.array_equal(z.cpu().numpy(), got[3, 1])


def test_errors_before_launch(pkg, engine):
    torch = pytest.importorskip("torch")
    B = pkg._binding
    api = pkg.api()
    n, length = 3, 8000
    pcms = [noise(800 + i, 2, length) for i in range(n)]
    made = [b_chain(pkg, engine.backend, i, pcms[i], True, length) for i in range(n)]
    b = pkg.Batch([c for c, _ in made])
    node = made[0][1]["node"].id
    with pytest.raises(pkg.WaeError) as e:
        b.run()
    assert e.value.status == 2 and "graph 0" in e.value.message and f"node {node}" in e.value.message
    good = tensor(torch, pcms)

    def raw(graph, nd, ptr, stride):
        item = B.SourceBinding(graph, nd, C.cast(C.c_void_p(ptr), B.c_float_p), stride)
        return api.batch_bind_sources(b.handle, C.byref(item), 1, None)

    host = np.stack(pcms)
    assert raw(0, node, host.ctypes.data, length) == 1                   # host (numpy) memory
    assert raw(0, node, good.data_ptr(), 1 << 40) == 1                    # extent outside any allocation
    assert raw(0, node, good.data_ptr(), length - 1) == 1                 # channel stride below the declared length
    assert raw(0, node + 3, good.data_ptr(), length) == 2                 # not a device input (the biquad)
    assert raw(n, node, good.data_ptr(), length) == 2                     # graph index out of range
    with pytest.raises(pkg.WaeError) as e:
        b.bind_sources(node, good[:, :, : length - 1])                  # shorter than the declared shape
    assert e.value.status == 1
    with pytest.raises(pkg.WaeError) as e:
        b.bind_sources(node, torch.zeros((n, 1, length), device="cuda"))  # channels differ
    assert e.value.status == 1
    with pytest.raises(pkg.WaeError) as e:
        b.run()
    assert e.value.status == 2  # nothing was bound by the failed calls
    for fn in (pkg.render_batch_oneshot, pkg.render_many):
        with pytest.raises(pkg.WaeError) as e:
            fn([b_chain(pkg, engine.backend, i, pcms[i], True, length)[0] for i in range(n)])
        assert e.value.status == 2
    b.bind_sources(node, good)
    b.run()
    b.sync()
    assert np.array_equal(b.fetch(), buf_render(pkg, engine, pcms, length))


def test_default_stream_ordering(pkg, engine):
    """torch's default stream is the legacy NULL stream: the input written there behind a long op, then bound and rendered, and the
    output read there behind a long op, then bound and rendered over — all without a synchronisation."""
    torch = pytest.importorskip("torch")
    n, length = 8, 100000
    A = [noise(900 + i, 2, length) for i in range(n)]
    Bp = [noise(950 + i, 2, length) for i in range(n)]
    want_a, want_b = buf_render(pkg, engine, A, length), buf_render(pkg, engine, Bp, length)
    b, node = dev_batch(pkg, engine, n, length)
    src_a, src_b = tensor(torch, A), tensor(torch, Bp)
    x = torch.zeros((n, 2, length), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    torch.cuda._sleep(100_000_000)  # ~50 ms: the write lands long after the host has bound and launched
    x.copy_(src_a)
    b.bind_sources(node, x)
    b.run()
    y = b.output_tensor()
    torch.cuda._sleep(100_000_000)  # the read of the output lands long after the next bind and run were queued
    ya = y.clone()
    x.copy_(src_b)
    b.bind_sources(node, x)
    b.run()
    yb = b.output_tensor().clone()
    torch.cuda.synchronize()
    b.sync()
    assert np.array_equal(ya.cpu().numpy(), want_a)
    assert np.array_equal(yb.cpu().numpy(), want_b)
    assert np.array_equal(b.fetch(), want_b)


def b_mono(pkg, be, i, pcm, dev, length):
    c = pkg.OfflineAudioContext(2, length, SR, be)
    s = source(pkg, c, pcm, dev)
    g = c.create_gain(0.7)
    s.connect(g)
    g.connect(c.destination())
    s.start()
    return c, {"node": s}


def test_mono_tensor_with_any_channel_stride(pkg, engine):
    torch = pytest.importorskip("torch")
    n, length = 3, 20001
    pcms = [noise(1000 + i, 1, length) for i in range(n)]
    want = buf_render(pkg, engine, pcms, length, build=b_mono)
    b, node = dev_batch(pkg, engine, n, length, build=b_mono, channels=1)
    flat = torch.from_numpy(np.stack(pcms).reshape(n, length)).cuda()
    for t in (flat.unsqueeze(1), torch.as_strided(flat, (n, 1, length), (length, 1, 1))):  # channel stride length, and 1
        b.bind_sources(node, t)
        b.run()
        b.sync()
        assert np.array_equal(b.fetch(), want)


def test_same_slot_twice_in_one_call(pkg, engine):
    torch = pytest.importorskip("torch")
    n, length = 2, 8000
    pcms = [noise(1100 + i, 2, length) for i in range(n)]
    b, node = dev_batch(pkg, engine, n, length)
    with pytest.raises(pkg.WaeError) as e:
        b.bind_sources(node, tensor(torch, [pcms[0], pcms[1]]), graphs=[1, 1])
    assert e.value.status == 1 and "twice" in e.value.message
    with pytest.raises(pkg.WaeError) as e:
        b.run()
    assert e.value.status == 2  # (nothing was bound)
    b.bind_sources(node, tensor(torch, pcms))
    b.run()
    b.sync()
    assert np.array_equal(b.fetch(), buf_render(pkg, engine, pcms, length))


def b_idle(pkg, be, i, pcm, dev, length):
    """a played source and a second device input that is never started (the planner gives it no slot)"""
    c, h = b_chain(pkg, be, i, pcm, dev, length)
    idle = source(pkg, c, pcm, dev)
    idle.connect(c.destination())
    h["idle"] = idle
    return c, h


def test_unstarted_device_input_binds_as_nothing(pkg, engine, oracle):
    torch = pytest.importorskip("torch")
    n, length = 3, 12000
    pcms = [noise(1200 + i, 2, length) for i in range(n)]
    made = [b_idle(pkg, engine.backend, i, pcms[i], True, length) for i in range(n)]
    b = pkg.Batch([c for c, _ in made])
    h = made[0][1]
    t = tensor(torch, pcms)
    b.bind_sources(h["node"], t)
    b.run()  # the idle input need not be bound
    b.sync()
    want = buf_render(pkg, engine, pcms, length, build=b_idle)
    assert np.array_equal(b.fetch(), want)
    both = torch.cat([t, t.flip(2)], 0)  # one call over both nodes of every graph: the idle ones are validated and copy nothing
    b.bind_sources([h["node"]] * n + [h["idle"]] * n, both, graphs=list(range(n)) * 2)
    b.run()
    b.sync()
    assert np.array_equal(b.fetch(), want)
    ora = pkg.render_batch([b_idle(pkg, oracle, i, pcms[i], False, length)[0] for i in range(n)])
    assert float(np.abs(want - np.stack([np.stack(x.channels) for x in ora])).max()) <= TOL
