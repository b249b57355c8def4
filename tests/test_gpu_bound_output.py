"""Prepared batches rendering into caller device memory (wae_batch_bind_output / Batch.bind_output).  Every case renders the batch into its
own buffer first, then fills that buffer and a bound tensor with NaN and renders again into the tensor: the bound render must equal the
first to the bit, every float of the tensor must be written, and the batch's own buffer must keep its NaNs.  The cases cover every stage
that writes a destination (k_mix, k_mix_dyn, the destination-direct k_chain, k_voice_sum, k_conv_mac_ifft and its accumulating twin), the
per-quantum stages of a DelayNode feedback cycle, a destination with no input and one muted in a cycle, a suspend point, batches of
different shapes, split groups, chunk sizes, a ring of two bound tensors, a slice of a larger tensor, unbinding, the read-outs and the
refusals.  Two cases hold a stream back (torch.cuda._sleep) to check the ordering between runs and the readers of a bound tensor."""
import ctypes as C

import numpy as np
import pytest

import graphs as G

pytestmark = pytest.mark.gpu
SR = G.SR


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


def bits(t):
    import torch
    return t.contiguous().view(torch.int32)


def same_bits(a, b):
    return a.shape == b.shape and bool((bits(a) == bits(b)).all())


def own_views(b):
    return [b.output_tensor(i) for i in range(b.n)]


def out_shape(b):
    return (b.n, b.channels, b.length) if b._one_shape() else (b.device_ptr()[1],)


def graph_views(b, out):
    flat = out.view(-1)
    views = []
    for i in range(b.n):
        off, ch, length = b.graph_output(i)
        views.append(flat[off:off + ch * length].view(ch, length))
    return views


def run(b, groups=False):
    if groups:
        for k in range(len(b.groups())):
            b.run_group(k)
    else:
        b.run()
    b.sync()


def check_bound(torch, b, groups=False, out=None):
    """renders `b` into its own buffer, then into `out` (default: a new tensor), both NaN-filled before the bound run; returns the
    bound tensor and the reference render per graph"""
    run(b, groups)
    own = own_views(b)
    ref = [v.clone() for v in own]
    for v in own:
        v.fill_(float("nan"))
    if out is None:
        out = torch.full(out_shape(b), float("nan"), device="cuda")
    else:
        out.fill_(float("nan"))
    b.bind_output(out)
    run(b, groups)
    for i, (got, want) in enumerate(zip(graph_views(b, out), ref)):
        assert same_bits(got, want), f"graph {i}: max |diff| {float((got - want).abs().max())}"
    for v in own:
        assert bool(torch.isnan(v).all()), "the batch's own buffer was written while an output was bound"
    return out, ref


def stage_names(b):
    return {name for name, _t, _k in b.stage_times()}


def build_mix(pkg, be, g, length=4096 + 37):
    c = pkg.OfflineAudioContext(2, length, SR, be)
    for v in range(3):
        o = c.create_oscillator(type_=pkg.SAWTOOTH, frequency=110.0 * (v + 1) + g)
        gn = c.create_gain(0.2)
        o.connect(gn)
        gn.connect(c.destination())
        o.start()
    return c


def build_mix_dyn(pkg, be, g, length=4096):
    c = pkg.OfflineAudioContext(2, length, SR, be)
    for v in range(4):
        o = c.create_oscillator(frequency=220.0 * (v + 1) + g)
        bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=2000.0, q=1.0)
        o.connect(bq)
        bq.connect(c.destination())
        o.start()
        if v == 1:
            o.stop_at(0.02)  # its layout changes (silent after the tail): the port is folded by k_mix_dyn
    return c


def build_chain(pkg, be, g, length=48000 + 5):
    c = pkg.OfflineAudioContext(2, length, SR, be)
    o = c.create_oscillator(frequency=330.0 + 7.0 * g)
    bq = c.create_biquad_filter(type_=pkg.BANDPASS, frequency=700.0, q=4.0)
    gn = c.create_gain(0.7)
    o.connect(bq)
    bq.connect(gn)
    gn.connect(c.destination())
    o.start()
    return c


def build_convolver(ir_channels, in_channels):
    def build(pkg, be, g, length=8192 * 2 + 300):
        c = pkg.OfflineAudioContext(2, length, SR, be)
        pcm = G.c2_source(g, length)[:in_channels]
        s = c.create_buffer_source(pkg.AudioBuffer(list(pcm), SR))
        ir = G.synthetic_ir(3000, ir_channels, seed=7 + g)
        cv = c.create_convolver(pkg.AudioBuffer(list(ir), SR))
        s.connect(cv)
        cv.connect(c.destination())
        s.start()
        return c
    return build


def build_feedback(pkg, be, g, length=128 * 25):
    pcm = G.c2_source(g, length)
    pcm[:, 128 * 3:] = 0
    c = pkg.OfflineAudioContext(2, length, SR, be)
    s = c.create_buffer_source(pkg.AudioBuffer([pcm[0], pcm[1]], SR))
    d = c.create_delay(max_delay_time=0.05, delay_time=0.0071)
    fb = c.create_gain(0.6)
    s.connect(d)
    d.connect(fb)
    fb.connect(d)
    d.connect(c.destination())
    s.connect(c.destination())
    s.start()
    return c


@pytest.mark.parametrize("case, build, kernel", [
    ("mix", build_mix, "k_mix"),
    ("mix_dyn", build_mix_dyn, "k_mix_dyn"),
    ("chain", build_chain, "k_chain"),
    ("convolver", build_convolver(2, 1), "k_conv_mac_ifft"),
    ("convolver_true_stereo", build_convolver(4, 2), "k_conv_mac_ifft(acc)"),
    ("feedback", build_feedback, "k_ring_write"),
])
def test_every_destination_writer(pkg, engine, torch, case, build, kernel):
    b = pkg.Batch([build(pkg, engine.backend, g) for g in range(3)])
    assert kernel in stage_names(b)
    if case in ("chain", "convolver", "convolver_true_stereo"):  # the chain / the convolver writes the rendered PCM itself
        assert not {"k_mix", "k_mix_dyn"} & stage_names(b)
    _, ref = check_bound(torch, b)
    assert max(float(r.abs().max()) for r in ref) > 1e-3


def test_voice_sum_ports(pkg, engine, torch, options):
    options(pkg.OPT_VOICE_SUM, 2)
    b = pkg.Batch([G.c3_many_voices(pkg, engine.backend, 40 + g, 2048 * 3 + 700) for g in range(2)])
    assert "k_voice_sum" in stage_names(b)
    check_bound(torch, b)


def test_destination_without_input_is_zeros(pkg, engine, torch):
    def build(g):
        c = pkg.OfflineAudioContext(2, 1000 + g, SR, engine.backend)
        o = c.create_oscillator()
        o.start()  # connected to nothing
        return c
    b = pkg.Batch([build(g) for g in range(3)], many=True)
    out, _ = check_bound(torch, b)
    assert bool((out == 0).all())


def test_destination_muted_in_a_cycle_is_zeros(pkg, engine, torch):
    """destination -> gain -> destination without a DelayNode: the Orderer mutes the cycle, no stage writes the destination, and runs
    into a bound output zero it (Group::out_zero) as the batch's own buffer was zeroed at prepare"""
    def build(g):
        c = pkg.OfflineAudioContext(2, 2048 + g, SR, engine.backend)
        o = c.create_oscillator(frequency=440.0 + g)
        o.connect(c.destination())
        o.start()
        gn = c.create_gain(0.5)
        c.destination().connect(gn)
        gn.connect(c.destination())
        return c
    b = pkg.Batch([build(g) for g in range(2)], many=True)
    assert not {"k_mix", "k_mix_dyn", "k_voice_sum", "k_conv_mac_ifft"} & stage_names(b)
    out, _ = check_bound(torch, b)
    assert bool((out == 0).all())


def test_suspend_point(pkg, engine, torch):
    def build(g):
        n = 128 * 40
        c = pkg.OfflineAudioContext(2, n, SR, engine.backend)
        o = c.create_oscillator(type_=pkg.SAWTOOTH, frequency=333.0 + g)
        gn = c.create_gain(0.3)
        o.connect(gn)
        gn.connect(c.destination())
        o.start()

        def later(ctx):
            k = ctx.create_constant_source(offset=0.05)
            k.connect(ctx.destination())
            k.start_at(ctx.current_time())
            gn.disconnect()
        c.suspend_sync(128 * 17 / SR, later)
        return c
    b = pkg.Batch([build(g) for g in range(2)])
    out, _ = check_bound(torch, b)
    assert float(out[:, :, 128 * 17:].abs().max()) == pytest.approx(0.05)


def test_batch_of_different_shapes(pkg, engine, torch):
    shapes = [(1, 1003), (2, 2001), (1, 777), (2, 1500 + 3)]

    def build(g, ch, n):
        c = pkg.OfflineAudioContext(ch, n, SR if g % 2 else 44100.0, engine.backend)
        o = c.create_oscillator(frequency=200.0 + 50.0 * g)
        bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=900.0)
        o.connect(bq)
        bq.connect(c.destination())
        o.start()
        return c
    b = pkg.Batch([build(g, ch, n) for g, (ch, n) in enumerate(shapes)], many=True)
    assert any(b.graph_output(i)[0] % 4 for i in range(b.n))
    out, _ = check_bound(torch, b)
    assert out.dim() == 1
    for i, v in enumerate(graph_views(b, out)):
        assert same_bits(b.output_tensor(i), v)


def test_run_group_over_split_groups(pkg, engine, torch, options):
    options(pkg.OPT_PIPELINE_GROUPS, 3)
    b = pkg.Batch([build_chain(pkg, engine.backend, g, 4096) for g in range(6)] +
                  [build_mix(pkg, engine.backend, g, 4096) for g in range(6)])
    assert len(b.groups()) > 1
    check_bound(torch, b, groups=True)


@pytest.mark.parametrize("chunk", [128, 1024, 0])
def test_chunk_sizes(pkg, engine, torch, options, chunk):
    options(pkg.OPT_CHUNK_FRAMES, chunk)
    ctxs = [build_mix_dyn(pkg, engine.backend, 0, 4096 + 128 * 3), build_chain(pkg, engine.backend, 1, 4096 + 128 * 3),
            build_feedback(pkg, engine.backend, 2, 4096 + 128 * 3)]
    check_bound(torch, pkg.Batch(ctxs))


def source_batch(pkg, engine, torch, n=4, frames=8192 + 77, sets=3):
    """n graphs of a device-input source -> lowpass -> destination, `sets` seeded source sets and each set's render into the batch's
    own buffer"""
    ctxs = []
    for g in range(n):
        c = pkg.OfflineAudioContext(2, frames, SR, engine.backend)
        s = c.create_buffer_source()
        s.set_device_input(2, frames, SR)
        bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=1500.0)
        s.connect(bq)
        bq.connect(c.destination())
        s.start()
        ctxs.append(c)
    b = pkg.Batch(ctxs)
    node = s.id
    gen = torch.Generator(device="cuda").manual_seed(3)
    srcs = [torch.rand((n, 2, frames), device="cuda", generator=gen) * 2 - 1 for _ in range(sets)]
    refs = []
    for src in srcs:
        b.bind_sources(node, src)
        b.run()
        b.sync()
        refs.append(b.output_tensor().clone())
    return b, node, srcs, refs


HOLD = 50_000_000  # torch.cuda._sleep cycles, about 25 ms: far longer than a run of source_batch


def test_ring_of_two_tensors_with_bound_sources(pkg, engine, torch):
    b, node, srcs, refs = source_batch(pkg, engine, torch)
    own = b.output_tensor()
    own.fill_(float("nan"))
    ys = [torch.full(refs[0].shape, float("nan"), device="cuda") for _ in range(2)]
    for step, src in enumerate(srcs):  # A, B, A
        b.bind_sources(node, src)
        b.bind_output(ys[step % 2])
        b.run()
    b.sync()
    assert same_bits(ys[0], refs[2]) and same_bits(ys[1], refs[1])
    assert bool(torch.isnan(own).all())


def test_ring_consumer_is_ordered_after_each_render(pkg, engine, torch):
    """the README ring without a host synchronise, its runs held back on the engine stream: the consumer, reading each half through
    output_tensor(), sees every render complete"""
    b, node, srcs, refs = source_batch(pkg, engine, torch, sets=4)
    ys = [torch.full(refs[0].shape, float("nan"), device="cuda") for _ in range(2)]
    got, prev = [], None
    for step, src in enumerate(srcs):
        b.bind_sources(node, src)
        b.bind_output(ys[step % 2])
        with torch.cuda.stream(b._engine_stream()):
            torch.cuda._sleep(HOLD)
        b.run()
        if prev is not None:
            got.append(prev.clone())
        prev = b.output_tensor()
    got.append(prev.clone())
    torch.cuda.synchronize()
    for k, (g, r) in enumerate(zip(got, refs)):
        assert same_bits(g, r), f"step {k}"


def test_a_kept_binding_waits_for_the_readers_of_its_views(pkg, engine, torch):
    """bound once, run twice: the second run is ordered after the work torch queued on a view of the first (held back, then writing the
    view in place), as a run into the batch's own buffer is"""
    b, node, srcs, refs = source_batch(pkg, engine, torch, sets=1)
    y = torch.full(refs[0].shape, float("nan"), device="cuda")
    b.bind_output(y)
    b.run()
    v = b.output_tensor()
    torch.cuda._sleep(HOLD)
    v.zero_()  # a reader that uses the render in place
    b.run()    # must land after it
    b.sync()
    torch.cuda.synchronize()
    assert same_bits(y, refs[0])


def test_slice_of_a_larger_tensor(pkg, engine, torch):
    b = pkg.Batch([build_chain(pkg, engine.backend, g, 4096 + 3) for g in range(3)])
    floats = b.device_ptr()[1]
    big = torch.full((floats + 64 * 4,), float("nan"), device="cuda")
    out = big[64:64 + floats].view(b.n, b.channels, b.length)
    check_bound(torch, b, out=out)
    assert bool(torch.isnan(big[:64]).all()) and bool(torch.isnan(big[64 + floats:]).all())


def test_unbind_and_read_outs(pkg, engine, torch):
    b = pkg.Batch([build_mix(pkg, engine.backend, g) for g in range(2)])
    out, ref = check_bound(torch, b)
    assert b.device_ptr() == (out.data_ptr(), out.numel())
    host = b.fetch()
    assert np.array_equal(host.view(np.int32), out.cpu().numpy().view(np.int32))
    for i in range(b.n):
        assert np.array_equal(b.fetch_graph(i).view(np.int32), ref[i].cpu().numpy().view(np.int32))
    kept = out.clone()
    b.bind_output(None)
    own = b.output_tensor()
    own.fill_(float("nan"))
    b.run()
    b.sync()
    assert same_bits(own, torch.stack(ref)) and same_bits(out, kept)  # back in the own buffer; the unbound tensor is left alone
    assert b.device_ptr()[0] != out.data_ptr()


def test_refusals(pkg, engine, torch):
    b = pkg.Batch([build_mix(pkg, engine.backend, g) for g in range(2)])
    floats = b.device_ptr()[1]
    fn = pkg.api().batch_bind_output
    big = torch.zeros(floats + 1024, device="cuda")
    seg = next(x for x in torch.cuda.memory_snapshot() if x["address"] <= big.data_ptr() < x["address"] + x["total_size"])
    end = seg["address"] + seg["total_size"]
    host = np.zeros(floats, np.float32)
    p = big.data_ptr()
    assert fn(b.handle, C.c_void_p(p + 4), floats, None) == 1                      # not 256-byte aligned
    assert fn(b.handle, C.c_void_p(p + 64), floats, None) == 1                     # 64 bytes: still not
    assert fn(b.handle, C.c_void_p(p), floats - 1, None) == 1                      # not the batch's output size
    assert fn(b.handle, C.c_void_p(host.ctypes.data), floats, None) == 1           # host memory
    assert fn(b.handle, C.c_void_p(end - 4 * floats + 256), floats, None) == 1     # runs past the end of its allocation
    assert fn(b.handle, None, 1, None) == 1                                        # unbind with a size
    with pytest.raises(pkg.WaeError) as e:
        b.bind_output(torch.zeros((b.n, b.channels, b.length + 1), device="cuda"))
    assert e.value.status == 1
    # nothing was changed: runs still write the own buffer
    assert b.device_ptr()[0] != p
    run(b)
    want = b.output_tensor().clone()
    out = torch.full((b.n, b.channels, b.length), float("nan"), device="cuda")
    b.bind_output(out)
    host_out = np.empty((b.n, b.channels, b.length), np.float32)
    with pytest.raises(pkg.WaeError) as e:
        b.run_pipelined(host_out.ctypes.data)
    assert e.value.status == 2 and "wae_batch_bind_output" in e.value.message
    run(b)
    assert same_bits(out, want)


def test_destination_feeding_another_node_is_refused(pkg, engine, torch):
    c = pkg.OfflineAudioContext(1, 2048, SR, engine.backend)
    o = c.create_oscillator()
    o.connect(c.destination())
    an = c.create_analyser()
    c.destination().connect(an)
    o.start()
    b = pkg.Batch([c])
    with pytest.raises(pkg.WaeError) as e:
        b.bind_output(torch.zeros((1, 1, 2048), device="cuda"))
    assert e.value.status == 2 and "destination" in e.value.message
    b.bind_output(None)  # (nothing is bound: unbinding is allowed)
