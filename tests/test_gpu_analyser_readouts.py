"""AnalyserNode read-outs at declared render times (wae_analyser_set_readouts) taken on the GPU during a run, against the oracle's
read-outs in suspend_sync callbacks at the same quanta (after the render for the end quantum), at the suite's analyser tolerances:
linear magnitudes within 1e-6, dB within 1e-2 where the bin is above 1e-4, time domain within 1e-5."""
import time

import numpy as np
import pytest

import test_analyser_readouts_cpu as RC

pytestmark = pytest.mark.gpu
RQ = 128
OPT_CHUNK_FRAMES = 1


def check(gpu_f, gpu_t, want_f, want_t):
    assert gpu_f.shape == want_f.shape and gpu_t.shape == want_t.shape
    lin_g, lin_c = 10.0 ** (gpu_f.astype(np.float64) / 20), 10.0 ** (want_f.astype(np.float64) / 20)
    assert np.abs(lin_g - lin_c).max() <= 1e-6
    loud = lin_c > 1e-4
    assert loud.any() and np.abs(gpu_f[loud] - want_f[loud]).max() <= 1e-2
    assert np.abs(gpu_t - want_t).max() <= 1e-5


def layout_graph(pkg, length, sr, fft_size, tau, seed=0):
    """a mono oscillator from the start and a stereo buffer source that starts late and stops early: the analyser's input switches
    between one and two channels"""
    rng = np.random.default_rng(seed)
    pcm = rng.uniform(-0.5, 0.5, (2, length // 2)).astype(np.float32)

    def build(be):
        c = pkg.OfflineAudioContext(2, length, sr, be)
        osc = c.create_oscillator(frequency=440.0 * (1 + seed % 5))
        src = c.create_buffer_source(pkg.AudioBuffer([pcm[0], pcm[1]], sr))
        a = c.create_analyser(fft_size=fft_size, smoothing_time_constant=tau)
        osc.connect(a)
        src.connect(a)
        a.connect(c.destination())
        osc.start()
        src.start_at(length / 4 / sr + 37.0 / sr)
        src.stop_at(length * 0.6 / sr)
        return c, a
    return build


def feedback_graph(pkg, length, sr, fft_size, tau):
    """an analyser inside a DelayNode feedback cycle"""
    def build(be):
        c = pkg.OfflineAudioContext(1, length, sr, be)
        osc = c.create_oscillator(frequency=330.0)
        d = c.create_delay(max_delay_time=0.1, delay_time=0.01)
        a = c.create_analyser(fft_size=fft_size, smoothing_time_constant=tau)
        g = c.create_gain(0.6)
        osc.connect(d)
        d.connect(a)
        a.connect(g)
        g.connect(d)
        a.connect(c.destination())
        osc.start()
        osc.stop_at(length / 3 / sr)
        return c, a
    return build


def gpu_readouts(pkg, eng, builds, times_of, many=False, runs=1):
    ctxs, nodes = [], []
    for k, build in enumerate(builds):
        c, a = build(eng.backend)
        a.set_readouts(times_of(k, c), frequency=True, time_domain=True)
        ctxs.append(c)
        nodes.append(a)
    b = pkg.context.Batch(ctxs, many=many)
    rows = []
    for _ in range(runs):
        b.run()
        b.sync()
        rows.append([(a.get_float_frequency_readouts(), a.get_float_time_domain_readouts()) for a in nodes])
    return b, ctxs, nodes, rows


def times_at(quanta, sr):
    # (half a frame before the quantum's first frame: ceil(t sr / 128) is exactly q, whatever the rounding of q * 128 / sr)
    return [max(q * RQ - 0.5, 0.0) / sr for q in quanta]


def engine_with_chunk(pkg, chunk):
    e = pkg.Engine(0)
    if chunk:
        e.set_option(OPT_CHUNK_FRAMES, chunk)
    return e


@pytest.mark.parametrize("fft_size,chunk", [(f, c) for f in (32, 2048, 32768) for c in (128, 1024, 0) if (f, c) != (32768, 128)])
@pytest.mark.parametrize("tau", [0.0, 0.8])
def test_readouts_match_oracle(pkg, engine, oracle, fft_size, tau, chunk):
    sr, length = 48000.0, RQ * 400 + 77
    total = -(-length // RQ)
    # quantum 0, mid-chunk, on a chunk boundary (chunk 0: the default chunk of a one-graph render is the whole render, so this is only
    # mid-render), duplicated, late, the end quantum
    boundary = chunk // RQ if chunk else total // 2
    quanta = sorted([0, 3, boundary, boundary, boundary + 5, 2 * boundary + 1, total - 40, total - 1, total])
    quanta = [min(q, total) for q in quanta]
    build = layout_graph(pkg, length, sr, fft_size, tau)
    eng = engine_with_chunk(pkg, chunk) if chunk else engine
    try:
        _, _, _, rows = gpu_readouts(pkg, eng, [build], lambda k, c: times_at(quanta, sr))
        want_f, want_t, _ = RC.oracle_readouts(pkg, oracle, build, times_at(quanta, sr))
        check(rows[0][0][0], rows[0][0][1], want_f, want_t)
    finally:
        if chunk:
            eng.close()


def test_long_chunk_with_late_readouts(pkg, oracle):
    # one chunk of 128 K frames (f0 = 0): every window comes from the input buffer, reaching further back than the ring holds
    sr, length = 48000.0, RQ * 1024
    quanta = [700, 900, 1000, 1023, 1024]
    build = layout_graph(pkg, length, sr, 32768, 0.8, seed=3)
    eng = engine_with_chunk(pkg, RQ * 1024)
    try:
        _, _, _, rows = gpu_readouts(pkg, eng, [build], lambda k, c: times_at(quanta, sr))
    finally:
        eng.close()
    want_f, want_t, _ = RC.oracle_readouts(pkg, oracle, build, times_at(quanta, sr))
    check(rows[0][0][0], rows[0][0][1], want_f, want_t)


def test_long_chunks_with_early_readouts(pkg, oracle):
    # two chunks of 64 K frames, longer than the ring (32 768 + 128 frames): the windows of read-outs early in the second chunk come
    # mostly from the ring, whose slots that chunk's own k_analyser rewrites; the read-outs must run first
    sr, length, chunk = 48000.0, RQ * 1024, RQ * 512
    quanta = [513, 517, 517, 612, 1024]
    build = layout_graph(pkg, length, sr, 32768, 0.8, seed=4)
    eng = engine_with_chunk(pkg, chunk)
    try:
        _, _, _, rows = gpu_readouts(pkg, eng, [build], lambda k, c: times_at(quanta, sr))
    finally:
        eng.close()
    want_f, want_t, _ = RC.oracle_readouts(pkg, oracle, build, times_at(quanta, sr))
    check(rows[0][0][0], rows[0][0][1], want_f, want_t)


def test_runs_into_a_bound_output_wait_for_readers_of_the_readout_view(pkg, engine):
    # the read-out rows are the batch's own memory even while the rendered PCM goes to a bound tensor: once a view of them is handed
    # out, a run waits for the work queued on torch's current stream (here a long sleep, then a copy of the view)
    import torch
    sr, length, n = 48000.0, RQ * 200, 8
    quanta = [0, 50, 100, 200]
    b, ctxs, nodes, rows = gpu_readouts(pkg, engine, [layout_graph(pkg, length, sr, 1024, 0.8, seed=k) for k in range(n)],
                                        lambda k, c: times_at(quanta, sr))
    out = torch.empty((n, 2, length), device="cuda")
    b.bind_output(out)
    b.run()
    view = b.analyser_readouts(nodes[0])
    torch.cuda._sleep(2_000_000_000)  # about one second of the current stream
    copy = view.clone()
    b.run()  # queued behind the sleep and the copy
    time.sleep(0.1)
    assert not b._engine_stream().query(), "the run did not wait for torch's readers of the read-out view"
    torch.cuda.synchronize()
    got = copy.cpu().numpy()  # (the rows of every run are equal: what is checked above is the order)
    for k in range(n):
        assert np.array_equal(got[k], rows[0][k][0])


@pytest.mark.parametrize("tau", [0.0, 0.8])
def test_analyser_inside_a_feedback_cycle(pkg, engine, oracle, tau):
    sr, length = 44100.0, RQ * 120
    quanta = [0, 1, 7, 7, 64, 65, 119, 120]
    build = feedback_graph(pkg, length, sr, 1024, tau)
    _, _, _, rows = gpu_readouts(pkg, engine, [build], lambda k, c: times_at(quanta, sr))
    want_f, want_t, _ = RC.oracle_readouts(pkg, oracle, build, times_at(quanta, sr))
    check(rows[0][0][0], rows[0][0][1], want_f, want_t)


def test_prepare_many_of_mixed_lengths_and_rates(pkg, engine, oracle):
    shapes = [(44100.0, RQ * 90 + 5), (48000.0, RQ * 200), (48000.0, RQ * 170 + 100), (22050.0, RQ * 60)]
    builds = [layout_graph(pkg, n, sr, 2048, 0.8, seed=k) for k, (sr, n) in enumerate(shapes)]

    def quanta(k):
        total = -(-shapes[k][1] // RQ)
        return [0, total // 3, total // 3, total - 1, total]
    _, _, _, rows = gpu_readouts(pkg, engine, builds, lambda k, c: times_at(quanta(k), shapes[k][0]), many=True)
    for k, build in enumerate(builds):
        want_f, want_t, _ = RC.oracle_readouts(pkg, oracle, build, times_at(quanta(k), shapes[k][0]))
        check(rows[0][k][0], rows[0][k][1], want_f, want_t)


@pytest.mark.parametrize("at_end", [False, True])
def test_post_render_readout_continues_the_smoothing_and_runs_repeat(pkg, engine, oracle, at_end):
    sr, length = 48000.0, RQ * 150
    quanta = [10, 80, 150] if at_end else [10, 80, 100]
    build = layout_graph(pkg, length, sr, 2048, 0.8, seed=1)
    _, _, nodes, rows = gpu_readouts(pkg, engine, [build], lambda k, c: times_at(quanta, sr), runs=2)
    assert np.array_equal(rows[0][0][0], rows[1][0][0]) and np.array_equal(rows[0][0][1], rows[1][0][1])
    post = nodes[0].get_float_frequency_data()
    # the oracle: the same read-outs in callbacks, then its own post-render read-out
    c, a = build(oracle)
    for q in quanta:
        if q < 150:
            c.suspend_sync(times_at([q], sr)[0], lambda ctx: a.get_float_frequency_data())
    c.start_rendering_sync()
    if at_end:
        a.get_float_frequency_data()
    want = a.get_float_frequency_data()
    check(post[None], np.zeros((1, 1)), want[None], np.zeros((1, 1)))
    if at_end:
        assert np.array_equal(post, rows[1][0][0][-1])


def test_a_thousand_graphs_through_the_batch_view(pkg, engine, oracle):
    import torch
    sr, length, n = 48000.0, RQ * 100, 1000
    quanta = [0, 8, 16, 50, 99, 100]
    builds = [layout_graph(pkg, length, sr, 256, 0.8, seed=k) for k in range(n)]
    b, ctxs, nodes, rows = gpu_readouts(pkg, engine, builds, lambda k, c: times_at(quanta, sr))
    view = b.analyser_readouts(nodes[0], "frequency")
    tview = b.analyser_readouts(nodes[0].id, "time_domain")
    assert tuple(view.shape) == (n, len(quanta), 128) and tuple(tview.shape) == (n, len(quanta), 256)
    torch.cuda.synchronize()
    vf, vt = view.cpu().numpy(), tview.cpu().numpy()
    for k in range(n):
        assert np.array_equal(vf[k], rows[0][k][0]) and np.array_equal(vt[k], rows[0][k][1])
    for k in (0, 517, 999):
        want_f, want_t, _ = RC.oracle_readouts(pkg, oracle, builds[k], times_at(quanta, sr))
        check(vf[k], vt[k], want_f, want_t)
