"""DynamicsCompressorNode reduction read-outs at declared render times (wae_compressor_set_readouts) taken on the GPU during a run, against
the oracle's reduction() in suspend_sync callbacks at the same quanta (after the render for the end quantum), within the suite's reduction
tolerance of 1e-3 dB x max(1, sr / 48000); the end quantum's row is bit-equal to wae_compressor_reduction after the render."""
import time

import numpy as np
import pytest

import test_compressor_readouts_cpu as CC
import test_gpu_witnesses_dynamics_spatial as W
from test_gpu_analyser_readouts import engine_with_chunk

pytestmark = pytest.mark.gpu
RQ = 128


def tol(sr):
    return 1e-3 * max(1.0, sr / 48000.0)


def switch_graph(pkg, length, sr, seed=0, params=None):
    """a mono source from the start and a stereo burst inside it: the compressor's input switches between one and two channels"""
    rng = np.random.default_rng(seed)
    mono = rng.uniform(-0.3, 0.3, (1, length + 1)).astype(np.float32)
    burst = rng.uniform(-0.9, 0.9, (2, length)).astype(np.float32)

    def build(be):
        c = pkg.OfflineAudioContext(2, length, sr, be)
        d = c.create_dynamics_compressor(**(params or {}))
        a = c.create_buffer_source(pkg.AudioBuffer(list(mono), sr))
        b = c.create_buffer_source(pkg.AudioBuffer(list(burst), sr))
        a.connect(d)
        b.connect(d)
        d.connect(c.destination())
        a.start()
        b.start_at(length / 4 / sr + 37.0 / sr)
        b.stop_at(length * 0.6 / sr)
        return c, d
    return build


def feedback_graph(pkg, length, sr):
    """a compressor inside a DelayNode feedback cycle"""
    def build(be):
        c = pkg.OfflineAudioContext(1, length, sr, be)
        osc = c.create_oscillator(frequency=330.0)
        dl = c.create_delay(max_delay_time=0.1, delay_time=0.01)
        d = c.create_dynamics_compressor(threshold=-40.0, attack=0.001, release=0.05)
        g = c.create_gain(0.9)
        osc.connect(dl)
        dl.connect(d)
        d.connect(g)
        g.connect(dl)
        d.connect(c.destination())
        osc.start()
        osc.stop_at(length / 3 / sr)
        return c, d
    return build


def gpu_readouts(pkg, eng, builds, quanta_of, many=False, runs=1):
    ctxs, nodes = [], []
    for k, build in enumerate(builds):
        c, d = build(eng.backend)
        d.set_readouts(CC.times_at(quanta_of(k), c._sample_rate))
        ctxs.append(c)
        nodes.append(d)
    b = pkg.context.Batch(ctxs, many=many)
    rows = []
    for _ in range(runs):
        b.run()
        b.sync()
        rows.append([d.get_reduction_readouts() for d in nodes])
    return b, ctxs, nodes, rows


def check(pkg, oracle, build, quanta, sr, got, node=None):
    want, q = CC.oracle_reduction_readouts(pkg, oracle, build, CC.times_at(quanta, sr))
    assert q == list(quanta)
    assert got.shape == want.shape
    assert np.abs(got - want).max() <= tol(sr), (got, want)
    for k in range(1, len(quanta)):
        if quanta[k] == quanta[k - 1]:
            assert got[k] == got[k - 1]
    for k, qk in enumerate(quanta):
        if qk == 0:
            assert got[k] == 0.0
    total = -(-build(oracle)[0]._length // RQ)
    if node is not None and quanta[-1] == total:
        assert got[-1] == np.float32(node.reduction())  # wae_compressor_reduction, bit for bit


@pytest.mark.parametrize("chunk", [128, 1024, 0])
def test_readouts_match_oracle(pkg, engine, oracle, chunk):
    sr, length = 48000.0, RQ * 400 + 77
    total = -(-length // RQ)
    boundary = chunk // RQ if chunk else total // 2
    quanta = sorted([0, 0, 1, 3, boundary, boundary, boundary + 5, 2 * boundary + 1, total - 40, total - 1, total])
    build = switch_graph(pkg, length, sr)
    eng = engine_with_chunk(pkg, chunk) if chunk else engine
    try:
        _, _, nodes, rows = gpu_readouts(pkg, eng, [build], lambda k: quanta)
        check(pkg, oracle, build, quanta, sr, rows[0][0], nodes[0])
    finally:
        if chunk:
            eng.close()


def test_one_chunk_with_a_readout_every_quantum(pkg, oracle):
    sr, length = 44100.0, RQ * 1024
    quanta = list(range(0, 1025))
    build = switch_graph(pkg, length, sr, seed=2, params=dict(attack=0.001, release=0.02))
    eng = engine_with_chunk(pkg, RQ * 1024)
    try:
        _, _, nodes, rows = gpu_readouts(pkg, eng, [build], lambda k: quanta)
        check(pkg, oracle, build, quanta, sr, rows[0][0], nodes[0])
        assert len(set(rows[0][0].tolist())) > 500  # the reduction moves from quantum to quantum
    finally:
        eng.close()


@pytest.mark.parametrize("chunk", [128, 0])
def test_automated_threshold_and_ratio(pkg, engine, oracle, chunk):
    sr, n = 32768.0, RQ * 160  # (a quantum is 2^-8 s: the steps land on quantum boundaries)
    rng = np.random.default_rng(4)
    comp = W._Comp(sr, n, W._comp_inputs(rng, sr, n, 2, "late"), dict(release=0.05),
                   steps=[("threshold", 30, -60.0), ("ratio", 70, 2.0), ("threshold", 100, -10.0), ("ratio", 130, 20.0)])
    quanta = [0, 29, 31, 32, 69, 71, 72, 101, 102, 131, 132, 159, 160]

    def build(be):
        return comp.build(pkg, be)
    eng = engine_with_chunk(pkg, chunk) if chunk else engine
    try:
        _, _, nodes, rows = gpu_readouts(pkg, eng, [build], lambda k: quanta)
        check(pkg, oracle, build, quanta, sr, rows[0][0], nodes[0])
    finally:
        if chunk:
            eng.close()


def test_compressor_inside_a_feedback_cycle(pkg, engine, oracle):
    sr, length = 44100.0, RQ * 120
    quanta = [0, 1, 7, 7, 64, 65, 119, 120]
    build = feedback_graph(pkg, length, sr)
    _, _, nodes, rows = gpu_readouts(pkg, engine, [build], lambda k: quanta)
    check(pkg, oracle, build, quanta, sr, rows[0][0], nodes[0])


def test_prepare_many_of_mixed_lengths_and_rates(pkg, engine, oracle):
    # the two 48 kHz graphs of different lengths share a group: the shorter one's rows stop at its own end
    shapes = [(44100.0, RQ * 90 + 5), (48000.0, RQ * 200), (48000.0, RQ * 170 + 100), (22050.0, RQ * 60), (96000.0, RQ * 300)]
    builds = [switch_graph(pkg, n, sr, seed=k) for k, (sr, n) in enumerate(shapes)]

    def quanta(k):
        total = -(-shapes[k][1] // RQ)
        return [0, total // 3, total // 3, total - 1, total]
    _, _, nodes, rows = gpu_readouts(pkg, engine, builds, quanta, many=True)
    for k, build in enumerate(builds):
        check(pkg, oracle, build, quanta(k), shapes[k][0], rows[0][k], nodes[k])


def test_runs_overwrite_the_rows(pkg, engine, oracle):
    import torch
    sr, length, n = 48000.0, RQ * 150, 4
    quanta = [0, 10, 80, 150]
    builds = [switch_graph(pkg, length, sr, seed=k) for k in range(n)]
    b, _, nodes, rows = gpu_readouts(pkg, engine, builds, lambda k: quanta)
    view = b.compressor_readouts(nodes[0])
    view.fill_(float("nan"))
    torch.cuda.synchronize()
    b.run()
    b.sync()
    again = [d.get_reduction_readouts() for d in nodes]
    for k in range(n):
        assert np.array_equal(again[k], rows[0][k])
    check(pkg, oracle, builds[1], quanta, sr, again[1], nodes[1])


def test_runs_into_a_bound_output_wait_for_readers_of_the_readout_view(pkg, engine):
    import torch
    sr, length, n = 48000.0, RQ * 200, 8
    quanta = [0, 50, 100, 200]
    b, ctxs, nodes, rows = gpu_readouts(pkg, engine, [switch_graph(pkg, length, sr, seed=k) for k in range(n)], lambda k: quanta)
    out = torch.empty((n, 2, length), device="cuda")
    b.bind_output(out)
    b.run()
    view = b.compressor_readouts(nodes[0])
    torch.cuda._sleep(2_000_000_000)  # about one second of the current stream
    copy = view.clone()
    b.run()  # queued behind the sleep and the copy
    time.sleep(0.1)
    assert not b._engine_stream().query(), "the run did not wait for torch's readers of the read-out view"
    torch.cuda.synchronize()
    got = copy.cpu().numpy()  # (the rows of every run are equal: what is checked above is the order)
    for k in range(n):
        assert np.array_equal(got[k], rows[0][k])


def test_a_thousand_graphs_through_the_batch_view(pkg, engine, oracle):
    import torch
    sr, length, n = 48000.0, RQ * 100, 1000
    quanta = [0, 8, 16, 50, 99, 100]
    builds = [switch_graph(pkg, length, sr, seed=k) for k in range(n)]
    b, ctxs, nodes, rows = gpu_readouts(pkg, engine, builds, lambda k: quanta)
    view = b.compressor_readouts(nodes[0].id)
    assert tuple(view.shape) == (n, len(quanta)) and view.dtype == torch.float32
    torch.cuda.synchronize()
    v = view.cpu().numpy()
    for k in range(n):
        assert np.array_equal(v[k], rows[0][k])
    for k in (0, 517, 999):
        check(pkg, oracle, builds[k], quanta, sr, v[k], nodes[k])


def test_undeclared_compressors_next_to_declared_ones_render_as_before(pkg, engine, oracle):
    # a batch where half the compressors declare read-outs: the other half run the undeclared kernel and render exactly what a batch
    # without any declaration renders; the declared half's PCM is the same too
    sr, length, n = 48000.0, RQ * 300, 6
    builds = [switch_graph(pkg, length, sr, seed=k) for k in range(n)]
    quanta = [0, 100, 299, 300]

    def render(declared):
        ctxs, nodes = [], []
        for k, build in enumerate(builds):
            c, d = build(engine.backend)
            if k in declared:
                d.set_readouts(CC.times_at(quanta, sr))
            ctxs.append(c)
            nodes.append(d)
        b = pkg.context.Batch(ctxs)
        b.run()
        b.sync()
        return [b.fetch_graph(k) for k in range(n)], nodes
    plain, _ = render(set())
    mixed, nodes = render({1, 3, 4})
    for k in range(n):
        assert np.array_equal(plain[k], mixed[k]), k
    for k in (1, 3, 4):
        check(pkg, oracle, builds[k], quanta, sr, nodes[k].get_reduction_readouts(), nodes[k])
