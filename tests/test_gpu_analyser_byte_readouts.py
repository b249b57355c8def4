"""AnalyserNode byte read-outs at declared render times (wae_analyser_set_byte_readouts) taken on the GPU during a run.  Each byte row is
exactly the reference's f32 formula applied to the GPU's own float row of the same run, and within 1 of the oracle's get_byte_* in
suspend_sync callbacks at the same quanta; the float rows are bit-identical to those of the same graphs declared without bytes."""
import numpy as np
import pytest

import test_analyser_byte_readouts_cpu as BC
from test_gpu_analyser_readouts import engine_with_chunk, feedback_graph, layout_graph, times_at

pytestmark = pytest.mark.gpu
RQ = 128


def gpu_readouts(pkg, eng, builds, quanta_of, byte=True, many=False, runs=1):
    """-> batch, analysers, [run][graph] (freq dB, time, byte freq, byte time)"""
    ctxs, nodes = [], []
    for k, build in enumerate(builds):
        c, a = build(eng.backend)
        a.set_readouts(times_at(quanta_of(k), c._sample_rate), frequency=True, time_domain=True)
        if byte:
            a.set_byte_readouts(frequency=True, time_domain=True)
        ctxs.append(c)
        nodes.append(a)
    b = pkg.context.Batch(ctxs, many=many)
    rows = []
    for _ in range(runs):
        b.run()
        b.sync()
        rows.append([(a.get_float_frequency_readouts(), a.get_float_time_domain_readouts()) +
                     ((a.get_byte_frequency_readouts(), a.get_byte_time_domain_readouts()) if byte else ()) for a in nodes])
    return b, nodes, rows


def check(pkg, oracle, build, quanta, got, min_db=-100.0, max_db=-30.0):
    f, t, bf, bt = got
    assert bf.dtype == np.uint8 and bt.dtype == np.uint8
    assert np.array_equal(bf, BC.byte_frequency(f, min_db, max_db))  # the formula of the GPU's own float rows
    assert np.array_equal(bt, BC.byte_time_domain(t))
    (_, _, wbf, wbt), _ = BC.oracle_all_readouts(pkg, oracle, build, times_at(quanta, build(oracle)[0]._sample_rate))
    assert bf.shape == wbf.shape and bt.shape == wbt.shape
    assert np.abs(bf.astype(int) - wbf).max() <= 1
    assert np.abs(bt.astype(int) - wbt).max() <= 1


@pytest.mark.parametrize("fft_size,chunk", [(32, 128), (2048, 1024), (2048, 0), (32768, 0)])
def test_byte_readouts_match_oracle_and_leave_the_float_rows(pkg, engine, oracle, fft_size, chunk):
    sr, length = 48000.0, RQ * 400 + 77
    total = -(-length // RQ)
    boundary = chunk // RQ if chunk else total // 2
    quanta = sorted([0, 3, boundary, boundary, boundary + 5, total - 1, total])
    build = layout_graph(pkg, length, sr, fft_size, 0.8)
    eng = engine_with_chunk(pkg, chunk) if chunk else engine
    try:
        _, nodes, rows = gpu_readouts(pkg, eng, [build], lambda k: quanta)
        _, _, plain = gpu_readouts(pkg, eng, [build], lambda k: quanta, byte=False)
        check(pkg, oracle, build, quanta, rows[0][0])
        assert np.array_equal(rows[0][0][0], plain[0][0][0]) and np.array_equal(rows[0][0][1], plain[0][0][1])
        # the end quantum: the post-render getters (which convert on the host) give the last rows
        assert np.array_equal(nodes[0].get_byte_frequency_data(), rows[0][0][2][-1])
        assert np.array_equal(nodes[0].get_byte_time_domain_data(), rows[0][0][3][-1])
    finally:
        if chunk:
            eng.close()


def test_decibel_range_and_clipping(pkg, engine, oracle):
    # a loud input: time-domain bytes clip at 0 and 255, spectra pass max_db; the node's min / max decibels at render time
    sr, length = 44100.0, RQ * 60
    quanta = [0, 3, 3, 17, 40, 59, 60]
    build = BC.loud_graph(pkg, length, sr, 256, 0.8, -60.0, -20.0)
    _, _, rows = gpu_readouts(pkg, engine, [build], lambda k: quanta)
    check(pkg, oracle, build, quanta, rows[0][0], -60.0, -20.0)
    bf, bt = rows[0][0][2], rows[0][0][3]
    assert (bt == 255).any() and (bt == 0).any() and (bf == 255).any() and (bf[0] == 0).all()


def test_feedback_cycle_and_repeated_runs(pkg, engine, oracle):
    sr, length = 44100.0, RQ * 120
    quanta = [0, 1, 7, 7, 64, 65, 119, 120]
    build = feedback_graph(pkg, length, sr, 1024, 0.8)
    _, _, rows = gpu_readouts(pkg, engine, [build], lambda k: quanta, runs=2)
    check(pkg, oracle, build, quanta, rows[0][0])
    for a, b in zip(rows[0][0], rows[1][0]):
        assert np.array_equal(a, b)


def test_prepare_many_with_some_graphs_declaring_bytes(pkg, engine, oracle):
    shapes = [(44100.0, RQ * 90 + 5), (48000.0, RQ * 200), (48000.0, RQ * 170 + 100), (22050.0, RQ * 60)]
    builds = [layout_graph(pkg, n, sr, 2048, 0.8, seed=k) for k, (sr, n) in enumerate(shapes)]

    def quanta(k):
        total = -(-shapes[k][1] // RQ)
        return [0, total // 3, total // 3, total - 1, total]
    ctxs, nodes = [], []
    for k, build in enumerate(builds):
        c, a = build(engine.backend)
        a.set_readouts(times_at(quanta(k), shapes[k][0]), frequency=True, time_domain=True)
        if k != 1:
            a.set_byte_readouts(frequency=True, time_domain=True)
        ctxs.append(c)
        nodes.append(a)
    b = pkg.context.Batch(ctxs, many=True)
    b.run()
    b.sync()
    with pytest.raises(pkg.WaeError):
        b.analyser_readouts(nodes[0], byte=True)  # graph 1 declares no bytes: no [n][K][row] view
    with pytest.raises(pkg.WaeError):
        nodes[1].get_byte_frequency_readouts()
    for k, build in enumerate(builds):
        if k == 1:
            continue
        a = nodes[k]
        got = (a.get_float_frequency_readouts(), a.get_float_time_domain_readouts(), a.get_byte_frequency_readouts(),
               a.get_byte_time_domain_readouts())
        check(pkg, oracle, build, quanta(k), got)


def test_a_thousand_graphs_through_the_byte_view(pkg, engine, oracle):
    import torch
    sr, length, n = 48000.0, RQ * 100, 1000
    quanta = [0, 8, 16, 50, 99, 100]
    builds = [layout_graph(pkg, length, sr, 256, 0.8, seed=k) for k in range(n)]
    b, nodes, rows = gpu_readouts(pkg, engine, builds, lambda k: quanta)
    view = b.analyser_readouts(nodes[0], "frequency", byte=True)
    tview = b.analyser_readouts(nodes[0].id, "time_domain", byte=True)
    assert tuple(view.shape) == (n, len(quanta), 128) and tuple(tview.shape) == (n, len(quanta), 256)
    assert view.dtype == torch.uint8 and tview.dtype == torch.uint8
    torch.cuda.synchronize()
    vf, vt = view.cpu().numpy(), tview.cpu().numpy()
    for k in range(n):
        assert np.array_equal(vf[k], rows[0][k][2]) and np.array_equal(vt[k], rows[0][k][3])
    for k in (0, 517, 999):
        check(pkg, oracle, builds[k], quanta, rows[0][k])
