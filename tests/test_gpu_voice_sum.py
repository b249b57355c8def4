"""k_voice_sum (csrc/wae_kernels.cu): a port fed by many oscillator -> [biquad] -> gain voices rendered by ONE kernel that keeps the running
sum in registers and walks the voices in the port's edge order — Graph::render's edge summation (graph.rs:489-535) fused with the voices
(examples/many_oscillators.rs, the north_star graph).  The planner only takes that path when the launch has enough (tile, port) work items
(tests/test_planner_cpu.py); here WAE_OPT_VOICE_SUM = 2 forces it on small graphs, and every case is rendered three ways: fused, unfused
(k_chain + k_mix) and on the oracle.  Tolerance 1e-5 absolute (north_star).  The option is OFF by default: on the north_star workload the
kernel measured slower than the two it replaces — it stays in the tree as a tested alternative."""
import numpy as np
import pytest

import graphs as G

pytestmark = pytest.mark.gpu
TOL = 1e-5


def _three_ways(pkg, engine, oracle, build, n, chunk=0):
    outs = []
    for mode in (2, 0):
        engine.set_option(pkg.OPT_VOICE_SUM, mode)
        engine.set_option(pkg.OPT_CHUNK_FRAMES, chunk)
        try:
            ctxs = [build(engine.backend, g) for g in range(n)]
            if mode == 2:
                batch = pkg.Batch(ctxs)
                names = {name for name, _t, _k in batch.stage_times()}
                batch.destroy()
                assert "k_voice_sum" in names, names
                ctxs = [build(engine.backend, g) for g in range(n)]
            outs.append(G.render(pkg, ctxs))
        finally:
            engine.set_option(pkg.OPT_VOICE_SUM, 0)
            engine.set_option(pkg.OPT_CHUNK_FRAMES, 0)
    cpu = G.render(pkg, [build(oracle, g) for g in range(n)])
    fused, unfused = outs
    assert np.isfinite(fused).all()
    assert float(np.abs(fused.astype(np.float64) - cpu).max()) <= TOL
    assert float(np.abs(unfused.astype(np.float64) - cpu).max()) <= TOL
    return fused, unfused, cpu


def test_north_star_voices_into_a_convolver(pkg, engine, oracle):
    ir = G.synthetic_ir(9000, 2, decay=0.2)
    length = 8192 * 2 + 128 * 5
    fused, unfused, cpu = _three_ways(pkg, engine, oracle, lambda be, g: G.north_star_voices_convolver(pkg, be, 40, length, ir, seed=g), 3)
    assert float(np.abs(cpu).max()) > 1e-3


def test_voices_summed_at_the_destination_partial_last_quantum(pkg, engine, oracle):
    # many_oscillators.rs shape: sine -> bandpass -> destination (mono voices, stereo destination: up-mix by copy), a render length that
    # is not a multiple of the quantum (the last quantum is cut, offline.rs:169-180)
    length = 2048 * 3 + 700
    fused, unfused, cpu = _three_ways(pkg, engine, oracle, lambda be, g: G.c3_many_voices(pkg, be, 48 + g, length), 2)
    assert np.array_equal(fused[:, 0], fused[:, 1])  # speakers 1 -> 2 is a copy


def test_state_is_carried_over_tiles_and_chunks(pkg, engine, oracle):
    # chunks of 4096 frames = 2 tiles: the biquad state of every voice goes tile -> tile through the hand-off slots and chunk -> chunk
    # through the filter's own state; the fused and the unfused path cut the render at the same frames, so they agree to the bit
    length = 4096 * 5 + 128 * 3
    fused, unfused, cpu = _three_ways(pkg, engine, oracle, lambda be, g: G.c3_many_voices(pkg, be, 33, length), 2, chunk=4096)
    assert np.array_equal(fused, unfused)


def test_voices_without_a_filter(pkg, engine, oracle):
    def build(be, g):
        c = pkg.OfflineAudioContext(1, 2048 * 2 + 128, 48000.0, be)
        types = [pkg.SINE, pkg.SAWTOOTH, pkg.SQUARE, pkg.TRIANGLE]
        for v in range(12):
            osc = c.create_oscillator(type_=types[v % 4], frequency=110.0 * (v + 1) + 3.0 * g, detune=7.0 * v)
            gn = c.create_gain(0.05 + 0.01 * v)
            osc.connect(gn)
            gn.connect(c.destination())
            osc.start()
        return c
    _three_ways(pkg, engine, oracle, build, 2)


def test_a_port_the_shape_does_not_fit_keeps_the_mixer(pkg, engine, oracle):
    # one voice that stops early has a layout that changes (silent after its tail): the port is folded by k_mix_dyn as before
    def build(be, g):
        c = pkg.OfflineAudioContext(2, 2048 * 2, 48000.0, be)
        for v in range(10):
            osc = c.create_oscillator(frequency=220.0 * (v + 1))
            bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=2000.0, q=1.0)
            osc.connect(bq)
            bq.connect(c.destination())
            osc.start()
            if v == 3:
                osc.stop_at(0.02)
        return c
    engine.set_option(pkg.OPT_VOICE_SUM, 2)
    try:
        batch = pkg.Batch([build(engine.backend, 0)])
        names = {name for name, _t, _k in batch.stage_times()}
        batch.destroy()
        assert "k_voice_sum" not in names
        gpu = G.render(pkg, [build(engine.backend, 0)])
    finally:
        engine.set_option(pkg.OPT_VOICE_SUM, 0)
    cpu = G.render(pkg, [build(oracle, 0)])
    assert float(np.abs(gpu.astype(np.float64) - cpu).max()) <= TOL
