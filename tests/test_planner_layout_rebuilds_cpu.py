"""Planner (CPU, wae_batch_plan): the two dynamic layouts that used to be refused — a ConvolverNode with a ONE-channel response whose input
switches between one and two channels (convolver.rs:378-400), and an over-sampled WaveShaperNode whose input changes its channel count
(waveshaper.rs:409-420) — are lowered, and the fuzz generator's graphs are planned without a single refusal."""
import os

import numpy as np
import pytest

import graphs as G

SR = 48000.0


@pytest.fixture
def be(pkg):
    so = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "web-audio-api-rs_b200", "libwae_b200.so")
    if not os.path.exists(so):
        pytest.skip("libwae_b200.so is not built (python -c 'import __graft_entry__ as g; g.build()')")
    return pkg.context.Backend(pkg.api(), None)


def stereo_source(pkg, c, seed, frames, start):
    pcm = np.random.default_rng(seed).uniform(-0.5, 0.5, (2, frames)).astype(np.float32)
    s = c.create_buffer_source(pkg.AudioBuffer(list(pcm), SR))
    s.start_at(start)
    return s


def late_stereo_into_convolver(pkg, be, ir_channels):
    c = pkg.OfflineAudioContext(2, int(SR), SR, be)
    cv = c.create_convolver(pkg.AudioBuffer(G.synthetic_ir(12000, ir_channels), SR))
    stereo_source(pkg, c, 1, 12000, 0.5).connect(cv)
    cv.connect(c.destination())
    return c


def panned_tone_into_convolver(pkg, be):
    c = pkg.OfflineAudioContext(2, int(1.2 * SR), SR, be)
    o = c.create_oscillator(frequency=440.0)
    o.start_at(0.1)
    o.stop_at(1.0)
    p = c.create_stereo_panner(0.3)
    cv = c.create_convolver(pkg.AudioBuffer(G.synthetic_ir(12000, 1), SR))
    o.connect(p)
    p.connect(cv)
    cv.connect(c.destination())
    return c


def late_stereo_into_x2_shaper(pkg, be):
    c = pkg.OfflineAudioContext(2, int(SR), SR, be)
    sh = c.create_wave_shaper(curve=np.linspace(-0.5, 1.0, 9).astype(np.float32), oversample=pkg.OVERSAMPLE_X2)
    stereo_source(pkg, c, 2, 12000, 0.5).connect(sh)
    sh.connect(c.destination())
    return c


def test_mono_response_behind_a_changing_input_gets_the_compacted_path(pkg, be):
    # stereo source started at 0.5 s -> mono response: path 0 on the usual kernels, path 1 on the compacted stage
    k = pkg.context.plan_batch([late_stereo_into_convolver(pkg, be, 1)])["kinds"]
    assert k.get("k_conv_compact") == 1 and "k_conv_fft_in" in k and "k_conv_mac_ifft" in k
    k = pkg.context.plan_batch([panned_tone_into_convolver(pkg, be)])["kinds"]
    assert k.get("k_conv_compact") == 1
    # a stereo response keeps its two ordinary paths (both convolvers are fed every quantum)
    k = pkg.context.plan_batch([late_stereo_into_convolver(pkg, be, 2)])["kinds"]
    assert "k_conv_compact" not in k and "k_conv_mac_ifft" in k


def test_over_sampled_shaper_behind_a_changing_input_is_lowered(pkg, be):
    k = pkg.context.plan_batch([late_stereo_into_x2_shaper(pkg, be)])["kinds"]
    assert "k_shaper_os" in k and "k_meta" in k  # (the output's layout track: a silent input still sounds, on one channel)


def test_the_new_graphs_batch_with_c4_graphs_and_suspend_points(pkg, be):
    ir = G.synthetic_ir(20000, 1)
    ctxs = [G.c4_convolver(pkg, be, g, 8192 * 3, ir) for g in range(2)]
    c = pkg.OfflineAudioContext(2, 8192 * 3, SR, be)
    cv = c.create_convolver(pkg.AudioBuffer(ir, SR))
    stereo_source(pkg, c, 3, 6000, 0.05).connect(cv)
    cv.connect(c.destination())
    c.suspend_sync(8192 / SR, lambda _c: stereo_source(pkg, _c, 4, 3000, 0.2).connect(cv))
    p = pkg.context.plan_batch(ctxs + [c])
    assert p["kinds"].get("k_conv_compact", 0) >= 1 and p["segments"] >= 2


@pytest.mark.parametrize("block", range(8))
def test_random_graphs_are_planned_without_refusal(pkg, be, block):
    # the seeds of test_planner_cpu.py::test_planner_accepts_random_graphs (8 x 40) and of tools/plan_digest_corpus.py (4000 - 4399):
    # no graph of the fuzz generator is refused any more
    import test_gpu_fuzz as F
    seeds = list(range(1000 + 40 * block, 1000 + 40 * (block + 1))) + list(range(4000 + 50 * block, 4000 + 50 * (block + 1)))
    for seed in seeds:
        p = pkg.context.plan_batch([F.random_graph(pkg, be, seed)])
        assert 1 <= p["stages"] <= 400, seed


def gap_into_mono_response(pkg, be, after):
    c = pkg.OfflineAudioContext(2, 8192 * 8, SR, be)
    cv = c.create_convolver(pkg.AudioBuffer(G.synthetic_ir(36000, 1), SR))
    stereo_source(pkg, c, 5, 20000, 0.0).connect(cv)
    stereo_source(pkg, c, 6, 15000, 41000 / SR).connect(cv)
    node = after(c)
    cv.connect(node)
    node.connect(c.destination())
    return c


def test_the_compacted_convolver_output_can_sound_on_one_channel(pkg, be):
    # while the response rings on a silent input the output is ONE sounding channel: a biquad behind it has to follow the count
    # (serial kernel, channels dropped and restarted), an over-sampled shaper through 0 has to rebuild its resamplers
    k = pkg.context.plan_batch([gap_into_mono_response(pkg, be, lambda c: c.create_biquad_filter())])["kinds"]
    assert "k_biquad_serial" in k  # (not the scan of k_chain, which assumes a constant count)
    tanh = np.tanh(np.linspace(-3, 3, 33)).astype(np.float32)
    k = pkg.context.plan_batch([gap_into_mono_response(pkg, be, lambda c: c.create_wave_shaper(curve=tanh, oversample=pkg.OVERSAMPLE_X2))])["kinds"]
    assert "k_shaper_os" in k


def test_a_mono_response_switching_paths_at_a_suspend_point_is_refused(pkg, be):
    # constant stereo input in the first segment (ordinary second path), a stop time set from the callback makes it change in the
    # second one (compacted path): the second convolver's history cannot be handed from one representation to the other
    c = pkg.OfflineAudioContext(2, 8192 * 4, SR, be)
    cv = c.create_convolver(pkg.AudioBuffer(G.synthetic_ir(12000, 1), SR))
    s = stereo_source(pkg, c, 7, 8192 * 4, 0.0)
    s.connect(cv)
    cv.connect(c.destination())
    c.suspend_sync(8192 * 2 / SR, lambda _c: s.stop_at(0.5))
    with pytest.raises(pkg.WaeError) as e:
        pkg.context.plan_batch([c])
    assert e.value.status == 4 and "suspend point" in str(e.value)
    # a tone alone, then a stereo source added from the callback: the second convolver was never fed before, the graph is lowered
    c = pkg.OfflineAudioContext(2, 8192 * 4, SR, be)
    cv = c.create_convolver(pkg.AudioBuffer(G.synthetic_ir(12000, 1), SR))
    o = c.create_oscillator()
    o.start()
    o.connect(cv)
    cv.connect(c.destination())
    c.suspend_sync(8192 * 2 / SR, lambda _c: stereo_source(pkg, _c, 8, 3000, 0.4).connect(cv))
    p = pkg.context.plan_batch([c])
    assert p["segments"] == 2 and p["kinds"].get("k_conv_compact") == 1
