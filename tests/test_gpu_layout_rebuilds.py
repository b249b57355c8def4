"""The two dynamic layouts the planner used to refuse, rendered on the GPU against the oracle (1e-5):

* a ConvolverNode with a ONE-channel response whose input switches between one and two channels: the reference's second convolver is
  fed the right channel of the two-channel quanta only and freezes in between (convolver.rs:378-400) — the compacted path
  (k_conv_compact: map, stream window, transforms over the stream's blocks, scatter back);
* an over-sampled WaveShaperNode (X2 / X4) whose input changes its channel count: its resamplers are rebuilt with zero state
  (waveshaper.rs:409-420) — k_shaper_os_prev records the rebuilds, k_shaper_os reads older history as zero."""
import numpy as np
import pytest

import graphs as G

pytestmark = pytest.mark.gpu
TOL = 1e-5
SR = G.SR


def maxdiff(a, b):
    return float(np.abs(a.astype(np.float64) - b.astype(np.float64)).max())


def check(pkg, engine, oracle, build, n=3, tol=TOL):
    gpu = G.render(pkg, [build(engine.backend, g) for g in range(n)])
    cpu = G.render(pkg, [build(oracle, g) for g in range(n)])
    assert np.isfinite(cpu).all()
    err = maxdiff(gpu, cpu)
    assert err <= tol, err
    return gpu, cpu


def stereo_pcm(seed, frames, amp=0.5):
    return np.random.default_rng(seed).uniform(-amp, amp, (2, frames)).astype(np.float32)


def stereo_source(pkg, c, seed, frames, start_frame):
    s = c.create_buffer_source(pkg.AudioBuffer(list(stereo_pcm(seed, frames)), SR))
    s.start_at(start_frame / SR)
    return s


def mono_ir(frames, seed=5, decay=0.3, gain=1.0):
    return [c * np.float32(gain) for c in G.synthetic_ir(frames, 1, seed=seed, decay=decay)]


# ---------------------------------------------------------------------------------------------- mono response, compacted second path
def test_mono_response_freezes_and_resumes(pkg, engine, oracle):
    """stereo source A, a gap, stereo source B into a response of several 8192-frame partitions: convolvers[1] stops with A's tail in
    its history and resumes from it when B starts"""
    n = 8192 * 9 + 333
    ir = mono_ir(36000, gain=0.01)  # (no normalization: outputs of order 1)
    a_len, b0 = 20000 + 77, 41000 + 45

    def build(be, g):
        c = pkg.OfflineAudioContext(2, n, SR, be)
        cv = c.create_convolver(pkg.AudioBuffer(ir, SR), disable_normalization=True)
        stereo_source(pkg, c, 10 + g, a_len, 0).connect(cv)
        stereo_source(pkg, c, 20 + g, 15000 + 100 * g, b0).connect(cv)
        cv.connect(c.destination())
        return c
    gpu, _ = check(pkg, engine, oracle, build)
    # not a trivial case: the right channel is not the unfrozen convolution of the right input
    r = np.zeros(n)
    r[:a_len] = stereo_pcm(10, a_len)[1]
    b = stereo_pcm(20, 15000)[1]
    r[b0:b0 + len(b)] = b
    unfrozen = np.convolve(r, ir[0].astype(np.float64))[:n]
    q0 = (b0 // 128) * 128
    assert np.abs(gpu[0, 1, q0:b0 + 15000] - unfrozen[q0:b0 + 15000]).max() > 1e-3


def test_mono_response_behind_a_panner_that_starts_and_stops(pkg, engine, oracle):
    n = 8192 * 4 + 1000

    def build(be, g):
        c = pkg.OfflineAudioContext(2, n, SR, be)
        o = c.create_oscillator(type_=pkg.SAWTOOTH, frequency=180.0 + 40 * g)
        o.start_at(0.05)
        o.stop_at(0.45)
        p = c.create_stereo_panner(0.4 - 0.3 * g)
        cv = c.create_convolver(pkg.AudioBuffer(mono_ir(12000), SR))
        o.connect(p)
        p.connect(cv)
        cv.connect(c.destination())
        return c
    check(pkg, engine, oracle, build)


def test_mono_response_behind_a_tone_and_a_stereo_source_that_ends(pkg, engine, oracle):
    n = 8192 * 4 + 500

    def build(be, g):
        c = pkg.OfflineAudioContext(2, n, SR, be)
        cv = c.create_convolver(pkg.AudioBuffer(mono_ir(17000), SR))
        o = c.create_oscillator(frequency=220.0 + 30 * g)
        o.start()
        o.connect(cv)
        stereo_source(pkg, c, 30 + g, 9000 + 500 * g, 3000).connect(cv)
        cv.connect(c.destination())
        return c
    gpu, _ = check(pkg, engine, oracle, build)
    assert np.array_equal(gpu[0, 0, 20000:], gpu[0, 1, 20000:])  # mono again once the stereo source has ended


def test_mono_response_runs_out_its_tail_on_a_silent_input(pkg, engine, oracle):
    n = 8192 * 5

    def build(be, g):
        c = pkg.OfflineAudioContext(2, n, SR, be)
        cv = c.create_convolver(pkg.AudioBuffer(mono_ir(9000), SR))
        stereo_source(pkg, c, 40 + g, 6000, 1000 + 300 * g).connect(cv)
        cv.connect(c.destination())
        return c
    gpu, _ = check(pkg, engine, oracle, build)
    assert np.abs(gpu[:, :, 30000:]).max() == 0.0  # silent once the input has been silent for the response's length


@pytest.mark.parametrize("chunk", [8192, 0])
def test_mono_response_does_not_depend_on_the_chunk_size(pkg, engine, oracle, chunk):
    """several chunks plus an odd remainder; the input switches between one and two channels inside chunks and across chunk boundaries,
    so the partial stream block is carried from chunk to chunk"""
    n = 8192 * 6 + 1234

    def build(be, g):
        c = pkg.OfflineAudioContext(2, n, SR, be)
        cv = c.create_convolver(pkg.AudioBuffer(mono_ir(26000, gain=0.01), SR), disable_normalization=True)
        o = c.create_oscillator(frequency=300.0 + 20 * g)
        o.start()
        o.connect(cv)
        for k, (start, frames) in enumerate([(5000, 12000), (16300, 9000), (30000 + 128 * g, 3000), (40900, 9500)]):
            stereo_source(pkg, c, 50 + 7 * g + k, frames, start).connect(cv)
        cv.connect(c.destination())
        return c
    engine.set_option(pkg.OPT_CHUNK_FRAMES, chunk)
    try:
        check(pkg, engine, oracle, build)
    finally:
        engine.set_option(pkg.OPT_CHUNK_FRAMES, 0)


def test_mono_response_lives_across_a_suspend_point_and_batches_with_c4(pkg, engine, oracle):
    n = 8192 * 4 + 100
    ir = mono_ir(20000)

    def build(be, g):
        if g % 2 == 1:  # C4-shaped: stereo source over the whole render -> stereo response
            return G.c4_convolver(pkg, be, g, n, G.synthetic_ir(20000, 2))
        c = pkg.OfflineAudioContext(2, n, SR, be)
        cv = c.create_convolver(pkg.AudioBuffer(ir, SR))
        stereo_source(pkg, c, 60 + g, 7000, 2000).connect(cv)
        cv.connect(c.destination())
        c.suspend_sync(8192 * 2 / SR, lambda _c: stereo_source(pkg, _c, 70 + g, 5000, 8192 * 2 + 3000).connect(cv))
        return c
    check(pkg, engine, oracle, build, n=4)


# ---------------------------------------------------------------------------------------------- over-sampled shaper, resampler rebuilds
def shaper_graph(pkg, be, g, kind, oversample, n):
    c = pkg.OfflineAudioContext(2, n, SR, be)
    if kind == "through_zero":  # curve maps 0 to 0: silent quanta are not processed; mono and stereo quanta alternate
        curve = np.tanh(np.linspace(-3, 3, 33)).astype(np.float32)
    else:                       # curve(0) != 0: silent quanta are processed as one zero channel
        curve = (np.linspace(-1, 1, 32) ** 2 * 0.8 + 0.1).astype(np.float32)
    sh = c.create_wave_shaper(curve=curve, oversample=oversample)
    if kind == "through_zero":
        o = c.create_oscillator(frequency=440.0 + 50 * g)
        o.start_at(128 * 3 / SR)
        o.stop_at(128 * 50 / SR)
        o.connect(sh)
        stereo_source(pkg, c, 80 + g, 128 * 9 + 50, 128 * 12 + 7).connect(sh)
        stereo_source(pkg, c, 90 + g, 128 * 6, 128 * 30).connect(sh)
    else:
        stereo_source(pkg, c, 100 + g, 128 * 20 + 9, 128 * 7 + 64).connect(sh)
    if kind == "feedback":  # shaper -> delay -> gain -> shaper: the shaper runs quantum by quantum inside the cycle
        d = c.create_delay(max_delay_time=0.1, delay_time=128 * 3 / SR)
        fb = c.create_gain(0.4)
        sh.connect(d)
        d.connect(fb)
        fb.connect(sh)
    sh.connect(c.destination())
    return c


@pytest.mark.parametrize("chunk", [128, 1024, 0])
@pytest.mark.parametrize("kind", ["through_zero", "not_through_zero", "feedback"])
@pytest.mark.parametrize("oversample", ["X2", "X4"])
def test_over_sampled_shaper_rebuilds_its_resamplers(pkg, engine, oracle, oversample, kind, chunk):
    os_ = pkg.OVERSAMPLE_X2 if oversample == "X2" else pkg.OVERSAMPLE_X4
    n = 128 * 70 + 17
    engine.set_option(pkg.OPT_CHUNK_FRAMES, chunk)
    try:
        check(pkg, engine, oracle, lambda be, g: shaper_graph(pkg, be, g, kind, os_, n))
    finally:
        engine.set_option(pkg.OPT_CHUNK_FRAMES, 0)


# ---------------------------------------------------------------------------------------------- what follows a compacted convolver
def gap_into_mono_response(pkg, be, g, n, after):
    """stereo A, a gap while the response still rings (ONE sounding output channel), stereo B -> mono response -> `after` -> destination:
    the convolver's sounding output changes between one and two channels"""
    c = pkg.OfflineAudioContext(2, n, SR, be)
    cv = c.create_convolver(pkg.AudioBuffer(mono_ir(36000, gain=0.01), SR), disable_normalization=True)
    stereo_source(pkg, c, 110 + g, 20000, 0).connect(cv)
    stereo_source(pkg, c, 120 + g, 15000, 41000 + 64 * g).connect(cv)
    node = after(c)
    cv.connect(node)
    node.connect(c.destination())
    return c


def test_biquad_behind_a_compacted_convolver(pkg, engine, oracle):
    # the filter drops its second channel in the gap and starts it again from zero state when B starts (biquad_filter.rs:796-809)
    n = 8192 * 8 + 99
    check(pkg, engine, oracle, lambda be, g: gap_into_mono_response(
        pkg, be, g, n, lambda c: c.create_biquad_filter(type_=pkg.LOWPASS, frequency=900.0 + 100 * g, q=3.0)))


@pytest.mark.parametrize("oversample", ["X2", "X4"])
def test_over_sampled_shaper_behind_a_compacted_convolver(pkg, engine, oracle, oversample):
    # a curve through 0 behind a convolver whose sounding output changes its count: the resamplers are rebuilt at every change
    os_ = pkg.OVERSAMPLE_X2 if oversample == "X2" else pkg.OVERSAMPLE_X4
    curve = np.tanh(np.linspace(-3, 3, 33)).astype(np.float32)
    n = 8192 * 8 + 99
    check(pkg, engine, oracle, lambda be, g: gap_into_mono_response(pkg, be, g, n, lambda c: c.create_wave_shaper(curve=curve, oversample=os_)))


# ---------------------------------------------------------------------------------------------- convolvers living across a suspend point
def test_stereo_response_keeps_its_history_across_a_suspend_point(pkg, engine, oracle):
    # the ordinary paths: a stereo source over the whole render -> gain -> stereo response; the callback changes the gain.  The response
    # spectra are shared by content, so the second segment's plan finds them in the cache: the node's own state must still be found
    n = 8192 * 4 + 300
    ir = G.synthetic_ir(20000, 2)

    def build(be, g):
        c = pkg.OfflineAudioContext(2, n, SR, be)
        s = stereo_source(pkg, c, 130 + g, n, 0)
        gn = c.create_gain(1.0)
        cv = c.create_convolver(pkg.AudioBuffer(ir, SR))
        s.connect(gn)
        gn.connect(cv)
        cv.connect(c.destination())
        c.suspend_sync(8192 * 2 / SR, lambda _c: gn.gain.set_value(0.25))
        return c
    gpu, cpu = check(pkg, engine, oracle, build)
    assert np.abs(cpu[:, :, 8192 * 2:8192 * 2 + 4000]).max() > 1e-2


def test_mono_response_turns_compacted_at_a_suspend_point(pkg, engine, oracle):
    # a tone alone (constant mono input) in the first segment; the callback adds a stereo source, so from the suspend point on the input
    # changes between one and two channels.  The first convolver's history (the tone's reverb) carries over, the second one starts empty
    n = 8192 * 4 + 300

    def build(be, g):
        c = pkg.OfflineAudioContext(2, n, SR, be)
        cv = c.create_convolver(pkg.AudioBuffer(mono_ir(20000), SR))
        o = c.create_oscillator(type_=pkg.SAWTOOTH, frequency=150.0 + 25 * g)
        o.start()
        o.connect(cv)
        cv.connect(c.destination())
        c.suspend_sync(8192 * 2 / SR, lambda _c: stereo_source(pkg, _c, 140 + g, 6000, 8192 * 2 + 2000).connect(cv))
        return c
    check(pkg, engine, oracle, build)
