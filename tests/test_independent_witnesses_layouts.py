"""Third statements of two layout rules, derived from neither oracle/ nor csrc/ (see tests/test_independent_witnesses.py):

* a ConvolverNode with a ONE-channel response builds two convolvers from it (convolver.rs:343-400); the second one is fed the right
  channel of the two-channel input quanta only, so it freezes through mono / silent stretches and resumes where it stopped.  Its output
  is numpy's linear convolution of the compacted right-channel stream, scattered back to the quanta it came from;
* an over-sampled WaveShaperNode rebuilds its resamplers with zero state whenever the channel count of a processed quantum changes
  (waveshaper.rs:409-420).  With the identity curve the node is a pure 128-frame delay (tests/test_oracle_kat.py), so the output
  quantum at a rebuild carries nothing from before it."""
import numpy as np

RQ = 128
SR = 48000.0


def merger_voice(pkg, c, f_left, f_right, start_frame, stop_frame, types=None):
    """a two-channel producer with an exact schedule: two oscillators into a ChannelMergerNode, sounding in the quanta that overlap
    [start_frame, stop_frame) and one silent channel elsewhere (oscillator.rs:382-392, channel_merger.rs:160-168)"""
    m = c.create_channel_merger(2)
    for ch, (f, ty) in enumerate(zip((f_left, f_right), types or (pkg.SAWTOOTH, pkg.TRIANGLE))):
        o = c.create_oscillator(type_=ty, frequency=f)
        o.start_at(start_frame / SR)
        o.stop_at(stop_frame / SR)
        o.connect_from_output_to_input(m, 0, ch)
    return m


def test_mono_response_second_convolver_is_the_convolution_of_the_compacted_right_channel(pkg, oracle):
    n_q = 120
    n = RQ * n_q
    a = (0, RQ * 40 + 60)           # quanta 0 .. 40 sound
    b = (RQ * 55 + 40, RQ * 100 + 7)  # quanta 55 .. 100: the response (3000 frames ~ 24 quanta) of A still rings in quanta 41 .. 54
    rng = np.random.default_rng(11)
    ir = (0.05 * rng.standard_normal(3000) * np.exp(-np.arange(3000) / 900.0)).astype(np.float32)

    def graph(with_convolver):
        c = pkg.OfflineAudioContext(2, n, SR, oracle)
        out = c.destination()
        if with_convolver:
            cv = c.create_convolver(pkg.AudioBuffer([ir], SR), disable_normalization=True)
            cv.connect(out)
            out = cv
        merger_voice(pkg, c, 220.0, 331.0, *a).connect(out)
        merger_voice(pkg, c, 523.0, 97.0, *b).connect(out)
        r = c.start_rendering_sync()
        return np.array([r.get_channel_data(0), r.get_channel_data(1)], np.float64)

    dry = graph(False)
    wet = graph(True)
    stereo_q = [q for q in range(n_q) if (q * RQ < a[1] and (q + 1) * RQ > a[0]) or (q * RQ < b[1] and (q + 1) * RQ > b[0])]
    assert 41 not in stereo_q and 55 in stereo_q and 54 not in stereo_q
    frames = np.concatenate([np.arange(q * RQ, (q + 1) * RQ) for q in stereo_q])
    stream = dry[1, frames]                                   # what convolvers[1] is fed: R of the two-channel quanta, gaps removed
    want = np.convolve(stream, ir.astype(np.float64))[:len(stream)]
    got = wet[1, frames]
    assert np.abs(got - want).max() <= 1e-6, np.abs(got - want).max()
    # not the unfrozen convolution: A's right-channel tail resumes in B's first quanta instead of having rung out in the gap
    timeline = np.zeros(n)
    timeline[frames] = stream
    unfrozen = np.convolve(timeline, ir.astype(np.float64))[:n][frames]
    assert np.abs(got - unfrozen).max() > 1e-3


def test_over_sampled_shaper_output_at_a_rebuild_carries_nothing_from_before(pkg, oracle):
    # identity curve (maps 0 to 0: silent quanta are not processed): a mono tone for quanta 0 .. 29, from quantum 30 on a two-channel
    # producer as well.  The quantum where the count turns to 2 rebuilds both resamplers: its output starts from zero history, the
    # quanta after it are the pure 128-frame delay again
    n = RQ * 60
    r = 30
    for oversample, tol in ((1, 1e-4), (2, 1e-3)):
        c = pkg.OfflineAudioContext(2, n, SR, oracle)
        sh = c.create_wave_shaper(curve=np.array([-1.0, 0.0, 1.0], np.float32), oversample=oversample)
        o = c.create_oscillator(frequency=1000.0)
        o.start()
        g_tone, g_voice = c.create_gain(0.5), c.create_gain(0.4)  # (inside the curve's [-1, 1])
        o.connect(g_tone)
        g_tone.connect(sh)
        merger_voice(pkg, c, 700.0, 1300.0, RQ * r, n, (pkg.SINE, pkg.SINE)).connect(g_voice)
        g_voice.connect(sh)
        sh.connect(c.destination())
        out = c.start_rendering_sync()
        y = np.array([out.get_channel_data(0), out.get_channel_data(1)], np.float64)
        t = np.arange(n) / SR
        # before the rebuild: the tone, 128 frames late
        assert np.abs(y[0, RQ * 10:RQ * r] - 0.5 * np.sin(2 * np.pi * 1000.0 * t[RQ * 9:RQ * (r - 1)])).max() <= tol
        # at the rebuild: the delayed input of quantum r - 1 is gone — only the transient of quantum r's own first frames
        at = y[:, RQ * r:RQ * r + 64]
        assert np.abs(at).max() < 1e-2, np.abs(at).max()
        assert np.abs(0.5 * np.sin(2 * np.pi * 1000.0 * t[RQ * (r - 1):RQ * (r - 1) + 64])).max() > 0.4
        # after it: the pure delay of the new two-channel input again (left: tone + 700 Hz, right: tone + 1300 Hz)
        tone = 0.5 * np.sin(2 * np.pi * 1000.0 * t)
        for ch, f in ((0, 700.0), (1, 1300.0)):
            x = tone + 0.4 * np.sin(2 * np.pi * f * (t - RQ * r / SR))
            assert np.abs(y[ch, RQ * (r + 4):] - x[RQ * (r + 3):n - RQ]).max() <= tol
