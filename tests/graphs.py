"""Graph builders shared by the parity tests, bench.py and smoke(): each function builds the SAME graph on any
backend (the CUDA engine or the CPU oracle) through the mirrored control API, so a parity test is
`render(build(gpu)) vs render(build(oracle))`.  The BASELINE.json configs C1..C5 (SURVEY §8d) are here."""
import numpy as np

SR = 48000.0


def c1_osc_biquad(pkg, backend, length=48000, sr=SR):
    """C1: OscillatorNode(440 Hz sine) -> BiquadFilterNode(lowpass 350 Hz, Q 1) -> destination (tests/offline.rs style)."""
    c = pkg.OfflineAudioContext(2, length, sr, backend)
    osc = c.create_oscillator()
    bq = c.create_biquad_filter()
    osc.connect(bq)
    bq.connect(c.destination())
    osc.start()
    return c


def c2_params(g):
    rng = np.random.default_rng(1000 + g)
    f0 = float(np.exp(rng.uniform(np.log(100.0), np.log(8000.0))))
    q = float(rng.uniform(0.5, 4.0))
    gain = float(rng.uniform(0.1, 0.9))
    return rng, f0, q, gain


def c2_source(g, frames):
    rng, *_ = c2_params(g)
    return rng.uniform(-1.0, 1.0, (2, frames)).astype(np.float32)


def c2_buffer_biquad_gain(pkg, backend, g, length, sr=SR, pcm=None):
    """C2: AudioBufferSource(stereo noise) -> Biquad(lowpass, seeded f0/Q) -> Gain -> destination."""
    _, f0, q, gain = c2_params(g)
    if pcm is None:
        pcm = c2_source(g, length)
    c = pkg.OfflineAudioContext(2, length, sr, backend)
    src = c.create_buffer_source(pkg.AudioBuffer([pcm[0], pcm[1]], sr))
    bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=f0, q=q)
    gn = c.create_gain(gain)
    src.connect(bq)
    bq.connect(gn)
    gn.connect(c.destination())
    src.start()
    return c


def c3_many_voices(pkg, backend, voices=4096, length=48000, sr=SR):
    """C3: `voices` x (sine osc f = 55*2^(v/512) -> bandpass f0 = 2f, Q 5), all summed at the destination."""
    c = pkg.OfflineAudioContext(2, length, sr, backend)
    for v in range(voices):
        f = 55.0 * 2.0 ** (v / 512.0)
        osc = c.create_oscillator(frequency=f)
        bq = c.create_biquad_filter(type_=pkg.BANDPASS, frequency=2.0 * f, q=5.0)
        osc.connect(bq)
        bq.connect(c.destination())
        osc.start()
    return c


def synthetic_ir(frames, channels=2, seed=99, decay=0.25, sr=SR):
    """Exponentially decaying noise (the shape of examples/benchmarks.rs:307-349 'Convolution reverb')."""
    rng = np.random.default_rng(seed)
    t = np.arange(frames) / sr
    env = np.exp(-t / decay)
    return [(rng.standard_normal(frames) * env).astype(np.float32) for _ in range(channels)]


def c4_convolver(pkg, backend, g, length, ir, sr=SR, burst=4096):
    """C4: stereo AudioBufferSource (noise burst + low-level noise) -> ConvolverNode(normalize) -> destination."""
    rng = np.random.default_rng(4000 + g)
    pcm = (rng.uniform(-1.0, 1.0, (2, length)) * 0.05).astype(np.float32)
    pcm[:, :burst] += rng.uniform(-0.5, 0.5, (2, min(burst, length))).astype(np.float32)
    c = pkg.OfflineAudioContext(2, length, sr, backend)
    src = c.create_buffer_source(pkg.AudioBuffer([pcm[0], pcm[1]], sr))
    cv = c.create_convolver(pkg.AudioBuffer(ir, sr))
    src.connect(cv)
    cv.connect(c.destination())
    src.start()
    return c


def north_star_voices_convolver(pkg, backend, voices, length, ir, sr=SR, seed=0):
    """north_star graph: `voices` x (oscillator -> biquad) summed into ONE ConvolverNode -> destination."""
    rng = np.random.default_rng(7000 + seed)
    c = pkg.OfflineAudioContext(2, length, sr, backend)
    cv = c.create_convolver(pkg.AudioBuffer(ir, sr))
    cv.connect(c.destination())
    types = [pkg.SINE, pkg.SAWTOOTH, pkg.SQUARE, pkg.TRIANGLE]
    for v in range(voices):
        f = float(55.0 * 2.0 ** rng.uniform(0.0, 6.0))
        osc = c.create_oscillator(type_=types[v % 4], frequency=f, detune=float(rng.uniform(-20, 20)))
        bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=min(4.0 * f, 18000.0), q=float(rng.uniform(0.5, 6.0)))
        gn = c.create_gain(1.0 / voices)
        osc.connect(bq)
        bq.connect(gn)
        gn.connect(cv)
        osc.start()
    return c


def c5_full_chain(pkg, backend, g, length, ir, sr=SR, curve_points=257):
    """C5 (configs[4]): Oscillator -> WaveShaper -> Biquad -> Convolver -> PannerNode(HRTF) -> Analyser -> destination.
    The backend must have an HRIR sphere at the context rate (synthetic_hrir_sphere)."""
    rng = np.random.default_rng(5000 + g)
    c = pkg.OfflineAudioContext(2, length, sr, backend)
    osc = c.create_oscillator(type_=[pkg.SAWTOOTH, pkg.SINE, pkg.SQUARE, pkg.TRIANGLE][g % 4], frequency=float(110.0 * 2.0 ** rng.uniform(0, 4)))
    x = np.linspace(-1.0, 1.0, curve_points)
    sh = c.create_wave_shaper(curve=np.tanh(x * (1.5 + g % 3)).astype(np.float32))
    bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=float(rng.uniform(800, 6000)), q=float(rng.uniform(0.7, 4.0)))
    cv = c.create_convolver(pkg.AudioBuffer(ir, sr))
    az = rng.uniform(0, 2 * np.pi)
    pn = c.create_panner(panning_model=pkg.context.HRTF, distance_model=1,
                         position=(float(3 * np.sin(az)), float(rng.uniform(-1, 1)), float(-3 * np.cos(az))))
    an = c.create_analyser(fft_size=2048)
    osc.connect(sh)
    sh.connect(bq)
    bq.connect(cv)
    cv.connect(pn)
    pn.connect(an)
    an.connect(c.destination())
    osc.start()
    c._test_analyser = an
    return c


def synthetic_hrir_sphere(sample_rate=48000, taps=256, subdivisions=2, seed=5):
    """An HRIR sphere in the container format of the reference's resources/IRC_1003_C.bin (see include/wae.h):
    a subdivided octahedron (z up) whose vertex responses are decaying noise with a direction-dependent inter-aural
    delay and level.  Test data only: the real sphere cannot travel to the GPU box."""
    import struct
    verts = [(1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1)]
    faces = [(0, 2, 4), (2, 1, 4), (1, 3, 4), (3, 0, 4), (2, 0, 5), (1, 2, 5), (3, 1, 5), (0, 3, 5)]
    verts = [np.array(v, np.float64) for v in verts]
    for _ in range(subdivisions):
        cache, nf = {}, []
        def mid(i, j):
            key = (min(i, j), max(i, j))
            if key not in cache:
                m = verts[i] + verts[j]
                verts.append(m / np.linalg.norm(m))
                cache[key] = len(verts) - 1
            return cache[key]
        for a, b, c in faces:
            ab, bc, ca = mid(a, b), mid(b, c), mid(c, a)
            nf += [(a, ab, ca), (b, bc, ab), (c, ca, bc), (ab, bc, ca)]
        faces = nf
    rng = np.random.default_rng(seed)
    t = np.arange(taps)
    out = [b"HRIR", struct.pack("<IIII", int(sample_rate), taps, len(verts), 3 * len(faces))]
    out.append(np.asarray(faces, "<u4").tobytes())
    for v in verts:
        out.append(np.asarray(v, "<f4").tobytes())
        for ear in (-1.0, 1.0):  # left ear at -x, right ear at +x
            lateral = ear * v[0]
            delay = 12.0 * (1.0 - lateral)
            env = np.where(t >= delay, np.exp(-(t - delay) / (10.0 + 6.0 * (1.0 + v[2]))), 0.0)
            h = (0.35 + 0.25 * lateral) * env * (0.6 * rng.standard_normal(taps) + np.where(np.abs(t - delay) < 1, 1.0, 0.0))
            out.append(h.astype("<f4").tobytes())
    return b"".join(out)


def reference_hrir_subset():
    """The reference's IRC_1003_C sphere as stored in tests/golden/irc_1003_c_subset.npz (tools/extract_hrir_subset.py): every
    vertex position and face, the responses of the vertices a source at x = 1 blends, zeros elsewhere.  Container bytes."""
    import os
    import struct
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "irc_1003_c_subset.npz"))
    pos, faces, taps = z["positions"], z["faces"], int(z["taps"])
    ir = np.zeros((len(pos), 2, taps), np.float32)
    ir[z["vertices"], 0], ir[z["vertices"], 1] = z["left"], z["right"]
    out = [b"HRIR", struct.pack("<IIII", int(z["sample_rate"]), taps, len(pos), faces.size), np.asarray(faces, "<u4").tobytes()]
    for v in range(len(pos)):
        out += [np.asarray(pos[v], "<f4").tobytes(), ir[v].astype("<f4").tobytes()]
    return b"".join(out)


def parse_hrir_sphere(data):
    """(sample_rate, positions [v][3], faces [f][3], left [v][taps], right [v][taps]) of an HRIR container."""
    import struct
    sr, taps, nv, ni = struct.unpack("<IIII", data[4:20])
    off = 20
    faces = np.frombuffer(data, "<u4", ni, off).reshape(-1, 3)
    off += 4 * ni
    rec = np.frombuffer(data, "<f4", nv * (3 + 2 * taps), off).reshape(nv, 3 + 2 * taps)
    return sr, rec[:, :3], faces, rec[:, 3:3 + taps], rec[:, 3 + taps:]


def render(pkg, contexts, threads=1):
    bufs = pkg.render_batch(contexts, threads=threads)
    return np.stack([np.stack(b.channels) for b in bufs])
