"""Third statements at the shapes where the CUDA kernels can go wrong.  tests/test_independent_witnesses.py states each operation from the
specification, scipy or numpy in f64 and checks the oracle with it on toy graphs; here the same kind of independent statement is checked on
the engine, at the shapes its kernels take different paths for: many graphs (many CTAs, ragged last tiles), long renders (time slabs of the
biquad scan), chunk edges, convolver partitions, the mixer's 16-edge direct path and 256-edge staging, parameters bound from device memory.

Every witness runs with two backends: `oracle` (unmarked: shows on a CPU-only machine that the witness and its budget are right) and
`engine` (the GPU).  None of the witness code is derived from oracle/ or csrc/; each formula cites the specification or the reference's
file:line.  The ordered sums are compared bit for bit, the f64 filters within a few f32 ulp of the output, the f32 convolver and analyser
against the reference's own accuracy (the oracle restates its f32 transforms)."""
import contextlib

import numpy as np
import pytest

import test_independent_witnesses as W
import test_independent_witnesses_layouts as WL
import test_reference_gaps as RG

scipy_signal = pytest.importorskip("scipy.signal")

RQ = 128
SR = 48000.0
F32 = np.float32


# ---------------------------------------------------------------------------------------------------------------------------------------
# backends
class _Backend:
    """`backend`: what OfflineAudioContext renders with; `options(...)`: engine launch options for a block (no-ops on the oracle, which
    has one code path); `variants(...)`: the option sets a witness is rendered under (the oracle renders once)."""

    def __init__(self, pkg, name, backend, engine=None):
        self.pkg, self.name, self.backend, self.engine = pkg, name, backend, engine

    @property
    def is_engine(self):
        return self.engine is not None

    @contextlib.contextmanager
    def options(self, chunk=0, fuse=1, serial=0, prepass=1):
        if self.engine is None:
            yield
            return
        p, e = self.pkg, self.engine
        e.set_option(p.OPT_CHUNK_FRAMES, chunk)
        e.set_option(p.OPT_FUSE, fuse)
        e.set_option(p.OPT_SERIAL_FILTERS, serial)
        e.set_option(p.OPT_CHAIN_PREPASS, prepass)
        try:
            yield
        finally:  # the defaults (include/wae.h)
            e.set_option(p.OPT_CHUNK_FRAMES, 0)
            e.set_option(p.OPT_FUSE, 1)
            e.set_option(p.OPT_SERIAL_FILTERS, 0)
            e.set_option(p.OPT_CHAIN_PREPASS, 1)

    def variants(self, *sets):
        return list(sets) if self.is_engine else [{}]


@pytest.fixture(params=["oracle", pytest.param("engine", marks=pytest.mark.gpu)])
def be(request, pkg, oracle):
    if request.param == "oracle":
        return _Backend(pkg, "oracle", oracle)
    engine = request.getfixturevalue("engine")
    return _Backend(pkg, "engine", engine.backend, engine)


def _render(pkg, contexts):
    """[graph][channel][frame] f32 of contexts of one shape"""
    return np.stack([np.stack(b.channels) for b in pkg.render_batch(contexts)])


# ---------------------------------------------------------------------------------------------------------------------------------------
# 1. the existing third statements, rendered by the engine
ENGINE_RERUNS = (
    [(W.test_biquad_render_vs_the_specification_and_scipy, (k,)) for k in W.KINDS]
    + [(W.test_biquad_detune_is_a_frequency_ratio, ())]
    + [(W.test_iir_render_vs_scipy, (o,)) for o in (1, 2, 3, 5, 8)]
    + [(W.test_analyser_spectrum_vs_numpy, (n,)) for n in (256, 2048)]
    + [(W.test_audioparam_curves_vs_closed_forms, ())]
    + [(W.test_delay_vs_linear_interpolation, (d,)) for d in (0.0, 1.0, 40.25, 127.5, 128.0, 300.75, 1000.5)]
    + [(W.test_stereo_panner_vs_the_specification, (p,)) for p in (-1.0, -0.3, 0.0, 0.45, 1.0)]
    + [(W.test_wave_shaper_vs_the_specification, (n,)) for n in (2, 3, 64, 1025)]
    + [(W.test_panner_distance_gain_vs_the_specification, (m,)) for m in ("linear", "inverse", "exponential")]
    + [(W.test_equal_power_panner_vs_the_specification, (s,)) for s in (False, True)]
    + [(W.test_panner_cone_gain_vs_the_specification, ()), (W.test_value_curve_vs_the_specification, ()),
       (W.test_sine_oscillator_and_detune_vs_numpy, ()), (W.test_looping_buffer_source_vs_modular_indexing, ()),
       (W.test_dynamics_compressor_vs_the_published_design, ())]
    + [(W.test_speaker_mixing_vs_the_specification, (k,)) for k in (1, 2, 3, 4, 6)]
    + [(W.test_buffer_source_resampling_vs_linear_interpolation, rb) for rb in ((0.5, 48000.0), (1.37, 48000.0), (2.0, 48000.0), (1.0, 32000.0),
                                                                               (0.8, 44100.0))]
    + [(WL.test_mono_response_second_convolver_is_the_convolution_of_the_compacted_right_channel, ()),
       (WL.test_over_sampled_shaper_output_at_a_rebuild_carries_nothing_from_before, ())]
    + [(RG.test_quantum_add_and_mix_through_a_graph, ()), (RG.test_convolver_response_from_the_options, ())]
)
# functions that also take `builder` (graph building checked on the product's graph half, renders on the engine)
ENGINE_RERUNS_WITH_BUILDER = [RG.test_oscillator_type_rules,
                              RG.test_offline_context_accessors_and_empty_graph, RG.test_option_values_apply_from_the_first_frame,
                              RG.test_constructors_and_their_defaults]


@pytest.mark.gpu
@pytest.mark.parametrize("case", ENGINE_RERUNS, ids=lambda c: c[0].__name__ + "".join("-%s" % (a,) for a in c[1]))
def test_third_statement_on_gpu(pkg, engine, case):
    fn, args = case
    fn(pkg, engine.backend, *args)


@pytest.mark.gpu
@pytest.mark.parametrize("fn", ENGINE_RERUNS_WITH_BUILDER, ids=lambda f: f.__name__)
def test_reference_gap_render_on_gpu(pkg, engine, fn):
    fn(pkg, engine.backend, engine.backend)


# ---------------------------------------------------------------------------------------------------------------------------------------
# 2. ordered sums, bit for bit
#
# An input port sums its edges in the processing order (graph.rs:498-535: every node adds its output to the inputs of its targets right after
# it processed): for sources created in order and connected to one port, last-created first (graph.rs:331-487; see
# tests/test_gpu_parity.py::test_c3_many_voices_summation_order).  Each add is AudioRenderQuantum::add (quantum.rs:532-569): the running sum
# and the edge are mixed to the port's computed channel count, then added channel by channel with AudioRenderQuantumChannel::add
# (quantum.rs:114-120), which takes the other channel as it is when the running one is the silent channel and skips a silent other channel.
# A quantum in which a source does not play is the silent quantum: one silent channel (quantum.rs:511-516).  Silence is None below.
SQRT05 = np.sqrt(F32(0.5))  # (0.5f32).sqrt(), quantum.rs:419 and on: IEEE sqrt is correctly rounded in numpy's f32 as in Rust's


def _z(ch, nf):
    return np.zeros(nf, F32) if ch is None else ch


def _fma32(a, b, c):
    # f32::mul_add: the product of two f32 is exact in the 64-bit significand of longdouble, so the sum is rounded twice only when the
    # 64-bit result lands exactly on an f32 rounding boundary
    return (np.longdouble(a) * np.asarray(b, np.longdouble) + np.asarray(c, np.longdouble)).astype(F32)


def _mix(q, n, speakers, nf):
    """AudioRenderQuantum::mix (quantum.rs:274-505), in its f32 operation order"""
    k = len(q)
    if k == n:
        return q
    if not speakers or k > 6 or n > 6:
        return (q + [None] * n)[:n]
    z = [_z(c, nf) for c in q]
    if (k, n) == (1, 2):
        return [q[0], q[0]]
    if (k, n) == (1, 4):
        return [q[0], q[0], None, None]
    if (k, n) == (1, 6):
        return [None, None, q[0], None, None, None]
    if (k, n) in ((2, 4), (2, 6)):
        return q + [None] * (n - 2)
    if (k, n) == (4, 5):
        return [q[0], q[1], None, q[2], q[3]]
    if (k, n) == (4, 6):
        return [q[0], q[1], None, None, q[2], q[3]]
    if (k, n) == (2, 1):
        return [F32(0.5) * (z[0] + z[1])]
    if (k, n) == (4, 1):
        return [F32(0.25) * (z[0] + z[1] + z[2] + z[3])]
    if (k, n) == (6, 1):
        return [_fma32(SQRT05, z[0] + z[1], _fma32(F32(0.5), z[4] + z[5], z[2]))]
    if (k, n) == (4, 2):
        return [F32(0.5) * (z[0] + z[2]), F32(0.5) * (z[1] + z[3])]
    if (k, n) == (6, 2):
        return [z[0] + SQRT05 * (z[2] + z[4]), z[1] + SQRT05 * (z[2] + z[5])]
    if (k, n) == (6, 4):  # swap_remove(3), swap_remove(2): [L, R, SL, SR]
        return [z[0] + SQRT05 * z[2], z[1] + SQRT05 * z[2], q[4], q[5]]
    return (q + [None] * n)[:n]


def _chan_add(a, b):
    if a is None:
        return b
    if b is None:
        return a
    return a + b


def _add(acc, other, mode, count, speakers, nf):
    """AudioRenderQuantum::add (quantum.rs:532-569); mode 0 max, 1 clamped-max, 2 explicit (include/wae.h)"""
    mx = max(len(acc), len(other))
    new = mx if mode == 0 else (min(mx, count) if mode == 1 else count)
    if speakers and all(c is acc[0] for c in acc) and all(c is other[0] for c in other):
        return _mix([_chan_add(acc[0], other[0])], new, speakers, nf)
    acc = _mix(acc, new, speakers, nf)
    other = _mix(list(other), new, speakers, nf)
    return [_chan_add(a, b) for a, b in zip(acc, other)]


class _Edge:
    """one AudioBufferSourceNode playing `pcm` [channels][frames] 1:1 from quantum `start_q` (its quanta outside the buffer are silent)"""

    def __init__(self, pcm, start_q):
        self.pcm, self.start_q = pcm, start_q

    def quantum_range(self):
        return self.start_q, self.start_q + -(-self.pcm.shape[1] // RQ)

    def frames(self, f0, f1):
        out = np.zeros((self.pcm.shape[0], f1 - f0), F32)
        a = self.start_q * RQ
        lo, hi = max(f0, a), min(f1, a + self.pcm.shape[1])
        if hi > lo:
            out[:, lo - f0:hi - f0] = self.pcm[:, lo - a:hi - a]
        return [out[c] for c in range(out.shape[0])]


def _port_sum(edges, order, n_q, mode, count, speakers):
    """the port's quanta [channel list per run of quanta with one silence pattern]: (q0, q1, channels)"""
    bounds = sorted({0, n_q} | {min(max(b, 0), n_q) for e in edges for b in e.quantum_range()})
    runs = []
    for q0, q1 in zip(bounds[:-1], bounds[1:]):
        if q0 == q1:
            continue
        nf = (q1 - q0) * RQ
        acc = [None]
        for i in order:
            e = edges[i]
            a, b = e.quantum_range()
            other = e.frames(q0 * RQ, q1 * RQ) if a <= q0 and q1 <= b else [None]
            acc = _add(acc, other, mode, count, speakers, nf)
        runs.append((q0, q1, acc))
    return runs


def _witness_sum(edges, order, n_q, out_ch, via_gain):
    """what the destination (count out_ch, explicit, speakers: offline.rs) renders from `edges` summed at the destination, or at a GainNode(1)
    (count 2, max, speakers: gain.rs) that feeds it (a gain of 1 multiplies every sample by 1.0: the bits pass unchanged, -0.0 included)"""
    n = n_q * RQ
    out = np.zeros((out_ch, n), F32)
    if via_gain:
        for q0, q1, acc in _port_sum(edges, order, n_q, 0, 2, True):
            silent = all(c is None for c in acc)
            dst = _add([None], [None] if silent else [_z(c, (q1 - q0) * RQ) * F32(1.0) for c in acc], 2, out_ch, True, (q1 - q0) * RQ)
            for c in range(out_ch):
                out[c, q0 * RQ:q1 * RQ] = _z(dst[c], (q1 - q0) * RQ)
    else:
        for q0, q1, acc in _port_sum(edges, order, n_q, 2, out_ch, True):
            for c in range(out_ch):
                out[c, q0 * RQ:q1 * RQ] = _z(acc[c], (q1 - q0) * RQ)
    return out


def _sum_samples(rng, ch, frames, neg_zero_frames):
    # u * 2^e with e in [-20, 4]: wide enough that the f32 sum depends on the order of the terms
    x = (rng.uniform(-1, 1, (ch, frames)) * 2.0 ** rng.integers(-20, 5, (ch, frames))).astype(F32)
    x[rng.uniform(size=(ch, frames)) < 0.02] = F32(-0.0)
    x[:, neg_zero_frames] = F32(-0.0)  # frames where every edge is -0.0: the sum is -0.0 only if the first edge is taken as it is
    return x


def _sum_graph(pkg, backend, spec, n_q):
    """spec = (n_edges, layout, port, timing, seed) -> (context, edges, processing order)"""
    n_edges, layout, port, timing, seed = spec
    rng = np.random.default_rng(seed)
    n = n_q * RQ
    neg_zero = rng.choice(n, 24, replace=False)
    edges = []
    for i in range(n_edges):
        ch = {"stereo": 2, "mono": 1, "mixed": (1, 2, 4, 6)[i % 4]}[layout]
        if timing == "full":
            start_q, frames = 0, n
        else:  # different starts and ends, some edges silent for whole stretches (the port's layout changes mid-render)
            start_q = int(rng.integers(0, n_q // 2))
            frames = int(rng.integers(RQ, (n_q - start_q) * RQ + 1))
        edges.append(_Edge(_sum_samples(rng, ch, frames, neg_zero[neg_zero < frames]), start_q))
    # 32768 Hz: start times on quantum boundaries are exact binary fractions, so the playhead sits on whole frames (no interpolation, which
    # would turn a -0.0 sample into +0.0: audio_buffer_source.rs:727-800)
    sr = 32768.0
    c = pkg.OfflineAudioContext(2, n, sr, backend)
    target = c.create_gain(1.0) if port == "gain" else c.destination()
    for e in edges:
        s = c.create_buffer_source(pkg.AudioBuffer(list(e.pcm), sr))
        s.connect(target)
        s.start_at(e.start_q * RQ / sr)
    if port == "gain":
        target.connect(c.destination())
    return c, edges, list(range(n_edges))[::-1]


EDGE_COUNTS = [1, 2, 8, 15, 16, 17, 255, 256, 257, 513]


def _check_sums(pkg, be, specs, n_q, opts):
    made = [_sum_graph(pkg, be.backend, s, n_q) for s in specs]
    with be.options(**opts):
        got = _render(pkg, [c for c, _, _ in made])
    for g, (spec, (_c, edges, order)) in enumerate(zip(specs, made)):
        want = _witness_sum(edges, order, n_q, 2, spec[2] == "gain")
        assert np.array_equal(got[g].view(np.uint32), want.view(np.uint32)), (spec, opts, int((got[g].view(np.uint32) != want.view(np.uint32)).sum()))
        if spec[0] >= 8 and spec[3] == "full":
            # the witness can tell the orders apart: summed in creation order, most frames come out different
            other = _witness_sum(edges, order[::-1], n_q, 2, spec[2] == "gain")
            assert (other != want).mean() > 0.5, spec
        assert np.signbit(want[want == 0]).any() or spec[3] != "full", spec  # (-0.0 frames survive in the witness)


@pytest.mark.parametrize("n_edges", EDGE_COUNTS + [1000])
def test_ordered_sum_one_graph_short_render(pkg, be, n_edges):
    # one graph, 12 quanta: few frames x few instances -> one frame per thread (k_mix<1> / k_mix_narrow<1>)
    specs = [(n_edges, layout, port, "full", 100 + n_edges) for layout in ("stereo", "mono") for port in ("dest", "gain")]
    for s in specs:
        _check_sums(pkg, be, [s], 12, {})


def _batch_specs():
    specs = [(n, "stereo" if k % 2 == 0 else "mono", "dest" if k % 3 else "gain", "full", 200 + k) for k, n in enumerate(EDGE_COUNTS)]
    specs += [(n, "mixed", port, "full", 300 + n) for n in (3, 8, 17) for port in ("dest", "gain")]
    specs += [(n, layout, port, "staggered", 400 + n) for n in (5, 16, 21) for layout in ("mixed", "mono", "stereo") for port in ("dest", "gain")]
    return specs


@pytest.mark.parametrize("opts", [dict(fuse=1, chunk=0), dict(fuse=0, chunk=0), dict(fuse=1, chunk=128), dict(fuse=0, chunk=128),
                                  dict(fuse=1, chunk=1024), dict(fuse=0, chunk=1024)], ids=lambda o: "fuse%d-chunk%d" % (o["fuse"], o["chunk"]))
def test_ordered_sums_in_one_batch(pkg, be, opts):
    # 38 graphs x 128 quanta: many instances x many frames -> four frames per thread (k_mix<4>) at chunk 0 and 1024, one at chunk 128;
    # mixed layouts take the general path, staggered sources the per-quantum layouts (k_mix_dyn)
    if not be.is_engine and opts != dict(fuse=1, chunk=0):
        pytest.skip("the oracle has one code path")
    _check_sums(pkg, be, _batch_specs(), 128, opts)


# ---------------------------------------------------------------------------------------------------------------------------------------
# 3. biquad and second-order IIR against scipy.signal.lfilter in f64
#
# BiquadFilterRenderer::process (biquad_filter.rs:764-899): coefficients in f64 from the f32 param values (computedFrequency = frequency * 2^(detune /
# 1200) in f32, :367-373, here detune 0), the specification's formulas (w3c_biquad), the recurrence in f64, the output cast to f32 (a non-normal y
# is flushed to 0).  Budget 4e-7 * max(1, peak), as the oracle's witness: an f32 output carries 6e-8 of its magnitude in rounding alone.
#
# Rule for the cases: a pole of radius r amplifies a relative error e of the f64 coefficients by about 1 / (1 - r)^2 in the output; one ulp
# (1.1e-16) stays below 1e-7 of the output when (1 - r)^2 >= 1e-8.  Cases outside the rule are dropped (_well_conditioned).
def _coefs(kind, sr, f0, q, gain):
    b, a = W.w3c_biquad(kind, float(F32(sr)), float(F32(f0)), float(F32(q)), float(F32(gain)))
    return np.array(b) / a[0], np.array(a) / a[0]


def _well_conditioned(a):
    r = np.abs(np.roots(a)).max() if len(a) > 1 else 0.0
    return (1.0 - r) ** 2 >= 1e-8


def _bq_cases(sr):
    nyq = sr / 2
    base = [(25.0, 30.0, 0.0), (0.97 * nyq, 1.0, 0.0), (0.9 * nyq, 8.0, 12.0), (1000.0, 0.1, 0.0), (700.0, 2.0, 30.0), (3000.0, 4.0, -30.0)]
    out = []
    for kind in W.KINDS:
        for f0, q, gain in base:
            if _well_conditioned(_coefs(kind, sr, f0, q, gain)[1]):
                out.append((kind, f0, q, gain))
    return out


def _bq_graph(pkg, backend, kind, f0, q, gain, x, n, bound=False):
    c = pkg.OfflineAudioContext(1, n, x.sr, backend)
    s = c.create_buffer_source(pkg.AudioBuffer([x.pcm], x.sr))
    bq = c.create_biquad_filter(type_=W.KINDS.index(kind), frequency=1000.0 if bound else f0, q=1.0 if bound else q, gain=0.0 if bound else gain)
    s.connect(bq)
    bq.connect(c.destination())
    s.start()
    if bound:
        for p in (bq.frequency, bq.q, bq.gain, bq.detune):
            p.set_device_value()
    return c, [bq.frequency, bq.q, bq.gain, bq.detune]


class _Pcm:
    def __init__(self, seed, n, sr):
        self.pcm = np.random.default_rng(seed).uniform(-1, 1, n).astype(F32)
        self.sr = float(F32(sr))


def _lfilter(b, a, x):
    y = scipy_signal.lfilter(b, a, np.asarray(x, np.float64))
    return np.where(np.abs(y) < np.finfo(np.float64).tiny, 0.0, y)


def _assert_filter(got, want, what):
    err = float(np.abs(got.astype(np.float64) - want).max())
    assert err <= 4e-7 * max(1.0, float(np.abs(want).max())), (what, err)
    return err


IIR2 = [scipy_signal.butter(2, 0.013), scipy_signal.cheby1(2, 1.0, 0.6)]


@pytest.mark.parametrize("sr", [22050.0, 48000.0, 96000.0])
def test_biquad_many_graphs_vs_scipy(pkg, be, sr):
    # 2048 * 12 + 5 frames: ragged last tile; every case its own graph (one CTA per graph and channel), plus order-2 IIRFilterNodes (the scan)
    n = 2048 * 12 + 5
    cases = _bq_cases(sr)
    assert len(cases) >= 40
    xs = [_Pcm(g, n, sr) for g in range(len(cases) + len(IIR2))]
    want = [_lfilter(*_coefs(k, sr, f0, q, gain), xs[g].pcm) for g, (k, f0, q, gain) in enumerate(cases)]
    want += [_lfilter(b, a, xs[len(cases) + i].pcm) for i, (b, a) in enumerate(IIR2)]
    for opts in be.variants(dict(), dict(serial=1), dict(chunk=128), dict(chunk=2048 * 36), dict(chunk=128, serial=1)):
        ctxs = [_bq_graph(pkg, be.backend, *case, xs[g], n)[0] for g, case in enumerate(cases)]
        for i, (b, a) in enumerate(IIR2):
            x = xs[len(cases) + i]
            c = pkg.OfflineAudioContext(1, n, x.sr, be.backend)
            s = c.create_buffer_source(pkg.AudioBuffer([x.pcm], x.sr))
            f = c.create_iir_filter(list(b * 3.0), list(a * 3.0))  # unnormalised: iir_filter.rs:282-309 divides by feedback[0]
            s.connect(f)
            f.connect(c.destination())
            s.start()
            ctxs.append(c)
        with be.options(**opts):
            got = _render(pkg, ctxs)
        for g in range(len(ctxs)):
            _assert_filter(got[g, 0], want[g], ((cases + IIR2)[g] if g < len(cases) else "iir2", opts))


@pytest.mark.parametrize("case", [("lowpass", 40.0, 12.0, 0.0), ("peaking", 150.0, 20.0, 9.0), ("highshelf", 5000.0, 1.0, -30.0)], ids=lambda c: c[0])
def test_biquad_long_mono_render_vs_scipy(pkg, be, case):
    # one graph, one channel, 21 s: the scan cuts the render into time slabs (with the pre-pass: slabs that find out the state they hand on)
    n = 48000 * 21 + 77
    assert _well_conditioned(_coefs(case[0], SR, *case[1:])[1])
    x = _Pcm(7, n, SR)
    want = _lfilter(*_coefs(case[0], SR, *case[1:]), x.pcm)
    for opts in be.variants(dict(), dict(prepass=0), dict(serial=1)):
        with be.options(**opts):
            got = _render(pkg, [_bq_graph(pkg, be.backend, *case, x, n)[0]])
        _assert_filter(got[0, 0], want, (case, opts))


@pytest.mark.gpu
def test_biquad_params_bound_from_device_memory_vs_scipy(pkg, engine):
    # the four params declared set_device_value and bound per run: coefficients derived on the device (k_derive_params, make_scan_coef)
    torch = pytest.importorskip("torch")
    be = _Backend(pkg, "engine", engine.backend, engine)
    n = 2048 * 7 + 5
    cases = _bq_cases(SR)
    xs = [_Pcm(50 + g, n, SR) for g in range(len(cases))]
    want = [_lfilter(*_coefs(k, SR, f0, q, gain), xs[g].pcm) for g, (k, f0, q, gain) in enumerate(cases)]
    for opts in (dict(), dict(serial=1)):
        made = [_bq_graph(pkg, engine.backend, *case, xs[g], n, bound=True) for g, case in enumerate(cases)]
        with be.options(**opts):
            b = pkg.Batch([c for c, _ in made])
            # (graphs of different filter types: each graph's params are named by its own node, so one bind call per graph)
            for g, (c, params) in enumerate(made):
                _k, f0, q, gain = cases[g]
                b.bind_params(params, torch.tensor([[f0, q, gain, 0.0]], dtype=torch.float32).cuda(), graphs=[g])
            b.run()
            b.sync()
        for g in range(len(cases)):
            _assert_filter(b.fetch_graph(g)[0], want[g], (cases[g], opts))
        b.destroy()


def test_biquad_frequency_ramp_vs_the_per_frame_recurrence(pkg, be):
    # a-rate frequency: coefficients per frame (biquad_filter.rs:820-845) from the f32 value of the linear ramp (spec 1.6.3: v(t) = V0 + (V1 - V0)
    # (t - T0) / (T1 - T0)), the recurrence y = b0 x + b1 x1 + b2 x2 - a1 y1 - a2 y2 in f64 (:869-885)
    n = RQ * 40
    x = _Pcm(3, n, SR)
    t = np.arange(n) / SR
    t1 = (n - 300) / SR
    freq = np.where(t < t1, 200.0 + (8000.0 - 200.0) * t / t1, 8000.0).astype(F32)
    for kind in ("lowpass", "bandpass", "peaking"):
        co = [_coefs(kind, SR, float(f), 3.0, 6.0) for f in freq]
        want = np.zeros(n)
        x1 = x2 = y1 = y2 = 0.0
        for i in range(n):
            (b0, b1, b2), (_a0, a1, a2) = co[i]
            xi = float(x.pcm[i])
            y = b0 * xi + b1 * x1 + b2 * x2 - a1 * y1 - a2 * y2
            x2, x1, y2, y1 = x1, xi, y1, y
            want[i] = y
        c, (fp, _q, _g, _d) = _bq_graph(pkg, be.backend, kind, 200.0, 3.0, 6.0, x, n)
        fp.linear_ramp_to_value_at_time(8000.0, t1)
        got = _render(pkg, [c])[0, 0]
        # the param evaluates the ramp in f32 (param.rs): its value may sit an ulp (6e-8 relative) from the f64 closed form rounded, a frequency
        # shift of that size moves the output by about Q times as much
        err = float(np.abs(got - want).max())
        assert err <= 2e-6 * max(1.0, float(np.abs(want).max())), (kind, err)


# ---------------------------------------------------------------------------------------------------------------------------------------
# 4. IIRFilterNode (k_iir_serial) up to the reference's 20 coefficients (iir_filter.rs:82-110), against lfilter in f64
def _iir_filters():
    return [("butter3", scipy_signal.butter(3, 0.3)), ("cheby6", scipy_signal.cheby1(6, 0.5, 0.45)), ("butter12", scipy_signal.butter(12, 0.5)),
            ("cheby19", scipy_signal.cheby1(19, 0.1, 0.7))]


@pytest.mark.parametrize("name", ["butter3", "cheby6", "butter12", "cheby19"])
def test_iir_high_orders_vs_scipy(pkg, be, name):
    b, a = dict(_iir_filters())[name]
    n = RQ * 300 + 45
    rng = np.random.default_rng(len(name))
    x = rng.uniform(-1, 1, n).astype(F32)
    x[n // 2:] = 0.0   # the input falls silent: the filter rings out (the tail check, iir_filter.rs:315-335)
    want = _lfilter(b, a, x)
    # the direct form is a witness only while it agrees with the cascade of second-order sections of the same filter
    sos = scipy_signal.tf2sos(b, a)
    assert np.abs(scipy_signal.sosfilt(sos, x.astype(np.float64)) - want).max() <= 1e-9 * max(1.0, np.abs(want).max()), name
    for suspend in (False, True):
        c = pkg.OfflineAudioContext(1, RQ * 300 + 128, SR, be.backend)
        s = c.create_buffer_source(pkg.AudioBuffer([x], SR))
        f = c.create_iir_filter(list(b * 2.5), list(a * 2.5))
        s.connect(f)
        f.connect(c.destination())
        s.start()
        if suspend:  # a render cut by a suspend point
            c.suspend_sync(RQ * 101 / SR, lambda ctx: None)
        got = _render(pkg, [c])[0, 0, :n]
        _assert_filter(got, want, (name, suspend))
        assert np.abs(want[-RQ:]).max() > 1e-12 or np.abs(got[-RQ:]).max() == 0.0


# ---------------------------------------------------------------------------------------------------------------------------------------
# 5. ConvolverNode against an f64 linear convolution
#
# Routing (convolver.rs:378-487): a mono response convolves each input channel; a stereo response convolves L with h0 and R with h1 (a mono input
# with both); four channels: L = xL * h0 + xR * h2, R = xL * h1 + xR * h3 (a mono input as both).  Normalisation
# (https://webaudio.github.io/web-audio-api/#dom-convolvernode-normalize, calculateNormalizationScale): 1 / max(sqrt(sum h^2 / (ch len)), 1.25e-4)
# * 0.00125 * 44100 / sr, halved for four channels.  The budget is the reference's own accuracy: the oracle restates its f32 fft-convolver, and
# the engine may be at most 3x its RMS error (see _check_conv) and 4x its max error (+ 1e-7 of the peak).
def _conv_truth(x, h, n, normalize, sr):
    x64, h64 = np.asarray(x, np.float64), np.asarray(h, np.float64)
    conv = lambda a, b: scipy_signal.fftconvolve(a, b)[:n] if len(b) > 1 else (a * b[0])[:n]
    if len(h64) == 1:
        y = [conv(xc, h64[0]) for xc in x64]
        if len(y) == 1:
            y = [y[0], y[0]]
        else:  # the second convolver is fed the two-channel quanta only (convolver.rs:343-400): once the input is silent, the output is
            #    the first one's, mono (tests/test_independent_witnesses_layouts.py)
            q_end = -(-x64.shape[1] // RQ) * RQ
            y[1] = np.concatenate([y[1][:q_end], y[0][q_end:]])
    elif len(h64) == 2:
        xl, xr = x64[0], x64[-1]
        y = [conv(xl, h64[0]), conv(xr, h64[1])]
    else:
        xl, xr = x64[0], x64[-1]
        y = [conv(xl, h64[0]) + conv(xr, h64[2]), conv(xl, h64[1]) + conv(xr, h64[3])]
    y = np.array([np.concatenate([c, np.zeros(max(0, n - len(c)))]) for c in y])
    if normalize:
        power = max(np.sqrt(np.sum(h64 ** 2) / h64.size), 0.000125)
        y *= 1 / power * 0.00125 * (44100.0 / sr) * (0.5 if len(h64) == 4 else 1.0)
    return y


IR_LENGTHS = [1, 127, 8191, 8192, 8193, 3 * 8192 + 1, 178899]


def _conv_cases():
    out = []
    for ir_len in IR_LENGTHS:
        routings = [(1, 1), (1, 2), (2, 1), (2, 2), (2, 4), (1, 4)] if ir_len in (127, 8193, 3 * 8192 + 1) else [(2, 2), (1, 4)]
        for r in routings:
            for norm in ((False, True) if ir_len != 178899 else (True,)):
                out.append((ir_len, r, norm))
    return out


def _conv_graph(pkg, backend, x, h, n, normalize, device=False):
    c = pkg.OfflineAudioContext(2, n, SR, backend)
    s = c.create_buffer_source(pkg.AudioBuffer(list(x), SR))
    if device:
        cv = c.create_convolver(disable_normalization=not normalize)
        cv.set_device_response(len(h), h.shape[1], SR)
    else:
        cv = c.create_convolver(pkg.AudioBuffer(list(h), SR), disable_normalization=not normalize)
    s.connect(cv)
    cv.connect(c.destination())
    s.start()
    return c, cv


def _conv_data(case, g):
    ir_len, (in_ch, ir_ch), _norm = case
    rng = np.random.default_rng(1000 + g)
    x = rng.uniform(-0.5, 0.5, (in_ch, 3 * 8192 + 1111)).astype(F32)
    env = np.exp(-np.arange(ir_len) / max(1.0, ir_len / 4.0))
    h = (rng.standard_normal((ir_ch, ir_len)) * env).astype(F32)
    return x, h


def _conv_errors(got, truth):
    d = got.astype(np.float64) - truth
    return float(np.sqrt(np.mean(d ** 2))), float(np.abs(d).max())


def _check_conv(pkg, be, cases, n, render_be):
    data = [_conv_data(case, g) for g, case in enumerate(cases)]
    truth = [_conv_truth(x, h, n, case[2], SR) for case, (x, h) in zip(cases, data)]
    ref = _render(pkg, [_conv_graph(pkg, be.pkg_oracle, x, h, n, case[2])[0] for case, (x, h) in zip(cases, data)])
    worst = 0.0
    for opts in be.variants(dict(), dict(chunk=8192)):
        got = render_be(data, opts)
        for g, case in enumerate(cases):
            if case[2]:
                # the reference sums the response's power in f32 (convolver.rs:14-45): its scale is off the f64 one by up to 2e-4 relative at
                # 178 899 frames x 2 channels.  The outputs are compared with the truth at the reference's own scale (fitted to the oracle's
                # render), which is checked to be that close to the specification's
                k = float((ref[g] * truth[g]).sum() / (truth[g] ** 2).sum())
                assert abs(k - 1) <= 5e-4, (case, k)
                truth[g] = truth[g] * k
            peak = float(np.abs(truth[g]).max())
            o_rms, o_max = _conv_errors(ref[g], truth[g])
            # the witness agrees with the reference's f32 convolver to f32 precision
            assert o_max <= 2e-5 * peak, (case, o_max, peak)
            e_rms, e_max = _conv_errors(got[g], truth[g])
            # RMS factor 3, not 2: on the H100 the engine's RMS error measured up to 2.4 x the oracle's where the oracle's is the rounding of a
            # single f32 product (one-tap responses) or little more (responses just past one 8192-frame partition) — every partition of the
            # engine goes through a 16384-point f32 forward and inverse transform, whose rounding is then the larger part of a tiny error
            assert e_rms <= 3 * o_rms + 1e-9 * peak and e_max <= 4 * o_max + 1e-7 * peak, (case, opts, e_rms, o_rms, e_max, o_max)
            worst = max(worst, e_rms / max(o_rms, 1e-30))
    return worst


@pytest.fixture
def cbe(be, oracle):
    be.pkg_oracle = oracle
    return be


@pytest.mark.parametrize("part", [0, 1, 2])
def test_convolver_vs_f64_linear_convolution(pkg, cbe, part):
    # input 3 * 8192 + 1111 frames (several partitions, not a multiple of 128) in a render that runs past it into the tail
    cases = [c for k, c in enumerate(_conv_cases()) if k % 3 == part]
    n = 4 * 8192 + 333

    def render(data, opts):
        with cbe.options(**opts):
            return _render(pkg, [_conv_graph(pkg, cbe.backend, x, h, n, case[2])[0] for case, (x, h) in zip(cases, data)])
    _check_conv(pkg, cbe, cases, n, render)


def test_convolver_in_place_source_and_destination_write(pkg, cbe):
    # source -> Convolver -> destination, the buffer covering the whole render: read in place, written straight to the destination
    cases = [(9000, (2, 2), True), (9000, (2, 1), False), (20000, (2, 2), False)]
    n = 3 * 8192 + 1111   # = the buffer's length

    def render(data, opts):
        with cbe.options(**opts):
            return _render(pkg, [_conv_graph(pkg, cbe.backend, x, h, n, case[2])[0] for case, (x, h) in zip(cases, data)])
    _check_conv(pkg, cbe, cases, n, render)


@pytest.mark.gpu
def test_convolver_responses_bound_from_device_memory(pkg, engine, oracle):
    torch = pytest.importorskip("torch")
    be = _Backend(pkg, "engine", engine.backend, engine)
    be.pkg_oracle = oracle
    cases = [(8193, (2, 2), True), (8193, (2, 2), False), (3 * 8192 + 1, (1, 4), True), (127, (2, 1), True)]
    n = 4 * 8192 + 333

    def render(data, opts):
        outs = []
        with be.options(**opts):
            for case, (x, h) in zip(cases, data):   # (responses of different shapes: one batch each)
                c, cv = _conv_graph(pkg, engine.backend, x, h, n, case[2], device=True)
                b = pkg.Batch([c])
                b.bind_responses(cv, torch.tensor(h[None]).cuda())
                b.run()
                b.sync()
                outs.append(b.fetch_graph(0))
                b.destroy()
        return np.stack(outs)
    _check_conv(pkg, be, cases, n, render)


# ---------------------------------------------------------------------------------------------------------------------------------------
# 6. DelayNode and AnalyserNode at GPU shapes
def _delay_want(x, d_frames):
    # y[n] = x(n - d): linear interpolation between the two neighbouring frames (delay.rs:640-700), x = 0 before the start
    n = np.arange(len(x))
    pos = n - d_frames
    k = np.floor(pos).astype(np.int64)
    f = pos - k
    xp = lambda i: np.where((i >= 0) & (i < len(x)), x[np.clip(i, 0, len(x) - 1)].astype(np.float64), 0.0)
    return (1 - f) * xp(k) + f * xp(k + 1)


def _smooth(rng, n):
    # a random walk scaled into [-1, 1]: steps of at most 0.05, so that a 1e-6 frame error of the read position stays far below the budget
    x = np.cumsum(rng.uniform(-0.05, 0.05, n))
    return (x / np.abs(x).max()).astype(F32)


def test_long_delays_across_the_ring_vs_linear_interpolation(pkg, be):
    # maxDelayTime 3 s, delays up to 2.9 s with fractional frames, an 8 s render (the ring wraps more than twice)
    n = RQ * 3000 + 64
    delays = [0.5, 127.25, 128.0, 1000.5, 48000 * 1.7 + 0.3, 48000 * 2.9 + 0.75, 48000 * 2.9]
    rng = np.random.default_rng(8)
    xs = [_smooth(rng, n) for _ in delays]
    for opts in be.variants(dict(), dict(chunk=128), dict(chunk=1024)):
        ctxs = []
        for d, x in zip(delays, xs):
            c = pkg.OfflineAudioContext(1, n, SR, be.backend)
            s = c.create_buffer_source(pkg.AudioBuffer([x], SR))
            dl = c.create_delay(3.0, d / SR)
            s.connect(dl)
            dl.connect(c.destination())
            s.start()
            ctxs.append(c)
        with be.options(**opts):
            got = _render(pkg, ctxs)
        for g, (d, x) in enumerate(zip(delays, xs)):
            d32 = float(F32(d / SR)) * SR   # delayTime is an f32 AudioParam
            err = float(np.abs(got[g, 0] - _delay_want(x, d32)).max())
            assert err <= 2e-6, (d, opts, err)


def test_delay_time_ramp_vs_linear_interpolation(pkg, be):
    # a-rate delayTime: a linear ramp from 0.1 s to 1.3 s (spec 1.6.3), read per frame (delay.rs:640-700)
    n = RQ * 800
    rng = np.random.default_rng(9)
    x = _smooth(rng, n)
    t = np.arange(n) / SR
    t1 = (n - 1000) / SR
    dt = np.where(t < t1, 0.1 + (1.3 - 0.1) * t / t1, 1.3).astype(F32).astype(np.float64)
    for opts in be.variants(dict(), dict(chunk=128), dict(chunk=1024)):
        c = pkg.OfflineAudioContext(1, n, SR, be.backend)
        s = c.create_buffer_source(pkg.AudioBuffer([x], SR))
        dl = c.create_delay(2.0, 0.1)
        dl.delay_time.linear_ramp_to_value_at_time(1.3, t1)
        s.connect(dl)
        dl.connect(c.destination())
        s.start()
        with be.options(**opts):
            got = _render(pkg, [c])[0, 0]
        want = _delay_want(x, dt * SR)
        # the ramp's f32 value may sit an ulp (1.2e-7 s = 0.006 frames at 1.3 s) from the rounded closed form; the input's slope is at most 0.05
        err = float(np.abs(got - want).max())
        assert err <= 2e-6 + 0.05 * 0.006, (opts, err)


@pytest.mark.parametrize("fft_size", [32, 2048, 32768])
def test_analyser_spectrum_vs_numpy_at_every_fft_size(pkg, be, oracle, fft_size):
    # |X_k| / N of the Blackman-windowed last fft_size frames (analysis.rs:281-369; as test_analyser_spectrum_vs_numpy), tau = 0, linear
    import test_oracle_analyser as AN
    rng = np.random.default_rng(fft_size)
    sr = 44100.0
    n = -(-(fft_size + 640) // RQ) * RQ   # (whole quanta: the window is the signal's last frames)
    sig = (0.5 * np.sin(2 * np.pi * 1000.0 * np.arange(n) / sr) + 0.1 * rng.uniform(-1, 1, n)).astype(F32)
    i = np.arange(fft_size)
    w = 0.42 - 0.5 * np.cos(2 * np.pi * i / fft_size) + 0.08 * np.cos(4 * np.pi * i / fft_size)
    want = np.abs(np.fft.rfft(sig[n - fft_size:].astype(np.float64) * w))[:fft_size // 2] / fft_size

    def err(backend):
        a, _c = AN._analyse(pkg, backend, sig, sr, fft_size=fft_size, smoothing_time_constant=0.0, min_decibels=-200.0)
        got = 10.0 ** (a.get_float_frequency_data().astype(np.float64) / 20.0)
        return float(np.abs(got - want).max())
    o = err(oracle)
    assert o <= 1e-6 * float(want.max()), o   # the witness: the reference's f32 transform is this close to numpy's f64 one
    assert err(be.backend) <= 2 * o + 1e-9, (o,)
