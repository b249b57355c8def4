"""Third statements of the DynamicsCompressorNode, the equal-power PannerNode and the StereoPannerNode at the shapes where their CUDA kernels
(k_compressor; k_panner_eq, k_panner_dyn, k_derive_spatial; k_stereo_panner) can go wrong: every sample rate the ABI takes (the compressor's
look-ahead of D = 1 to 36 quanta), inputs whose channel count and silence change per quantum, chunks shorter than the look-ahead, more than one
CTA of instances, batches that mix sample rates and lengths, moving sources and listeners, poses bound from device memory.

As in tests/test_gpu_witnesses.py, every witness runs with two backends: `oracle` (unmarked: shows on a CPU-only machine that the witness and
its budget are right) and `engine` (the GPU).  None of the witness code is derived from oracle/ or csrc/; each formula cites the
specification, the JAES 2012 paper or the reference's file:line."""
import numpy as np
import pytest

from test_gpu_witnesses import _Backend

RQ = 128
F32 = np.float32
S = np.sqrt(0.5)


@pytest.fixture(params=["oracle", pytest.param("engine", marks=pytest.mark.gpu)])
def be(request, pkg, oracle):
    if request.param == "oracle":
        return _Backend(pkg, "oracle", oracle)
    engine = request.getfixturevalue("engine")
    return _Backend(pkg, "engine", engine.backend, engine)


def _render_each(pkg, be, ctxs):
    """[graph] -> [channel][frame] f32, for contexts of any mix of lengths and sample rates"""
    if be.is_engine:
        b = pkg.Batch(ctxs, many=True)
        b.run()
        b.sync()
        return [b.fetch_graph(g).reshape(c._channels, c._length) for g, c in enumerate(ctxs)]
    return [np.stack(a.channels) for a in pkg.render_many(ctxs)]


# ---------------------------------------------------------------------------------------------------------------------------------------
# A. DynamicsCompressorNode
#
# The specification's compression curve and makeup gain, the gain computer (eq. 4) and branching peak detector (eq. 7, 16) of Giannoulis,
# Massberg and Reiss, "Digital Dynamic Range Compressor Design" (JAES 2012), as dynamics_compressor.rs:330-478 follows them, with the layout
# of the reference's look-ahead:
# - D = ceil(sr * 0.006 / 128) quanta, computed in f32 (dynamics_compressor.rs:253-254: a ring of D + 1 whole quanta, read one slot ahead of
#   the write, :452-461).  The output of quantum q is input quantum q - D, WITH its channel count and silence; the ring starts out silent
#   (:343-349); a silent delayed quantum gives the silent output (:465-468).
# - The detector takes per frame the max |x| over the channels the CURRENT input quantum has (:400-407); a silent quantum is one zero channel:
#   lin_to_db(0) = -1000 dB.
# - Params are k-rate: the first value of each quantum (:353-377).
# - reduction() is the dB gain of the last frame the node rendered (:440, :450).
# The node's input port is count 2, clamped-max, speakers (:57-58): a 6-channel input reaches it down-mixed to stereo (spec: 5.1 -> stereo),
# a mono one stays mono and reaches a stereo destination as L = R.
def _comp_d(sr):
    return int(np.ceil(F32(F32(sr) * F32(0.006)) / F32(RQ)))


def _time_step(sr):
    """the longest 2^-m s (m <= 12) that is a whole number of frames at `sr`: start and stop times on its multiples are exact binary fractions
    that land on whole frames, so no sub-sample scheduling enters the witness"""
    for m in range(13):
        if (sr * 2.0 ** -m) != int(sr * 2.0 ** -m):
            return 2.0 ** -(m - 1)
    return 2.0 ** -12


class _Src:
    """one AudioBufferSourceNode at rate 1: `pcm` [ch][frames] plays from frame `a` and is stopped at frame `b` (the buffer is longer: the stop
    time ends it)"""

    def __init__(self, pcm, a, b):
        assert pcm.shape[1] > b - a
        self.pcm, self.a, self.b = pcm, a, b

    def active(self, q):  # plays in quantum q: it renders its own channel count there, zeros outside [a, b)
        return self.a < (q + 1) * RQ and self.b > q * RQ


def _to_port(x, k):
    """spec: speakers up / down-mix of k channels to the compressor's port (at most 2: clamped-max 2)"""
    if k == 1:
        return [x[0]]
    if k == 2:
        return [x[0], x[1]]
    if k == 6:  # 5.1 -> stereo: L + sqrt(1/2) (C + SL), R + sqrt(1/2) (C + SR)
        return [x[0] + S * (x[2] + x[4]), x[1] + S * (x[2] + x[5])]
    raise ValueError(k)


class _Comp:
    """one graph: sources -> DynamicsCompressorNode -> destination (2 channels).  params: dict name -> value; steps: [(name, quantum, value)]
    set with setValueAtTime on a quantum boundary (sample rates where a quantum is a binary fraction of a second)"""
    NAMES = ("attack", "knee", "ratio", "release", "threshold")

    def __init__(self, sr, n, srcs, params=None, steps=()):
        assert n % RQ == 0
        self.sr, self.n, self.srcs, self.steps = float(F32(sr)), n, srcs, list(steps)
        self.params = dict(attack=0.003, knee=30.0, ratio=12.0, release=0.25, threshold=-24.0)
        self.params.update(params or {})
        if self.steps:
            assert (RQ / self.sr) == 2.0 ** np.round(np.log2(RQ / self.sr)), "steps need quanta that are binary fractions of a second"

    def build(self, pkg, backend):
        c = pkg.OfflineAudioContext(2, self.n, self.sr, backend)
        d = c.create_dynamics_compressor(**self.params)
        for s in self.srcs:
            src = c.create_buffer_source(pkg.AudioBuffer(list(s.pcm), self.sr))
            src.connect(d)
            src.start_at(s.a / self.sr)
            src.stop_at(s.b / self.sr)
        for name, q, v in self.steps:
            getattr(d, name).set_value_at_time(v, q * RQ / self.sr)
        d.connect(c.destination())
        return c, d

    def port(self):
        """the compressor's input: x [2][n] f64 (a mono quantum has x[1] = x[0]) and its layout per quantum: 0 silent, 1 mono, 2 stereo"""
        n_q = self.n // RQ
        x = np.zeros((2, self.n))
        lay = np.zeros(n_q, np.int64)
        for s in self.srcs:
            frames = np.zeros((s.pcm.shape[0], self.n))
            hi = min(s.b, self.n)
            frames[:, s.a:hi] = s.pcm[:, :hi - s.a]
            s.port = _to_port(frames, s.pcm.shape[0])
            for q in range(n_q):
                if s.active(q):
                    lay[q] = max(lay[q], len(s.port))
        for s in self.srcs:
            for q in range(n_q):
                if s.active(q):
                    sl = slice(q * RQ, (q + 1) * RQ)
                    x[0, sl] += s.port[0][sl]
                    x[1, sl] += s.port[-1][sl]   # (mono up-mixed to the port's stereo: L = R; a mono port keeps x[1] = x[0])
        return x, lay

    def param_track(self):
        """[5][n_q] f64: the k-rate value of each param per quantum (f32 AudioParam values).  A k-rate param gives a block the intrinsic
        value the block started with, before the block's events are applied (param.rs:1543-1544): a step at the start of quantum q is heard
        from quantum q + 1 on"""
        n_q = self.n // RQ
        t = {k: np.full(n_q, float(F32(v))) for k, v in self.params.items()}
        for name, q, v in sorted(self.steps, key=lambda s: s[1]):
            t[name][q + 1:] = float(F32(v))
        return [t[k] for k in self.NAMES]


def _comp_witness(graphs):
    """-> [(out [2][n] f64, reduction dB)], the detector's recurrence vectorised over the graphs"""
    G = len(graphs)
    n_max = max(g.n for g in graphs)
    lvl = np.zeros((G, n_max))
    xs, lays = [], []
    thr = np.zeros((G, n_max)); knee = np.zeros((G, n_max)); ratio = np.ones((G, n_max))
    a_tau = np.zeros((G, n_max)); r_tau = np.zeros((G, n_max)); makeup = np.zeros((G, n_max))
    for i, g in enumerate(graphs):
        x, lay = g.port()
        xs.append(x)
        lays.append(lay)
        live = np.repeat(lay > 0, RQ)
        lvl[i, :g.n] = np.where(live, np.maximum(np.abs(x[0]), np.abs(x[1])), 0.0)
        at, kn, ra, re, th = (np.repeat(v, RQ) for v in g.param_track())
        sl = slice(0, g.n)
        # compression curve with the knee centred on the shifted threshold (paper's W around T; dynamics_compressor.rs:356-371)
        thr[i, sl] = np.where(kn > 0, th + kn / 2, th)
        knee[i, sl], ratio[i, sl] = kn, ra
        with np.errstate(divide="ignore"):
            a_tau[i, sl] = np.exp(-1.0 / (at * g.sr))   # eq. 7 (attack 0: tau 0, the detector follows at once)
            r_tau[i, sl] = np.exp(-1.0 / (re * g.sr))
        # spec: full range gain = the curve applied to 0 dB, makeup = (1 / full range gain)^0.6, in dB
        makeup[i, sl] = -0.6 * (thr[i, sl] - thr[i, sl] / ratio[i, sl])
    with np.errstate(divide="ignore"):
        xg = np.where(lvl == 0, -1000.0, 20 * np.log10(lvl))
    T, W, R = thr, knee, ratio
    # eq. 4
    yg = np.where(2 * (xg - T) < -W, xg,
                  np.where(2 * np.abs(xg - T) <= W, xg + (1 / R - 1) * (xg - T + W / 2) ** 2 / np.where(W > 0, 2 * W, 1.0), T + (xg - T) / R))
    xl = xg - yg
    yl = np.zeros((G, n_max))
    prev = np.zeros(G)
    for f in range(n_max):   # eq. 16, the branching peak detector
        att = xl[:, f] > prev
        tau = np.where(att, a_tau[:, f], r_tau[:, f])
        prev = tau * prev + (1 - tau) * xl[:, f]
        yl[:, f] = prev
    red = -yl + makeup
    out = []
    for i, g in enumerate(graphs):
        D = _comp_d(g.sr)
        gain = 10.0 ** (red[i, :g.n] / 20)
        delayed = np.zeros((2, g.n))
        delayed[:, D * RQ:] = xs[i][:, :g.n - D * RQ]
        lay_out = np.concatenate([np.zeros(D, np.int64), lays[i]])[:g.n // RQ]
        delayed *= np.repeat(lay_out > 0, RQ)
        out.append((delayed * gain, float(red[i, g.n - 1])))
    return out


def _noise(rng, ch, frames, amp):
    return (amp * rng.uniform(-1, 1, (ch, frames))).astype(F32)


def _comp_inputs(rng, sr, n, ch, kind):
    """sources for one graph: 'constant' (from 0 to the end), 'late' (starts late), 'stop' (stops well before the end: the look-ahead's last
    quanta come out after the input fell silent), 'switch' (a mono source from 0 and a stereo burst that starts and stops inside it)"""
    u = int(round(_time_step(sr) * sr))   # frames per time step
    steps = n // u
    if kind == "constant":
        return [_Src(np.full((ch, n + 1), 0.7, F32) * np.linspace(1.0, 0.5, ch, dtype=F32)[:, None], 0, n)]
    if kind == "late":
        a = u * max(1, steps // 3)
        return [_Src(_noise(rng, ch, n, 0.9), a, n)]
    if kind == "stop":
        a = u * (steps // 4)
        b = u * max(steps // 4 + 1, (2 * steps) // 3)
        return [_Src(_noise(rng, ch, n, 0.9), a, b)]
    if kind == "switch":
        a = u * max(1, steps // 4)
        b = u * max(steps // 4 + 1, steps // 2)
        return [_Src(_noise(rng, 1, n + 1, 0.3), 0, n), _Src(_noise(rng, 2, n, 0.8), a, b)]
    raise ValueError(kind)


def _comp_budget(sr):
    """(output, relative to max(1, peak); reduction, dB).  The reference runs the detector in f32 (dynamics_compressor.rs:378-379, :431-436):
    1 - tau is a few hundred f32 ulps at high rates (release 0.25 s at 768 kHz: 5e-6), so each step's rounding is a relative error of the
    attack / release rate, which grows with the rate.  Measured on the oracle: 2.0e-4 of the peak at 176.4 kHz, 3.8e-4 at 768 kHz; the
    reduction, read at the end of a long release (release 1 s), up to 3e-3 dB at 32 kHz and 3.7e-2 dB of a 10 dB reduction at 176.4 kHz.
    The budgets grow with the square root of the rate, about 1.5x the measured error at the rates where it peaks."""
    return 2e-4 * max(1.0, np.sqrt(sr / 96000.0)), 6e-3 * max(1.0, np.sqrt(sr / 24000.0))


def _check_comp(pkg, be, graphs, opts=None, what=""):
    want = _comp_witness(graphs)
    made = [g.build(pkg, be.backend) for g in graphs]
    with be.options(**(opts or {})):
        got = _render_each(pkg, be, [c for c, _ in made])
    if be.is_engine:   # the engine also stays within f32 transcendental noise of the reference's own f32 arithmetic (tests/test_gpu_parity.py)
        ref_made = [g.build(pkg, be.pkg_oracle.backend) for g in graphs]
        ref = _render_each(pkg, be.pkg_oracle, [c for c, _ in ref_made])
    for i, g in enumerate(graphs):
        w, red = want[i]
        out_budget, red_budget = _comp_budget(g.sr)
        peak = max(1.0, float(np.abs(w).max()))
        err = float(np.abs(got[i] - w).max())
        assert err <= out_budget * peak, (what, i, g.sr, err, peak)
        got_red = made[i][1].reduction()
        assert abs(got_red - red) <= red_budget * max(1.0, abs(red) / 4), (what, i, g.sr, got_red, red)
        if be.is_engine:
            assert float(np.abs(got[i] - ref[i]).max()) <= 5e-5 * peak, (what, i, g.sr)
            assert abs(got_red - ref_made[i][1].reduction()) <= 1e-3 * max(1.0, g.sr / 48000.0), (what, i, g.sr)


@pytest.fixture
def cbe(be, oracle):
    be.pkg_oracle = _Backend(be.pkg, "oracle", oracle)
    return be


RATES = [3000.0, 22050.0, 44100.0, 48000.0, 96000.0, 176400.0, 192000.0, 384000.0, 768000.0]


def test_compressor_look_ahead_is_whole_quanta_from_1_to_36():
    # the reference's f32 ceiling; from 176.4 kHz on the look-ahead holds more than 8 quanta
    assert [_comp_d(sr) for sr in RATES] == [1, 2, 3, 3, 5, 9, 9, 18, 36]


@pytest.mark.parametrize("sr", RATES)
def test_compressor_every_sample_rate_vs_the_published_design(pkg, cbe, sr):
    # one graph per input kind and width (the 'switch' graphs are mono + stereo); ~0.4 s, at least 3 whole time steps
    u = int(round(_time_step(sr) * sr))
    n = -(-max(3 * u, int(0.4 * sr)) // RQ) * RQ
    rng = np.random.default_rng(int(sr))
    graphs = [_Comp(sr, n, _comp_inputs(rng, sr, n, ch, kind)) for kind in ("constant", "late", "stop") for ch in (1, 2, 6)]
    graphs.append(_Comp(sr, n, _comp_inputs(rng, sr, n, 1, "switch")))
    for opts in cbe.variants(dict(), dict(chunk=128), dict(chunk=1024)):
        _check_comp(pkg, cbe, graphs, opts, (sr, opts))


def _mixed_graphs(rng, sr, n, count):
    kinds = [(k, ch) for k in ("constant", "late", "stop") for ch in (1, 2, 6)] + [("switch", 1)]
    return [_Comp(sr, n, _comp_inputs(rng, sr, n, kinds[g % len(kinds)][1], kinds[g % len(kinds)][0])) for g in range(count)]


def test_compressor_many_instances_in_one_batch(pkg, cbe):
    # 600 graphs at 48 kHz and 200 at 192 kHz: one thread per instance, 32 per CTA -> many CTAs and a ragged last one
    rng = np.random.default_rng(5)
    for sr, count, secs in ((48000.0, 600, 0.25), (192000.0, 200, 0.125)):
        n = int(sr * secs) // RQ * RQ
        graphs = _mixed_graphs(rng, sr, n, count)
        for opts in cbe.variants(dict(), dict(chunk=128)):
            _check_comp(pkg, cbe, graphs, opts, (sr, count, opts))


def test_compressor_batch_of_mixed_sample_rates_and_lengths(pkg, cbe):
    # every rate in one batch, each graph its own length: a different look-ahead per instance and graphs that end before the batch does
    rng = np.random.default_rng(6)
    graphs = []
    for k, sr in enumerate(RATES):
        u = int(round(_time_step(sr) * sr))
        n = -(-max(3 * u, int((0.15 + 0.05 * k) * sr)) // RQ) * RQ
        graphs += _mixed_graphs(rng, sr, n, 4 + k % 3)
    for opts in cbe.variants(dict(), dict(chunk=128), dict(chunk=1024)):
        _check_comp(pkg, cbe, graphs, opts, opts)


def test_compressor_long_render_at_192k(pkg, cbe):
    # 3 s at 192 kHz (D = 9): sources that stop and switch their channel count many chunks into the render
    sr, n = 192000.0, 192000 * 3
    rng = np.random.default_rng(7)
    u = int(_time_step(sr) * sr)
    graphs = [_Comp(sr, n, [_Src(_noise(rng, 2, n, 0.9), u * 100, u * 1000)]),
              _Comp(sr, n, [_Src(_noise(rng, 1, n + 1, 0.3), 0, n)] + [_Src(_noise(rng, 2, n, 0.8), u * a, u * b) for a, b in ((7, 9), (700, 1300))]),
              _Comp(sr, n, [_Src(_noise(rng, 6, n, 0.5), u * 3, u * 1499)], dict(release=1.0, attack=0.0))]
    for opts in cbe.variants(dict(), dict(chunk=1024)):
        _check_comp(pkg, cbe, graphs, opts, opts)


EXTREMES = [dict(knee=0.0), dict(ratio=1.0), dict(ratio=20.0), dict(attack=0.0), dict(release=1.0), dict(threshold=0.0), dict(threshold=-100.0),
            dict(knee=0.0, ratio=20.0, attack=0.0, threshold=-100.0), dict(knee=40.0, ratio=1.0, release=1.0, threshold=0.0),
            dict(knee=0.0, attack=0.05, release=0.0, threshold=-60.0)]


@pytest.mark.parametrize("sr", [48000.0, 176400.0])
def test_compressor_extreme_params(pkg, cbe, sr):
    rng = np.random.default_rng(8)
    u = int(round(_time_step(sr) * sr))
    n = -(-max(3 * u, int(0.3 * sr)) // RQ) * RQ
    graphs = [_Comp(sr, n, _comp_inputs(rng, sr, n, ch, kind), p) for p in EXTREMES for kind, ch in (("stop", 2), ("switch", 1), ("late", 6))]
    for opts in cbe.variants(dict(), dict(chunk=128)):
        _check_comp(pkg, cbe, graphs, opts, (sr, opts))


@pytest.mark.parametrize("sr", [32768.0, 262144.0])
def test_compressor_k_rate_automation_of_every_param(pkg, cbe, sr):
    # setValueAtTime on quantum boundaries (a quantum is 2^-8 s at 32768 Hz, 2^-11 s at 262144 Hz: the times are exact); at 262144 Hz D = 13
    rng = np.random.default_rng(9)
    n_q = 160
    n = n_q * RQ
    graphs = []
    for g in range(40):
        steps = [("threshold", 10 + g % 7, float(rng.uniform(-80, -5))), ("knee", 30 + g % 5, float(rng.choice([0.0, 3.0, 40.0]))),
                 ("ratio", 45 + g % 11, float(rng.choice([1.0, 2.5, 20.0]))), ("attack", 60, float(rng.choice([0.0, 0.001, 0.2]))),
                 ("release", 61 + g % 3, float(rng.choice([0.01, 0.3, 1.0]))), ("threshold", 100 + g % 13, -30.0), ("ratio", 120, 6.0)]
        graphs.append(_Comp(sr, n, _comp_inputs(rng, sr, n, (1, 2, 6)[g % 3], ("constant", "late", "stop")[g % 3]) if g % 4 else
                            _comp_inputs(rng, sr, n, 1, "switch"), steps=steps))
    for opts in cbe.variants(dict(), dict(chunk=128)):
        _check_comp(pkg, cbe, graphs, opts, (sr, opts))


# ---------------------------------------------------------------------------------------------------------------------------------------
# B. equal-power PannerNode, C. StereoPannerNode
#
# 32768 Hz: a quantum is 2^-8 s, so sources start and stop, and ramps end, on exact quantum boundaries.
PSR = 32768.0


def _unit(v):
    n = np.linalg.norm(v, axis=-1, keepdims=True)
    return v / np.where(n == 0, 1.0, n)


def _acos_deg(c):
    return np.degrees(np.arccos(np.clip(c, -1.0, 1.0)))


def _spatial(src, ori, lp, fwd, up, model, ref, mx, roll, inner, outer, outer_gain):
    """spatial.rs:205-299 and panner.rs:927-985 in f64, vectorised over poses [N, 3] (f32 values): -> (azimuth, gain, arguments of every acos)
    - azimuth: the source-listener vector projected on the plane orthogonal to up' = right x forward (right = forward x up), measured from
      right, 360 - angle behind the listener, then relative to forward; (0, 0) for a coincident source or forward parallel to up, azimuth 0
      for a source straight above or below (spatial.rs:213-267)
    - distance gain: the three models of the specification with the reference's clamps (panner.rs:955-985)
    - cone gain: the angle between the orientation and the vector from the LISTENER to the SOURCE (spatial.rs:277-299, DESIGN.md §6), 1 with
      no cone or a zero orientation, linear between the half-angles (panner.rs:927-953)"""
    src, ori, lp, fwd, up = (np.asarray(a, np.float64) for a in (src, ori, lp, fwd, up))
    rel = src - lp
    coincident = (rel ** 2).sum(-1) <= np.finfo(F32).tiny
    sl = _unit(rel)
    right = np.cross(fwd, up)
    no_right = (right ** 2).sum(-1) == 0
    rn, fn = _unit(right), _unit(fwd)
    up2 = np.cross(rn, fn)
    el_arg = (sl * up2).sum(-1)
    proj = sl - el_arg[:, None] * up2
    no_proj = (proj ** 2).sum(-1) == 0
    pn = _unit(proj)
    az_arg = (pn * rn).sum(-1)
    az = _acos_deg(az_arg)
    az = np.where((pn * fn).sum(-1) < 0, 360 - az, az)
    az = np.where((az >= 0) & (az <= 270), 90 - az, 450 - az)
    az = np.where(coincident | no_right | no_proj, 0.0, az)
    d = np.sqrt((rel ** 2).sum(-1))
    if model == "linear":
        lo, hi = min(ref, mx), max(ref, mx)
        dg = 1 - min(max(roll, 0.0), 1.0) * (np.clip(d, lo, hi) - lo) / (hi - lo)
    elif model == "inverse":
        r = max(roll, 0.0)
        dg = np.where(d > 0, ref / (ref + r * (np.maximum(d, ref) - ref)), 1.0)
    else:
        dg = (np.maximum(d, ref) / ref) ** -max(roll, 0.0)
    cone_arg = (sl * _unit(ori)).sum(-1)
    angle = np.where(((ori ** 2).sum(-1) == 0) | coincident, 0.0, np.abs(_acos_deg(cone_arg)))
    hi_, ho = abs(inner) / 2, abs(outer) / 2
    if hi_ >= 180 and ho >= 180:
        cg = np.ones_like(angle)
    else:
        x = (angle - hi_) / np.where(ho - hi_ == 0, 1.0, ho - hi_)
        cg = np.where(angle < hi_, 1.0, np.where(angle >= ho, outer_gain, (1 - x) + outer_gain * x))
    live = ~(coincident | no_right)
    args = [np.where(live, el_arg, 0.0), np.where(live & ~no_proj, az_arg, 0.0), np.where(((ori ** 2).sum(-1) > 0) & ~coincident, cone_arg, 0.0)]
    return az, dg * cg, args


def _equal_power(az, g, x):
    """panner.rs:988-1057: x [1 or 2][N] -> [2][N]; azimuth clamped to [-180, 180] and folded into [-90, 90]"""
    az = np.clip(az, -180, 180)
    az = np.where(az < -90, -180 - az, np.where(az > 90, 180 - az, az))
    if len(x) == 1:
        p = (az + 90) / 180 * np.pi / 2
        return np.array([x[0] * np.cos(p) * g, x[0] * np.sin(p) * g])
    p = np.where(az <= 0, (az + 90) / 90, az / 90) * np.pi / 2
    gl, gr = np.cos(p), np.sin(p)
    return np.where(az <= 0, [(x[0] + x[1] * gl) * g, x[1] * gr * g], [x[0] * gl * g, (x[1] + x[0] * gr) * g])


def _pan_err(got, want):
    return float(np.abs(got - want).max()) / max(1.0, float(np.abs(want).max()))


POSE_FIELDS = ("src", "ori", "lp", "fwd", "up")
EDGE_POSES = [  # (src, orientation, listener position, forward, up, model, ref, max, rolloff, inner, outer, outer gain)
    ((0, 0, 0), (1, 0, 0), (0, 0, 0), (0, 0, -1), (0, 1, 0), "inverse", 1.0, 10000.0, 1.0, 360.0, 360.0, 0.0),       # at the listener
    ((1, 2, 3), (1, 0, 0), (1, 2, 3), (0, 0, -1), (0, 1, 0), "inverse", 1.0, 10000.0, 1.0, 90.0, 200.0, 0.3),        # (and a cone)
    ((0, 5, 0), (1, 0, 0), (0, 0, 0), (0, 0, -1), (0, 1, 0), "inverse", 1.0, 10000.0, 1.0, 360.0, 360.0, 0.0),       # straight overhead
    ((0, -3, 0), (0, 1, 0), (0, 0, 0), (0, 0, -1), (0, 1, 0), "exponential", 1.0, 100.0, 0.5, 40.0, 120.0, 0.2),     # straight below
    ((2, 0, -1), (0, 0, 0), (0, 0, 0), (0, 0, -1), (0, 1, 0), "inverse", 1.0, 10000.0, 1.0, 30.0, 60.0, 0.1),        # zero orientation
    ((2, 1, -1), (1, 0, 0), (0, 0, 0), (0, 1, 0), (0, 1, 0), "inverse", 1.0, 10000.0, 1.0, 360.0, 360.0, 0.0),       # forward = up
    ((2, 1, -1), (1, 0, 0), (0, 0, 0), (0, 0, -2), (0, 0, 3), "inverse", 1.0, 10000.0, 1.0, 360.0, 360.0, 0.0),     # forward || up
    ((0, 0, -4), (1, 0, 0), (0, 0, 0), (0, 0, -1), (0, 1, 0), "linear", 1.0, 10.0, 0.5, 360.0, 360.0, 0.0),          # azimuth 0
    ((3, 0, 0), (1, 0, 0), (0, 0, 0), (0, 0, -1), (0, 1, 0), "linear", 1.0, 10.0, 0.5, 360.0, 360.0, 0.0),           # azimuth 90
    ((-3, 0, 0), (1, 0, 0), (0, 0, 0), (0, 0, -1), (0, 1, 0), "linear", 1.0, 10.0, 0.5, 360.0, 360.0, 0.0),          # azimuth -90
    ((0, 0, 2), (1, 0, 0), (0, 0, 0), (0, 0, -1), (0, 1, 0), "linear", 1.0, 10.0, 0.5, 360.0, 360.0, 0.0),           # azimuth 180
    ((2, 0.5, 3), (1, 0, 0), (0, 0, 0), (0, 0, -1), (0, 1, 0), "inverse", 1.0, 10000.0, 1.0, 360.0, 360.0, 0.0),     # behind, right
    ((-2, -0.5, 1), (1, 0, 0), (0, 0, 0), (0, 0, -1), (0, 1, 0), "inverse", 1.0, 10000.0, 1.0, 360.0, 360.0, 0.0),   # behind, left
    ((1, 0, -5), (1, 0, 0), (0, 0, 0), (0, 0, -1), (0, 1, 0), "linear", 8.0, 2.0, 0.7, 360.0, 360.0, 0.0),           # ref > max
    ((1, 0, -5), (1, 0, 0), (0, 0, 0), (0, 0, -1), (0, 1, 0), "linear", 1.0, 20.0, 3.0, 360.0, 360.0, 0.0),          # rolloff > 1
    ((0, 0, 0), (1, 0, 0), (0, 0, 0), (0, 0, -1), (0, 1, 0), "inverse", 2.0, 10000.0, 1.0, 360.0, 360.0, 0.0),       # inverse at 0
    ((4, 1, -5), (1, 0, 0), (0, 0, 0), (0, 0, -1), (0, 1, 0), "exponential", 1.0, 100.0, 0.0, 360.0, 360.0, 0.0),    # rolloff 0
    ((4, 1, -5), (1, 0, 0), (0, 0, 0), (0, 0, -1), (0, 1, 0), "inverse", 1.0, 100.0, 0.0, 360.0, 360.0, 0.0),
    ((1, 1, -2), (-1, 0, 0.5), (0, 0, 0), (0, 0, -1), (0, 1, 0), "inverse", 1.0, 10000.0, 1.0, 300.0, 60.0, 0.25),   # inner > outer
    ((1, 1, -2), (0.3, 0.2, -1), (0.5, -1, 2), (1, 0, -1), (0, 1, 0), "exponential", 0.5, 100.0, 1.5, 100.0, 250.0, 0.4),
]
MODELS = {"linear": 0, "inverse": 1, "exponential": 2}


def _pose_lists(rng, n):
    """n random static poses, and the edge poses"""
    out = []
    for _ in range(n):
        fwd = rng.uniform(-1, 1, 3)
        up = rng.uniform(-1, 1, 3)
        model = ("linear", "inverse", "exponential")[int(rng.integers(3))]
        ref, mx = float(rng.uniform(0.2, 3)), float(rng.uniform(4, 30))
        inner = float(rng.uniform(0, 360))
        out.append((tuple(rng.uniform(-8, 8, 3)), tuple(rng.uniform(-1, 1, 3)), tuple(rng.uniform(-2, 2, 3)), tuple(fwd), tuple(up), model, ref, mx,
                    float(rng.uniform(0, 1.5)), inner, float(rng.uniform(inner, 360)), float(rng.uniform(0, 1))))
    return out + EDGE_POSES


class _PanInput:
    """the sources in front of a panner: 'mono' / 'stereo' play from frame 0 to the end; 'switch' is a mono source that starts late and stops
    early, and a stereo burst inside it (whole quanta: the times are exact at 32768 Hz).  x [2][n] f64 is the panner's input (a mono quantum
    has x[1] = x[0]) and lay its layout per quantum: 0 silent, 1 mono, 2 stereo (the port is count 2, clamped-max: panner.rs:162-163)"""

    def __init__(self, seed, n, kind):
        rng = np.random.default_rng(seed)
        if kind in ("mono", "stereo"):
            self.srcs = [(rng.uniform(-1, 1, (1 if kind == "mono" else 2, n)).astype(F32), 0, n)]
        else:
            a, b = RQ * (3 + seed % 5), n - RQ * (4 + seed % 7)
            c = a + RQ * (5 + seed % 13)
            d = min(b, c + RQ * (10 + seed % 17))
            self.srcs = [(rng.uniform(-0.5, 0.5, (1, n)).astype(F32), a, b), (rng.uniform(-0.5, 0.5, (2, n)).astype(F32), c, d)]
        self.x = np.zeros((2, n))
        self.lay = np.zeros(n // RQ, np.int64)
        for pcm, a, b in self.srcs:
            self.x[:, a:b] += pcm[:, :b - a]   # (mono up-mixed to stereo: L = R)
            self.lay[a // RQ:-(-b // RQ)] = np.maximum(self.lay[a // RQ:-(-b // RQ)], len(pcm))

    def connect(self, pkg, c, node):
        for pcm, a, b in self.srcs:
            s = c.create_buffer_source(pkg.AudioBuffer(list(pcm), PSR))
            s.connect(node)
            s.start_at(a / PSR)
            if b < c.length():
                s.stop_at(b / PSR)

    def want(self, az, gain):
        """each quantum panned with the law of its own layout (panner.rs:846-894); a silent quantum is silent (panner.rs:698-708) -> (output,
        silent frames)"""
        per = np.repeat(self.lay, RQ)
        out = np.where(per == 2, _equal_power(az, gain, self.x), np.where(per == 1, _equal_power(az, gain, self.x[:1]), 0.0))
        return out, per == 0


def _pose_graph(pkg, backend, pose, inp, n, bound=False):
    src, ori, lp, fwd, up, model, ref, mx, roll, inner, outer, og = pose
    c = pkg.OfflineAudioContext(2, n, PSR, backend)
    p = c.create_panner(distance_model=MODELS[model], position=(0.0, 0.0, 0.0) if bound else tuple(map(float, src)),
                        orientation=(1.0, 0.0, 0.0) if bound else tuple(map(float, ori)), ref_distance=ref, max_distance=mx, rolloff_factor=roll,
                        cone_inner_angle=inner, cone_outer_angle=outer, cone_outer_gain=og)
    lis = c.listener()
    lparams = [lis.position_x, lis.position_y, lis.position_z, lis.forward_x, lis.forward_y, lis.forward_z, lis.up_x, lis.up_y, lis.up_z]
    if not bound:
        for prm, v in zip(lparams, list(lp) + list(fwd) + list(up)):
            prm.set_value(float(v))
    inp.connect(pkg, c, p)
    p.connect(c.destination())
    return c, [p.position_x, p.position_y, p.position_z, p.orientation_x, p.orientation_y, p.orientation_z] + lparams


def _pose_want(pose, inp):
    src, ori, lp, fwd, up, model, ref, mx, roll, inner, outer, og = pose
    vec = [np.array([v], F32).astype(np.float64) for v in (src, ori, lp, fwd, up)]
    az, g, args = _spatial(*vec, model, ref, mx, roll, inner, outer, og)
    ill = max(float(np.abs(a).max()) for a in args) >= 1 - 1e-3
    return inp.want(az[0], g[0]) + (ill,)


# Where an acos argument is within 1e-3 of +-1, f32 acos is ill-conditioned (d acos / dx = 1 / sqrt(1 - x^2)): an argument one f32 ulp off
# moves the angle by up to sqrt(2 * 6e-8) = 3.5e-4 rad, so the reference's own f32 evaluation strays from the f64 witness there.  The oracle
# is held to 1e-3 of the peak at those poses, the engine to twice the oracle's error for the same case.  The degenerate rules (a coincident
# source, forward parallel to up, a source straight above: azimuth 0; spatial.rs:213-250) zero those arguments in the witness: such poses
# are not ill-conditioned and fall under the 1e-5 budget.
def _assert_pan(got, want, silent, ill, ref, what):
    assert np.all(got[:, silent] == 0.0), what
    err = _pan_err(got, want)
    if not ill:
        assert err <= 1e-5, (what, err)
    elif ref is None:
        assert err <= 1e-3, (what, err)
    else:
        assert err <= 2 * _pan_err(ref, want) + 1e-6, (what, err)


def _check_static(pkg, be, oracle_backend, poses, inps, n, render):
    got = render(poses)
    ref = render(poses, oracle_backend) if be.is_engine else None
    for i, pose in enumerate(poses):
        want, silent, ill = _pose_want(pose, inps[i])
        _assert_pan(got[i], want, silent, ill, None if ref is None else ref[i], (i, pose))


@pytest.mark.parametrize("stereo", [False, True])
def test_equal_power_panner_static_poses(pkg, be, oracle, stereo):
    # ~1000 graphs of random poses and the edge poses (k_panner_eq: one set of spatial params per graph), 24 quanta
    rng = np.random.default_rng(11 + stereo)
    n = RQ * 24
    poses = _pose_lists(rng, 980)
    inps = [_PanInput(1000 * stereo + g, n, "stereo" if stereo else "mono") for g in range(len(poses))]

    def render(ps, backend=None):
        return _render_each(pkg, _Backend(pkg, "oracle", backend) if backend else be,
                            [_pose_graph(pkg, backend or be.backend, p, inps[i], n)[0] for i, p in enumerate(ps)])
    _check_static(pkg, be, oracle, poses, inps, n, render)


@pytest.mark.gpu
@pytest.mark.parametrize("stereo", [False, True])
def test_equal_power_panner_poses_bound_from_device_memory(pkg, engine, oracle, stereo):
    # the 15 spatial params bound per run (k_derive_spatial): the batch is run three times with three different pose sets, the witness taken
    # at the bound values clamped to the declared range
    torch = pytest.importorskip("torch")
    be = _Backend(pkg, "engine", engine.backend, engine)
    rng = np.random.default_rng(21 + stereo)
    n = RQ * 16
    inps = [_PanInput(2000 * stereo + g, n, "stereo" if stereo else "mono") for g in range(300 + len(EDGE_POSES))]
    made = None
    for run in range(3):
        poses = _pose_lists(rng, 300)
        if run == 2:
            poses = poses[::-1]
        if made is None:
            made = [_pose_graph(pkg, engine.backend, p, inps[i], n, bound=True) for i, p in enumerate(poses)]
            for _c, params in made:
                for prm in params:
                    prm.set_device_value(-6.0, 6.0)   # (random positions reach +-8: the bound values are clamped to the declared range)
            b = pkg.Batch([c for c, _ in made])
        vals = torch.tensor([list(p[0]) + list(p[1]) + list(p[2]) + list(p[3]) + list(p[4]) for p in poses], dtype=torch.float32).cuda()
        b.bind_params(made[0][1], vals)
        b.run()
        b.sync()
        got = [b.fetch_graph(g) for g in range(len(poses))]
        # the graphs were built with the models / cones of the first run's poses: the witness takes those, at the bound positions
        first = poses if run == 0 else first
        eff = [tuple(tuple(np.clip(np.asarray(v, F32), -6.0, 6.0)) for v in p[:5]) + tuple(f[5:]) for p, f in zip(poses, first)]

        def render(ps, backend=None, eff=eff):
            if backend is None:
                return got
            return _render_each(pkg, _Backend(pkg, "oracle", backend), [_pose_graph(pkg, backend, p, inps[i], n)[0] for i, p in enumerate(ps)])
        _check_static(pkg, be, oracle, eff, inps, n, render)
    b.destroy()


def _stereo_pan(pan, x):
    """https://webaudio.github.io/web-audio-api/#stereopanner-algorithm: x [1 or 2][N], pan [N] -> [2][N]"""
    if len(x) == 1:
        p = (pan + 1) / 2 * np.pi / 2
        return np.array([x[0] * np.cos(p), x[0] * np.sin(p)])
    p = np.where(pan <= 0, pan + 1, pan) * np.pi / 2
    gl, gr = np.cos(p), np.sin(p)
    return np.where(pan <= 0, [x[0] + x[1] * gl, x[1] * gr], [x[0] * gl, x[1] + x[0] * gr])


@pytest.mark.parametrize("layout", ["mono", "stereo", "switch"])
def test_stereo_panner_vs_the_specification_in_many_graphs(pkg, be, layout):
    # 1000 graphs: constant pans (0 sits on the pan <= 0 branch) and an a-rate linear ramp from -1 to 1 over the render (spec 1.6.3, evaluated
    # in f32 by the param: a pan an ulp off moves the gains by 1e-7).  'switch': a mono source and a stereo burst on quanta 8-19: the input's
    # channel count changes per quantum, and silent quanta before a late start stay silent
    n = 40 * RQ
    pans = [-1.0, -0.5, 0.0, 0.5, 1.0, "ramp"]
    t = np.arange(n) / PSR

    def build():
        rng = np.random.default_rng({"mono": 31, "stereo": 32, "switch": 33}[layout])
        ctxs, wants = [], []
        for g in range(1000):
            pan = pans[g % len(pans)]
            c = pkg.OfflineAudioContext(2, n, PSR, be.backend)
            sp = c.create_stereo_panner(-1.0 if pan == "ramp" else pan)
            if pan == "ramp":
                sp.pan.linear_ramp_to_value_at_time(1.0, n / PSR)
                pv = (-1.0 + 2.0 * t / (n / PSR)).astype(F32).astype(np.float64)
            else:
                pv = np.full(n, pan)
            x = np.zeros((2, n))
            late = RQ * (g % 5)   # a late start: silent quanta first
            if layout in ("mono", "switch"):
                m = rng.uniform(-0.5, 0.5, (1, n)).astype(F32)
                s = c.create_buffer_source(pkg.AudioBuffer(list(m), PSR))
                s.connect(sp)
                s.start_at(late / PSR)
                x[:, late:] += m[0, :n - late]
            if layout in ("stereo", "switch"):
                st = rng.uniform(-0.5, 0.5, (2, n)).astype(F32)
                a, b = (8 * RQ, 20 * RQ) if layout == "switch" else (late, n)
                s = c.create_buffer_source(pkg.AudioBuffer(list(st), PSR))
                s.connect(sp)
                s.start_at(a / PSR)
                s.stop_at(b / PSR)
                x[:, a:b] += st[:, :b - a]
            sp.connect(c.destination())
            ctxs.append(c)
            if layout == "mono":
                w = _stereo_pan(pv, x[:1])
            elif layout == "stereo":
                w = _stereo_pan(pv, x)
            else:   # mono quanta are panned with the mono law, stereo quanta (the burst plays) with the stereo law
                w = np.where((np.arange(n) >= 8 * RQ) & (np.arange(n) < 20 * RQ), _stereo_pan(pv, x), _stereo_pan(pv, x[:1]))
            wants.append(w)
        return ctxs, wants

    for opts in be.variants(dict(), dict(chunk=128)):
        ctxs, wants = build()
        with be.options(**opts):
            got = _render_each(pkg, be, ctxs)
        for g in range(len(ctxs)):
            err = _pan_err(got[g], wants[g])
            assert err <= 1e-6, (layout, g, pans[g % len(pans)], opts, err)


def _check_moving(pkg, be, oracle, n_q, kinds, seed):
    """k_panner_dyn: one graph per entry of `kinds` (its input, _PanInput).  The source's position and orientation ramp linearly (spec 1.6.3,
    f32 param values) over the whole render.  While every listener param is single-valued in a quantum, the reference evaluates the spatial
    params once, at the quantum's first frame, even for a moving source (panner.rs:833-855); otherwise per frame.  Odd graphs move the
    listener too, with a ramp that ends in the middle of quantum 100: quanta up to 100 take the per-frame path, later ones the first-frame
    path."""
    n = n_q * RQ
    T = n / PSR
    t = np.arange(n) / PSR
    t_l = (100 * RQ + 64) / PSR
    rng = np.random.default_rng(seed)
    specs = [(rng.uniform(-6, 6, 3), rng.uniform(-6, 6, 3), rng.uniform(-1, 1, 3), rng.uniform(-1, 1, 3), rng.uniform(-2, 2, 3) if g % 2 else None,
              _PanInput(seed + g, n, kind)) for g, kind in enumerate(kinds)]

    def ramp(v0, v1, t1):
        return np.where(t < t1, v0 + (v1 - v0) * t / t1, v1).astype(F32).astype(np.float64)

    def build(backend):
        ctxs = []
        for p0, p1, o0, o1, l1, inp in specs:
            c = pkg.OfflineAudioContext(2, n, PSR, backend)
            p = c.create_panner(position=tuple(map(float, p0)), orientation=tuple(map(float, o0)), cone_inner_angle=60.0, cone_outer_angle=240.0,
                                cone_outer_gain=0.2, ref_distance=1.5, rolloff_factor=0.8)
            for prm, v in zip([p.position_x, p.position_y, p.position_z, p.orientation_x, p.orientation_y, p.orientation_z], list(p1) + list(o1)):
                prm.linear_ramp_to_value_at_time(float(v), T)
            if l1 is not None:
                lis = c.listener()
                for k, prm in enumerate([lis.position_x, lis.position_y, lis.position_z]):
                    prm.linear_ramp_to_value_at_time(float(l1[k]), t_l)
            inp.connect(pkg, c, p)
            p.connect(c.destination())
            ctxs.append(c)
        return ctxs

    wants = []
    for p0, p1, o0, o1, l1, inp in specs:
        src = np.stack([ramp(float(F32(a)), float(F32(b)), T) for a, b in zip(p0, p1)], -1)
        ori = np.stack([ramp(float(F32(a)), float(F32(b)), T) for a, b in zip(o0, o1)], -1)
        lp = np.zeros((n, 3)) if l1 is None else np.stack([ramp(0.0, float(F32(v)), t_l) for v in l1], -1)
        per_frame = np.zeros(n, bool) if l1 is None else np.repeat(np.arange(n_q) <= 100, RQ)
        idx = np.where(per_frame, np.arange(n), np.repeat(np.arange(n_q) * RQ, RQ))   # the frame whose spatial params a frame is panned with
        fwd, up = np.tile([0.0, 0.0, -1.0], (n, 1)), np.tile([0.0, 1.0, 0.0], (n, 1))
        az, gain, args = _spatial(src[idx], ori[idx], lp[idx], fwd, up, "inverse", 1.5, 10000.0, 0.8, 60.0, 240.0, 0.2)
        ill = np.max(np.abs(args), axis=0) >= 1 - 1e-3
        wants.append(inp.want(az, gain) + (ill,))
    ref = _render_each(pkg, _Backend(pkg, "oracle", oracle), build(oracle)) if be.is_engine else None
    for opts in be.variants(dict(), dict(chunk=128)):
        with be.options(**opts):
            got = _render_each(pkg, be, build(be.backend))
        for g, (want, silent, ill) in enumerate(wants):   # frame by frame: the frames near an acos singularity as in _assert_pan
            _assert_pan(got[g][:, ~ill], want[:, ~ill], silent[~ill], False, None, (g, opts))
            if ill.any():
                _assert_pan(got[g][:, ill], want[:, ill], silent[ill], True, None if ref is None else ref[g][:, ill], (g, opts))


def test_equal_power_panner_moving_source_and_listener(pkg, be, oracle):
    # 96 graphs of 4 s at 32768 Hz (the f64 witness evaluates every frame of every graph: 12.6 M poses keep its CPU time near 20 s); mono and
    # stereo inputs each with a static and a moving listener
    _check_moving(pkg, be, oracle, 4 * 256, [("mono", "mono", "stereo", "stereo")[g % 4] for g in range(96)], 41)


@pytest.mark.parametrize("poses", ["static", "moving"])
def test_equal_power_panner_input_that_changes_layout(pkg, be, oracle, poses):
    # a late mono source that stops early, with a stereo burst inside it: each quantum takes the mono or the stereo law by its own layout,
    # and the silent quanta before and after come out silent.  Static poses: k_panner_eq (random and edge poses); moving: k_panner_dyn
    n_q = 200
    if poses == "moving":
        _check_moving(pkg, be, oracle, n_q, ["switch"] * 64, 51)
        return
    n = n_q * RQ
    ps = _pose_lists(np.random.default_rng(61), 300)
    inps = [_PanInput(3000 + g, n, "switch") for g in range(len(ps))]
    assert all(set(i.lay) == {0, 1, 2} for i in inps)

    def render(pp, backend=None):
        return _render_each(pkg, _Backend(pkg, "oracle", backend) if backend else be,
                            [_pose_graph(pkg, backend or be.backend, p, inps[i], n)[0] for i, p in enumerate(pp)])
    for opts in be.variants(dict(), dict(chunk=128)):
        with be.options(**opts):
            _check_static(pkg, be, oracle, ps, inps, n, render)
