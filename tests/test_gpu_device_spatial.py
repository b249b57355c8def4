"""PannerNode positions / orientations and the AudioListener's pose bound from device memory (wae_param_set_device_value +
wae_batch_bind_params) on the GPU.  Every case renders three ways: bound from a torch tensor, host-built with the same values, and on
the oracle; every render is within 1e-5 of the oracle.  The bound render runs the spatial math on the device (acosf, sinf / cosf, pow),
so it is not promised bit-equality with its host twin: near a face of the sphere the device may pick the neighbouring triangle.  The
cases print how far each bound render is from its twin, and the bit-equal ones are counted."""
import numpy as np
import pytest

import graphs as G

pytestmark = pytest.mark.gpu
TOL = 1e-5
SR = 48000.0
LENGTH = 9600
EQ, HRTF = 0, 1
BIT_EQUAL = {"equal": 0, "all": 0}

# the bindable spatial params: ("p", i) panner param i (position xyz, orientation xyz), ("l", i) listener param i (position, forward, up)
SOURCE = [("p", 0), ("p", 1), ("p", 2)]
LISTENER_FWD = [("l", 3), ("l", 4), ("l", 5)]
PANNER_NAMES = ["position_x", "position_y", "position_z", "orientation_x", "orientation_y", "orientation_z"]
LISTENER_NAMES = ["position_x", "position_y", "position_z", "forward_x", "forward_y", "forward_z", "up_x", "up_y", "up_z"]
PANNER_DEFAULTS = [0.0, 0.0, 0.0, 1.0, 0.0, 0.0]
LISTENER_DEFAULTS = [0.0, 0.0, 0.0, 0.0, 0.0, -1.0, 0.0, 1.0, 0.0]
RANGE = (-20.0, 20.0)


def set_sphere(engine, oracle, rate=int(SR), taps=256):
    data = G.synthetic_hrir_sphere(rate, taps)
    oracle.set_hrir_sphere(data)
    engine.backend.set_hrir_sphere(data)


def run(batch):
    batch.set_timing(True)
    batch.run()
    batch.sync()
    return batch.fetch()


def maxdiff(a, b):
    return float(np.abs(a.astype(np.float64) - b.astype(np.float64)).max())


def stage_names(batch):
    return sorted((name, k) for name, _t, k in batch.stage_times())


def target(c, pns, key, k=0):
    kind, i = key
    return getattr(pns[k], PANNER_NAMES[i]) if kind == "p" else getattr(c.listener(), LISTENER_NAMES[i])


def clamp(v, default):
    return default if not np.isfinite(v) else min(max(float(np.float32(v)), RANGE[0]), RANGE[1])


def host_values(row, spec):
    """the values a bind gives: clamped to RANGE, a non-finite value -> the param's default"""
    out = []
    for (kind, i), v in zip(spec["bind"], row):
        out.append(clamp(v, (PANNER_DEFAULTS if kind == "p" else LISTENER_DEFAULTS)[i]))
    return out


def make(pkg, be, spec, row, declare):
    """spec["src"] ("mono" oscillator, "stereo": oscillator -> StereoPannerNode) -> PannerNode (spec["panners"] of them, sharing the
    listener) -> destination.  `row`: the values of spec["bind"]; `declare`: those params declared over RANGE (planned at a
    placeholder), else the host twin sets them."""
    c = pkg.OfflineAudioContext(2, LENGTH, SR, be)
    pns = []
    for k in range(spec.get("panners", 1)):
        osc = c.create_oscillator(type_=pkg.SAWTOOTH, frequency=220.0 * (k + 1))
        last = osc
        if spec.get("src") == "stereo":
            sp = c.create_stereo_panner(pan=0.3)
            osc.connect(sp)
            last = sp
        cone = spec.get("cone", (360.0, 360.0))
        pn = c.create_panner(panning_model=spec.get("model", HRTF), distance_model=spec.get("distance", 1),
                             position=spec.get("pos", (1.0, 0.5, -2.0)), orientation=spec.get("orient", (1.0, 0.0, 0.0)),
                             ref_distance=1.0, max_distance=50.0, rolloff_factor=spec.get("rolloff", 1.0),
                             cone_inner_angle=cone[0], cone_outer_angle=cone[1], cone_outer_gain=0.3)
        last.connect(pn)
        pn.connect(c.destination())
        osc.start_at(spec.get("start", 0.0))
        pns.append(pn)
    for i, v in spec.get("listener", {}).items():
        getattr(c.listener(), LISTENER_NAMES[i]).set_value(v)
    if spec.get("moving"):  # another spatial param automated: k_panner_dyn / k_hrtf_sel
        pns[0].orientation_z.linear_ramp_to_value_at_time(0.5, 0.1)
    for key, v in zip(spec["bind"], row):
        for k in range(len(pns) if key[0] == "p" else 1):
            p = target(c, pns, key, k)
            if declare:
                p.set_value(3.0 if key[0] == "p" else 0.5)  # (any placeholder: the bound value replaces it)
                p.set_device_value(*RANGE)
            else:
                p.set_value(v)
    if spec.get("suspend"):
        c.suspend_sync(4096 / SR, lambda ctx: None)
    return c, pns


def render_three(pkg, engine, oracle, spec, rows, chunk=0, expect=None):
    torch = pytest.importorskip("torch")
    engine.set_option(pkg.OPT_CHUNK_FRAMES, chunk)
    try:
        made = [make(pkg, engine.backend, spec, r, True) for r in rows]
        b = pkg.Batch([c for c, _ in made])
        tw = pkg.Batch([make(pkg, engine.backend, spec, host_values(r, spec), False)[0] for r in rows])
    finally:
        engine.set_option(pkg.OPT_CHUNK_FRAMES, 0)
    c0, pns0 = made[0]
    params = [target(c0, pns0, key) for key in spec["bind"]]
    try:
        b.bind_params(params, torch.tensor(np.array(rows, np.float32)).cuda())
        got = run(b)
        twin = run(tw)
        stages = (stage_names(b), stage_names(tw))
    finally:
        b.destroy()
        tw.destroy()
    want = np.stack([np.stack(x.channels) for x in
                     pkg.render_batch([make(pkg, oracle, spec, host_values(r, spec), False)[0] for r in rows])])
    assert np.isfinite(got).all()
    assert maxdiff(twin, want) <= TOL
    assert maxdiff(got, want) <= TOL, (spec, maxdiff(got, want))
    assert stages[0] == stages[1], stages
    if expect:
        names = {n for n, _ in stages[0]}
        assert expect in names, (expect, names)
    for g in range(len(rows)):
        BIT_EQUAL["all"] += 1
        BIT_EQUAL["equal"] += int(np.array_equal(got[g], twin[g]))
    print(f"{spec}: max |bound - twin| = {maxdiff(got, twin):.3e}, max |bound - oracle| = {maxdiff(got, want):.3e}, "
          f"bit-equal renders so far {BIT_EQUAL['equal']} / {BIT_EQUAL['all']}")
    return got, twin


def directions(n, seed, with_forward=True):
    """rows of (source x, y, z[, listener forward x, y, z]) around the listener at 0.5 .. 8 m"""
    rng = np.random.default_rng(seed)
    rows = []
    for _ in range(n):
        az, el, d = rng.uniform(0, 2 * np.pi), rng.uniform(-1.2, 1.2), rng.uniform(0.5, 8.0)
        r = [d * np.sin(az) * np.cos(el), d * np.sin(el), -d * np.cos(az) * np.cos(el)]
        if with_forward:
            fa = rng.uniform(-np.pi, np.pi)
            r += [np.sin(fa), 0.0, -np.cos(fa)]
        rows.append(r)
    return rows


# ---- the five paths ---------------------------------------------------------------------------------------------------------------
PATHS = {
    "eq_static": (dict(model=EQ), "k_panner_eq"),
    "eq_moving": (dict(model=EQ, moving=True), "k_panner_dyn"),
    "hrtf_moving": (dict(moving=True), "k_hrtf_fir"),
    "hrtf_fir": (dict(start=0.0123), "k_hrtf_fir"),  # a late start: the input's layout changes
    "hrtf_conv": (dict(), "k_conv_fft_in"),
}


@pytest.mark.parametrize("path", list(PATHS))
@pytest.mark.parametrize("src", ["mono", "stereo"])
def test_paths(pkg, engine, oracle, path, src):
    set_sphere(engine, oracle)
    spec, kernel = PATHS[path]
    spec = dict(spec, src=src, bind=SOURCE + LISTENER_FWD)
    render_three(pkg, engine, oracle, spec, directions(5, 11), expect=kernel)


@pytest.mark.parametrize("path", ["hrtf_conv", "hrtf_fir"])
def test_resampled_sphere(pkg, engine, oracle, path):
    set_sphere(engine, oracle, rate=44100)  # resampled to the context's 48 kHz
    spec, kernel = PATHS[path]
    render_three(pkg, engine, oracle, dict(spec, bind=SOURCE + LISTENER_FWD), directions(4, 12), expect=kernel)


@pytest.mark.parametrize("which", ["source", "listener"])
@pytest.mark.parametrize("path", ["eq_static", "hrtf_conv"])
def test_source_only_or_listener_only(pkg, engine, oracle, which, path):
    set_sphere(engine, oracle)
    spec, _ = PATHS[path]
    if which == "source":
        render_three(pkg, engine, oracle, dict(spec, bind=SOURCE), directions(4, 13, with_forward=False))
    else:
        rows = [r[3:] for r in directions(4, 14)]
        render_three(pkg, engine, oracle, dict(spec, bind=LISTENER_FWD), rows)


@pytest.mark.parametrize("distance", [0, 1, 2])
@pytest.mark.parametrize("path", ["eq_static", "hrtf_fir"])
def test_distance_models(pkg, engine, oracle, distance, path):
    set_sphere(engine, oracle)
    spec, _ = PATHS[path]
    render_three(pkg, engine, oracle, dict(spec, distance=distance, rolloff=0.8, bind=SOURCE + LISTENER_FWD), directions(4, 15))


@pytest.mark.parametrize("path", ["eq_static", "hrtf_conv"])
def test_cone_with_bound_orientation(pkg, engine, oracle, path):
    set_sphere(engine, oracle)
    spec, _ = PATHS[path]
    rows = [[2.0, 0.0, -1.0, np.cos(a), 0.0, np.sin(a)] for a in np.linspace(0, 2 * np.pi, 6, endpoint=False)]
    render_three(pkg, engine, oracle, dict(spec, cone=(60.0, 200.0), bind=SOURCE + [("p", 3), ("p", 4), ("p", 5)]), rows)


@pytest.mark.parametrize("path", ["eq_static", "hrtf_conv", "hrtf_fir"])
def test_degenerate_poses(pkg, engine, oracle, path):
    set_sphere(engine, oracle)
    spec, _ = PATHS[path]
    bind = SOURCE + LISTENER_FWD + [("l", 6), ("l", 7), ("l", 8)]
    rows = [[0.0, 0.0, 0.0, 0.0, 0.0, -1.0, 0.0, 1.0, 0.0],   # the source at the listener's position
            [1.0, 2.0, -3.0, 0.0, 1.0, 0.0, 0.0, 1.0, 0.0],   # forward parallel to up
            [1.0, 2.0, -3.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0]]   # a zero forward
    render_three(pkg, engine, oracle, dict(spec, bind=bind), rows)


@pytest.mark.parametrize("path", ["eq_static", "hrtf_conv"])
def test_two_panners_share_one_bound_listener(pkg, engine, oracle, path):
    set_sphere(engine, oracle)
    spec, _ = PATHS[path]
    rows = [r[3:] for r in directions(4, 16)]
    render_three(pkg, engine, oracle, dict(spec, panners=2, bind=LISTENER_FWD), rows)


@pytest.mark.parametrize("path", ["eq_static", "hrtf_fir"])
def test_suspend_point_after_the_declaration(pkg, engine, oracle, path):
    set_sphere(engine, oracle)
    spec, _ = PATHS[path]
    render_three(pkg, engine, oracle, dict(spec, suspend=True, bind=SOURCE + LISTENER_FWD), directions(3, 17))


@pytest.mark.parametrize("chunk", [128, 1024, 0])
@pytest.mark.parametrize("path", ["hrtf_conv", "hrtf_moving"])
def test_chunks(pkg, engine, oracle, chunk, path):
    set_sphere(engine, oracle)
    spec, _ = PATHS[path]
    render_three(pkg, engine, oracle, dict(spec, bind=SOURCE + LISTENER_FWD), directions(3, 18), chunk=chunk)


@pytest.mark.parametrize("path", ["eq_static", "hrtf_conv", "hrtf_moving"])
def test_clamped_and_non_finite_values(pkg, engine, oracle, path):
    set_sphere(engine, oracle)
    spec, _ = PATHS[path]
    rows = [[100.0, -1e30, 5.0, np.nan, 0.0, -1.0],
            [np.inf, 1.0, -np.inf, 0.5, np.nan, np.nan],
            [-25.0, 0.0, 30.0, 1.0, 0.0, 0.0]]
    render_three(pkg, engine, oracle, dict(spec, bind=SOURCE + LISTENER_FWD), rows)


# ---- the bind contract ------------------------------------------------------------------------------------------------------------
def test_rebinding_a_b_a_renders_a_again(pkg, engine, oracle):
    torch = pytest.importorskip("torch")
    set_sphere(engine, oracle)
    spec = dict(bind=SOURCE + LISTENER_FWD)
    rows_a, rows_b = directions(4, 19), directions(4, 20)
    made = [make(pkg, engine.backend, spec, r, True) for r in rows_a]
    b = pkg.Batch([c for c, _ in made])
    params = [target(made[0][0], made[0][1], key) for key in spec["bind"]]
    try:
        b.bind_params(params, torch.tensor(np.array(rows_a, np.float32)).cuda())
        a1 = run(b).copy()
        b.bind_params(params, torch.tensor(np.array(rows_b, np.float32)).cuda())
        bb = run(b).copy()
        b.bind_params(params, torch.tensor(np.array(rows_a, np.float32)).cuda())
        a2 = run(b)
    finally:
        b.destroy()
    assert np.array_equal(a1, a2)
    assert not np.array_equal(a1, bb)


def test_runs_and_one_shot_renders_are_refused_until_the_bind(pkg, engine, oracle):
    torch = pytest.importorskip("torch")
    set_sphere(engine, oracle)
    spec = dict(bind=SOURCE)
    made = [make(pkg, engine.backend, spec, r, True) for r in directions(2, 21, with_forward=False)]
    b = pkg.Batch([c for c, _ in made])
    try:
        with pytest.raises(Exception) as e:
            b.run()
        assert e.value.status == 2 and "wae_batch_bind_params" in str(e.value)
        b.bind_params([made[0][1][0].position_x], torch.zeros(2, device="cuda"))  # one of three: still refused
        with pytest.raises(Exception) as e:
            b.run()
        assert e.value.status == 2
    finally:
        b.destroy()
    with pytest.raises(Exception) as e:
        pkg.render_batch([make(pkg, engine.backend, spec, [1.0, 2.0, 3.0], True)[0]])
    assert e.value.status == 2


def test_listener_without_panner_is_validated_and_reaches_nothing(pkg, engine, oracle):
    torch = pytest.importorskip("torch")

    def graph(declare):
        c = pkg.OfflineAudioContext(1, LENGTH, SR, engine.backend)
        osc = c.create_oscillator(frequency=330.0)
        osc.connect(c.destination())
        osc.start()
        if declare:
            c.listener().forward_x.set_device_value(-1.0, 1.0)
        return c
    c = graph(True)
    b = pkg.Batch([c])
    tw = pkg.Batch([graph(False)])
    try:
        with pytest.raises(Exception) as e:  # runs still wait for it
            b.run()
        assert e.value.status == 2
        with pytest.raises(Exception) as e:  # validated: an undeclared listener param is refused
            b.bind_params([c.listener().forward_y], torch.zeros(1, device="cuda"))
        assert e.value.status == 2
        b.bind_params([c.listener().forward_x], torch.full((1,), 0.7, device="cuda"))
        got, want = run(b), run(tw)
    finally:
        b.destroy()
        tw.destroy()
    assert np.array_equal(got, want)


@pytest.mark.parametrize("path", ["hrtf_conv", "hrtf_fir"])
def test_bind_after_the_sphere_was_replaced_is_refused(pkg, engine, oracle, path):
    torch = pytest.importorskip("torch")
    set_sphere(engine, oracle)
    spec, _ = PATHS[path]
    spec = dict(spec, bind=SOURCE)
    made = [make(pkg, engine.backend, spec, r, True) for r in directions(2, 22, with_forward=False)]
    b = pkg.Batch([c for c, _ in made])
    params = [target(made[0][0], made[0][1], key) for key in spec["bind"]]
    try:
        values = torch.ones(2, 3, device="cuda")
        b.bind_params(params, values)  # (bound once: the refusal below is the sphere's, not the declarations')
        engine.backend.set_hrir_sphere(G.synthetic_hrir_sphere(int(SR), 256, seed=6))
        with pytest.raises(Exception) as e:
            b.bind_params(params, values)
        assert e.value.status == 2 and "wae_engine_set_hrir_sphere" in str(e.value)
    finally:
        b.destroy()  # (never run against the freed sphere)
    set_sphere(engine, oracle)


def test_equal_power_batches_ignore_the_sphere(pkg, engine, oracle):
    torch = pytest.importorskip("torch")
    set_sphere(engine, oracle)
    spec = dict(model=EQ, bind=SOURCE)
    made = [make(pkg, engine.backend, spec, r, True) for r in directions(2, 23, with_forward=False)]
    b = pkg.Batch([c for c, _ in made])
    params = [target(made[0][0], made[0][1], key) for key in spec["bind"]]
    try:
        set_sphere(engine, oracle)
        b.bind_params(params, torch.ones(2, 3, device="cuda"))
        run(b)
    finally:
        b.destroy()
