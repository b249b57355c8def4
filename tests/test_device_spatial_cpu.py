"""PannerNode positions / orientations and the AudioListener's pose bound from device memory, on the host (no GPU): the declaration rules
of wae_param_set_device_value applied to panner params 0..5 and listener params 0..8 (node 1, created on declaration), the spatial
bound (ranges beyond +-1e9 refused), listener value
curves still refused, one-shot renders refused, and plans (stages and plan digests) equal to host twins at the placeholder on the two
equal-power paths (static: k_panner_eq, moving because another spatial param is automated: k_panner_dyn).  The host-only planner has
no HRIR sphere, so the three HRTF paths are compared with their twins on the GPU (tests/test_gpu_device_spatial.py)."""
import os
import subprocess
import sys
import textwrap

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "web-audio-api-rs_b200", "libwae_b200.so")
SR = 48000.0


@pytest.fixture
def host(pkg):
    if not os.path.exists(LIB):
        pytest.skip("libwae_b200.so is not built (python -c 'import __graft_entry__ as g; g.build()')")
    return pkg.context.Backend(pkg.api(), None)


def status_of(fn):
    with pytest.raises(Exception) as e:
        fn()
    return e.value.status


def panner_ctx(pkg, host, position=(1.0, 0.5, -2.0)):
    c = pkg.OfflineAudioContext(2, 4096, SR, host)
    osc = c.create_oscillator(frequency=330.0)
    pn = c.create_panner(position=position)
    osc.connect(pn)
    pn.connect(c.destination())
    osc.start()
    return c, pn


PANNER_PARAMS = ["position_x", "position_y", "position_z", "orientation_x", "orientation_y", "orientation_z"]
LISTENER_PARAMS = ["position_x", "position_y", "position_z", "forward_x", "forward_y", "forward_z", "up_x", "up_y", "up_z"]


# ---- declarations -----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", PANNER_PARAMS)
def test_panner_params_are_accepted(pkg, host, name):
    c, pn = panner_ctx(pkg, host)
    getattr(pn, name).set_device_value(-10.0, 10.0)
    pkg.plan_batch([c])


@pytest.mark.parametrize("name", LISTENER_PARAMS)
def test_listener_params_are_accepted_and_create_the_listener(pkg, host, name):
    c = pkg.OfflineAudioContext(2, 4096, SR, host)  # no listener yet: the declaration creates it
    getattr(c.listener(), name).set_device_value(-1.0, 1.0)
    pkg.plan_batch([c])  # (a listener without panners plans)


def test_one_shot_renders_refuse_declared_graphs(pkg, host):
    import ctypes
    import numpy as np
    api = pkg.api()
    c1, pn = panner_ctx(pkg, host)
    pn.position_z.set_device_value(-10.0, 10.0)
    c2 = pkg.OfflineAudioContext(2, 4096, SR, host)  # a declared listener without a panner counts too
    c2.listener().up_y.set_device_value(-1.0, 1.0)
    for c in (c1, c2):
        arr = (ctypes.c_void_p * 1)(c._g)
        out = np.zeros((1, 2, 4096), np.float32)
        assert api.render_batch(None, arr, 1, out.ctypes.data_as(ctypes.c_void_p), 0) == 2
        assert b"wae_batch_bind_params" in api.last_error()


def test_generic_rules_apply_to_spatial_params(pkg, host):
    c, pn = panner_ctx(pkg, host)
    for lo, hi in ((1.0, -1.0), (float("nan"), 1.0), (0.0, float("inf"))):
        assert status_of(lambda: pn.position_x.set_device_value(lo, hi)) == 1, (lo, hi)
        assert status_of(lambda: c.listener().up_y.set_device_value(lo, hi)) == 1, (lo, hi)
    pn.position_x.set_device_value(-5.0, 5.0)
    assert status_of(lambda: pn.position_x.set_device_value(-5.0, 5.0)) == 2  # declared twice
    assert status_of(lambda: pn.position_x.set_value(1.0)) == 2  # no events after
    assert status_of(lambda: pn.position_x.linear_ramp_to_value_at_time(1.0, 0.01)) == 2
    lfo = c.create_oscillator(frequency=2.0)
    assert status_of(lambda: lfo.connect(pn.position_x)) == 2  # no audio-rate input after
    c.listener().forward_x.set_device_value(-1.0, 1.0)
    assert status_of(lambda: c.listener().forward_x.set_value(0.5)) == 2  # wae_listener_param_event_push goes through the same rule
    assert status_of(lambda: c.listener().forward_x.set_value_at_time(0.5, 0.01)) == 2
    assert status_of(lambda: lfo.connect(c.listener().forward_x)) == 2
    assert status_of(lambda: c.listener().forward_x.set_device_value(-1.0, 1.0)) == 2
    c, pn = panner_ctx(pkg, host)
    pn.position_y.set_value_at_time(1.0, 0.01)
    assert status_of(lambda: pn.position_y.set_device_value(-5.0, 5.0)) == 2  # events before
    c.listener().up_x.set_value_at_time(0.1, 0.01)
    assert status_of(lambda: c.listener().up_x.set_device_value(-1.0, 1.0)) == 2
    c, pn = panner_ctx(pkg, host)
    lfo = c.create_oscillator(frequency=2.0)
    lfo.connect(c.listener().position_z)
    assert status_of(lambda: c.listener().position_z.set_device_value(-1.0, 1.0)) == 2  # an audio-rate input


@pytest.mark.parametrize("lo,hi", [(None, None), (-1e10, 0.0), (0.0, 1.5e9), (-3e38, 3e38)])
def test_ranges_beyond_the_spatial_bound_are_refused(pkg, host, lo, hi):
    # the f32 spatial math squares differences and cross products: values beyond +-1e9 overflow, so such ranges answer WAE_UNSUPPORTED
    c, pn = panner_ctx(pkg, host)
    for p in (pn.position_x, pn.orientation_z, c.listener().position_y, c.listener().up_x):
        assert status_of(lambda: p.set_device_value(lo, hi)) == 4
    for p in (pn.position_x, pn.orientation_z, c.listener().position_y, c.listener().up_x):
        p.set_device_value(-1e9, 1e9)  # (the failed calls declared nothing; the bound itself is inside)


def test_listener_param_index_out_of_range(pkg, host):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    assert pkg.api().param_set_device_value(c._g, 1, 9, 0.0, 1.0) == 1  # the listener has params 0..8


def test_listener_value_curves_stay_refused(pkg, host):
    c, _ = panner_ctx(pkg, host)
    assert status_of(lambda: c.listener().position_x.set_device_value_curve(2, 0.0, 0.01)) == 1
    api = host.api
    assert api.param_set_device_value_curve(c._g, 1, 0, 2, 0.0, 0.01) == 1  # the C entry point itself


def test_declaration_after_a_suspend_point(pkg, host):
    c, pn = panner_ctx(pkg, host)
    c.suspend_sync(1024 / SR, lambda ctx: c.listener().forward_x.set_device_value(-1.0, 1.0))
    assert status_of(lambda: pkg.plan_batch([c])) == 2


# ---- plans equal to host twins ----------------------------------------------------------------------------------------------------
def spatial_graph(pkg, backend, case, declare):
    """One panner (or two sharing the listener) at the case's position and listener pose.  `declare`: case["bind"] ("source", "listener"
    or "both") declared over ranges that hold the host twin's values, so the placeholder is the twin's value."""
    c = pkg.OfflineAudioContext(2, 4800, SR, backend)
    pos = case.get("pos", (2.0, 0.5, -1.0))
    fwd = case.get("fwd", (0.3, 0.0, -1.0))
    panners = []
    for k in range(case.get("panners", 1)):
        src = c.create_oscillator(frequency=220.0 * (k + 1))
        pn = c.create_panner(panning_model=case.get("model", pkg.context.EQUALPOWER), distance_model=case.get("distance", 1),
                             position=tuple(p + k for p in pos), orientation=case.get("orient", (1.0, 0.0, 0.0)),
                             cone_inner_angle=case.get("cone", (360.0, 360.0))[0], cone_outer_angle=case.get("cone", (360.0, 360.0))[1],
                             cone_outer_gain=0.25)
        src.connect(pn)
        pn.connect(c.destination())
        src.start_at(case.get("start", 0.0))
        panners.append(pn)
    lis = c.listener()
    for name, v in zip(("forward_x", "forward_y", "forward_z"), fwd):
        getattr(lis, name).set_value(v)
    if case.get("moving"):  # another spatial param automated: the moving paths
        panners[0].orientation_y.linear_ramp_to_value_at_time(0.5, 0.05)
    if declare:
        bind = case.get("bind", "both")
        for pn in panners:
            if bind in ("source", "both"):
                for name in ("position_x", "position_y", "position_z"):
                    getattr(pn, name).set_device_value(-50.0, 50.0)
            if case.get("cone") and bind in ("source", "both"):
                pn.orientation_x.set_device_value(-1.0, 1.0)
        if bind in ("listener", "both"):
            for name in ("forward_x", "forward_y", "forward_z"):
                getattr(lis, name).set_device_value(-1.0, 1.0)
    return c


DIGEST_CASES = {
    "static_source": dict(bind="source"),
    "static_listener": dict(bind="listener"),
    "static_both_linear": dict(distance=0),
    "static_both_exponential_cone": dict(distance=2, cone=(60.0, 180.0)),
    "static_two_panners": dict(panners=2),
    "moving_source": dict(moving=True, bind="source"),
    "moving_both": dict(moving=True),
}


def plan_digests(declare, env=None):
    script = textwrap.dedent(f"""
        import sys
        sys.path.insert(0, {os.path.join(ROOT, 'tests')!r}); sys.path.insert(0, {ROOT!r})
        from conftest import load_package
        import test_device_spatial_cpu as T
        pkg = load_package()
        be = pkg.context.Backend(pkg.api(), None)
        for name, case in T.DIGEST_CASES.items():
            sys.stderr.write("case " + name + "\\n")
            p = pkg.plan_batch([T.spatial_graph(pkg, be, case, {declare!r}) for _ in range(2)])
            sys.stderr.write("kinds " + repr(sorted(p["kinds"].items())) + "\\n")
            sys.stderr.write("stages " + repr(p["stages"]) + "\\n")
    """)
    r = subprocess.run([sys.executable, "-c", script], env=dict(os.environ, WAE_PLAN_DIGEST="1", **(env or {})), capture_output=True,
                       text=True, check=True)
    got, name = {}, None
    for line in r.stderr.splitlines():
        if line.startswith("case "):
            name = line[5:]
            got[name] = []
        elif line.startswith(("kinds ", "stages ")):
            got[name].append(line)
        elif "[wae plan digest]" in line:
            got[name].append(line.rsplit(": ", 1)[1])
    return got


@pytest.mark.parametrize("env", [{}, {"WAE_PLAN_PARALLEL": "1"}])
def test_declared_plans_equal_host_twins(pkg, host, env):
    declared, twins = plan_digests(True, env), plan_digests(False, env)
    assert set(declared) == set(DIGEST_CASES)
    assert declared == twins
    kinds = {name: dict(eval(next(x for x in lines if x.startswith("kinds "))[6:])) for name, lines in declared.items()}
    for name in DIGEST_CASES:
        want = "k_panner_dyn" if DIGEST_CASES[name].get("moving") else "k_panner_eq"
        assert kinds[name].get(want), (name, kinds[name])
