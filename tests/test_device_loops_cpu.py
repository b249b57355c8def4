"""AudioBufferSourceNode loop points bound from device memory (wae_buffer_source_set_device_loop), on the host (no GPU): the declaration
rules, the playback path and output layout the planner picks from the declared windows and rates, plans of graphs without declarations
unchanged, and the shared playhead walk (absn_loop_segments) against a frame-by-frame replay of the reference's loop bookkeeping."""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "web-audio-api-rs_b200", "libwae_b200.so")
SR = 48000.0
F64_MAX = 1.7976931348623157e308
BOUND = "k_buffer_source_slow(bound)"
SERIAL = "k_buffer_source_serial"


@pytest.fixture
def host(pkg):
    if not os.path.exists(LIB):
        pytest.skip("libwae_b200.so is not built (python -c 'import __graft_entry__ as g; g.build()')")
    return pkg.context.Backend(pkg.api(), None)


def status_of(fn):
    with pytest.raises(Exception) as e:
        fn()
    return e.value.status


def loop_graph(pkg, backend, start=(0.1, 0.3), end=(0.8, 1.2), rate=1.0, rng=None, det=None, automate_detune=False, frames=72000,
               length=96000, when=0.0, stop=None, duration=None, schedule=False, biquad=True, declare=True, loop_points=None):
    """1.5 s clip -> looping source (loop points declared over `start` / `end`, or host-built at `loop_points`) -> [lowpass] -> destination"""
    c = pkg.OfflineAudioContext(2, length, SR, backend)
    pcm = np.random.default_rng(frames).uniform(-0.5, 0.5, (2, frames)).astype(np.float32)
    ls, le = loop_points if loop_points is not None else (start[0], end[0])
    s = c.create_buffer_source(pkg.AudioBuffer(list(pcm), SR), playback_rate=rate, loop=True)
    s.set_loop_start(ls)
    s.set_loop_end(le)
    if rng is not None:
        s.playback_rate.set_device_value(*rng)
    if det is not None:
        s.detune.set_device_value(*det)
    if automate_detune:
        s.detune.linear_ramp_to_value_at_time(100.0, 0.5)
    last = s
    if biquad:
        bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=1000.0)
        s.connect(bq)
        last = bq
    last.connect(c.destination())
    s.start_at_with_offset_and_duration(when, 0.0, F64_MAX if duration is None else duration)
    if stop is not None:
        s.stop_at(stop)
    if schedule:
        s.set_device_schedule((when, when + 0.1))
    if declare:
        s.set_device_loop(start, end)
    return c


def kinds(pkg, c):
    return pkg.plan_batch([c])["kinds"]


def test_declaration_rules(pkg, host):
    api = pkg.api()
    c = pkg.OfflineAudioContext(1, 4096, SR, host)
    s = c.create_buffer_source(pkg.AudioBuffer.zeros(1, 4800, SR))
    s.connect(c.destination())
    assert api.buffer_source_set_device_loop(c._g, s.id, 0.0, 0.01, 0.05, 0.08) == 2  # loop is false
    s.set_loop(True)
    osc = c.create_oscillator()
    assert api.buffer_source_set_device_loop(c._g, osc.id, 0.0, 0.01, 0.05, 0.08) == 1  # not a buffer source
    assert api.buffer_source_set_device_loop(c._g, 12345, 0.0, 0.01, 0.05, 0.08) == 1  # unknown node
    for lo, hi in ((0.02, 0.01), (-0.01, 0.05), (0.0, float("inf")), (float("nan"), 1.0)):
        assert api.buffer_source_set_device_loop(c._g, s.id, lo, hi, 0.05, 0.08) == 1, (lo, hi)
        assert api.buffer_source_set_device_loop(c._g, s.id, 0.0, 0.01, lo, hi) == 1, (lo, hi)
    assert api.buffer_source_set_device_loop(c._g, s.id, 0.0, 0.01, 0.05, 0.08) == 0
    assert api.buffer_source_set_device_loop(c._g, s.id, 0.0, 0.01, 0.05, 0.08) == 2  # declared twice
    for setter in (lambda: s.set_loop(False), lambda: s.set_loop_start(0.0), lambda: s.set_loop_end(0.1)):
        assert status_of(setter) == 2
    assert api.graph_suspend(c._g, 1024 / SR) == 2
    assert c._device_loops == set()  # (declared through the C ABI, not the Python method)


def test_declaration_in_graph_with_suspend_point(pkg, host):
    c = pkg.OfflineAudioContext(1, 4096, SR, host)
    s = c.create_buffer_source(pkg.AudioBuffer.zeros(1, 4800, SR), loop=True)
    s.connect(c.destination())
    s.start()
    assert pkg.api().graph_suspend(c._g, 1024 / SR) == 0
    assert status_of(lambda: s.set_device_loop((0.0, 0.01), (0.05, 0.08))) == 2


def test_python_declaration(pkg, host):
    c = pkg.OfflineAudioContext(1, 4096, SR, host)
    s = c.create_buffer_source(pkg.AudioBuffer.zeros(1, 4800, SR), loop=True)
    assert status_of(lambda: s.set_device_loop((0.5, 0.1), (0.05, 0.08))) == 1
    assert s.set_device_loop((0.0, 0.01), (0.05, 0.08)) is s
    assert c._device_loops == {s.id}


PATHS = {
    "constant_rate": (dict(), BOUND),
    "rate_range": (dict(rng=(0.9, 1.1)), BOUND),
    "rate_detune": (dict(rng=(0.5, 2.0), det=(-100.0, 100.0)), BOUND),
    "schedule": (dict(rng=(0.9, 1.1), schedule=True), BOUND),
    "one_point_windows": (dict(start=(0.2, 0.2), end=(1.0, 1.0), rng=(0.9, 1.1)), BOUND),
    "overlapping_windows": (dict(start=(0.1, 0.9), end=(0.8, 1.2)), SERIAL),
    "end_window_from_zero": (dict(start=(0.0, 0.0), end=(0.0, 1.0)), SERIAL),
    "range_to_zero": (dict(rng=(0.0, 1.0)), SERIAL),
    "negative_rate": (dict(rate=-1.0), SERIAL),
    "automated_detune": (dict(rng=(0.9, 1.1), automate_detune=True), SERIAL),
    "tiny_rate": (dict(rng=(1e-4, 1.0)), SERIAL),  # a step narrower than a loop point's snap zone
    "short_loop": (dict(start=(0.0, 0.0), end=(1e-4, 1e-4), rng=(1.0, 2.0)), SERIAL),  # under four frames at the top rate
    # ~0.5 ms loops over 10 s at up to 2x: more segments than a table holds
    "over_capacity": (dict(start=(0.0, 0.01), end=(0.0105, 0.02), rng=(1.0, 2.0), length=480000), SERIAL),
}


@pytest.mark.parametrize("name", list(PATHS))
def test_stage(pkg, host, name):
    case, stage = PATHS[name]
    k = kinds(pkg, loop_graph(pkg, host, **case))
    assert k.get(stage) == 1, k
    assert "k_buffer_source" not in k and "k_buffer_source_slow" not in k, k
    assert (BOUND if stage == SERIAL else SERIAL) not in k, k


def test_capacity_edge_stays_on_the_bound_track(pkg, host):
    # the shortest loop of these windows at the top rate over the whole render fits the table
    k = kinds(pkg, loop_graph(pkg, host, start=(0.0, 0.01), end=(0.05, 0.06), rng=(1.0, 2.0)))
    assert k.get(BOUND) == 1, k


def test_layout_decision(pkg, host):
    # a looping source that starts at frame 0 with no stop and no duration plays to the end of the render: a constant layout
    assert kinds(pkg, loop_graph(pkg, host, rng=(0.9, 1.1), biquad=False)) == {BOUND: 1, "k_mix": 1}
    assert kinds(pkg, loop_graph(pkg, host, biquad=False)) == {BOUND: 1, "k_mix": 1}
    for kw in (dict(when=0.01), dict(stop=1.5), dict(duration=1.0), dict(schedule=True)):
        k = kinds(pkg, loop_graph(pkg, host, rng=(0.9, 1.1), biquad=False, **kw))
        assert k == {BOUND: 1, "k_mix_dyn": 1}, (kw, k)


# WAE_PLAN_DIGEST of looping sources without a loop declaration (host-built slow and fast tracks, bound rates and schedules on the serial
# kernel), recorded before loop points could be bound: they plan as they did
DIGEST_CASES = {
    "slow": dict(rate=0.7, declare=False),
    "fast": dict(loop_points=(0.0, 0.0), declare=False, biquad=False),
    "bound_rate": dict(rng=(0.9, 1.1), declare=False),
    "bound_schedule": dict(schedule=True, declare=False),
    "late_stop": dict(rate=1.25, when=0.0123, stop=1.5, declare=False),
}
PINNED = {
    "slow": "aa4ab02a7bb88549",
    "fast": "7fdb91f145fd1c15",
    "bound_rate": "b7131061dbe0c442",
    "bound_schedule": "b7131061dbe0c442",
    "late_stop": "7f6627285e5e47a6",
}


def plan_digests():
    script = textwrap.dedent(f"""
        import sys
        sys.path.insert(0, {os.path.join(ROOT, 'tests')!r}); sys.path.insert(0, {ROOT!r})
        from conftest import load_package
        import test_device_loops_cpu as T
        pkg = load_package()
        be = pkg.context.Backend(pkg.api(), None)
        for name, kw in T.DIGEST_CASES.items():
            sys.stderr.write("case " + name + "\\n")
            pkg.plan_batch([T.loop_graph(pkg, be, **kw)])
    """)
    r = subprocess.run([sys.executable, "-c", script], env=dict(os.environ, WAE_PLAN_DIGEST="1"), capture_output=True, text=True, check=True)
    got, name = {}, None
    for line in r.stderr.splitlines():
        if line.startswith("case "):
            name = line[5:]
        elif "[wae plan digest]" in line:
            got[name] = line.rsplit(": ", 1)[1]
    return got


def test_plans_without_declarations_unchanged(pkg, host):
    assert plan_digests() == PINNED


# absn_loop_segments (wae_kernels.h) compiled for the host against a literal frame-by-frame replay of audio_buffer_source.rs:676-770, and
# the segment count against the capacity the planner reserves for windows that contain the points (absn_loop_capacity, restated)
WALK_CHECK = r"""
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <algorithm>
#include <limits>
#include <random>
#include <vector>
#include "wae_kernels.h"
using namespace wae;
int main() {
    std::mt19937_64 g(4321);
    std::uniform_real_distribution<double> u(0., 1.);
    const double srs[3] = {44100., 48000., 96000.};
    const double tol = 1.4901161193847656e-8;
    int bad = 0, over = 0, checked_cap = 0;
    std::vector<int64_t> seg_n(1 << 20);
    std::vector<double> seg_bt(1 << 20);
    for (int it = 0; it < 4000; it++) {
        const double sr = srs[it % 3], dt = 1. / sr;
        const double buffer_rate = srs[(it / 3) % 3];
        const double duration = std::floor(64. + u(g) * 96000.) / buffer_rate;
        const double rate = it % 11 == 0 ? 1. : 0.05 + 3. * u(g);
        // raw loop points: inside, at 0, at the buffer end, inverted, past the end, one ulp around almost::equal of each other
        double ls = u(g) * duration, le = ls + u(g) * (duration - ls);
        switch (it % 8) {
            case 1: ls = 0.; break;
            case 2: le = duration; break;
            case 3: std::swap(ls, le); break;
            case 4: le = duration * (1. + u(g)); break;
            case 5: ls = duration * (1. + u(g)); break;
            default: break;
        }
        const AbsnLoopPoints lp = absn_loop_points(ls, le, duration);
        double offset = u(g) * duration * 1.2;
        if (it % 7 == 0) offset = 0.;
        if (it % 13 == 0) offset = lp.actual_end;
        if (it % 17 == 0) offset = lp.actual_start + (it % 2 ? 1. : -1.) * (tol * std::max(1., lp.actual_start));
        if (it % 19 == 0) offset = std::nextafter(lp.actual_end - tol * std::max(1., lp.actual_end), it % 2 ? 0. : 1e300);
        const double delta = it % 3 == 0 ? 0. : u(g) * dt;
        const int64_t n_first = (int64_t)(u(g) * 1000.);
        const int64_t frames = 1000 + (int64_t)(u(g) * 60000.);
        const int64_t n_end = n_first + frames;
        const AbsnSlowDerived d = absn_slow_derive(dt, rate, offset, delta, duration, 1.7976931348623157e308, true, lp.actual_end, n_first,
                                                   SCHED_NEVER);
        const int32_t k = absn_loop_segments(lp.actual_start, lp.actual_end, d.step, n_first, n_end, d.offset0, seg_n.data(), seg_bt.data(),
                                             (int32_t)seg_n.size());
        if (k < 1) { bad++; continue; }
        // the replay: buffer_time per frame as the reference computes it
        const double als = lp.actual_start, ale = lp.actual_end;
        double bt = d.offset0;
        bool entered = false;
        int32_t s = 0;
        for (int64_t m = 0; m < frames; m++) {
            if (almost_equal(bt, ale)) bt = ale;
            if (almost_equal(bt, als)) bt = als;
            if (!entered) {
                if (d.offset0 < ale && bt >= als) entered = true;
                if (d.offset0 >= ale && bt < ale) entered = true;
            }
            if (entered) {
                while (bt >= ale) bt -= ale - als;
                while (bt < als) bt += ale - als;
            }
            const int64_t n = n_first + m;
            while (s + 1 < k && seg_n[s + 1] <= n) s++;
            const double tab = std::fma((double)(n - seg_n[s]), d.step, seg_bt[s]);
            if (!(std::fabs(tab - bt) <= 1e-9 * (1. + std::fabs(bt)))) {
                if (bad < 5) std::fprintf(stderr, "it %d frame %lld: table %.17g replay %.17g\n", it, (long long)m, tab, bt);
                bad++;
                break;
            }
            bt += d.step;
        }
        // the capacity the planner reserves for windows around these points (restated from absn_loop_capacity)
        const double w = u(g) * 0.01 * duration;
        const double s_hi = std::min(lp.actual_start + w, duration), e_lo = std::max(lp.actual_end - w, 0.);
        const double shortest = std::min(e_lo, duration) - s_hi;
        if (lp.actual_start < lp.actual_end && shortest > 4. * d.step && d.step > 6.0e-8 * (1. + duration)) {
            const double cap = 2. * (std::floor((double)frames * d.step / shortest) + 1. + 1.) + 4.;
            checked_cap++;
            if ((double)k > cap) over++;
        }
    }
    std::printf("%d %d %d\n", bad, over, checked_cap);
    return 0;
}
"""


def test_shared_walk_matches_the_reference_replay(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cuda_inc = os.path.join(os.path.dirname(os.path.dirname(nvcc)), "include")
    if not os.path.exists(os.path.join(cuda_inc, "cuda_runtime.h")):
        pytest.skip("no CUDA headers next to nvcc")
    src = tmp_path / "walk.cpp"
    src.write_text(WALK_CHECK)
    exe = tmp_path / "walk"
    # the library's host flags: no floating-point contraction
    subprocess.check_call(["g++", "-std=c++17", "-O3", "-ffp-contract=off", "-I", os.path.join(ROOT, "web-audio-api-rs_b200", "csrc"),
                           "-I", cuda_inc, str(src), "-o", str(exe)])
    bad, over, checked = (int(x) for x in subprocess.check_output([str(exe)], text=True).split())
    assert bad == 0 and over == 0, (bad, over)
    assert checked > 1000, checked
