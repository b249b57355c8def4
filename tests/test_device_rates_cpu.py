"""AudioBufferSourceNode playbackRate / detune bound from device memory, on the host (no GPU): the declaration rules, the playback path
and output layout the planner picks from the declared range, plans of graphs without declarations unchanged, and the shared derivation
of the slow track's rate-dependent constants against the planner's expressions as they stood before it was shared."""
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "web-audio-api-rs_b200", "libwae_b200.so")
SR = 48000.0
BOUND = "k_buffer_source_slow(bound)"


@pytest.fixture
def host(pkg):
    if not os.path.exists(LIB):
        pytest.skip("libwae_b200.so is not built (python -c 'import __graft_entry__ as g; g.build()')")
    return pkg.context.Backend(pkg.api(), None)


def status_of(fn):
    with pytest.raises(Exception) as e:
        fn()
    return e.value.status


def rate_graph(pkg, backend, rate=1.0, rng=None, det=None, frames=96000, length=48000, start=0.0, offset=0.0, duration=None,
               biquad=True, loop=False, started=True, automate_detune=False, buffer_rate=SR):
    """clip -> source (playbackRate declared over `rng`, detune over `det`) -> [lowpass] -> destination"""
    c = pkg.OfflineAudioContext(2, length, SR, backend)
    pcm = np.random.default_rng(frames).uniform(-0.5, 0.5, (2, frames)).astype(np.float32)
    s = c.create_buffer_source(pkg.AudioBuffer(list(pcm), buffer_rate), playback_rate=rate, loop=loop)
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
    if started:
        s.start_at_with_offset_and_duration(start, offset, 1.7976931348623157e308 if duration is None else duration)
    return c


def kinds(pkg, c):
    return pkg.plan_batch([c])["kinds"]


def test_both_params_accepted(pkg, host):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    s = c.create_buffer_source()
    s.detune.set_device_value(-100.0, 100.0)
    s.playback_rate.set_device_value(0.5, 2.0)
    api = pkg.api()
    assert api.param_set_device_value(c._g, s.id, 2, 0.0, 1.0) == 1  # (a buffer source has two params)


def test_declaration_rules(pkg, host):
    c = pkg.OfflineAudioContext(2, 1024, SR, host)
    s = c.create_buffer_source()
    s.playback_rate.set_device_value(0.5, 2.0)
    assert status_of(lambda: s.playback_rate.set_value(1.5)) == 2  # events after the declaration
    assert status_of(lambda: s.playback_rate.linear_ramp_to_value_at_time(2.0, 0.01)) == 2
    assert status_of(lambda: s.playback_rate.set_device_value(0.5, 2.0)) == 2  # declared twice
    lfo = c.create_oscillator()
    assert status_of(lambda: lfo.connect(s.playback_rate)) == 2  # an audio-rate input
    t = c.create_buffer_source()
    t.detune.set_value_at_time(100.0, 0.01)
    assert status_of(lambda: t.detune.set_device_value(-100.0, 100.0)) == 2  # events before it
    lfo.connect(t.playback_rate)
    assert status_of(lambda: t.playback_rate.set_device_value(0.5, 2.0)) == 2


def test_declaration_after_suspend_point(pkg, host):
    c = pkg.OfflineAudioContext(2, 4096, SR, host)
    s = c.create_buffer_source(pkg.AudioBuffer.zeros(2, 4096, SR))
    s.connect(c.destination())
    s.start()
    c.suspend_sync(1024 / SR, lambda ctx: s.playback_rate.set_device_value(0.5, 2.0))
    assert status_of(lambda: pkg.plan_batch([c])) == 2


def test_set_value_from_suspend_callback(pkg, host):
    c = pkg.OfflineAudioContext(2, 4096, SR, host)
    s = c.create_buffer_source(pkg.AudioBuffer.zeros(2, 4096, SR))
    s.connect(c.destination())
    s.start()
    s.detune.set_device_value(-100.0, 100.0)
    c.suspend_sync(1024 / SR, lambda ctx: s.detune.set_value(50.0))
    assert status_of(lambda: pkg.plan_batch([c])) == 2


@pytest.mark.parametrize("rng,det", [((0.9, 1.1), None), ((1.0 / 3.0, 2.0), (-100.0, 100.0)), (None, (-1200.0, 1200.0)), ((1.0, 1.0), None)],
                         ids=["rate", "rate_detune", "detune", "one_value"])
def test_positive_range_takes_the_bound_slow_track(pkg, host, rng, det):
    k = kinds(pkg, rate_graph(pkg, host, rng=rng, det=det))
    assert k.get(BOUND) == 1, k
    assert "k_buffer_source_serial" not in k and "k_buffer_source_slow" not in k and "k_buffer_source" not in k, k
    # never fused: the lowpass reads the source's arena buffer (the host-built graph at rate 1 has the source inside k_chain)
    assert k == {BOUND: 1, "k_chain": 1}, k
    assert kinds(pkg, rate_graph(pkg, host, rate=1.0)) == {"k_chain": 1}


@pytest.mark.parametrize("case", ["zero", "negative", "loop", "automated_detune", "detune_underflow"])
def test_serial_path(pkg, host, case):
    kw = {"zero": dict(rng=(0.0, 1.0)), "negative": dict(rng=(-0.5, 1.0)), "loop": dict(rng=(0.9, 1.1), loop=True),
          "automated_detune": dict(rng=(0.9, 1.1), automate_detune=True),
          # exp2(detune / 1200) is 0 in f64 at the low corner of the default range: the range allows a rate of 0
          "detune_underflow": dict(det=(-3.0e38, 3.0e38))}[case]
    k = kinds(pkg, rate_graph(pkg, host, **kw))
    assert k.get("k_buffer_source_serial") == 1, k
    assert BOUND not in k, k


def test_never_started_source_has_no_source_stage(pkg, host):
    for c in (rate_graph(pkg, host, rng=(0.9, 1.1), started=False), rate_graph(pkg, host, rng=(0.0, 1.0), started=False)):
        k = kinds(pkg, c)
        assert not any(name.startswith("k_buffer_source") for name in k), k


def test_layout_decision(pkg, host):
    # two seconds of clip at up to 1.1x cover the one-second render: a constant layout, the destination takes the plain mix, a downstream
    # biquad stays on the k_chain scan
    long = rate_graph(pkg, host, rng=(0.9, 1.1), frames=96000, biquad=False)
    assert kinds(pkg, long) == {BOUND: 1, "k_mix": 1}
    assert kinds(pkg, rate_graph(pkg, host, rng=(0.9, 1.1), frames=96000)) == {BOUND: 1, "k_chain": 1}
    # a clip that can end inside the render at the top of the range (1.05 s at 0.9x covers it, at 1.1x it does not): a layout track
    for kw in (dict(frames=50400), dict(start=0.01), dict(duration=0.5), dict(offset=1.5), dict(det=(0.0, 1200.0), frames=60000)):
        k = kinds(pkg, rate_graph(pkg, host, rng=(0.9, 1.1), biquad=False, **kw))
        assert k == {BOUND: 1, "k_mix_dyn": 1}, (kw, k)
    # a rate range whose top is exactly where the clip ends with the render: detune bound (exp2 may round either way) needs a quantum more
    exact = dict(rng=(0.5, 1.0), frames=48000 + 64, biquad=False)
    assert kinds(pkg, rate_graph(pkg, host, **exact)) == {BOUND: 1, "k_mix": 1}
    assert kinds(pkg, rate_graph(pkg, host, det=(-10.0, 0.0), **exact)) == {BOUND: 1, "k_mix_dyn": 1}


# WAE_PLAN_DIGEST of host-built buffer-source graphs (fast, fused, slow, looping slow, serial, late, offset, stop, duration, 44.1 kHz
# buffer), recorded before the slow track's constants were derived by absn_slow_derive: graphs without declarations plan as they did
DIGEST_CASES = {
    "fast": dict(rate=1.0, biquad=False),
    "fused": dict(rate=1.0),
    "slow": dict(rate=0.9),
    "slow_short": dict(rate=1.1, frames=40000),
    "loop": dict(rate=0.75, loop=True, frames=20000),
    "serial": dict(rate=-0.5),
    "late_offset": dict(rate=1.1, start=0.0123, offset=0.05),
    "duration": dict(rate=2.0, duration=0.3),
    "44k1": dict(rate=1.0, buffer_rate=44100.0),
}
PINNED = {
    "fast": "83a594215d67e4ca",
    "fused": "26a27f434a6018b3",
    "slow": "a72e9ffdc342b2d6",
    "slow_short": "9c76c8c40713e43a",
    "loop": "8ec55b282d70d91a",
    "serial": "a811d11f4e5ce88a",
    "late_offset": "a6d84e4edcecd317",
    "duration": "2768ae407fd66676",
    "44k1": "ec4fab0655d8a62a",
}


def plan_digests():
    script = textwrap.dedent(f"""
        import sys
        sys.path.insert(0, {os.path.join(ROOT, 'tests')!r}); sys.path.insert(0, {ROOT!r})
        from conftest import load_package
        import test_device_rates_cpu as T
        pkg = load_package()
        be = pkg.context.Backend(pkg.api(), None)
        for name, kw in T.DIGEST_CASES.items():
            sys.stderr.write("case " + name + "\\n")
            pkg.plan_batch([T.rate_graph(pkg, be, **kw)])
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


# The pre-refactor expressions of Planner::absn_slow, restated, against absn_slow_derive (wae_kernels.h) compiled for the host, bit for bit
DERIVE_CHECK = r"""
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <algorithm>
#include <limits>
#include <random>
#include "wae_kernels.h"
using namespace wae;
static bool same(double a, double b) { return std::memcmp(&a, &b, 8) == 0; }
int main() {
    std::mt19937_64 g(1234);
    std::uniform_real_distribution<double> u(0., 1.);
    const double srs[3] = {44100., 48000., 96000.};
    int bad = 0;
    for (int it = 0; it < 200000; it++) {
        const double sr = srs[it % 3], dt = 1. / sr;
        const double buffer_rate = srs[(it / 3) % 3];
        const double duration = std::floor(1. + u(g) * 200000.) / buffer_rate;  // the buffer's
        const float rate = (float)(it % 7 == 0 ? 1. : 0.05 + 4. * u(g));
        const float detune = (float)(it % 5 == 0 ? 0. : -2400. + 4800. * u(g));
        const double computed_rate = (double)rate * std::exp2((double)detune / 1200.);
        const double offset = it % 4 == 0 ? 0. : u(g) * duration * 1.2;
        const double delta = it % 3 == 0 ? 0. : u(g) * dt;
        const double dur = it % 6 == 0 ? u(g) * 3. : std::numeric_limits<double>::max();
        const bool loop = it % 9 == 0;
        const double loop_end = loop ? u(g) * duration : duration;
        const int64_t n_first = (int64_t)(u(g) * 100000.);
        const int64_t n_stop = it % 8 == 0 ? n_first + (int64_t)(u(g) * 200000.) : std::numeric_limits<int64_t>::max();
        // Planner::absn_slow before absn_slow_derive
        const double step = dt * computed_rate;
        double off = offset + delta * computed_rate;
        off = std::min(std::max(off, 0.), duration);
        if (loop && off > loop_end) off = loop_end;
        const double elapsed0 = std::fabs(delta * computed_rate);
        int64_t n_end = n_stop;
        if (step > 0.) {
            if (!loop) n_end = std::min<int64_t>(n_end, n_first + (int64_t)std::ceil(std::max(0., duration - off) / step));
            if (dur < 1e300) n_end = std::min<int64_t>(n_end, n_first + (int64_t)std::ceil(std::max(0., dur - elapsed0) / step));
        }
        const AbsnSlowDerived d = absn_slow_derive(dt, computed_rate, offset, delta, duration, dur, loop, loop_end, n_first, n_stop);
        if (!same(d.step, step) || !same(d.offset0, off) || !same(d.elapsed0, elapsed0) || d.n_end != n_end) bad++;
    }
    std::printf("%d\n", bad);
    return 0;
}
"""


def test_shared_derivation_matches_the_planner(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cuda_inc = os.path.join(os.path.dirname(os.path.dirname(nvcc)), "include")
    if not os.path.exists(os.path.join(cuda_inc, "cuda_runtime.h")):
        pytest.skip("no CUDA headers next to nvcc")
    src = tmp_path / "derive.cpp"
    src.write_text(DERIVE_CHECK)
    exe = tmp_path / "derive"
    # the library's host flags: no floating-point contraction
    subprocess.check_call(["g++", "-std=c++17", "-O3", "-ffp-contract=off", "-I", os.path.join(ROOT, "web-audio-api-rs_b200", "csrc"),
                           "-I", cuda_inc, str(src), "-o", str(exe)])
    assert subprocess.check_output([str(exe)], text=True).strip() == "0"
