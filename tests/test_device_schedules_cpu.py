"""Start / stop times of scheduled sources bound from device memory, on the host (no GPU): the declaration rules, the ABI layout, the
playback path an AudioBufferSourceNode takes, plans equal to host twins started late inside the render, and the shared scheduling
functions against the planner's expressions as they stood before they were shared."""
import ctypes as C
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


def kinds(pkg, c):
    return pkg.plan_batch([c])["kinds"]


def test_binding_layout(pkg):
    B = pkg._binding if hasattr(pkg, "_binding") else sys.modules[pkg.__name__ + "._binding"]
    assert C.sizeof(B.ScheduleBinding) == 16
    assert [B.ScheduleBinding.graph_index.offset, B.ScheduleBinding.node.offset, B.ScheduleBinding.times.offset] == [0, 4, 8]


def test_declaration_rules(pkg, host):
    c = pkg.OfflineAudioContext(2, 4096, SR, host)
    osc = c.create_oscillator()
    osc.connect(c.destination())
    assert status_of(lambda: osc.set_device_schedule((0.0, 0.05))) == 2  # not started
    osc.start_at(0.01)
    for bad in ((0.02, 0.01), (-0.01, 0.05), (0.0, float("inf")), (float("nan"), 1.0)):
        assert status_of(lambda: osc.set_device_schedule(bad)) == 1, bad
    assert status_of(lambda: osc.set_device_schedule((0.0, 0.05), stop=(0.03, 0.02))) == 1
    osc.set_device_schedule((0.0, 0.05))
    assert status_of(lambda: osc.set_device_schedule((0.0, 0.05))) == 2  # declared twice
    assert status_of(lambda: osc.start_at(0.02)) == 2
    assert status_of(lambda: osc.stop_at(0.04)) == 2
    gain = c.create_gain()
    assert pkg.api().source_set_device_schedule(c._g, gain.id, 0.0, 0.05, 0, 0.0, 0.0) == 1  # not a scheduled source
    cs = c.create_constant_source()
    cs.start()
    cs.set_device_schedule((0.0, 0.05), stop=(0.01, 0.08))
    s = c.create_buffer_source(pkg.AudioBuffer.zeros(1, 512, SR))
    s.start_at_with_offset_and_duration(0.0, 0.001, 0.002)
    s.set_device_schedule((0.0, 1.0))


def test_declaration_after_suspend_point(pkg, host):
    c = pkg.OfflineAudioContext(2, 4096, SR, host)
    osc = c.create_oscillator()
    osc.connect(c.destination())
    osc.start()
    c.suspend_sync(1024 / SR, lambda ctx: None)
    c._run_suspend_callbacks()
    assert status_of(lambda: osc.set_device_schedule((0.0, 0.05))) == 2


def test_suspend_point_after_declaration(pkg, host):
    c = pkg.OfflineAudioContext(2, 4096, SR, host)
    osc = c.create_oscillator()
    osc.connect(c.destination())
    osc.start()
    osc.set_device_schedule((0.0, 0.05))
    c.suspend_sync(1024 / SR, lambda ctx: None)
    assert status_of(lambda: pkg.plan_batch([c])) == 2


def osc_graph(pkg, backend, start, stop=None, declare=False, type_=None, biquad=True, automate=False, const=False):
    """source -> [lowpass] -> destination; `declare`: the start (and stop) declared with windows whose low ends are `start` / `stop`"""
    c = pkg.OfflineAudioContext(1, 4800, SR, backend)
    if const:
        src = c.create_constant_source()
    else:
        src = c.create_oscillator()
        if type_ is not None:
            src.set_type(type_)
        src.frequency.set_value(440.0)
        if automate:
            src.frequency.linear_ramp_to_value_at_time(880.0, 0.05)
    last = src
    if biquad:
        bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=1000.0)
        src.connect(bq)
        last = bq
    last.connect(c.destination())
    src.start_at(start)
    if stop is not None and not declare:
        src.stop_at(stop)
    if declare:
        src.set_device_schedule((start, start + 0.5), stop=None if stop is None else (stop, stop + 0.5))
    return c


DIGEST_CASES = {
    "osc_fused": dict(start=0.0123),
    "osc_stop": dict(start=0.0123, stop=0.05),
    "osc_unfused": dict(start=0.0123, biquad=False),
    "osc_arate": dict(start=0.0123, automate=True),
    "square": dict(start=0.02, stop=0.07, type_=1),
    "const_fused": dict(start=0.0101, stop=0.03, const=True),
    "const_unfused": dict(start=0.0101, const=True, biquad=False),
}


def plan_digests(declare):
    script = textwrap.dedent(f"""
        import sys
        sys.path.insert(0, {os.path.join(ROOT, 'tests')!r}); sys.path.insert(0, {ROOT!r})
        from conftest import load_package
        import test_device_schedules_cpu as T
        pkg = load_package()
        be = pkg.context.Backend(pkg.api(), None)
        for name, kw in T.DIGEST_CASES.items():
            sys.stderr.write("case " + name + "\\n")
            c = T.osc_graph(pkg, be, declare={declare!r}, **kw)
            sys.stderr.write("kinds " + repr(sorted(pkg.plan_batch([c])["kinds"].items())) + "\\n")
    """)
    r = subprocess.run([sys.executable, "-c", script], env=dict(os.environ, WAE_PLAN_DIGEST="1"), capture_output=True, text=True, check=True)
    got, name = {}, None
    for line in r.stderr.splitlines():
        if line.startswith("case "):
            name = line[5:]
            got[name] = []
        elif line.startswith("kinds "):
            got[name].append(line[6:])
        elif "[wae plan digest]" in line:
            got[name].append(line.rsplit(": ", 1)[1])
    return got


def test_declared_plans_equal_host_twins_started_late(pkg, host):
    """The record fields of a declared source hold the windows' low ends: the plan (stages and digest) is the host twin's started there,
    which is gated as well."""
    declared, twins = plan_digests(True), plan_digests(False)
    assert set(declared) == set(DIGEST_CASES)
    assert declared == twins


def test_declared_source_at_zero_is_gated(pkg, host):
    # a host source started at 0 that plays to the end has a constant layout; a declared one is gated (its output gets a layout track)
    def graph(declare):
        c = pkg.OfflineAudioContext(1, 4800, SR, host)
        osc = c.create_oscillator()
        g = c.create_gain(gain=0.5)
        osc.connect(c.destination())
        osc.connect(g)
        g.connect(c.destination())
        osc.start()
        if declare:
            osc.set_device_schedule((0.0, 0.01))
        return kinds(pkg, c)
    assert "k_meta" not in graph(False) and "k_mix_dyn" not in graph(False), graph(False)
    k = graph(True)
    assert "k_mix_dyn" in k, k


def absn_graph(pkg, backend, rate=1.0, loop=False, automate=False, rate_range=None, biquad=True, start=0.01):
    c = pkg.OfflineAudioContext(2, 9600, SR, backend)
    pcm = np.random.default_rng(3).uniform(-0.5, 0.5, (2, 4800)).astype(np.float32)
    s = c.create_buffer_source(pkg.AudioBuffer(list(pcm), SR), playback_rate=rate, loop=loop)
    if automate:
        s.playback_rate.linear_ramp_to_value_at_time(2.0, 0.1)
    if rate_range is not None:
        s.playback_rate.set_device_value(*rate_range)
    last = s
    if biquad:
        bq = c.create_biquad_filter(type_=pkg.LOWPASS, frequency=1000.0)
        s.connect(bq)
        last = bq
    last.connect(c.destination())
    s.start_at(start)
    s.set_device_schedule((start, start + 0.1))
    return c


@pytest.mark.parametrize("case,stage", [
    (dict(), BOUND),                                  # rate 1: the bound slow track (1:1 where the start is aligned)
    (dict(rate=0.9), BOUND),
    (dict(rate_range=(0.5, 2.0)), BOUND),
    (dict(loop=True), "k_buffer_source_serial"),
    (dict(automate=True), "k_buffer_source_serial"),
    (dict(rate_range=(0.0, 2.0)), "k_buffer_source_serial"),  # a bound range that allows a rate <= 0
    (dict(rate=-1.0), "k_buffer_source_serial"),
], ids=["rate1", "rate09", "bound_range", "loop", "automated", "range_to_zero", "negative"])
def test_buffer_source_stage(pkg, host, case, stage):
    k = kinds(pkg, absn_graph(pkg, host, **case))
    assert k.get(stage) == 1, k
    assert "k_buffer_source" not in k and "k_buffer_source_slow" not in k, k
    # never fused into k_chain as a source: the lowpass reads the source's buffer
    if stage == BOUND:
        assert k == {BOUND: 1, "k_chain": 1}, k


# The planner's expressions before they were shared (SchedClock of the host math, Planner::lower_osc, lower_absn, absn_start and
# absn_fast_end), restated, against the shared WAE_HD functions (wae_kernels.h) compiled for the host, bit for bit
SCHED_CHECK = r"""
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
struct OldClock {
    double sample_rate, dt;
    explicit OldClock(float sr) : sample_rate((double)sr), dt(1. / (double)sr) {}
    double block_time(int64_t q) const { return (double)(q * 128) / sample_rate; }
    double next_block_time(int64_t q) const { return block_time(q) + dt * 128.; }
    int64_t quantum_containing(double T) const {
        if (!(T < 1e15)) return std::numeric_limits<int64_t>::max() / 256;
        int64_t q = (int64_t)std::floor(T * sample_rate / 128.) - 2;
        if (q < 0) q = 0;
        while (!(T < next_block_time(q))) q++;
        return q;
    }
    int64_t first_frame_at_or_after(double T, double* time_out = nullptr) const {
        int64_t q = quantum_containing(T);
        if (q >= std::numeric_limits<int64_t>::max() / 512) return std::numeric_limits<int64_t>::max();
        double t = block_time(q);
        for (int i = 0; i < 128; i++) {
            if (t >= T) { if (time_out) *time_out = t; return q * 128 + i; }
            t += dt;
        }
        if (time_out) *time_out = block_time(q + 1);
        return (q + 1) * 128;
    }
};
static bool old_almost_equal(double x, double y) {
    if (x == y) return true;
    const double tol = 1.4901161193847656e-8;
    double d = std::fabs(y - x);
    return d <= tol || d <= std::max(std::fabs(x), std::fabs(y)) * tol;
}
int main(int argc, char** argv) {
    std::mt19937_64 g(99);
    std::uniform_real_distribution<double> u(0., 1.);
    const float srs[2] = {44100.f, 48000.f};
    int bad = 0;
    long n = 0;
    for (int it = 0; it < 240000; it++) {
        const float sr = srs[it % 2];
        const OldClock oc(sr);
        const SchedClock nc(sr);
        const int64_t q0 = (int64_t)(u(g) * 40000.);
        double T;
        switch ((it / 2) % 6) {
            case 0: T = u(g) * 120.; break;                                    // anywhere
            case 1: T = oc.block_time(q0); break;                              // on a block boundary
            case 2: T = std::nextafter(oc.block_time(q0), 0.); break;          // one ulp below
            case 3: T = std::nextafter(oc.block_time(q0), 1e300); break;       // one ulp above
            case 4: T = oc.block_time(q0) + (double)(it % 128) * oc.dt; break; // on an accumulated frame time
            default: T = (double)(q0 * 128) / (double)sr; T = std::nextafter(T, (it & 4) ? 0. : 1e300); break;
        }
        const double stop = (it % 3) ? T + u(g) * 2. : 1.7976931348623157e308;
        const double incr = (it % 5 == 0) ? 0.75 + u(g) : u(g) * 0.3;
        const bool outside = incr >= 0.5;
        n++;
        // SchedClock
        double ta = 0., tb = 0.;
        if (oc.quantum_containing(T) != nc.quantum_containing(T) || !same(oc.block_time(q0), nc.block_time(q0))) bad++;
        if (oc.first_frame_at_or_after(T, &ta) != nc.first_frame_at_or_after(T, &tb) || !same(ta, tb)) bad++;
        // Planner::lower_osc
        {
            int64_t q = oc.quantum_containing(T);
            double start = T;
            if (start < oc.block_time(q)) start = oc.block_time(q);
            double cur = oc.block_time(q);
            int i = 0;
            for (; i < 128; i++) { if (!(cur < start)) break; cur += oc.dt; }
            int64_t n_first = q * 128 + i;
            double phase0 = 0., ratio0 = 0.;
            if (i < 128 && cur > start) {
                double ratio = (cur - start) / oc.dt;
                ratio0 = ratio;
                double ph = incr * ratio;
                if (outside) { ph = std::fmod(ph, 1.); if (ph < 0.) ph += 1.; }
                else ph = ph >= 1. ? ph - 1. : (ph < 0. ? ph + 1. : ph);
                phase0 = ph;
            }
            int64_t n_stop = std::numeric_limits<int64_t>::max();
            if (stop < 1e300) {
                int64_t qs = oc.quantum_containing(stop);
                n_stop = stop <= oc.block_time(qs) ? qs * 128 : oc.first_frame_at_or_after(stop);
            }
            const OscStart s = osc_start(nc, T, incr, outside);
            if (s.n_first != n_first || !same(s.phase0, phase0) || !same(s.start_ratio, ratio0) || osc_stop_frame(nc, stop) != n_stop) bad++;
        }
        // Planner::lower_absn (the q + 1 snap), absn_start, absn_fast_end
        {
            int64_t q = oc.quantum_containing(T);
            if (T > oc.block_time(q) && T == oc.block_time(q + 1)) q = q + 1;
            if (absn_start_quantum(nc, T) != q) bad++;
            int64_t nf = -1, ns = std::numeric_limits<int64_t>::max();
            double t_first = 0., st = T;
            int64_t qq = oc.quantum_containing(st);
            for (int guard = 0; guard < 3 && nf < 0; guard++, qq++) {
                double bt0 = oc.block_time(qq);
                for (int i = 0; i < 128; i++) {
                    double t = bt0 + (double)i * oc.dt;
                    if (old_almost_equal(t, st)) st = t;
                    if (!(t < st)) { nf = qq * 128 + i; t_first = t; break; }
                }
            }
            if (nf < 0) nf = qq * 128;
            if (stop < 1e300) {
                int64_t qs = oc.quantum_containing(stop);
                ns = (qs + 1) * 128;
                double bt0 = oc.block_time(qs);
                for (int i = 0; i < 128; i++)
                    if (bt0 + (double)i * oc.dt >= stop) { ns = qs * 128 + i; break; }
            }
            const AbsnStart a = absn_start(nc, T, stop);
            if (a.n_first != nf || a.n_stop != ns || !same(a.t_first, t_first) || !same(a.start, st)) bad++;
            const double duration = u(g) * 20.;
            const int64_t lq = 480000, n_start = q * 128;
            const double block_duration = oc.dt * 128.;
            const int64_t max_q = (lq - n_start) / 128 + 2;
            int64_t played = 0;
            double bt = 0.;
            while (played < max_q) { bt += block_duration; played++; if (bt >= duration) break; }
            if (absn_fast_end(nc, lq, n_start, duration) != n_start + played * 128) bad++;
        }
    }
    std::printf("%d %ld\n", bad, n);
    return 0;
}
"""


def test_shared_scheduling_functions_match_the_planner(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cuda_inc = os.path.join(os.path.dirname(os.path.dirname(nvcc)), "include")
    if not os.path.exists(os.path.join(cuda_inc, "cuda_runtime.h")):
        pytest.skip("no CUDA headers next to nvcc")
    src = tmp_path / "sched.cpp"
    src.write_text(SCHED_CHECK)
    exe = tmp_path / "sched"
    # the library's host flags: no floating-point contraction
    subprocess.check_call(["g++", "-std=c++17", "-O3", "-ffp-contract=off", "-I", os.path.join(ROOT, "web-audio-api-rs_b200", "csrc"),
                           "-I", cuda_inc, str(src), "-o", str(exe)])
    bad, n = subprocess.check_output([str(exe)], text=True).split()
    assert int(bad) == 0 and int(n) >= 100000

