"""GPU parity of the reference's criterion / iai benchmark graphs (benches/my_benchmark.rs), of graphs configured through the
post-construction setters, of the WPT buffer-stitching case, and of the two AudioParam kernels against each other."""

import numpy as np
import pytest

import benchmark_scenarios as BS
import test_node_setters as NS
import test_oracle_absn as A

pytestmark = pytest.mark.gpu
SECONDS = 3.0


@pytest.mark.parametrize("name,build", BS.CRITERION, ids=[n for n, _ in BS.CRITERION])
def test_criterion_bench_matches_the_oracle(pkg, engine, oracle, name, build):
    """benches/my_benchmark.rs (criterion / iai), GPU vs oracle at 1e-5."""
    import graphs as G
    if "hrtf" in name:
        sphere = G.synthetic_hrir_sphere(44100, 256)
        oracle.set_hrir_sphere(sphere)
        engine.backend.set_hrir_sphere(sphere)
    got = build(pkg, engine.backend, 2.0).start_rendering_sync()
    want = build(pkg, oracle, 2.0).start_rendering_sync()
    for ch in range(2):
        d = np.abs(got.get_channel_data(ch).astype(np.float64) - want.get_channel_data(ch))
        assert d.max() <= 1e-5, (name, ch, float(d.max()))


def test_graph_built_with_setters_on_gpu(pkg, engine, oracle):
    # tests/test_node_setters.py: the library only records the setters in the graph description, the plan is proven identical on the CPU
    got = NS._variants(pkg, engine.backend, True).start_rendering_sync()
    want = NS._variants(pkg, oracle, False).start_rendering_sync()
    for ch in range(2):
        assert np.abs(got.get_channel_data(ch).astype(np.float64) - want.get_channel_data(ch)).max() <= 1e-5


def test_buffer_source_setters_on_gpu(pkg, engine):
    NS.test_buffer_source_configured_the_way_the_reference_examples_do(pkg, engine.backend)


@pytest.mark.parametrize("rates", [(44100.0, 44100.0, 9.0957e-5), (44100.0, 43800.0, 3.8986e-3)])
def test_buffer_source_stitching_on_gpu(pkg, engine, rates):
    A.test_construct_with_options_and_run(pkg, engine.backend)
    A.test_subsample_buffer_stitching(pkg, engine.backend, *rates)


AUTOMATED = ["Granular synthesis", "Synth (Sawtooth with Envelope)", "Substractive Synth", "Stereo panning with automation", "Sawtooth with automation"]


@pytest.mark.parametrize("name", AUTOMATED)
def test_parallel_param_kernel_matches_the_oracle(pkg, engine, oracle, name):
    """The AudioParam kernels on the automation-heavy scenarios of the reference's benchmark suite: the default (one CTA per param, 32
    quanta walked speculatively from predicted states and verified, csrc/wae_kernels.cu k_param_spec) against the oracle AND, bit for
    bit, against the two kernels that walk quantum after quantum (WAE_OPT_PARAM_PARALLEL = 1: the warp evaluates the fills,
    csrc/wae_param_walk.h; 0: lane 0 evaluates every frame)."""
    build = dict(BS.SCENARIOS)[name]
    want = build(pkg, oracle, SECONDS).start_rendering_sync()
    got = build(pkg, engine.backend, SECONDS).start_rendering_sync()
    others = []
    try:
        for mode in (0, 1):
            engine.set_option(pkg.OPT_PARAM_PARALLEL, mode)
            others.append(build(pkg, engine.backend, SECONDS).start_rendering_sync())
    finally:
        engine.set_option(pkg.OPT_PARAM_PARALLEL, 2)
    for ch in range(want.number_of_channels()):
        assert np.abs(got.get_channel_data(ch).astype(np.float64) - want.get_channel_data(ch)).max() <= 1e-5 * max(1.0, float(np.abs(want.get_channel_data(ch)).max()))
        for o in others:
            assert np.array_equal(got.get_channel_data(ch), o.get_channel_data(ch))
