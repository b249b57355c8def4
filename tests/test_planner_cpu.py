"""The planner — the largest piece of host logic of the library (csrc/wae_engine.cu: fusion, stage grouping, scheduling classes of
feedback loops, render segments of suspend points, chunk sizing, what is refused) — exercised WITHOUT a GPU through wae_batch_plan,
which runs the sizing pass wae_batch_prepare runs first (it touches no device memory) and reports what the batch would be lowered to."""
import os

import numpy as np
import pytest

import benchmark_scenarios as BS
import graphs as G

RQ = 128


@pytest.fixture
def be(pkg):
    so = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "web-audio-api-rs_b200", "libwae_b200.so")
    if not os.path.exists(so):
        pytest.skip("libwae_b200.so is not built (python -c 'import __graft_entry__ as g; g.build()')")
    return pkg.context.Backend(pkg.api(), None)


def plan(pkg, ctxs):
    return pkg.context.plan_batch(ctxs)


def test_c2_is_one_fused_launch_for_the_whole_render(pkg, be):
    # BASELINE configs[1]: AudioBufferSource -> Biquad -> Gain -> destination: one k_chain stage, no arena, one chunk = the whole render
    p = plan(pkg, [G.c2_buffer_biquad_gain(pkg, be, g, 48000) for g in range(8)])
    assert p["kinds"] == {"k_chain": 1} and p["arena_floats_per_frame"] == 0 and p["chunks"] == 1 and p["chunk_frames"] == 48000
    assert p["source_floats"] == 8 * 2 * 48000 and not p["has_feedback"]
    # >= 512 graphs: 32 pipeline groups, each its own stage
    p = plan(pkg, [G.c2_buffer_biquad_gain(pkg, be, g, 1280) for g in range(512)])
    assert p["groups"] == 32 and p["kinds"] == {"k_chain": 32}


def test_c1_c3_voices_fuse_and_meet_in_one_mix(pkg, be):
    p = plan(pkg, [G.c1_osc_biquad(pkg, be, 48000)])
    assert p["kinds"] == {"k_chain": 1}  # the single chain writes the destination directly (mono -> stereo by copy)
    p = plan(pkg, [G.c3_many_voices(pkg, be, 64, 48000)])
    assert p["kinds"] == {"k_chain": 1, "k_mix": 1}  # 64 oscillator -> biquad chains in ONE launch, one ordered sum
    assert p["arena_floats_per_frame"] == 64           # 64 mono voices


def test_c4_north_star_c5_stage_lists(pkg, be):
    ir = G.synthetic_ir(20000, 2, decay=0.6)
    p = plan(pkg, [G.c4_convolver(pkg, be, g, 8192 * 3, ir) for g in range(4)])
    # the source buffer covers the render 1:1 and the convolver is the destination's only input: the forward transforms read the asset,
    # the inverse transforms write the rendered PCM — no copy stage on either side
    assert set(p["kinds"]) == {"k_conv_fft_in", "k_conv_mac_ifft"} and p["chunk_frames"] % 8192 == 0 and p["arena_floats_per_frame"] == 0
    # a second input at the destination needs the mix again ...
    def two_inputs(g):
        c = G.c4_convolver(pkg, be, g, 8192 * 3, ir)
        o = c.create_constant_source()
        o.connect(c.destination())
        o.start()
        return c
    k = plan(pkg, [two_inputs(g) for g in range(2)])["kinds"]
    assert "k_mix" in k and k.get("k_chain") == 1   # (that chain is the constant source; the buffer source is still read in place)
    # ... and a source that does not cover the render 1:1 (here: looping) is copied by the chain kernel as before
    def looping(g):
        c = pkg.OfflineAudioContext(2, 8192 * 3, 48000.0, be)
        src = c.create_buffer_source(pkg.AudioBuffer([np.ones(5000, np.float32)] * 2, 48000.0), loop=True)
        cv = c.create_convolver(pkg.AudioBuffer(ir, 48000.0))
        src.connect(cv)
        cv.connect(c.destination())
        src.start()
        return c
    k = plan(pkg, [looping(g) for g in range(2)])["kinds"]
    assert "k_chain" in k and "k_mix" not in k
    p = plan(pkg, [G.north_star_voices_convolver(pkg, be, 50, 8192 * 3, ir, seed=g) for g in range(2)])
    assert p["kinds"]["k_chain"] == 1 and "k_conv_mac_ifft" in p["kinds"]
    # enough (2048-frame tile, graph) work items to fill the machine about twice: the voices and their ordered sum become ONE kernel
    # (k_voice_sum), no voice is written to the arena (what is left is the convolver's mono input), the render is one chunk
    big = [G.north_star_voices_convolver(pkg, be, 12, 8192 * 48, ir, seed=g) for g in range(8)]
    assert "k_voice_sum" not in plan(pkg, big)["kinds"]  # (off by default: measured slower than k_chain + k_mix)
    os.environ["WAE_VOICE_SUM"] = "1"
    try:
        p = plan(pkg, big)
        assert p["kinds"].get("k_voice_sum") == 1 and "k_chain" not in p["kinds"] and "k_mix" not in p["kinds"]
        assert p["arena_floats_per_frame"] == 8 and p["chunks"] == 1
        # ... C3 (one graph, a short render) keeps k_chain + k_mix: its parallelism is in the voices, not in (tile, graph) items
        p = plan(pkg, [G.c3_many_voices(pkg, be, 64, 48000)])
        assert "k_voice_sum" not in p["kinds"]
    finally:
        del os.environ["WAE_VOICE_SUM"]
    with pytest.raises(pkg.WaeError) as e:  # an HRTF panner needs the sphere the engine is given (wae_engine_set_hrir_sphere)
        plan(pkg, [G.c5_full_chain(pkg, be, 0, 8192, ir)])
    assert e.value.status == 4 and "HRIR sphere" in str(e.value)


@pytest.mark.parametrize("name,build", BS.SCENARIOS, ids=[n for n, _ in BS.SCENARIOS])
def test_every_reference_benchmark_scenario_is_lowered(pkg, be, name, build):
    # examples/benchmarks.rs: none of the 24 scenarios may be refused (WAE_UNSUPPORTED) by the planner
    p = plan(pkg, [build(pkg, be, 3.0) for _ in range(2)])
    assert p["stages"] >= 1 and p["segments"] == p["groups"]
    if name.startswith("Simple source test without resampling (Mono)"):
        assert p["kinds"] == {"k_chain": 1}


def test_feedback_loop_is_scheduled_and_a_convolver_inside_it_is_refused(pkg, be):
    def echo(with_conv):
        c = pkg.OfflineAudioContext(2, RQ * 16, 48000.0, be)
        src = c.create_constant_source()
        g = c.create_gain(0.5)
        d = c.create_delay(1.0, 0.01)
        src.connect(g)
        g.connect(d)
        if with_conv:
            conv = c.create_convolver(pkg.AudioBuffer([np.ones(8, np.float32)], 48000.0))
            d.connect(conv)
            conv.connect(g)
        else:
            d.connect(g)
        g.connect(c.destination())
        src.start()
        return c

    p = plan(pkg, [echo(False)])
    assert p["has_feedback"] and "k_delay_read" in p["kinds"] and "k_ring_write" in p["kinds"]
    with pytest.raises(pkg.WaeError) as e:  # a ConvolverNode inside the loop is not lowered (DESIGN.md §6)
        plan(pkg, [echo(True)])
    assert e.value.status == 4 and "feedback cycle" in str(e.value)


def test_suspend_points_cut_the_render_into_segments(pkg, be):
    def build(cut_frames, with_conv):
        sr = 48000.0
        c = pkg.OfflineAudioContext(1, 8192 * 3, sr, be)
        src = c.create_constant_source()
        node = c.create_convolver(pkg.AudioBuffer([np.ones(4, np.float32)], sr)) if with_conv else c.create_gain(0.5)
        src.connect(node)
        node.connect(c.destination())
        src.start()
        c.suspend_sync(cut_frames / sr, lambda ctx: src.offset.set_value(0.25))
        return c

    p = plan(pkg, [build(RQ * 5, False)])
    assert p["segments"] == 2
    p = plan(pkg, [build(8192, True)])   # a convolver needs the cut on a partition boundary
    assert p["segments"] == 2
    with pytest.raises(pkg.WaeError) as e:
        plan(pkg, [build(RQ * 5, True)])
    assert e.value.status == 4
    # graphs with different suspend points are planned in different groups
    p = plan(pkg, [build(RQ * 5, False), build(RQ * 9, False)])
    assert p["groups"] == 2 and p["segments"] == 4


def test_batch_shape_errors(pkg, be):
    a = pkg.OfflineAudioContext(2, 256, 48000.0, be)
    b = pkg.OfflineAudioContext(1, 256, 48000.0, be)
    with pytest.raises(pkg.WaeError):
        plan(pkg, [a, b])  # all graphs of a batch share channels / length / sample rate


def _one(pkg, be, build, length=RQ * 8, channels=2, sr=48000.0):
    c = pkg.OfflineAudioContext(channels, length, sr, be)
    build(c)
    return plan(pkg, [c])["kinds"]


def test_which_kernel_a_node_variant_is_lowered_to(pkg, be):
    noise = np.random.default_rng(3).uniform(-1, 1, 4096).astype(np.float32)

    def src_to(c, node):
        s = c.create_buffer_source(pkg.AudioBuffer([noise, noise], 48000.0))
        s.connect(node)
        node.connect(c.destination())
        s.start()
        return s

    # canonical chain order: source -> gain -> biquad -> gain -> biquad -> gain -> shaper -> gain is ONE fused launch
    def long_chain(c):
        s = c.create_buffer_source(pkg.AudioBuffer([noise, noise], 48000.0))
        nodes = [c.create_gain(0.9), c.create_biquad_filter(), c.create_gain(0.8), c.create_biquad_filter(type_=pkg.HIGHPASS), c.create_gain(0.7),
                 c.create_wave_shaper(curve=np.linspace(-1, 1, 9).astype(np.float32)), c.create_gain(0.6)]
        prev = s
        for n in nodes:
            prev.connect(n)
            prev = n
        prev.connect(c.destination())
        s.start()
    assert _one(pkg, be, long_chain) == {"k_chain": 1}
    # a third biquad does not fit the chain shape: the chain is materialised and a second one starts
    def three_biquads(c):
        s = c.create_buffer_source(pkg.AudioBuffer([noise, noise], 48000.0))
        prev = s
        for _ in range(3):
            b = c.create_biquad_filter()
            prev.connect(b)
            prev = b
        prev.connect(c.destination())
        s.start()
    k = _one(pkg, be, three_biquads)
    assert k.get("k_chain", 0) == 2 and "k_biquad_serial" not in k
    # IIR filter, compressor, analyser, stereo panner, delay: their own stages
    # an IIR of order <= 2 on a constant layout IS a biquad: it rides the time-parallel scan of k_chain; order >= 3 keeps the serial kernel
    k = _one(pkg, be, lambda c: src_to(c, c.create_iir_filter([0.5, 0.5], [1.0, -0.2])))
    assert "k_chain" in k and "k_iir_serial" not in k
    assert "k_iir_serial" in _one(pkg, be, lambda c: src_to(c, c.create_iir_filter([0.5, 0.5, 0.1, 0.05], [1.0, -0.2, 0.1, 0.01])))
    assert "k_compressor" in _one(pkg, be, lambda c: src_to(c, c.create_dynamics_compressor()))
    assert "k_analyser" in _one(pkg, be, lambda c: src_to(c, c.create_analyser()))
    assert "k_stereo_panner" in _one(pkg, be, lambda c: src_to(c, c.create_stereo_panner(0.3)))
    k = _one(pkg, be, lambda c: src_to(c, c.create_delay(1.0, 0.01)))
    assert "k_delay_read" in k and "k_ring_write" in k
    # equal-power panner: static source and listener -> k_panner_eq; an automated position -> k_param + k_panner_dyn
    assert "k_panner_eq" in _one(pkg, be, lambda c: src_to(c, c.create_panner(position=(1.0, 0.0, -1.0))))

    def moving(c):
        p = c.create_panner(position=(1.0, 0.0, -1.0))
        p.position_x.linear_ramp_to_value_at_time(-3.0, 0.01)
        src_to(c, p)
    k = _one(pkg, be, moving)
    assert "k_panner_dyn" in k and "k_param" in k and "k_panner_eq" not in k
    # over-sampled shaper
    assert "k_shaper_os" in _one(pkg, be, lambda c: src_to(c, c.create_wave_shaper(curve=np.linspace(-1, 1, 9).astype(np.float32), oversample=pkg.OVERSAMPLE_X2)))


def test_automation_selects_the_a_rate_kernels(pkg, be):
    def osc_fm(c):  # an LFO on the carrier's frequency: audio-rate param input -> k_param + k_osc_arate
        lfo = c.create_oscillator(frequency=5.0)
        depth = c.create_gain(30.0)
        car = c.create_oscillator(frequency=440.0)
        lfo.connect(depth)
        depth.connect(car.frequency)
        car.connect(c.destination())
        lfo.start()
        car.start()
    k = _one(pkg, be, osc_fm)
    assert "k_osc_arate" in k and "k_param" in k

    def filter_sweep(c):
        o = c.create_oscillator(type_=pkg.SAWTOOTH, frequency=110.0)
        f = c.create_biquad_filter()
        f.frequency.exponential_ramp_to_value_at_time(4000.0, 0.02)
        o.connect(f)
        f.connect(c.destination())
        o.start()
    k = _one(pkg, be, filter_sweep)
    assert "k_biquad_arate" in k and "k_param" in k

    def rate_automation(c):  # playbackRate automation: the renderer's own frame loop, one warp per source
        s = c.create_buffer_source(pkg.AudioBuffer([np.ones(4096, np.float32)], 48000.0))
        s.playback_rate.linear_ramp_to_value_at_time(2.0, 0.02)
        s.connect(c.destination())
        s.start()
    assert "k_buffer_source_serial" in _one(pkg, be, rate_automation)

    def resampled(c):  # a 38 kHz asset in a 48 kHz context: the closed-form slow track
        s = c.create_buffer_source(pkg.AudioBuffer([np.ones(4096, np.float32)], 38000.0), loop=True)
        s.connect(c.destination())
        s.start()
    assert "k_buffer_source_slow" in _one(pkg, be, resampled)


def test_chunk_sizing_follows_the_arena(pkg, be):
    # no arena (fully fused): one chunk; 64 mono voices at 1 GiB / (4 B x 64 floats per frame) would be 4 M frames -> capped to the render;
    # a long render with many edges is cut into chunks of >= 8192 frames, multiples of 2048
    p = plan(pkg, [G.c3_many_voices(pkg, be, 300, 48000 * 40)])
    assert p["arena_floats_per_frame"] == 300 and p["chunks"] > 1
    assert p["chunk_frames"] % 2048 == 0 and p["chunk_frames"] >= 8192
    assert p["chunk_frames"] * 4 * p["arena_floats_per_frame"] <= 1 << 30


@pytest.mark.parametrize("name,build", BS.CRITERION, ids=[n for n, _ in BS.CRITERION])
def test_every_criterion_bench_graph_is_lowered(pkg, be, name, build):
    # benches/my_benchmark.rs: planned without a GPU; the HRTF one stops at "needs an HRIR sphere" (the sphere belongs to an engine)
    if "hrtf" in name:
        with pytest.raises(pkg.WaeError) as e:
            plan(pkg, [build(pkg, be, 2.0)])
        assert e.value.status == 4 and "HRIR sphere" in str(e.value)
        return
    p = plan(pkg, [build(pkg, be, 2.0) for _ in range(3)])
    assert p["stages"] >= 1
    if name in ("bench_sine", "bench_sine_gain", "bench_buffer_src", "bench_buffer_src_biquad", "bench_constant_source"):
        assert p["kinds"] == {"k_chain": 1}  # fully fused into the destination


@pytest.mark.parametrize("block", range(8))
def test_planner_accepts_random_graphs(pkg, be, block):
    # the generator of tests/test_gpu_fuzz.py (random DAGs of every lowered node kind, stereo sources that end, automation, feedback
    # loops, suspend points) on the CPU: 8 x 40 seeds through the planner's sizing pass — no crash, a sane plan; the only refusals are the
    # two documented layout combinations (DESIGN.md §6), and they are rare
    import test_gpu_fuzz as F
    refused = 0
    for seed in range(1000 + 40 * block, 1000 + 40 * (block + 1)):
        try:
            p = plan(pkg, [F.random_graph(pkg, be, seed)])
        except pkg.WaeError as e:
            assert e.status == 4 and ("mono response" in str(e) or "over-sampled WaveShaperNode" in str(e)), (seed, str(e))
            refused += 1
            continue
        assert 1 <= p["stages"] <= 400 and p["segments"] >= 1 and p["chunk_frames"] >= 128, seed
    assert refused <= 6, refused


@pytest.mark.parametrize("block", range(4))
def test_the_checker_renders_the_same_random_graphs(pkg, oracle, block):
    # the oracle side of the fuzz pairs: 4 x 20 of the graphs above rendered on the CPU — finite, not silent, reproducible
    import test_gpu_fuzz as F
    for seed in range(1000 + 20 * block, 1000 + 20 * (block + 1)):
        a = F.random_graph(pkg, oracle, seed).start_rendering_sync()
        pcm = np.array([a.get_channel_data(0), a.get_channel_data(1)])
        assert np.isfinite(pcm).all(), seed
        if seed % 10 == 0:
            b = F.random_graph(pkg, oracle, seed).start_rendering_sync()
            assert np.array_equal(pcm[0], b.get_channel_data(0)) and np.array_equal(pcm[1], b.get_channel_data(1))


def test_an_audio_buffer_played_by_many_nodes_is_held_once(pkg, be):
    # the reference clones an Arc<AudioBuffer> into every AudioBufferSourceNode (src/buffer.rs:69-72): the grains of
    # examples/benchmarks.rs:351-388 all play ONE buffer.  The graph keeps one host copy per distinct PCM (copy_buffer) and the planner
    # one copy per buffer in the device slab — same samples in another array count as the same buffer, different samples do not
    rng = np.random.default_rng(3)
    pcm = rng.uniform(-1, 1, (2, 1000)).astype(np.float32)   # stride 1000 floats per channel
    other = pcm.copy()
    other[1, 999] += 0.5                                       # same shape, differs in the very last sample

    def graph(buffers):
        c = pkg.OfflineAudioContext(2, 128 * 20, 48000.0, be)
        for i, bufr in enumerate(buffers):
            s = c.create_buffer_source(pkg.AudioBuffer(list(bufr), 48000.0))
            s.connect(c.destination())
            s.start_at_with_offset_and_duration(i * 0.001, 0.0005 * i, 0.01)
        return c
    assert plan(pkg, [graph([pcm] * 12)])["source_floats"] == 2 * 1000
    assert plan(pkg, [graph([pcm, pcm.copy(), other, pcm, other.copy()])])["source_floats"] == 2 * 2 * 1000
    # not shared across graphs (each context owns its assets) ...
    assert plan(pkg, [graph([pcm] * 3), graph([pcm] * 3)])["source_floats"] == 2 * 2 * 1000
    # ... and a shorter buffer with the same leading samples is its own asset
    assert plan(pkg, [graph([pcm, pcm[:, :996]])])["source_floats"] == 2 * 1000 + 2 * 996
    # set_buffer goes through the same door
    c = pkg.OfflineAudioContext(2, 128 * 20, 48000.0, be)
    for _ in range(4):
        s = c.create_buffer_source()
        s.set_buffer(pkg.AudioBuffer(list(pcm), 48000.0))
        s.connect(c.destination())
        s.start()
    assert plan(pkg, [c])["source_floats"] == 2 * 1000


def test_split_sizing_of_a_group_agrees_with_the_serial_pass():
    # one-shot renders size a group of few, large graphs on several workers (prep_begin: size_group_split); with WAE_PLAN_PARALLEL=1
    # wae_batch_plan sizes every multi-graph group both ways and refuses with "internal: ..." when arena floats, slab size, the recorded
    # source copies, feedback or the in-cycle delay layouts differ.  (The switch is read once per process: a child process.)
    import subprocess
    import sys
    code = r"""
import sys
sys.path.insert(0, %r)
import conftest, graphs as G, test_gpu_fuzz as F, benchmark_scenarios as BS
pkg = conftest.load_package()
be = pkg.context.Backend(pkg.api(), None)
ir = G.synthetic_ir(20000, 2, decay=0.6)
batches = [[G.c2_buffer_biquad_gain(pkg, be, g, 12800) for g in range(5)],
           [G.c2_buffer_biquad_gain(pkg, be, g, 2560) for g in range(70)],
           [G.north_star_voices_convolver(pkg, be, 40, 48000, ir, seed=g) for g in range(4)],
           [G.c3_many_voices(pkg, be, 50, 4800) for _ in range(3)]]
batches += [[fn(pkg, be, 2.0) for _ in range(3)] for _name, fn in BS.SCENARIOS]
n = refused = 0
for seed in range(3000, 3120, 4):
    batches.append([F.random_graph(pkg, be, seed + i) for i in range(4)])
for ctxs in batches:
    try:
        pkg.context.plan_batch(ctxs)
        n += 1
    except pkg.WaeError as e:
        assert "internal" not in str(e), str(e)
        refused += 1
print("planned", n, "refused", refused)
""" % os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, WAE_PLAN_PARALLEL="2")  # 2: the runs of the check on real worker threads
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    planned = int(r.stdout.split()[1])
    assert planned >= 40, r.stdout


def test_plan_digests_are_reproducible_across_processes():
    # WAE_PLAN_DIGEST=1 hashes every instance record the sizing pass builds (tools/plan_digest_corpus.py compares them across library versions):
    # that only works when no record carries uninitialised bytes or host addresses — two processes must print the same digests
    import subprocess
    import sys
    code = r"""
import sys
sys.path.insert(0, %r)
import conftest, graphs as G, test_gpu_fuzz as F, benchmark_scenarios as BS
pkg = conftest.load_package()
be = pkg.context.Backend(pkg.api(), None)
ir = G.synthetic_ir(20000, 2, decay=0.6)
for ctxs in ([G.c1_osc_biquad(pkg, be, 4800)], [G.c2_buffer_biquad_gain(pkg, be, g, 2560) for g in range(6)], [G.c3_many_voices(pkg, be, 40, 4800)],
             [G.north_star_voices_convolver(pkg, be, 30, 24576, ir, seed=g) for g in range(2)]):
    pkg.context.plan_batch(ctxs)
for name, fn in BS.SCENARIOS:
    pkg.context.plan_batch([fn(pkg, be, 2.0)])
for seed in range(6000, 6060):
    try:
        pkg.context.plan_batch([F.random_graph(pkg, be, seed)])
    except pkg.WaeError:
        pass
""" % os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, WAE_PLAN_DIGEST="1")
    outs = []
    for _ in range(2):
        r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-2000:]
        outs.append([ln for ln in r.stderr.splitlines() if "plan digest" in ln])
    assert len(outs[0]) >= 80 and outs[0] == outs[1]
