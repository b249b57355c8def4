"""The reference's OWN known-answer tests, run through the CUDA path (C ABI -> sm_90a kernels) instead of the oracle.

tests/test_oracle_kat.py and tests/test_oracle_offline.py restate the reference's `#[test]`s (each names its file:line) and
pin the oracle with them; the graph-rendering ones only need a backend, so the very same functions are executed here with
the GPU engine as the backend — the parity tests then read like the reference's own tests.  Helper-only KATs (frequency
response formulas, mix matrices, Blackman window) exercise oracle hooks that have no GPU counterpart and stay CPU-only."""
import pytest

import test_oracle_kat as K
import test_oracle_offline as O

pytestmark = pytest.mark.gpu

CASES = [
    O.test_offline_render, O.test_start_stop, O.test_delayed_constant_source, O.test_audio_param_graph, O.test_cycle,
    O.test_cycle_breaker,
    K.test_iir_fir_case_exact, K.test_oscillator_sine_matches_sin, K.test_oscillator_polyblep_values,
    K.test_oscillator_start_in_middle_of_quantum, K.test_convolver_passthrough_zeroed_identity_two_id, K.test_convolver_tail_time,
    K.test_convolver_argument_errors, K.test_convolver_matches_direct_convolution, K.test_mixing_channel_count_modes,
    K.test_denormals_are_flushed, K.test_waveshaper_curves, K.test_delay_integer_and_fractional, K.test_stereo_panner_mono_and_stereo,
    K.test_equal_power_panner_positions, K.test_compressor_lookahead_delay, K.test_buffer_source_fast_and_slow_track,
    K.test_param_automation_vectors, K.test_filter_node_frequency_response_methods, K.test_iir_coefficient_validation,
    K.test_iir_one_zero_different_lengths,
]


@pytest.mark.parametrize("case", CASES, ids=lambda f: f.__name__)
def test_reference_case_on_gpu(pkg, engine, case):
    case(pkg, engine.backend)


def test_oscillator_triangle_on_gpu(pkg, engine):
    # oscillator.rs:933-998 triangle_raw demands bit equality with the f64-accumulated phase; the fused chain keeps the phase in
    # 64-bit fixed point (DESIGN.md §6): equal up to the f32 rounding of isolated samples
    K.test_oscillator_triangle_exact(pkg, engine.backend, exact=False)


@pytest.mark.parametrize("case", range(6))
def test_convolver_channel_config_on_gpu(pkg, engine, case):
    # the reference asserts abs <= 1e-7 with its 2048-point FFTs; the engine's 16384-point f32 FFT (8192-frame partitions)
    # returns 1 - 2^-23 for a unit tap: one f32 ulp at 1.0, so the bound here is 2 ulp
    K.test_convolver_channel_config(pkg, engine.backend, case, tol=2.4e-7)


# ---- src/node/audio_buffer_source.rs:974-1890, restated in tests/test_oracle_absn.py -------------------------------------
import test_oracle_absn as A  # noqa: E402

ABSN_CASES = [
    A.test_sub_quantum_start_1, A.test_sub_quantum_start_2, A.test_sub_sample_start, A.test_sub_quantum_stop, A.test_sub_sample_stop,
    A.test_start_in_the_past, A.test_playback_rate_and_detune, A.test_negative_playback_rate, A.test_end_of_file,
    A.test_with_duration_and_offset, A.test_reverse_playback_with_duration, A.test_offset_larger_than_buffer_duration,
    A.test_reverse_loop_boundaries,
]


@pytest.mark.parametrize("case", ABSN_CASES, ids=lambda f: f.__name__)
def test_buffer_source_reference_case_on_gpu(pkg, engine, case):
    case(pkg, engine.backend)


@pytest.mark.parametrize("buf_sr", [22500, 38000, 43800, 48000, 96000])
def test_buffer_source_resampling_on_gpu(pkg, engine, buf_sr):
    A.test_audio_buffer_resampling(pkg, engine.backend, buf_sr)


@pytest.mark.parametrize("buffer_len", A.LOOP_LENS)
def test_buffer_source_loops_on_gpu(pkg, engine, buffer_len):
    A.test_track_loop_mono(pkg, engine.backend, buffer_len)
    A.test_track_loop_stereo(pkg, engine.backend, buffer_len)


@pytest.mark.parametrize("bounds", [(-2.0, -1.0, 0.0), (-1.0, -2.0, 0.0), (0.0, 0.0, 0.0), (-1.0, 2.0, 0.0), (2.0, -1.0, 1e-10), (1.0, 1.0, 1e-10),
                                    (2.0, 3.0, 1e-10), (3.0, 2.0, 1e-10)])
def test_buffer_source_loop_out_of_bounds_on_gpu(pkg, engine, bounds):
    A.test_loop_out_of_bounds(pkg, engine.backend, *bounds)


# ---- src/node/delay.rs:766-1200, restated in tests/test_oracle_delay.py ----------------------------------------------------
import test_oracle_delay as D  # noqa: E402

DELAY_CASES = [D.test_sample_accurate, D.test_sub_sample_accurate, D.test_multichannel, D.test_input_number_of_channels_change,
               D.test_node_stays_alive_long_enough, D.test_subquantum_delay, D.test_min_delay_when_in_loop, D.test_max_delay,
               D.test_max_delay_smaller_than_quantum_size, D.test_max_delay_multiple_of_quantum_size, D.test_subquantum_delay_dynamic_lifetime]


@pytest.mark.parametrize("case", DELAY_CASES, ids=lambda f: f.__name__)
def test_delay_reference_case_on_gpu(pkg, engine, case):
    case(pkg, engine.backend)


# ---- src/node/oscillator.rs:806-1455, restated in tests/test_oracle_osc.py ---------------------------------------------------
import test_oracle_osc as OS  # noqa: E402

OSC_CASES = [OS.test_sine_raw, OS.test_square_and_sawtooth_raw_away_from_the_steps, OS.test_periodic_wave, OS.test_sub_quantum_and_sub_sample_start,
             OS.test_sub_quantum_and_sub_sample_stop, OS.test_stop_disarms_future_start, OS.test_start_in_the_past,
             OS.test_computed_frequency_outside_nyquist_is_silent, OS.test_delayed_start_and_negative_frequency]


@pytest.mark.parametrize("case", OSC_CASES, ids=lambda f: f.__name__)
def test_oscillator_reference_case_on_gpu(pkg, engine, case):
    case(pkg, engine.backend)


# ---- panner / constant source / merger / splitter / stereo panner / wave shaper unit tests, restated in tests/test_oracle_nodes.py ---
import test_oracle_nodes as N  # noqa: E402

NODE_CASES = [N.test_equal_power_mono_to_stereo, N.test_equal_power_azimuth_mono_to_stereo, N.test_equal_power_stereo_to_stereo,
              N.test_constant_source_start_stop, N.test_constant_source_start_in_the_past, N.test_constant_source_start_in_the_future_while_dropped,
              N.test_channel_merger, N.test_channel_merger_disconnect, N.test_channel_merger_splitter_option_errors, N.test_channel_splitter,
              N.test_stereo_panner_mono_panning, N.test_stereo_panner_stereo_panning, N.test_wave_shaper_boundaries, N.test_wave_shaper_interpolation,
              N.test_up_down_mix_rules_through_a_graph, N.test_mixing_integration_cases,
              N.test_channel_config_setters_take_effect_at_a_suspend_point, N.test_channel_config_constraints]


@pytest.mark.parametrize("case", NODE_CASES, ids=lambda f: f.__name__)
def test_node_reference_case_on_gpu(pkg, engine, case):
    case(pkg, engine.backend)


# ---- src/analysis.rs:414-868, restated in tests/test_oracle_analyser.py ---------------------------------------------------------
import test_oracle_analyser as AN  # noqa: E402

ANALYSER_CASES = [AN.test_time_domain_data_vs_fft_size, AN.test_time_domain_data_is_the_most_recent_window, AN.test_byte_time_domain_data,
                  AN.test_frequency_data_vs_frequency_bin_count, AN.test_option_constraints]


@pytest.mark.parametrize("case", ANALYSER_CASES, ids=lambda f: f.__name__)
def test_analyser_reference_case_on_gpu(pkg, engine, case):
    case(pkg, engine.backend)


@pytest.mark.parametrize("bins", [range(1, 128, 9), range(5, 128, 9)], ids=["a", "b"])
def test_analyser_sine_bins_on_gpu(pkg, engine, bins):
    AN.test_float_frequency_data_peaks_at_the_sine_bin(pkg, engine.backend, bins)


# ---- src/buffer.rs:716-816 AudioBuffer::resample, restated in tests/test_oracle_buffer.py; here through wae_resample_linear -------
import test_oracle_buffer as BU  # noqa: E402


def test_resample_up_down_and_edges_on_gpu(pkg, engine):
    BU.check_up_and_downsample(engine.resample)
    BU.check_resample_edge_cases(engine.resample)


@pytest.mark.parametrize("source_sr", [22500, 38000, 48000, 96000])
def test_resample_stereo_on_gpu(pkg, engine, source_sr):
    BU.check_resample_stereo(engine.resample, source_sr)

