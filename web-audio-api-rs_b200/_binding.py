"""ctypes binding of the C ABI declared in include/wae.h.

`Api(lib, prefix)` binds one shared library: the product (`libwae_b200.so`, prefix ``wae_``) or — from
tests/, bench.py's cpu_baseline leg and __graft_entry__.smoke() only — the CPU oracle
(prefix ``wao_``), which exports the same graph-building surface.  Nothing in this package loads the
oracle itself.
"""
import ctypes as C

import numpy as np

c_float_p = C.POINTER(C.c_float)
c_double_p = C.POINTER(C.c_double)


class ChannelConfig(C.Structure):
    _fields_ = [("count", C.c_uint32), ("count_mode", C.c_uint32), ("interpretation", C.c_uint32)]


class AudioBufferDesc(C.Structure):
    _fields_ = [("number_of_channels", C.c_uint32), ("length", C.c_uint64), ("sample_rate", C.c_float),
                ("channels", C.POINTER(c_float_p))]


class OscillatorOptions(C.Structure):
    _fields_ = [("type", C.c_uint32), ("frequency", C.c_float), ("detune", C.c_float),
                ("periodic_wave", c_float_p), ("periodic_wave_len", C.c_uint32)]


class BiquadOptions(C.Structure):
    _fields_ = [("type", C.c_uint32), ("q", C.c_float), ("detune", C.c_float), ("frequency", C.c_float),
                ("gain", C.c_float), ("channel_config", ChannelConfig)]


class IirOptions(C.Structure):
    _fields_ = [("feedforward", c_double_p), ("feedforward_len", C.c_uint32), ("feedback", c_double_p),
                ("feedback_len", C.c_uint32), ("channel_config", ChannelConfig)]


class GainOptions(C.Structure):
    _fields_ = [("gain", C.c_float), ("channel_config", ChannelConfig)]


class BufferSourceOptions(C.Structure):
    _fields_ = [("buffer", C.POINTER(AudioBufferDesc)), ("detune", C.c_float), ("playback_rate", C.c_float),
                ("loop", C.c_uint32), ("loop_start", C.c_double), ("loop_end", C.c_double)]


class ConstantSourceOptions(C.Structure):
    _fields_ = [("offset", C.c_float)]


class ConvolverOptions(C.Structure):
    _fields_ = [("buffer", C.POINTER(AudioBufferDesc)), ("disable_normalization", C.c_uint32),
                ("channel_config", ChannelConfig)]


class WaveShaperOptions(C.Structure):
    _fields_ = [("curve", c_float_p), ("curve_len", C.c_uint32), ("oversample", C.c_uint32),
                ("channel_config", ChannelConfig)]


class DelayOptions(C.Structure):
    _fields_ = [("max_delay_time", C.c_double), ("delay_time", C.c_double), ("channel_config", ChannelConfig)]


class StereoPannerOptions(C.Structure):
    _fields_ = [("pan", C.c_float), ("channel_config", ChannelConfig)]


class PannerOptions(C.Structure):
    _fields_ = [("panning_model", C.c_uint32), ("distance_model", C.c_uint32),
                ("position_x", C.c_float), ("position_y", C.c_float), ("position_z", C.c_float),
                ("orientation_x", C.c_float), ("orientation_y", C.c_float), ("orientation_z", C.c_float),
                ("ref_distance", C.c_double), ("max_distance", C.c_double), ("rolloff_factor", C.c_double),
                ("cone_inner_angle", C.c_double), ("cone_outer_angle", C.c_double), ("cone_outer_gain", C.c_double),
                ("channel_config", ChannelConfig)]


class AnalyserOptions(C.Structure):
    _fields_ = [("fft_size", C.c_uint32), ("smoothing_time_constant", C.c_double), ("min_decibels", C.c_double),
                ("max_decibels", C.c_double), ("channel_config", ChannelConfig)]


class DynamicsCompressorOptions(C.Structure):
    _fields_ = [("attack", C.c_float), ("knee", C.c_float), ("ratio", C.c_float), ("release", C.c_float),
                ("threshold", C.c_float), ("channel_config", ChannelConfig)]


class ChannelMergerOptions(C.Structure):
    _fields_ = [("number_of_inputs", C.c_uint32)]


class ChannelSplitterOptions(C.Structure):
    _fields_ = [("number_of_outputs", C.c_uint32)]


class ParamEvent(C.Structure):
    _fields_ = [("type", C.c_uint32), ("value", C.c_float), ("time", C.c_double), ("aux", C.c_double),
                ("values", c_float_p), ("values_len", C.c_uint32)]


(ATTR_LOOP, ATTR_LOOP_START, ATTR_LOOP_END, ATTR_NORMALIZE, ATTR_OVERSAMPLE, ATTR_PANNING_MODEL, ATTR_DISTANCE_MODEL, ATTR_REF_DISTANCE,
 ATTR_MAX_DISTANCE, ATTR_ROLLOFF_FACTOR, ATTR_CONE_INNER_ANGLE, ATTR_CONE_OUTER_ANGLE, ATTR_CONE_OUTER_GAIN, ATTR_FFT_SIZE,
 ATTR_SMOOTHING_TIME_CONSTANT, ATTR_MIN_DECIBELS, ATTR_MAX_DECIBELS) = range(1, 18)


class PlanInfo(C.Structure):
    _fields_ = [("groups", C.c_uint32), ("segments", C.c_uint32), ("stages", C.c_uint32), ("has_feedback", C.c_uint32),
                ("chunk_frames", C.c_uint64), ("chunks", C.c_uint64), ("arena_floats_per_frame", C.c_uint64), ("source_floats", C.c_uint64),
                ("stage_kinds", C.c_char * 512)]


class BatchStats(C.Structure):
    _fields_ = [("kernel_launches_per_run", C.c_uint64), ("stages", C.c_uint64), ("chunks", C.c_uint64),
                ("arena_bytes", C.c_uint64), ("asset_bytes", C.c_uint64), ("algorithmic_bytes", C.c_uint64),
                ("graph_quanta", C.c_uint64), ("last_run_ms", C.c_float), ("dominant_kernel_ms", C.c_float),
                ("dominant_kernel", C.c_char * 64)]


class SourceBinding(C.Structure):
    """wae_source_binding: device audio for one device input of a prepared batch (wae_batch_bind_sources)."""
    _fields_ = [("graph_index", C.c_uint32), ("node", C.c_uint32), ("pcm", c_float_p), ("channel_stride", C.c_uint64)]


class ParamBinding(C.Structure):
    """wae_param_binding: the device address of one param value of a prepared batch (wae_batch_bind_params)."""
    _fields_ = [("graph_index", C.c_uint32), ("node", C.c_uint32), ("param_index", C.c_uint32), ("value", c_float_p)]


class ResponseBinding(C.Structure):
    """wae_response_binding: the device impulse response of one declared ConvolverNode of a prepared batch (wae_batch_bind_responses)."""
    _fields_ = [("graph_index", C.c_uint32), ("node", C.c_uint32), ("pcm", c_float_p), ("channel_stride", C.c_uint64)]


class CurveBinding(C.Structure):
    """wae_curve_binding: the device curve of one declared WaveShaperNode of a prepared batch (wae_batch_bind_curves)."""
    _fields_ = [("graph_index", C.c_uint32), ("node", C.c_uint32), ("curve", c_float_p)]


class PeriodicWaveBinding(C.Structure):
    """wae_periodic_wave_binding: the device coefficients of one declared custom OscillatorNode of a prepared batch
    (wae_batch_bind_periodic_waves); either pointer may be NULL (zeros)."""
    _fields_ = [("graph_index", C.c_uint32), ("node", C.c_uint32), ("real", c_float_p), ("imag", c_float_p)]


class IirBinding(C.Structure):
    """wae_iir_binding: the device f64 coefficients of one declared IIRFilterNode of a prepared batch (wae_batch_bind_iir_coefficients)."""
    _fields_ = [("graph_index", C.c_uint32), ("node", C.c_uint32), ("feedforward", c_double_p), ("feedback", c_double_p)]


class ValueCurveBinding(C.Structure):
    """wae_value_curve_binding: the device values of one declared SetValueCurveAtTime of a prepared batch (wae_batch_bind_value_curves)."""
    _fields_ = [("graph_index", C.c_uint32), ("node", C.c_uint32), ("param_index", C.c_uint32), ("values", c_float_p)]


class ScheduleBinding(C.Structure):
    """wae_schedule_binding: the device row start, [stop], [offset], [duration] of one declared scheduled source of a prepared batch
    (wae_batch_bind_schedules)."""
    _fields_ = [("graph_index", C.c_uint32), ("node", C.c_uint32), ("times", c_double_p)]


class LoopBinding(C.Structure):
    """wae_loop_binding: the device row loop_start, loop_end of one declared looping AudioBufferSourceNode of a prepared batch
    (wae_batch_bind_loops)."""
    _fields_ = [("graph_index", C.c_uint32), ("node", C.c_uint32), ("points", c_double_p)]


STATUS_NAMES = {0: "OK", 1: "INVALID_ARGUMENT", 2: "INVALID_STATE", 3: "NOT_SUPPORTED", 4: "UNSUPPORTED",
                5: "CUDA_ERROR", 6: "OUT_OF_MEMORY", 7: "NO_DEVICE"}


class WaeError(RuntimeError):
    """A non-zero wae_status. `.status` is the code, the message is wae_last_error() (the reference's
    panic text, e.g. 'NotSupportedError - ...')."""

    def __init__(self, status, message):
        super().__init__(f"[{STATUS_NAMES.get(status, status)}] {message}")
        self.status = status
        self.message = message


CREATE_FUNCS = {
    "create_oscillator": OscillatorOptions, "create_biquad_filter": BiquadOptions, "create_iir_filter": IirOptions,
    "create_gain": GainOptions, "create_buffer_source": BufferSourceOptions,
    "create_constant_source": ConstantSourceOptions, "create_convolver": ConvolverOptions,
    "create_wave_shaper": WaveShaperOptions, "create_delay": DelayOptions,
    "create_stereo_panner": StereoPannerOptions, "create_panner": PannerOptions, "create_analyser": AnalyserOptions,
    "create_dynamics_compressor": DynamicsCompressorOptions, "create_channel_merger": ChannelMergerOptions,
    "create_channel_splitter": ChannelSplitterOptions,
}

READOUT_FREQUENCY, READOUT_TIME_DOMAIN = 1, 2  # WAE_READOUT_*

# every symbol include/wae.h declares (tests check the product exports all of them)
WAE_SYMBOLS = [
    "wae_engine_create", "wae_engine_destroy", "wae_last_error", "wae_version", "wae_engine_set_option", "wae_engine_stream",
    "wae_graph_create", "wae_graph_destroy",
] + ["wae_" + n for n in CREATE_FUNCS] + [
    "wae_connect", "wae_connect_param", "wae_disconnect", "wae_param_event_push", "wae_param_set_automation_rate",
    "wae_listener_param_event_push", "wae_source_start", "wae_source_stop", "wae_oscillator_set_type",
    "wae_biquad_set_type", "wae_render_batch", "wae_batch_prepare", "wae_batch_upload", "wae_batch_set_timing", "wae_batch_run", "wae_batch_run_pipelined", "wae_batch_sync", "wae_batch_group_count", "wae_batch_group_range", "wae_batch_run_group", "wae_host_alloc", "wae_host_free", "wae_host_register", "wae_host_unregister", "wae_selftest_conv_fft", "wae_param_sim_speculation",
    "wae_batch_output_device_ptr", "wae_batch_fetch", "wae_batch_destroy", "wae_batch_get_stats", "wae_batch_stage_time",
    "wae_analyser_get_float_time_domain_data", "wae_analyser_get_float_frequency_data", "wae_resample_linear", "wae_compressor_reduction", "wae_analyser_get_byte_time_domain_data", "wae_analyser_get_byte_frequency_data", "wae_engine_set_hrir_sphere", "wae_graph_suspend", "wae_param_sim_create", "wae_param_sim_destroy", "wae_param_sim_push",
    "wae_param_sim_set_automation_rate", "wae_param_sim_compute", "wae_biquad_coefs", "wae_biquad_frequency_response", "wae_iir_frequency_response",
    "wae_node_set_channel_count", "wae_node_set_channel_count_mode", "wae_node_set_channel_interpretation", "wae_graph_render_order", "wae_hrir_resample", "wae_batch_plan", "wae_buffer_source_set_buffer", "wae_convolver_set_buffer", "wae_wave_shaper_set_curve",
    "wae_oscillator_set_periodic_wave", "wae_node_set_attribute", "wae_disconnect_from", "wae_disconnect_param", "wae_periodic_wave_table", "wae_param_sim_set_walker", "wae_sched_first_frame_at_or_after", "wae_spatial_params", "wae_hrtf_locate",
    "wae_render_many", "wae_batch_prepare_many", "wae_batch_graph_output", "wae_batch_fetch_graph", "wae_batch_plan_many", "wae_batch_plan_quanta",
    "wae_buffer_source_set_device_input", "wae_buffer_source_set_device_input_by_reference", "wae_batch_bind_sources",
    "wae_param_set_device_value", "wae_batch_bind_params",
    "wae_convolver_set_device_response", "wae_batch_bind_responses",
    "wae_wave_shaper_set_device_curve", "wae_batch_bind_curves",
    "wae_oscillator_set_device_periodic_wave", "wae_batch_bind_periodic_waves",
    "wae_iir_filter_set_device_coefficients", "wae_batch_bind_iir_coefficients",
    "wae_param_set_device_value_curve", "wae_batch_bind_value_curves",
    "wae_source_set_device_schedule", "wae_batch_bind_schedules", "wae_buffer_source_set_device_offset",
    "wae_buffer_source_set_device_loop", "wae_batch_bind_loops",
    "wae_batch_bind_output",
    "wae_analyser_set_readouts", "wae_batch_analyser_readouts_device_ptr", "wae_batch_fetch_analyser_readouts",
    "wae_analyser_set_byte_readouts", "wae_batch_analyser_byte_readouts_device_ptr", "wae_batch_fetch_analyser_byte_readouts",
    "wae_compressor_set_readouts", "wae_batch_compressor_readouts_device_ptr", "wae_batch_fetch_compressor_readouts",
]


class Api:
    """One bound library. `prefix` is 'wae_' (product) or 'wao_' (oracle)."""

    def __init__(self, lib, prefix):
        self.lib = lib
        self.prefix = prefix
        self.is_product = prefix == "wae_"
        f = self._f
        f("last_error", C.c_char_p, [])
        gp = C.c_void_p
        for name, opt in CREATE_FUNCS.items():
            f(name, C.c_int32, [gp, C.POINTER(opt), C.POINTER(C.c_uint32)])
        f("graph_destroy", C.c_int32, [gp])
        if self.is_product:
            f("graph_render_order", C.c_int32, [gp, C.POINTER(C.c_uint32), C.c_uint32, C.POINTER(C.c_uint32)])
        else:
            f("render_order", C.c_uint32, [gp, C.POINTER(C.c_uint32), C.c_uint32])
        f("graph_suspend", C.c_int32, [gp, C.c_double])
        f("param_sim_create", C.c_int32, [C.c_uint32, C.c_float, C.c_float, C.c_float, C.POINTER(C.c_void_p)])
        f("param_sim_destroy", C.c_int32, [C.c_void_p])
        f("param_sim_push", C.c_int32, [C.c_void_p, C.POINTER(ParamEvent)])
        f("param_sim_set_automation_rate", C.c_int32, [C.c_void_p, C.c_uint32])
        f("param_sim_compute", C.c_int32, [C.c_void_p, C.c_double, C.c_double, C.c_uint32, c_float_p, C.POINTER(C.c_uint32)])
        if self.is_product:
            f("param_sim_set_walker", C.c_int32, [C.c_void_p, C.c_uint32])
            f("param_sim_speculation", C.c_int32, [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)])
            f("selftest_conv_fft", C.c_int32, [c_float_p, C.c_uint32])
            f("sched_first_frame_at_or_after", C.c_int32, [C.c_float, C.c_double, C.POINTER(C.c_int64), C.POINTER(C.c_double)])
        f("connect", C.c_int32, [gp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32])
        f("connect_param", C.c_int32, [gp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32])
        f("disconnect", C.c_int32, [gp, C.c_uint32])
        f("disconnect_from", C.c_int32, [gp, C.c_uint32, C.c_int32, C.c_uint32, C.c_int32])
        f("disconnect_param", C.c_int32, [gp, C.c_uint32, C.c_int32, C.c_uint32, C.c_uint32])
        f("param_event_push", C.c_int32, [gp, C.c_uint32, C.c_uint32, C.POINTER(ParamEvent)])
        f("param_set_automation_rate", C.c_int32, [gp, C.c_uint32, C.c_uint32, C.c_uint32])
        f("listener_param_event_push", C.c_int32, [gp, C.c_uint32, C.POINTER(ParamEvent)])
        f("source_start", C.c_int32, [gp, C.c_uint32, C.c_double, C.c_double, C.c_double])
        f("source_stop", C.c_int32, [gp, C.c_uint32, C.c_double])
        f("oscillator_set_type", C.c_int32, [gp, C.c_uint32, C.c_uint32])
        f("biquad_set_type", C.c_int32, [gp, C.c_uint32, C.c_uint32])
        f("buffer_source_set_buffer", C.c_int32, [gp, C.c_uint32, C.POINTER(AudioBufferDesc)])
        f("convolver_set_buffer", C.c_int32, [gp, C.c_uint32, C.POINTER(AudioBufferDesc)])
        f("wave_shaper_set_curve", C.c_int32, [gp, C.c_uint32, c_float_p, C.c_uint32])
        f("oscillator_set_periodic_wave", C.c_int32, [gp, C.c_uint32, c_float_p, C.c_uint32])
        f("node_set_attribute", C.c_int32, [gp, C.c_uint32, C.c_uint32, C.c_double])
        f("spatial_params", C.c_int32, [C.c_uint32, c_double_p, c_float_p, c_float_p])
        f("hrtf_locate", C.c_int32, [c_float_p, C.POINTER(C.c_uint32), C.c_uint32, c_float_p, C.POINTER(C.c_uint32), c_float_p])
        f("periodic_wave_table", C.c_int32, [c_float_p, c_float_p, C.c_uint32, C.c_uint32, c_float_p, C.c_uint32])
        f("hrir_resample", C.c_int32, [c_float_p, C.c_uint32, C.c_double, c_float_p, C.c_uint32, C.POINTER(C.c_uint32)])
        for name in ("node_set_channel_count", "node_set_channel_count_mode", "node_set_channel_interpretation"):
            f(name, C.c_int32, [gp, C.c_uint32, C.c_uint32])
        f("biquad_coefs", None, [C.c_uint32, C.c_double, C.c_double, C.c_double, C.c_double, c_double_p])
        f("biquad_frequency_response", None, [C.c_uint32, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float,
                                              c_float_p, c_float_p, c_float_p, C.c_uint32])
        f("iir_frequency_response", None, [c_double_p, C.c_uint32, c_double_p, C.c_uint32, C.c_float,
                                           c_float_p, c_float_p, c_float_p, C.c_uint32])
        if self.is_product:
            f("version", C.c_char_p, [])
            f("engine_create", C.c_int32, [C.c_int32, C.POINTER(C.c_void_p)])
            f("engine_destroy", C.c_int32, [C.c_void_p])
            f("engine_set_option", C.c_int32, [C.c_void_p, C.c_uint32, C.c_int64])
            f("engine_stream", C.c_int32, [C.c_void_p, C.POINTER(C.c_void_p)])
            f("graph_create", C.c_int32, [C.c_void_p, C.c_uint32, C.c_uint64, C.c_float, C.POINTER(C.c_void_p)])
            f("render_batch", C.c_int32, [C.c_void_p, C.POINTER(C.c_void_p), C.c_uint32, C.c_void_p, C.c_uint32])
            f("batch_prepare", C.c_int32, [C.c_void_p, C.POINTER(C.c_void_p), C.c_uint32, C.POINTER(C.c_void_p)])
            f("batch_plan", C.c_int32, [C.POINTER(C.c_void_p), C.c_uint32, C.POINTER(PlanInfo)])
            f("batch_upload", C.c_int32, [C.c_void_p])
            f("batch_set_timing", C.c_int32, [C.c_void_p, C.c_uint32])
            f("batch_run", C.c_int32, [C.c_void_p])
            f("batch_run_pipelined", C.c_int32, [C.c_void_p, C.c_void_p])
            f("batch_sync", C.c_int32, [C.c_void_p])
            f("host_alloc", C.c_int32, [C.c_void_p, C.c_uint64, C.POINTER(C.c_void_p)])
            f("host_free", C.c_int32, [C.c_void_p, C.c_void_p])
            f("host_register", C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint64])
            f("host_unregister", C.c_int32, [C.c_void_p, C.c_void_p])
            f("batch_group_count", C.c_int32, [C.c_void_p, C.POINTER(C.c_uint32)])
            f("batch_group_range", C.c_int32, [C.c_void_p, C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)])
            f("batch_run_group", C.c_int32, [C.c_void_p, C.c_uint32])
            f("batch_output_device_ptr", C.c_int32, [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)])
            f("batch_fetch", C.c_int32, [C.c_void_p, C.c_void_p])
            f("batch_destroy", C.c_int32, [C.c_void_p])
            f("batch_get_stats", C.c_int32, [C.c_void_p, C.POINTER(BatchStats)])
            f("batch_stage_time", C.c_int32, [C.c_void_p, C.c_uint32, C.c_char_p, c_float_p, C.POINTER(C.c_uint32)])
            f("analyser_get_float_time_domain_data", C.c_int32, [C.c_void_p, C.c_uint32, C.c_uint32, c_float_p, C.c_uint32])
            f("analyser_get_float_frequency_data", C.c_int32, [C.c_void_p, C.c_uint32, C.c_uint32, c_float_p, C.c_uint32])
            f("compressor_reduction", C.c_int32, [C.c_void_p, C.c_uint32, C.c_uint32, c_float_p])
            f("analyser_get_byte_time_domain_data", C.c_int32, [C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(C.c_uint8), C.c_uint32])
            f("analyser_get_byte_frequency_data", C.c_int32, [C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(C.c_uint8), C.c_uint32])
            f("engine_set_hrir_sphere", C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint64])
            f("resample_linear", C.c_int32, [C.c_void_p, c_float_p, C.c_uint64, C.c_float, C.c_float, c_float_p, C.c_uint64, C.POINTER(C.c_uint64)])
            # contexts of different shapes in one batch
            f("render_many", C.c_int32, [C.c_void_p, C.POINTER(C.c_void_p), C.c_uint32, C.POINTER(c_float_p)])
            f("batch_prepare_many", C.c_int32, [C.c_void_p, C.POINTER(C.c_void_p), C.c_uint32, C.POINTER(C.c_void_p)])
            f("batch_graph_output", C.c_int32, [C.c_void_p, C.c_uint32, C.POINTER(C.c_uint64), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)])
            f("batch_fetch_graph", C.c_int32, [C.c_void_p, C.c_uint32, c_float_p])
            f("batch_plan_many", C.c_int32, [C.POINTER(C.c_void_p), C.c_uint32, C.POINTER(PlanInfo)])
            f("batch_plan_quanta", C.c_int32, [C.POINTER(C.c_void_p), C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)])
            # source audio bound from device memory
            f("buffer_source_set_device_input", C.c_int32, [gp, C.c_uint32, C.c_uint32, C.c_uint64, C.c_float])
            f("buffer_source_set_device_input_by_reference", C.c_int32, [gp, C.c_uint32, C.c_uint32, C.c_uint64, C.c_float])
            f("batch_bind_sources", C.c_int32, [C.c_void_p, C.POINTER(SourceBinding), C.c_uint32, C.c_void_p])
            # param values bound from device memory
            f("param_set_device_value", C.c_int32, [gp, C.c_uint32, C.c_uint32, C.c_float, C.c_float])
            f("batch_bind_params", C.c_int32, [C.c_void_p, C.POINTER(ParamBinding), C.c_uint32, C.c_void_p])
            # convolver responses bound from device memory
            f("convolver_set_device_response", C.c_int32, [gp, C.c_uint32, C.c_uint32, C.c_uint64, C.c_float])
            f("batch_bind_responses", C.c_int32, [C.c_void_p, C.POINTER(ResponseBinding), C.c_uint32, C.c_void_p])
            # WaveShaper curves bound from device memory
            f("wave_shaper_set_device_curve", C.c_int32, [gp, C.c_uint32, C.c_uint32])
            f("batch_bind_curves", C.c_int32, [C.c_void_p, C.POINTER(CurveBinding), C.c_uint32, C.c_void_p])
            # periodic waves bound from device memory
            f("oscillator_set_device_periodic_wave", C.c_int32, [gp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32])
            f("batch_bind_periodic_waves", C.c_int32, [C.c_void_p, C.POINTER(PeriodicWaveBinding), C.c_uint32, C.c_void_p])
            # IIR coefficients bound from device memory
            f("iir_filter_set_device_coefficients", C.c_int32, [gp, C.c_uint32])
            f("batch_bind_iir_coefficients", C.c_int32, [C.c_void_p, C.POINTER(IirBinding), C.c_uint32, C.c_void_p])
            # AudioParam value curves bound from device memory
            f("param_set_device_value_curve", C.c_int32, [gp, C.c_uint32, C.c_uint32, C.c_uint32, C.c_double, C.c_double])
            f("batch_bind_value_curves", C.c_int32, [C.c_void_p, C.POINTER(ValueCurveBinding), C.c_uint32, C.c_void_p])
            # start / stop times bound from device memory
            f("source_set_device_schedule", C.c_int32, [gp, C.c_uint32, C.c_double, C.c_double, C.c_int32, C.c_double, C.c_double])
            f("batch_bind_schedules", C.c_int32, [C.c_void_p, C.POINTER(ScheduleBinding), C.c_uint32, C.c_void_p])
            f("buffer_source_set_device_offset", C.c_int32, [gp, C.c_uint32, C.c_double, C.c_double, C.c_int32, C.c_double, C.c_double])
            # loop points bound from device memory
            f("buffer_source_set_device_loop", C.c_int32, [gp, C.c_uint32, C.c_double, C.c_double, C.c_double, C.c_double])
            f("batch_bind_loops", C.c_int32, [C.c_void_p, C.POINTER(LoopBinding), C.c_uint32, C.c_void_p])
            # rendered PCM written to caller device memory
            f("batch_bind_output", C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p])
            # analyser read-outs at declared render times
            f("analyser_set_readouts", C.c_int32, [gp, C.c_uint32, c_double_p, C.c_uint32, C.c_uint32])
            f("batch_analyser_readouts_device_ptr", C.c_int32, [C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(c_float_p), C.POINTER(C.c_uint64)])
            f("batch_fetch_analyser_readouts", C.c_int32, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, c_float_p, C.c_uint64])
            f("analyser_set_byte_readouts", C.c_int32, [gp, C.c_uint32, C.c_uint32])
            f("batch_analyser_byte_readouts_device_ptr", C.c_int32, [C.c_void_p, C.c_uint32, C.c_uint32, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)])
            f("batch_fetch_analyser_byte_readouts", C.c_int32, [C.c_void_p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p, C.c_uint64])
            # compressor reduction read-outs at declared render times
            f("compressor_set_readouts", C.c_int32, [gp, C.c_uint32, c_double_p, C.c_uint32])
            f("batch_compressor_readouts_device_ptr", C.c_int32, [C.c_void_p, C.c_uint32, C.POINTER(c_float_p), C.POINTER(C.c_uint64)])
            f("batch_fetch_compressor_readouts", C.c_int32, [C.c_void_p, C.c_uint32, C.c_uint32, c_float_p, C.c_uint64])
        else:
            f("graph_create", C.c_int32, [C.c_uint32, C.c_uint64, C.c_float, C.POINTER(C.c_void_p)])
            f("render", C.c_int32, [gp, c_float_p])
            f("render_many", C.c_int32, [C.POINTER(C.c_void_p), C.c_uint32, c_float_p, C.c_uint32, c_double_p])
            f("analyser_get_float_time_domain_data", C.c_int32, [gp, C.c_uint32, c_float_p, C.c_uint32])
            f("analyser_get_float_frequency_data", C.c_int32, [gp, C.c_uint32, c_float_p, C.c_uint32])
            f("analyser_get_byte_frequency_data", C.c_int32, [gp, C.c_uint32, C.POINTER(C.c_uint8), C.c_uint32])
            f("analyser_get_byte_time_domain_data", C.c_int32, [gp, C.c_uint32, C.POINTER(C.c_uint8), C.c_uint32])
            f("compressor_reduction", C.c_int32, [gp, C.c_uint32, c_float_p])
            f("blackman", None, [C.c_uint32, c_float_p])
            f("db_to_lin", C.c_float, [C.c_float])
            f("lin_to_db", C.c_float, [C.c_float])
            f("set_hrir_sphere", C.c_int32, [C.c_void_p, C.c_uint64])
            f("convolver_normalize", C.c_float, [C.POINTER(AudioBufferDesc)])
            f("resample_linear", C.c_uint64, [c_float_p, C.c_uint64, C.c_float, C.c_float, c_float_p, C.c_uint64])
            f("mix", None, [c_float_p, C.c_uint32, C.c_uint32, C.c_uint32, c_float_p])

    def _f(self, name, restype, argtypes):
        fn = getattr(self.lib, self.prefix + name)
        fn.restype = restype
        fn.argtypes = argtypes
        setattr(self, name, fn)

    def check(self, status):
        if status != 0:
            msg = self.last_error()
            raise WaeError(status, msg.decode() if msg else "")


def as_f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def fptr(a):
    return a.ctypes.data_as(c_float_p)


def buffer_desc(channels, sample_rate):
    """channels: list of contiguous float32 arrays of equal length. Returns (desc, keepalive)."""
    chans = [as_f32(c) for c in channels]
    n = len(chans)
    arr = (c_float_p * n)(*[fptr(c) for c in chans])
    d = AudioBufferDesc(n, len(chans[0]) if n else 0, float(sample_rate), arr)
    return d, (chans, arr)
