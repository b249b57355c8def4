"""Host-side mirror of the reference's control API for the OfflineAudioContext path.

Same names and argument meaning as web-audio-api-rs:
  OfflineAudioContext::new / create_* / destination / start_rendering_sync   (src/context/offline.rs, base.rs)
  AudioNode::connect / connect_from_output_to_input / disconnect               (src/node/audio_node.rs:224-466)
  AudioScheduledSourceNode::start / start_at / stop / stop_at                  (src/node/scheduled_source.rs)
  AudioParam::value / set_value / *_at_time                                    (src/param.rs:336-662)
so that the parity tests read like the reference's own `#[test]`s.  Everything is forwarded through the
C ABI of include/wae.h; errors surface as WaeError carrying the reference's panic text.

One addition that the reference does not have: `render_batch([ctx, ...])` renders many independent
OfflineAudioContexts in ONE engine call — the whole point of the GPU engine.
"""
import ctypes as C
import math

import numpy as np

from . import _binding as B

F64_MAX = 1.7976931348623157e308

# enums, same order as the reference
SINE, SQUARE, SAWTOOTH, TRIANGLE, CUSTOM = range(5)
LOWPASS, HIGHPASS, BANDPASS, NOTCH, ALLPASS, PEAKING, LOWSHELF, HIGHSHELF = range(8)
MAX, CLAMPED_MAX, EXPLICIT = range(3)
SPEAKERS, DISCRETE = range(2)
EQUALPOWER, HRTF = range(2)
LINEAR, INVERSE, EXPONENTIAL = range(3)
OVERSAMPLE_NONE, OVERSAMPLE_X2, OVERSAMPLE_X4 = range(3)


class Backend:
    """An Api plus (for the product) an engine handle."""

    def __init__(self, api, engine=None, device=0):
        import weakref
        self.api = api
        self.engine = engine
        self.device = device  # CUDA device ordinal of the engine
        self.batches = weakref.WeakSet()  # live wae_batch handles: destroyed before their engine (Engine.close)
        self.closed = False

    def close_batches(self):
        for b in list(self.batches):
            b.destroy()
        self.closed = True

    def set_hrir_sphere(self, data):
        """load_hrtf_processor (src/node/panner.rs:39-68): hand over the bytes of the HRIR sphere (IRC_1003_C.bin format)."""
        buf = C.create_string_buffer(bytes(data), len(data))
        if self.api.is_product:
            self.api.check(self.api.engine_set_hrir_sphere(self.engine, C.cast(buf, C.c_void_p), len(data)))
        else:
            self.api.check(self.api.set_hrir_sphere(C.cast(buf, C.c_void_p), len(data)))


class AudioBuffer:
    """Planar f32 PCM (src/buffer.rs:69-72)."""

    def __init__(self, channels, sample_rate):
        self.channels = [B.as_f32(c) for c in channels]
        # AudioBuffer::from (src/buffer.rs:96-117) panics on ragged channels
        if any(len(c) != len(self.channels[0]) for c in self.channels):
            raise B.WaeError(2, "all channels of an AudioBuffer must have the same length")
        self.sample_rate = float(np.float32(sample_rate))

    @classmethod
    def zeros(cls, number_of_channels, length, sample_rate):
        return cls([np.zeros(length, np.float32) for _ in range(number_of_channels)], sample_rate)

    def number_of_channels(self):
        return len(self.channels)

    def length(self):
        return len(self.channels[0]) if self.channels else 0

    def duration(self):
        return self.length() / self.sample_rate

    def get_channel_data(self, i):
        return self.channels[i]

    def copy_to_channel(self, data, i):
        d = B.as_f32(data)
        self.channels[i][: len(d)] = d

    def _desc(self):
        return B.buffer_desc(self.channels, self.sample_rate)


def channel_config(count=0, count_mode=MAX, interpretation=SPEAKERS):
    """AudioNodeOptions; count == 0 selects the node's default config."""
    return B.ChannelConfig(count, count_mode, interpretation)


class AudioParam:
    def __init__(self, ctx, node_id, index, value, min_value=-3.4028234663852886e38, max_value=3.4028234663852886e38):
        self._ctx, self._node, self._index = ctx, node_id, index
        self._value = float(np.float32(value))
        self._min, self._max = min_value, max_value

    def _push(self, type_, value=0.0, time=0.0, aux=0.0, values=None):
        ev = B.ParamEvent(type_, float(value), float(time), float(aux), None, 0)
        keep = None
        if values is not None:
            keep = B.as_f32(values)
            ev.values = B.fptr(keep)
            ev.values_len = len(keep)
        api = self._ctx._api
        if self._node == "listener":
            api.check(api.listener_param_event_push(self._ctx._g, self._index, C.byref(ev)))
        else:
            api.check(api.param_event_push(self._ctx._g, self._node, self._index, C.byref(ev)))
        return self

    def value(self):
        return self._value

    def set_value(self, v):
        self._push(0, v)
        self._value = min(max(float(np.float32(v)), self._min), self._max)
        return self

    def set_value_at_time(self, v, start_time):
        return self._push(1, v, start_time)

    def linear_ramp_to_value_at_time(self, v, end_time):
        return self._push(2, v, end_time)

    def exponential_ramp_to_value_at_time(self, v, end_time):
        return self._push(3, v, end_time)

    def cancel_scheduled_values(self, cancel_time):
        return self._push(4, 0.0, cancel_time)

    def set_target_at_time(self, v, start_time, time_constant):
        return self._push(5, v, start_time, time_constant)

    def cancel_and_hold_at_time(self, cancel_time):
        return self._push(6, 0.0, cancel_time)

    def set_value_curve_at_time(self, values, start_time, duration):
        return self._push(7, 0.0, start_time, duration, values)

    def set_device_value(self, lo=None, hi=None):
        """wae_param_set_device_value (product only): the param's value is supplied per run from device memory by Batch.bind_params,
        clamped to [lo, hi] within [minValue, maxValue] (default: the whole range).  It renders as a constant over the render; until
        bound, the batch is planned with the current value clamped to the range.  An OscillatorNode's frequency and detune need a range
        whose computed frequencies (with the other param's range or value) all lie in (0, sampleRate / 2), so the whole range is refused
        (WaeError status 4): bind a wider pitch with set_device_value_curve.  A PannerNode's position and orientation and the
        AudioListener's position, forward and up are bindable too, over a range inside [-1e9, 1e9] (a wider one, the default
        included, is refused with status 4): a static panner keeps its static lowering (HRTF as a convolver included), and the bind
        re-derives its direction, gains and HRTF response."""
        api = self._ctx._api
        if not api.is_product:
            raise B.WaeError(3, "params bound from device memory are a feature of the GPU engine")
        lo = -3.4028234663852886e38 if lo is None else float(lo)
        hi = 3.4028234663852886e38 if hi is None else float(hi)
        api.check(api.param_set_device_value(self._ctx._g, 1 if self._node == "listener" else self._node, self._index, lo, hi))
        return self

    def set_device_value_curve(self, length, start_time, duration):
        """wae_param_set_device_value_curve (product only): one setValueCurveAtTime of `length` values at [start_time, start_time +
        duration) whose values Batch.bind_value_curves supplies from device memory before each run.  The param takes no further events."""
        api = self._ctx._api
        if not api.is_product:
            raise B.WaeError(3, "value curves bound from device memory are a feature of the GPU engine")
        if self._node == "listener":
            raise B.WaeError(1, "AudioListener params cannot be bound from device memory")
        api.check(api.param_set_device_value_curve(self._ctx._g, self._node, self._index, int(length), float(start_time), float(duration)))
        self._ctx._device_value_curves[(int(self._node), int(self._index))] = int(length)
        return self

    def set_automation_rate(self, rate):
        api = self._ctx._api
        api.check(api.param_set_automation_rate(self._ctx._g, self._node, self._index, 0 if rate in ("a", "A", 0) else 1))


class AudioNode:
    def __init__(self, ctx, node_id, n_inputs=1, n_outputs=1):
        self._ctx, self.id = ctx, node_id
        self._n_inputs, self._n_outputs = n_inputs, n_outputs

    def number_of_inputs(self):
        return self._n_inputs

    def number_of_outputs(self):
        return self._n_outputs

    def _set_attribute(self, attribute, value):
        api = self._ctx._api
        api.check(api.node_set_attribute(self._ctx._g, self.id, attribute, float(value)))

    def _set_buffer(self, fn, buffer):
        d, keep = buffer._desc()
        self._ctx._keep.append((d, keep))
        api = self._ctx._api
        api.check(getattr(api, fn)(self._ctx._g, self.id, C.byref(d)))

    # AudioNode::set_channel_count / set_channel_count_mode / set_channel_interpretation (src/node/audio_node.rs:417-441)
    def set_channel_count(self, count):
        api = self._ctx._api
        api.check(api.node_set_channel_count(self._ctx._g, self.id, int(count)))

    def set_channel_count_mode(self, mode):
        api = self._ctx._api
        api.check(api.node_set_channel_count_mode(self._ctx._g, self.id, int(mode)))

    def set_channel_interpretation(self, interpretation):
        api = self._ctx._api
        api.check(api.node_set_channel_interpretation(self._ctx._g, self.id, int(interpretation)))

    def connect(self, dest):
        return self.connect_from_output_to_input(dest, 0, 0)

    def connect_from_output_to_input(self, dest, output, input):
        api = self._ctx._api
        if isinstance(dest, AudioParam):
            api.check(api.connect_param(self._ctx._g, self.id, output, 1 if dest._node == "listener" else dest._node, dest._index))
        else:
            if dest._ctx is not self._ctx:
                raise B.WaeError(1, "InvalidAccessError - Attempting to connect nodes from different contexts")
            api.check(api.connect(self._ctx._g, self.id, output, dest.id, input))
        return dest

    def disconnect(self):
        api = self._ctx._api
        api.check(api.disconnect(self._ctx._g, self.id))

    # the selective forms, src/node/audio_node.rs:304-405
    def _disconnect_from(self, output, dest, input):
        api = self._ctx._api
        if isinstance(dest, AudioParam):
            owner = 1 if dest._node == "listener" else dest._node
            api.check(api.disconnect_param(self._ctx._g, self.id, output, owner, dest._index))
        else:
            if dest is not None and dest._ctx is not self._ctx:
                raise B.WaeError(1, "InvalidAccessError - Attempting to disconnect nodes from different contexts")
            api.check(api.disconnect_from(self._ctx._g, self.id, output, 0xFFFFFFFF if dest is None else dest.id, input))

    def disconnect_dest(self, dest):
        self._disconnect_from(-1, dest, -1)

    def disconnect_output(self, output):
        self._disconnect_from(output, None, -1)

    def disconnect_dest_from_output(self, dest, output):
        self._disconnect_from(output, dest, -1)

    def disconnect_dest_from_output_to_input(self, dest, output, input):
        self._disconnect_from(output, dest, input)


class AudioScheduledSourceNode(AudioNode):
    def start(self):
        self.start_at(0.0)  # context.current_time() is 0 before an offline render

    def start_at(self, when):
        api = self._ctx._api
        api.check(api.source_start(self._ctx._g, self.id, when, 0.0, F64_MAX))

    def stop(self):
        self.stop_at(0.0)

    def stop_at(self, when):
        api = self._ctx._api
        api.check(api.source_stop(self._ctx._g, self.id, when))

    def set_device_schedule(self, start, stop=None):
        """wae_source_set_device_schedule (product only): the start time of this started source (and, given `stop`, its stop time) is
        supplied by Batch.bind_schedules from device memory before each run, clamped to the window `start` = (lo, hi) (`stop` = (lo, hi)).
        The node takes no further start / stop."""
        api = self._ctx._api
        if not api.is_product:
            raise B.WaeError(3, "schedules bound from device memory are a feature of the GPU engine")
        s_lo, s_hi = (float(x) for x in start)
        t_lo, t_hi = (0.0, 0.0) if stop is None else (float(x) for x in stop)
        api.check(api.source_set_device_schedule(self._ctx._g, self.id, s_lo, s_hi, 0 if stop is None else 1, t_lo, t_hi))
        self._ctx._device_schedules[self.id] = (stop is not None, False, False)
        return self


class OscillatorNode(AudioScheduledSourceNode):
    def set_periodic_wave(self, table):
        """OscillatorNode::set_periodic_wave (oscillator.rs:334-337); `table` = PeriodicWave's wavetable (periodic_wave.rs:163-209)."""
        t = B.as_f32(table)
        api = self._ctx._api
        api.check(api.oscillator_set_periodic_wave(self._ctx._g, self.id, B.fptr(t), len(t)))

    def set_device_periodic_wave(self, coefficients, table_length=8192, disable_normalization=False):
        """wae_oscillator_set_device_periodic_wave (product only): the node plays the wavetable of `table_length` points (8192, the
        reference's PERIODIC_WAVE_TABLE_LENGTH, by default) that Batch.bind_periodic_waves synthesises from `coefficients` (real, imag)
        pairs of device memory before each run.  Counts as the node's set_periodic_wave."""
        api = self._ctx._api
        if not api.is_product:
            raise B.WaeError(3, "periodic waves bound from device memory are a feature of the GPU engine")
        api.check(api.oscillator_set_device_periodic_wave(self._ctx._g, self.id, int(coefficients), int(table_length),
                                                          1 if disable_normalization else 0))
        self._ctx._device_waves[self.id] = int(coefficients)

    def set_type(self, type_):
        api = self._ctx._api
        api.check(api.oscillator_set_type(self._ctx._g, self.id, type_))


class AudioBufferSourceNode(AudioScheduledSourceNode):
    # audio_buffer_source.rs:278-349
    def set_buffer(self, buffer):
        self._set_buffer("buffer_source_set_buffer", buffer)

    def set_device_input(self, number_of_channels, length, sample_rate, by_reference=False):
        """wae_buffer_source_set_device_input (product only): the node plays audio of this shape that Batch.bind_sources supplies from
        device memory before each run, instead of an AudioBuffer.  Counts as the node's buffer.
        by_reference (wae_buffer_source_set_device_input_by_reference): the runs read the bound tensor where it lies, and the batch keeps
        no copy of it.  The tensor must then stay unchanged while runs that read it are queued: write it in place only after
        Batch.output_tensor() or Batch.sync() has ordered torch after those runs (a ring of input tensors follows that rule)."""
        api = self._ctx._api
        if not api.is_product:
            raise B.WaeError(3, "device inputs are a feature of the GPU engine")
        declare = api.buffer_source_set_device_input_by_reference if by_reference else api.buffer_source_set_device_input
        api.check(declare(self._ctx._g, self.id, int(number_of_channels), int(length), float(sample_rate)))
        self._ctx._device_inputs[self.id] = (int(number_of_channels), int(length))
        if by_reference:
            self._ctx._source_refs.add(self.id)

    def set_loop(self, value):
        self._set_attribute(B.ATTR_LOOP, 1.0 if value else 0.0)

    def set_loop_start(self, value):
        self._set_attribute(B.ATTR_LOOP_START, value)

    def set_loop_end(self, value):
        self._set_attribute(B.ATTR_LOOP_END, value)

    def start_at_with_offset(self, start, offset):
        self.start_at_with_offset_and_duration(start, offset, F64_MAX)

    def start_at_with_offset_and_duration(self, start, offset, duration):
        api = self._ctx._api
        api.check(api.source_start(self._ctx._g, self.id, start, offset, duration))

    def set_device_schedule(self, start, stop=None, offset=None, duration=None):
        """As for every scheduled source; given `offset` = (lo, hi) (and `duration` = (lo, hi)), the offset (and duration) of
        start_at_with_offset_and_duration are supplied by Batch.bind_schedules as well (wae_buffer_source_set_device_offset).  A
        duration is declared together with an offset."""
        if duration is not None and offset is None:
            raise B.WaeError(1, "set_device_schedule: a duration window needs an offset window")
        o_lo, o_hi = (0.0, 0.0) if offset is None else (float(x) for x in offset)
        d_lo, d_hi = (0.0, 0.0) if duration is None else (float(x) for x in duration)
        # (checked before the start is declared, so that a refused call declares nothing)
        if not all(math.isfinite(lo) and math.isfinite(hi) and 0.0 <= lo <= hi for lo, hi in ((o_lo, o_hi), (d_lo, d_hi))):
            raise B.WaeError(1, "RangeError - an offset / duration window must be finite with 0 <= lo <= hi")
        super().set_device_schedule(start, stop)
        if offset is not None:
            api = self._ctx._api
            api.check(api.buffer_source_set_device_offset(self._ctx._g, self.id, o_lo, o_hi, 0 if duration is None else 1, d_lo, d_hi))
            self._ctx._device_schedules[self.id] = (stop is not None, True, duration is not None)
        return self

    def set_device_loop(self, start, end):
        """wae_buffer_source_set_device_loop (product only): the loopStart and loopEnd of this looping source are supplied by
        Batch.bind_loops from device memory before each run, clamped to the windows `start` = (lo, hi) and `end` = (lo, hi).  Pin one of
        them with a one-point window.  The node takes no further set_loop / set_loop_start / set_loop_end."""
        api = self._ctx._api
        if not api.is_product:
            raise B.WaeError(3, "loop points bound from device memory are a feature of the GPU engine")
        s_lo, s_hi = (float(x) for x in start)
        e_lo, e_hi = (float(x) for x in end)
        api.check(api.buffer_source_set_device_loop(self._ctx._g, self.id, s_lo, s_hi, e_lo, e_hi))
        self._ctx._device_loops.add(self.id)
        return self


def _response_arrays(frequency_hz):
    f = np.ascontiguousarray(frequency_hz, dtype=np.float32)
    return f, np.zeros(len(f), np.float32), np.zeros(len(f), np.float32)


class ConvolverNode(AudioNode):
    # convolver.rs:259-328
    def set_buffer(self, buffer):
        self._set_buffer("convolver_set_buffer", buffer)

    def set_device_response(self, number_of_channels, length, sample_rate):
        """wae_convolver_set_device_response (product only): the node convolves with a response of this shape that
        Batch.bind_responses supplies from device memory before each run, instead of an AudioBuffer.  Counts as the node's set_buffer
        (the normalisation is decided now)."""
        api = self._ctx._api
        if not api.is_product:
            raise B.WaeError(3, "convolver responses bound from device memory are a feature of the GPU engine")
        api.check(api.convolver_set_device_response(self._ctx._g, self.id, int(number_of_channels), int(length), float(sample_rate)))
        self._ctx._device_responses[self.id] = (int(number_of_channels), int(length))

    def set_normalize(self, value):
        self._set_attribute(B.ATTR_NORMALIZE, 1.0 if value else 0.0)


class WaveShaperNode(AudioNode):
    # waveshaper.rs:203-229
    def set_curve(self, curve):
        c = B.as_f32(curve)
        api = self._ctx._api
        api.check(api.wave_shaper_set_curve(self._ctx._g, self.id, B.fptr(c), len(c)))

    def set_device_curve(self, length):
        """wae_wave_shaper_set_device_curve (product only): the node shapes with a curve of `length` points that Batch.bind_curves
        supplies from device memory before each run.  Counts as the node's set_curve."""
        api = self._ctx._api
        if not api.is_product:
            raise B.WaeError(3, "WaveShaper curves bound from device memory are a feature of the GPU engine")
        api.check(api.wave_shaper_set_device_curve(self._ctx._g, self.id, int(length)))
        self._ctx._device_curves[self.id] = int(length)

    def set_oversample(self, oversample):
        self._set_attribute(B.ATTR_OVERSAMPLE, oversample)


class PannerNode(AudioNode):
    # panner.rs:545-657
    def set_panning_model(self, v):
        self._set_attribute(B.ATTR_PANNING_MODEL, v)

    def set_distance_model(self, v):
        self._set_attribute(B.ATTR_DISTANCE_MODEL, v)

    def set_ref_distance(self, v):
        self._set_attribute(B.ATTR_REF_DISTANCE, v)

    def set_max_distance(self, v):
        self._set_attribute(B.ATTR_MAX_DISTANCE, v)

    def set_rolloff_factor(self, v):
        self._set_attribute(B.ATTR_ROLLOFF_FACTOR, v)

    def set_cone_inner_angle(self, v):
        self._set_attribute(B.ATTR_CONE_INNER_ANGLE, v)

    def set_cone_outer_angle(self, v):
        self._set_attribute(B.ATTR_CONE_OUTER_ANGLE, v)

    def set_cone_outer_gain(self, v):
        self._set_attribute(B.ATTR_CONE_OUTER_GAIN, v)


class BiquadFilterNode(AudioNode):
    def set_type(self, type_):
        api = self._ctx._api
        api.check(api.biquad_set_type(self._ctx._g, self.id, type_))
        self.type_ = type_

    def get_frequency_response(self, frequency_hz):
        """BiquadFilterNode::get_frequency_response (src/node/biquad_filter.rs:657-735) -> (mag_response, phase_response)."""
        f, mag, phase = _response_arrays(frequency_hz)
        self._ctx._api.biquad_frequency_response(self.type_, self._ctx._sample_rate, self.frequency.value(), self.detune.value(), self.q.value(),
                                                 self.gain.value(), f.ctypes.data_as(B.c_float_p), mag.ctypes.data_as(B.c_float_p),
                                                 phase.ctypes.data_as(B.c_float_p), len(f))
        return mag, phase


class IIRFilterNode(AudioNode):
    def set_device_coefficients(self):
        """wae_iir_filter_set_device_coefficients (product only): the node filters with the feedforward / feedback coefficients that
        Batch.bind_iir_coefficients supplies from device memory before each run, as many of each as the node was constructed with.
        Plans are made with the constructed coefficients."""
        api = self._ctx._api
        if not api.is_product:
            raise B.WaeError(3, "IIR coefficients bound from device memory are a feature of the GPU engine")
        api.check(api.iir_filter_set_device_coefficients(self._ctx._g, self.id))
        self._ctx._device_iirs[self.id] = (len(self.feedforward), len(self.feedback))

    def get_frequency_response(self, frequency_hz):
        """IIRFilterNode::get_frequency_response (src/node/iir_filter.rs:215-265) -> (mag_response, phase_response)."""
        if self.id in self._ctx._device_iirs:
            raise B.WaeError(2, "get_frequency_response: the coefficients of this IIRFilterNode are bound from device memory "
                                "(set_device_coefficients)")
        f, mag, phase = _response_arrays(frequency_hz)
        ff, fb = self.feedforward, self.feedback
        self._ctx._api.iir_frequency_response(ff.ctypes.data_as(B.c_double_p), len(ff), fb.ctypes.data_as(B.c_double_p), len(fb), self._ctx._sample_rate,
                                              f.ctypes.data_as(B.c_float_p), mag.ctypes.data_as(B.c_float_p), phase.ctypes.data_as(B.c_float_p), len(f))
        return mag, phase


class DynamicsCompressorNode(AudioNode):
    def reduction(self):
        """DynamicsCompressorNode::reduction (src/node/dynamics_compressor.rs:204-206) after the render."""
        ctx, api = self._ctx, self._ctx._api
        out = C.c_float(0)
        if api.is_product:
            if ctx._batch is None:
                raise B.WaeError(2, "reduction is available after rendering")
            api.check(api.compressor_reduction(ctx._batch.handle, ctx._batch_index, self.id, C.byref(out)))
        else:
            api.check(api.compressor_reduction(ctx._g, self.id, C.byref(out)))
        return out.value

    # wae_compressor_set_readouts: reduction() taken on the GPU during the render, at `times` (seconds, non-decreasing), each quantised
    # like a suspend_sync callback's (ceil(t * sampleRate / 128) quanta)
    def set_readouts(self, times):
        times = np.ascontiguousarray(times, np.float64).reshape(-1)
        api = self._ctx._api
        if not api.is_product:
            raise B.WaeError(4, "compressor read-outs are taken by the GPU engine")
        api.check(api.compressor_set_readouts(self._ctx._g, self.id, times.ctypes.data_as(B.c_double_p), len(times)))
        self._readouts = len(times)
        self._ctx._comp_readout_nodes[self.id] = self

    def get_reduction_readouts(self):
        """[K] reduction (dB) of the declared read-outs of the last render"""
        ctx = self._ctx
        out = ctx._readout_array("compressor", (getattr(self, "_readouts", 0),), np.float32)
        ctx._api.check(ctx._api.batch_fetch_compressor_readouts(ctx._batch.handle, ctx._batch_index, self.id, B.fptr(out), out.size))
        return out


class AnalyserNode(AudioNode):
    def __init__(self, ctx, node_id, fft_size):
        super().__init__(ctx, node_id)
        self.fft_size = fft_size

    # analyser.rs:148-222
    def set_fft_size(self, fft_size):
        self._set_attribute(B.ATTR_FFT_SIZE, fft_size)
        self.fft_size = int(fft_size)

    def set_smoothing_time_constant(self, v):
        self._set_attribute(B.ATTR_SMOOTHING_TIME_CONSTANT, v)

    def set_min_decibels(self, v):
        self._set_attribute(B.ATTR_MIN_DECIBELS, v)

    def set_max_decibels(self, v):
        self._set_attribute(B.ATTR_MAX_DECIBELS, v)

    def frequency_bin_count(self):
        return self.fft_size // 2

    # `out`: a caller-owned array (like the reference's `&mut [f32]` / `&mut [u8]`): only the first min(len, fft_size or
    # frequency_bin_count) entries are written, the rest is left as it was
    def get_float_time_domain_data(self, n=None, out=None):
        return self._ctx._analyser_read(self, "time", n or self.fft_size, out=out)

    def get_float_frequency_data(self, n=None, out=None):
        return self._ctx._analyser_read(self, "freq", n or self.fft_size // 2, out=out)

    def get_byte_time_domain_data(self, n=None, out=None):
        return self._ctx._analyser_read(self, "time", n or self.fft_size, byte=True, out=out)

    def get_byte_frequency_data(self, n=None, out=None):
        return self._ctx._analyser_read(self, "freq", n or self.fft_size // 2, byte=True, out=out)

    # wae_analyser_set_readouts: read-outs taken on the GPU during the render, at `times` (seconds, non-decreasing), each quantised
    # like a suspend_sync callback's (ceil(t * sampleRate / 128) quanta); fftSize and the smoothing are the node's at render time
    def set_readouts(self, times, frequency=True, time_domain=False):
        times = np.ascontiguousarray(times, np.float64).reshape(-1)
        kinds = (B.READOUT_FREQUENCY if frequency else 0) | (B.READOUT_TIME_DOMAIN if time_domain else 0)
        api = self._ctx._api
        if not api.is_product:
            raise B.WaeError(4, "analyser read-outs are taken by the GPU engine")
        api.check(api.analyser_set_readouts(self._ctx._g, self.id, times.ctypes.data_as(B.c_double_p), len(times), kinds))
        self._readouts = len(times)
        self._ctx._readout_nodes[self.id] = self

    def get_float_frequency_readouts(self):
        """[K][fftSize / 2] dB of the declared read-outs of the last render"""
        return self._ctx._readouts(self, B.READOUT_FREQUENCY, self.fft_size // 2)

    def get_float_time_domain_readouts(self):
        """[K][fftSize] samples of the declared read-outs of the last render"""
        return self._ctx._readouts(self, B.READOUT_TIME_DOMAIN, self.fft_size)

    # wae_analyser_set_byte_readouts: the declared read-outs of these kinds (declared by set_readouts) delivered as bytes too, as
    # get_byte_frequency_data / get_byte_time_domain_data return them; minDecibels / maxDecibels are the node's at render time
    def set_byte_readouts(self, frequency=False, time_domain=False):
        kinds = (B.READOUT_FREQUENCY if frequency else 0) | (B.READOUT_TIME_DOMAIN if time_domain else 0)
        api = self._ctx._api
        if not api.is_product:
            raise B.WaeError(4, "analyser read-outs are taken by the GPU engine")
        api.check(api.analyser_set_byte_readouts(self._ctx._g, self.id, kinds))
        self._byte_readouts = kinds

    def get_byte_frequency_readouts(self):
        """[K][fftSize / 2] uint8 of the declared byte read-outs of the last render"""
        return self._ctx._readouts(self, B.READOUT_FREQUENCY, self.fft_size // 2, byte=True)

    def get_byte_time_domain_readouts(self):
        """[K][fftSize] uint8 of the declared byte read-outs of the last render"""
        return self._ctx._readouts(self, B.READOUT_TIME_DOMAIN, self.fft_size, byte=True)


class AudioListener:
    def __init__(self, ctx):
        names = ["position_x", "position_y", "position_z", "forward_x", "forward_y", "forward_z", "up_x", "up_y", "up_z"]
        defaults = [0, 0, 0, 0, 0, -1, 0, 1, 0]
        for i, (n, d) in enumerate(zip(names, defaults)):
            setattr(self, n, AudioParam(ctx, "listener", i, d))


class OfflineAudioContext:
    """OfflineAudioContext::new(number_of_channels, length, sample_rate), src/context/offline.rs:78."""

    def __init__(self, number_of_channels, length, sample_rate, backend):
        self._backend = backend
        self._api = backend.api
        self._channels, self._length = int(number_of_channels), int(length)
        self._sample_rate = float(np.float32(sample_rate))
        g = C.c_void_p()
        if self._api.is_product:
            self._api.check(self._api.graph_create(backend.engine, self._channels, self._length, self._sample_rate, C.byref(g)))
        else:
            self._api.check(self._api.graph_create(self._channels, self._length, self._sample_rate, C.byref(g)))
        self._g = g
        self._keep = []
        self._dest = AudioNode(self, 0, 1, 1)
        self._batch = None
        self._batch_index = 0
        self._listener = None
        self._suspends = []
        self._readout_nodes = {}  # node id -> AnalyserNode with declared read-outs (set_readouts)
        self._comp_readout_nodes = {}  # node id -> DynamicsCompressorNode with declared read-outs (set_readouts)
        self._current_time = 0.0
        self._device_inputs = {}  # node id -> (channels, length) declared with set_device_input
        self._source_refs = set()  # ids of the device inputs declared by_reference
        self._device_responses = {}  # node id -> (channels, length) declared with set_device_response
        self._device_curves = {}  # node id -> length declared with set_device_curve
        self._device_waves = {}  # node id -> coefficient count declared with set_device_periodic_wave
        self._device_iirs = {}  # node id -> (feedforward count, feedback count) declared with set_device_coefficients
        self._device_value_curves = {}  # (node id, param index) -> length declared with set_device_value_curve
        self._device_schedules = {}  # node id -> whether set_device_schedule declared the stop time too
        self._device_loops = set()  # ids of the nodes declared with set_device_loop

    def __del__(self):
        try:
            if self._g:
                self._api.graph_destroy(self._g)
                self._g = None
        except Exception:
            pass

    def render_order(self):
        """Ids in per-quantum processing order (Graph::order_nodes, src/render/graph.rs:331-487); host work on both libraries."""
        ids = (C.c_uint32 * 4096)()
        if self._api.is_product:
            n = C.c_uint32(0)
            self._api.check(self._api.graph_render_order(self._g, ids, 4096, C.byref(n)))
            n = n.value
        else:
            n = self._api.render_order(self._g, ids, 4096)
        return list(ids[:min(n, 4096)])

    # ---- BaseAudioContext
    def destination(self):
        return self._dest

    def sample_rate(self):
        return self._sample_rate

    def length(self):
        return self._length

    def listener(self):
        if self._listener is None:
            self._listener = AudioListener(self)
        return self._listener

    def create_buffer(self, number_of_channels, length, sample_rate):
        return AudioBuffer.zeros(number_of_channels, length, sample_rate)

    def _create(self, fn, opts):
        nid = C.c_uint32()
        self._api.check(getattr(self._api, fn)(self._g, C.byref(opts), C.byref(nid)))
        return nid.value

    def create_oscillator(self, type_=SINE, frequency=440.0, detune=0.0, periodic_wave=None):
        o = B.OscillatorOptions(type_, frequency, detune, None, 0)
        if periodic_wave is not None:
            pw = B.as_f32(periodic_wave)
            self._keep.append(pw)
            o.periodic_wave, o.periodic_wave_len, o.type = B.fptr(pw), len(pw), CUSTOM
        nid = self._create("create_oscillator", o)
        n = OscillatorNode(self, nid, 0, 1)
        nyq = self._sample_rate / 2
        n.frequency = AudioParam(self, nid, 0, frequency, -nyq, nyq)
        n.detune = AudioParam(self, nid, 1, detune, -153600.0, 153600.0)
        return n

    def create_biquad_filter(self, type_=LOWPASS, frequency=350.0, q=1.0, detune=0.0, gain=0.0, cfg=None):
        o = B.BiquadOptions(type_, q, detune, frequency, gain, cfg or channel_config())
        nid = self._create("create_biquad_filter", o)
        n = BiquadFilterNode(self, nid)
        n.type_ = type_
        n.q = AudioParam(self, nid, 0, q)
        n.detune = AudioParam(self, nid, 1, detune, -153600.0, 153600.0)
        n.frequency = AudioParam(self, nid, 2, frequency, 0.0, self._sample_rate / 2)
        n.gain = AudioParam(self, nid, 3, gain)
        return n

    def create_iir_filter(self, feedforward, feedback, cfg=None):
        ff = np.ascontiguousarray(feedforward, dtype=np.float64)
        fb = np.ascontiguousarray(feedback, dtype=np.float64)
        o = B.IirOptions(ff.ctypes.data_as(B.c_double_p), len(ff), fb.ctypes.data_as(B.c_double_p), len(fb),
                         cfg or channel_config())
        n = IIRFilterNode(self, self._create("create_iir_filter", o))
        n.feedforward, n.feedback = ff, fb
        return n

    def create_gain(self, gain=1.0, cfg=None):
        nid = self._create("create_gain", B.GainOptions(gain, cfg or channel_config()))
        n = AudioNode(self, nid)
        n.gain = AudioParam(self, nid, 0, gain)
        return n

    def create_buffer_source(self, buffer=None, detune=0.0, playback_rate=1.0, loop=False, loop_start=0.0, loop_end=0.0):
        o = B.BufferSourceOptions(None, detune, playback_rate, 1 if loop else 0, loop_start, loop_end)
        if buffer is not None:
            d, keep = buffer._desc()
            self._keep.append((d, keep))
            o.buffer = C.pointer(d)
        nid = self._create("create_buffer_source", o)
        n = AudioBufferSourceNode(self, nid, 0, 1)
        n.detune = AudioParam(self, nid, 0, detune)
        n.playback_rate = AudioParam(self, nid, 1, playback_rate)
        return n

    def create_constant_source(self, offset=1.0):
        nid = self._create("create_constant_source", B.ConstantSourceOptions(offset))
        n = AudioScheduledSourceNode(self, nid, 0, 1)
        n.offset = AudioParam(self, nid, 0, offset)
        return n

    def create_convolver(self, buffer=None, disable_normalization=False, cfg=None):
        o = B.ConvolverOptions(None, 1 if disable_normalization else 0, cfg or channel_config())
        if buffer is not None:
            d, keep = buffer._desc()
            self._keep.append((d, keep))
            o.buffer = C.pointer(d)
        return ConvolverNode(self, self._create("create_convolver", o))

    def create_wave_shaper(self, curve=None, oversample=OVERSAMPLE_NONE, cfg=None):
        o = B.WaveShaperOptions(None, 0, oversample, cfg or channel_config())
        if curve is not None:
            c = B.as_f32(curve)
            self._keep.append(c)
            o.curve, o.curve_len = B.fptr(c), len(c)
        return WaveShaperNode(self, self._create("create_wave_shaper", o))

    def create_delay(self, max_delay_time=1.0, delay_time=0.0, cfg=None):
        nid = self._create("create_delay", B.DelayOptions(max_delay_time, delay_time, cfg or channel_config()))
        n = AudioNode(self, nid)
        n.delay_time = AudioParam(self, nid, 0, delay_time, 0.0, max_delay_time)
        return n

    def create_stereo_panner(self, pan=0.0, cfg=None):
        nid = self._create("create_stereo_panner", B.StereoPannerOptions(pan, cfg or channel_config()))
        n = AudioNode(self, nid)
        n.pan = AudioParam(self, nid, 0, pan, -1.0, 1.0)
        return n

    def create_panner(self, panning_model=EQUALPOWER, distance_model=INVERSE, position=(0.0, 0.0, 0.0),
                      orientation=(1.0, 0.0, 0.0), ref_distance=1.0, max_distance=10000.0, rolloff_factor=1.0,
                      cone_inner_angle=360.0, cone_outer_angle=360.0, cone_outer_gain=0.0, cfg=None):
        o = B.PannerOptions(panning_model, distance_model, *position, *orientation, ref_distance, max_distance,
                            rolloff_factor, cone_inner_angle, cone_outer_angle, cone_outer_gain, cfg or channel_config())
        nid = self._create("create_panner", o)
        n = PannerNode(self, nid)
        for i, name in enumerate(["position_x", "position_y", "position_z", "orientation_x", "orientation_y", "orientation_z"]):
            setattr(n, name, AudioParam(self, nid, i, (list(position) + list(orientation))[i]))
        return n

    def create_analyser(self, fft_size=2048, smoothing_time_constant=0.8, min_decibels=-100.0, max_decibels=-30.0, cfg=None):
        o = B.AnalyserOptions(fft_size, smoothing_time_constant, min_decibels, max_decibels, cfg or channel_config())
        return AnalyserNode(self, self._create("create_analyser", o), fft_size)

    def create_dynamics_compressor(self, attack=0.003, knee=30.0, ratio=12.0, release=0.25, threshold=-24.0, cfg=None):
        o = B.DynamicsCompressorOptions(attack, knee, ratio, release, threshold, cfg or channel_config())
        nid = self._create("create_dynamics_compressor", o)
        n = DynamicsCompressorNode(self, nid)
        for i, (name, v) in enumerate([("attack", attack), ("knee", knee), ("ratio", ratio), ("release", release), ("threshold", threshold)]):
            setattr(n, name, AudioParam(self, nid, i, v))
        return n

    def create_channel_merger(self, number_of_inputs=6):
        return AudioNode(self, self._create("create_channel_merger", B.ChannelMergerOptions(number_of_inputs)), number_of_inputs, 1)

    def create_channel_splitter(self, number_of_outputs=6):
        return AudioNode(self, self._create("create_channel_splitter", B.ChannelSplitterOptions(number_of_outputs)), 1, number_of_outputs)

    def current_time(self):
        """BaseAudioContext::current_time: 0 before rendering, the suspend time inside a suspend_sync callback."""
        return self._current_time

    def suspend_sync(self, suspend_time, callback):
        """OfflineAudioContext::suspend_sync (src/context/offline.rs:330-387): `callback(context)` runs when the render reaches
        suspend_time (quantised up to a render quantum) and may mutate the graph."""
        self._suspends.append((float(suspend_time), callback))

    def _run_suspend_callbacks(self):
        """The control half of the render loop (src/render/thread.rs:271-290): take the suspend points in time order."""
        todo, self._suspends = sorted(self._suspends, key=lambda sc: sc[0]), []
        for t, cb in todo:
            self._api.check(self._api.graph_suspend(self._g, t))
            self._current_time = math.ceil(t * self._sample_rate / 128.0) * 128.0 / self._sample_rate
            cb(self)
        self._current_time = 0.0

    # ---- rendering
    def start_rendering_sync(self):
        """OfflineAudioContext::start_rendering_sync (src/context/offline.rs:157-185): a batch of one."""
        return render_batch([self])[0]

    def _readout_array(self, what, shape, dtype):
        if self._batch is None:
            raise B.WaeError(2, f"{what} read-outs are available after rendering")
        return np.empty(shape, dtype)

    def _readouts(self, node, kind, row, byte=False):
        out = self._readout_array("analyser", (getattr(node, "_readouts", 0), row), np.uint8 if byte else np.float32)
        api, h = self._api, self._batch.handle
        if byte:
            api.check(api.batch_fetch_analyser_byte_readouts(h, self._batch_index, node.id, kind, out.ctypes.data_as(C.c_void_p), out.size))
        else:
            api.check(api.batch_fetch_analyser_readouts(h, self._batch_index, node.id, kind, B.fptr(out), out.size))
        return out

    def _analyser_read(self, node, kind, n, byte=False, out=None):
        if out is None:
            out = np.zeros(n, np.uint8 if byte else np.float32)
        else:
            assert out.dtype == (np.uint8 if byte else np.float32) and out.flags.c_contiguous
            n = len(out)
        ptr = out.ctypes.data_as(C.POINTER(C.c_uint8)) if byte else B.fptr(out)
        api = self._api
        name = "analyser_get_%s_%s_data" % ("byte" if byte else "float", "time_domain" if kind == "time" else "frequency")
        fn = getattr(api, name)
        if api.is_product:
            if self._batch is None:
                raise B.WaeError(2, "analyser data is available after rendering")
            api.check(fn(self._batch.handle, self._batch_index, node.id, ptr, n))
        else:
            api.check(fn(self._g, node.id, ptr, n))
        return out


def _readout_kind(kind):
    kinds = {"frequency": B.READOUT_FREQUENCY, "time_domain": B.READOUT_TIME_DOMAIN}
    if kind not in kinds:
        raise B.WaeError(1, f"kind must be one of {sorted(kinds)}")
    return kinds[kind]


class Batch:
    """wae_batch_prepare / run / fetch: a compiled batch of contexts (product only).  many=True: wae_batch_prepare_many, contexts of
    any mix of channel counts, lengths and sample rates (read each one's PCM with fetch_graph)."""

    def __init__(self, contexts, many=False):
        ctx0 = contexts[0]
        self.api = ctx0._api
        self.contexts = contexts
        self.n = len(contexts)
        self.channels, self.length = ctx0._channels, ctx0._length
        for c in contexts:
            c._run_suspend_callbacks()
        arr = (C.c_void_p * self.n)(*[c._g for c in contexts])
        h = C.c_void_p()
        prepare = self.api.batch_prepare_many if many else self.api.batch_prepare
        self.api.check(prepare(ctx0._backend.engine, arr, self.n, C.byref(h)))
        self.handle = h
        self._guard = None  # bind_sources: torch stream the bound tensors are recorded on
        self._views_out = False  # output_tensor was called: runs into the batch's own buffer are ordered after torch's current stream
        self._out = None  # bind_output: the tensor runs write
        self._out_viewed = False  # output_tensor handed out views of the bound tensor since it was bound: runs into it wait for torch
        self._readouts_viewed = False  # analyser_readouts / compressor_readouts handed out views of read-out rows: every run (bound output or not) waits for torch
        self._src_refs = {}  # bind_sources: (graph, node id) -> the tensor a device input declared by_reference reads
        self._ref_tensors = []  # the distinct tensors of _src_refs
        self._has_refs = any(c._source_refs for c in contexts)
        self._backend = ctx0._backend
        self._backend.batches.add(self)
        for i, c in enumerate(contexts):
            c._batch, c._batch_index = self, i

    def run(self):
        self._after_torch_readers()
        self._after_torch_writers()
        self.api.check(self.api.batch_run(self.handle))
        self._out_written()
        self._refs_read()

    def upload(self):
        self.api.check(self.api.batch_upload(self.handle))

    def set_timing(self, per_stage):
        self.api.check(self.api.batch_set_timing(self.handle, 1 if per_stage else 0))

    def sync(self):
        self.api.check(self.api.batch_sync(self.handle))

    def groups(self):
        """[(first_graph, last_graph)] of the batch's graph groups (rendered one after the other)."""
        n = C.c_uint32()
        self.api.check(self.api.batch_group_count(self.handle, C.byref(n)))
        out = []
        for k in range(n.value):
            a, b = C.c_uint32(), C.c_uint32()
            self.api.check(self.api.batch_group_range(self.handle, k, C.byref(a), C.byref(b)))
            out.append((a.value, b.value))
        return out

    def run_group(self, k):
        """render of ONE graph group, asynchronous on the engine stream (call the groups in order)"""
        self._after_torch_readers()
        self._after_torch_writers()
        self.api.check(self.api.batch_run_group(self.handle, k))
        self._out_written()
        self._refs_read()

    def run_pipelined(self, host_out_ptr):
        """H2D + render + D2H, overlapped per graph group; `host_out_ptr` = address of [n][ch][length] f32 (pinned)."""
        self._after_torch_readers()
        self._after_torch_writers()
        self.api.check(self.api.batch_run_pipelined(self.handle, host_out_ptr))
        self._refs_read()

    def fetch(self, out=None):
        if out is None:
            out = np.empty((self.n, self.channels, self.length), np.float32)
        self.api.check(self.api.batch_fetch(self.handle, out.ctypes.data_as(C.c_void_p)))
        return out

    def graph_output(self, i):
        """(offset in floats, channels, length) of context i in the packed device output (device_ptr)."""
        off, ch, length = C.c_uint64(), C.c_uint32(), C.c_uint64()
        self.api.check(self.api.batch_graph_output(self.handle, i, C.byref(off), C.byref(ch), C.byref(length)))
        return off.value, ch.value, length.value

    def fetch_graph(self, i, out=None):
        """context i's rendered PCM, [channels][length] float32."""
        _, ch, length = self.graph_output(i)
        if out is None:
            out = np.empty((ch, length), np.float32)
        assert out.dtype == np.float32 and out.flags.c_contiguous and out.size >= ch * length
        self.api.check(self.api.batch_fetch_graph(self.handle, i, B.fptr(out)))
        return out

    def device_ptr(self):
        p, n = C.c_void_p(), C.c_uint64()
        self.api.check(self.api.batch_output_device_ptr(self.handle, C.byref(p), C.byref(n)))
        return p.value, n.value

    def _engine_stream(self):
        import torch
        p = C.c_void_p()
        self.api.check(self.api.engine_stream(self._backend.engine, C.byref(p)))
        return torch.cuda.ExternalStream(p.value or 0, device=self._device())

    def _device(self):
        import torch
        return torch.device("cuda", self._backend.device)

    def _torch_stream_handle(self):
        """cudaStream_t of torch's current stream.  torch reports its default stream, the legacy NULL stream, as 0, which the library
        reads as 'no ordering' (and the non-blocking engine stream does not wait for the legacy stream by itself): cudaStreamLegacy."""
        import torch
        return torch.cuda.current_stream(self._device()).cuda_stream or 1  # 1 = cudaStreamLegacy

    def _after_torch_readers(self):
        """A run overwrites the device output: once output_tensor views of the buffer it writes were handed out, order it after the work
        torch has queued so far on its current stream (the readers of the last output).  Views of another buffer do not hold a run into a
        bound output up: bind_output ordered it after the work queued before the bind, and the readers of the other buffer may run while it
        renders.  Views of the analyser read-out rows hold every run up: the rows are the batch's own memory whether or not an output is
        bound, and every run rewrites them."""
        if (self._views_out and self._out is None) or (self._out_viewed and self._out is not None) or self._readouts_viewed:
            import torch
            self._engine_stream().wait_stream(torch.cuda.current_stream(self._device()))

    def bind_sources(self, nodes, pcm, graphs=None):
        """wae_batch_bind_sources: pcm[k] ([channels][length] of a float32 CUDA tensor [n][channels][length], unit stride on the last
        dimension) becomes the audio of device input nodes[k] of context graphs[k] (default: 0..n-1).  `nodes`: one node (or id) for all
        graphs (graphs built the same way share ids) or one per graph.  One call, ordered after torch's current stream (its default
        stream included); the copy runs on the engine stream, and the tensor's memory is kept from reuse until it has (record_stream).
        Inputs declared by_reference are not copied: the batch keeps `pcm` until they are bound again or the batch is destroyed, and each
        run reads it (see AudioBufferSourceNode.set_device_input).  A tensor of one shape [1][channels][length] expanded to n rows
        (stride 0 on the first dimension) names the same memory for every graph."""
        items, n = self._pcm_items("bind_sources", "pcm", nodes, pcm, graphs, "_device_inputs", B.SourceBinding)
        self._bind(self.api.batch_bind_sources, items, n, pcm)
        if self._has_refs:
            gs, ids = self._graphs_and_nodes("bind_sources", nodes, graphs, n)
            keys = [(g, int(nid)) for g, nid in zip(gs, ids) if int(nid) in self.contexts[g]._source_refs]
            if keys:
                self._src_refs.update(dict.fromkeys(keys, pcm))
                self._ref_tensors = list({id(t): t for t in self._src_refs.values()}.values())

    def _after_torch_writers(self):
        """While a device input declared by_reference is bound, a run reads caller memory: order it after the work torch has queued so
        far on its current stream (in-place writes to the bound tensors made after the bind included)."""
        if self._src_refs:
            import torch
            self._engine_stream().wait_stream(torch.cuda.current_stream(self._device()))

    def _refs_read(self):
        """Keeps the tensors read by reference from reuse until the runs queued so far have read them (as bind_output's tensor)."""
        for t in self._ref_tensors:
            self._keep_until_read(t)

    def bind_responses(self, nodes, ir, graphs=None):
        """wae_batch_bind_responses: ir[k] ([channels][length] of a float32 CUDA tensor [n][channels][length], unit stride on the last
        dimension) becomes the impulse response of ConvolverNode nodes[k] (declared with set_device_response) of context graphs[k]
        (default: 0..n-1).  `nodes` as for bind_sources.  One call, ordered after torch's current stream; the response is normalised,
        trimmed and transformed on the engine stream, and the tensor's memory is kept from reuse until it has been read."""
        items, n = self._pcm_items("bind_responses", "ir", nodes, ir, graphs, "_device_responses", B.ResponseBinding)
        self._bind(self.api.batch_bind_responses, items, n, ir)

    def bind_curves(self, nodes, curves, graphs=None):
        """wae_batch_bind_curves: curves[k] (a row of a float32 CUDA tensor [n][length], unit stride on the last dimension) becomes the
        curve of WaveShaperNode nodes[k] (declared with set_device_curve) of context graphs[k] (default: 0..n-1).  `nodes` as for
        bind_sources.  One call, ordered after torch's current stream; the curves are copied on the engine stream, and the tensor's memory
        is kept from reuse until they have been."""
        import torch
        if not (isinstance(curves, torch.Tensor) and curves.is_cuda and curves.dtype == torch.float32 and curves.dim() == 2):
            raise B.WaeError(1, "bind_curves: curves must be a float32 CUDA tensor [n][length]")
        n = curves.shape[0]
        graphs, ids = self._graphs_and_nodes("bind_curves", nodes, graphs, n)
        if n and curves.stride(1) != 1:
            raise B.WaeError(1, "bind_curves: the points of a curve must be contiguous (unit stride on the last dimension)")
        items = (B.CurveBinding * max(n, 1))()
        base = curves.data_ptr()
        for k, (g, nid) in enumerate(zip(graphs, ids)):
            declared = self.contexts[g]._device_curves.get(int(nid))
            # (the tensor's own shape: the library checks only the CUDA allocation, which may hold several tensors)
            if declared is not None and curves.shape[1] != declared:
                raise B.WaeError(1, f"bind_curves: curves[{k}] has {curves.shape[1]} points, node {nid} of graph {g} was declared with "
                                    f"{declared}")
            items[k] = B.CurveBinding(g, int(nid), C.cast(C.c_void_p(base + 4 * k * curves.stride(0)), B.c_float_p))
        self._bind(self.api.batch_bind_curves, items, n, curves)

    def bind_periodic_waves(self, nodes, real, imag=None, graphs=None):
        """wae_batch_bind_periodic_waves: real[k] and imag[k] (rows of float32 CUDA tensors [n][coefficients], unit stride on the last
        dimension; either may be None = zeros) become the PeriodicWave coefficients of OscillatorNode nodes[k] (declared with
        set_device_periodic_wave) of context graphs[k] (default: 0..n-1).  `nodes` as for bind_sources.  One call, ordered after torch's
        current stream; the wavetables are synthesised on the engine stream, and the tensors' memory is kept from reuse until they have
        been."""
        import torch
        given = [t for t in (real, imag) if t is not None]
        if not given:
            raise B.WaeError(1, "bind_periodic_waves: real and imag are both None")
        for t in given:
            if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float32 and t.dim() == 2):
                raise B.WaeError(1, "bind_periodic_waves: real and imag must be float32 CUDA tensors [n][coefficients]")
        if len(given) == 2 and real.shape != imag.shape:
            raise B.WaeError(1, f"bind_periodic_waves: real {tuple(real.shape)} and imag {tuple(imag.shape)} differ in shape")
        n, count = given[0].shape
        graphs, ids = self._graphs_and_nodes("bind_periodic_waves", nodes, graphs, n)
        if n and any(t.stride(1) != 1 for t in given):
            raise B.WaeError(1, "bind_periodic_waves: the coefficients of a wave must be contiguous (unit stride on the last dimension)")

        def row(t, k):
            return None if t is None else C.cast(C.c_void_p(t.data_ptr() + 4 * k * t.stride(0)), B.c_float_p)
        items = (B.PeriodicWaveBinding * max(n, 1))()
        for k, (g, nid) in enumerate(zip(graphs, ids)):
            declared = self.contexts[g]._device_waves.get(int(nid))
            # (the tensor's own shape: the library checks only the CUDA allocation, which may hold several tensors)
            if declared is not None and count != declared:
                raise B.WaeError(1, f"bind_periodic_waves: row {k} has {count} coefficients, node {nid} of graph {g} was declared "
                                    f"with {declared}")
            items[k] = B.PeriodicWaveBinding(g, int(nid), row(real, k), row(imag, k))
        self._bind(self.api.batch_bind_periodic_waves, items, n, *given)

    def bind_iir_coefficients(self, nodes, feedforward, feedback, graphs=None):
        """wae_batch_bind_iir_coefficients: feedforward[k] and feedback[k] (rows of float64 CUDA tensors [n][nff] and [n][nfb], unit
        stride on the last dimension) become the coefficients of IIRFilterNode nodes[k] (declared with set_device_coefficients) of context
        graphs[k] (default: 0..n-1).  `nodes` as for bind_sources.  One call, ordered after torch's current stream; the coefficients are
        read on the engine stream, and the tensors' memory is kept from reuse until they have been."""
        import torch
        for t in (feedforward, feedback):
            if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float64 and t.dim() == 2):
                raise B.WaeError(1, "bind_iir_coefficients: feedforward and feedback must be float64 CUDA tensors [n][count]")
        n = feedforward.shape[0]
        if feedback.shape[0] != n:
            raise B.WaeError(1, f"bind_iir_coefficients: {n} feedforward rows and {feedback.shape[0]} feedback rows")
        graphs, ids = self._graphs_and_nodes("bind_iir_coefficients", nodes, graphs, n)
        if n and (feedforward.stride(1) != 1 or feedback.stride(1) != 1):
            raise B.WaeError(1, "bind_iir_coefficients: the coefficients of a filter must be contiguous (unit stride on the last dimension)")

        def row(t, k):
            return C.cast(C.c_void_p(t.data_ptr() + 8 * k * t.stride(0)), B.c_double_p)
        items = (B.IirBinding * max(n, 1))()
        for k, (g, nid) in enumerate(zip(graphs, ids)):
            declared = self.contexts[g]._device_iirs.get(int(nid))
            # (the tensors' own shapes: the library checks only the CUDA allocations, which may hold several tensors)
            if declared is not None and (feedforward.shape[1], feedback.shape[1]) != declared:
                raise B.WaeError(1, f"bind_iir_coefficients: row {k} has {feedforward.shape[1]} feedforward and {feedback.shape[1]} "
                                    f"feedback coefficients, node {nid} of graph {g} was declared with {declared[0]} and {declared[1]}")
            items[k] = B.IirBinding(g, int(nid), row(feedforward, k), row(feedback, k))
        self._bind(self.api.batch_bind_iir_coefficients, items, n, feedforward, feedback)

    def bind_value_curves(self, params, values, graphs=None):
        """wae_batch_bind_value_curves: values[j][i] (a float32 CUDA tensor [n][length] per param, unit stride on the last dimension)
        becomes the curve of params[j] (declared with set_device_value_curve) in context graphs[i] (default: 0..n-1).  `params`: one
        AudioParam or a list (AudioListener params are not bound as curves); a param of a context built like the others shares its node
        id and index, so the params of context 0 name those of every context.  `values`: one tensor, or a list of tensors, one per param.  One call, ordered after torch's current
        stream; the values are copied on the engine stream, and the tensors' memory is kept from reuse until they have been."""
        import torch
        params = list(params) if isinstance(params, (list, tuple)) else [params]
        tensors = list(values) if isinstance(values, (list, tuple)) else [values]
        if len(tensors) != len(params):
            raise B.WaeError(1, f"bind_value_curves: {len(tensors)} tensors for {len(params)} params")
        for t in tensors:
            if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float32 and t.dim() == 2):
                raise B.WaeError(1, "bind_value_curves: values must be float32 CUDA tensors [n][length]")
        n = tensors[0].shape[0] if tensors else 0
        if any(t.shape[0] != n for t in tensors):
            raise B.WaeError(1, "bind_value_curves: the tensors differ in their number of rows")
        graphs = self._graphs("bind_value_curves", graphs, n, "rows")
        if n and any(t.stride(1) != 1 for t in tensors):
            raise B.WaeError(1, "bind_value_curves: the values of a curve must be contiguous (unit stride on the last dimension)")
        items = (B.ValueCurveBinding * max(n * len(params), 1))()
        for j, (prm, t) in enumerate(zip(params, tensors)):
            if prm._node == "listener":
                raise B.WaeError(2, "bind_value_curves: AudioListener params are not bound from device memory")
            key = (int(prm._node), int(prm._index))
            for i, g in enumerate(graphs):
                declared = self.contexts[g]._device_value_curves.get(key)
                # (the tensor's own shape: the library checks only the CUDA allocation, which may hold several tensors)
                if declared is not None and t.shape[1] != declared:
                    raise B.WaeError(1, f"bind_value_curves: values[{j}] has {t.shape[1]} points, param {key[1]} of node {key[0]} of "
                                        f"graph {g} was declared with {declared}")
                ptr = C.cast(C.c_void_p(t.data_ptr() + 4 * i * t.stride(0)), B.c_float_p)
                items[j * n + i] = B.ValueCurveBinding(g, key[0], key[1], ptr)
        self._bind(self.api.batch_bind_value_curves, items, n * len(params), *tensors)

    def bind_schedules(self, nodes, starts, stops=None, offsets=None, durations=None, graphs=None):
        """wae_batch_bind_schedules: starts[i] (and stops[i]) become the start (and stop) times of the scheduled source `nodes` (declared
        with set_device_schedule) in context graphs[i] (default: 0..n-1), and offsets[i] (and durations[i]) the offset (and duration) of
        an AudioBufferSourceNode declared with them.  Each is a float64 CUDA tensor [n] for one node, or [n][k] for a list of k nodes;
        `stops`, `offsets` and `durations` are given exactly when the nodes were declared with those windows.  One call, ordered after
        torch's current stream; the values are read on the engine stream, and their memory is kept from reuse until they have been."""
        import torch
        cols = {"stops": stops, "offsets": offsets, "durations": durations}
        for t in [starts] + [t for t in cols.values() if t is not None]:
            if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float64 and t.dim() in (1, 2)):
                raise B.WaeError(1, "bind_schedules: starts / stops / offsets / durations must be float64 CUDA tensors [n] or [n][k]")
        many = isinstance(nodes, (list, tuple))
        ids = [int(getattr(x, "id", x)) for x in nodes] if many else [int(getattr(nodes, "id", nodes))]
        n, k = starts.shape[0], len(ids)
        if (starts.dim() == 2) != many or (many and starts.shape[1] != k):
            raise B.WaeError(1, f"bind_schedules: starts is {list(starts.shape)} for {k} node(s): [n] for one node, [n][k] for a list")
        for name, t in cols.items():
            if t is not None and t.shape != starts.shape:
                raise B.WaeError(1, f"bind_schedules: {name} is {list(t.shape)}, starts {list(starts.shape)}")
        graphs = self._graphs("bind_schedules", graphs, n, "rows")
        given = tuple(t is not None for t in cols.values())
        for g in graphs:
            for nid in ids:
                declared = self.contexts[g]._device_schedules.get(nid)
                if declared is None:
                    continue
                for name, what, d, h in zip(cols, ("a stop", "an offset", "a duration"), declared, given):
                    if d != h:
                        raise B.WaeError(1, f"bind_schedules: node {nid} of graph {g} was declared {'with' if d else 'without'} {what} "
                                            f"window, {name} is {'missing' if d else 'given'}")
        # one item reads its row start, [stop], [offset], [duration] from adjacent memory: the values are packed on torch's current stream
        rest = [t.reshape(n, k) for t in cols.values() if t is not None]
        times = (torch.stack([starts.reshape(n, k)] + rest, dim=2) if rest else starts.reshape(n, k, 1)).contiguous()
        width = times.shape[2]
        items = (B.ScheduleBinding * max(n * k, 1))()
        base = times.data_ptr()
        for i, g in enumerate(graphs):
            for j, nid in enumerate(ids):
                items[i * k + j] = B.ScheduleBinding(g, nid, C.cast(C.c_void_p(base + 8 * width * (i * k + j)), B.c_double_p))
        self._bind(self.api.batch_bind_schedules, items, n * k, times)

    def bind_loops(self, nodes, starts, ends, graphs=None):
        """wae_batch_bind_loops: starts[i] and ends[i] become the loopStart and loopEnd of the AudioBufferSourceNode `nodes` (declared
        with set_device_loop) in context graphs[i] (default: 0..n-1).  Each is a float64 CUDA tensor [n] for one node, or [n][k] for a
        list of k nodes.  One call, ordered after torch's current stream; the values are read on the engine stream, and their memory is
        kept from reuse until they have been."""
        import torch
        for t in (starts, ends):
            if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == torch.float64 and t.dim() in (1, 2)):
                raise B.WaeError(1, "bind_loops: starts / ends must be float64 CUDA tensors [n] or [n][k]")
        many = isinstance(nodes, (list, tuple))
        ids = [int(getattr(x, "id", x)) for x in nodes] if many else [int(getattr(nodes, "id", nodes))]
        n, k = starts.shape[0], len(ids)
        if (starts.dim() == 2) != many or (many and starts.shape[1] != k):
            raise B.WaeError(1, f"bind_loops: starts is {list(starts.shape)} for {k} node(s): [n] for one node, [n][k] for a list")
        if ends.shape != starts.shape:
            raise B.WaeError(1, f"bind_loops: ends is {list(ends.shape)}, starts {list(starts.shape)}")
        graphs = self._graphs("bind_loops", graphs, n, "rows")
        # one item reads its row loop_start, loop_end from adjacent memory: the values are packed on torch's current stream
        points = torch.stack([starts.reshape(n, k), ends.reshape(n, k)], dim=2).contiguous()
        items = (B.LoopBinding * max(n * k, 1))()
        base = points.data_ptr()
        for i, g in enumerate(graphs):
            for j, nid in enumerate(ids):
                items[i * k + j] = B.LoopBinding(g, nid, C.cast(C.c_void_p(base + 16 * (i * k + j)), B.c_double_p))
        self._bind(self.api.batch_bind_loops, items, n * k, points)

    def _graphs(self, fn, graphs, n, rows, ids=None):
        """The graph indices of n rows of binding items: `graphs` (default 0..n-1), each in range; `ids`: the node ids of the rows, whose
        count is checked with the graphs'."""
        graphs = list(range(n)) if graphs is None else [int(g) for g in graphs]
        if len(graphs) != n or (ids is not None and len(ids) != n):
            raise B.WaeError(1, f"{fn}: {n} {rows} for {len(graphs)} graphs" + ("" if ids is None else f" and {len(ids)} nodes"))
        for g in graphs:
            if not 0 <= g < self.n:
                raise B.WaeError(2, f"{fn}: graph index {g} is out of range")
        return graphs

    def _graphs_and_nodes(self, fn, nodes, graphs, n):
        """The graph index and node id of each of n binding items: `graphs` (default 0..n-1), `nodes` one node (or id) for all graphs or
        one per graph."""
        if isinstance(nodes, (list, tuple)):
            ids = [getattr(x, "id", x) for x in nodes]
        else:
            ids = [getattr(nodes, "id", nodes)] * n
        return self._graphs(fn, graphs, n, "tensors", ids), ids

    def _pcm_items(self, fn, arg, nodes, pcm, graphs, declarations, Struct):
        """The binding items (graph index, node, device pointer, channel stride) of bind_sources / bind_responses: `declarations` names
        the contexts' {node id: (channels, length)} the tensor's shape is checked against."""
        import torch
        if not (isinstance(pcm, torch.Tensor) and pcm.is_cuda and pcm.dtype == torch.float32 and pcm.dim() == 3):
            raise B.WaeError(1, f"{fn}: {arg} must be a float32 CUDA tensor [n][channels][length]")
        n = pcm.shape[0]
        graphs, ids = self._graphs_and_nodes(fn, nodes, graphs, n)
        if n and pcm.stride(2) != 1:
            raise B.WaeError(1, f"{fn}: the frames of a channel must be contiguous (unit stride on the last dimension)")
        items = (Struct * max(n, 1))()
        base = pcm.data_ptr()
        # (torch may give the channel dimension of a one-channel tensor any stride: only channel 0 is read then)
        channel_stride = pcm.stride(1) if pcm.shape[1] > 1 else pcm.shape[2]
        for k, (g, nid) in enumerate(zip(graphs, ids)):
            declared = getattr(self.contexts[g], declarations).get(int(nid))
            # the library checks the CUDA allocation; torch's caching allocator may hold several tensors in one, so the tensor's own
            # shape is checked here
            if declared is not None and (pcm.shape[1], pcm.shape[2]) != declared:
                raise B.WaeError(1, f"{fn}: {arg}[{k}] is [{pcm.shape[1]}][{pcm.shape[2]}], node {nid} of graph {g} was declared "
                                    f"[{declared[0]}][{declared[1]}]")
            items[k] = Struct(g, int(nid), C.cast(C.c_void_p(base + 4 * k * pcm.stride(0)), B.c_float_p), channel_stride)
        return items, n

    def _bind(self, fn, items, n, *tensors):
        """One call of the bind entry point `fn`, ordered after torch's current stream; the bound tensors are kept from reuse until the
        engine stream has read them."""
        self.api.check(fn(self.handle, items, n, C.c_void_p(self._torch_stream_handle())))
        for t in tensors:
            self._keep_until_read(t)

    def _keep_until_read(self, t):
        """Keeps torch's caching allocator from reusing a bound tensor's memory before the engine stream has read it.  The tensor is
        recorded on a torch-owned stream that waits for the engine stream, not on the engine stream itself: the allocator records an event
        on that stream whenever the tensor is freed, which may be after the engine (and its stream) are gone."""
        import torch
        if self._guard is None:
            self._guard = torch.cuda.Stream(device=self._device())
        self._guard.wait_stream(self._engine_stream())
        t.record_stream(self._guard)

    def bind_params(self, params, values, graphs=None):
        """wae_batch_bind_params: values[i][j] (a float32 CUDA tensor [n][k], or [n] for one param) becomes the value of params[j] in
        context graphs[i] (default: 0..n-1).  `params`: AudioParams declared with set_device_value, one per column (an oscillator's
        frequency / detune included: the bind re-derives its phase fields; a PannerNode's position / orientation and the AudioListener's
        position / forward / up included: the bind re-derives the panner's direction, gains and HRTF response); a param of a context built
        like the others shares its node id and index, so the params of context 0 name those of every context.  One call, ordered after torch's current stream; the values
        are read on the engine stream, and the tensor is kept from reuse until they have been."""
        import torch
        if not (isinstance(values, torch.Tensor) and values.is_cuda and values.dtype == torch.float32 and values.dim() in (1, 2)):
            raise B.WaeError(1, "bind_params: values must be a float32 CUDA tensor [n] or [n][k]")
        params = list(params) if isinstance(params, (list, tuple)) else [params]
        v2 = values if values.dim() == 2 else values.unsqueeze(1)
        n, k = v2.shape
        if k != len(params):
            raise B.WaeError(1, f"bind_params: {k} value columns for {len(params)} params")
        graphs = self._graphs("bind_params", graphs, n, "value rows")
        items = (B.ParamBinding * max(n * k, 1))()
        base = v2.data_ptr()
        s0, s1 = v2.stride()
        for i, g in enumerate(graphs):
            for j, prm in enumerate(params):
                ptr = C.cast(C.c_void_p(base + 4 * (i * s0 + j * s1)), B.c_float_p)
                node = 1 if prm._node == "listener" else int(prm._node)
                items[i * k + j] = B.ParamBinding(g, node, int(prm._index), ptr)
        self._bind(self.api.batch_bind_params, items, n * k, values)

    def bind_output(self, out):
        """wae_batch_bind_output: later runs write the rendered PCM into `out`, a contiguous float32 CUDA tensor on the engine's device,
        [n][channels][length] for a batch of one shape, else 1-D of the batch's output floats in the layout output_tensor(i) addresses.  The
        call is ordered after torch's current stream; the tensor is kept while it is bound, and from reuse until the runs into it are done.
        None: back to the batch's own buffer."""
        import torch
        if out is None:
            self.api.check(self.api.batch_bind_output(self.handle, None, 0, C.c_void_p(self._torch_stream_handle())))
            self._out, self._out_viewed = None, False
            return
        p, floats = C.c_void_p(), C.c_uint64()
        self.api.check(self.api.batch_output_device_ptr(self.handle, C.byref(p), C.byref(floats)))
        shape = (self.n, self.channels, self.length) if self._one_shape() else (floats.value,)
        if not (isinstance(out, torch.Tensor) and out.is_cuda and out.dtype == torch.float32):
            raise B.WaeError(1, "bind_output: out must be a float32 CUDA tensor")
        if out.device != self._device():
            raise B.WaeError(1, f"bind_output: out is on {out.device}, the batch renders on {self._device()}")
        if tuple(out.shape) != shape or not out.is_contiguous():
            raise B.WaeError(1, f"bind_output: out must be a contiguous tensor of shape {list(shape)}, not {list(out.shape)}")
        self.api.check(self.api.batch_bind_output(self.handle, C.c_void_p(out.data_ptr()), floats.value,
                                                  C.c_void_p(self._torch_stream_handle())))
        self._out, self._out_viewed = out, False

    def _out_written(self):
        if self._out is not None:
            self._keep_until_read(self._out)

    def _one_shape(self):
        return len({(c._channels, c._length) for c in self.contexts}) == 1

    def output_tensor(self, i=None):
        """Zero-copy torch view of the rendered output on the device: [n][channels][length] for a batch of one shape, [channels_i][length_i]
        of context i; while an output is bound (bind_output), views of that tensor.  The view keeps the batch alive; torch's current stream
        is made to wait for the engine stream first (read a bound tensor through this call: it orders the read after the run), and later
        runs of the batch into the same memory (which overwrite the view) wait for the work then queued on torch's current stream."""
        import torch
        if self._out is not None:
            self._out_viewed = True
            torch.cuda.current_stream(self._device()).wait_stream(self._engine_stream())
            if i is None:
                if not self._one_shape():
                    raise B.WaeError(2, "output_tensor: the contexts of this batch differ in shape; view one with output_tensor(i)")
                return self._out
            off, ch, length = self.graph_output(i)
            return self._out.view(-1)[off:off + ch * length].view(ch, length)
        base, _ = self.device_ptr()
        if i is None:
            if not self._one_shape():
                raise B.WaeError(2, "output_tensor: the contexts of this batch differ in shape; view one with output_tensor(i)")
            off, shape = 0, (self.n, self.channels, self.length)
        else:
            off, ch, length = self.graph_output(i)
            shape = (ch, length)
        view = torch.as_tensor(_DeviceView(self, base + 4 * off, shape), device=self._device())
        self._views_out = True
        torch.cuda.current_stream(self._device()).wait_stream(self._engine_stream())
        return view

    def analyser_readouts(self, node, kind="frequency", byte=False):
        """Zero-copy torch view [n][K][row] of the declared read-outs (AnalyserNode.set_readouts) of `node` (an AnalyserNode of context 0,
        or its id) over the batch, when every context declares them alike on the same node id; otherwise fetch them per context
        (AnalyserNode.get_float_frequency_readouts / get_float_time_domain_readouts).  byte=True: the uint8 rows of
        AnalyserNode.set_byte_readouts.  Ordered like output_tensor: torch's current stream waits for the engine stream, and later runs,
        which overwrite the rows, wait for the work then queued on torch's stream."""
        kind_id = _readout_kind(kind)
        node_id = int(getattr(node, "id", node))
        count = C.c_uint64()
        if byte:
            p = C.c_void_p()
            self.api.check(self.api.batch_analyser_byte_readouts_device_ptr(self.handle, node_id, kind_id, C.byref(p), C.byref(count)))
        else:
            p = B.c_float_p()
            self.api.check(self.api.batch_analyser_readouts_device_ptr(self.handle, node_id, kind_id, C.byref(p), C.byref(count)))
        shapes = set()
        for c in self.contexts:
            a = c._readout_nodes.get(node_id)
            shapes.add(None if a is None else (a._readouts, a.fft_size // 2 if kind_id == B.READOUT_FREQUENCY else a.fft_size))
        return self._readout_view("analyser_readouts", p, count.value, shapes, "|u1" if byte else "<f4")

    def compressor_readouts(self, node):
        """Zero-copy torch view [n][K] of the declared reduction read-outs (DynamicsCompressorNode.set_readouts) of `node` (a
        DynamicsCompressorNode of context 0, or its id) over the batch, when every context declares them alike on the same node id;
        otherwise fetch them per context (DynamicsCompressorNode.get_reduction_readouts).  Ordered like analyser_readouts."""
        node_id = int(getattr(node, "id", node))
        p, count = B.c_float_p(), C.c_uint64()
        self.api.check(self.api.batch_compressor_readouts_device_ptr(self.handle, node_id, C.byref(p), C.byref(count)))
        shapes = set()
        for c in self.contexts:
            r = c._comp_readout_nodes.get(node_id)
            shapes.add(None if r is None else (r._readouts,))
        return self._readout_view("compressor_readouts", p, count.value, shapes, "<f4")

    def _readout_view(self, what, p, count, shapes, typestr):
        """[n][*shape] view of read-out rows at `p` (`count` elements over the batch) when every context has the one shape in `shapes`"""
        import torch
        shape = shapes.pop() if len(shapes) == 1 else None
        if shape is None or self.n * int(np.prod(shape)) != count:
            raise B.WaeError(2, f"{what}: the contexts declare different read-outs on this node; fetch them per context")
        addr = C.cast(p, C.c_void_p).value
        view = torch.as_tensor(_DeviceView(self, addr, (self.n,) + shape, typestr), device=self._device())
        self._readouts_viewed = True
        torch.cuda.current_stream(self._device()).wait_stream(self._engine_stream())
        return view

    def stats(self):
        s = B.BatchStats()
        self.api.check(self.api.batch_get_stats(self.handle, C.byref(s)))
        return s

    def stage_times(self):
        """[(kernel name, ms over the last run, instances)] — needs set_timing(True) before run()."""
        out, i = [], 0
        while True:
            name = C.create_string_buffer(64)
            ms, n = C.c_float(), C.c_uint32()
            if self.api.batch_stage_time(self.handle, i, name, C.byref(ms), C.byref(n)) != 0:
                break
            out.append((name.value.decode(), ms.value, n.value))
            i += 1
        return out

    def destroy(self):
        self._src_refs, self._ref_tensors = {}, []
        if self.handle:
            if not self._backend.closed:  # a batch must not outlive its engine
                self.api.batch_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.destroy()
        except Exception:
            pass


class _DeviceView:
    """__cuda_array_interface__ of a float32 (or, typestr "|u1", uint8) range of a batch's device memory; torch.as_tensor keeps this
    object, and so the batch, alive as long as the tensor."""

    def __init__(self, batch, ptr, shape, typestr="<f4"):
        self.batch = batch
        self.__cuda_array_interface__ = {"shape": tuple(int(s) for s in shape), "typestr": typestr, "data": (int(ptr), False),
                                         "version": 2}


def plan_batch(contexts):
    """wae_batch_plan: what the contexts would be lowered to (host only, no GPU) -> dict; raises what prepare would raise."""
    api = contexts[0]._api
    assert api.is_product
    for c in contexts:
        c._run_suspend_callbacks()
    arr = (C.c_void_p * len(contexts))(*[c._g for c in contexts])
    info = B.PlanInfo()
    api.check(api.batch_plan(arr, len(contexts), C.byref(info)))
    return _plan_dict(info)


def _plan_dict(info):
    kinds = {}
    for part in info.stage_kinds.decode().split(", "):
        if part:
            name, n = part.rsplit(" x ", 1)
            kinds[name] = int(n)
    return {"groups": info.groups, "segments": info.segments, "stages": info.stages, "has_feedback": bool(info.has_feedback),
            "chunk_frames": info.chunk_frames, "chunks": info.chunks, "arena_floats_per_frame": info.arena_floats_per_frame,
            "source_floats": info.source_floats, "kinds": kinds}


def plan_many(contexts):
    """wae_batch_plan_many: plan_batch for contexts of any mix of shapes -> the same dict, plus the grouping: "group_of" (the group of
    each context), "rendered_quanta" (each context rendered to its group's length) and "needed_quanta" (sum of ceil(length / 128))."""
    api = contexts[0]._api
    assert api.is_product
    for c in contexts:
        c._run_suspend_callbacks()
    n = len(contexts)
    arr = (C.c_void_p * n)(*[c._g for c in contexts])
    info = B.PlanInfo()
    api.check(api.batch_plan_many(arr, n, C.byref(info)))
    group_of = (C.c_uint32 * n)()
    rendered, needed = C.c_uint64(), C.c_uint64()
    api.check(api.batch_plan_quanta(arr, n, group_of, C.byref(rendered), C.byref(needed)))
    return dict(_plan_dict(info), group_of=list(group_of), rendered_quanta=rendered.value, needed_quanta=needed.value)


def render_many(contexts, outs=None):
    """ONE wae_render_many call for contexts of any mix of channel counts, lengths and sample rates -> a list of AudioBuffer, each of its
    context's own shape.  `outs`: optional list of float32 arrays, outs[i] with at least channels_i * length_i contiguous floats
    (pageable, or the numpy view of page-locked memory); the buffers then view them.  Product: one call; oracle (tests only): each
    context rendered on its own."""
    api = contexts[0]._api
    for c in contexts:
        c._run_suspend_callbacks()
    n = len(contexts)
    if outs is None:
        outs = [np.empty((c._channels, c._length), np.float32) for c in contexts]
    for c, o in zip(contexts, outs):
        assert o.dtype == np.float32 and o.flags.c_contiguous and o.size >= c._channels * c._length
    if api.is_product:
        arr = (C.c_void_p * n)(*[c._g for c in contexts])
        ptrs = (B.c_float_p * n)(*[B.fptr(o) for o in outs])
        api.check(api.render_many(contexts[0]._backend.engine, arr, n, ptrs))
    else:
        for c, o in zip(contexts, outs):
            secs = C.c_double()
            one = (C.c_void_p * 1)(c._g)
            api.check(api.render_many(one, 1, B.fptr(o), 1, C.byref(secs)))
    result = []
    for c, o in zip(contexts, outs):
        pcm = o.reshape(-1)[:c._channels * c._length].reshape(c._channels, c._length)
        result.append(AudioBuffer([pcm[k] for k in range(c._channels)], c._sample_rate))
    return result


def render_batch_oneshot(contexts, out=None):
    """ONE wae_render_batch(engine, graphs, n, out, HOST) call: sizing, planning, H2D of the source PCM, render and D2H overlapped inside
    the library (csrc/wae_engine.cu: render_oneshot_host) — the call the Rust binding makes from start_rendering_sync
    (INTEGRATION.md).  `out`: optional [n][channels][length] float32 array (pageable numpy memory, or the numpy view of a pinned torch
    tensor: the library copies straight into page-locked memory).  Product only."""
    ctx0 = contexts[0]
    api = ctx0._api
    n, ch, length = len(contexts), ctx0._channels, ctx0._length
    for c in contexts:
        c._run_suspend_callbacks()
    if out is None:
        out = np.empty((n, ch, length), np.float32)
    arr = (C.c_void_p * n)(*[c._g for c in contexts])
    api.check(api.render_batch(ctx0._backend.engine, arr, n, out.ctypes.data_as(C.c_void_p), 0))
    return out


def render_batch(contexts, threads=1):
    """Render many OfflineAudioContexts. Returns a list of AudioBuffer (one per context).

    Product: one wae_render_batch call.  Oracle (tests only): wao_render per context (optionally threaded)."""
    ctx0 = contexts[0]
    api = ctx0._api
    n, ch, length = len(contexts), ctx0._channels, ctx0._length
    for c in contexts:
        c._run_suspend_callbacks()
    out = np.empty((n, ch, length), np.float32)
    arr = (C.c_void_p * n)(*[c._g for c in contexts])
    if api.is_product:
        b = Batch(contexts)
        b.run()
        b.sync()
        b.fetch(out)
    else:
        secs = C.c_double()
        api.check(api.render_many(arr, n, B.fptr(out), threads, C.byref(secs)))
    return [AudioBuffer([out[i, c] for c in range(ch)], ctx0._sample_rate) for i in range(n)]
