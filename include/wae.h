/*
 * wae.h — C ABI of the H100 render-quantum engine ("wae" = web-audio engine).
 *
 * This is the drop-in boundary for web-audio-api-rs's OfflineAudioContext hot path.
 * The reference has NO FFI today: its plug-in point is the Rust trait
 *     AudioProcessor::process(inputs, outputs, params, scope) -> bool   (src/render/processor.rs:131-196)
 * driven one 128-frame quantum at a time by Graph::render (src/render/graph.rs:490-591) inside
 * RenderThread::render_audiobuffer_sync (src/render/thread.rs:260-302).  A per-quantum FFI is useless
 * for a GPU, so the boundary is graph-level and batch-level: the Rust side keeps its AudioNode /
 * AudioProcessor surface, forwards node construction / connect / param events / start-stop to the
 * calls below (they mirror the ControlMessage enum, src/message.rs:13-87), and replaces the quantum
 * loop of render_audiobuffer_sync with ONE call to wae_render_batch for many contexts at once.
 *
 * Conventions
 *   - every function returns wae_status (0 = ok); nothing unwinds across the boundary;
 *     wae_last_error() returns a thread-local, NUL-terminated description of the last failure.
 *     Reference behaviour being mirrored: argument validation panics on the control thread with
 *     DOMException-style messages (e.g. src/node/convolver.rs:264-275) -> WAE_INVALID_ARGUMENT /
 *     WAE_INVALID_STATE / WAE_NOT_SUPPORTED with the same message text.
 *   - plain pointers and sizes only; inputs are borrowed for the duration of the call and copied;
 *     outputs are caller-allocated.
 *   - node ids follow the reference's allocation exactly (src/context/concrete_base.rs:240,
 *     src/context/mod.rs:24-40): destination = 0, listener = 1, listener params = 2..=10, first user
 *     node = 11; a node takes its id BEFORE its AudioParams (oscillator N -> frequency N+1, detune N+2).
 *     The render order and therefore the f32 summation order of the mixer depend on these ids
 *     (src/render/graph.rs:443-479).
 *   - one host thread per engine at a time (the reference renders a context on the calling thread,
 *     src/context/offline.rs:157-185).
 *
 * The oracle (oracle/, test infrastructure only) exports the same graph-building surface with the
 * prefix wao_ so that parity tests can build one graph twice.
 */
#ifndef WAE_H
#define WAE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef WAE_API
#define WAE_API __attribute__((visibility("default")))
#endif

#define WAE_RENDER_QUANTUM_SIZE 128u /* src/lib.rs:18 */
#define WAE_MAX_CHANNELS 32u         /* src/lib.rs:21 */

typedef int32_t wae_status;
enum {
    WAE_OK = 0,
    WAE_INVALID_ARGUMENT = 1, /* RangeError / IndexSizeError / TypeError style panics          */
    WAE_INVALID_STATE = 2,    /* InvalidStateError (start twice, stop before start, ...)       */
    WAE_NOT_SUPPORTED = 3,    /* NotSupportedError in the reference (e.g. 3-channel IR)        */
    WAE_UNSUPPORTED = 4,      /* valid in the reference, not lowered to the GPU yet -> caller  */
                              /* falls back to the CPU renderer                                */
    WAE_CUDA_ERROR = 5,
    WAE_OUT_OF_MEMORY = 6,
    WAE_NO_DEVICE = 7
};

typedef struct wae_engine wae_engine; /* one per GPU / per process rank                        */
typedef struct wae_graph wae_graph;   /* one OfflineAudioContext (src/context/offline.rs:78)   */
typedef uint32_t wae_node_id;

/* ChannelCountMode / ChannelInterpretation, src/node/audio_node.rs (enum order kept) */
enum { WAE_COUNT_MODE_MAX = 0, WAE_COUNT_MODE_CLAMPED_MAX = 1, WAE_COUNT_MODE_EXPLICIT = 2 };
enum { WAE_INTERPRETATION_SPEAKERS = 0, WAE_INTERPRETATION_DISCRETE = 1 };

/* AudioNodeOptions (src/node/audio_node.rs:54-71). count == 0 means "node default". */
typedef struct wae_channel_config {
    uint32_t count;
    uint32_t count_mode;
    uint32_t interpretation;
} wae_channel_config;

/* AudioBuffer: planar f32 channels (src/buffer.rs:69-72). */
typedef struct wae_audio_buffer {
    uint32_t number_of_channels;
    uint64_t length; /* frames per channel */
    float sample_rate;
    const float* const* channels; /* [number_of_channels] pointers to `length` floats */
} wae_audio_buffer;

/* ---- node option structs: one per renderer of SURVEY §8(a) ------------------------------------- */

/* OscillatorType, src/node/oscillator.rs:74-87 */
enum { WAE_OSC_SINE = 0, WAE_OSC_SQUARE = 1, WAE_OSC_SAWTOOTH = 2, WAE_OSC_TRIANGLE = 3, WAE_OSC_CUSTOM = 4 };
/* OscillatorOptions, src/node/oscillator.rs:48-70. Params: 0 = frequency, 1 = detune. */
typedef struct wae_oscillator_options {
    uint32_t type;
    float frequency;
    float detune;
    const float* periodic_wave; /* custom only: precomputed wavetable (src/periodic_wave.rs:163-209) */
    uint32_t periodic_wave_len;
} wae_oscillator_options;
enum { WAE_OSC_PARAM_FREQUENCY = 0, WAE_OSC_PARAM_DETUNE = 1 };

/* BiquadFilterType, src/node/biquad_filter.rs:392-403 */
enum {
    WAE_BIQUAD_LOWPASS = 0, WAE_BIQUAD_HIGHPASS = 1, WAE_BIQUAD_BANDPASS = 2, WAE_BIQUAD_NOTCH = 3,
    WAE_BIQUAD_ALLPASS = 4, WAE_BIQUAD_PEAKING = 5, WAE_BIQUAD_LOWSHELF = 6, WAE_BIQUAD_HIGHSHELF = 7
};
/* BiquadFilterOptions, src/node/biquad_filter.rs:430-450. Params in creation order
 * (src/node/biquad_filter.rs:555-593): 0 = Q, 1 = detune, 2 = frequency, 3 = gain. */
typedef struct wae_biquad_options {
    uint32_t type;
    float q;
    float detune;
    float frequency;
    float gain;
    wae_channel_config channel_config;
} wae_biquad_options;
enum { WAE_BIQUAD_PARAM_Q = 0, WAE_BIQUAD_PARAM_DETUNE = 1, WAE_BIQUAD_PARAM_FREQUENCY = 2, WAE_BIQUAD_PARAM_GAIN = 3 };

/* IIRFilterOptions, src/node/iir_filter.rs (feedforward/feedback, 1..=20 coefficients, f64) */
typedef struct wae_iir_options {
    const double* feedforward;
    uint32_t feedforward_len;
    const double* feedback;
    uint32_t feedback_len;
    wae_channel_config channel_config;
} wae_iir_options;

/* GainOptions, src/node/gain.rs. Param 0 = gain. */
typedef struct wae_gain_options {
    float gain;
    wae_channel_config channel_config;
} wae_gain_options;

/* AudioBufferSourceOptions, src/node/audio_buffer_source.rs. Params: 0 = detune, 1 = playbackRate
 * (creation order). */
typedef struct wae_buffer_source_options {
    const wae_audio_buffer* buffer; /* may be NULL */
    float detune;
    float playback_rate;
    uint32_t loop;
    double loop_start;
    double loop_end;
} wae_buffer_source_options;
enum { WAE_ABSN_PARAM_DETUNE = 0, WAE_ABSN_PARAM_PLAYBACK_RATE = 1 };

/* ConstantSourceOptions, src/node/constant_source.rs. Param 0 = offset. */
typedef struct wae_constant_source_options {
    float offset;
} wae_constant_source_options;

/* ConvolverOptions, src/node/convolver.rs:55-81 (default channel config ClampedMax / 2 / Speakers) */
typedef struct wae_convolver_options {
    const wae_audio_buffer* buffer; /* may be NULL: pass-through (convolver.rs:368-375) */
    uint32_t disable_normalization;
    wae_channel_config channel_config;
} wae_convolver_options;

/* OverSampleType, src/node/waveshaper.rs */
enum { WAE_OVERSAMPLE_NONE = 0, WAE_OVERSAMPLE_X2 = 1, WAE_OVERSAMPLE_X4 = 2 };
typedef struct wae_wave_shaper_options {
    const float* curve; /* may be NULL: pass-through */
    uint32_t curve_len;
    uint32_t oversample;
    wae_channel_config channel_config;
} wae_wave_shaper_options;

/* DelayOptions, src/node/delay.rs. Param 0 = delayTime. */
typedef struct wae_delay_options {
    double max_delay_time; /* default 1.0 */
    double delay_time;
    wae_channel_config channel_config;
} wae_delay_options;

/* StereoPannerOptions, src/node/stereo_panner.rs. Param 0 = pan. */
typedef struct wae_stereo_panner_options {
    float pan;
    wae_channel_config channel_config;
} wae_stereo_panner_options;

/* PannerOptions, src/node/panner.rs. Params in creation order:
 * 0..2 = positionX/Y/Z, 3..5 = orientationX/Y/Z. */
enum { WAE_PANNING_EQUALPOWER = 0, WAE_PANNING_HRTF = 1 };
enum { WAE_DISTANCE_LINEAR = 0, WAE_DISTANCE_INVERSE = 1, WAE_DISTANCE_EXPONENTIAL = 2 };
typedef struct wae_panner_options {
    uint32_t panning_model;
    uint32_t distance_model;
    float position_x, position_y, position_z;
    float orientation_x, orientation_y, orientation_z;
    double ref_distance, max_distance, rolloff_factor;
    double cone_inner_angle, cone_outer_angle, cone_outer_gain;
    wae_channel_config channel_config;
} wae_panner_options;

/* AnalyserOptions, src/node/analyser.rs */
typedef struct wae_analyser_options {
    uint32_t fft_size; /* 32..32768, power of two, default 2048 */
    double smoothing_time_constant; /* default 0.8 */
    double min_decibels;            /* default -100 */
    double max_decibels;            /* default -30 */
    wae_channel_config channel_config;
} wae_analyser_options;

/* DynamicsCompressorOptions, src/node/dynamics_compressor.rs. Params in creation order:
 * 0 = attack, 1 = knee, 2 = ratio, 3 = release, 4 = threshold. */
typedef struct wae_dynamics_compressor_options {
    float attack, knee, ratio, release, threshold;
    wae_channel_config channel_config;
} wae_dynamics_compressor_options;

typedef struct wae_channel_merger_options {
    uint32_t number_of_inputs; /* default 6 */
} wae_channel_merger_options;
typedef struct wae_channel_splitter_options {
    uint32_t number_of_outputs; /* default 6 */
} wae_channel_splitter_options;

/* AudioParamEventType, src/param.rs:160-170 (enum order kept) */
enum {
    WAE_EVENT_SET_VALUE = 0,
    WAE_EVENT_SET_VALUE_AT_TIME = 1,
    WAE_EVENT_LINEAR_RAMP_TO_VALUE_AT_TIME = 2,
    WAE_EVENT_EXPONENTIAL_RAMP_TO_VALUE_AT_TIME = 3,
    WAE_EVENT_CANCEL_SCHEDULED_VALUES = 4,
    WAE_EVENT_SET_TARGET_AT_TIME = 5,
    WAE_EVENT_CANCEL_AND_HOLD_AT_TIME = 6,
    WAE_EVENT_SET_VALUE_CURVE_AT_TIME = 7
};
enum { WAE_AUTOMATION_RATE_A = 0, WAE_AUTOMATION_RATE_K = 1 };

/* AudioParam automation call (src/param.rs:403-640): `time` is start/end/cancel time as in the
 * method of the same name; `aux` = timeConstant (set_target) or duration (set_value_curve);
 * `values` only for set_value_curve. */
typedef struct wae_param_event {
    uint32_t type;
    float value;
    double time;
    double aux;
    const float* values;
    uint32_t values_len;
} wae_param_event;

/* ---- engine ------------------------------------------------------------------------------------ */

/* device_ordinal: CUDA device of this process rank. Fails with WAE_NO_DEVICE when no sm_90 GPU (H100) is
 * usable — there is NO CPU fallback in this library. */
WAE_API wae_status wae_engine_create(int32_t device_ordinal, wae_engine** out_engine);
WAE_API wae_status wae_engine_destroy(wae_engine* engine);
WAE_API const char* wae_last_error(void);
WAE_API const char* wae_version(void);

/* Engine tunables (all optional). */
enum {
    WAE_OPT_CHUNK_FRAMES = 1,   /* frames rendered per time chunk (multiple of 128; 0 = auto)      */
    WAE_OPT_FUSE = 2,           /* 1 (default): fuse source->filter->gain chains; 0: one stage/node */
    WAE_OPT_SERIAL_FILTERS = 3, /* 1: bit-faithful serial recurrences (thread per channel)          */
    WAE_OPT_PIPELINE_GROUPS = 4, /* graph groups of the H2D/render/D2H pipeline (0 = auto: 8)       */
    WAE_OPT_PARAM_PARALLEL = 5,  /* AudioParam kernel. 2 (default): one CTA per param, 32 quanta walked speculatively at once and verified;
                                  * 1: one warp per param, the fills of a quantum evaluated by the warp; 0: one lane evaluates every frame.
                                  * The three are bit-identical (tests/test_gpu_criterion_and_setters.py). */
    WAE_OPT_BIND_NUMA = 6,       /* 1: pin the calling thread and the engine's host workers to the CPUs of the GPU's NUMA node (before the first render) */
    WAE_OPT_HOST_WORKERS = 7,    /* host worker threads (planning, copy-out to pageable buffers); 0 = auto (hardware threads / 8, 2..16) */
    WAE_OPT_CHAIN_TMA = 8,       /* process-wide: 1 = the fused chain kernel streams PCM with cp.async.bulk (TMA), 0 = with cp.async */
    WAE_OPT_CHAIN_WAVES = 9,     /* process-wide: time slabs of the fused chain kernel are sized for this many waves of CTAs; 0 = one slab */
    WAE_OPT_CHAIN_PREPASS = 10,  /* process-wide, 1 (default): few (graph, channel) pairs with long renders through one biquad are cut into time slabs
                                  * that find out what they hand on before they render (one extra read of the source), so that the slabs of
                                  * a pair run concurrently; 0: one CTA per pair walks the whole render */
    WAE_OPT_VOICE_SUM = 11       /* 0 (default): oscillator voices are rendered into buffers by the chain kernel and summed by the mixer kernel;
                                  * 1: an input fed by many oscillator -> [biquad] -> gain voices is rendered by ONE kernel that keeps the running
                                  * sum in registers and walks the voices in edge order (no voice is written to memory) when the launch has enough
                                  * (time tile, port) work items; 2: whenever the port has the shape (tests).  Measured slower than the two
                                  * kernels it replaces (DESIGN.md section 2): kept as an option */
};
WAE_API wae_status wae_engine_set_option(wae_engine* engine, uint32_t option, int64_t value);
/* the cudaStream_t every kernel of this engine is launched on (callers that time with their own CUDA events) */
WAE_API wae_status wae_engine_stream(wae_engine* engine, void** out_stream);

/* ---- graph construction = OfflineAudioContext::new + BaseAudioContext::create_* ----------------- */

/* OfflineAudioContext::new(number_of_channels, length, sample_rate), src/context/offline.rs:78.
 * `engine` may be NULL: graph construction is host work (validation, id allocation, the event queues), the graph meets a
 * device only when it is handed to wae_batch_prepare / wae_render_batch, which take the engine themselves. */
WAE_API wae_status wae_graph_create(wae_engine* engine, uint32_t number_of_channels, uint64_t length,
                                    float sample_rate, wae_graph** out_graph);
/* The order the graph's nodes are processed in within one quantum, as the planner derives it: Graph::order_nodes
 * (src/render/graph.rs:331-487: depth-first over ascending ids, reversed post-order, DelayWriters of a cycle lose their
 * outgoing edges, nodes of a cycle without a delay are dropped).  Fills at most `cap` ids, *n = the full count. Host work. */
WAE_API wae_status wae_graph_render_order(wae_graph* graph, wae_node_id* ids, uint32_t cap, uint32_t* n);
WAE_API wae_status wae_graph_destroy(wae_graph* graph);

/* BaseAudioContext::create_* (src/context/base.rs:26-361) / XxxNode::new(context, options). */
WAE_API wae_status wae_create_oscillator(wae_graph*, const wae_oscillator_options*, wae_node_id* out);
WAE_API wae_status wae_create_biquad_filter(wae_graph*, const wae_biquad_options*, wae_node_id* out);
WAE_API wae_status wae_create_iir_filter(wae_graph*, const wae_iir_options*, wae_node_id* out);
WAE_API wae_status wae_create_gain(wae_graph*, const wae_gain_options*, wae_node_id* out);
WAE_API wae_status wae_create_buffer_source(wae_graph*, const wae_buffer_source_options*, wae_node_id* out);
WAE_API wae_status wae_create_constant_source(wae_graph*, const wae_constant_source_options*, wae_node_id* out);
WAE_API wae_status wae_create_convolver(wae_graph*, const wae_convolver_options*, wae_node_id* out);
WAE_API wae_status wae_create_wave_shaper(wae_graph*, const wae_wave_shaper_options*, wae_node_id* out);
WAE_API wae_status wae_create_delay(wae_graph*, const wae_delay_options*, wae_node_id* out);
WAE_API wae_status wae_create_stereo_panner(wae_graph*, const wae_stereo_panner_options*, wae_node_id* out);
WAE_API wae_status wae_create_panner(wae_graph*, const wae_panner_options*, wae_node_id* out);
WAE_API wae_status wae_create_analyser(wae_graph*, const wae_analyser_options*, wae_node_id* out);
WAE_API wae_status wae_create_dynamics_compressor(wae_graph*, const wae_dynamics_compressor_options*, wae_node_id* out);
WAE_API wae_status wae_create_channel_merger(wae_graph*, const wae_channel_merger_options*, wae_node_id* out);
WAE_API wae_status wae_create_channel_splitter(wae_graph*, const wae_channel_splitter_options*, wae_node_id* out);

/* AudioNode::connect_from_output_to_input (src/node/audio_node.rs:259-289); destination is node 0. */
WAE_API wae_status wae_connect(wae_graph*, wae_node_id from, uint32_t output, wae_node_id to, uint32_t input);
/* AudioNode::connect(&param): audio-rate modulation of a param (src/param.rs:762-796). */
/* Host-side simulation of ONE AudioParam, block by block (no GPU involved): the engine's event folding and per-quantum state
 * machine — the code the planner and the k_param kernel run — driven like the reference's unit tests drive
 * AudioParamProcessor (src/param.rs:1766-3545: handle_incoming_event, then compute_intrinsic_values(block_time, dt, count)).
 * `out` holds `count` (<= 128) floats; *len = 1 for a single-valued block, else count. */
typedef struct wae_param_sim wae_param_sim;
WAE_API wae_status wae_param_sim_create(uint32_t a_rate, float default_value, float min_value, float max_value, wae_param_sim** out);
WAE_API wae_status wae_param_sim_destroy(wae_param_sim* sim);
WAE_API wae_status wae_param_sim_push(wae_param_sim* sim, const wae_param_event* event);
WAE_API wae_status wae_param_sim_set_automation_rate(wae_param_sim* sim, uint32_t a_rate);
/* which implementation of the state machine wae_param_sim_compute runs: 0 = csrc/wae_param_core.h (k_param), 1 / 2 = the sink-based
 * walker with its serial / recording sink (csrc/wae_param_walk.h; k_param_parallel), 3 = the recording sink walked from predicted states
 * that are verified against the previous quantum's result first, as the default kernel k_param_spec does with 32 quanta at a time.
 * wae_param_sim_speculation reports how many predictions walker 3 made and how many held. */
WAE_API wae_status wae_param_sim_set_walker(wae_param_sim* sim, uint32_t walker);
WAE_API wae_status wae_param_sim_speculation(wae_param_sim* sim, uint64_t* tried, uint64_t* hits);
WAE_API wae_status wae_param_sim_compute(wae_param_sim* sim, double block_time, double dt, uint32_t count, float* out, uint32_t* len);

/* OfflineAudioContext::suspend_sync(suspend_time, callback) (src/context/offline.rs:330-387): call this, then run the
 * callback; graph mutations issued afterwards (new nodes, connections, param events, start / stop) take effect at the
 * suspend frame (suspend_time quantised up to a render quantum).  Suspend points must be taken in increasing time order. */
WAE_API wae_status wae_graph_suspend(wae_graph* graph, double suspend_time);

/* `to` = 1 (WAE_LISTENER_NODE) addresses the AudioListener's params: 0..8 = position xyz, forward xyz, up xyz */
WAE_API wae_status wae_connect_param(wae_graph*, wae_node_id from, uint32_t output, wae_node_id to, uint32_t param_index);
/* AudioNode::disconnect() — removes all outgoing connections of `from`. */
WAE_API wae_status wae_disconnect(wae_graph*, wae_node_id from);
/* The selective forms (src/node/audio_node.rs:304-405), all of them ConcreteBaseAudioContext::disconnect(from, Option<output>, Option<to>,
 * Option<input>) (src/context/concrete_base.rs:474-507): disconnect_output(o) = (from, o, WAE_NODE_NONE, -1); disconnect_dest(d) =
 * (from, -1, d, -1); disconnect_dest_from_output(d, o) = (from, o, d, -1); disconnect_dest_from_output_to_input(d, o, i) = (from, o, d, i).
 * Naming a destination that is not connected answers "InvalidAccessError - attempting to disconnect unconnected nodes". */
#define WAE_NODE_NONE 0xFFFFFFFFu
WAE_API wae_status wae_disconnect_from(wae_graph*, wae_node_id from, int32_t output, wae_node_id to, int32_t input);
/* ... and towards an AudioParam of `to` (node.disconnect_dest(&param)) */
WAE_API wae_status wae_disconnect_param(wae_graph*, wae_node_id from, int32_t output, wae_node_id to, uint32_t param_index);

/* AudioParam methods (src/param.rs:336-662). */
WAE_API wae_status wae_param_event_push(wae_graph*, wae_node_id node, uint32_t param_index, const wae_param_event* event);
WAE_API wae_status wae_param_set_automation_rate(wae_graph*, wae_node_id node, uint32_t param_index, uint32_t rate);
/* AudioListener params (src/spatial.rs): index 0..8 = position xyz, forward xyz, up xyz. */
WAE_API wae_status wae_listener_param_event_push(wae_graph*, uint32_t param_index, const wae_param_event* event);

/* AudioScheduledSourceNode (src/node/scheduled_source.rs:12-54): start_at / stop_at, and
 * AudioBufferSourceNode::start_at_with_offset_and_duration. Pass offset = 0, duration = +inf
 * (or any value >= 1e300) for the plain start_at. */
WAE_API wae_status wae_source_start(wae_graph*, wae_node_id node, double when, double offset, double duration);
WAE_API wae_status wae_source_stop(wae_graph*, wae_node_id node, double when);

/* Setters that exist as control messages in the reference. */
WAE_API wae_status wae_oscillator_set_type(wae_graph*, wae_node_id node, uint32_t type);
WAE_API wae_status wae_biquad_set_type(wae_graph*, wae_node_id node, uint32_t type);

/* ---- rendering = OfflineAudioContext::start_rendering_sync for a whole batch ------------------- */

enum {
    WAE_RENDER_OUT_HOST = 0,   /* `out` is host memory (pageable or pinned)                         */
    WAE_RENDER_OUT_DEVICE = 1  /* `out` is device memory on the engine's GPU                       */
};

/* Renders every graph of the batch from frame 0 to its length. All graphs of one batch must have
 * the same number_of_channels, length and sample_rate (independent OfflineAudioContexts that only
 * differ in their node graphs / assets).  Output layout: planar [n_graphs][number_of_channels][length]
 * f32, i.e. the AudioBuffer each start_rendering_sync would return (src/render/thread.rs:298-301),
 * back to back.  The call is synchronous: on return `out` is complete. */
WAE_API wae_status wae_render_batch(wae_engine* engine, wae_graph* const* graphs, uint32_t n_graphs,
                                    float* out, uint32_t flags);

/* Page-locked host memory for output buffers a caller keeps around: with WAE_RENDER_OUT_HOST the rendered PCM is DMA-ed straight into a
 * page-locked `out` (pageable memory goes through staging slots and copy-out threads inside the library).  wae_host_register
 * page-locks memory the caller allocated itself; it must stay allocated until wae_host_unregister. */
WAE_API wae_status wae_host_alloc(wae_engine* engine, uint64_t bytes, void** out);
WAE_API wae_status wae_host_free(wae_engine* engine, void* p);
WAE_API wae_status wae_host_register(wae_engine* engine, void* p, uint64_t bytes);
WAE_API wae_status wae_host_unregister(wae_engine* engine, void* p);

/* Diagnostics: runs the convolver's 8192-point shared-memory transforms on the HOST with the same butterfly / index / twiddle code the
 * kernels compile (no GPU needed), in place on 16384 floats.  mode 0: complex forward, natural order in, bit-reversed ("position") order
 * out; 1: complex inverse (unnormalised), position order in, natural out; 2: 16384 reals -> 8192 packed bins (bin 0 = DC, Nyquist) in
 * position order; 3: the inverse of 2 (scaled).  tests/test_conv_fft_host.py pins them against numpy. */
WAE_API wae_status wae_selftest_conv_fft(float* data, uint32_t mode);

/* Two-phase variant used by bench.py and by callers that render the same batch repeatedly or keep
 * PCM on the device for the NCCL gather: prepare uploads assets and compiles the stage schedule,
 * run renders (device-resident output owned by the engine), fetch copies to the host. */
typedef struct wae_batch wae_batch;
WAE_API wae_status wae_batch_prepare(wae_engine* engine, wae_graph* const* graphs, uint32_t n_graphs, wae_batch** out_batch);
/* re-upload the source PCM of every AudioBufferSourceNode from host memory (pinned at prepare) — the H2D
 * leg of an end-to-end step when the same batch is rendered repeatedly */
WAE_API wae_status wae_batch_upload(wae_batch* batch);                    /* async on the engine stream   */
/* per_stage != 0: record CUDA events around every stage (diagnostic: serialises chunks) */
WAE_API wae_status wae_batch_set_timing(wae_batch* batch, uint32_t per_stage);
WAE_API wae_status wae_batch_run(wae_batch* batch);                       /* async on the engine stream   */
/* End-to-end render of a PREPARED batch with HOST buffers: per graph group H2D(source PCM) -> render -> D2H into host_out
 * ([n_graphs][channels][length] f32, ideally page-locked), the three legs of neighbouring groups overlapped on three
 * streams.  Synchronous.  Source PCM is copied from where wae_create_buffer_source / set_buffer put it (page-locked when the
 * graph has an engine; otherwise a pinned mirror is built on the first call).  The one-shot equivalent — planning included and
 * overlapped, pageable `out` served through staging slots — is wae_render_batch(..., WAE_RENDER_OUT_HOST). */
WAE_API wae_status wae_batch_run_pipelined(wae_batch* batch, float* host_out);
/* Graph groups of a prepared batch (contiguous graph ranges [first, last) rendered one after the other) and the render of ONE
 * group, asynchronous on the engine stream: lets a caller interleave its own work per group — bench.py overlaps the NCCL
 * all-gather of group k's PCM with the render of group k+1.  Group 0 also resets the per-run node state; call the groups in order. */
WAE_API wae_status wae_batch_group_count(wae_batch* batch, uint32_t* n_groups);
WAE_API wae_status wae_batch_group_range(wae_batch* batch, uint32_t group, uint32_t* first_graph, uint32_t* last_graph);
WAE_API wae_status wae_batch_run_group(wae_batch* batch, uint32_t group);
WAE_API wae_status wae_batch_sync(wae_batch* batch);                      /* wait for the stream           */
WAE_API wae_status wae_batch_output_device_ptr(wae_batch* batch, float** out_dev, uint64_t* out_floats);
WAE_API wae_status wae_batch_fetch(wae_batch* batch, float* host_out);   /* D2H of the whole output       */
WAE_API wae_status wae_batch_destroy(wae_batch* batch);

/* Introspection used by bench.py / tests (counts since prepare). */
typedef struct wae_batch_stats {
    uint64_t kernel_launches_per_run; /* launches of OUR kernels per wae_batch_run                  */
    uint64_t stages;                  /* stages in the compiled schedule                            */
    uint64_t chunks;                  /* time chunks per run                                        */
    uint64_t arena_bytes;             /* device bytes of edge buffers + state                        */
    uint64_t asset_bytes;             /* device bytes of uploaded assets (buffers, IR spectra, ...)  */
    uint64_t algorithmic_bytes;       /* SURVEY §8(d) compulsory HBM bytes per run                   */
    uint64_t graph_quanta;            /* n_graphs * ceil(length / 128)                               */
    float last_run_ms;                /* CUDA-event time of the last completed run                   */
    float dominant_kernel_ms;         /* CUDA-event time of the dominant stage kernel in last run    */
    char dominant_kernel[64];
} wae_batch_stats;
WAE_API wae_status wae_batch_get_stats(wae_batch* batch, wae_batch_stats* out);
/* device time of stage `index` summed over the chunks of the last run (needs wae_batch_set_timing(batch, 1));
 * returns WAE_INVALID_ARGUMENT past the last stage */
WAE_API wae_status wae_batch_stage_time(wae_batch* batch, uint32_t index, char* name64, float* ms, uint32_t* n_instances);

/* AnalyserNode read-out after a render (src/node/analyser.rs:246-264, src/analysis.rs:347-401):
 * state of the analyser at the end of the render. */
WAE_API wae_status wae_analyser_get_float_time_domain_data(wae_batch*, uint32_t graph_index, wae_node_id node, float* out, uint32_t len);
WAE_API wae_status wae_analyser_get_float_frequency_data(wae_batch*, uint32_t graph_index, wae_node_id node, float* out, uint32_t len);

/* AnalyserNode read-outs at declared render times, taken on the GPU during a run of a prepared batch.
 *
 * wae_analyser_set_readouts declares read-outs at `times` (seconds, n >= 1, non-decreasing).  Each time is quantised as
 * suspend_sync quantises it (q = ceil(t * sampleRate / 128), offline.rs:248-251, 0 <= q <= the graph's whole quanta): read-out k
 * is what Analyser::get_float_frequency_data / get_float_time_domain_data return in a suspend callback at quantum q, i.e. at
 * current_time = q * 128 / sampleRate over the fftSize frames before frame q * 128 (frames before the render are zeros).
 * Frequency read-outs smooth in time order from a zero state each run; two read-outs on one quantum give the same row.  The
 * post-render wae_analyser_get_float_frequency_data continues that smoothing.  `kinds`: WAE_READOUT_* bits.
 * Refused: a node that is not an analyser, n == 0, a negative / non-finite / decreasing time, a quantum past the render, kinds
 * 0 or unknown bits (WAE_INVALID_ARGUMENT); a second declaration on the node or a graph with a suspend point
 * (WAE_INVALID_STATE; wae_graph_suspend refuses a graph with a declaration).  One-shot renders refuse declared graphs.
 *
 * After a run: wae_batch_analyser_readouts_device_ptr gives the device memory of one (node, kind) over the whole batch, graphs
 * in the order they were passed to prepare, each [k][row] (row = fftSize / 2 dB values or fftSize samples; a graph without the
 * declaration takes no space), `floats` in all; wae_batch_fetch_analyser_readouts copies one graph's [k][row] to the host
 * (`floats` must be K * row).  Each run overwrites the rows. */
enum { WAE_READOUT_FREQUENCY = 1, WAE_READOUT_TIME_DOMAIN = 2 };
WAE_API wae_status wae_analyser_set_readouts(wae_graph* graph, wae_node_id node, const double* times, uint32_t n, uint32_t kinds);
WAE_API wae_status wae_batch_analyser_readouts_device_ptr(wae_batch* batch, wae_node_id node, uint32_t kind, float** ptr, uint64_t* floats);
WAE_API wae_status wae_batch_fetch_analyser_readouts(wae_batch* batch, uint32_t graph_index, wae_node_id node, uint32_t kind, float* host_out,
                                                     uint64_t floats);

/* Byte read-outs: wae_analyser_set_byte_readouts delivers the declared read-outs of `kinds` (a non-empty subset of the kinds given to
 * wae_analyser_set_readouts) as bytes too, at the same times: row k is what Analyser::get_byte_frequency_data /
 * get_byte_time_domain_data return in a suspend callback at quantum q_k (src/analysis.rs:266-276, 371-401).  A byte frequency row is
 * (u8) clamp(255 / (maxDecibels - minDecibels) * (dB - minDecibels), 0, 255) in f32 of the float row's dB (one smoothing step serves
 * both, as last_fft_time makes it in the reference; minDecibels / maxDecibels are the node's at render time); a byte time-domain row
 * is (u8) clamp(128 * (1 + x), 0, 255), NaN -> 0.  The float rows are unchanged by the declaration.  Refused: a node that is not an
 * analyser, kinds 0, unknown bits (WAE_INVALID_ARGUMENT) or not declared by wae_analyser_set_readouts (WAE_INVALID_ARGUMENT); no
 * read-outs declared yet, a second declaration or a graph with a suspend point (WAE_INVALID_STATE).
 * wae_batch_analyser_byte_readouts_device_ptr / wae_batch_fetch_analyser_byte_readouts: as the float pair, laid out alike (one
 * allocation per (node, kind), graphs in prepare order, each [k][row]; a graph without the byte declaration takes no space). */
WAE_API wae_status wae_analyser_set_byte_readouts(wae_graph* graph, wae_node_id node, uint32_t kinds);
WAE_API wae_status wae_batch_analyser_byte_readouts_device_ptr(wae_batch* batch, wae_node_id node, uint32_t kind, uint8_t** ptr,
                                                               uint64_t* bytes);
WAE_API wae_status wae_batch_fetch_analyser_byte_readouts(wae_batch* batch, uint32_t graph_index, wae_node_id node, uint32_t kind,
                                                          uint8_t* host_out, uint64_t bytes);

/* DynamicsCompressorNode::reduction at declared render times, taken on the GPU during a run of a prepared batch.
 *
 * wae_compressor_set_readouts declares read-outs at `times` (seconds), validated and quantised as wae_analyser_set_readouts does:
 * read-out k is what DynamicsCompressorNode::reduction returns in a suspend callback at quantum q_k, i.e. the reduction (dB) of the
 * last frame of quantum q_k - 1 (dynamics_compressor.rs:440, 450), 0 for q_k = 0; at the end quantum it equals what
 * wae_compressor_reduction answers after the render.  Refused: a node that is not a DynamicsCompressorNode, n == 0, a negative /
 * non-finite / decreasing time, a quantum past the render (WAE_INVALID_ARGUMENT); a second declaration on the node or a graph with a
 * suspend point (WAE_INVALID_STATE; wae_graph_suspend refuses a graph with a declaration).  One-shot renders refuse declared graphs.
 *
 * After a run: wae_batch_compressor_readouts_device_ptr gives the device memory of one node's rows over the whole batch, graphs in the
 * order they were passed to prepare, each [k] (a graph without the declaration takes no space), `floats` in all;
 * wae_batch_fetch_compressor_readouts copies one graph's [k] to the host (`floats` must be K).  Each run overwrites the rows. */
WAE_API wae_status wae_compressor_set_readouts(wae_graph* graph, wae_node_id node, const double* times, uint32_t n);
WAE_API wae_status wae_batch_compressor_readouts_device_ptr(wae_batch* batch, wae_node_id node, float** ptr, uint64_t* floats);
WAE_API wae_status wae_batch_fetch_compressor_readouts(wae_batch* batch, uint32_t graph_index, wae_node_id node, float* host_out,
                                                       uint64_t floats);

/* load_hrtf_processor (src/node/panner.rs:39-68): the HRIR sphere the reference embeds with include_bytes!
 * ("resources/IRC_1003_C.bin": "HRIR" | u32 rate | u32 taps | u32 #vertices | u32 #indices | indices | per vertex xyz,
 * left[taps], right[taps]).  Must be set before a batch with PanningModelType::HRTF panners is prepared; contexts whose
 * sample rate differs from the sphere's are WAE_UNSUPPORTED (the hrtf crate's rubato resampling is not lowered). */
WAE_API wae_status wae_engine_set_hrir_sphere(wae_engine* engine, const void* data, uint64_t len);

/* Analyser::get_byte_time_domain_data / get_byte_frequency_data (src/analysis.rs:266-276, 371-401) */
WAE_API wae_status wae_analyser_get_byte_time_domain_data(wae_batch* batch, uint32_t graph_index, wae_node_id node, uint8_t* out, uint32_t len);
WAE_API wae_status wae_analyser_get_byte_frequency_data(wae_batch* batch, uint32_t graph_index, wae_node_id node, uint8_t* out, uint32_t len);

/* DynamicsCompressorNode::reduction (src/node/dynamics_compressor.rs:204-206): gain reduction (dB) at the end of the render */
WAE_API wae_status wae_compressor_reduction(wae_batch* batch, uint32_t graph_index, wae_node_id node, float* out);
/* (the reduction over the render: wae_compressor_set_readouts above) */

/* AudioBuffer::resample (src/buffer.rs:311-363) on the GPU: linear interpolation keeping the first and last frame; the
 * input side of the path (decode_audio_data resamples buffers to the context rate).  Host pointers. */
WAE_API wae_status wae_resample_linear(wae_engine* engine, const float* in, uint64_t len, float from_rate, float to_rate, float* out,
                                       uint64_t out_cap, uint64_t* out_len);

/* What wae_batch_prepare would lower `graphs` to, computed on the host only (no engine, no device, default engine options): the planner's
 * sizing pass.  Errors are the ones prepare would report (WAE_UNSUPPORTED for what is not lowered, WAE_INVALID_ARGUMENT ...). */
typedef struct wae_plan_info {
    uint32_t groups;                 /* graph groups of the H2D / render / D2H pipeline                                  */
    uint32_t segments;               /* render segments over all groups (1 per group without wae_graph_suspend points)    */
    uint32_t stages;                 /* kernel launches per chunk, summed over groups and segments                        */
    uint32_t has_feedback;           /* some graph has a cycle broken by a DelayNode                                      */
    uint64_t chunk_frames;           /* frames rendered per time chunk                                                    */
    uint64_t chunks;                 /* chunks per render                                                                 */
    uint64_t arena_floats_per_frame; /* edge buffers of the largest group, floats per frame                               */
    uint64_t source_floats;          /* AudioBuffer PCM resident on the device, floats                                    */
    char stage_kinds[512];           /* "k_chain x 1, k_mix x 1": the stages by kernel                                    */
} wae_plan_info;
WAE_API wae_status wae_batch_plan(wae_graph* const* graphs, uint32_t n_graphs, wae_plan_info* info);

/* ---- batches of contexts that differ in number_of_channels, length or sample_rate --------------------------------------------
 * The calls above take graphs of one shape and refuse anything else.  The calls below take any mix.  Graphs are grouped by
 * sample rate, suspend frames and length; a group renders all its graphs to its longest graph's length (whole quanta), and the
 * shortest graph of a group is at least 3/4 of the longest.  Each graph's output, analyser and compressor read-outs are exactly
 * what it renders alone.  A batch whose graphs all share one shape is planned exactly as by wae_batch_prepare / wae_batch_plan. */

/* OfflineAudioContext::start_rendering_sync for each graph, in one call: outs[i] = [channels_i][length_i] f32 host memory (pageable
 * or page-locked) of graph i.  Synchronous. */
WAE_API wae_status wae_render_many(wae_engine* engine, wae_graph* const* graphs, uint32_t n_graphs, float* const* outs);
/* wae_batch_prepare for any mix of shapes.  run / run_group / sync / stats / destroy, the analyser read-outs and
 * wae_compressor_reduction work on the batch (graph_index = the graph's index in `graphs`).  The device output is packed: see
 * wae_batch_graph_output.  On a batch whose graphs differ in shape wae_batch_fetch and wae_batch_run_pipelined answer
 * WAE_INVALID_STATE, and the ranges of wae_batch_group_range index the batch's own order (graphs sorted into groups). */
WAE_API wae_status wae_batch_prepare_many(wae_engine* engine, wae_graph* const* graphs, uint32_t n_graphs, wae_batch** out_batch);
/* where graph `graph_index` lies in wae_batch_output_device_ptr's buffer: [channels][length] f32 from offset_floats on */
WAE_API wae_status wae_batch_graph_output(wae_batch* batch, uint32_t graph_index, uint64_t* offset_floats, uint32_t* channels, uint64_t* length);
/* D2H of one graph's rendered PCM into `out` ([channels][length] f32) */
WAE_API wae_status wae_batch_fetch_graph(wae_batch* batch, uint32_t graph_index, float* out);
/* wae_batch_plan for any mix of shapes (host only) */
WAE_API wae_status wae_batch_plan_many(wae_graph* const* graphs, uint32_t n_graphs, wae_plan_info* info);
/* The grouping wae_batch_plan_many / wae_batch_prepare_many / wae_render_many make under the default engine options (host only):
 * group_of[i] (may be NULL; n_graphs entries) = the group of graph i; *rendered = render quanta over all graphs (each graph rendered
 * to its group's length); *needed = the sum over graphs of ceil(length_i / 128). */
WAE_API wae_status wae_batch_plan_quanta(wae_graph* const* graphs, uint32_t n_graphs, uint32_t* group_of, uint64_t* rendered, uint64_t* needed);

/* ---- source audio bound from device memory ---------------------------------------------------------------------------------
 * A prepared batch renders the PCM its graphs were built with; the calls below let it render new audio that already lives on the GPU
 * (decoded, augmented or generated there) without building, planning or uploading anything again: declare the source at build time,
 * prepare once, then any number of times bind new device audio, run, and read the output on the device (wae_batch_output_device_ptr).
 * wae_render_batch and wae_render_many answer WAE_INVALID_STATE on graphs with device inputs (a one-shot call leaves no point to bind
 * at); wae_batch_plan / wae_batch_plan_many plan them as usual. */

/* An AudioBufferSourceNode whose PCM is supplied per run from device memory (wae_batch_bind_sources) instead of an AudioBuffer.
 * Counts as the node's buffer: the node then behaves exactly like one given an AudioBuffer of this shape.  Same validation and texts
 * as AudioBuffer::new (channels 1..32, length > 0), same "cannot assign buffer twice" rule as set_buffer, in both directions. */
WAE_API wae_status wae_buffer_source_set_device_input(wae_graph* graph, wae_node_id node, uint32_t number_of_channels,
                                                      uint64_t length, float sample_rate);

/* A device input read where the caller keeps it: validated and counted as wae_buffer_source_set_device_input (the same texts, the same
 * "cannot assign buffer twice" rule against set_buffer and either declaration), but the batch gives it no slab memory and its bind
 * copies no audio.  wae_batch_bind_sources records the item's `pcm` and `channel_stride` in every planned record that plays the node;
 * later runs read that memory.  The contract differs from a copy: after a copy bind the caller may free or overwrite the tensor at once,
 * after a reference bind it keeps the memory alive and unchanged for every run that reads it, until it binds other memory.  Writes to
 * it are ordered by the caller: a write queued on another stream before a run is read by the run only if the engine stream waits for
 * that stream, and a write after a run waits for the engine stream.  Several declarations may name the same memory; the memory must not
 * overlap the output the runs write.  wae_render_batch and wae_render_many refuse graphs with such inputs as they refuse device inputs. */
WAE_API wae_status wae_buffer_source_set_device_input_by_reference(wae_graph* graph, wae_node_id node, uint32_t number_of_channels,
                                                                   uint64_t length, float sample_rate);

typedef struct wae_source_binding {
    uint32_t graph_index;    /* caller's index, as wae_batch_fetch_graph (also for wae_batch_prepare_many batches) */
    wae_node_id node;        /* a node declared with wae_buffer_source_set_device_input */
    const float* pcm;        /* device memory on the engine's GPU, 4-byte aligned: channel c is `length` floats at
                                pcm + c * channel_stride */
    uint64_t channel_stride; /* floats, >= the declared length; channels need no 16-byte alignment */
} wae_source_binding;

/* Copies the audio into the batch's source slab, asynchronously on the engine stream, after the work already queued on `stream`
 * (a cudaStream_t of the engine's device, or cudaStreamLegacy for the legacy default stream, or cudaStreamPerThread; NULL = no extra
 * ordering: the engine stream is non-blocking and does NOT wait for the legacy default stream by itself).  All-or-nothing: every item
 * is validated before anything is enqueued.  Bound audio stays until it is bound again; runs never alter it.  A device input that is
 * never started renders silence and reads nothing: binding it is validated and copies nothing.  WAE_INVALID_ARGUMENT: `pcm` is null,
 * not 4-byte aligned or not device (or managed) memory of the engine's GPU, or the extent
 * [pcm, pcm + (channels - 1) * channel_stride + length) does not lie
 * inside one allocation, or channel_stride is below the declared length, or one (graph, node) is named twice in the call.
 * WAE_INVALID_STATE: graph_index out of range, or the node is not a device input.
 * An input declared with wae_buffer_source_set_device_input_by_reference is not copied: the bind writes `pcm` and `channel_stride` into
 * the batch's records (one small kernel on the engine stream, no host synchronisation), and runs read the caller's memory.  One call
 * may mix copied and referenced items.  A referenced extent that overlaps the batch's own output buffer or the output bound with
 * wae_batch_bind_output answers WAE_INVALID_ARGUMENT.
 * wae_batch_run, wae_batch_run_group and wae_batch_run_pipelined answer WAE_INVALID_STATE while a device input of the batch has never
 * been bound. */
WAE_API wae_status wae_batch_bind_sources(wae_batch* batch, const wae_source_binding* items, uint32_t n, void* stream);

/* ---- param values bound from device memory ----------------------------------------------------------------------------------
 * Declares a param whose value is supplied per run from device memory (wae_batch_bind_params) instead of at build time, so that one
 * prepared batch renders any number of parameter sets (EQ, gain, pan, compressor settings drawn on the GPU) without being built and
 * planned again.  The param renders as a constant for the whole render, as a param with only a value does.  param_index numbers the
 * params as wae_param_event_push does.  Bindable: GainNode gain; BiquadFilterNode q, detune, frequency, gain (0..3); StereoPannerNode
 * pan; DynamicsCompressorNode attack, knee, ratio, release, threshold (0..4); AudioBufferSourceNode detune, playbackRate (0, 1);
 * OscillatorNode frequency, detune (0, 1); PannerNode positionX/Y/Z, orientationX/Y/Z (0..5); the AudioListener's positionX/Y/Z,
 * forwardX/Y/Z, upX/Y/Z (0..8, addressed as node 1: declaring one creates the listener, as wae_connect_param does).  A
 * bound value is clamped to [max(lo, minValue), min(hi, maxValue)], as AudioParam::set_value clamps to [minValue, maxValue].  The range
 * decides what is planned, never the value: a GainNode whose range excludes |gain| <= 1e-6 can never answer with silence, so its output
 * keeps the layout of its input.  An AudioBufferSourceNode's two ranges give the computed rates rate * 2^(detune / 1200) it may play
 * at: a source that does not loop, whose other param is not automated and whose rates are all > 0 is rendered time-parallel (give
 * detune a range: the default one allows a rate of 0), its output has a constant layout only when the clip lasts to the end of the
 * render at the highest rate; any other source takes the serial renderer, which is right for every value but slow.  An
 * OscillatorNode keeps its fused path (k_chain, k_voice_sum) when every computed frequency frequency * 2^(detune / 1200) its ranges allow
 * (the other param's range, or its current value when it is not declared) lies in (0, sampleRate / 2); a range that allows any other
 * frequency answers WAE_UNSUPPORTED (bind such a pitch with wae_param_set_device_value_curve).  The rule is not needed while the other
 * param is automated or driven at audio rate.  The other param may change after the declaration, so wae_batch_prepare and wae_batch_plan
 * check the rule again and answer WAE_UNSUPPORTED, naming the graph and the node, when it no longer holds.  With a start time declared as
 * well (wae_source_set_device_schedule) the two binds may come in either order.  A PannerNode whose position, orientation or listener is
 * declared keeps the lowering of its placeholder (equal-power or HRTF, static or moving when another of its 15 spatial params is
 * automated).  Its range, and a listener param's, must lie inside [-1e9, 1e9], where the f32 spatial math (squared differences, the
 * cross product of forward and up) stays finite; a wider range, the default one included, answers WAE_UNSUPPORTED.  A static HRTF panner
 * lowered to a convolver gets response spectra of its own (2 x 24 x 8192 float2, 3 MiB), which every
 * wae_batch_bind_params rewrites.  A listener param reaches every panner of its graph; in a graph without a panner it is validated and
 * reaches nothing, and runs still wait for its bind.  Bound spatial math runs on the device (acosf, sinf / cosf, pow), which may round the
 * last bit differently from the host: near a face of the HRIR sphere the device may pick the neighbouring triangle.
 * Deviation: a non-finite bound value renders as the param's default value (the reference panics on a non-finite set_value, which a
 * device bind cannot do; this is its rule for a NaN computed value); an oscillator's frequency and detune take the default clamped to the
 * declared range.
 * WAE_INVALID_ARGUMENT: lo > hi, a non-finite bound, or a range outside [minValue, maxValue].  WAE_UNSUPPORTED: another node kind or
 * param, an oscillator pitch range that breaks the rule above, or a spatial range beyond [-1e9, 1e9].  WAE_INVALID_STATE: the param has automation events or an audio-rate input, is declared twice, or the graph already has a
 * suspend point; after the declaration, events (set_value included, also from a suspend callback) and wae_connect_param to it answer
 * WAE_INVALID_STATE.  wae_render_batch and wae_render_many answer WAE_INVALID_STATE on graphs with such params; wae_batch_plan plans
 * them with the param's current value clamped to the range. */
WAE_API wae_status wae_param_set_device_value(wae_graph* graph, wae_node_id node, uint32_t param_index, float lo, float hi);

typedef struct wae_param_binding {
    uint32_t graph_index;  /* caller's index, as wae_batch_fetch_graph */
    wae_node_id node;      /* the param's node */
    uint32_t param_index;  /* declared with wae_param_set_device_value */
    const float* value;    /* one float of device (or managed) memory on the engine's GPU, 4-byte aligned */
} wae_param_binding;

/* Reads the values on the device, asynchronously on the engine stream after the work already queued on `stream` (as
 * wae_batch_bind_sources), and re-derives every planned record they reach (filter coefficients and scan constants, gain products,
 * panner gains, compressor settings) in every render segment.  All-or-nothing: every item is validated before anything is enqueued.
 * Bound values stay until they are bound again.  WAE_INVALID_ARGUMENT: `value` is null, not 4-byte aligned, not device (or managed)
 * memory of the engine's GPU or its 4 bytes are not in one allocation, or one param is named twice in the call.  WAE_INVALID_STATE:
 * graph_index out of range, the param was not declared, or the batch has HRTF panners whose source or listener is bound and
 * wae_engine_set_hrir_sphere has replaced the sphere since the batch was prepared (nothing is enqueued: prepare the batch again).  The
 * spatial values re-derive each static panner's direction and gains, and for HRTF its triangle, weights and, for one lowered to a
 * convolver, its blended response and spectra.  wae_batch_run, wae_batch_run_group and wae_batch_run_pipelined answer WAE_INVALID_STATE while a declared
 * param of the batch has never been bound. */
WAE_API wae_status wae_batch_bind_params(wae_batch* batch, const wae_param_binding* items, uint32_t n, void* stream);

/* ---- ConvolverNode responses bound from device memory -----------------------------------------------------------------------
 * Declares a ConvolverNode whose impulse response is supplied per run from device memory (wae_batch_bind_responses) instead of an
 * AudioBuffer, so that one prepared batch convolves with any number of response sets (room impulse responses drawn or generated on the
 * GPU) without being built and planned again.  The declaration counts as the node's set_buffer: it fixes the normalisation (the
 * `normalize` attribute as it is now), with set_buffer's checks and texts (WAE_NOT_SUPPORTED: a channel count other than 1, 2 or 4, a
 * rate other than the context's; AudioBuffer::new's text for length 0).  The node is planned with ceil(length / 8192) partitions on
 * every channel, as an untrimmed response of that length would be; normalisation and the trimming of the quiet tail run on the device
 * in the bind, so a bound response renders exactly as an AudioBuffer of the same content given to set_buffer.
 * WAE_INVALID_STATE: the node already has a response, is declared twice, or the graph already has a suspend point; set_buffer after the
 * declaration answers WAE_INVALID_STATE.  Suspend points added later are allowed (every segment reads the one bound response).
 * wae_render_batch and wae_render_many answer WAE_INVALID_STATE on graphs with such nodes; wae_batch_plan plans them. */
WAE_API wae_status wae_convolver_set_device_response(wae_graph* graph, wae_node_id node, uint32_t number_of_channels,
                                                     uint64_t length, float sample_rate);

typedef struct wae_response_binding {
    uint32_t graph_index;    /* caller's index, as wae_batch_fetch_graph */
    wae_node_id node;        /* declared with wae_convolver_set_device_response */
    const float* pcm;        /* device memory of the engine's GPU, 4-byte aligned: channel c is `length` floats at
                                pcm + c * channel_stride */
    uint64_t channel_stride; /* floats, >= the declared length; channels need no 16-byte alignment */
} wae_response_binding;

/* Normalises, trims and transforms the responses on the device, asynchronously on the engine stream after the work already queued on
 * `stream` (as wae_batch_bind_sources).  All-or-nothing: every item is validated before anything is enqueued.  A bound response stays
 * until it is bound again.  WAE_INVALID_ARGUMENT: `pcm` is null, not 4-byte aligned or not device (or managed) memory of the engine's
 * GPU, the extent does not lie
 * in one allocation, channel_stride is below the declared length, one (graph, node) is named twice in the call, or the call has more
 * than 65535 items that the batch renders.  WAE_INVALID_STATE:
 * graph_index out of range, or the node was not declared.  wae_batch_run, wae_batch_run_group and wae_batch_run_pipelined answer
 * WAE_INVALID_STATE while a declared response of the batch has never been bound. */
WAE_API wae_status wae_batch_bind_responses(wae_batch* batch, const wae_response_binding* items, uint32_t n, void* stream);

/* ---- WaveShaperNode curves bound from device memory -------------------------------------------------------------------------
 * Declares a WaveShaperNode whose curve of `length` points is supplied per run from device memory (wae_batch_bind_curves) instead of
 * set_curve, so that one prepared batch shapes with any number of curve sets (saturation / distortion curves drawn on the GPU) without
 * being built and planned again.  The declaration counts as the node's set_curve; the oversample attribute stays settable.  Any length
 * >= 1 is accepted (WAE_INVALID_ARGUMENT: 0).  WAE_INVALID_STATE: the node already has a curve (options or set_curve), is declared
 * twice, or the graph already has a suspend point; set_curve after the declaration answers WAE_INVALID_STATE.  Suspend points added
 * later are allowed (every segment reads the one bound curve).  Whether the curve maps 0 to 0 (can_propagate_silence) is decided
 * per bind on the device; the plan covers both answers.  wae_render_batch and wae_render_many answer WAE_INVALID_STATE on graphs with
 * such nodes; wae_batch_plan plans them. */
WAE_API wae_status wae_wave_shaper_set_device_curve(wae_graph* graph, wae_node_id node, uint32_t length);

typedef struct wae_curve_binding {
    uint32_t graph_index;   /* caller's index, as wae_batch_fetch_graph */
    wae_node_id node;       /* declared with wae_wave_shaper_set_device_curve */
    const float* curve;     /* device memory of the engine's GPU: `length` floats, 4-byte aligned */
} wae_curve_binding;

/* Copies the curves into the batch, asynchronously on the engine stream after the work already queued on `stream` (as
 * wae_batch_bind_sources).  The values are used bit for bit, NaN and infinities included.  All-or-nothing: every item is validated before
 * anything is enqueued.  A bound curve stays until it is bound again.  WAE_INVALID_ARGUMENT: `curve` is null, not 4-byte aligned or
 * not device (or managed)
 * memory of the engine's GPU, [curve, curve + length) does not lie in one allocation, or one (graph, node) is named twice in the call.
 * WAE_INVALID_STATE: graph_index out of range, or the node was not declared.  wae_batch_run, wae_batch_run_group and
 * wae_batch_run_pipelined answer WAE_INVALID_STATE while a declared curve of the batch has never been bound. */
WAE_API wae_status wae_batch_bind_curves(wae_batch* batch, const wae_curve_binding* items, uint32_t n, void* stream);

/* ---- OscillatorNode periodic waves bound from device memory -----------------------------------------------------------------
 * Declares an OscillatorNode whose PeriodicWave of `coefficients` (real, imag) pairs is supplied per run from device memory
 * (wae_batch_bind_periodic_waves) instead of set_periodic_wave, so that one prepared batch plays any number of timbres (harmonic
 * amplitudes predicted by a network, randomised wavetables) without being built and planned again.  The bind synthesises the wavetable
 * of `table_len` points on the device as wae_periodic_wave_table does (normalised unless `disable_normalization`).  The declaration
 * counts as the node's set_periodic_wave: the type becomes Custom for good, and an earlier host wave is replaced.
 * WAE_INVALID_ARGUMENT: not an oscillator, `coefficients` < 2 or `table_len` 0.  WAE_INVALID_STATE: the node is declared twice, or the
 * graph already has a suspend point; set_periodic_wave after the declaration answers WAE_INVALID_STATE.  Suspend points added later are
 * allowed (every segment reads the one bound table).  wae_render_batch and wae_render_many answer WAE_INVALID_STATE on graphs with such
 * nodes; wae_batch_plan plans them. */
WAE_API wae_status wae_oscillator_set_device_periodic_wave(wae_graph* graph, wae_node_id node, uint32_t coefficients, uint32_t table_len,
                                                           uint32_t disable_normalization);

typedef struct wae_periodic_wave_binding {
    uint32_t graph_index;   /* caller's index, as wae_batch_fetch_graph */
    wae_node_id node;       /* declared with wae_oscillator_set_device_periodic_wave */
    const float* real;      /* device memory of the engine's GPU: `coefficients` floats, 4-byte aligned, or NULL (= zeros) */
    const float* imag;      /* likewise; not both NULL */
} wae_periodic_wave_binding;

/* Synthesises the wavetables into the batch, asynchronously on the engine stream after the work already queued on `stream` (as
 * wae_batch_bind_sources).  real[0] and imag[0] (DC) are ignored, as PeriodicWave ignores them.  All-or-nothing: every item is validated
 * before anything is enqueued.  A bound wave stays until it is bound again.  WAE_INVALID_ARGUMENT: `real` and `imag` are both null, one
 * of them is not 4-byte aligned, not device (or managed) memory of the engine's GPU or does not hold `coefficients` floats in one
 * allocation, or one
 * (graph, node) is named twice in the call.  WAE_INVALID_STATE: graph_index out of range, or the node was not declared.  wae_batch_run,
 * wae_batch_run_group and wae_batch_run_pipelined answer WAE_INVALID_STATE while a declared wave of the batch has never been bound. */
WAE_API wae_status wae_batch_bind_periodic_waves(wae_batch* batch, const wae_periodic_wave_binding* items, uint32_t n, void* stream);

/* ---- IIRFilterNode coefficients bound from device memory --------------------------------------------------------------------
 * The IIRFilterNode's coefficients are supplied per run from device memory (wae_batch_bind_iir_coefficients) instead of its options, so
 * that one prepared batch filters with any number of coefficient sets (an EQ a network predicts, random filters for augmentation) without
 * being built and planned again.  The counts are the node's own (as constructed); the constructed coefficients are what wae_batch_plan
 * plans with (the lowering depends on the counts only, so the plan is that of the constructed node).  WAE_INVALID_ARGUMENT: not an
 * IIRFilterNode.  WAE_INVALID_STATE: the node is declared twice, or the graph already has a suspend point.  Suspend points added later
 * are allowed (every segment reads the one bound set).  wae_render_batch and wae_render_many answer WAE_INVALID_STATE on graphs with
 * such nodes; wae_batch_plan plans them. */
WAE_API wae_status wae_iir_filter_set_device_coefficients(wae_graph* graph, wae_node_id node);

typedef struct wae_iir_binding {
    uint32_t graph_index;      /* caller's index, as wae_batch_fetch_graph */
    wae_node_id node;          /* declared with wae_iir_filter_set_device_coefficients */
    const double* feedforward; /* device memory of the engine's GPU: the node's feedforward count of doubles, any 8 B alignment */
    const double* feedback;    /* likewise, the node's feedback count */
} wae_iir_binding;

/* Writes the coefficients into the batch, asynchronously on the engine stream after the work already queued on `stream` (as
 * wae_batch_bind_sources).  They are normalised by feedback[0] in f64 as the constructor's coefficients are, so bound coefficients render
 * bit for bit what a node constructed with them renders; NaN and infinities are used as they are.  Deviation: the reference refuses
 * feedback[0] == 0 at construction; such an item writes all-zero coefficients, and the filter outputs zeros.  All-or-nothing: every
 * item is validated before anything is enqueued.  A bound set stays until it is bound again.  WAE_INVALID_ARGUMENT: a null pointer, one
 * that is not 8-byte aligned or not device (or managed) memory of the engine's GPU, an extent that does not lie in one allocation, or
 * one (graph, node) named twice in the call.  WAE_INVALID_STATE: graph_index out of range, or the node was not declared.  wae_batch_run,
 * wae_batch_run_group and wae_batch_run_pipelined answer WAE_INVALID_STATE while a declared IIR filter of the batch has never been
 * bound. */
WAE_API wae_status wae_batch_bind_iir_coefficients(wae_batch* batch, const wae_iir_binding* items, uint32_t n, void* stream);

/* ---- AudioParam value curves bound from device memory -----------------------------------------------------------------------
 * Declares one SetValueCurveAtTime event of `length` values at [start_time, start_time + duration) whose values are supplied per run
 * from device memory (wae_batch_bind_value_curves), so that one prepared batch renders any number of envelopes, filter sweeps, pitch
 * contours, pan trajectories or delay-time modulations without being built and planned again.  It works on every param
 * wae_param_event_push accepts, including the ones wae_param_set_device_value refuses (OscillatorNode frequency / detune, DelayNode
 * delayTime, PannerNode positions, ConstantSourceNode offset): no planning decision reads the values of an automated param.  The event is
 * pushed in arrival order exactly as wae_param_event_push pushes a host curve, so folding, sorting, cancel handling and overlap errors
 * (WAE_NOT_SUPPORTED at plan time) are the host's, and a bound curve renders bit for bit what the same values given to
 * wae_param_event_push render.  The values are used as they are, NaN and infinities included (the reference checks only the length,
 * start time and duration).  An audio-rate input (wae_connect_param) stays allowed.
 * WAE_INVALID_ARGUMENT: an unknown node or param (AudioListener params included), an invalid start time, a duration that is not > 0.
 * WAE_INVALID_STATE: length < 2, a param bound with wae_param_set_device_value, a second declaration on the param, or a graph that
 * already has a suspend point.  After the declaration the param takes no further events (also from a suspend callback: WAE_INVALID_STATE);
 * suspend points added later are allowed.  wae_render_batch and wae_render_many answer WAE_INVALID_STATE on graphs with declarations;
 * wae_batch_plan plans them. */
WAE_API wae_status wae_param_set_device_value_curve(wae_graph* graph, wae_node_id node, uint32_t param_index, uint32_t length,
                                                    double start_time, double duration);

typedef struct wae_value_curve_binding {
    uint32_t graph_index;  /* caller's index, as wae_batch_fetch_graph */
    wae_node_id node;      /* the param's node */
    uint32_t param_index;  /* declared with wae_param_set_device_value_curve */
    const float* values;   /* device memory of the engine's GPU: the declared `length` floats, 4-byte aligned */
} wae_value_curve_binding;

/* Copies the values into the batch, asynchronously on the engine stream after the work already queued on `stream` (as
 * wae_batch_bind_sources).  All-or-nothing: every item is validated before anything is enqueued.  A bound curve stays until it is bound
 * again.  WAE_INVALID_ARGUMENT: `values` is null, not 4-byte aligned or not device (or managed) memory of the engine's GPU,
 * [values, values + length) does not lie in one allocation, or one param is named twice in the call.  WAE_INVALID_STATE: graph_index
 * out of range, or the param has no declaration.  wae_batch_run, wae_batch_run_group and wae_batch_run_pipelined answer
 * WAE_INVALID_STATE while a declared curve of the batch has never been bound (a declared param the batch never renders needs no bind). */
WAE_API wae_status wae_batch_bind_value_curves(wae_batch* batch, const wae_value_curve_binding* items, uint32_t n, void* stream);

/* ---- Start and stop times of scheduled sources bound from device memory -------------------------------------------------------------
 * Declares that the start time of a started AudioBufferSourceNode, OscillatorNode or ConstantSourceNode (and, with `bind_stop`, its stop
 * time) is supplied per run from device memory (wae_batch_bind_schedules), so that one prepared batch renders any number of event
 * onsets, note sequences or onset jitters without being built and planned again.  The `when` given to wae_source_start becomes a
 * placeholder (as does the stop time with `bind_stop`); an AudioBufferSourceNode's offset and duration stay the ones given to
 * wae_source_start unless wae_buffer_source_set_device_offset declares them too.  A bound time is clamped to its window [lo, hi] (a NaN becomes lo); the reference panics on a negative or non-finite
 * `when`, which a bind on the device cannot do.  The source is always planned with a gated output layout, and its path never depends on
 * the bound times: a non-looping AudioBufferSourceNode whose computed playback rates are all > 0 and not automated takes the bound slow
 * track (k_buffer_source_slow(bound), which plays a rate of 1 from an aligned start 1:1), a looping one the path of its loop declaration
 * (wae_buffer_source_set_device_loop), every other one the serial kernel.  A declared
 * source is never fused into k_chain.
 * WAE_INVALID_ARGUMENT: not a scheduled source node, a window that is not finite with 0 <= lo <= hi.  WAE_INVALID_STATE: a source that
 * has not been started, a second declaration, or a graph with a suspend point.  After the declaration, wae_source_start / wae_source_stop
 * on the node and wae_graph_suspend on the graph answer WAE_INVALID_STATE.  wae_render_batch and wae_render_many answer
 * WAE_INVALID_STATE on graphs with declarations; wae_batch_plan plans them. */
WAE_API wae_status wae_source_set_device_schedule(wae_graph* graph, wae_node_id node, double start_lo, double start_hi, int32_t bind_stop,
                                                  double stop_lo, double stop_hi);

/* Extends the schedule declaration of an AudioBufferSourceNode with the `offset` of start_at_with_offset_and_duration (and, with
 * `bind_duration`, its `duration`), supplied per run by wae_batch_bind_schedules, so that one prepared batch plays any excerpt of a long
 * clip.  A caller who only wants a per-run offset declares the start window [when, when].  The offset (and duration) given to
 * wae_source_start become placeholders: the windows' low ends, and the plan is the one of a source started with them.  A bound value is
 * clamped to its window (a NaN becomes lo); the reference panics on a negative or non-finite offset or duration.  The playback path is the
 * declared schedule's (see above); an offset of 0 from an aligned start still plays 1:1 at a rate of 1, a declared duration never does.
 * WAE_INVALID_ARGUMENT: not an AudioBufferSourceNode, a window that is not finite with 0 <= lo <= hi.  WAE_INVALID_STATE: the node's
 * schedule has not been declared with wae_source_set_device_schedule, or a second declaration. */
WAE_API wae_status wae_buffer_source_set_device_offset(wae_graph* graph, wae_node_id node, double offset_lo, double offset_hi,
                                                       int32_t bind_duration, double duration_lo, double duration_hi);

typedef struct wae_schedule_binding {
    uint32_t graph_index;  /* caller's index, as wae_batch_fetch_graph */
    wae_node_id node;      /* declared with wae_source_set_device_schedule */
    const double* times;   /* device memory of the engine's GPU, 8-byte aligned: the row start, [stop], [offset], [duration], holding
                              only what was declared (bind_stop; wae_buffer_source_set_device_offset, bind_duration) */
} wae_schedule_binding;

/* Writes the times into the batch, asynchronously on the engine stream after the work already queued on `stream` (as
 * wae_batch_bind_sources).  All-or-nothing: every item is validated before anything is enqueued.  A bound schedule stays until it is
 * bound again.  WAE_INVALID_ARGUMENT: `times` is null, not 8-byte aligned or not device (or managed) memory of the engine's GPU, the
 * declared row does not lie in one allocation, or one node is named twice in the call.  WAE_INVALID_STATE: graph_index out of range, or
 * the node has no declaration.  wae_batch_run, wae_batch_run_group and wae_batch_run_pipelined answer WAE_INVALID_STATE while a declared
 * schedule of the batch has never been bound (a declared source the batch never renders needs no bind). */
WAE_API wae_status wae_batch_bind_schedules(wae_batch* batch, const wae_schedule_binding* items, uint32_t n, void* stream);

/* ---- Loop points of AudioBufferSourceNodes bound from device memory ----------------------------------------------------------------
 * Declares that the loopStart and loopEnd of a looping AudioBufferSourceNode are supplied per run from device memory
 * (wae_batch_bind_loops), so that one prepared batch loops any region of its clip without being built and planned again.  Both are
 * declared together: a caller who wants only one pins the other with a window [v, v].  The current loop_start / loop_end become
 * placeholders, the windows' low ends: the plan is the one of a source built with them.  A bound value is clamped to its window (a NaN
 * becomes lo); the reference stores any f64.  The reference's clamp_loop_boundaries and actual-loop-point rules then apply on the device.
 * The playback path is decided from the windows and the declared rates, never from the bound values: a source whose computed playback
 * rates are all > 0 and not automated, whose shortest possible loop is longer than four output frames at the top rate, and whose
 * playhead table fits 65536 segments, takes the bound slow track (k_buffer_source_slow(bound)), whose table is derived on the device
 * after each bind; every other one the serial kernel.  A looping source with a bound playbackRate / detune or a bound schedule but no
 * loop declaration stays on the serial kernel: to put it on the bound slow track, declare its loop with one-point windows [ls, ls],
 * [le, le].
 * WAE_INVALID_ARGUMENT: not an AudioBufferSourceNode, a window that is not finite with 0 <= lo <= hi.  WAE_INVALID_STATE: the node's
 * `loop` is false, a second declaration, or a graph with a suspend point.  After the declaration, wae_node_set_attribute with
 * WAE_ATTR_LOOP / _LOOP_START / _LOOP_END on the node and wae_graph_suspend on the graph answer WAE_INVALID_STATE.  wae_render_batch and
 * wae_render_many answer WAE_INVALID_STATE on graphs with declarations; wae_batch_plan plans them. */
WAE_API wae_status wae_buffer_source_set_device_loop(wae_graph* graph, wae_node_id node, double start_lo, double start_hi, double end_lo,
                                                     double end_hi);

typedef struct wae_loop_binding {
    uint32_t graph_index;  /* caller's index, as wae_batch_fetch_graph */
    wae_node_id node;      /* declared with wae_buffer_source_set_device_loop */
    const double* points;  /* device memory of the engine's GPU, 8-byte aligned: the row loop_start, loop_end */
} wae_loop_binding;

/* Writes the loop points into the batch, asynchronously on the engine stream after the work already queued on `stream` (as
 * wae_batch_bind_sources).  All-or-nothing: every item is validated before anything is enqueued.  Bound loop points stay until they are
 * bound again.  WAE_INVALID_ARGUMENT: `points` is null, not 8-byte aligned or not device (or managed) memory of the engine's GPU, the row
 * does not lie in one allocation, or one node is named twice in the call.  WAE_INVALID_STATE: graph_index out of range, or the node has
 * no declaration.  wae_batch_run, wae_batch_run_group and wae_batch_run_pipelined answer WAE_INVALID_STATE while declared loop points of
 * the batch have never been bound (a declared source the batch never renders needs no bind).  wae_batch_sync answers WAE_CUDA_ERROR if a
 * playhead table derived on the device ever needed more segments than were planned for it (a defect: the render is wrong). */
WAE_API wae_status wae_batch_bind_loops(wae_batch* batch, const wae_loop_binding* items, uint32_t n, void* stream);

/* ---- Rendered PCM written to caller device memory ---------------------------------------------------------------------------------
 * Points the rendered PCM of later runs at caller device memory instead of the batch's own buffer.  `out` takes the layout of that buffer:
 * packed, graph j at the offset wae_batch_graph_output reports, [channels_j][length_j] f32; `floats` must be the out_floats of
 * wae_batch_output_device_ptr.  The call is ordered after the work already queued on `stream` (as wae_batch_bind_sources) and rewrites the
 * batch's output pointers on the engine stream; later wae_batch_run / wae_batch_run_group write `out`, every float of it (a graph whose
 * destination has no input, or whose destination is muted in a cycle, renders zeros there, as in the batch's own buffer).  A null `out`
 * with floats == 0 returns the batch to its own buffer, which a run into `out` leaves untouched.  The binding stays until it is changed.
 * Runs are asynchronous on the engine stream (wae_engine_stream) and never wait for another stream by themselves, as for the batch's own
 * buffer: a reader of `out` on another stream waits for the engine stream after the run, and a run into memory whose last render is still
 * being read is ordered after that reader by the caller (binding again orders it after `stream`).  While it holds,
 * wae_batch_output_device_ptr reports `out` and wae_batch_fetch / wae_batch_fetch_graph read it.  WAE_INVALID_ARGUMENT, with nothing
 * changed: `out` is not 256-byte aligned (as cudaMalloc aligns the batch's own buffer; a torch allocation is, and so is a slice of it at
 * a multiple of 64 floats), not device (or managed) memory of the engine's GPU or [out, out + floats) does not lie in one allocation,
 * `floats` is not the batch's out_floats, a null `out` comes with floats != 0, or [out, out + floats) overlaps the memory a device input
 * declared by reference is bound to.  WAE_INVALID_STATE: a graph of the batch connects its
 * destination to another node (that node reads the batch's own buffer).  wae_batch_run_pipelined, which streams the batch's own buffer
 * to host memory, answers WAE_INVALID_STATE while an output is bound.  wae_render_batch and wae_render_many are not affected. */
WAE_API wae_status wae_batch_bind_output(wae_batch* batch, float* out, uint64_t floats, void* stream);

/* PeriodicWave::new(context, PeriodicWaveOptions { real, imag, disable_normalization }) (src/periodic_wave.rs:104-209): fills `table`
 * (PERIODIC_WAVE_TABLE_LENGTH = 8192 in the reference) with the wavetable an OscillatorNode of type Custom plays.  `real` / `imag` may be
 * NULL (= zeros); both NULL = the sine default.  Host math, no engine needed. */
WAE_API wae_status wae_periodic_wave_table(const float* real, const float* imag, uint32_t len, uint32_t disable_normalization, float* table,
                                           uint32_t table_len);

/* Test hook: the scheduling clock start / stop times are lowered with.  The reference's renderers compare a start time with a time that is
 * `frame / sample_rate` at the head of a quantum and then grows by `+= dt` per frame (oscillator.rs:511-557, constant_source.rs:231-246,
 * audio_buffer_source.rs): the first frame at or after `time` under that clock, and its accumulated time. */
WAE_API wae_status wae_sched_first_frame_at_or_after(float sample_rate, double time, int64_t* frame, double* frame_time);

/* Test hook: the spatial math of PannerNode as the planner and the moving-source kernels evaluate it (csrc/wae_spatial.h; panner.rs:927-986,
 * spatial.rs:205-299).  v15 = source position, source orientation, listener position, forward, up; model6 = refDistance, maxDistance,
 * rolloffFactor, coneInnerAngle, coneOuterAngle, coneOuterGain; out4 = distance gain, cone gain, azimuth, elevation (degrees). */
WAE_API wae_status wae_spatial_params(uint32_t distance_model, const double* model6, const float* v15, float* out4);

/* Test hook: the HRIR-sphere lookup of HRTF panning (the hrtf crate's ray / triangle query + barycentric weights): 1 when `dir` crosses a
 * face; idx = its 3 vertices, weights = the blend weights of their impulse responses.  pos: [vertex][3], faces: 3 indices per face. */
WAE_API int32_t wae_hrtf_locate(const float* pos, const uint32_t* faces, uint32_t n_faces, const float* dir, uint32_t* idx, float* weights);

/* ---- attributes set after construction (the reference posts one control message per setter) --------------------------------
 * AudioBufferSourceNode::set_buffer (once; src/node/audio_buffer_source.rs:278-288), ConvolverNode::set_buffer (convolver.rs:259-317; the
 * normalisation is decided at this call from the current `normalize` attribute), WaveShaperNode::set_curve (once; waveshaper.rs:203-213),
 * OscillatorNode::set_periodic_wave (oscillator.rs:334-337; `table` = the wavetable of PeriodicWave::new, the type becomes Custom). */
WAE_API wae_status wae_buffer_source_set_buffer(wae_graph* graph, wae_node_id node, const wae_audio_buffer* buffer);
WAE_API wae_status wae_convolver_set_buffer(wae_graph* graph, wae_node_id node, const wae_audio_buffer* buffer);
WAE_API wae_status wae_wave_shaper_set_curve(wae_graph* graph, wae_node_id node, const float* curve, uint32_t len);
WAE_API wae_status wae_oscillator_set_periodic_wave(wae_graph* graph, wae_node_id node, const float* table, uint32_t len);
/* the scalar setters: AudioBufferSourceNode::set_loop / set_loop_start / set_loop_end (audio_buffer_source.rs:324-349),
 * ConvolverNode::set_normalize (convolver.rs:325-328), WaveShaperNode::set_oversample (waveshaper.rs:226-229), PannerNode::set_*
 * (panner.rs:545-657), AnalyserNode::set_* (analyser.rs:148-222).  Enumerated values (models, oversample) are passed as their enum
 * value, booleans as 0 / 1.  Range errors answer the reference's panic text.  Called after wae_graph_suspend the change applies from
 * that point on; two changes at a suspend point are answered WAE_UNSUPPORTED (the graph keeps the CPU renderer): the loop attributes of
 * a source that was already started, and a second impulse response for a ConvolverNode. */
enum {
    WAE_ATTR_LOOP = 1, WAE_ATTR_LOOP_START = 2, WAE_ATTR_LOOP_END = 3,
    WAE_ATTR_NORMALIZE = 4,
    WAE_ATTR_OVERSAMPLE = 5,
    WAE_ATTR_PANNING_MODEL = 6, WAE_ATTR_DISTANCE_MODEL = 7, WAE_ATTR_REF_DISTANCE = 8, WAE_ATTR_MAX_DISTANCE = 9,
    WAE_ATTR_ROLLOFF_FACTOR = 10, WAE_ATTR_CONE_INNER_ANGLE = 11, WAE_ATTR_CONE_OUTER_ANGLE = 12, WAE_ATTR_CONE_OUTER_GAIN = 13,
    WAE_ATTR_FFT_SIZE = 14, WAE_ATTR_SMOOTHING_TIME_CONSTANT = 15, WAE_ATTR_MIN_DECIBELS = 16, WAE_ATTR_MAX_DECIBELS = 17
};
WAE_API wae_status wae_node_set_attribute(wae_graph* graph, wae_node_id node, uint32_t attribute, double value);

/* AudioNode::set_channel_count / set_channel_count_mode / set_channel_interpretation (src/node/audio_node.rs:417-441), with the
 * constraints of the nodes that narrow them (destination.rs:55-96, channel_merger.rs:39-110, channel_splitter.rs:36-134, convolver.rs:187-197,
 * dynamics_compressor.rs:168-178, stereo_panner.rs:143-152, panner.rs:363-372, param.rs:325-333, spatial.rs:113-121): a value the reference
 * panics on answers WAE_NOT_SUPPORTED with the panic text.  `node` is the id create_* returned; 0 addresses the destination.  Called
 * between wae_graph_suspend points the change applies from that point on, like the reference's control message. */
WAE_API wae_status wae_node_set_channel_count(wae_graph* graph, wae_node_id node, uint32_t count);
WAE_API wae_status wae_node_set_channel_count_mode(wae_graph* graph, wae_node_id node, uint32_t count_mode);
WAE_API wae_status wae_node_set_channel_interpretation(wae_graph* graph, wae_node_id node, uint32_t interpretation);

/* HrirSphere::new(reader, context_rate) of the hrtf crate (src/node/panner.rs:39-68 is the call site): when the context rate differs from
 * the sphere's, every impulse response is resampled once with an asynchronous windowed-sinc resampler (ratio = context_rate / sphere_rate).
 * The engine does this to the whole sphere on first use of a rate; this entry point applies it to one response (host work, for tests). */
WAE_API wae_status wae_hrir_resample(const float* hrir, uint32_t len, double ratio, float* out, uint32_t cap, uint32_t* out_len);

/* Control-side read-outs of the filter nodes; host math only, no engine needed.
 * wae_biquad_frequency_response = BiquadFilterNode::get_frequency_response (src/node/biquad_filter.rs:657-735): the node's type and the
 * current value of its frequency / detune / q / gain params; frequencies outside [0, sample_rate / 2] answer NaN.
 * wae_iir_frequency_response = IIRFilterNode::get_frequency_response (src/node/iir_filter.rs:215-265).
 * wae_biquad_coefs = calculate_coefs (src/node/biquad_filter.rs:42-390): {b0, b1, b2, a1, a2} normalised by a0, as the kernels use them. */
WAE_API void wae_biquad_coefs(uint32_t type, double sample_rate, double computed_frequency, double gain, double q, double* out5);
WAE_API void wae_biquad_frequency_response(uint32_t type, float sample_rate, float frequency, float detune, float q, float gain,
                                           const float* frequency_hz, float* mag_response, float* phase_response, uint32_t n);
WAE_API void wae_iir_frequency_response(const double* feedforward, uint32_t n_feedforward, const double* feedback, uint32_t n_feedback,
                                        float sample_rate, const float* frequency_hz, float* mag_response, float* phase_response, uint32_t n);

#ifdef __cplusplus
}
#endif
#endif /* WAE_H */
