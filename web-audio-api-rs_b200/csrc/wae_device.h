// Device-visible POD descriptors shared by the planner (wae_plan.cpp) and the kernels (wae_kernels.cu).
//
// Execution model: a batch of G independent graphs is lowered to STAGES.  A stage is one kernel launch over
// all node instances of one kind at one topological level, for ONE time chunk [f0, f0+nf) of the render.
// Edge buffers live in a per-chunk arena (planar [ch][chunk_frames] f32, reused every chunk so they stay
// L2-resident); node state that crosses chunks (filter state, delay/compressor/analyser rings, convolver
// spectra) lives in persistent device memory.
#pragma once
#include <cstdint>
#include <vector_types.h>

#include "wae_spatial.h"

namespace wae {

// Dynamic layout (src/render/quantum.rs:109-111,179-260): in the reference a node output is a quantum of 1..32 channels whose count
// can change from one render quantum to the next, and "silent" is a property of the quantum (one shared zero buffer), which
// processors branch on.  A buffer whose layout the planner cannot prove constant carries a per-quantum META track:
//   meta[row * meta_stride + qi], rows = the buffer's static (maximum) channel count, qi = quantum index inside the chunk's arena;
//   low 6 bits = channels of that quantum (row 0 is authoritative), bit 7 = "this row's channel is silent";
//   the quantum is silent <=> every row has bit 7 (rows let per-channel CTAs / threads report their own filter tail).
// PCM of channels >= count, and of silent quanta, is unspecified: consumers of a buffer with a meta track read only what the
// track says exists.  meta == nullptr: the layout is constant (count = static channels, never silent) and nothing is looked up.
struct BufRef {
    float* p;           // channel 0, frame 0 of the chunk (arena) or of the whole render (absolute)
    uint32_t stride;    // floats between channels
    uint32_t absolute;  // 1: index with f0 + n (final output / assets), 0: index with n (arena)
    uint8_t* meta;      // per-quantum layout track or nullptr (constant layout)
    uint32_t meta_stride;
    uint32_t meta_pad;
};
constexpr uint8_t WAE_META_SILENT = 0x80;

struct ChunkInfo {
    int64_t f0;  // first frame of this chunk
    int32_t nf;  // frames in this chunk (multiple of 128 except nothing: render is padded to whole quanta)
    int32_t sub;  // offset of these frames inside the chunk's arena buffers: 0 for a whole chunk, q * 128 when the stages of
                  // a DelayNode feedback cycle are replayed quantum by quantum inside a chunk (f0 then includes it)
};

struct OscInst {
    BufRef out;
    int32_t type;             // WAE_OSC_*
    int32_t outside_nyquist;  // |computed_freq| >= nyquist -> zeros (oscillator.rs:542-555)
    double incr;              // phase increment per frame = computedFrequency / sampleRate
    double phase0;            // phase at frame n_first
    int64_t n_first, n_stop;  // active frames [n_first, n_stop)
    const float* table;       // sine table (2048) or periodic wave
    int32_t table_len;
    int32_t fast;             // (host) 0 < incr < 1/2, inside Nyquist, table of 2048 entries or no table: the fixed-point phase paths of k_chain apply
    double inv_incr;          // 1 / incr (polyBLEP of constant-frequency oscillators)
};

struct ConstInst {
    BufRef out;
    float value;
    int32_t pad;
    int64_t n_first, n_stop;
    BufRef track;  // p != nullptr: automated offset
};

struct AbsnInst {
    BufRef out;
    const float* buf;  // planar [ch][buf_len]
    int64_t buf_len;     // frames per channel
    int64_t buf_stride;  // floats between channels (>= buf_len, multiple of 4)
    int64_t n_start, n_stop;  // output frames [n_start, n_stop) play buf[n - n_start + buf_offset] (fast track)
    int64_t buf_offset;
    int32_t ch;
    int32_t loop;  // 1: wrap modulo buf_len (default loop points)
};

// AudioBufferSourceRenderer slow track (audio_buffer_source.rs:625-823): fractional playhead, offset / duration / stop,
// custom loop points, buffer sample rate != context sample rate; constant positive playback rate
struct AbsnSlowInst {
    BufRef out;
    const float* buf;
    int64_t buf_len, buf_stride;
    int64_t n_first, n_stop;     // frames [n_first, n_stop) may play
    double offset0;              // buffer time (s) at n_first
    double step;                 // dt * computed_playback_rate
    double elapsed0, duration;   // buffer_time_elapsed at n_first / explicit duration (f64::MAX: none)
    double buffer_duration;
    double pos_scale;            // sampling_ratio * sample_rate: playhead (frames) = buffer_time * pos_scale
    double loop_start, loop_end; // actual loop points (s)
    double sample_rate;
    int32_t ch;
    int32_t loop;
    // playhead segments: buffer_time(n) = seg_bt[k] + (n - seg_n[k]) * step for seg_n[k] <= n < seg_n[k+1]; a new
    // segment starts wherever the reference modifies buffer_time (loop wrap, sticky snap to a loop point)
    const int64_t* seg_n;
    const double* seg_bt;
    int32_t n_seg;
    int32_t pad;
};

// A non-looping slow-track source whose playbackRate / detune are bound from device memory (wae_param_set_device_value) over a range of
// positive computed rates (k_buffer_source_slow<true>).  The record holds what does not depend on the rate; each run derives the rest
// from `rate` and `detune` (patched by wae_batch_bind_params) with absn_slow_derive, the planner's own expressions.
struct AbsnBoundInst {
    AbsnSlowInst s;        // step, offset0, elapsed0 are derived per run; the segment table too (one segment) unless s.loop, whose
                           // table k_absn_loop_schedule derives after each bind that reaches it (loop points bound from device memory)
    double dt;             // the planner clock's frame duration
    double offset;         // start(when, offset): the requested offset
    double start_delta;    // t_first - start: the first playing frame's time after the start time
    int64_t n_start;       // fast track: output frames [n_start, fast_end) play buf[n - n_start]
    int64_t fast_end;
    int32_t fast_ok;       // aligned start, sampling ratio 1, default loop points, no stop / duration: a computed rate of 1 is the fast track
    float rate, detune;    // the bound (or planned constant) param values
    int32_t pad;
};

// AudioBufferSourceRenderer::process restated frame by frame (audio_buffer_source.rs:422-845) for everything the two
// closed-form tracks do not cover: automated playbackRate / detune (k-rate), zero / negative rates, very short loops.
// One warp per instance: lane 0 walks the renderer's state machine of a quantum, all lanes interpolate.
struct AbsnSerialState {
    double start_time, offset, buffer_time, buffer_time_elapsed;
    int32_t started, entered_loop, ended, is_aligned;
    int32_t inited, pad;  // 0 after the per-run memset
};
struct AbsnSerialInst {
    BufRef out;
    const float* buf;
    int64_t buf_len, buf_stride;
    double start_time, stop_time, offset, duration;  // start(when, offset, duration) / stop(when)
    double loop_start, loop_end;                     // after clamp_loop_boundaries (:400-417)
    double buffer_duration, buffer_sample_rate, sample_rate;
    BufRef rate_track, detune_track;                 // p != nullptr: automated (first value of every quantum)
    float rate, detune;
    int32_t ch, loop;
    AbsnSerialState* state;
};

struct BiquadInst {
    BufRef in, out;
    double b0, b1, b2, a1, a2;
    double* state;  // [ch][4] = x1, x2, y1, y2 (biquad_filter.rs:761)
    int32_t ch;
    int32_t pad;
    int32_t* dyn_len;  // [ch] (dynamic input layout only): `xy.len()`, the channel count of the last non-silent input quantum
};

struct IirInst {
    BufRef in, out;
    double b[20], a[20];  // normalised by a0 (iir_filter.rs:301-309)
    double* state;        // [ch][20]
    int32_t n;            // number of coefficients
    int32_t ch;
    int32_t* dyn_len;     // [ch] (dynamic input layout only): `states.len()` of the reference
};

struct GainInst {
    BufRef in, out;
    float gain;
    int32_t ch;
    BufRef gain_track;  // p != nullptr: a-rate / automated gain, one value per frame (k_param output)
};

struct ShaperInst {
    BufRef in, out;
    const float* curve;  // nullptr: pass-through
    int32_t n;
    int32_t ch;
};

// over-sampled WaveShaper (waveshaper.rs:409-480): 128 -> 128 * factor frames up (FFT resampler), curve, back down
struct ShaperOsInst {
    BufRef in, out;
    const float* curve;
    const float2* f_up;  // [128] filter bins of the up-sampler
    const float2* f_dn;  // [128] filter bins of the down-sampler
    float* hist;         // [ch][256] the two input quanta before the chunk
    // dynamic input layout, curve that maps 0 to 0: the reference returns early on a silent input WITHOUT feeding its resamplers
    // (waveshaper.rs:395-398), so their state is the last PROCESSED quanta, however long ago.  prev[2 q], prev[2 q + 1] = chunk index of
    // the two processed quanta before quantum q (-1 / -2: the history slots), prev[2 nq], prev[2 nq + 1]: the same after the chunk.
    int32_t* prev;
    int32_t n;           // curve length
    int32_t ch;
    int32_t factor;      // 2 or 4
    // != 0: the input changes its channel count.  Before a processed quantum whose count differs from the one the resamplers were built
    // for (initially 1) both are rebuilt with zero state (waveshaper.rs:409-420,527-531): history older than the last rebuild reads as
    // zero, and the down-sampler's overlap (the dn_{q-1} term) is zero at the rebuild quantum itself.  1: the curve does not map 0 to 0,
    // every quantum is processed (a silent one as ONE zero channel); 2: it does, silent quanta are not processed (waveshaper.rs:395-398).
    // prev then holds [0] the count the resamplers were built for (0: not yet, i.e. 1), [1] processed quanta since the last rebuild
    // (capped at 2) — both carried across chunks — followed by the table above and, at 2 nq + 2 + q, OS_INFO words of quantum q.
    int32_t rebuild;
};
// k_shaper_os_prev -> k_shaper_os: per quantum, its channel count, whether it is processed, and the processed quanta since the last rebuild
constexpr int32_t OS_INFO_PROCESSED = 0x40;
constexpr int OS_INFO_SINCE_SHIFT = 8;

struct SPanInst {
    BufRef in, out;
    float pan;
    int32_t in_ch;
    BufRef pan_track;  // p != nullptr: automated pan
};

struct PanInst {  // equal-power panner with static source/listener (panner.rs:839-870,988-1057)
    BufRef in, out;
    float dist_gain, cone_gain, azimuth;
    int32_t in_ch;
};

// HRTF panner (panner.rs:215-271,781-830 + the hrtf crate's process_samples with interpolation_steps = 1): per quantum a
// sphere triangle (v) and blend weights (w) select the L-tap left / right responses; out = gain * FIR(in)
struct HrtfSel {
    uint32_t v[3];
    float w[3];
    float gain;  // cone_gain * dist_gain
    float pad;
};
struct HrtfInst {
    BufRef in, out;
    const float* sphere_ir;  // [vertex][2][L]
    float* hist;             // [L-1] mono input before the chunk
    const HrtfSel* sel;      // per-quantum table of the chunk (moving source / listener) or nullptr: static_sel
    HrtfSel static_sel;
    int32_t L;
    int32_t in_ch;
    float correction;        // 2 for stereo input (panner.rs:805-812)
    int32_t dyn;             // 1: the input's layout changes.  A silent input is processed only while the node's tail budget lasts
                             // (tail_time_counter < L, never reset: panner.rs:697-711); afterwards the node returns early and its
                             // convolution history FREEZES.  The FIR therefore runs over the PROCESSED quanta only:
    int32_t* cmap;           // cmap[0] = processed quanta of this chunk, cmap[1 + k] = chunk quantum of the k-th of them
    int64_t* tail;           // tail_time_counter, carried across chunks
};

// the 15 spatial params of a panner (source position / orientation, listener position / forward / up); an automated one
// is a k_param track: channel 0 = value per frame, channel 1 [first frame of a quantum] = 1 if the reference's param
// buffer is single-valued in that quantum (panner.rs:833-841 branches on the listener params' lengths)
struct SpatialTracks {
    BufRef track[15];  // p == nullptr: value[i]
    float value[15];
    int32_t pad;
};
struct PanDynInst {  // equal-power panner with moving source / listener (panner.rs:833-897)
    BufRef in, out;
    SpatialTracks sp;
    spatial::PanModel model;
    int32_t in_ch;
    int32_t pad;
};
struct HrtfSelInst {  // per-quantum triangle / weights / gain of an HRTF panner with moving source / listener
    SpatialTracks sp;
    spatial::PanModel model;
    const float* pos;     // sphere vertices [v][3]
    const uint32_t* tri;  // sphere faces
    int32_t n_faces;
    int32_t pad;
    HrtfSel* sel;         // [quanta per chunk]
};

struct MixEdge {
    BufRef src;
    int32_t src_ch;
    int32_t pad;
};

struct MixInst {  // AudioRenderQuantum::add over all incoming edges of one input port, reference order
    BufRef out;
    int32_t out_ch;
    int32_t interp;  // 0 speakers, 1 discrete
    int32_t n_edges;
    uint32_t edge_offset;
    int64_t limit;  // frames >= limit are not written (destination: render length); < 0: no limit
    int32_t simple;    // every edge has out_ch channels or is mono up-mixed by copy (speakers 1 -> 2): vector fast path
    int32_t all_mono;  // simple and every edge is mono: sum once, write to all channels
};

struct DelayInst {
    BufRef in, out;
    float* ring;         // [ch][ring_len]
    uint32_t ring_len;   // power of two
    int32_t ch;
    // dynamic input layout (static channels <= 2): the reference re-mixes its whole ring whenever the input's channel count changes
    // (delay.rs:470-488), i.e. a stereo sample collapses to its mono down-mix as soon as a one-channel (or silent) quantum is written
    // after it.  mono_at[q mod mono_len] = absolute index of the last quantum <= q whose input had one channel (-1: none).
    int64_t* mono_at;
    int32_t mono_len;    // power of two >= quanta of the ring + quanta of a chunk
    int32_t dyn;         // 1: layout tracks in use
    int64_t fl;          // floor(-delay * sr): integer part of the (negative) read offset
    float k;             // fractional part
    int32_t in_cycle;    // 1: the reader runs before the writer (cycle breaker applied): history comes from the ring only
    BufRef delay_track;  // p != nullptr: automated delayTime (seconds per frame)
    float sample_rate;
    int32_t pad;
};

// slots of CompInst::meta_ring: more than the look-ahead of quanta at the highest sample rate (37 at 768 kHz), a power of two
constexpr int COMP_META_RING = 64;

struct CompInst {
    BufRef in, out;
    uint8_t* meta_ring;  // dynamic input layout: the layout bytes of the quanta inside the look-ahead ring ([COMP_META_RING], index = quantum & (COMP_META_RING - 1))
    float* ring;         // [ch][ring_len] input history
    float* state;        // [0] = prev_detector_value, [1] = last reduction (dB)
    uint32_t ring_len;   // power of two
    int32_t ch;
    int32_t delay_frames;  // (ring_size - 1) * 128
    float threshold, knee, ratio, attack, release, sample_rate;
    int32_t pad;
    int64_t end;      // the graph's last rendered frame + 1: the detector state and `reduction` stop there (a shorter graph of a longer group)
    BufRef track[5];  // attack, knee, ratio, release, threshold: p != nullptr -> automated (k-rate: first value of a quantum)
};

struct AnalyserInst {
    BufRef in, out;
    float* ring;  // 32768 + 128 floats (analysis.rs:74)
    int32_t ch;
    int32_t pad;
    int64_t end;  // the graph's last rendered frame + 1: the ring is not written from there on (a shorter graph of a longer group)
};

// One declared analyser read-out (wae_analyser_set_readouts) at frame F = q * 128: its window is the fftSize mono frames before F,
// taken from the ring for frames < f0 and from the input buffer for [f0, F) by the read-out kernels of the chunk (f0, f0 + nf] holding F
// (F = 0: the first chunk), which run before k_analyser writes that chunk into the ring.  A stage's records are sorted by F.
struct ReadoutInst {
    BufRef in;            // the analyser's input (AnalyserInst::in)
    const float* ring;    // the analyser's ring (AnalyserInst::ring)
    float* row;           // frequency: fftSize / 2 linear magnitudes (dB after k_readout_smooth); time domain: fftSize samples
    int64_t frame;        // F
    int32_t ch;
    int32_t fft_size;
    uint8_t* bytes;       // time domain with wae_analyser_set_byte_readouts: fftSize bytes of the same window; nullptr: none
};

// The frequency read-outs of one analyser, for k_readout_smooth: one thread per bin walks those of a chunk in time order
struct ReadoutSmoothInst {
    const int64_t* frames;  // [K] F of each read-out, non-decreasing
    float* rows;            // [K][bins]
    float* last_fft;        // the analyser's smoothing state (AnalyserRec::d_last_fft), zeroed per run
    float* db;              // the analyser's post-render read-out (AnalyserRec::d_db): the last row's dB
    int32_t n;              // K
    int32_t bins;
    float smoothing;
    int32_t pad;
    uint8_t* bytes;         // [K][bins] byte rows (wae_analyser_set_byte_readouts) of the same dB; nullptr: none
    float min_db, max_db;   // the node's at render time (the byte rows' range)
};

// The declared reduction read-outs of one compressor (wae_compressor_set_readouts), parallel to its CompInst in a stage that runs
// k_compressor<true>: read-out k is the reduction at frame frames[k] = 128 q_k, written when the quantum that ends there ends
struct CompReadoutInst {
    const int64_t* frames;  // [K] non-decreasing
    float* rows;            // [K]
    int32_t n;              // K
    int32_t pad;
};


struct RouteInst {  // channel merger / splitter: copy one channel
    BufRef in, out;
    int32_t in_channel, out_channel;
    int32_t zero;  // 1: write zeros (splitter output beyond the input's channels)
    int32_t in_ch;  // static channels of `in` (rows of its meta track); splitter with a dynamic input: zeros wherever in_channel >= count
};

// ---- layout tracks of nodes whose PCM does not depend on the layout (or that are handled by their own kernel) ----------------
// k_meta walks the quanta of a chunk serially, one thread per instance, and writes the output track from the input track(s).
enum MetaMode : int32_t {
    META_SOURCE = 0,     // scheduled source: silent outside [n_first, n_stop) (oscillator.rs:382-392, constant_source.rs:197-205,
                         // audio_buffer_source.rs:430-471), `count` channels inside
    META_COPY = 1,       // same layout as the input (gain, analyser pass-through, wave-shaper that propagates silence)
    META_SHAPER = 2,     // wave-shaper whose curve does not map 0 to 0: a silent input still produces sound, on its ONE channel (waveshaper.rs:395-400)
    META_PAN = 3,        // stereo / equal-power panner: silent in -> silent out, else 2 channels (stereo_panner.rs:230-235, panner.rs:698-708)
    META_CONV = 4,       // convolver: tail counter (convolver.rs:357-366), output channels from (input count, response channels) (:378-487)
    META_SPLIT = 5,      // splitter output `aux`: one channel, silent when the input has no such channel (channel_splitter.rs:196-206)
    META_MERGE = 6,      // merger: `count` channels when any input is not silent, else silent (channel_merger.rs:160-168); inputs in `more`
    META_CONST = 7,      // constant layout `count`, `aux` != 0: always silent
};
struct MetaInst {
    BufRef in, out;
    int32_t mode;
    int32_t in_ch, out_ch;   // static channels (= rows of the tracks)
    int32_t count;           // META_SOURCE / META_MERGE / META_CONST: channels when not silent
    int32_t aux;             // META_CONV: response channels; META_SPLIT: channel index; META_CONST: silent flag
    int32_t n_more;          // META_MERGE: number of inputs
    int64_t n_first, n_stop; // META_SOURCE
    int64_t tail_len;        // META_CONV: impulse length in frames
    int64_t* state;          // META_CONV: tail_count, carried across chunks
    const BufRef* more;      // META_MERGE: the inputs (device table)
};

// Mixer with per-quantum layouts: AudioRenderQuantum::add folded over the edges in processing order (quantum.rs:532-569), the
// running channel count re-mixed edge by edge.  Writes canonical PCM: channels >= count hold the speakers up-mix of the sum
// (static channels <= 2) so that layout-agnostic consumers (convolver, delay line, compressor ring) can read all static channels.
struct MixDynInst {
    BufRef out;
    int32_t out_ch;    // static channels of the port (maximum)
    int32_t interp;    // 0 speakers, 1 discrete
    int32_t mode;      // WAE_COUNT_MODE_*
    int32_t cfg_count; // channelCount of the node
    int32_t n_edges;
    uint32_t edge_offset;
    int64_t limit;
    int32_t stereo4;   // every edge and the port have at most two static channels and 16-byte aligned arena buffers: four frames per thread
    int32_t pad;
};


// oscillator with automated / audio-rate frequency or detune (oscillator.rs:447-459): phase = running sum of the
// per-frame increments
struct OscArInst {
    OscInst base;        // type, table, n_first, n_stop (incr / phase0 unused)
    BufRef freq, detune; // p == nullptr: constant f_val / d_val
    float f_val, d_val;
    double start_ratio;  // (t_first - start_time) / dt: sub-sample start (oscillator.rs:527-540)
    double* phase;       // carried phase (before the first frame of the next chunk)
    float sample_rate;
    int32_t pad;
};

// biquad with automated parameters: coefficients per frame (biquad_filter.rs:837-855), serial recurrence
struct BiquadArInst {
    BufRef in, out;
    BufRef q, detune, freq, gain;  // p == nullptr: constant *_val
    float q_val, detune_val, freq_val, gain_val;
    double* state;
    float sample_rate;
    int32_t type;
    int32_t ch;
    int32_t pad;
    int32_t* dyn_len;  // see BiquadInst
    BufRef coefs;      // [5][chunk frames] f64 (b0, b1, b2, a1, a2 of every frame), written by k_biquad_coefs: the per-frame coefficient
                       // formulas (sin / cos / pow in f64) run one thread per frame, only the 9-flop recurrence stays serial
};

// ---- AudioParam automation (AudioParamProcessor, src/param.rs:664-1600) -------------------------------------
struct ParamEvDev {  // AudioParamEvent (param.rs:172-181) after handle_incoming_event
    int32_t type;    // WAE_EVENT_*
    float value;
    double time;
    double aux;          // time constant (setTarget) / duration (value curve)
    double cancel_time;  // cancel_and_hold
    int32_t has_cancel;
    int32_t values_off, values_len;  // value curve samples in the curve pool
    int32_t pad;
};
struct ParamState {  // render-side state of one param, carried across chunks
    float intrinsic;
    int32_t head;        // events [0, head) have been popped
    int32_t has_last;
    int32_t override_valid;  // replace_peek(): the event at `head` is `override_ev`
    int32_t inited;          // 0 after the per-run memset: the first quantum this param is rendered initialises the state
    int32_t pad;
    ParamEvDev last;
    ParamEvDev override_ev;
};
struct ParamInst {
    const ParamEvDev* events;
    const float* curves;
    ParamState* state;
    BufRef in;   // summed audio-rate input (mono), p == nullptr: none
    BufRef out;  // 1 channel: the computed value of every frame
    float def, mn, mx, intrinsic0;
    float sample_rate;
    int32_t n_events;
    int32_t a_rate;
    int32_t has_last0;  // render-side `last_event` the state starts with (params whose events were extended at a suspend point)
    ParamEvDev last0;
};

// ---- fused chain: source -> {biquad | gain | shaper}* -> buffer or destination, one pass over the PCM -------
enum ChainSrc : int32_t { CHAIN_SRC_BUFFER = 0, CHAIN_SRC_ABSN = 1, CHAIN_SRC_OSC = 2, CHAIN_SRC_CONST = 3 };
struct ChainBiquad {
    double b0, b1, b2, a1, a2;
    double* state;  // [ch][4] = x1, x2, y1, y2
    int32_t coef;   // index into the ScanCoef table of the stage
    int32_t pad;
};
constexpr int CHAIN_MAX_BIQUADS = 2;
// canonical chain: src -> *g[0] -> [biquad A] -> *g[1] -> [biquad B] -> *g[2] -> [shaper] -> *g[3] -> out
struct ChainInst {
    int32_t src_kind;
    int32_t ch;          // channels processed (one CTA each)
    int32_t n_biquad;    // 0..2
    int32_t has_shaper;
    float g[4];
    int32_t out_dup;     // >1: the (mono) result is written to channels 0..out_dup-1 (speaker up-mix 1->2 by copy)
    int32_t shaper_n;    // curve length
    int32_t shaper_keeps_silence;  // can_propagate_silence (waveshaper.rs:480-503): the curve maps 0 to 0
    int32_t pad2;
    const float* curve;  // nullptr: pass-through
    BufRef in;           // CHAIN_SRC_BUFFER
    AbsnInst absn;       // CHAIN_SRC_ABSN (out unused)
    OscInst osc;         // CHAIN_SRC_OSC (out unused)
    ConstInst cst;       // CHAIN_SRC_CONST (out unused)
    BufRef out;
    int64_t limit;       // frames >= limit are not written (destination); < 0: none
    int64_t end;         // the graph's render end (its length in whole quanta): a work item starting there has nothing to render
    ChainBiquad bq[CHAIN_MAX_BIQUADS];
};

// k_chain work decomposition (see the kernel): time slabs handed out in ticket order, filter state handed from slab to slab
constexpr int CHAIN_MAX_SLABS = 64;
constexpr int CHAIN_MAX_PRE_SLABS = 256;  // (PRE: few pairs, long renders)
struct ChainSched {
    int32_t n_slabs;         // time slabs per (instance, channel)
    int32_t tiles_per_slab;  // whole 2048-frame tiles per slab
    int32_t max_ch;          // channel slots per instance in the item numbering
    int32_t slab_stride;     // hand-off slots per (instance, channel)
    uint32_t epoch;          // launch number of this stage: the value a hand-off flag written by this launch carries
    int32_t pre_log2;        // >= 0: k_chain<..., PRE> — slabs of WAE_CHAIN_PRE_TILES << pre_log2 tiles publish the next slab's state before they render
    unsigned* ticket;        // one counter per stage (zero between launches); nullptr: item = blockIdx.x
    double* handoff;         // [(instance * max_ch + channel) * slab_stride + slab][CHAIN_MAX_BIQUADS][4]: state ENTERING the slab
    unsigned* flags;         // same indexing: == epoch once that state is written
};
struct ChainAux {  // per-stage device memory of the slab hand-off (engine-owned)
    unsigned* ticket = nullptr;
    double* handoff = nullptr;
    unsigned* flags = nullptr;
    int32_t slab_stride = 0;
    uint32_t epoch = 0;
};

// k_voice_sum: the voices (oscillator -> [biquad] -> gain chains, mono, static layout) of one input port, summed in the port's edge
// order without ever being written out.  The group's ChainInst records are consecutive in the stage's instance table.
struct VoiceGroup {
    int32_t first;     // first ChainInst of the group
    int32_t n_voices;
    BufRef out;        // the mono sum (arena buffer or the rendered PCM)
    int32_t out_dup;   // channels the sum is written to (speaker up-mix 1 -> 2 by copy), >= 1
    int32_t pad;
    int64_t limit;     // frames >= limit are not written (destination); < 0: none
};

// ---- convolver (uniformly partitioned overlap-save, block WAE_CONV_BLOCK, time-batched) -----------------
struct ConvInput {   // one input channel of one convolver instance
    BufRef in;
    float* prev;     // [block] last block of the previous chunk
    float2* xring;   // [xring_blocks][block] input spectra ring
    int32_t in_channel;
    int32_t xring_blocks;
    int64_t end;     // the graph's render end (its length in whole quanta): input from there on is zero, blocks starting there are not built
};
struct ConvPath {    // one FFTConvolver of the reference: (input channel, IR channel) -> output channel
    BufRef out;
    const float2* h;  // [S][block] IR segment spectra
    float2* y;        // [blocks per chunk][block] output spectra of the chunk (scratch between k_conv_mac and k_conv_ifft)
    int32_t input;    // index into the ConvInput table
    int32_t S;        // IR segments
    int32_t out_channel;
    int32_t accumulate;  // 1: out += (true-stereo mix-down, convolver.rs:436-452)
    int64_t limit;       // >= 0: `out` is the rendered PCM itself (the convolver is the destination's only input): frames from `limit` on do not exist
    int64_t end;         // the graph's render end (its length in whole quanta): output blocks starting there are not computed
};
// Second path of a ConvolverNode with a ONE-channel response whose input switches between one and two channels (convolver.rs:343-400):
// the reference's convolvers[1] is fed the R channel of the two-channel quanta only and freezes (history, partly filled block and all)
// whenever the input is mono or silent.  Its input is therefore the STREAM of those quanta with the gaps removed: per chunk the map kernel
// lists the chunk quanta it processes and advances the stream cursor, the stream window [previous full stream block | partial block
// carried from the last chunk | new frames] is transformed block by block (a partial block again once it holds more frames, like the
// reference re-transforms its partly filled block), the MAC / inverse transform run over the stream's blocks, and the output frames of
// the new stream frames are scattered back to channel 1 of the quanta they came from.
struct ConvCmpInst {
    BufRef in;         // canonical PCM of the input (2 static channels, layout track)
    ConvInput x;       // x.xring: input spectra at the stream's absolute block index (x.in / prev / in_channel unused)
    ConvPath path;     // h, S, y ([window blocks][block] scratch), out (channel 1 = out_channel); input / accumulate / limit unused
    int64_t* cursor;   // [1] frames fed to convolvers[1] so far (persistent)
    float* carry;      // [2 block] the stream's last full block before the cursor | its partial block (persistent)
    float* win;        // [(window blocks + 1) block] stream window of the chunk, from block cursor / block - 1 on (scratch)
    int32_t* qmap;     // [quanta per chunk] chunk quanta processed this chunk, in order (scratch)
    int64_t* wdesc;    // [2] cursor before the chunk, new frames of the chunk (scratch, written by the map kernel)
    int32_t in_ch;     // static channels of `in`
    int32_t pad;
};

// ---- wae_batch_bind_sources: device audio -> a device-input slot of a group's source slab --------------------------------------
struct BindItem {
    float* dst;          // the slot: [channels][stride], 16 B aligned (slab offsets are multiples of 4 floats)
    const float* src;    // caller's device audio: channel c is `len` floats at src + c * src_stride (any alignment)
    int64_t stride;      // slot channel stride, floats (len rounded up to 4; [len, stride) is written as zeros)
    int64_t src_stride;  // floats
    int64_t len;
    int32_t channels;
    int32_t pad;
};

// ---- wae_batch_bind_responses: caller device audio -> the IR spectra of a declared ConvolverNode response --------------------------
struct RespBindItem {
    const float* src;    // caller's response: channel c is `len` floats at src + c * src_stride (any alignment)
    float2* h;           // the node's spectra: [channels][S + WAE_CONV_H_PAD][WAE_CONV_SPEC], padding partitions zero
    int64_t src_stride;  // floats
    int64_t len;         // declared length
    float sample_rate;   // the response's rate (normalisation)
    int32_t channels;    // 1, 2 or 4
    int32_t S;           // partitions: ceil(len / WAE_CONV_BLOCK)
    int32_t normalize;
    // written on the device by the bind's kernels: the scale (1 when not normalising) and per channel the trimmed length m (0 on entry)
    float scale;
    int32_t m[4];
    int32_t pad;
};

// ---- wae_batch_bind_curves: caller device curve -> the curve memory of a declared WaveShaperNode, and the records its value decides --
// A record field that depends on whether the curve maps 0 to 0 (can_propagate_silence): ChainInst::shaper_keeps_silence, the
// MetaInst::mode of the node's output track, ShaperOsInst::rebuild.  The bind writes `keeps` or `other` into it.
struct CurvePatch {
    int32_t* dst;
    int32_t keeps, other;
};
struct CurveBindItem {
    const float* src;            // caller's curve (any alignment)
    float* dst;                  // the node's curve memory: 16 B aligned, `n` rounded up to 4 floats
    const CurvePatch* patches;   // the node's entries
    int32_t n;                   // curve length
    int32_t n_patches;
};

// ---- wae_batch_bind_periodic_waves: caller coefficients -> the wavetable of a declared custom OscillatorNode ------------------------
struct WaveBindItem {
    const float* re;   // caller's coefficients (null: zeros)
    const float* im;
    float* dst;        // the node's wavetable memory: `len` floats
    int32_t n;         // coefficient count (>= 2)
    int32_t len;       // wavetable length
    int32_t normalize;
    int32_t pad;
};

// ---- wae_batch_bind_iir_coefficients: caller f64 coefficients -> the records of a declared IIRFilterNode ---------------------------
// One record the coefficients reach: an IirInst (k_iir_serial; `b` = IirInst::b, `a` = IirInst::a, n = max(nff, nfb) of each) or the
// ChainBiquad of a k_chain record (`b` = ChainBiquad::b0: b0, b1, b2, a1, a2; `a` null) with its scan constants (`scan`, null: none).
struct IirPatch {
    double* b;
    double* a;
    void* scan;  // ScanCoef
};
struct IirBindItem {
    const double* ff;         // caller's coefficients (8 B aligned)
    const double* fb;
    const IirPatch* patches;  // the node's entries
    int32_t nff, nfb;         // 1..20 each
    int32_t n_patches;
    int32_t pad;
};

// ---- wae_batch_bind_value_curves: caller values -> the SetValueCurveAtTime values of a declared param (ParamInst::curves + values_off)
struct ValueCurveBindItem {
    const float* src;  // caller's values (4 B aligned)
    float* dst;        // in the param's curve pool
    int32_t n;         // the declared length
    int32_t pad;
};

// ---- wae_batch_bind_schedules: caller start / stop times -> the record fields of a declared scheduled source they reach ------------
// One entry per record; the bind re-derives the fields from the times with the planner's own functions (wae_kernels.h).
enum SchedKind : int32_t {
    SCHED_OSC = 0,          // OscInst (S_OSC, ChainInst::osc): n_first, n_stop, phase0
    SCHED_OSC_AR = 1,       // OscArInst: base.n_first, base.n_stop, base.phase0, start_ratio
    SCHED_CONST = 2,        // ConstInst (S_CONST, ChainInst::cst): n_first, n_stop
    SCHED_META_OSC = 3,     // MetaInst (META_SOURCE) of an oscillator's gated output: n_first, n_stop
    SCHED_META_CONST = 4,   // MetaInst (META_SOURCE) of a constant source's gated output: n_first, n_stop
    SCHED_ABSN_BOUND = 5,   // AbsnBoundInst: s.n_first, s.n_stop, start_delta, n_start, fast_end, fast_ok
    SCHED_ABSN_SERIAL = 6,  // AbsnSerialInst: start_time, stop_time (the kernel takes them raw)
};
struct SchedPatch {
    void* dst;            // the record
    int32_t kind;
    int32_t flag;         // SCHED_ABSN_BOUND: fast_ok but for the start and stop (sampling ratio 1, default loop points, no duration)
    float sample_rate;    // the graph's (the clock)
    int32_t pad;
    double* start_out;    // SCHED_OSC of an oscillator whose pitch is bound from device memory: the clamped start is also written here,
                          // where its PATCH_OSC entry reads it (nullptr: none).  SCHED_OSC* take the phase increment from the record.
    double offset;        // SCHED_ABSN_BOUND: start(when, offset), taken when the offset is not bound
    double duration;      // SCHED_ABSN_BOUND: the buffer's duration
    double stop_time;     // the planned stop time, taken when the stop is not bound (>= 1e300: none)
    int64_t lq;           // SCHED_ABSN_BOUND: the render length of the plan (absn_fast_end)
};
enum SchedBinds : int32_t {  // the declared values after the start, in the order they follow it in the caller's row
    SCHED_BIND_STOP = 1,
    SCHED_BIND_OFFSET = 2,    // AudioBufferSourceNode: start(when, offset)
    SCHED_BIND_DURATION = 4,  // AudioBufferSourceNode: start(when, offset, duration)
};
struct SchedBindItem {
    const double* times;        // caller's row: start, [stop], [offset], [duration] (8 B aligned)
    const SchedPatch* patches;  // the node's entries
    double lo[4], hi[4];        // the declared windows the values are clamped to (a NaN becomes lo): start, stop, offset, duration
    int32_t n_patches;
    int32_t binds;              // SchedBinds
};

// ---- wae_batch_bind_loops: caller loop points -> the records of a declared looping AudioBufferSourceNode ------------------------------
enum LoopKind : int32_t {
    LOOP_BOUND = 0,   // AbsnBoundInst: s.loop_start / s.loop_end = the actual loop points (k_absn_loop_schedule then walks its table)
    LOOP_SERIAL = 1,  // AbsnSerialInst: loop_start / loop_end after clamp_loop_boundaries (the kernel takes them as they are)
};
struct LoopPatch {
    void* dst;               // the record
    int32_t kind;
    int32_t pad;
    double buffer_duration;  // of the source's buffer (clamp_loop_boundaries)
};
struct LoopBindItem {
    const double* points;     // caller's row: loop_start, loop_end (8 B aligned)
    const LoopPatch* patches;  // the node's entries
    double lo[2], hi[2];       // the declared windows the values are clamped to (a NaN becomes lo): start, end
    int32_t n_patches;
    int32_t pad;
};
// A looping record of the bound slow track whose playhead table is derived on the device (k_absn_loop_schedule, one thread per walk)
// from its loop points, rate, detune, start, offset and duration, into the table the record points at (s.seg_n / s.seg_bt, `cap`
// segments).  `lq`: the frames its group renders.
struct LoopWalk {
    AbsnBoundInst* rec;
    int64_t lq;
    int32_t cap;
    int32_t pad;
};

// ---- wae_batch_bind_params: per-run values of params planned as constants ------------------------------------------------------
struct ParamBindItem {  // one float of the caller's device memory -> value slot `slot`
    const float* src;
    int32_t slot;
    int32_t pad;
};
struct ParamSlotInfo {  // how a slot takes a bound value: clamped to [lo, hi]; non-finite -> def (the param's default value)
    float lo, hi, def;
    int32_t pad;
};
// A patch entry: one planned record field that a bound value reaches, re-derived from the value slots and the planned constants.
// Operand i is slot[i] (>= 0) or the constant val[i].
enum PatchKind : int32_t {
    PATCH_GAIN = 0,    // float *dst = the product of the n operands in node order, each bound one after gain.rs's 1e-6 shortcuts
    PATCH_META = 1,    // int32 *dst (MetaInst::mode of a gain that may answer with silence): META_CONST when that product is 0, else META_COPY
    PATCH_BIQUAD = 2,  // operands q, detune, frequency, gain: double *dst = b0, b1, b2, a1, a2; ScanCoef *dst2 (k_chain) or nullptr
    PATCH_SPAN = 3,    // operand pan: float *dst = pan, float2 *dst2 = the stereo gains for n input channels
    PATCH_RAW = 4,     // float *dst = operand 0
    PATCH_OSC = 5,     // operands frequency, detune: OscInst *dst = incr, inv_incr, outside_nyquist, and phase0 from the start time at
                       // const double *dst2 (the planned one, or the slot a bound schedule writes: SchedPatch::start_out)
};
constexpr int PATCH_OPS = 8;
struct ParamPatch {
    int32_t kind;
    int32_t n;          // PATCH_GAIN / PATCH_META: operands; PATCH_BIQUAD: filter type; PATCH_SPAN: input channels
    float sample_rate;  // PATCH_BIQUAD, PATCH_OSC
    int32_t pad;
    void* dst;
    void* dst2;
    int32_t slot[PATCH_OPS];
    float val[PATCH_OPS];
};

// A spatial entry: one static panner whose source or listener is bound from device memory (panner params 0..5, listener params 0..8),
// re-derived by k_derive_spatial after k_derive_params.  Operand i (the 15 spatial params in SpatialTracks order) is slot[i] (>= 0) or
// the constant val[i].
enum SpatialKind : int32_t {
    SPATIAL_PAN = 0,   // PanInst *dst = azimuth, dist_gain, cone_gain (S_PAN)
    SPATIAL_SEL = 1,   // HrtfSel *dst = triangle, weights, gain (HrtfInst::static_sel)
    SPATIAL_RESP = 2,  // HrtfSel *dst as SPATIAL_SEL, then the blended pair into resp [2][taps] (k_spatial_blend), which k_resp_fft
                       // transforms into the node's spectra
};
struct SpatialPatch {
    int32_t kind;
    int32_t n_faces;         // SPATIAL_SEL / SPATIAL_RESP: the sphere's faces
    void* dst;
    const float* pos;        // sphere vertices [v][3]
    const uint32_t* tri;     // sphere faces
    const float* ir;         // SPATIAL_RESP: the sphere's responses at the context rate [v][2][taps]
    float* resp;             // SPATIAL_RESP: the blended pair [2][taps]
    int32_t taps;
    float correction;        // SPATIAL_RESP: 2 for a two-channel input (panner.rs:805-812)
    spatial::PanModel model;
    int32_t slot[15];
    float val[15];
};

// An output entry: one planned record field that points into the batch's rendered PCM (the BufRef::p of a destination writer: k_mix,
// k_mix_dyn, k_chain, k_voice_sum, k_conv_mac_ifft).  wae_batch_bind_output writes base + off into it (k_bind_output).
struct OutPatch {
    float** dst;
    uint64_t off;  // floats from the start of the packed output
};

// A source-reference entry: the PCM pointer and channel stride of one planned record that plays an AudioBufferSourceNode declared with
// wae_buffer_source_set_device_input_by_reference (AbsnInst on k_buffer_source or inside a ChainInst, AbsnSlowInst, AbsnBoundInst::s,
// AbsnSerialInst).  wae_batch_bind_sources writes the caller's pointer and stride into them (k_bind_source_refs).
struct SrcRefPatch {
    const float** buf;
    int64_t* stride;
};
// one row of k_bind_source_refs: entry `entry` of the batch now reads `pcm`, channel c at pcm + c * stride
struct SrcRefBindItem {
    const float* pcm;
    int64_t stride;  // floats, >= the declared length, any value
    int32_t entry;
    int32_t pad;
};

}  // namespace wae
