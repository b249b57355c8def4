// Launch wrappers of the sm_90a kernels (wae_kernels.cu).
#pragma once
#include "wae_device.h"

#include <cuda_runtime.h>

namespace wae {

// Per-biquad constants of the time-parallel recurrence (host-computed in f64).  M = [[-a1,-a2],[1,0]] advances the
// state (y[n-1], y[n-2]) by one frame; A = M^WAE_CHAIN_K advances it by one thread (WAE_CHAIN_K frames).
constexpr int WAE_CHAIN_K = 16;  // frames per thread of k_chain
constexpr int WAE_CONV_BLOCK = 8192;            // frames per convolver partition (the reference's 1024 is a latency choice, see wae_kernels.cu)
constexpr int WAE_CONV_SPEC = WAE_CONV_BLOCK;   // float2 per block spectrum (packed real FFT of 2 * block: bin 0 = (DC, Nyquist))
// IR spectra of one response channel: [WAE_CONV_H_PAD_LO zero partitions][S partitions][zero partitions up to WAE_CONV_H_PAD in total] —
// k_conv_mac walks the partitions in groups of 8 x 8 products whose first and last group reach 7 / up to 15 partitions past the ends
constexpr int WAE_CONV_H_PAD_LO = 7;
constexpr int WAE_CONV_H_PAD = 7 + 16;
struct ScanCoef {
    double Pshfl[5][4];    // A^(2^d), d = 0..4: warp-level Kogge-Stone steps
    double Plane[32][4];   // A^(lane+1): carries a warp's incoming state to each lane
    double Pwarp[4];       // A^32: one warp
    double GL[16];         // G^L, L = WAE_CHAIN_PRE_TILES tiles: (x1, x2, y1, y2) entering a slab of L frames -> its share of the state leaving it
};
constexpr int WAE_CHAIN_PRE_TILES = 16;  // 32768 frames (k_chain PRE: slabs of WAE_CHAIN_PRE_TILES << pre_log2 tiles)

// The scan constants of one biquad, in f64: one source for the planner (host) and for k_bind_params (device, bound coefficients).  The
// build compiles without FMA contraction on both sides, so equal coefficients give bit-equal constants.
struct ScanM2 {
    double a, b, c, d;
};
WAE_HD ScanM2 scan_mul(const ScanM2& x, const ScanM2& y) {
    return ScanM2{x.a * y.a + x.b * y.c, x.a * y.b + x.b * y.d, x.c * y.a + x.d * y.c, x.c * y.b + x.d * y.d};
}
WAE_HD void make_scan_coef(double b1, double b2, double a1, double a2, ScanCoef& sc) {
    const ScanM2 M{-a1, -a2, 1., 0.};
    ScanM2 r{1., 0., 0., 1.};
    for (int j = 0; j < WAE_CHAIN_K; j++) r = scan_mul(M, r);
    const ScanM2 A = r;  // M^K: one thread of k_chain
    ScanM2 pw = A;
    for (int d = 0; d < 5; d++) {
        sc.Pshfl[d][0] = pw.a; sc.Pshfl[d][1] = pw.b; sc.Pshfl[d][2] = pw.c; sc.Pshfl[d][3] = pw.d;
        pw = scan_mul(pw, pw);
    }
    sc.Pwarp[0] = pw.a; sc.Pwarp[1] = pw.b; sc.Pwarp[2] = pw.c; sc.Pwarp[3] = pw.d;  // A^32
    ScanM2 pl = A;
    for (int l = 0; l < 32; l++) {
        sc.Plane[l][0] = pl.a; sc.Plane[l][1] = pl.b; sc.Plane[l][2] = pl.c; sc.Plane[l][3] = pl.d;
        pl = scan_mul(A, pl);
    }
    // one frame with zero input: (x1, x2, y1, y2) -> (0, x1, b1 x1 + b2 x2 - a1 y1 - a2 y2, y1); G^L by squaring (L = 2^15 frames)
    static_assert(WAE_CHAIN_PRE_TILES * WAE_CHAIN_K * 128 == 1 << 15, "GL below is G^(2^15)");
    double g[16] = {0., 0., 0., 0., 1., 0., 0., 0., b1, b2, -a1, -a2, 0., 0., 1., 0.}, h[16];
    for (int sq = 0; sq < 15; sq++) {
        for (int rr = 0; rr < 4; rr++)
            for (int cc = 0; cc < 4; cc++) {
                double a = 0.;
                for (int k = 0; k < 4; k++) a += g[4 * rr + k] * g[4 * k + cc];
                h[4 * rr + cc] = a;
            }
        for (int i = 0; i < 16; i++) g[i] = h[i];
    }
    for (int i = 0; i < 16; i++) sc.GL[i] = g[i];
}

// The rate-dependent constants of a slow-track source (audio_buffer_source.rs:660-678,826-838), in f64: one source for the planner
// (host, absn_slow) and for k_buffer_source_slow<true> (device, rates bound from device memory).  `delta`: t_first - start; `n_stop`: the
// stop frame; `duration`: the explicit duration (>= 1e300: none).  n_end is the frame after the last one the source can play.
struct AbsnSlowDerived {
    double step, offset0, elapsed0;
    int64_t n_end;
};
WAE_HD AbsnSlowDerived absn_slow_derive(double dt, double computed_rate, double offset, double delta, double buffer_duration, double duration,
                                        bool loop, double loop_end, int64_t n_first, int64_t n_stop) {
    auto mx = [](double a, double b) { return a < b ? b : a; };  // std::max / std::min, -0. and all
    auto mn = [](double a, double b) { return b < a ? b : a; };
    AbsnSlowDerived d;
    d.step = dt * computed_rate;
    double off = offset + delta * computed_rate;  // :672-674
    off = mn(mx(off, 0.), buffer_duration);
    if (loop && off > loop_end) off = loop_end;  // :676-678 (rate >= 0)
    d.offset0 = off;
    d.elapsed0 = fabs(delta * computed_rate);
    // the source has ended after the stop frame, the explicit duration, or (not looping) the end of the buffer
    d.n_end = n_stop;
    if (d.step > 0.) {
        if (!loop) {
            const int64_t e = n_first + (int64_t)ceil(mx(0., buffer_duration - off) / d.step);
            d.n_end = e < d.n_end ? e : d.n_end;
        }
        if (duration < 1e300) {
            const int64_t e = n_first + (int64_t)ceil(mx(0., duration - d.elapsed0) / d.step);
            d.n_end = e < d.n_end ? e : d.n_end;
        }
    }
    return d;
}

// ---- Sample-accurate scheduling of AudioScheduledSourceNodes, in f64 without transcendentals: one source for the planner (host, times
// given when the graph is built) and for k_bind_schedules (device, times bound from device memory, wae_batch_bind_schedules).  The build
// compiles without FMA contraction on both sides, so equal times give bit-equal frames and phases.
constexpr int64_t SCHED_NEVER = 0x7fffffffffffffffll;
WAE_HD bool almost_equal(double x, double y) {  // `almost` crate 0.2: absolute or relative sqrt(eps)
    if (x == y) return true;
    const double tol = 1.4901161193847656e-8;
    const double d = fabs(y - x), m = fabs(x) < fabs(y) ? fabs(y) : fabs(x);
    return d <= tol || d <= m * tol;
}
// The reference walks quanta (current_time = frame / sample_rate, src/render/thread.rs:357-360) and, inside the quantum that contains a
// start/stop time, accumulates `current_time += dt` per frame (oscillator.rs:511-557, constant_source.rs:231-246).
// first_frame_at_or_after(T) returns the first frame whose accumulated time is >= T, reproducing that walk.
struct SchedClock {
    double sample_rate, dt;
    WAE_HD explicit SchedClock(float sr) : sample_rate((double)sr), dt(1. / (double)sr) {}
    WAE_HD double block_time(int64_t q) const { return (double)(q * 128) / sample_rate; }
    WAE_HD double next_block_time(int64_t q) const { return block_time(q) + dt * 128.; }
    // first quantum whose next_block_time is > T (i.e. the node is not skipped by `T >= next_block_time`)
    WAE_HD int64_t quantum_containing(double T) const {
        if (!(T < 1e15)) return SCHED_NEVER / 256;
        int64_t q = (int64_t)floor(T * sample_rate / 128.) - 2;
        if (q < 0) q = 0;
        while (!(T < next_block_time(q))) q++;
        return q;
    }
    // returns frame index; *time_out = accumulated time of that frame
    WAE_HD int64_t first_frame_at_or_after(double T, double* time_out = nullptr) const {
        int64_t q = quantum_containing(T);
        if (q >= SCHED_NEVER / 512) return SCHED_NEVER;
        double t = block_time(q);
        for (int i = 0; i < 128; i++) {
            if (t >= T) {
                if (time_out) *time_out = t;
                return q * 128 + i;
            }
            t += dt;
        }
        if (time_out) *time_out = block_time(q + 1);
        return (q + 1) * 128;
    }
};
// OscillatorNode (oscillator.rs:391-428,511-540): the first rendered frame and its phase (`incr` = computed frequency / sample rate), and
// the sub-sample start (t_first - start) / dt that the a-rate kernel adds its own increment with
struct OscStart {
    int64_t n_first;
    double phase0, start_ratio;
};
WAE_HD OscStart osc_start(const SchedClock& clock, double start_time, double incr, bool outside_nyquist) {
    OscStart r{0, 0., 0.};
    const int64_t q = clock.quantum_containing(start_time);
    double start = start_time;
    if (start < clock.block_time(q)) start = clock.block_time(q);  // "prevent scheduling in the past"
    double cur = clock.block_time(q);  // the accumulated per-frame clock of that quantum
    int i = 0;
    for (; i < 128; i++) {
        if (!(cur < start)) break;
        cur += clock.dt;
    }
    r.n_first = q * 128 + i;
    if (i < 128 && cur > start) {
        const double ratio = (cur - start) / clock.dt;
        r.start_ratio = ratio;
        double ph = incr * ratio;
        if (outside_nyquist) {
            ph = fmod(ph, 1.);
            if (ph < 0.) ph += 1.;
        } else {
            ph = ph >= 1. ? ph - 1. : (ph < 0. ? ph + 1. : ph);  // unroll_phase
        }
        r.phase0 = ph;
    }
    return r;
}
WAE_HD int64_t osc_stop_frame(const SchedClock& clock, double stop_time) {
    if (!(stop_time < 1e300)) return SCHED_NEVER;
    const int64_t qs = clock.quantum_containing(stop_time);
    return stop_time <= clock.block_time(qs) ? qs * 128 : clock.first_frame_at_or_after(stop_time);
}
// AudioBufferSourceNode: the quantum its start time falls in.  A start time that IS the next block boundary but compares below
// next_block_time by one rounding: the reference goes through one all-silent slow-track quantum, then aligns (audio_buffer_source.rs:521-523)
WAE_HD int64_t absn_start_quantum(const SchedClock& clock, double start_time) {
    int64_t q = clock.quantum_containing(start_time);
    if (start_time > clock.block_time(q) && start_time == clock.block_time(q + 1)) q = q + 1;
    return q;
}
// the slow track's first playing frame: current_time = block_time + i * dt (:648), sticky within almost::equal (:652-654); the first
// frame with current_time >= stop_time (:663)
struct AbsnStart {
    int64_t n_first, n_stop;
    double t_first, start;  // the time of frame n_first, the start time (snapped to it when almost equal)
};
WAE_HD AbsnStart absn_start(const SchedClock& clock, double start_time, double stop_time) {
    AbsnStart r{-1, SCHED_NEVER, 0., start_time};
    int64_t qq = clock.quantum_containing(r.start);
    for (int guard = 0; guard < 3 && r.n_first < 0; guard++, qq++) {
        const double bt0 = clock.block_time(qq);
        for (int i = 0; i < 128; i++) {
            const double t = bt0 + (double)i * clock.dt;
            if (almost_equal(t, r.start)) r.start = t;
            if (!(t < r.start)) {
                r.n_first = qq * 128 + i;
                r.t_first = t;
                break;
            }
        }
    }
    if (r.n_first < 0) r.n_first = qq * 128;
    if (stop_time < 1e300) {
        const int64_t qs = clock.quantum_containing(stop_time);
        int64_t ns = (qs + 1) * 128;
        const double bt0 = clock.block_time(qs);
        for (int i = 0; i < 128; i++)
            if (bt0 + (double)i * clock.dt >= stop_time) {
                ns = qs * 128 + i;
                break;
            }
        r.n_stop = ns;
    }
    return r;
}
// the fast track of a non-looping source: the frame after the quantum in which it has `ended`.  The reference accumulates
// buffer_time += block_duration and stops once it reaches the buffer's duration (audio_buffer_source.rs:609,826-838) — replayed, not
// divided.  lq: the render length the walk stops after.
WAE_HD int64_t absn_fast_end(const SchedClock& clock, int64_t lq, int64_t n_start, double duration) {
    const double block_duration = clock.dt * 128.;
    const int64_t max_q = (lq - n_start) / 128 + 2;
    int64_t played = 0;
    double bt = 0.;
    while (played < max_q) {
        bt += block_duration;
        played++;
        if (bt >= duration) break;
    }
    return n_start + played * 128;
}

// The loop points a looping slow-track source plays (audio_buffer_source.rs:400-417 clamp_loop_boundaries, then the actual loop points
// of :627-636): one source for the planner (host, loop points bound from device memory: the placeholders) and for k_bind_loops (device).
struct AbsnLoopPoints {
    double start, end;        // after clamp_loop_boundaries (AbsnSerialInst)
    double actual_start, actual_end;  // the loop the slow track plays (AbsnSlowInst)
};
WAE_HD AbsnLoopPoints absn_loop_points(double loop_start, double loop_end, double buffer_duration) {
    AbsnLoopPoints p;
    p.start = loop_start < 0. ? 0. : (loop_start > buffer_duration ? buffer_duration : loop_start);
    p.end = (loop_end <= 0. || loop_end > buffer_duration) ? buffer_duration : loop_end;
    const bool custom = p.start >= 0. && p.end > 0. && p.start < p.end;
    p.actual_start = custom ? p.start : 0.;
    p.actual_end = custom ? p.end : buffer_duration;
    return p;
}

// The playhead schedule of a looping slow-track source (AbsnSlowInst::seg_n / seg_bt): the reference's per-frame loop bookkeeping
// (audio_buffer_source.rs:730-770) walked from event to event — a frame where buffer_time is snapped to a loop point (almost::equal) or
// wrapped starts a new segment.  One source for the planner (host-built loop points) and for k_absn_loop_schedule (loop points bound from
// device memory); the build compiles without FMA contraction on both sides, so equal inputs give bit-equal tables.  ls2 / le2: the actual
// loop points; off: buffer_time at n_first (absn_slow_derive's offset0); frames [n_first, n_end) are walked.  Writes at most `cap` (>= 1)
// segments and returns their number, or -1 when the walk needs more than `cap` (the first `cap` are written and valid).  A source that
// starts at or past the loop end never enters the loop (:700-707): one segment.
WAE_HD int32_t absn_loop_segments(double ls2, double le2, double step, int64_t n_first, int64_t n_end, double off, int64_t* seg_n,
                                  double* seg_bt, int32_t cap) {
    seg_n[0] = n_first;
    seg_bt[0] = off;
    int32_t k = 1;
    if (!(off < le2)) return k;
    const double len2 = le2 - ls2;
    int64_t m = 0;   // frames since n_first
    double v = off;  // buffer_time of frame m
    bool entered = false;
    auto tz = [](double x) { return 3.0e-8 * (1.0 + fabs(x)); };  // a little wider than almost::equal
    while (n_first + m < n_end) {
        // frames until the playhead can touch the tolerance zone of a loop point
        const double to_ls = v < ls2 - tz(ls2) ? (ls2 - tz(ls2) - v) / step : 0.;
        const double to_le = v < le2 - tz(le2) ? (le2 - tz(le2) - v) / step : 0.;
        // (until the loop is entered, the loop start's zone is walked frame by frame too: a frame that lands in it is snapped to it)
        const double skip = !entered ? (to_le < to_ls ? to_le : to_ls) : to_le;
        const int64_t adv = (int64_t)floor(skip);
        if (adv > 0) {
            v += (double)adv * step;
            m += adv;
            continue;
        }
        // exact per-frame logic of the reference
        double w = v;
        if (almost_equal(w, le2)) w = le2;
        if (almost_equal(w, ls2)) w = ls2;
        if (!entered && w >= ls2) entered = true;
        if (entered) {
            while (w >= le2) w -= len2;
            while (w < ls2) w += len2;
        }
        if (w != v && n_first + m > seg_n[k - 1]) {
            if (k == cap) return -1;
            seg_n[k] = n_first + m;
            seg_bt[k] = w;
            k++;
        } else if (w != v) {
            seg_bt[k - 1] = w;
        }
        v = w + step;
        m += 1;
    }
    return k;
}

void upload_twiddles();                         // convolver FFT tables (computed in wae_kernels.cu, f64 -> f32)
void conv_fft_selftest(float* data, int mode);   // host emulation of the convolver transforms (wae_selftest_conv_fft)
void launch_oscillator(const OscInst* d, int n, ChunkInfo ci, cudaStream_t s);
void launch_constant(const ConstInst* d, int n, ChunkInfo ci, cudaStream_t s);
void launch_buffer_source(const AbsnInst* d, int n, ChunkInfo ci, cudaStream_t s);
void launch_buffer_source_slow(const AbsnSlowInst* d, int n, ChunkInfo ci, cudaStream_t s);
void launch_buffer_source_bound(const AbsnBoundInst* d, int n, ChunkInfo ci, cudaStream_t s);  // k_buffer_source_slow<true>
void launch_mix(const MixInst* d, const MixEdge* e, int n, ChunkInfo ci, cudaStream_t s, int max_edges);  // max_edges: widest port of the stage (host)
void launch_mix_dyn(const MixDynInst* d, const MixEdge* e, int n, ChunkInfo ci, cudaStream_t s);
void launch_meta(const MetaInst* d, int n, ChunkInfo ci, cudaStream_t s);
void launch_biquad_serial(const BiquadInst* d, int n, int max_ch, ChunkInfo ci, cudaStream_t s);
void launch_chain(int variant, const ChainInst* d, const ScanCoef* c, int n, int max_ch, ChunkInfo ci, cudaStream_t s, ChainAux aux);
// voices summed in edge order inside one kernel (k_voice_sum); nb = biquads per voice (0 / 1).  aux: ticket, progress counters
// [n_groups][aux.slab_stride tiles], state hand-off [voices][2][4]
void launch_voice_sum(int nb, const ChainInst* d, const ScanCoef* c, const VoiceGroup* g, int n_groups, ChunkInfo ci, cudaStream_t s, ChainAux aux);
int voice_sum_slots();  // resident CTAs of k_voice_sum on the machine (host: is a launch big enough to be worth it?)
void set_num_sms(int n);  // SM count of the engine's device (launch geometry; 132 on an H100 SXM until an engine sets it)
void chain_plan_slabs(int n, int max_ch, int nf, int nb, int* n_slabs, int* tiles_per_slab, int* pre_log2 = nullptr);  // launch geometry of k_chain (host); *pre_log2 >= 0: slabs publish their end state before they render
void chain_set_prepass(int on);            // WAE_OPT_CHAIN_PREPASS / WAE_CHAIN_PREPASS (default on)
void chain_set_tuning(int tma, int waves);  // < 0: keep (defaults: WAE_CHAIN_TMA / WAE_CHAIN_WAVES or 0 / 20)
void launch_iir(const IirInst* d, int n, int max_ch, ChunkInfo ci, cudaStream_t s);
void launch_gain(const GainInst* d, int n, ChunkInfo ci, cudaStream_t s);
void launch_shaper(const ShaperInst* d, int n, ChunkInfo ci, cudaStream_t s);
void launch_stereo_panner(const SPanInst* d, const float2* gains, int n, ChunkInfo ci, cudaStream_t s);
void launch_hrtf(const HrtfInst* d, int n, const HrtfSelInst* sel, int n_sel, int max_taps, ChunkInfo ci, cudaStream_t s);
void launch_buffer_source_serial(const AbsnSerialInst* d, int n, ChunkInfo ci, cudaStream_t s);
void launch_shaper_os(const ShaperOsInst* d, int n, int max_ch, ChunkInfo ci, cudaStream_t s);
void launch_panner_dyn(const PanDynInst* d, int n, ChunkInfo ci, cudaStream_t s);
void launch_panner_eq(const PanInst* d, int n, ChunkInfo ci, cudaStream_t s);
void launch_route(const RouteInst* d, int n, ChunkInfo ci, cudaStream_t s);
void launch_delay_read(const DelayInst* d, int n, ChunkInfo ci, cudaStream_t s);
void launch_delay_mono(const DelayInst* d, int n, ChunkInfo ci, cudaStream_t s);
void launch_ring_write(const DelayInst* d, int n, ChunkInfo ci, cudaStream_t s);
void launch_osc_arate(const OscArInst* d, int n, ChunkInfo ci, cudaStream_t s);
void launch_biquad_arate(const BiquadArInst* d, int n, int max_ch, ChunkInfo ci, cudaStream_t s);
void launch_analyser_fft(const float* ring, uint32_t write_index, int fft_size, float smoothing, float* last_fft, float* out_db, cudaStream_t s);
void launch_resample_linear(const float* in, int64_t len, float* out, int64_t target_len, cudaStream_t s);
void launch_param(const ParamInst* d, int n, ChunkInfo ci, cudaStream_t s, int mode);  // 0: k_param, 1: k_param_parallel, 2: k_param_spec
// ro != nullptr: the instances' reduction read-outs (wae_compressor_set_readouts), parallel to d
void launch_compressor(const CompInst* d, const CompReadoutInst* ro, int n, ChunkInfo ci, cudaStream_t s);
void launch_analyser(const AnalyserInst* d, int n, ChunkInfo ci, cudaStream_t s);
// declared analyser read-outs (wae_analyser_set_readouts): `d` = the chunk's n records, max_fft / max_bins = the largest of the stage
void launch_readout_fft(const ReadoutInst* d, int n, int max_fft, ChunkInfo ci, cudaStream_t s);
void launch_readout_time(const ReadoutInst* d, int n, int max_fft, ChunkInfo ci, cudaStream_t s);
void launch_readout_smooth(const ReadoutSmoothInst* d, int n, int max_bins, ChunkInfo ci, cudaStream_t s);
void launch_conv_fft_in(const ConvInput* d, int n, ChunkInfo ci, cudaStream_t s);
void launch_conv_mac_ifft(const ConvPath* p, const ConvInput* in, int n, ChunkInfo ci, cudaStream_t s);
void launch_conv_compact(const ConvCmpInst* d, int n, ChunkInfo ci, cudaStream_t s);
// one launch for all items of a bind call; max_vec = the largest slot stride / 4, max_ch = the most channels of an item
void launch_bind_sources(const BindItem* d, int n, int64_t max_vec, int max_ch, cudaStream_t s);
// a bind of n param values into their slots (k_bind_params), then every patch entry of the batch re-derived from the slots (k_derive_params)
void launch_bind_params(const ParamBindItem* d, int n, const ParamSlotInfo* info, float* values, const ParamPatch* patches, int n_patches,
                        cudaStream_t s);
// after a param bind, the n spatial entries of the batch re-derived from the slots (k_derive_spatial); then the blended pair of each
// SPATIAL_RESP entry (k_spatial_blend) and its spectra (k_resp_fft over `resp`, one item per such entry); max_* over those entries
void launch_derive_spatial(const SpatialPatch* patches, int n, const float* values, const RespBindItem* resp, int n_resp, int max_taps,
                           int max_S, cudaStream_t s);
// a bind of n convolver responses: the power of the normalising items (k_resp_power, when any_normalize), the trimmed lengths
// (k_resp_trim), the spectra (k_resp_fft); max_* over the items
void launch_bind_responses(RespBindItem* d, int n, bool any_normalize, int64_t max_len, int max_S, int max_ch, cudaStream_t s);
// a bind of n WaveShaper curves (k_bind_curves): copy, can_propagate_silence, the patch entries it decides
void launch_bind_curves(const CurveBindItem* d, int n, cudaStream_t s);
// a bind of n periodic waves: the wavetables (k_bind_waves, max_len = the longest), then their normalisation (k_wave_normalize, when
// any_normalize)
void launch_bind_waves(const WaveBindItem* d, int n, int max_len, bool any_normalize, cudaStream_t s);
// a bind of n IIR coefficient sets (k_bind_iir): normalised by feedback[0], written to every patch entry of each item
void launch_bind_iir(const IirBindItem* d, int n, cudaStream_t s);
// a bind of n param value curves (k_bind_value_curves): each item's values copied bit for bit, max_len = the longest
void launch_bind_value_curves(const ValueCurveBindItem* d, int n, int64_t max_len, cudaStream_t s);
// a bind of n schedules (start, [stop], [offset], [duration]; k_bind_schedules, one thread per item): clamped, then every patch entry of
// each item re-derived
void launch_bind_schedules(const SchedBindItem* d, int n, cudaStream_t s);
// a bind of n loop-point pairs (k_bind_loops, one thread per item): clamped, then every patch entry of each item written
void launch_bind_loops(const LoopBindItem* d, int n, cudaStream_t s);
// the playhead tables of the n looping bound slow-track records of a batch (k_absn_loop_schedule, one thread per record); *overflow is
// set when a walk needs more segments than its table holds
void launch_absn_loop_schedule(const LoopWalk* d, int n, int* overflow, cudaStream_t s);
// a bind of the output (k_bind_output, one thread per entry): base + off into each of the n output entries of a batch
void launch_bind_output(const OutPatch* d, int n, float* base, cudaStream_t s);
// the reference half of a bind of sources (k_bind_source_refs, one thread per row): each of the n rows writes its pointer and stride into
// its entry of `entries`
void launch_bind_source_refs(const SrcRefBindItem* d, int n, const SrcRefPatch* entries, cudaStream_t s);
void launch_conv_ir_fft(const float* ir, int64_t ir_len, int64_t ir_stride, float2* h, int S, int channels, cudaStream_t s);

}  // namespace wae
