// Hand-written sm_90a kernels of the render-quantum engine, one per node renderer of SURVEY §8(a).
//
// All kernels are HBM/latency-bound streaming or scan kernels (no dense contraction -> no tensor cores):
// coalesced planar f32 loads/stores, f64 only where the reference computes in f64 (biquad / IIR state,
// oscillator phase), grids sized over (time tiles x node instances).  Each kernel cites the reference
// renderer whose arithmetic it reproduces; parity target is 1e-5 absolute on f32 PCM.
#include "wae_kernels.h"
#include "wae_param_core.h"
#include "wae_param_walk.h"
#include "../../include/wae.h"

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <vector>
#include <type_traits>
#include <cuda_runtime.h>
#include <math_constants.h>

namespace wae {

#define DEVI __device__ __forceinline__

DEVI float* chan(const BufRef& b, int c, const ChunkInfo& ci) { return b.p + (size_t)c * b.stride + (b.absolute ? ci.f0 : ci.sub); }

// ---- dynamic layout tracks (BufRef::meta, wae_device.h) ----------------------------------------------------------------
DEVI int meta_qi(const ChunkInfo& ci, int n) { return (ci.sub + n) >> 7; }  // quantum slot of chunk frame n inside the chunk's arena
DEVI bool buf_silent(const BufRef& b, int rows, int qi) {                   // AudioRenderQuantum::is_silent (quantum.rs:257-259)
    if (!b.meta) return false;
    for (int r = 0; r < rows; r++)
        if (!(b.meta[(size_t)r * b.meta_stride + qi] & WAE_META_SILENT)) return false;
    return true;
}
DEVI int buf_count(const BufRef& b, int ch_static, int qi) { return b.meta ? (int)(b.meta[qi] & 0x3f) : ch_static; }
DEVI void meta_put(const BufRef& b, int row, int qi, int count, bool silent) {
    b.meta[(size_t)row * b.meta_stride + qi] = (uint8_t)((count & 0x3f) | (silent ? WAE_META_SILENT : 0));
}
DEVI void meta_put_all(const BufRef& b, int rows, int qi, int count, bool silent) {
    for (int r = 0; r < rows; r++) meta_put(b, r, qi, count, silent);
}

// ---------------------------------------------------------------------------------------------------------
// Oscillator — OscillatorRenderer::process + generate_* (src/node/oscillator.rs:364-676), constant
// frequency/detune.  The reference advances phase by repeated `phase += incr` (f64); here phase is the
// closed form frac(phase0 + (n - n_first) * incr), which differs by < 1e-10 over minutes of audio.
// ---------------------------------------------------------------------------------------------------------
DEVI double osc_poly_blep(double t, double dt) {  // oscillator.rs:645-659 (release build: enabled)
    if (t < dt) {
        t /= dt;
        return t + t - t * t - 1.0;
    } else if (t > 1.0 - dt) {
        t = (t - 1.0) / dt;
        return fma(t, t, t) + t + 1.0;
    }
    return 0.0;
}
// same with a precomputed 1/dt (constant-frequency oscillators): t * (1/dt) differs from t / dt by <= 1 ulp of f64
DEVI double osc_poly_blep_r(double t, double dt, double inv_dt) {
    if (t < dt) {
        t *= inv_dt;
        return t + t - t * t - 1.0;
    } else if (t > 1.0 - dt) {
        t = (t - 1.0) * inv_dt;
        return fma(t, t, t) + t + 1.0;
    }
    return 0.0;
}
// the rare frames inside a polyBLEP window, out of line so that the common path of the fused chain stays small
__device__ __noinline__ float osc_saw_blep(unsigned long long p2, double inc, double inv) {
    const double t = (double)p2 * 5.42101086242752217e-20;  // 2^-64
    return (float)(2.0 * t - 1.0 - osc_poly_blep_r(t, inc, inv));
}
__device__ __noinline__ float osc_square_blep(unsigned long long ph, unsigned long long p2, double inc, double inv) {
    const double t = (double)ph * 5.42101086242752217e-20, t2 = (double)p2 * 5.42101086242752217e-20;
    // the half-cycle sign comes from the fixed-point phase itself: `t` may round to exactly 0.5 (or 1.0) while p2 is still
    // just below the wrap, and deciding the sign from the rounded value would pair +-1 with the wrong polyBLEP branch
    return (float)(((long long)ph >= 0 ? 1.0 : -1.0) + osc_poly_blep_r(t, inc, inv) - osc_poly_blep_r(t2, inc, inv));
}
DEVI double osc_unroll(double p) { return p >= 1. ? p - 1. : (p < 0. ? p + 1. : p); }

DEVI float osc_sample(const OscInst& o, double phase, double incr) {
    switch (o.type) {
        case 0:
        case 4: {  // sine (:571-585) / custom (:622-637): table lookup + lerp with fmaf
            double position = phase * (double)o.table_len;
            double floored = floor(position);
            int prev = (int)floored;
            if (prev >= o.table_len) prev = o.table_len - 1;  // guards phase == 1-ulp rounding up
            int next = prev + 1;
            if (next == o.table_len) next = 0;
            float k = (float)(position - floored);
            return fmaf(o.table[prev], 1.f - k, o.table[next] * k);  // generic loads: the table may sit in shared memory
        }
        case 2: {  // sawtooth, :588-595
            double ph = osc_unroll(phase + 0.5);
            double s = 2.0 * ph - 1.0;
            s -= osc_poly_blep(ph, incr);
            return (float)s;
        }
        case 1: {  // square, :598-606
            double s = phase < 0.5 ? 1.0 : -1.0;
            s += osc_poly_blep(phase, incr);
            s -= osc_poly_blep(osc_unroll(phase + 0.5), incr);
            return (float)s;
        }
        default: {  // triangle, :609-619
            double s = -4. * phase + 2.;
            if (s > 1.)
                s = 2. - s;
            else if (s < -1.)
                s = -2. - s;
            return (float)s;
        }
    }
}

DEVI double osc_phase_at(const OscInst& o, int64_t n) {
    double d = (double)(n - o.n_first);
    double p = fma(d, o.incr, o.phase0);
    p -= floor(p);
    if (p >= 1.) p = 0.;
    return p;
}

__global__ void __launch_bounds__(256) k_oscillator(const OscInst* __restrict__ insts, int n_inst, ChunkInfo ci) {
    for (int ii = blockIdx.y; ii < n_inst; ii += gridDim.y) {
        const OscInst o = insts[ii];
        float* out = chan(o.out, 0, ci);
        int n0 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
        if (n0 >= ci.nf) continue;
        float v[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {
            int64_t n = ci.f0 + n0 + j;
            float s = 0.f;
            if (n >= o.n_first && n < o.n_stop && !o.outside_nyquist) s = osc_sample(o, osc_phase_at(o, n), o.incr);
            v[j] = s;
        }
        *reinterpret_cast<float4*>(out + n0) = make_float4(v[0], v[1], v[2], v[3]);
    }
}

// ConstantSourceRenderer (src/node/constant_source.rs:190-262), constant offset
__global__ void __launch_bounds__(256) k_constant(const ConstInst* __restrict__ insts, int n_inst, ChunkInfo ci) {
    for (int ii = blockIdx.y; ii < n_inst; ii += gridDim.y) {
        const ConstInst o = insts[ii];
        float* out = chan(o.out, 0, ci);
        int n0 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
        if (n0 >= ci.nf) continue;
        float v[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {
            int64_t n = ci.f0 + n0 + j;
            v[j] = (n >= o.n_first && n < o.n_stop) ? (o.track.p ? chan(o.track, 0, ci)[n0 + j] : o.value) : 0.f;
        }
        *reinterpret_cast<float4*>(out + n0) = make_float4(v[0], v[1], v[2], v[3]);
    }
}

// AudioBufferSourceRenderer fast track (src/node/audio_buffer_source.rs:554-624): aligned copy, optional loop
__global__ void __launch_bounds__(256) k_buffer_source(const AbsnInst* __restrict__ insts, int n_inst, ChunkInfo ci) {
    for (int ii = blockIdx.y; ii < n_inst; ii += gridDim.y) {
        const AbsnInst o = insts[ii];
        int n0 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
        if (n0 >= ci.nf) continue;
        for (int c = 0; c < o.ch; c++) {
            float* out = chan(o.out, c, ci);
            const float* src = o.buf + (size_t)c * o.buf_stride;
            float v[4];
#pragma unroll
            for (int j = 0; j < 4; j++) {
                int64_t n = ci.f0 + n0 + j;
                float s = 0.f;
                if (n >= o.n_start && n < o.n_stop) {
                    int64_t idx = n - o.n_start + o.buf_offset;
                    if (o.loop)
                        s = __ldg(src + (idx % o.buf_len));
                    else if (idx < o.buf_len)
                        s = __ldg(src + idx);
                }
                v[j] = s;
            }
            *reinterpret_cast<float4*>(out + n0) = make_float4(v[0], v[1], v[2], v[3]);
        }
    }
}

// AudioBufferSourceRenderer slow track (src/node/audio_buffer_source.rs:625-823) for a constant positive playback
// rate.  The reference advances `buffer_time += dt * rate` per frame; here the playhead of frame n is the closed form
// offset0 + (n - n_first) * step (loop wrap applied arithmetically), which differs by rounding only; the linear
// interpolation is continuous across frame boundaries, so the PCM agrees to ~1e-7.
DEVI bool almost_eq(double a, double b) {  // `almost` crate 0.2: absolute or relative sqrt(eps)
    if (a == b) return true;
    const double tol = 1.4901161193847656e-8;
    double d = fabs(b - a);
    if (d <= tol) return true;
    return d <= fmax(fabs(a), fabs(b)) * tol;
}
// chunk frame n of a slow-track source
DEVI void absn_slow_frame(const AbsnSlowInst& o, int n, const ChunkInfo& ci) {
    const int64_t na = ci.f0 + n;
    bool play = na >= o.n_first && na < o.n_stop;
    int64_t pfi = 0;
    double k = 0.;
    if (play) {
        const double m = (double)(na - o.n_first);
        double elapsed = fma(m, fabs(o.step), o.elapsed0);
        if (almost_eq(elapsed, o.duration)) elapsed = o.duration;
        if (elapsed >= o.duration) play = false;
        // segment of the playhead schedule that contains this frame (binary search), then the linear playhead
        int lo = 0, hi = o.n_seg - 1;
        while (lo < hi) {
            int mid = (lo + hi + 1) >> 1;
            if (o.seg_n[mid] <= na) lo = mid;
            else hi = mid - 1;
        }
        double bt = fma((double)(na - o.seg_n[lo]), o.step, o.seg_bt[lo]);
        if (fabs(bt) < 1.4901161193847656e-8) bt = 0.;
        if (play && bt >= 0. && bt < o.buffer_duration) {
            double playhead = bt * o.pos_scale;
            double fl = floor(playhead);
            pfi = (int64_t)fl;
            k = playhead - fl;
            if (pfi >= o.buf_len) play = false;
        } else {
            play = false;
        }
    }
    for (int c = 0; c < o.ch; c++) {
        float v = 0.f;
        if (play) {
            const float* b = o.buf + (size_t)c * o.buf_stride;
            double prev = (double)__ldg(b + pfi), next;
            if (pfi + 1 < o.buf_len) {
                next = (double)__ldg(b + pfi + 1);
            } else if (o.loop) {  // :788-800 (rate >= 0): first frame at / after the loop start
                double sp = o.loop_start * o.sample_rate;
                int64_t si = floor(sp) == sp ? (int64_t)sp : (int64_t)sp + 1;
                next = (double)__ldg(b + (si < o.buf_len ? si : o.buf_len - 1));
            } else if (almost_eq(k, 1.) || pfi == 0) {
                next = 0.;
            } else {
                next = 2. * prev - (double)__ldg(b + pfi - 1);  // extrapolate past the end (:815-819)
            }
            v = (float)fma(1. - k, prev, k * next);
        }
        chan(o.out, c, ci)[n] = v;
    }
}

// A source whose playback rate is bound from device memory, ABSN_BOUND_TILES tiles of 256 chunk frames from frame n0 (called by every
// thread of the CTA).  Thread 0 derives the instance's constants from the bound rate with the planner's expressions: the fast track's 1:1
// copy where the planner would have taken it (k_buffer_source), else the slow track over one playhead segment.  A gated output also gets
// its layout track here, silent outside the frames that play, as k_meta's META_SOURCE writes it for a planned source.
constexpr int ABSN_BOUND_TILES = 8;
DEVI void absn_bound_tiles(const AbsnBoundInst& r, int n0, const ChunkInfo& ci) {
    __shared__ AbsnSlowInst s_o;
    __shared__ int64_t s_seg_n, s_first, s_end;
    __shared__ double s_seg_bt;
    __shared__ int s_fast;
    __syncthreads();  // (the CTA's previous instance is done with them)
    if (threadIdx.x == 0) {
        AbsnSlowInst o = r.s;
        const double computed_rate = (double)r.rate * exp2((double)r.detune / 1200.);
        const AbsnSlowDerived d = absn_slow_derive(r.dt, computed_rate, r.offset, r.start_delta, o.buffer_duration, o.duration, o.loop != 0,
                                                   o.loop_end, o.n_first, o.n_stop);
        o.step = d.step;
        o.offset0 = d.offset0;
        o.elapsed0 = d.elapsed0;
        if (!o.loop) {  // (a looping record reads the table k_absn_loop_schedule derived from the same values)
            o.n_seg = 1;
            o.seg_n = &s_seg_n;
            o.seg_bt = &s_seg_bt;
            s_seg_n = o.n_first;
            s_seg_bt = d.offset0;
        }
        const bool fast = r.fast_ok && computed_rate == 1.;
        s_fast = fast;
        s_first = fast ? r.n_start : o.n_first;
        s_end = fast ? r.fast_end : d.n_end;
        s_o = o;
    }
    __syncthreads();
    const AbsnSlowInst o = s_o;
    const bool fast = s_fast;
    for (int t = 0; t < ABSN_BOUND_TILES; t++) {
        const int n = n0 + t * 256 + (int)threadIdx.x;
        if (n >= ci.nf) return;
        const int64_t na = ci.f0 + n;
        if (fast) {
            for (int c = 0; c < o.ch; c++) {
                float v = 0.f;
                if (na >= r.n_start && na < r.fast_end && na - r.n_start < o.buf_len) v = __ldg(o.buf + (size_t)c * o.buf_stride + (na - r.n_start));
                chan(o.out, c, ci)[n] = v;
            }
        } else {
            absn_slow_frame(o, n, ci);
        }
        if (o.out.meta && (n & 127) == 0) {
            const bool silent = s_end <= na || s_first >= na + 128;
            meta_put_all(o.out, o.ch, meta_qi(ci, n), silent ? 1 : o.ch, silent);
        }
    }
}

// One thread per frame (BOUND: per frame of each of ABSN_BOUND_TILES tiles).  BOUND: the records are AbsnBoundInst (a playback rate
// bound from device memory), else AbsnSlowInst.
template <bool BOUND>
struct AbsnSlowRecord {
    using T = AbsnSlowInst;
};
template <>
struct AbsnSlowRecord<true> {
    using T = AbsnBoundInst;
};
template <bool BOUND>
__global__ void __launch_bounds__(256) k_buffer_source_slow(const typename AbsnSlowRecord<BOUND>::T* __restrict__ insts, int n_inst, ChunkInfo ci) {
    for (int ii = blockIdx.y; ii < n_inst; ii += gridDim.y) {
        if constexpr (BOUND) {
            absn_bound_tiles(insts[ii], blockIdx.x * ABSN_BOUND_TILES * 256, ci);
        } else {
            const int n = blockIdx.x * blockDim.x + threadIdx.x;
            const AbsnSlowInst o = insts[ii];
            if (n >= ci.nf) continue;
            absn_slow_frame(o, n, ci);
        }
    }
}

// AudioBufferSourceRenderer::process, general form (audio_buffer_source.rs:422-845): one warp per instance, lane 0 runs
// the renderer's per-frame bookkeeping for a quantum (exactly the reference's sequence of f64 operations), then the 32
// lanes produce the 128 samples of every channel.
constexpr int ABSN_SERIAL_WARPS = 4;
__global__ void __launch_bounds__(32 * ABSN_SERIAL_WARPS) k_buffer_source_serial(const AbsnSerialInst* __restrict__ insts, int n_inst, ChunkInfo ci) {
    __shared__ long long s_idx[ABSN_SERIAL_WARPS][128];  // frame of the buffer to read, -1: silence
    __shared__ double s_k[ABSN_SERIAL_WARPS][128];      // interpolation weight, < 0: plain copy (fast track)
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ii = blockIdx.x * ABSN_SERIAL_WARPS + warp;
    if (ii >= n_inst) return;
    const AbsnSerialInst& o = insts[ii];
    long long* idx = s_idx[warp];
    double* kk = s_k[warp];
    AbsnSerialState st;
    if (lane == 0) {
        st = *o.state;
        if (!st.inited) st = AbsnSerialState{o.start_time, o.offset, 0., 0., 0, 0, 0, 0, 1, 0};  // first quantum of this source in this run
    }
    const double sample_rate = o.sample_rate, dt = 1. / sample_rate, block_duration = dt * 128.;
    const double buffer_duration = o.buffer_duration;
    const double sampling_ratio = o.buffer_sample_rate / sample_rate;
    const bool is_looping = o.loop != 0;
    for (int q0 = 0; q0 < ci.nf; q0 += 128) {
        float playback_rate_f = o.rate_track.p ? chan(o.rate_track, 0, ci)[q0] : o.rate;
        double actual_loop_start = 0., actual_loop_end = 0.;
        if (is_looping) {  // :627-636 (only read by the slow track)
            if (o.loop_start >= 0. && o.loop_end > 0. && o.loop_start < o.loop_end) {
                actual_loop_start = o.loop_start;
                actual_loop_end = o.loop_end;
            } else {
                actual_loop_end = buffer_duration;
            }
        }
        if (lane == 0) {
            for (int i = 0; i < 128; i++) idx[i] = -1;
            const double block_time = (double)(ci.f0 + q0) / sample_rate;
            const double next_block_time = block_time + block_duration;
            bool run = !st.ended;
            if (run && st.start_time >= next_block_time) {  // :470-481
                if (o.stop_time <= next_block_time) st.ended = 1;
                run = false;
            }
            if (run) {
                const double detune_v = (double)(o.detune_track.p ? chan(o.detune_track, 0, ci)[q0] : o.detune);
                const double computed_playback_rate = (double)playback_rate_f * exp2(detune_v / 1200.);
                double buffer_time = st.buffer_time;
                if (!st.started && st.start_time < block_time) st.start_time = block_time;  // :519-523
                if (st.start_time == block_time && st.offset == 0.) st.is_aligned = 1;
                if (sampling_ratio != 1. || computed_playback_rate != 1.) st.is_aligned = 0;
                if (o.loop_start != 0. || o.loop_end != buffer_duration) st.is_aligned = 0;
                if (buffer_time + block_duration > o.duration || block_time + block_duration > o.stop_time) st.is_aligned = 0;
                if (st.is_aligned) {  // fast track (:554-624)
                    if (st.start_time == block_time) st.started = 1;
                    long long start_index = llround(buffer_time * sample_rate);
                    if (buffer_time + block_duration > buffer_duration) {
                        const long long end_index = o.buf_len;
                        bool has_loop_point = false;
                        int loop_point_index = 0;
                        long long off = 0;
                        for (int i = 0; i < 128; i++) {
                            long long bi = start_index + i - off;
                            if (bi >= end_index) {
                                if (is_looping) {
                                    has_loop_point = true;
                                    loop_point_index = i;
                                    start_index = 0;
                                    off = i;
                                    bi = 0;
                                } else {
                                    bi = -1;
                                }
                            }
                            idx[i] = bi;
                            kk[i] = -1.;
                        }
                        if (has_loop_point)
                            buffer_time = fmod((double)(128 - loop_point_index) / sample_rate, buffer_duration);
                        else
                            buffer_time += block_duration;
                    } else {
                        for (int i = 0; i < 128; i++) {
                            idx[i] = start_index + i;
                            kk[i] = -1.;
                        }
                        buffer_time += block_duration;
                    }
                    st.buffer_time_elapsed += block_duration;
                } else {  // slow track (:625-823)
                    if (!is_looping) st.entered_loop = 0;
                    for (int i = 0; i < 128; i++) {
                        const double current_time = block_time + (double)i * dt;
                        if (!st.started && almost_eq(current_time, st.start_time)) st.start_time = current_time;
                        if (almost_eq(st.buffer_time_elapsed, o.duration)) st.buffer_time_elapsed = o.duration;
                        if (current_time < st.start_time || current_time >= o.stop_time || st.buffer_time_elapsed >= o.duration) continue;
                        if (!st.started) {
                            const double delta = current_time - st.start_time;
                            st.offset += delta * computed_playback_rate;
                            st.offset = fmin(fmax(st.offset, 0.), buffer_duration);
                            if (is_looping && computed_playback_rate >= 0. && st.offset > actual_loop_end) st.offset = actual_loop_end;
                            if (is_looping && computed_playback_rate < 0. && st.offset < actual_loop_start) st.offset = actual_loop_start;
                            buffer_time = st.offset;
                            st.buffer_time_elapsed = fabs(delta * computed_playback_rate);
                            st.started = 1;
                        }
                        if (is_looping) {
                            if (almost_eq(buffer_time, actual_loop_end)) buffer_time = actual_loop_end;
                            if (almost_eq(buffer_time, actual_loop_start)) buffer_time = actual_loop_start;
                            if (!st.entered_loop) {
                                if (st.offset < actual_loop_end && buffer_time >= actual_loop_start) st.entered_loop = 1;
                                if (st.offset >= actual_loop_end && buffer_time < actual_loop_end) st.entered_loop = 1;
                            }
                            if (st.entered_loop) {
                                while (buffer_time >= actual_loop_end) buffer_time -= actual_loop_end - actual_loop_start;
                                while (buffer_time < actual_loop_start) buffer_time += actual_loop_end - actual_loop_start;
                            }
                        }
                        if (fabs(buffer_time) < 1.4901161193847656e-8) buffer_time = 0.;
                        if (buffer_time >= 0. && buffer_time < buffer_duration) {
                            const double position = buffer_time * sampling_ratio;
                            const double playhead = position * sample_rate;
                            const double fl = floor(playhead);
                            const long long pfi = (long long)fl;
                            if (pfi < o.buf_len) {
                                idx[i] = pfi;
                                kk[i] = playhead - fl;
                            }
                        }
                        const double time_incr = dt * computed_playback_rate;
                        buffer_time += time_incr;
                        st.buffer_time_elapsed += fabs(time_incr);
                    }
                }
                st.buffer_time = buffer_time;
                if (next_block_time >= o.stop_time || st.buffer_time_elapsed >= o.duration ||
                    (!is_looping && ((computed_playback_rate > 0. && buffer_time >= buffer_duration) || (computed_playback_rate < 0. && buffer_time < 0.))))
                    st.ended = 1;  // :826-838
            }
            if (o.out.meta) meta_put_all(o.out, o.ch, meta_qi(ci, q0), run ? o.ch : 1, !run);  // make_silent: one silent channel (:434-471)
        }
        __syncwarp();
        for (int c = 0; c < o.ch; c++) {
            const float* b = o.buf + (size_t)c * o.buf_stride;
            float* out = chan(o.out, c, ci) + q0;
            for (int i = lane; i < 128; i += 32) {
                const long long pfi = idx[i];
                float v = 0.f;
                if (pfi >= 0) {
                    const double k = kk[i];
                    if (k < 0.) {
                        v = __ldg(b + pfi);
                    } else {
                        const double prev = (double)__ldg(b + pfi);
                        double next;
                        if (pfi + 1 < o.buf_len) {
                            next = (double)__ldg(b + pfi + 1);
                        } else if (is_looping) {  // :788-800
                            long long j;
                            if (playback_rate_f >= 0.f) {
                                const double sp = actual_loop_start * sample_rate;
                                j = floor(sp) == sp ? (long long)sp : (long long)sp + 1;
                            } else {
                                j = (long long)(actual_loop_end * sample_rate);
                            }
                            next = (double)__ldg(b + (j < o.buf_len ? j : o.buf_len - 1));
                        } else if (almost_eq(k, 1.) || pfi == 0) {
                            next = 0.;
                        } else {
                            next = 2. * prev - (double)__ldg(b + pfi - 1);
                        }
                        v = (float)fma(1. - k, prev, k * next);
                    }
                }
                out[i] = v;
            }
        }
        __syncwarp();
    }
    if (lane == 0) *o.state = st;
}

// ---------------------------------------------------------------------------------------------------------
// Mixer — AudioRenderQuantum::add / mix (src/render/quantum.rs:274-569): per input port, the incoming edges
// are summed in the reference's processing order, each up/down-mixed to the port's computed channel count.
// One thread per frame; sequential f32 adds over the edges => same summation order as the reference.
// ---------------------------------------------------------------------------------------------------------
// channel c of a quantum of s channels (read through ld) mixed to dst_ch channels (quantum.rs:274-505)
template <typename LD>
DEVI float mix_channel(LD ld, int s, int dst_ch, int c, int interp) {
    if (s == dst_ch) return ld(c);
    if (interp == 1 || s > 6 || dst_ch > 6) return c < s ? ld(c) : 0.f;  // discrete: zero-fill / truncate
    const float sqrt05 = 0.70710678118654752440f;                          // (0.5f32).sqrt()
    switch (s * 16 + dst_ch) {
        case 1 * 16 + 2: return ld(0);
        case 1 * 16 + 4: return c < 2 ? ld(0) : 0.f;
        case 1 * 16 + 6: return c == 2 ? ld(0) : 0.f;
        case 2 * 16 + 4:
        case 2 * 16 + 6: return c < 2 ? ld(c) : 0.f;
        case 4 * 16 + 5: return c < 2 ? ld(c) : (c == 2 ? 0.f : ld(c - 1));
        case 4 * 16 + 6: return c < 2 ? ld(c) : (c < 4 ? 0.f : ld(c - 2));
        case 2 * 16 + 1: return 0.5f * (ld(0) + ld(1));
        case 4 * 16 + 1: return 0.25f * (ld(0) + ld(1) + ld(2) + ld(3));
        case 6 * 16 + 1: return fmaf(sqrt05, ld(0) + ld(1), fmaf(0.5f, ld(4) + ld(5), ld(2)));
        case 4 * 16 + 2: return 0.5f * (ld(c) + ld(c + 2));
        case 6 * 16 + 2: return ld(c) + sqrt05 * (ld(2) + ld(4 + c));
        case 6 * 16 + 4: return c < 2 ? ld(c) + sqrt05 * ld(2) : ld(c + 2);
        default: return c < s ? ld(c) : 0.f;
    }
}
// Where channel c of a quantum of s channels mixed to dst_ch channels comes from (quantum.rs:292-502): the channel it moves or copies
// (>= 0), the silent channel the mix pushes (-1), or a sum it computes (-2).  AudioRenderQuantumChannel::add (quantum.rs:114-120) skips a
// silent channel instead of adding its zeros and takes the other one as it is onto a silent one, so a -0.0 keeps the sign an added +0.0
// would take from it.
DEVI int mix_source(int s, int dst_ch, int c, int interp) {
    if (s == dst_ch) return c;
    if (interp == 1 || s > 6 || dst_ch > 6) return c < s ? c : -1;
    switch (s * 16 + dst_ch) {
        case 1 * 16 + 2: return 0;
        case 1 * 16 + 4: return c < 2 ? 0 : -1;
        case 1 * 16 + 6: return c == 2 ? 0 : -1;
        case 2 * 16 + 4:
        case 2 * 16 + 6: return c < 2 ? c : -1;
        case 4 * 16 + 5: return c < 2 ? c : (c == 2 ? -1 : c - 1);
        case 4 * 16 + 6: return c < 2 ? c : (c < 4 ? -1 : c - 2);
        case 2 * 16 + 1: case 4 * 16 + 1: case 6 * 16 + 1: case 4 * 16 + 2: case 6 * 16 + 2: return -2;
        case 6 * 16 + 4: return c < 2 ? -2 : c + 2;
        default: return c < s ? c : -1;
    }
}
DEVI bool mix_is_silence(int s, int dst_ch, int c, int interp) { return mix_source(s, dst_ch, c, interp) == -1; }
DEVI float mixed_sample(const MixEdge& e, int dst_ch, int c, int interp, int n, const ChunkInfo& ci) {
    return mix_channel([&](int ch) { return chan(e.src, ch, ci)[n]; }, e.src_ch, dst_ch, c, interp);
}

// Mixer with per-quantum layouts (MixDynInst): AudioRenderQuantum::add (quantum.rs:532-569) folded over the edges in processing
// order.  Every add first brings the running sum to computedNumberOfChannels(max(sum's count, edge's count)) — so with three or more
// layouts the intermediate counts matter (mono, then stereo, then 5.1: 1 -> 2 -> 6, the mono lands in L / R, not in C) — then mixes the
// edge to that count and adds channel by channel; silent edges only take part in the count.  One thread per frame.
// up to two channels everywhere (the usual case): four frames per thread, the running sum in two float4, the layout bytes read once per
// four frames.  Same fold, same order of additions as the general path below.
DEVI void mix_dyn_stereo4(const MixDynInst& m, const MixEdge* __restrict__ edges, int n0, const ChunkInfo& ci) {
    const int qi = meta_qi(ci, n0);
    float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f), a1 = a0;
    int cnt = 1;
    bool silent = true;
    bool held1 = false;  // channel 1 of the running sum is not the silent channel (a discrete 1 -> 2 mix pushes silence: mix_source)
    const bool speakers = m.interp == 0;
    for (int e = 0; e < m.n_edges; e++) {
        const MixEdge& ed = edges[m.edge_offset + e];
        const int ce = buf_count(ed.src, ed.src_ch, qi);
        const bool se = buf_silent(ed.src, ed.src_ch, qi);
        const int mx = cnt > ce ? cnt : ce;
        const int nw = m.mode == WAE_COUNT_MODE_MAX ? mx : (m.mode == WAE_COUNT_MODE_EXPLICIT ? m.cfg_count : (mx < m.cfg_count ? mx : m.cfg_count));
        if (!silent && nw != cnt) {  // self.mix(new_channels): 1 -> 2 copy (speakers) / zero-fill (discrete); 2 -> 1 half sum / truncate
            if (nw == 2) {
                a1 = speakers ? a0 : make_float4(0.f, 0.f, 0.f, 0.f);
                held1 = speakers;
            } else if (speakers) {
                a0 = make_float4(0.5f * (a0.x + a1.x), 0.5f * (a0.y + a1.y), 0.5f * (a0.z + a1.z), 0.5f * (a0.w + a1.w));
            }
        }
        cnt = nw;
        if (!se) {
            const float4 v0 = *reinterpret_cast<const float4*>(chan(ed.src, 0, ci) + n0);
            float4 v1 = v0;
            if (ce == 2) v1 = *reinterpret_cast<const float4*>(chan(ed.src, 1, ci) + n0);
            float4 x0 = v0, x1 = v1;  // the edge mixed to nw channels
            if (nw == 1 && ce == 2 && speakers) x0 = make_float4(0.5f * (v0.x + v1.x), 0.5f * (v0.y + v1.y), 0.5f * (v0.z + v1.z), 0.5f * (v0.w + v1.w));
            const bool x1_silence = nw == 2 && ce == 1 && !speakers;
            if (silent) {
                a0 = x0;
            } else {
                a0.x += x0.x; a0.y += x0.y; a0.z += x0.z; a0.w += x0.w;
            }
            if (nw == 2 && !x1_silence) {
                if (silent || !held1) a1 = x1;
                else { a1.x += x1.x; a1.y += x1.y; a1.z += x1.z; a1.w += x1.w; }
                held1 = true;
            } else if (silent) {
                a1 = make_float4(0.f, 0.f, 0.f, 0.f);
            }
            silent = false;
        }
    }
    if ((n0 & 127) == 0 && m.out.meta) meta_put_all(m.out, m.out_ch, qi, cnt, silent);
    if (silent) a0 = a1 = make_float4(0.f, 0.f, 0.f, 0.f);
    else if (cnt == 1) a1 = speakers ? a0 : make_float4(0.f, 0.f, 0.f, 0.f);  // canonical fill of the second static channel
    for (int c = 0; c < m.out_ch; c++) {
        const float4 v = c == 0 ? a0 : a1;
        float* out = chan(m.out, c, ci) + n0;
        if ((reinterpret_cast<uintptr_t>(out) & 15) == 0 && (m.limit < 0 || ci.f0 + n0 + 4 <= m.limit)) {
            *reinterpret_cast<float4*>(out) = v;
        } else {
            const float w[4] = {v.x, v.y, v.z, v.w};
            for (int j = 0; j < 4; j++)
                if (m.limit < 0 || ci.f0 + n0 + j < m.limit) out[j] = w[j];
        }
    }
}
__global__ void __launch_bounds__(128) k_mix_dyn(const MixDynInst* __restrict__ insts, const MixEdge* __restrict__ edges, int n_inst, ChunkInfo ci) {
    for (int ii = blockIdx.y; ii < n_inst; ii += gridDim.y) {
        const MixDynInst m = insts[ii];
        if (m.stereo4) {  // (instance-uniform)
            const int n0 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
            if (n0 < ci.nf) mix_dyn_stereo4(m, edges, n0, ci);
            continue;
        }
        for (int sub = 0; sub < 4; sub++) {  // (the grid is sized for four frames per thread)
        const int n = (blockIdx.x * blockDim.x + threadIdx.x) * 4 + sub;
        if (n >= ci.nf) continue;
        const int qi = meta_qi(ci, n);
        float acc[32], tmp[32];
        uint32_t held = 0;  // bit c: channel c of the running sum is not the silent channel
        int cnt = 1;
        bool silent = true;
        for (int e = 0; e < m.n_edges; e++) {
            const MixEdge ed = edges[m.edge_offset + e];
            const int ce = buf_count(ed.src, ed.src_ch, qi);
            const bool se = buf_silent(ed.src, ed.src_ch, qi);
            const int mx = cnt > ce ? cnt : ce;
            const int nw = m.mode == WAE_COUNT_MODE_MAX ? mx : (m.mode == WAE_COUNT_MODE_EXPLICIT ? m.cfg_count : (mx < m.cfg_count ? mx : m.cfg_count));
            if (!silent && nw != cnt) {  // self.mix(new_channels, interpretation)
                uint32_t h = 0;
                for (int c = 0; c < nw; c++) {
                    tmp[c] = mix_channel([&](int ch) { return acc[ch]; }, cnt, nw, c, m.interp);
                    const int from = mix_source(cnt, nw, c, m.interp);  // a moved channel stays what it was, a computed one is held
                    if (from == -2 || (from >= 0 && ((held >> from) & 1u))) h |= 1u << c;
                }
                for (int c = 0; c < nw; c++) acc[c] = tmp[c];
                held = h;
            }
            cnt = nw;
            if (!se) {
                for (int c = 0; c < nw; c++) {
                    if (mix_is_silence(ce, nw, c, m.interp)) continue;
                    const float v = mix_channel([&](int ch) { return chan(ed.src, ch, ci)[n]; }, ce, nw, c, m.interp);
                    acc[c] = (held >> c) & 1u ? acc[c] + v : v;
                    held |= 1u << c;
                }
                silent = false;
            }
        }
        for (int c = 0; c < cnt; c++)
            if (!((held >> c) & 1u)) acc[c] = 0.f;
        if ((n & 127) == 0 && m.out.meta) meta_put_all(m.out, m.out_ch, qi, cnt, silent);
        if (m.limit >= 0 && ci.f0 + n >= m.limit) continue;
        for (int c = 0; c < m.out_ch; c++) {
            float v = 0.f;
            if (!silent) v = c < cnt ? acc[c] : mix_channel([&](int ch) { return acc[ch]; }, cnt, m.out_ch, c, m.interp);  // canonical fill
            chan(m.out, c, ci)[n] = v;
        }
        }
    }
}

// Layout tracks of nodes whose PCM path does not look at the layout (MetaInst): one thread per instance walks the chunk's quanta.
__global__ void __launch_bounds__(64) k_meta(const MetaInst* __restrict__ insts, int n_inst, ChunkInfo ci) {
    const int ii = blockIdx.x * blockDim.x + threadIdx.x;
    if (ii >= n_inst) return;
    const MetaInst m = insts[ii];
    int64_t tail = m.mode == META_CONV ? *m.state : 0;
    for (int q = 0; q < ci.nf / 128; q++) {
        const int qi = meta_qi(ci, q * 128);
        const int64_t f = ci.f0 + (int64_t)q * 128;
        bool si = false;
        int ci_ = m.in_ch;
        if (m.mode != META_SOURCE && m.mode != META_MERGE && m.mode != META_CONST) {
            si = buf_silent(m.in, m.in_ch, qi);
            ci_ = buf_count(m.in, m.in_ch, qi);
        }
        int co = 1;
        bool so = true;
        switch (m.mode) {
            case META_SOURCE:
                so = m.n_stop <= f || m.n_first >= f + 128;
                co = so ? 1 : m.count;
                break;
            case META_COPY:
                so = si;
                co = ci_;
                break;
            case META_SHAPER:
                so = false;
                co = ci_;
                break;
            case META_PAN:
                so = si;
                co = si ? 1 : 2;
                break;
            case META_CONV: {
                bool out_silent = false;
                if (si) {
                    if (tail >= m.tail_len) out_silent = true;
                    else tail += 128;
                } else {
                    tail = 0;
                }
                so = out_silent;
                co = out_silent ? 1 : ((ci_ == 1 && m.aux == 1) ? 1 : 2);
                break;
            }
            case META_SPLIT:
                so = si || m.aux >= ci_;
                co = 1;
                break;
            case META_MERGE: {
                bool any = false;
                for (int k = 0; k < m.n_more; k++) any = any || !buf_silent(m.more[k], 1, qi);
                so = !any;
                co = any ? m.count : 1;
                break;
            }
            default:  // META_CONST
                so = m.aux != 0;
                co = so ? 1 : m.count;
                break;
        }
        meta_put_all(m.out, m.out_ch, qi, co, so);
    }
    if (m.mode == META_CONV) *m.state = tail;
}

// Fast path (MixInst::simple): every edge either has the port's channel count or is a mono signal up-mixed by
// copy (speakers 1 -> 2).  One thread owns 4 consecutive frames; the edge loop issues 8 independent 16-byte loads
// before the 8 dependent adds, so a 4096-edge fan-in (config C3) is bandwidth-, not latency-bound, while the f32
// summation order stays the reference's.  When all edges are mono the sum is computed once and written to every
// output channel (the reference's "all channels identical" fast path, quantum.rs:549-558).
template <int VEC>
struct MixVec;
template <>
struct MixVec<4> {
    float4 v;
    DEVI void load(const float* p) { v = *reinterpret_cast<const float4*>(p); }
    DEVI void add(const MixVec& o) { v.x += o.v.x; v.y += o.v.y; v.z += o.v.z; v.w += o.v.w; }
    DEVI void zero() { v = make_float4(0.f, 0.f, 0.f, 0.f); }
    DEVI float get(int j) const { return j == 0 ? v.x : (j == 1 ? v.y : (j == 2 ? v.z : v.w)); }
};
template <>
struct MixVec<1> {
    float v;
    DEVI void load(const float* p) { v = *p; }
    DEVI void add(const MixVec& o) { v += o.v; }
    DEVI void zero() { v = 0.f; }
    DEVI float get(int) const { return v; }
};

// The CTA first resolves the channel pointers of up to MIX_STAGE edges into shared memory (every thread of the CTA follows the same
// edges: one global read of the edge table per CTA instead of one per thread, and no pointer load in front of every sample load),
// then each thread walks them in two alternating batches: the loads of one batch are in flight while the other one is added, in edge
// order, so the f32 summation order stays the reference's.
constexpr int MIX_STAGE = 256;
template <int VEC>
struct MixBatch { static constexpr int N = VEC == 1 ? 16 : 4; };

template <int VEC, int B>
DEVI void mix_load(MixVec<VEC> (&v)[B], const float* const* src, int k, int n0) {
#pragma unroll
    for (int u = 0; u < B; u++) v[u].load(src[k + u] + n0);
}
template <int VEC, int B>
DEVI void mix_add(MixVec<VEC>& acc, const MixVec<VEC> (&v)[B], bool first) {
#pragma unroll
    for (int u = 0; u < B; u++) {
        if (u == 0 && first) acc = v[0];  // the first edge is taken as it is (a sum that starts from -0.0 keeps its sign)
        else acc.add(v[u]);
    }
}
// `cnt` edges whose pointers are in src[]; first: src[0] is the port's first edge
template <int VEC>
DEVI void mix_run(const float* const* src, int cnt, int n0, bool first, MixVec<VEC>& acc) {
    constexpr int B = MixBatch<VEC>::N;
    MixVec<VEC> a[B], b[B];
    const int nb = cnt / B;
    if (nb > 0) mix_load<VEC, B>(a, src, 0, n0);
    for (int bi = 0; bi < nb; bi += 2) {
        if (bi + 1 < nb) mix_load<VEC, B>(b, src, (bi + 1) * B, n0);
        mix_add<VEC, B>(acc, a, first && bi == 0);
        if (bi + 2 < nb) mix_load<VEC, B>(a, src, (bi + 2) * B, n0);
        if (bi + 1 < nb) mix_add<VEC, B>(acc, b, false);
    }
    for (int k = nb * B; k < cnt; k++) {
        MixVec<VEC> v;
        v.load(src[k] + n0);
        if (k == 0 && first) acc = v;
        else acc.add(v);
    }
}

// few edges: the loads of up to 8 edges are issued together, then added in edge order
template <int VEC>
DEVI void mix_direct(const MixInst& m, const MixEdge* __restrict__ edges, int c, int n0, const ChunkInfo& ci, MixVec<VEC>& acc) {
    const MixEdge* e = edges + m.edge_offset;
    int k = 0;
    for (; k + 8 <= m.n_edges; k += 8) {
        MixVec<VEC> v[8];
#pragma unroll
        for (int u = 0; u < 8; u++) v[u].load(chan(e[k + u].src, e[k + u].src_ch == 1 ? 0 : c, ci) + n0);
#pragma unroll
        for (int u = 0; u < 8; u++) {
            if (k + u == 0) acc = v[u];
            else acc.add(v[u]);
        }
    }
    for (; k < m.n_edges; k++) {
        MixVec<VEC> v;
        v.load(chan(e[k].src, e[k].src_ch == 1 ? 0 : c, ci) + n0);
        if (k == 0) acc = v;
        else acc.add(v);
    }
}

template <int VEC>
__global__ void __launch_bounds__(256) k_mix(const MixInst* __restrict__ insts, const MixEdge* __restrict__ edges, int n_inst,
                                             ChunkInfo ci) {
    __shared__ const float* s_src[MIX_STAGE];
    for (int ii = blockIdx.y; ii < n_inst; ii += gridDim.y) {  // (CTA-uniform loop: the barriers below are reached by every thread)
        const MixInst m = insts[ii];
        const int n0 = (blockIdx.x * blockDim.x + threadIdx.x) * VEC;
        const bool live = n0 < ci.nf;
        if (m.simple) {
            const int n_sum = m.all_mono ? 1 : m.out_ch;
            for (int c = 0; c < n_sum; c++) {
                MixVec<VEC> acc;
                acc.zero();
                if (m.n_edges < 16) {  // a handful of edges (the usual port): straight from the edge table, no staging, no barriers
                    if (live) mix_direct<VEC>(m, edges, c, n0, ci, acc);
                } else
                for (int base = 0; base < m.n_edges; base += MIX_STAGE) {
                    __syncthreads();  // the previous stage's pointers have been used by everyone
                    if (base + (int)threadIdx.x < m.n_edges) {
                        const MixEdge& ed = edges[m.edge_offset + base + threadIdx.x];
                        s_src[threadIdx.x] = chan(ed.src, ed.src_ch == 1 ? 0 : c, ci);
                    }
                    __syncthreads();
                    if (live) mix_run<VEC>(s_src, min(MIX_STAGE, m.n_edges - base), n0, base == 0, acc);
                }
                if (!live) continue;
                for (int oc = c; oc < (m.all_mono ? m.out_ch : c + 1); oc++) {
                    float* out = chan(m.out, oc, ci) + n0;
                    const bool vec = VEC == 4 && (reinterpret_cast<uintptr_t>(out) & 15) == 0 && (m.limit < 0 || ci.f0 + n0 + 4 <= m.limit);
                    if (vec) {
                        *reinterpret_cast<float4*>(out) = make_float4(acc.get(0), acc.get(1), acc.get(2), acc.get(3));
                    } else {
                        for (int j = 0; j < VEC; j++)
                            if (m.limit < 0 || ci.f0 + n0 + j < m.limit) out[j] = acc.get(j);
                    }
                }
            }
            continue;
        }
        if (!live) continue;
        for (int j = 0; j < VEC; j++) {
            const int n = n0 + j;
            if (m.limit >= 0 && ci.f0 + n >= m.limit) continue;
            for (int c = 0; c < m.out_ch; c++) {
                float acc = 0.f;
                bool any = false;
                for (int e = 0; e < m.n_edges; e++) {
                    const MixEdge& ed = edges[m.edge_offset + e];
                    if (mix_is_silence(ed.src_ch, m.out_ch, c, m.interp)) continue;
                    const float v = mixed_sample(ed, m.out_ch, c, m.interp, n, ci);
                    acc = any ? acc + v : v;
                    any = true;
                }
                chan(m.out, c, ci)[n] = acc;
            }
        }
    }
}

// stages whose ports all have fewer than 16 edges (the usual graph): no staging, no barriers, 40 registers — the mixer is memory-bound and
// lives on resident warps (the staged kernel above needs 64+)
template <int VEC>
__global__ void __launch_bounds__(256) k_mix_narrow(const MixInst* __restrict__ insts, const MixEdge* __restrict__ edges, int n_inst, ChunkInfo ci) {
    for (int ii = blockIdx.y; ii < n_inst; ii += gridDim.y) {
        const MixInst m = insts[ii];
        const int n0 = (blockIdx.x * blockDim.x + threadIdx.x) * VEC;
        if (n0 >= ci.nf) continue;
        if (m.simple) {
            const int n_sum = m.all_mono ? 1 : m.out_ch;
            for (int c = 0; c < n_sum; c++) {
                MixVec<VEC> acc;
                acc.zero();
                mix_direct<VEC>(m, edges, c, n0, ci, acc);
                for (int oc = c; oc < (m.all_mono ? m.out_ch : c + 1); oc++) {
                    float* out = chan(m.out, oc, ci) + n0;
                    const bool vec = VEC == 4 && (reinterpret_cast<uintptr_t>(out) & 15) == 0 && (m.limit < 0 || ci.f0 + n0 + 4 <= m.limit);
                    if (vec) {
                        *reinterpret_cast<float4*>(out) = make_float4(acc.get(0), acc.get(1), acc.get(2), acc.get(3));
                    } else {
                        for (int j = 0; j < VEC; j++)
                            if (m.limit < 0 || ci.f0 + n0 + j < m.limit) out[j] = acc.get(j);
                    }
                }
            }
            continue;
        }
        for (int j = 0; j < VEC; j++) {
            const int n = n0 + j;
            if (m.limit >= 0 && ci.f0 + n >= m.limit) continue;
            for (int c = 0; c < m.out_ch; c++) {
                float acc = 0.f;
                bool any = false;
                for (int e = 0; e < m.n_edges; e++) {
                    const MixEdge& ed = edges[m.edge_offset + e];
                    if (mix_is_silence(ed.src_ch, m.out_ch, c, m.interp)) continue;
                    const float v = mixed_sample(ed, m.out_ch, c, m.interp, n, ci);
                    acc = any ? acc + v : v;
                    any = true;
                }
                chan(m.out, c, ci)[n] = acc;
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
// BiquadFilter — BiquadFilterRenderer::process (src/node/biquad_filter.rs:764-899), constant coefficients.
// (1) serial: one thread per (instance, channel), the reference's exact f64 operation order (bit-faithful).
// (2) scan: one CTA per (instance, channel); the chunk is processed in tiles of 256 x 8 frames.  Each thread
//     runs the recurrence on its 8 frames from zero state, a block-wide Kogge-Stone scan over the 2x2
//     state-transition powers propagates the true state, and the homogeneous response is added back:
//         y[j] = y0[j] + h1[j] * y[-1] + h2[j] * y[-2].
//     Same filter in exact arithmetic; rounding differs from the serial order by ~1e-15 relative.
// ---------------------------------------------------------------------------------------------------------
DEVI bool isnormal_d(double v) {
    const double a = fabs(v);
    return a >= 2.2250738585072014e-308 && a <= 1.7976931348623157e308;
}
// BiquadFilterRenderer / IirFilterRenderer with an input whose layout changes (biquad_filter.rs:778-815, iir_filter.rs:336-376), as seen
// by the thread of ONE channel `c` at the start of quantum `qi`:
//   input silent: the filter keeps its channel count `len`; a channel whose state has no normal value left is in its "ended" state —
//     the reference stops processing once ALL channels are (processing an ended channel yields exact zeros, so deciding per channel
//     is the same PCM); the quantum is reported silent when every row says so.
//   input not silent: `len` becomes the input's count; a channel the input does not have loses its state (truncate), one that
//     appears starts from zeros (push([0.; 4])).
// skip: write zeros, leave the state alone.  absent: channel c does not exist in this quantum (state zeroed, output don't-care).
DEVI void filter_layout_step(const BufRef& in, const BufRef& out, int rows, int c, int qi, int& len, bool state_normal, bool& skip, bool& absent) {
    const bool silent = buf_silent(in, rows, qi);
    if (!silent) len = buf_count(in, rows, qi);
    const bool gone = c >= len;
    skip = (silent && !state_normal) || gone;
    absent = gone || silent;  // no input samples to read for this channel in this quantum: zeros (`gone` also drops the state, below)
    if (out.meta) meta_put(out, c, qi, len > 0 ? len : 1, skip);
}

__global__ void __launch_bounds__(128) k_biquad_serial(const BiquadInst* __restrict__ insts, int n_inst, int max_ch, ChunkInfo ci) {
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    int ii = t / max_ch, c = t % max_ch;
    if (ii >= n_inst) return;
    const BiquadInst q = insts[ii];
    if (c >= q.ch) return;
    const float* in = chan(q.in, c, ci);
    float* out = chan(q.out, c, ci);
    double* st = q.state + 4 * c;
    double x1 = st[0], x2 = st[1], y1 = st[2], y2 = st[3];
    const bool dyn = q.in.meta != nullptr;
    int len = dyn ? q.dyn_len[c] : q.ch;  // xy.len() of the reference
    bool skip = false, absent = false;
    for (int n = 0; n < ci.nf; n++) {
        if (dyn && (n & 127) == 0) {  // biquad_filter.rs:778-815, per channel (see filter_layout_step)
            filter_layout_step(q.in, q.out, q.ch, c, meta_qi(ci, n), len, isnormal_d(x1) || isnormal_d(x2) || isnormal_d(y1) || isnormal_d(y2), skip, absent);
            if (c >= len) x1 = x2 = y1 = y2 = 0.;
        }
        if (skip) {
            out[n] = 0.f;
            continue;
        }
        double x = absent ? 0. : (double)in[n];
        // b0*x + b1*x1 + b2*x2 - a1*y1 - a2*y2, left to right, unfused (biquad_filter.rs:878)
        double y = __dsub_rn(__dsub_rn(__dadd_rn(__dadd_rn(__dmul_rn(q.b0, x), __dmul_rn(q.b1, x1)), __dmul_rn(q.b2, x2)),
                                       __dmul_rn(q.a1, y1)),
                             __dmul_rn(q.a2, y2));
        // `if !y.is_normal() { y = 0. }` (:881-883) incl. FTZ of subnormals
        double ay = fabs(y);
        if (!(ay >= 2.2250738585072014e-308 && ay <= 1.7976931348623157e308)) y = 0.;
        x2 = x1;
        x1 = x;
        y2 = y1;
        y1 = y;
        out[n] = (float)y;
    }
    st[0] = x1;
    st[1] = x2;
    st[2] = y1;
    st[3] = y2;
    if (dyn) q.dyn_len[c] = len;
}

DEVI float shaper_apply(const float* curve, int len, float input);

constexpr int CH_K = WAE_CHAIN_K;  // frames per thread
#ifndef WAE_CH_THREADS
#define WAE_CH_THREADS 128
#endif
constexpr int CH_THREADS = WAE_CH_THREADS;  // threads per CTA -> tile = 16 frames per thread
constexpr int CH_WARPS = CH_THREADS / 32;

// ---------------------------------------------------------------------------------------------------------
// Fused chain — source -> gain -> [biquad A] -> gain -> [biquad B] -> gain -> [wave-shaper] -> gain -> buffer or
// destination, in ONE pass over the PCM.  One CTA per (instance, channel); the chunk is walked in tiles of
// 128 threads x 16 frames, the next tile's source frames are prefetched while the current tile is filtered.
// Replaces, for chain-shaped sub-graphs, AudioBufferSourceRenderer / OscillatorRenderer / ConstantSourceRenderer +
// BiquadFilterRenderer + GainRenderer + WaveShaperRenderer + the destination copy (src/node/{audio_buffer_source,
// oscillator,constant_source,biquad_filter,gain,waveshaper,destination}.rs), so that a graph-quantum costs only its
// compulsory HBM bytes (SURVEY §8d: source read + destination write).  The kernel is compiled per chain shape
// <source kind, number of biquads, shaper> so that the per-step dispatch costs no instructions.
//
// Biquad = time-parallel recurrence in f64: pass 1 runs the thread's 16 frames from zero state to get its end
// state, the end states are scanned (5 shuffle steps with A^(2^d) inside a warp, then the 4 warp totals are chained
// with A^32), pass 2 re-runs the recurrence from the true incoming state.  Same filter as the reference's serial
// loop (biquad_filter.rs:876-891) in exact arithmetic; rounding differs by ~1e-15 relative.
// ---------------------------------------------------------------------------------------------------------
DEVI void mat2_fma(const double* P, double a, double b, double& accA, double& accB) {
    accA = fma(P[0], a, fma(P[1], b, accA));
    accB = fma(P[2], a, fma(P[3], b, accB));
}

template <int SRC>
DEVI void chain_load_source(const ChainInst& q, int c, const ChunkInfo& ci, int n0, float v[CH_K], const float2* tab2 = nullptr) {
    // n0: first frame (chunk-relative) of this thread's 16 frames; caller guarantees n0 < ci.nf
    if (SRC == CHAIN_SRC_BUFFER) {
        const float4* in = reinterpret_cast<const float4*>(chan(q.in, c, ci) + n0);
#pragma unroll
        for (int u = 0; u < CH_K / 4; u++) {
            float4 a = in[u];
            v[4 * u] = a.x; v[4 * u + 1] = a.y; v[4 * u + 2] = a.z; v[4 * u + 3] = a.w;
        }
    } else if (SRC == CHAIN_SRC_ABSN) {
        const AbsnInst& o = q.absn;
        const float* src = o.buf + (size_t)c * o.buf_stride;
        const int64_t n = ci.f0 + n0;
        const int64_t idx = n - o.n_start + o.buf_offset;
        if (!o.loop && n >= o.n_start && idx + CH_K <= o.buf_len && ((reinterpret_cast<uintptr_t>(src + idx) & 15) == 0)) {
            const float4* in = reinterpret_cast<const float4*>(src + idx);  // aligned interior: 4 x LDG.128
#pragma unroll
            for (int u = 0; u < CH_K / 4; u++) {
                float4 a = __ldg(in + u);
                v[4 * u] = a.x; v[4 * u + 1] = a.y; v[4 * u + 2] = a.z; v[4 * u + 3] = a.w;
            }
        } else {
            // ragged / looping runs, frame by frame; a looping buffer costs ONE modulo per thread and then a wrapping index (was: a 64-bit
            // modulo per frame).  (Kept this small: the out-of-line gather's register needs are saved and restored around every call
            // in k_chain — a float4 fast path for loops here made the streamed kernel spill.)
            int64_t pos = 0;
            if (o.loop) {
                pos = idx % o.buf_len;
                if (pos < 0) pos += o.buf_len;  // (frames before the start: never read, but the index keeps step)
            }
#pragma unroll
            for (int j = 0; j < CH_K; j++) {
                const int64_t m = n + j;
                float s = 0.f;
                if (m >= o.n_start && m < o.n_stop) {
                    if (o.loop) s = __ldg(src + pos);
                    else if (idx + j < o.buf_len) s = __ldg(src + idx + j);
                }
                if (o.loop) pos = pos + 1 == o.buf_len ? 0 : pos + 1;
                v[j] = s;
            }
        }
    } else if (SRC == CHAIN_SRC_OSC) {
        const OscInst& o = q.osc;
        const int64_t na = ci.f0 + n0;
        if (o.fast && na >= o.n_first && na + CH_K <= o.n_stop) {
            // Fully active run.  The reference accumulates `phase += incr` (wrapping at 1) in f64; here the phase of the
            // first frame comes from the closed form and then runs as a 64-bit fixed-point fraction of a cycle (wraps for
            // free, 2^-64 resolution): |phase - reference phase| stays ~1e-14, far below the f32 output resolution, and the
            // per-frame work is integer / f32 instead of f64 compare-and-wrap + f64 <-> f32 conversions.
            const double inc = o.incr, inv = o.inv_incr;
            unsigned long long ph = __double2ull_rn(osc_phase_at(o, na) * 9223372036854775808.0) << 1;
            const unsigned long long dph = __double2ull_rn(inc * 18446744073709551616.0);
            const unsigned long long HALF = 0x8000000000000000ull;
            const int type = o.type;
            if (type == 0 || type == 4) {  // sine (:571-585) / custom (:622-637): 2048-entry table + lerp with fmaf
                if (tab2) {  // the CTA's shared copy of the table as (entry, next entry) pairs: one 8-byte shared load per frame
#pragma unroll
                    for (int j = 0; j < CH_K; j++) {
                        const unsigned hi = (unsigned)(ph >> 32), lo = (unsigned)ph;
                        const float2 e = tab2[hi >> 21];
                        const float k = __uint_as_float(0x3f800000u | ((hi << 11 | lo >> 21) >> 9)) - 1.0f;
                        v[j] = fmaf(e.x, 1.f - k, e.y * k);
                        asm("add.u64 %0, %0, %1;" : "+l"(ph) : "l"(dph));  // opaque: keeps ONE running phase instead of 16 precomputed ones
                    }
                } else {
#pragma unroll
                    for (int j = 0; j < CH_K; j++) {
                        const unsigned hi = (unsigned)(ph >> 32), lo = (unsigned)ph;
                        const int prev = (int)(hi >> 21);
                        const int next = (prev + 1) & 2047;
                        const float k = __uint_as_float(0x3f800000u | ((hi << 11 | lo >> 21) >> 9)) - 1.0f;
                        v[j] = fmaf(__ldg(o.table + prev), 1.f - k, __ldg(o.table + next) * k);
                        asm("add.u64 %0, %0, %1;" : "+l"(ph) : "l"(dph));
                    }
                }
            } else if (type == 2 || type == 1) {
                // sawtooth (:588-595): 2 * unroll(phase + 0.5) - 1 - polyBLEP;  square (:598-606): +-1 + polyBLEP(phase) - polyBLEP(phase + 0.5).
                // Pass 1 writes the plain wave and notes, one bit per frame, the frames that MAY lie in a polyBLEP window: with
                // u = phase + dph the sawtooth's window around the wrap of phase + 0.5 is u + 2^63 < 2 dph, the square's two windows
                // (around 0 and 0.5) are u mod 2^63 < 2 dph; the test looks at the high words only, so it flags a few frames too many —
                // the out-of-line evaluation decides exactly, in f64, and returns the plain wave for those.  Pass 2 visits the flagged
                // frames lane by lane: a warp whose lanes have their windows at different frames runs the f64 evaluation as often as its
                // busiest lane has flagged frames (1 - 2 times per tile at 440 Hz) instead of once per frame that ANY lane flags (7 of 16:
                // the polyBLEP lines were a large share of the oscillator chain's instructions).
                const unsigned long long ph0 = ph;
                const unsigned thr = (unsigned)((dph + dph) >> 32);
                unsigned mask = 0;
                if (type == 2) {
                    const unsigned long long cw = HALF + dph;
#pragma unroll
                    for (int j = 0; j < CH_K; j++) {
                        v[j] = __ll2float_rn((long long)ph) * 1.08420217248550443e-19f;  // (2 p2 - 1) = signed(ph) / 2^63
                        if ((unsigned)((ph + cw) >> 32) <= thr) mask |= 1u << j;
                        asm("add.u64 %0, %0, %1;" : "+l"(ph) : "l"(dph));
                    }
                    while (mask) {
                        const int jw = __ffs((int)mask) - 1;
                        mask &= mask - 1;
                        const unsigned long long pj = ph0 + (unsigned long long)jw * dph;
                        const float sw = osc_saw_blep(pj + HALF, inc, inv);
#pragma unroll
                        for (int j = 0; j < CH_K; j++) v[j] = j == jw ? sw : v[j];
                    }
                } else {
                    const bool wide = dph >= 0x4000000000000000ull;  // incr >= 1/4: the two windows cover every frame
#pragma unroll
                    for (int j = 0; j < CH_K; j++) {
                        v[j] = (long long)ph >= 0 ? 1.0f : -1.0f;
                        if (((unsigned)((ph + dph) >> 32) & 0x7fffffffu) <= thr) mask |= 1u << j;
                        asm("add.u64 %0, %0, %1;" : "+l"(ph) : "l"(dph));
                    }
                    if (wide) mask = (1u << CH_K) - 1u;
                    while (mask) {
                        const int jw = __ffs((int)mask) - 1;
                        mask &= mask - 1;
                        const unsigned long long pj = ph0 + (unsigned long long)jw * dph;
                        const float sw = osc_square_blep(pj, pj + HALF, inc, inv);
#pragma unroll
                        for (int j = 0; j < CH_K; j++) v[j] = j == jw ? sw : v[j];
                    }
                }
            } else {  // triangle (:609-619): fold(-4 phase + 2) = 1 - 4 |phase - 1/4| with the difference taken modulo 1
#pragma unroll
                for (int j = 0; j < CH_K; j++) {
                    long long q = (long long)(ph - 0x4000000000000000ull);
                    q = q < 0 ? -q : q;  // |q| * 2^64, <= 2^63 (q = -2^63 maps to itself: phase 3/4, value -1)
                    // 1 - 4 |q| / 2^64 = (2^62 - |q|) / 2^62: the integer is exact, its conversion is the one f32 rounding
                    v[j] = __ll2float_rn((long long)(0x4000000000000000ull - (unsigned long long)q)) * 2.16840434497100887e-19f;
                    asm("add.u64 %0, %0, %1;" : "+l"(ph) : "l"(dph));  // opaque: keeps ONE running phase instead of 16 precomputed ones
                }
            }
        } else {
#pragma unroll
            for (int j = 0; j < CH_K; j++) {
                int64_t n = na + j;
                float s = 0.f;
                if (n >= o.n_first && n < o.n_stop && !o.outside_nyquist) s = osc_sample(o, osc_phase_at(o, n), o.incr);
                v[j] = s;
            }
        }
    } else {
        const ConstInst& o = q.cst;
#pragma unroll
        for (int j = 0; j < CH_K; j++) {
            int64_t n = ci.f0 + n0 + j;
            v[j] = (n >= o.n_first && n < o.n_stop) ? o.value : 0.f;
        }
    }
}

// ragged / looping / unaligned source regions: the thread's 16 frames gathered one by one and put into the warp's staging region
// (kept out of line: it is rare, and inlined it is repeated in every prefetch stage of the pipeline)
template <int SRC>
__device__ __noinline__ void chain_stage_gather(const ChainInst* q, int c, ChunkInfo ci, int n0, float4* region, int lane, int xq) {
    float tmp[CH_K];
    chain_load_source<SRC>(*q, c, ci, n0, tmp);
#pragma unroll
    for (int u = 0; u < CH_K / 4; u++) region[4 * lane + (u ^ xq)] = make_float4(tmp[4 * u], tmp[4 * u + 1], tmp[4 * u + 2], tmp[4 * u + 3]);
}

struct ChainSmem {
    ChainInst q;
    double state[CHAIN_MAX_BIQUADS][4];  // x1, x2, y1, y2 carried from tile to tile
    double P[CHAIN_MAX_BIQUADS][24];     // Pshfl[5][4], Pwarp[4]
    double plane[CHAIN_MAX_BIQUADS][32][4];  // A^(lane+1): carries a warp's incoming state to each lane (read once per tile: not worth registers)
    double wtot[CH_WARPS][2];            // per-warp end state (zero incoming state)
    double replay[4];                    // serial replay of a tile (non-finite input): state handed from warp to warp
    float edge[CH_WARPS][2];             // last two step inputs of every warp
    int flushed;                         // a tile of this slab went through the non-finite handling (its end state no longer depends on the state it started from)
};

// one biquad over the thread's 16 frames (v in/out), see the header comment
// clean: (threads that start a render quantum) the filter state entering this thread's frames has no normal value — the filter's
// "tail has ended" test (biquad_filter.rs:778-794), used for the layout track of the chain's output
struct NoReload {};
// reload(x): (biquad A of a chain that streams its source) puts the thread's 16 INPUT samples of this tile back into x — the staging
// region still holds them — for the serial replay of a tile that a NaN / Inf went through.
template <typename RL>
DEVI void chain_biquad(ChainSmem& sm, int bq, const double b0, const double b1, const double b2, const double a1, const double a2,
                       const double* Plane, float v[CH_K], bool active, int n_active, int t, int lane, int warp, bool want_clean, bool& clean,
                       RL reload) {
    const double* Psh = sm.P[bq];
    const double* Pw = sm.P[bq] + 20;
    // previous two step inputs: neighbour lane, previous warp, or the carried state
    const float xl1 = active ? v[CH_K - 1] : 0.f, xl2 = active ? v[CH_K - 2] : 0.f;
    if (lane == 31) {
        sm.edge[warp][0] = xl1;
        sm.edge[warp][1] = xl2;
    }
    const float p1 = __shfl_up_sync(0xffffffffu, xl1, 1);
    const float p2 = __shfl_up_sync(0xffffffffu, xl2, 1);
    __syncthreads();
    double x1, x2;
    if (lane == 0) {
        if (warp == 0) {
            x1 = sm.state[bq][0];
            x2 = sm.state[bq][1];
        } else {
            x1 = (double)sm.edge[warp - 1][0];
            x2 = (double)sm.edge[warp - 1][1];
        }
    } else {
        x1 = (double)p1;
        x2 = (double)p2;
    }
    const bool x_normal = want_clean && (isnormal_d(x1) || isnormal_d(x2));
    // FIR part and pass 1 (zero incoming state): end state only
    double w[CH_K];
    double r1 = 0., r2 = 0.;
    const double na1 = -a1, na2 = -a2;
#pragma unroll
    for (int j = 0; j < CH_K; j++) {
        const double x = (double)v[j];
        w[j] = fma(b2, x2, fma(b1, x1, b0 * x));
        const double y = fma(na1, r1, fma(na2, r2, w[j]));
        x2 = x1;
        x1 = x;
        r2 = r1;
        r1 = y;
    }
    // warp-level inclusive scan of end states: S_t = A S_{t-1} + (r1, r2)
    double va = active ? r1 : 0., vb = active ? r2 : 0.;
#pragma unroll
    for (int d = 0; d < 5; d++) {
        const double oa = __shfl_up_sync(0xffffffffu, va, 1 << d);
        const double ob = __shfl_up_sync(0xffffffffu, vb, 1 << d);
        if (lane >= (1 << d)) mat2_fma(Psh + 4 * d, oa, ob, va, vb);
    }
    if (lane == 31) {
        sm.wtot[warp][0] = va;
        sm.wtot[warp][1] = vb;
    }
    const double ea = __shfl_up_sync(0xffffffffu, va, 1);  // inclusive value of the previous lane
    const double eb = __shfl_up_sync(0xffffffffu, vb, 1);
    __syncthreads();
    // state entering this warp: chain the previous warps' totals through A^32
    double wa = sm.state[bq][2], wb = sm.state[bq][3];
#pragma unroll
    for (int k = 0; k < CH_WARPS - 1; k++) {
        if (k < warp) {
            double ta = sm.wtot[k][0], tb = sm.wtot[k][1];
            mat2_fma(Pw, wa, wb, ta, tb);
            wa = ta;
            wb = tb;
        }
    }
    // state entering this thread: warp-incoming state carried over `lane` threads + exclusive prefix inside the warp
    double e1 = wa, e2 = wb;
    if (lane != 0) {
        e1 = ea;
        e2 = eb;
        mat2_fma(Plane, wa, wb, e1, e2);
    }
    if (want_clean) clean = !(x_normal || isnormal_d(e1) || isnormal_d(e2));  // (CTA-uniform: only chains that write a layout track)
    // pass 2: the recurrence from the true state
    r1 = e1;
    r2 = e2;
#pragma unroll
    for (int j = 0; j < CH_K; j++) {
        const double y = fma(na1, r1, fma(na2, r2, w[j]));
        r2 = r1;
        r1 = y;
        v[j] = (float)y;  // `*o = y as f32` between nodes (biquad_filter.rs:890)
    }
    // (barrier: everyone has read state / wtot / edge of this step.)  A NaN / Inf that went through the recurrence is still in the state
    // the tile ends with: the reference flushes every non-normal y to 0 sample by sample (`if !y.is_normal() { y = 0. }`,
    // biquad_filter.rs:881-883) and recovers three samples after a bad input sample, which no linear scan reproduces.
    const bool last = active && t == n_active - 1;
    const bool poisoned = last && (!(fabs(r1) <= 1.7976931348623157e308) || !(fabs(r2) <= 1.7976931348623157e308));
#ifdef WAE_CHAIN_NOCHECK  // (tuning builds only: what the non-finite check costs)
    __syncthreads();
    if (false) {
#else
    if (__syncthreads_or(poisoned)) {
#endif
        if (t == 0) sm.flushed = 1;
        if constexpr (!std::is_same<RL, NoReload>::value) {
            // rare: run the tile again serially, thread after thread, in the reference's own operation order, from the tile's inputs
            float x[CH_K];
            reload(x);
            double sx1 = sm.state[bq][0], sx2 = sm.state[bq][1], sy1 = sm.state[bq][2], sy2 = sm.state[bq][3];
            __syncthreads();
#pragma unroll 1
            for (int wv = 0; wv < CH_WARPS; wv++) {
                if (warp == wv) {
#pragma unroll 1
                    for (int l = 0; l < 32; l++) {
                        double qx1 = sx1, qx2 = sx2, qy1 = sy1, qy2 = sy2;
                        if (lane == l && active) {
#pragma unroll
                            for (int j = 0; j < CH_K; j++) {  // (unrolled: x[] / v[] stay in registers)
                                const double xi = (double)x[j];
                                double y = __dsub_rn(__dsub_rn(__dadd_rn(__dadd_rn(__dmul_rn(b0, xi), __dmul_rn(b1, qx1)), __dmul_rn(b2, qx2)), __dmul_rn(a1, qy1)),
                                                     __dmul_rn(a2, qy2));
                                if (!isnormal_d(y)) y = 0.;
                                qx2 = qx1;
                                qx1 = xi;
                                qy2 = qy1;
                                qy1 = y;
                                v[j] = (float)y;
                            }
                        }
                        sx1 = __shfl_sync(0xffffffffu, qx1, l);
                        sx2 = __shfl_sync(0xffffffffu, qx2, l);
                        sy1 = __shfl_sync(0xffffffffu, qy1, l);
                        sy2 = __shfl_sync(0xffffffffu, qy2, l);
                    }
                    if (lane == 0) {
                        sm.replay[0] = sx1;
                        sm.replay[1] = sx2;
                        sm.replay[2] = sy1;
                        sm.replay[3] = sy2;
                    }
                }
                __syncthreads();
                sx1 = sm.replay[0];
                sx2 = sm.replay[1];
                sy1 = sm.replay[2];
                sy2 = sm.replay[3];
                __syncthreads();
            }
            if (t == 0) {
                sm.state[bq][0] = sx1;
                sm.state[bq][1] = sx2;
                sm.state[bq][2] = sy1;
                sm.state[bq][3] = sy2;
            }
            return;
        } else {
            // (a filter fed by another node of the chain: its input is finite, it has run off by itself — the reference's flush would have
            // reset it; do not carry the poison)
            if (last) r1 = r2 = 0.;
        }
    }
    if (last) {
        sm.state[bq][0] = (double)xl1;
        sm.state[bq][1] = (double)xl2;
        sm.state[bq][2] = r1;
        sm.state[bq][3] = r2;
    }
}

// ---- Hopper async-copy primitives used by the TMA variant of k_chain (1-D bulk copies, mbarrier completion) ----
DEVI unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
DEVI void mbar_init(uint64_t* bar, unsigned count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory"); }
DEVI void mbar_expect_tx(uint64_t* bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
DEVI void mbar_wait(uint64_t* bar, unsigned parity) {
    unsigned ok;
    do {
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
            "selp.u32 %0, 1, 0, p;\n"
            "}\n"
            : "=r"(ok)
            : "r"(smem_u32(bar)), "r"(parity)
            : "memory");
    } while (!ok);
}
// global -> shared, completion counted in bytes on `bar` (SASS: UBLKCP)
DEVI void bulk_load(void* smem_dst, const void* gsrc, unsigned bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)), "l"(gsrc),
                 "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
// shared -> global, tracked by the issuing thread's bulk async-groups
DEVI void bulk_store(void* gdst, const void* smem_src, unsigned bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)), "r"(bytes) : "memory");
}
DEVI void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
DEVI void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
DEVI void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

#ifndef WAE_CH_STAGES
#define WAE_CH_STAGES 4
#endif
constexpr int CH_STAGES = WAE_CH_STAGES;  // source tiles in flight per CTA (8 KB each)

// conditional exchange of two 16-byte pieces (the un-permutation of the bank-conflict-free access order, see k_chain)
DEVI void cswap4(bool p, float4& a, float4& b) {
    const float4 ta = a, tb = b;
    a.x = p ? tb.x : ta.x; a.y = p ? tb.y : ta.y; a.z = p ? tb.z : ta.z; a.w = p ? tb.w : ta.w;
    b.x = p ? ta.x : tb.x; b.y = p ? ta.y : tb.y; b.z = p ? ta.z : tb.z; b.w = p ? ta.w : tb.w;
}

// Work decomposition.  A work item is (time slab, instance, channel); items are numbered slab-major and handed out in
// order of CTA start (one atomic ticket per CTA), so the slab before a given one of the same (instance, channel) always
// belongs to a CTA that is already running or done: waiting for the filter state it leaves behind cannot deadlock.
// With S slabs the launch has S x more, S x shorter CTAs: the tail of the last wave (equal whole-render CTAs
// leave the machine partly empty for the last fraction of the run) shrinks to one short item.  Chains without a filter carry no
// state: their slabs are independent.  TMA = true: the source tiles arrive through 1-D bulk copies (cp.async.bulk +
// mbarrier), results leave through bulk stores; TMA = false: 16-byte cp.async pieces / coalesced stores (kept as the
// reference data path: WAE_OPT_CHAIN_TMA = 0).
#ifndef WAE_CH_MINB
#define WAE_CH_MINB 6
#endif
// resident CTAs per SM the register budget is cut for: 6 (80 registers) for the streamed chains, which live on memory-level parallelism;
// one fewer with two filters; the oscillator chains are bound by issue slots and latency, not by DRAM, and spill at 80 registers
// (56 bytes of stack in <OSC, 1>): WAE_CH_MINB_OSC CTAs (96+ registers)
#ifndef WAE_CH_MINB_OSC
#define WAE_CH_MINB_OSC 5
#endif
constexpr int chain_min_blocks(int src, int nb) {
    const int base = src == CHAIN_SRC_OSC ? WAE_CH_MINB_OSC : WAE_CH_MINB;
    return ((nb == 2 ? base - 1 : base) * 128) / CH_THREADS;
}
template <int SRC, int NB, bool SHAPER, bool TMA, bool PRE = false>
__global__ void __launch_bounds__(CH_THREADS, chain_min_blocks(SRC, NB)) k_chain(const ChainInst* __restrict__ insts, const ScanCoef* __restrict__ coefs,
                                                                        int n_inst, ChunkInfo ci, ChainSched sc) {
    __shared__ ChainSmem sm;
    __shared__ int s_item;
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    int item = (int)blockIdx.x;
    if (NB > 0 && sc.ticket != nullptr) {
        if (t == 0) {
            const unsigned tk = atomicAdd(sc.ticket, 1u);
            if (tk == gridDim.x - 1) atomicExch(sc.ticket, 0u);  // the last ticket of this launch: leave the counter ready for the next one
            s_item = (int)tk;
        }
        __syncthreads();
        item = s_item;
    }
    const int per_slab = n_inst * sc.max_ch;
    const int slab = item / per_slab;
    const int rem = item - slab * per_slab;
    const int c = rem / n_inst;
    const int inst = rem - c * n_inst;
    {
        const int* src = reinterpret_cast<const int*>(insts + inst);
        int* dst = reinterpret_cast<int*>(&sm.q);
        for (int i = t; i < (int)(sizeof(ChainInst) / 4); i += CH_THREADS) dst[i] = src[i];
    }
    __syncthreads();
    // A work item that starts at or after its graph's end (a graph shorter than its group) has nothing to render: it leaves before any
    // copy.  No slab waits for it: the later slabs of its (instance, channel) start later still and leave here too, before they wait for
    // a hand-off (PRE slabs included).  (An output with a layout track is rendered to the end: its consumers read the track.)
    if (ci.f0 + (int64_t)slab * sc.tiles_per_slab * (CH_THREADS * CH_K) >= sm.q.end && sm.q.out.meta == nullptr) return;
    // oscillator wavetable -> shared memory, as (entry, next entry) pairs: the 128 threads of a CTA are 16 frames apart, so their table
    // indices fall in different 128-byte lines (a 32-wavefront global gather per load); shared memory only pays bank conflicts, and the
    // pair makes the two taps of the interpolation one 8-byte load
    __shared__ float2 s_table2[SRC == CHAIN_SRC_OSC ? 2048 : 1];
    const float2* tab2 = nullptr;
    if (SRC == CHAIN_SRC_OSC && sm.q.osc.table_len == 2048 && (sm.q.osc.type == 0 || sm.q.osc.type == 4)) {
        const float* gt = sm.q.osc.table;
        for (int i = t; i < 2048; i += CH_THREADS) s_table2[i] = make_float2(__ldg(gt + i), __ldg(gt + ((i + 1) & 2047)));
        tab2 = s_table2;
        __syncthreads();
    }
    const ChainInst& q = sm.q;
    if (c >= q.ch) return;
    constexpr int tile = CH_THREADS * CH_K;
    const int n_tiles = (ci.nf + tile - 1) / tile;
    const int tile0 = slab * sc.tiles_per_slab;
    if (tile0 >= n_tiles) return;
    const int slab_begin = tile0 * tile;
    const int slab_end = min(ci.nf, (tile0 + sc.tiles_per_slab) * tile);
    const bool first_slab = slab == 0, last_slab = slab_end >= ci.nf;
    const size_t ho = ((size_t)inst * sc.max_ch + c) * sc.slab_stride + slab;  // hand-off slot of the state ENTERING this slab
    // per-CTA constants -> registers / shared
    double cb[NB > 0 ? NB : 1][5];
    // PRE (few (instance, channel) pairs, long renders: chain_plan_slabs): a slab that is not the last one first runs over its frames from
    // ZERO state without storing anything, which gives the part of its end state that its own input causes; the rest is the state it
    // starts from carried through the slab, G^L s_in with a host-computed matrix.  So it can publish the state the NEXT slab starts
    // from as soon as its own s_in arrives — before it renders — and the slabs of one pair render concurrently instead of one after
    // the other (one extra read of the source; the chain of hand-offs costs a couple of microseconds per slab).
    const bool pre = PRE && NB == 1 && sc.pre_log2 >= 0 && !last_slab;
    auto wait_handoff = [&]() {  // the slab before this one (same instance, channel) publishes the state it ends with
        if (t == 0) {
            const unsigned* f = sc.flags + ho;
            unsigned seen;
            for (;;) {
                asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(seen) : "l"(f) : "memory");
                if (seen == sc.epoch) break;
                __nanosleep(256);
            }
        }
        __syncthreads();
    };
    if (NB > 0 && !first_slab && !pre) wait_handoff();
#pragma unroll
    for (int k = 0; k < NB; k++) {
        const ChainBiquad& bq = q.bq[k];
        cb[k][0] = bq.b0; cb[k][1] = bq.b1; cb[k][2] = bq.b2; cb[k][3] = bq.a1; cb[k][4] = bq.a2;
        const ScanCoef& scf = coefs[bq.coef];
        if (t < 20) sm.P[k][t] = (&scf.Pshfl[0][0])[t];
        if (t < 4) {
            sm.P[k][20 + t] = scf.Pwarp[t];
            sm.state[k][t] = pre ? 0. : (first_slab ? bq.state[4 * c + t] : __ldcg(sc.handoff + ho * (CHAIN_MAX_BIQUADS * 4) + 4 * k + t));
        }
        for (int i = t; i < 128; i += CH_THREADS) (&sm.plane[k][0][0])[i] = (&scf.Plane[0][0])[i];
    }
    const float g0 = q.g[0], g1 = q.g[1], g2 = q.g[2], g3 = q.g[3];

    constexpr bool STREAMED = SRC == CHAIN_SRC_BUFFER || SRC == CHAIN_SRC_ABSN;  // PCM read from memory: prefetched
    constexpr bool USE_TMA = TMA && STREAMED;
    constexpr int NST = STREAMED ? CH_STAGES : 1;
    // Per-warp staging of source / result frames.  A warp owns 512 consecutive frames (2 KB) of the tile; global memory is
    // touched with whole 2 KB regions (one bulk copy, or 4 coalesced 512-byte warp accesses), while thread tt works on the
    // contiguous pieces f = 4*tt + uu.  cp.async path: an XOR swizzle makes both access patterns conflict-free for 128-bit
    // shared accesses.  Bulk copies are linear, so there a thread visits its own four pieces in the order u ^ xq (conflict-free
    // for the same reason) and puts them back in place with two conditional exchanges.
    constexpr int WF = 32 * CH_K / 4;  // float4 pieces per warp region (128)
    __shared__ __align__(128) float4 s_io[NST][CH_WARPS][WF];
    __shared__ __align__(8) uint64_t s_bar[USE_TMA ? NST : 1];  // TMA: one barrier per stage, armed with the tile's 8 KB
    // swizzle f -> f ^ ((f >> 3) & 3).  For the coalesced pieces f = 32u + lane it only touches the lane part, for the
    // thread's own pieces f = 4 lane + u only the u part: both reduce to one per-thread constant plus a compile-time offset
    const int lane_sw = lane ^ ((lane >> 3) & 3);  // coalesced piece 32u + lane lives at 32u + lane_sw
    const int xq = (lane >> 1) & 3;                // own piece 4 lane + u lives at 4 lane + (u ^ xq)
    const int wbase = warp * 32 * CH_K;  // first frame of the warp region inside a tile
    if (USE_TMA) {
        if (t == 0) {
#pragma unroll
            for (int s = 0; s < NST; s++) mbar_init(&s_bar[s], 1);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        }
    }
    __syncthreads();

    // Per-warp invariants of the slab, so that the hot loop only compares tile bases: the warp's 2 KB source region at tile base `tb` is
    // one aligned run  s_ptr0 + tb  for  s_lo <= tb <= s_hi  (tile bases are multiples of the tile: the alignment does not change),
    // and its results leave as coalesced 2 KB stores to  o_ptr0 + tb  (+ channel stride for an up-mixed copy) for  tb <= o_hi.
    int s_lo = 1, s_hi = 0;  // (tile bases are ints: the bounds are clamped into the int range)
    const float* s_ptr0 = nullptr;
    auto clamp_i = [](long long x) { return (int)max(-2000000000ll, min(2000000000ll, x)); };
    if (STREAMED) {
        if (SRC == CHAIN_SRC_BUFFER) {
            const float* p0 = chan(q.in, c, ci) + wbase;
            if ((reinterpret_cast<uintptr_t>(p0) & 15) == 0) {
                s_ptr0 = p0;
                s_lo = 0;
                s_hi = ci.nf - wbase - 32 * CH_K;  // nf is a multiple of 128 = 8 threads: the region may be ragged at the end
            }
        } else {
            const AbsnInst& o = q.absn;
            const long long off = (long long)ci.f0 + wbase - o.n_start + o.buf_offset;  // buffer index of the region's first frame at tb = 0
            const float* p0 = o.buf + (size_t)c * o.buf_stride + off;
            if (!o.loop && (reinterpret_cast<uintptr_t>(p0) & 15) == 0) {
                s_ptr0 = p0;
                s_lo = clamp_i(max(0ll, (long long)o.n_start - ci.f0 - wbase));
                s_hi = clamp_i(min((long long)ci.nf - wbase - 32 * CH_K, (long long)o.buf_len - 32 * CH_K - off));
            }
        }
    }
    auto region_src = [&](int tile_base) -> const float* {
        return (tile_base >= s_lo && tile_base <= s_hi) ? s_ptr0 + tile_base : nullptr;
    };
    const int n_out = q.out_dup > 1 ? q.out_dup : 1;
    float* const o_ptr0 = chan(q.out, q.out_dup > 1 ? 0 : c, ci) + wbase;
    int o_hi = ci.nf - wbase - 32 * CH_K;
    if (q.limit >= 0) o_hi = clamp_i(min((long long)o_hi, (long long)q.limit - ci.f0 - wbase - 32 * CH_K));
    if ((reinterpret_cast<uintptr_t>(o_ptr0) & 15) != 0 || (q.out_dup > 1 && (q.out.stride & 3) != 0)) o_hi = -1;
    // cp.async path: 16-byte pieces into the swizzled layout, per-thread gather for ragged / looping / unaligned regions
    auto stage_source = [&](int buf, int tile_base) {
        if (!STREAMED || tile_base >= slab_end) return;
        const int nw = tile_base + wbase;
        if (nw >= ci.nf) return;
        const float* gp = region_src(tile_base);
        if (gp) {
#pragma unroll
            for (int u = 0; u < CH_K / 4; u++) {
                const int f = 32 * u + lane;
                const unsigned dst = smem_u32(&s_io[buf][warp][32 * u + lane_sw]);
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(gp + 4 * f) : "memory");
            }
        } else if (nw + lane * CH_K < ci.nf) {
            chain_stage_gather<SRC>(&sm.q, c, ci, nw + lane * CH_K, &s_io[buf][warp][0], lane, xq);
        }
    };
    // TMA path: whole tile (2048 frames, 8 KB) readable as one aligned run?  (CTA-uniform, pure function)
    auto tile_src = [&](int tile_base) -> const float* {
        if (!STREAMED || tile_base + tile > ci.nf) return nullptr;
        if (SRC == CHAIN_SRC_BUFFER) {
            const float* gp = chan(q.in, c, ci) + tile_base;
            return (reinterpret_cast<uintptr_t>(gp) & 15) == 0 ? gp : nullptr;
        } else {
            const AbsnInst& o = q.absn;
            const float* src = o.buf + (size_t)c * o.buf_stride;
            const int64_t n = ci.f0 + tile_base;
            const int64_t idx = n - o.n_start + o.buf_offset;
            if (!o.loop && n >= o.n_start && idx + tile <= o.buf_len && ((reinterpret_cast<uintptr_t>(src + idx) & 15) == 0)) return src + idx;
            return nullptr;
        }
    };
    // TMA path (thread 0 only): one 8 KB bulk copy per tile, completion on the stage's mbarrier
    auto issue_bulk = [&](int buf, int tile_base) {
        if (tile_base >= slab_end) return;
        const float* gp = tile_src(tile_base);
        if (gp) {
            mbar_expect_tx(&s_bar[buf], tile * 4);
            bulk_load(&s_io[buf][0][0], gp, tile * 4, &s_bar[buf]);
        }
    };
    unsigned par = 0;  // TMA path: phase parity of every stage's barrier (bit s), flipped each time the stage is consumed
    // the slab, tile by tile.  emit = false (PRE): filter state only — nothing is stored, no layout track written
    auto run_slab = [&](const bool emit) {
    float v[CH_K];
    if (STREAMED) {
        if (USE_TMA) {
            if (t == 0)
#pragma unroll
                for (int s = 0; s < NST - 1; s++) issue_bulk(s, slab_begin + s * tile);
        } else {
#pragma unroll
            for (int s = 0; s < NST - 1; s++) {
                stage_source(s, slab_begin + s * tile);
                asm volatile("cp.async.commit_group;" ::: "memory");
            }
        }
    }
    int buf = 0;
    for (int base = slab_begin; base < slab_end; base += tile) {
        const int n0 = base + t * CH_K;
        const bool active = n0 < ci.nf;  // nf is a multiple of 128, K divides 128: a thread is fully in or out
        const int n_active = min(CH_THREADS, (ci.nf - base) / CH_K);
        const int pbuf = buf == 0 ? NST - 1 : buf - 1;  // stage of the tile before this one = stage of the tile NST-1 ahead
        if (STREAMED && !USE_TMA) {
            stage_source(pbuf, base + (NST - 1) * tile);  // prefetch while this tile is filtered
            asm volatile("cp.async.commit_group;" ::: "memory");
            asm volatile("cp.async.wait_group %0;" ::"n"(NST - 1) : "memory");  // this tile's pieces have landed ...
            __syncwarp();                                                          // ... for every lane of the warp
            if (active) {
#pragma unroll
                for (int u = 0; u < CH_K / 4; u++) {
                    const float4 a = s_io[buf][warp][4 * lane + (u ^ xq)];
                    v[4 * u] = a.x; v[4 * u + 1] = a.y; v[4 * u + 2] = a.z; v[4 * u + 3] = a.w;
                }
            }
        } else if (USE_TMA) {
            if (tile_src(base) != nullptr) {  // CTA-uniform: the tile arrived by bulk copy (all threads are active)
                mbar_wait(&s_bar[buf], (par >> buf) & 1u);
                par ^= 1u << buf;
                float4 a[CH_K / 4];
#pragma unroll
                for (int u = 0; u < CH_K / 4; u++) a[u] = s_io[buf][warp][4 * lane + (u ^ xq)];  // a[u] = piece u ^ xq
                cswap4((xq & 1) != 0, a[0], a[1]);
                cswap4((xq & 1) != 0, a[2], a[3]);
                cswap4((xq & 2) != 0, a[0], a[2]);
                cswap4((xq & 2) != 0, a[1], a[3]);
#pragma unroll
                for (int u = 0; u < CH_K / 4; u++) {
                    v[4 * u] = a[u].x; v[4 * u + 1] = a[u].y; v[4 * u + 2] = a[u].z; v[4 * u + 3] = a[u].w;
                }
            } else if (active) {
                chain_load_source<SRC>(q, c, ci, n0, v, tab2);
            }
        } else if (active) {
            chain_load_source<SRC>(q, c, ci, n0, v, tab2);
        }
        bool clean0 = true, clean1 = true;
        const bool want_clean = q.out.meta != nullptr;
        if (g0 != 1.f) {  // x * 1.0f == x bit for bit: skip the multiply (uniform branch)
#pragma unroll
            for (int j = 0; j < CH_K; j++) v[j] *= g0;
        }
        if (NB >= 1) {
            if constexpr (STREAMED) {
                // the tile's source samples are still in the staging region (it is overwritten by the results only further down)
                auto reload = [&](float x[CH_K]) {
                    float4 a[CH_K / 4];
#pragma unroll
                    for (int u = 0; u < CH_K / 4; u++) a[u] = s_io[buf][warp][4 * lane + (u ^ xq)];
                    if (USE_TMA) {  // linear layout, pieces visited in the order u ^ xq
                        cswap4((xq & 1) != 0, a[0], a[1]);
                        cswap4((xq & 1) != 0, a[2], a[3]);
                        cswap4((xq & 2) != 0, a[0], a[2]);
                        cswap4((xq & 2) != 0, a[1], a[3]);
                    }
#pragma unroll
                    for (int u = 0; u < CH_K / 4; u++) {
                        x[4 * u] = a[u].x * g0; x[4 * u + 1] = a[u].y * g0; x[4 * u + 2] = a[u].z * g0; x[4 * u + 3] = a[u].w * g0;
                    }
                };
                chain_biquad(sm, 0, cb[0][0], cb[0][1], cb[0][2], cb[0][3], cb[0][4], sm.plane[0][lane > 0 ? lane - 1 : 0], v, active, n_active, t, lane, warp, want_clean, clean0, reload);
            } else {
                chain_biquad(sm, 0, cb[0][0], cb[0][1], cb[0][2], cb[0][3], cb[0][4], sm.plane[0][lane > 0 ? lane - 1 : 0], v, active, n_active, t, lane, warp, want_clean, clean0, NoReload{});
            }
            if (g1 != 1.f) {
#pragma unroll
                for (int j = 0; j < CH_K; j++) v[j] *= g1;
            }
        }
        if (NB >= 2) {
            chain_biquad(sm, 1, cb[NB - 1][0], cb[NB - 1][1], cb[NB - 1][2], cb[NB - 1][3], cb[NB - 1][4], sm.plane[1][lane > 0 ? lane - 1 : 0], v, active,
                         n_active, t, lane, warp, want_clean, clean1, NoReload{});
            if (g2 != 1.f) {
#pragma unroll
                for (int j = 0; j < CH_K; j++) v[j] *= g2;
            }
        }
        if (SHAPER) {
            const float* curve = q.curve;
            const int cn = q.shaper_n;
            if (curve) {
#pragma unroll
                for (int j = 0; j < CH_K; j++) v[j] = cn == 0 ? 0.f : shaper_apply(curve, cn, v[j]);
            }
#pragma unroll
            for (int j = 0; j < CH_K; j++) v[j] *= g3;
        }
        if (emit && q.out.meta && active && (n0 & 127) == 0) {
            // Layout track of the chain's output, row c (this CTA's channel), for the quantum this thread starts: the nodes of the
            // chain in order.  source: silent outside its schedule; gain: silent in -> silent out, a gain of (about) zero silences
            // (gain.rs:153-169); biquad: silent once its input is silent AND its state has no normal value left, until then it keeps
            // its channels (biquad_filter.rs:778-815); wave-shaper: passes silence on only if its curve maps 0 to 0, else it answers
            // on the one channel a silent quantum has (waveshaper.rs:395-400).
            const int qi = meta_qi(ci, n0);
            const int64_t f = ci.f0 + n0;
            bool sl;
            int cnt = q.ch;
            if (SRC == CHAIN_SRC_BUFFER) {
                sl = buf_silent(q.in, q.ch, qi);
                cnt = buf_count(q.in, q.ch, qi);
            } else if (SRC == CHAIN_SRC_OSC) {
                sl = q.osc.n_stop <= f || q.osc.n_first >= f + 128;
            } else if (SRC == CHAIN_SRC_CONST) {
                sl = q.cst.n_stop <= f || q.cst.n_first >= f + 128;
            } else {
                sl = q.absn.n_stop <= f || q.absn.n_start >= f + 128;
            }
            if (g0 == 0.f) sl = true;
            if (sl) cnt = 1;
            if (NB >= 1) {
                if (sl && !clean0) {
                    sl = false;
                    cnt = q.ch;
                }
                if (g1 == 0.f) sl = true;
                if (sl) cnt = 1;
            }
            if (NB >= 2) {
                if (sl && !clean1) {
                    sl = false;
                    cnt = q.ch;
                }
                if (g2 == 0.f) sl = true;
                if (sl) cnt = 1;
            }
            if (SHAPER) {
                if (sl && q.curve && !q.shaper_keeps_silence) sl = false;  // (cnt stays 1)
                if (g3 == 0.f) sl = true;
            }
            meta_put(q.out, c, qi, cnt, sl || c >= cnt);
        }
        if (emit) {
            // results: through the warp's staging region (the source pieces of this tile are consumed), so that global
            // memory sees whole 2 KB regions; per-thread stores for ragged / unaligned / length-limited regions
            const int nw = base + wbase;
            // TMA path: the whole tile leaves as one 8 KB bulk store per output channel (CTA-uniform condition)
            const bool tile_out = USE_TMA && base + tile <= ci.nf && (q.limit < 0 || ci.f0 + base + tile <= q.limit) &&
                                  (reinterpret_cast<uintptr_t>(chan(q.out, q.out_dup > 1 ? 0 : c, ci) + base) & 15) == 0 &&
                                  (q.out_dup <= 1 || (q.out.stride & 3) == 0);
            if (USE_TMA) {
                if (tile_out) {
                    float4 a[CH_K / 4];
#pragma unroll
                    for (int u = 0; u < CH_K / 4; u++) a[u] = make_float4(v[4 * u], v[4 * u + 1], v[4 * u + 2], v[4 * u + 3]);
                    cswap4((xq & 2) != 0, a[0], a[2]);
                    cswap4((xq & 2) != 0, a[1], a[3]);
                    cswap4((xq & 1) != 0, a[0], a[1]);
                    cswap4((xq & 1) != 0, a[2], a[3]);  // a[u] = piece u ^ xq
#pragma unroll
                    for (int u = 0; u < CH_K / 4; u++) s_io[buf][warp][4 * lane + (u ^ xq)] = a[u];
                    fence_proxy_async_smem();  // generic-proxy writes -> visible to the bulk store's async-proxy reads
                } else if (active) {
                    const int64_t nabs = ci.f0 + n0;
                    for (int oc = 0; oc < n_out; oc++) {
                        float* out = chan(q.out, q.out_dup > 1 ? oc : c, ci) + n0;
#pragma unroll
                        for (int j = 0; j < CH_K; j++)
                            if (q.limit < 0 || nabs + j < q.limit) out[j] = v[j];
                    }
                }
                __syncthreads();  // the tile is staged (and the carried filter state of this tile is visible to the next)
                if (t == 0) {
                    if (tile_out)
                        for (int oc = 0; oc < n_out; oc++) bulk_store(chan(q.out, q.out_dup > 1 ? oc : c, ci) + base, &s_io[buf][0][0], tile * 4);
                    bulk_commit();        // this tile's stores (possibly none) form one group ...
                    bulk_wait_read<1>();  // ... and the group of the tile before has finished reading its stage: refill it
                    issue_bulk(pbuf, base + (NST - 1) * tile);
                }
            } else if (base <= o_hi) {  // warp-uniform
                __syncwarp();
#pragma unroll
                for (int u = 0; u < CH_K / 4; u++)
                    s_io[buf][warp][4 * lane + (u ^ xq)] = make_float4(v[4 * u], v[4 * u + 1], v[4 * u + 2], v[4 * u + 3]);
                __syncwarp();
                for (int oc = 0; oc < n_out; oc++) {
                    float4* out = reinterpret_cast<float4*>(o_ptr0 + (size_t)oc * q.out.stride + base);
#pragma unroll
                    for (int u = 0; u < CH_K / 4; u++) {
                        out[32 * u + lane] = s_io[buf][warp][32 * u + lane_sw];
                    }
                }
                __syncwarp();
            } else if (active) {
                const int64_t nabs = ci.f0 + n0;
                for (int oc = 0; oc < n_out; oc++) {
                    float* out = chan(q.out, q.out_dup > 1 ? oc : c, ci) + n0;
#pragma unroll
                    for (int j = 0; j < CH_K; j++)
                        if (q.limit < 0 || nabs + j < q.limit) out[j] = v[j];
                }
            }
        }
        if (NB > 0 && !USE_TMA) __syncthreads();  // the carried state of this tile is visible before the next tile reads it
        buf = buf + 1 == NST ? 0 : buf + 1;
    }
    if (STREAMED && !USE_TMA) asm volatile("cp.async.wait_group 0;" ::: "memory");  // (prefetches past the slab's end are empty groups)
    };
    if constexpr (PRE && NB == 1 && !TMA) {
        if (pre) {
            if (t == 0) sm.flushed = 0;
            __syncthreads();
            run_slab(false);  // leaves the slab's zero-state end state in sm.state[0]
            __syncthreads();
            if (!first_slab) wait_handoff();
            if (t == 0) {
                double sin_[4], g[16], h[16];
                const ScanCoef& scf = coefs[q.bq[0].coef];
                for (int i = 0; i < 4; i++) sin_[i] = first_slab ? q.bq[0].state[4 * c + i] : __ldcg(sc.handoff + ho * (CHAIN_MAX_BIQUADS * 4) + i);
                for (int i = 0; i < 16; i++) g[i] = scf.GL[i];
                for (int sq = 0; sq < sc.pre_log2; sq++) {  // G^(2L) = G^L G^L: slabs of CHAIN_PRE_TILES << pre_log2 tiles
                    for (int r = 0; r < 4; r++)
                        for (int cc = 0; cc < 4; cc++) {
                            double a = 0.;
                            for (int k = 0; k < 4; k++) a = fma(g[4 * r + k], g[4 * k + cc], a);
                            h[4 * r + cc] = a;
                        }
                    for (int i = 0; i < 16; i++) g[i] = h[i];
                }
                for (int r = 0; r < 4; r++) {
                    double o = sm.state[0][r];  // what the slab's own input leaves behind
                    if (!sm.flushed)            // (a slab that flushed a NaN / Inf ends in the same state wherever it started)
                        for (int k = 0; k < 4; k++) o = fma(g[4 * r + k], sin_[k], o);
                    __stcg(sc.handoff + (ho + 1) * (CHAIN_MAX_BIQUADS * 4) + r, o);
                }
                __threadfence();
                asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(sc.flags + ho + 1), "r"(sc.epoch) : "memory");
                for (int i = 0; i < 4; i++) sm.state[0][i] = sin_[i];
            }
            __syncthreads();
        }
    }
    run_slab(true);
    if (USE_TMA && t == 0) bulk_wait_read<0>();  // shared memory stays valid until the last bulk store has read it
    // carry the filter state: to the next slab of this launch, or (last slab) to the next chunk
    if (NB > 0) {
        if (last_slab) {
#pragma unroll
            for (int k = 0; k < NB; k++)
                if (t < 4) q.bq[k].state[4 * c + t] = sm.state[k][t];
        } else if (!pre) {
            if (t < 4 * NB) __stcg(sc.handoff + (ho + 1) * (CHAIN_MAX_BIQUADS * 4) + t, sm.state[t >> 2][t & 3]);
            __threadfence();
            __syncthreads();
            if (t == 0) asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(sc.flags + ho + 1), "r"(sc.epoch) : "memory");
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
// k_voice_sum — Graph::render's edge summation (graph.rs:489-535, AudioRenderQuantum::add, quantum.rs:532-569) for a port fed by
// many oscillator -> [biquad] -> gain voices (many_oscillators.rs, the north_star graph), fused with the voices themselves: the
// voices are never written to memory.  f32 addition does not associate and the reference adds the edges one after the other, so the
// sum of a frame is a serial chain over the voices; the parallelism is over time.  A work item is (2048-frame tile, group): the CTA
// keeps the tile's partial sum in registers (16 frames per thread) and walks the group's voices in edge order — oscillator into
// registers, biquad as the block scan of k_chain, gain, add.  The biquad state a voice leaves at the end of tile s is what tile s + 1
// of the same voice starts from: items are handed out in ticket order, tile-major, so the CTA of tile s - 1 is always running or
// done when tile s starts, and it publishes, voice by voice, the state it ends with (two slots per voice, indexed by tile parity)
// and a progress counter "voices finished" that tile s polls — only when its cached copy does not already cover the voice it is at:
// the CTAs of consecutive tiles follow each other one voice apart, like a pipeline along the time axis.
// Replaces, for such ports, k_chain (one 8 KB store per voice tile) + k_mix (one 8 KB load per voice tile).
// ---------------------------------------------------------------------------------------------------------
#ifndef WAE_VS_MINB
#define WAE_VS_MINB 5
#endif
template <int NB>
__global__ void __launch_bounds__(CH_THREADS, WAE_VS_MINB * 128 / CH_THREADS) k_voice_sum(const ChainInst* __restrict__ insts, const ScanCoef* __restrict__ coefs,
                                                                                          const VoiceGroup* __restrict__ groups, int n_groups, ChunkInfo ci,
                                                                                          ChainSched sc) {
    __shared__ ChainSmem sm;
    __shared__ int s_item;
    __shared__ float2 s_table2[2048];
    const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
    if (t == 0) {
        const unsigned tk = atomicAdd(sc.ticket, 1u);
        if (tk == gridDim.x - 1) atomicExch(sc.ticket, 0u);  // the last ticket of this launch: leave the counter ready for the next one
        s_item = (int)tk;
    }
    __syncthreads();
    const int item = s_item;
    const int slab = item / n_groups, gi = item - slab * n_groups;
    const VoiceGroup grp = groups[gi];
    constexpr int tile = CH_THREADS * CH_K;
    const int base = slab * tile;
    if (base >= ci.nf) return;
    const int n0 = base + t * CH_K;
    const bool active = n0 < ci.nf;
    const int n_active = min(CH_THREADS, (ci.nf - base) / CH_K);
    const bool first_slab = slab == 0, last_slab = base + tile >= ci.nf;
    const unsigned tag = (sc.epoch & 0xfffu) << 20;
    const unsigned* prog_prev = sc.flags + (size_t)gi * sc.slab_stride + (slab > 0 ? slab - 1 : 0);
    unsigned* prog_mine = sc.flags + (size_t)gi * sc.slab_stride + slab;
    unsigned seen = 0;  // (thread 0) voices the tile before this one is known to have finished
    const float* cur_table = nullptr;
    float acc[CH_K];
#pragma unroll
    for (int j = 0; j < CH_K; j++) acc[j] = 0.f;
    // The record and the filter constants of the NEXT voice are loaded into registers while the current voice is computed (one 4-byte
    // word of the 512-byte record, one or two doubles of the 152 scan constants per thread) and put into shared memory at the top of
    // the next iteration: the voice loop never waits for a table read.  Voice k of the stage owns coefficient set k (plan_graph).
    constexpr int REC_W = (int)(sizeof(ChainInst) / 4 + CH_THREADS - 1) / CH_THREADS;
    constexpr int PL_W = (128 + CH_THREADS - 1) / CH_THREADS;
    static_assert(CH_THREADS >= 24, "scan constants: one of Pshfl / Pwarp per thread");
    int rec_n[REC_W];
    double pl_n[PL_W], pw_n = 0.;
    auto prefetch = [&](int vi) {
        const int inst = grp.first + vi;
        const int* src = reinterpret_cast<const int*>(insts + inst);
#pragma unroll
        for (int i = 0; i < REC_W; i++) rec_n[i] = (t + i * CH_THREADS) < (int)(sizeof(ChainInst) / 4) ? __ldg(src + t + i * CH_THREADS) : 0;
        if (NB > 0) {
            const ScanCoef& scf = coefs[inst];
#pragma unroll
            for (int i = 0; i < PL_W; i++) pl_n[i] = (t + i * CH_THREADS) < 128 ? (&scf.Plane[0][0])[t + i * CH_THREADS] : 0.;
            if (t < 20) pw_n = (&scf.Pshfl[0][0])[t];
            else if (t < 24) pw_n = scf.Pwarp[t - 20];
        }
    };
    prefetch(0);
    // No hand-off duty sits in front of a CTA barrier.  Incoming (warp 0): the state a voice enters the tile with is needed only inside
    // chain_biquad (behind ITS first barrier), so it is fetched after barrier (1), while the other warps already compute their
    // oscillator frames; whether the tile before this one has finished voice vi + 1 as well is asked at the start of voice vi (a load
    // whose result is not waited for) and looked at when voice vi is done: if so — the usual case once the CTAs of consecutive tiles
    // have settled a voice apart — the state of vi + 1 is loaded right then, a whole voice before it is needed; only when it has not
    // does warp 0 poll at the start of vi + 1.  Outgoing (lane 0 of warp 1): two 16-byte stores + a release store of the progress
    // counter, after barrier (1) of the next voice.  The counter is read with relaxed loads (no L1 invalidation per poll) and the
    // state with L2 loads issued only once the counter's value is known: the writer's release orders state before counter at L2.
    const bool handoff_in = NB > 0 && !first_slab, handoff_out = NB > 0 && !last_slab;
    auto poll_ok = [&](unsigned x, int v) { return (x & 0xfff00000u) == tag && (x & 0xfffffu) > (unsigned)v; };
    double st_next = 0.;        // (lanes 0-3 of warp 0) incoming state of the next voice, when it could be loaded early
    bool st_next_valid = false;
    constexpr int PUB_T = CH_WARPS > 1 ? 32 : 0;     // the publishing thread
    double pe0 = 0., pe1 = 0., pe2 = 0., pe3 = 0.;  // (thread PUB_T) end state of the voice before, not yet published
    double* pub_ptr = nullptr;
    int pub_vi = -1;
    auto publish = [&]() {  // thread PUB_T
        if (pub_vi < 0) return;
        if (last_slab) {  // carried to the next chunk
            pub_ptr[0] = pe0; pub_ptr[1] = pe1; pub_ptr[2] = pe2; pub_ptr[3] = pe3;
        } else {
            double* dst = sc.handoff + ((size_t)(grp.first + pub_vi) * 2 + ((slab + 1) & 1)) * 4;
            asm volatile("st.global.cg.v2.f64 [%0], {%1, %2};" ::"l"(dst), "d"(pe0), "d"(pe1) : "memory");
            asm volatile("st.global.cg.v2.f64 [%0], {%1, %2};" ::"l"(dst + 2), "d"(pe2), "d"(pe3) : "memory");
            asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(prog_mine), "r"(tag | (unsigned)(pub_vi + 1)) : "memory");
        }
        pub_vi = -1;
    };
    for (int vi = 0; vi < grp.n_voices; vi++) {
        const int inst = grp.first + vi;
        // (everyone is past barrier (3) of the voice before: its record and constants are dead)
#pragma unroll
        for (int i = 0; i < REC_W; i++)
            if ((t + i * CH_THREADS) < (int)(sizeof(ChainInst) / 4)) reinterpret_cast<int*>(&sm.q)[t + i * CH_THREADS] = rec_n[i];
        if (NB > 0) {
#pragma unroll
            for (int i = 0; i < PL_W; i++)
                if ((t + i * CH_THREADS) < 128) (&sm.plane[0][0][0])[t + i * CH_THREADS] = pl_n[i];
            if (t < 24) sm.P[0][t] = pw_n;  // [0, 20): Pshfl, [20, 24): Pwarp
        }
        __syncthreads();  // (1) record and constants of the voice are in shared memory (nothing global was waited for)
        if (vi + 1 < grp.n_voices) prefetch(vi + 1);
        const ChainInst& q = sm.q;
        double st_cur = 0.;
        unsigned xa = 0;
        if (NB > 0 && t == PUB_T) publish();  // the voice before this one
        if (NB > 0 && warp == 0) {
            if (st_next_valid) {
                st_cur = st_next;
            } else if (first_slab) {
                if (lane < 4) st_cur = q.bq[0].state[lane];  // (carried from the chunk before)
            } else {
                if (lane == 0 && seen <= (unsigned)vi) {
                    for (;;) {
                        unsigned x;
                        asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(x) : "l"(prog_prev) : "memory");
                        if (poll_ok(x, vi)) {
                            seen = x & 0xfffffu;
                            break;
                        }
                        __nanosleep(20);
                    }
                }
                __syncwarp();
                if (lane < 4) st_cur = __ldcg(sc.handoff + ((size_t)inst * 2 + (slab & 1)) * 4 + lane);
            }
            // has the tile before this one finished the NEXT voice as well?  asked now, looked at when this voice is done
            if (handoff_in && lane == 0 && vi + 1 < grp.n_voices && seen <= (unsigned)(vi + 1))
                asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(xa) : "l"(prog_prev));
        }
        const float2* tab2 = nullptr;
        if ((q.osc.type == 0 || q.osc.type == 4) && q.osc.table_len == 2048) {
            if (q.osc.table != cur_table) {  // (CTA-uniform) sine voices share one table: staged once per CTA
                const float* gt = q.osc.table;
                for (int i = t; i < 2048; i += CH_THREADS) s_table2[i] = make_float2(__ldg(gt + i), __ldg(gt + ((i + 1) & 2047)));
                cur_table = gt;
                __syncthreads();
            }
            tab2 = s_table2;
        }
        double cb[5] = {0., 0., 0., 0., 0.};
        double* st_ptr = nullptr;
        if (NB > 0) {
            const ChainBiquad& bq = q.bq[0];
            cb[0] = bq.b0; cb[1] = bq.b1; cb[2] = bq.b2; cb[3] = bq.a1; cb[4] = bq.a2;
            st_ptr = bq.state;
        }
        const float g0 = q.g[0], g1 = q.g[1];
        float v[CH_K];
        if (active) chain_load_source<CHAIN_SRC_OSC>(q, 0, ci, n0, v, tab2);
        if (g0 != 1.f) {
#pragma unroll
            for (int j = 0; j < CH_K; j++) v[j] *= g0;
        }
        if (NB > 0) {
            if (warp == 0 && lane < 4) sm.state[0][lane] = st_cur;  // (read behind chain_biquad's first barrier)
            bool clean = true;
            chain_biquad(sm, 0, cb[0], cb[1], cb[2], cb[3], cb[4], sm.plane[0][lane > 0 ? lane - 1 : 0], v, active, n_active, t, lane, warp, false, clean, NoReload{});
            if (g1 != 1.f) {
#pragma unroll
                for (int j = 0; j < CH_K; j++) v[j] *= g1;
            }
        }
        if (active) {
            if (vi == 0) {  // the first edge is taken as it is (AudioRenderQuantum::add onto a silent input = copy)
#pragma unroll
                for (int j = 0; j < CH_K; j++) acc[j] = v[j];
            } else {
#pragma unroll
                for (int j = 0; j < CH_K; j++) acc[j] += v[j];
            }
        }
        if (NB > 0 && first_slab && warp == 0) {  // the head of the pipeline sets everyone's pace: its next state is loaded a voice early too
            st_next_valid = vi + 1 < grp.n_voices;
            if (st_next_valid && lane < 4) st_next = insts[inst + 1].bq[0].state[lane];
        }
        if (handoff_in && warp == 0) {
            st_next_valid = false;
            if (vi + 1 < grp.n_voices) {
                if (lane == 0 && seen <= (unsigned)(vi + 1) && poll_ok(xa, vi + 1)) seen = xa & 0xfffffu;
                st_next_valid = __shfl_sync(0xffffffffu, seen > (unsigned)(vi + 1) ? 1 : 0, 0) != 0;
                if (st_next_valid && lane < 4) st_next = __ldcg(sc.handoff + ((size_t)(inst + 1) * 2 + (slab & 1)) * 4 + lane);
            }
        }
        __syncthreads();  // (3) everyone is done with the voice's record and constants; its end state is in sm.state[0]
        if (NB > 0 && t == PUB_T) {
            pe0 = sm.state[0][0]; pe1 = sm.state[0][1]; pe2 = sm.state[0][2]; pe3 = sm.state[0][3];
            pub_ptr = st_ptr;
            pub_vi = vi;
        }
    }
    if (NB > 0 && t == PUB_T) publish();
    (void)handoff_out;
    if (!active) return;
    const int64_t nabs = ci.f0 + n0;
    for (int oc = 0; oc < grp.out_dup; oc++) {
        float* out = chan(grp.out, oc, ci) + n0;
        if ((reinterpret_cast<uintptr_t>(out) & 15) == 0 && (grp.limit < 0 || nabs + CH_K <= grp.limit)) {
#pragma unroll
            for (int u = 0; u < CH_K / 4; u++) reinterpret_cast<float4*>(out)[u] = make_float4(acc[4 * u], acc[4 * u + 1], acc[4 * u + 2], acc[4 * u + 3]);
        } else {
#pragma unroll
            for (int j = 0; j < CH_K; j++)
                if (grp.limit < 0 || nabs + j < grp.limit) out[j] = acc[j];
        }
    }
}

// Oscillator with automated / audio-rate frequency or detune (oscillator.rs:447-459,511-557): the phase of frame n is
// the running sum of the per-frame increments f[n] * 2^(d[n]/1200) / sr.  One CTA per oscillator; tiles of 256 x 8
// frames, Kogge-Stone scan of the tile's increments in f64, the phase is carried from tile to tile and chunk to chunk.
__global__ void __launch_bounds__(256) k_osc_arate(const OscArInst* __restrict__ insts, int n_inst, ChunkInfo ci) {
    __shared__ double s_sum[256];
    __shared__ double s_carry;
    const OscArInst q = insts[blockIdx.x];
    const OscInst& o = q.base;
    float* out = chan(o.out, 0, ci);
    const float* ft = q.freq.p ? chan(q.freq, 0, ci) : nullptr;
    const float* dtk = q.detune.p ? chan(q.detune, 0, ci) : nullptr;
    const int t = threadIdx.x;
    const double sr = (double)q.sample_rate, nyq = sr / 2.;
    if (t == 0) s_carry = *q.phase;  // zeroed before every run
    __syncthreads();
    for (int base = 0; base < ci.nf; base += 2048) {
        const int n0 = base + t * 8;
        double inc[8];
        bool act[8], oob[8];
        double local = 0.;
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const int n = n0 + j;
            const int64_t na = ci.f0 + n;
            act[j] = n < ci.nf && na >= o.n_first && na < o.n_stop;
            double cf = 0.;
            if (n < ci.nf) {
                float f = ft ? ft[n] : q.f_val, d = dtk ? dtk[n] : q.d_val;
                cf = (double)f * exp2((double)d / 1200.);  // get_computed_freq, oscillator.rs:30-32
            }
            oob[j] = fabs(cf) >= nyq;
            inc[j] = cf / sr;
            double add = act[j] ? inc[j] : 0.;
            if (act[j] && na == o.n_first) add += q.start_ratio * inc[j];  // sub-sample start: phase = incr * ratio
            local += add;
        }
        s_sum[t] = local;
        __syncthreads();
        for (int off = 1; off < 256; off <<= 1) {
            double v = t >= off ? s_sum[t - off] : 0.;
            __syncthreads();
            s_sum[t] += v;
            __syncthreads();
        }
        double ph = s_carry + (t > 0 ? s_sum[t - 1] : 0.);
        float v[8];
#pragma unroll
        for (int j = 0; j < 8; j++) {
            const int64_t na = ci.f0 + n0 + j;
            double p = ph;
            if (act[j] && na == o.n_first) p += q.start_ratio * inc[j];
            p -= floor(p);
            if (p >= 1.) p = 0.;
            v[j] = (act[j] && !oob[j]) ? osc_sample(o, p, inc[j]) : 0.f;
            if (act[j]) ph = p + inc[j];
        }
        if (n0 < ci.nf) {
            *reinterpret_cast<float4*>(out + n0) = make_float4(v[0], v[1], v[2], v[3]);
            *reinterpret_cast<float4*>(out + n0 + 4) = make_float4(v[4], v[5], v[6], v[7]);
        }
        __syncthreads();
        if (t == 255) {
            double c = s_carry + s_sum[255];
            s_carry = c - floor(c);
        }
        __syncthreads();
    }
    if (t == 0) *q.phase = s_carry;
}

// calculate_coefs on the device (src/node/biquad_filter.rs:28-390) for per-frame coefficients
struct BqC {
    double b0, b1, b2, a1, a2;
};
DEVI BqC bq_norm(double b0, double b1, double b2, double a0, double a1, double a2) {
    double s = 1. / a0;
    return BqC{b0 * s, b1 * s, b2 * s, a1 * s, a2 * s};
}
DEVI BqC bq_coefs(int type, double sample_rate, double f0, double gain, double q) {
    const BqC wire{1., 0., 0., 0., 0.}, zero{0., 0., 0., 0., 0.};
    const double PI64 = 3.14159265358979323846;
    double f = f0 / (sample_rate / 2.);
    f = f < 0. ? 0. : (f > 1. ? 1. : f);
    const double w0 = PI64 * f, sn = sin(w0), c = cos(w0);
    const double A = pow(10., gain / 40.);
    switch (type) {
        case 0: {
            if (f == 1.) return wire;
            double a = sn / (2. * pow(10., q / 20.)), beta = (1. - c) / 2.;
            return bq_norm(beta, 2. * beta, beta, 1. + a, -2. * c, 1. - a);
        }
        case 1: {
            if (f == 1.) return zero;
            if (f == 0.) return wire;
            double a = sn / (2. * pow(10., q / 20.)), beta = (1. + c) / 2.;
            return bq_norm(beta, -2. * beta, beta, 1. + a, -2. * c, 1. - a);
        }
        case 2: {
            if (!(f > 0. && f < 1.)) return zero;
            if (!(q > 0.)) return wire;
            double a = sn / (2. * q);
            return bq_norm(a, 0., -a, 1. + a, -2. * c, 1. - a);
        }
        case 3: {
            if (!(f > 0. && f < 1.)) return wire;
            if (!(q > 0.)) return zero;
            double a = sn / (2. * q);
            return bq_norm(1., -2. * c, 1., 1. + a, -2. * c, 1. - a);
        }
        case 4: {
            if (!(f > 0. && f < 1.)) return wire;
            if (!(q > 0.)) return BqC{-1., 0., 0., 0., 0.};
            double a = sn / (2. * q);
            return bq_norm(1. - a, -2. * c, 1. + a, 1. + a, -2. * c, 1. - a);
        }
        case 5: {
            if (!(f > 0. && f < 1.)) return wire;
            if (!(q > 0.)) return BqC{A * A, 0., 0., 0., 0.};
            double a = sn / (2. * q);
            return bq_norm(1. + a * A, -2. * c, 1. - a * A, 1. + a / A, -2. * c, 1. - a / A);
        }
        case 6: {
            if (f == 1.) return BqC{A * A, 0., 0., 0., 0.};
            if (f == 0.) return wire;
            double as = sn / 2. * 1.41421356237309504880168872420969808;
            double tt = 2. * as * sqrt(A), ap = A + 1., am = A - 1.;
            return bq_norm(A * (ap - am * c + tt), 2. * A * (am - ap * c), A * (ap - am * c - tt), ap + am * c + tt, -2. * (am + ap * c),
                           ap + am * c - tt);
        }
        default: {
            if (f == 1.) return wire;
            if (!(f > 0.)) return BqC{A * A, 0., 0., 0., 0.};
            double as = sn / 2. * 1.41421356237309504880168872420969808;
            double tt = 2. * as * sqrt(A), ap = A + 1., am = A - 1.;
            return bq_norm(A * (ap + am * c + tt), -2. * A * (am + ap * c), A * (ap + am * c - tt), ap - am * c + tt, 2. * (am - ap * c),
                           ap - am * c - tt);
        }
    }
}

// BiquadFilter with automated parameters, step 1: the coefficients of every frame (biquad_filter.rs:837-855), one thread per frame.
// The formulas are a function of the frame's parameter values only, so they do not belong in the serial recurrence.
__global__ void __launch_bounds__(256) k_biquad_coefs(const BiquadArInst* __restrict__ insts, int n_inst, ChunkInfo ci) {
    for (int ii = blockIdx.y; ii < n_inst; ii += gridDim.y) {
        const BiquadArInst& q = insts[ii];
        const int n = blockIdx.x * blockDim.x + threadIdx.x;
        if (n >= ci.nf) continue;
        const float vq = q.q.p ? chan(q.q, 0, ci)[n] : q.q_val, vd = q.detune.p ? chan(q.detune, 0, ci)[n] : q.detune_val;
        const float vf = q.freq.p ? chan(q.freq, 0, ci)[n] : q.freq_val, vg = q.gain.p ? chan(q.gain, 0, ci)[n] : q.gain_val;
        const float computed = vd != 0.f ? vf * exp2f(vd / 1200.f) : vf;  // get_computed_freq, biquad_filter.rs:393-399
        const BqC cf = bq_coefs(q.type, (double)q.sample_rate, (double)computed, (double)vg, (double)vq);
        double* base = reinterpret_cast<double*>(q.coefs.p) + ci.sub + n;
        const size_t cs = q.coefs.stride;  // doubles between coefficient planes
        base[0] = cf.b0;
        base[cs] = cf.b1;
        base[2 * cs] = cf.b2;
        base[3 * cs] = cf.a1;
        base[4 * cs] = cf.a2;
    }
}
// step 2: the recurrence with those coefficients, one WARP per (instance, channel), a quantum at a time.  The lanes stage the quantum's
// coefficients and input in shared memory with coalesced loads (the next quantum's loads are already in flight in registers).  With
// per-frame coefficients the filter is still linear in its state:  (y[n], y[n-1]) = M_n (y[n-1], y[n-2]) + (t_n, 0),
// M_n = [[-a1_n, -a2_n], [1, 0]],  t_n = (b0_n x[n] + b1_n x[n-1]) + b2_n x[n-2]  — so the quantum is a scan over affine maps: every lane
// composes the maps of its four frames, a Kogge-Stone scan over the 32 lanes gives each lane the map from the quantum's start to its
// first frame, and the lane then runs its four frames from that state in the reference's own operation order (biquad_filter.rs:869-883,
// with its flush of non-normal values).  About 25 dependent f64 operations per quantum instead of 640 (a dependent f64 operation
// of a lone warp costs on the order of 100 cycles; "Substractive Synth", 64 graphs x 120 s, is the case that needs it).
// Differs from the serial evaluation by the re-association of the state carried between lanes (~1e-16 relative); a NaN / Inf going
// through the recurrence (the reference recovers from it sample by sample) sends the quantum to the serial code, which stays below.
constexpr int BQA_WARPS = 2;
struct Aff2 {  // s -> A s + b
    double a00, a01, a10, a11, b0, b1;
};
DEVI Aff2 aff_after(const Aff2& g, const Aff2& f) {  // g o f: first f, then g
    Aff2 r;
    r.a00 = fma(g.a00, f.a00, g.a01 * f.a10);
    r.a01 = fma(g.a00, f.a01, g.a01 * f.a11);
    r.a10 = fma(g.a10, f.a00, g.a11 * f.a10);
    r.a11 = fma(g.a10, f.a01, g.a11 * f.a11);
    r.b0 = fma(g.a00, f.b0, fma(g.a01, f.b1, g.b0));
    r.b1 = fma(g.a10, f.b0, fma(g.a11, f.b1, g.b1));
    return r;
}
DEVI Aff2 aff_shfl_up(const Aff2& v, int d) {
    Aff2 r;
    r.a00 = __shfl_up_sync(0xffffffffu, v.a00, d); r.a01 = __shfl_up_sync(0xffffffffu, v.a01, d);
    r.a10 = __shfl_up_sync(0xffffffffu, v.a10, d); r.a11 = __shfl_up_sync(0xffffffffu, v.a11, d);
    r.b0 = __shfl_up_sync(0xffffffffu, v.b0, d);   r.b1 = __shfl_up_sync(0xffffffffu, v.b1, d);
    return r;
}
__global__ void __launch_bounds__(32 * BQA_WARPS) k_biquad_arate(const BiquadArInst* __restrict__ insts, int n_inst, int max_ch, ChunkInfo ci) {
    __shared__ __align__(16) double s_cf[BQA_WARPS][5][128];
    __shared__ __align__(16) float s_x[BQA_WARPS][128];
    __shared__ __align__(16) float s_y[BQA_WARPS][128];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int t = blockIdx.x * BQA_WARPS + wib;
    const int ii = t / max_ch, c = t % max_ch;
    if (ii >= n_inst) return;
    const BiquadArInst q = insts[ii];
    if (c >= q.ch) return;
    const float* in = chan(q.in, c, ci);
    float* out = chan(q.out, c, ci);
    double* st = q.state + 4 * c;
    double x1 = st[0], x2 = st[1], y1 = st[2], y2 = st[3];  // (every lane keeps a copy of the carried state)
    const double* cbase = reinterpret_cast<const double*>(q.coefs.p) + ci.sub;
    const size_t cs = q.coefs.stride;
    const bool dyn = q.in.meta != nullptr;
    int len = dyn ? q.dyn_len[c] : q.ch;
    double (*cf)[128] = s_cf[wib];
    float* sx = s_x[wib];
    float* sy = s_y[wib];
    // frames lane + 32 k of the quantum at n0 (k < 4), zero past the chunk
    double pre[5][4];
    float prex[4];
    auto fetch = [&](int n0) {
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const int n = n0 + lane + 32 * k;
            const bool ok = n < ci.nf;
#pragma unroll
            for (int j = 0; j < 5; j++) pre[j][k] = ok ? cbase[(size_t)j * cs + n] : 0.;
            prex[k] = ok ? in[n] : 0.f;
        }
    };
    auto step = [](double tt, double a1, double a2, double ym1, double ym2, bool& bad) {
        double y = __dsub_rn(__dsub_rn(tt, __dmul_rn(a1, ym1)), __dmul_rn(a2, ym2));
        const double ay = fabs(y);
        if (!(ay <= 1.7976931348623157e308)) bad = true;  // NaN / Inf: the states handed between the lanes are poisoned too
        if (!(ay >= 2.2250738585072014e-308 && ay <= 1.7976931348623157e308)) y = 0.;
        return y;
    };
    fetch(0);
    for (int n0 = 0; n0 < ci.nf; n0 += 128) {
#pragma unroll
        for (int k = 0; k < 4; k++) {
#pragma unroll
            for (int j = 0; j < 5; j++) cf[j][lane + 32 * k] = pre[j][k];
            sx[lane + 32 * k] = prex[k];
        }
        __syncwarp();
        if (n0 + 128 < ci.nf) fetch(n0 + 128);  // in flight while this quantum is filtered
        const int cnt = min(128, ci.nf - n0);     // (a multiple of 128: the render is padded to whole quanta)
        bool skip = false, absent = false;
        if (dyn) {  // (identical in every lane; lane 0 writes the layout track)
            BufRef none = q.out;
            if (lane != 0) none.meta = nullptr;
            filter_layout_step(q.in, none, q.ch, c, meta_qi(ci, n0), len, isnormal_d(x1) || isnormal_d(x2) || isnormal_d(y1) || isnormal_d(y2), skip, absent);
            if (c >= len) x1 = x2 = y1 = y2 = 0.;
        }
        if (skip) {
            *reinterpret_cast<float4*>(&sy[4 * lane]) = make_float4(0.f, 0.f, 0.f, 0.f);
        } else {
            const int i = 4 * lane;
            double cq[5][4];
#pragma unroll
            for (int j = 0; j < 5; j++) {
                const double2 lo = *reinterpret_cast<const double2*>(&cf[j][i]), hi = *reinterpret_cast<const double2*>(&cf[j][i + 2]);
                cq[j][0] = lo.x, cq[j][1] = lo.y, cq[j][2] = hi.x, cq[j][3] = hi.y;
            }
            const float4 xf = *reinterpret_cast<const float4*>(&sx[i]);
            const double xa = absent ? 0. : (double)xf.x, xb = absent ? 0. : (double)xf.y, xc = absent ? 0. : (double)xf.z,
                         xd = absent ? 0. : (double)xf.w;
            // the two inputs before this lane's frames: the carried state (lane 0) or the neighbour's last two
            const double pm1 = lane == 0 ? x1 : (absent ? 0. : (double)sx[i - 1]), pm2 = lane == 0 ? x2 : (absent ? 0. : (double)sx[i - 2]);
            const double t0 = __dadd_rn(__dadd_rn(__dmul_rn(cq[0][0], xa), __dmul_rn(cq[1][0], pm1)), __dmul_rn(cq[2][0], pm2));
            const double t1 = __dadd_rn(__dadd_rn(__dmul_rn(cq[0][1], xb), __dmul_rn(cq[1][1], xa)), __dmul_rn(cq[2][1], pm1));
            const double t2 = __dadd_rn(__dadd_rn(__dmul_rn(cq[0][2], xc), __dmul_rn(cq[1][2], xb)), __dmul_rn(cq[2][2], xa));
            const double t3 = __dadd_rn(__dadd_rn(__dmul_rn(cq[0][3], xd), __dmul_rn(cq[1][3], xc)), __dmul_rn(cq[2][3], xb));
            const double tt[4] = {t0, t1, t2, t3};
            // the affine map of this lane's four frames
            Aff2 m{1., 0., 0., 1., 0., 0.};
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const double na1 = -cq[3][j], na2 = -cq[4][j];
                Aff2 r;
                r.a00 = fma(na1, m.a00, na2 * m.a10);
                r.a01 = fma(na1, m.a01, na2 * m.a11);
                r.a10 = m.a00;
                r.a11 = m.a01;
                r.b0 = fma(na1, m.b0, fma(na2, m.b1, tt[j]));
                r.b1 = m.b0;
                m = r;
            }
            // inclusive scan: lane L ends up with the map from the quantum's start to the end of its frames
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const Aff2 o = aff_shfl_up(m, d);
                if (lane >= d) m = aff_after(m, o);
            }
            const Aff2 e = aff_shfl_up(m, 1);  // ... to the start of its frames (lane 0: the identity)
            double s1 = y1, s2 = y2;
            if (lane != 0) {
                s1 = fma(e.a00, y1, fma(e.a01, y2, e.b0));
                s2 = fma(e.a10, y1, fma(e.a11, y2, e.b1));
            }
            bool bad = !(fabs(s1) <= 1.7976931348623157e308) || !(fabs(s2) <= 1.7976931348623157e308);
            const double ya = step(t0, cq[3][0], cq[4][0], s1, s2, bad);
            const double yb = step(t1, cq[3][1], cq[4][1], ya, s1, bad);
            const double yc = step(t2, cq[3][2], cq[4][2], yb, ya, bad);
            const double yd = step(t3, cq[3][3], cq[4][3], yc, yb, bad);
            if (!__any_sync(0xffffffffu, bad)) {
                *reinterpret_cast<float4*>(&sy[i]) = make_float4((float)ya, (float)yb, (float)yc, (float)yd);
                y1 = __shfl_sync(0xffffffffu, yd, 31);
                y2 = __shfl_sync(0xffffffffu, yc, 31);
            } else if (lane == 0) {
                // rare: a NaN / Inf went through — the reference's own serial evaluation, sample by sample with its flush
                double qx1 = x1, qx2 = x2, qy1 = y1, qy2 = y2;
                bool ignore = false;
                for (int k = 0; k < cnt; k++) {
                    const double x = absent ? 0. : (double)sx[k];
                    const double tk = __dadd_rn(__dadd_rn(__dmul_rn(cf[0][k], x), __dmul_rn(cf[1][k], qx1)), __dmul_rn(cf[2][k], qx2));
                    const double y = step(tk, cf[3][k], cf[4][k], qy1, qy2, ignore);
                    qx2 = qx1; qx1 = x; qy2 = qy1; qy1 = y;
                    sy[k] = (float)y;
                }
                y1 = qy1;
                y2 = qy2;
            }
            if (__any_sync(0xffffffffu, bad)) {
                y1 = __shfl_sync(0xffffffffu, y1, 0);
                y2 = __shfl_sync(0xffffffffu, y2, 0);
            }
            x1 = absent ? 0. : (double)sx[127];
            x2 = absent ? 0. : (double)sx[126];
        }
        __syncwarp();
        for (int k = lane; k < cnt; k += 32) out[n0 + k] = sy[k];
        __syncwarp();
    }
    if (lane == 0) {
        st[0] = x1; st[1] = x2; st[2] = y1; st[3] = y2;
        if (dyn) q.dyn_len[c] = len;
    }
}

// IIRFilter — IirFilterRenderer::process (src/node/iir_filter.rs:323-414): transposed DF-II in f64, serial
__global__ void __launch_bounds__(64) k_iir_serial(const IirInst* __restrict__ insts, int n_inst, int max_ch, ChunkInfo ci) {
    int t = blockIdx.x * blockDim.x + threadIdx.x;
    int ii = t / max_ch, c = t % max_ch;
    if (ii >= n_inst) return;
    const IirInst& q = insts[ii];
    if (c >= q.ch) return;
    const float* in = chan(q.in, c, ci);
    float* out = chan(q.out, c, ci);
    double s[20];
    const int nc = q.n;
    for (int i = 0; i < 20; i++) s[i] = q.state[20 * c + i];
    const bool dyn = q.in.meta != nullptr;
    int len = dyn ? q.dyn_len[c] : q.ch;
    bool skip = false, absent = false;
    for (int n = 0; n < ci.nf; n++) {
        if (dyn && (n & 127) == 0) {  // iir_filter.rs:336-376
            bool normal = false;
            for (int i = 0; i < 20; i++) normal = normal || isnormal_d(s[i]);
            filter_layout_step(q.in, q.out, q.ch, c, meta_qi(ci, n), len, normal, skip, absent);
            if (c >= len)
                for (int i = 0; i < 20; i++) s[i] = 0.;
        }
        if (skip) {
            out[n] = 0.f;
            continue;
        }
        double x = absent ? 0. : (double)in[n];
        double y = fma(q.b[0], x, s[0]);  // b0.mul_add(input, last_state), :391
        double ay = fabs(y);
        if (!(ay >= 2.2250738585072014e-308 && ay <= 1.7976931348623157e308)) y = 0.;
#pragma unroll
        for (int i = 0; i < 19; i++)
            if (i + 1 < nc) s[i] = __dadd_rn(__dsub_rn(__dmul_rn(q.b[i + 1], x), __dmul_rn(q.a[i + 1], y)), s[i + 1]);
        out[n] = (float)y;
    }
    for (int i = 0; i < 20; i++) q.state[20 * c + i] = s[i];
    if (dyn) q.dyn_len[c] = len;
}

// ---------------------------------------------------------------------------------------------------------
// Element-wise renderers
// ---------------------------------------------------------------------------------------------------------
// GainRenderer (src/node/gain.rs:147-199), scalar gain (the ~0 / ~1 shortcuts yield the same values up to
// 1e-6 relative only when |gain| or |1-gain| <= 1e-6: handled on the host by folding gain to 0 / 1)
__global__ void __launch_bounds__(256) k_gain(const GainInst* __restrict__ insts, int n_inst, ChunkInfo ci) {
    for (int ii = blockIdx.y; ii < n_inst; ii += gridDim.y) {
        const GainInst g = insts[ii];
        int n0 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
        if (n0 >= ci.nf) continue;
        for (int c = 0; c < g.ch; c++) {
            float4 v = *reinterpret_cast<const float4*>(chan(g.in, c, ci) + n0);
            if (g.gain_track.p) {  // a-rate gain (gain.rs:189-197)
                float4 t = *reinterpret_cast<const float4*>(chan(g.gain_track, 0, ci) + n0);
                v.x *= t.x; v.y *= t.y; v.z *= t.z; v.w *= t.w;
            } else {
                v.x *= g.gain; v.y *= g.gain; v.z *= g.gain; v.w *= g.gain;
            }
            *reinterpret_cast<float4*>(chan(g.out, c, ci) + n0) = v;
        }
    }
}

// apply_curve, src/node/waveshaper.rs:555-572
DEVI float shaper_apply(const float* curve, int len, float input) {
    float n = (float)len;
    float v = (n - 1.f) / 2.0f * (input + 1.f);
    if (v <= 0.f) return __ldg(curve);
    if (v >= n - 1.f) return __ldg(curve + (int)(n - 1.f));
    float k = floorf(v);
    float f = v - k;
    return __fadd_rn(__fmul_rn(1.f - f, __ldg(curve + (int)k)), __fmul_rn(f, __ldg(curve + (int)(k + 1.f))));
}
__global__ void __launch_bounds__(256) k_shaper(const ShaperInst* __restrict__ insts, int n_inst, ChunkInfo ci) {
    for (int ii = blockIdx.y; ii < n_inst; ii += gridDim.y) {
        const ShaperInst s = insts[ii];
        int n0 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
        if (n0 >= ci.nf) continue;
        for (int c = 0; c < s.ch; c++) {
            float4 v = *reinterpret_cast<const float4*>(chan(s.in, c, ci) + n0);
            if (s.curve) {
                if (s.n == 0) {
                    v = make_float4(0.f, 0.f, 0.f, 0.f);
                } else {
                    v.x = shaper_apply(s.curve, s.n, v.x);
                    v.y = shaper_apply(s.curve, s.n, v.y);
                    v.z = shaper_apply(s.curve, s.n, v.z);
                    v.w = shaper_apply(s.curve, s.n, v.w);
                }
            }
            *reinterpret_cast<float4*>(chan(s.out, c, ci) + n0) = v;
        }
    }
}

// StereoPannerRenderer (src/node/stereo_panner.rs:218-318), constant pan; gains are computed on the host
// with the reference's f32 expressions (get_stereo_gains, :74-79) and passed in `pan`-derived fields.
__global__ void __launch_bounds__(256) k_stereo_panner(const SPanInst* __restrict__ insts, const float2* __restrict__ gains, int n_inst,
                                                       ChunkInfo ci) {
    for (int ii = blockIdx.y; ii < n_inst; ii += gridDim.y) {
        const SPanInst s = insts[ii];
        float gl = gains[ii].x, gr = gains[ii].y;
        int n = blockIdx.x * blockDim.x + threadIdx.x;
        if (n >= ci.nf) continue;
        float pan = s.pan;
        // dynamic input layout: the mono / stereo formulas are chosen per quantum (stereo_panner.rs:242), a silent input gives
        // a silent output (:230-233; the layout track of the output is written by k_meta)
        int in_ch = s.in_ch;
        if (s.in.meta) {
            const int qi = meta_qi(ci, n);
            if (buf_silent(s.in, s.in_ch, qi)) {
                chan(s.out, 0, ci)[n] = 0.f;
                chan(s.out, 1, ci)[n] = 0.f;
                continue;
            }
            in_ch = buf_count(s.in, s.in_ch, qi);
        }
        if (s.pan_track.p || in_ch != s.in_ch) {  // a-rate pan: gains per frame (stereo_panner.rs:259-271, 293-313)
            if (s.pan_track.p) pan = chan(s.pan_track, 0, ci)[n];
            const float PI32 = 3.14159265358979323846f;
            float x = in_ch == 1 ? (pan + 1.f) * 0.5f : (pan <= 0.f ? pan + 1.f : pan);
            gl = sinf((1.f - x) * PI32 / 2.f);
            gr = sinf(x * PI32 / 2.f);
        }
        float* l = chan(s.out, 0, ci);
        float* r = chan(s.out, 1, ci);
        if (in_ch == 1) {
            float x = chan(s.in, 0, ci)[n];
            l[n] = x * gl;
            r[n] = x * gr;
        } else {
            float il = chan(s.in, 0, ci)[n], ir = chan(s.in, 1, ci)[n];
            if (pan <= 0.f) {
                l[n] = fmaf(ir, gl, il);
                r[n] = ir * gr;
            } else {
                l[n] = il * gl;
                r[n] = fmaf(il, gr, ir);
            }
        }
    }
}

// equal-power gains of one frame (panner.rs:988-1057)
__device__ __forceinline__ void pan_eq_frame(const spatial::SpatialParams& sp, int in_ch, float il, float ir, float& l, float& r) {
    const float PI32 = 3.14159265358979323846f;
    float az = fminf(fmaxf(sp.azimuth, -180.f), 180.f);
    if (az < -90.f)
        az = -180.f - az;
    else if (az > 90.f)
        az = 180.f - az;
    if (in_ch == 1) {
        float x = (az + 90.f) / 180.f;
        float gl = cosf(x * PI32 / 2.f), gr = sinf(x * PI32 / 2.f);
        l = il * (gl * sp.dist_gain * sp.cone_gain);
        r = il * (gr * sp.dist_gain * sp.cone_gain);
    } else {
        float x = az <= 0.f ? (az + 90.f) / 90.f : az / 90.f;
        float gl = cosf(x * PI32 / 2.f), gr = sinf(x * PI32 / 2.f);
        if (az <= 0.f) {
            l = (il + ir * gl) * sp.dist_gain * sp.cone_gain;
            r = ir * gr * sp.dist_gain * sp.cone_gain;
        } else {
            l = il * gl * sp.dist_gain * sp.cone_gain;
            r = (ir + il * gr) * sp.dist_gain * sp.cone_gain;
        }
    }
}

// PannerRenderer equal-power branch, static source/listener (src/node/panner.rs:839-870, 988-1057)
__global__ void __launch_bounds__(256) k_panner_eq(const PanInst* __restrict__ insts, int n_inst, ChunkInfo ci) {
    for (int ii = blockIdx.y; ii < n_inst; ii += gridDim.y) {
        const PanInst p = insts[ii];
        int n = blockIdx.x * blockDim.x + threadIdx.x;
        if (n >= ci.nf) continue;
        spatial::SpatialParams sp{p.dist_gain, p.cone_gain, p.azimuth, 0.f};
        int in_ch = p.in_ch;
        if (p.in.meta) {  // dynamic input layout (panner.rs:698-708,846,872)
            const int qi = meta_qi(ci, n);
            if (buf_silent(p.in, p.in_ch, qi)) {
                chan(p.out, 0, ci)[n] = 0.f;
                chan(p.out, 1, ci)[n] = 0.f;
                continue;
            }
            in_ch = buf_count(p.in, p.in_ch, qi);
        }
        float il = chan(p.in, 0, ci)[n], ir = in_ch == 2 ? chan(p.in, 1, ci)[n] : 0.f;
        float l, r;
        pan_eq_frame(sp, in_ch, il, ir, l, r);
        chan(p.out, 0, ci)[n] = l;
        chan(p.out, 1, ci)[n] = r;
    }
}

// ---------------------------------------------------------------------------------------------------------
// Over-sampled WaveShaper (waveshaper.rs:409-480 over rubato::FftFixedInOut): per render quantum q
//     up_j   = irFFT_{2 fo}( rFFT_256([x_j | 0]) * F_up )            fo = 128 * factor
//     u_j    = curve( up_j[0 .. fo) + up_{j-1}[fo .. 2 fo) )
//     dn_j   = irFFT_256( rFFT_{2 fo}([u_j | 0])[0 .. 128) * F_dn )
//     out_q  = dn_q[0 .. 128) + dn_{q-1}[128 .. 256)
// One CTA per (quantum, channel, instance) recomputes the three up-transforms and two down-transforms its output
// depends on, so the only state between chunks is two quanta of input.  Plain complex FFTs (<= 1024 points) in smem.
// ---------------------------------------------------------------------------------------------------------
DEVI void fft_small(float2* s, int n, int logn, int sign) {  // 128 threads, in place, natural order in and out
    const int t = threadIdx.x;
    for (int i = t; i < n; i += 128) {
        const int r = (int)(__brev((unsigned)i) >> (32 - logn));
        if (i < r) {
            const float2 tmp = s[i];
            s[i] = s[r];
            s[r] = tmp;
        }
    }
    __syncthreads();
    for (int len = 2; len <= n; len <<= 1) {
        const int half = len >> 1;
        for (int b = t; b < n / 2; b += 128) {
            const int j = b & (half - 1);
            const int i0 = ((b - j) << 1) + j, i1 = i0 + half;
            float sn, cs;
            sincospif((float)sign * 2.f * (float)j / (float)len, &sn, &cs);
            const float2 u = s[i0], x = s[i1];
            const float2 v = make_float2(x.x * cs - x.y * sn, x.x * sn + x.y * cs);
            s[i0] = make_float2(u.x + v.x, u.y + v.y);
            s[i1] = make_float2(u.x - v.x, u.y - v.y);
        }
        __syncthreads();
    }
}
// z <- irFFT_{n_out}( rFFT_{n_in}(real input in z[0 .. n_in)) [0 .. 128) * F ): the real result is left in z[i].x
DEVI void os_resample(float2* z, int n_in, int log_in, int n_out, int log_out, const float2* __restrict__ F) {
    const int t = threadIdx.x;
    fft_small(z, n_in, log_in, -1);
    float2 y = make_float2(0.f, 0.f);
    {
        const float2 x = z[t], f = __ldg(F + t);  // bins 0 .. 127 (n_in >= 256)
        y = make_float2(x.x * f.x - x.y * f.y, x.x * f.y + x.y * f.x);
        if (t == 0) y.y = 0.f;  // realfft ignores the imaginary part of the DC bin
    }
    __syncthreads();
    for (int i = t; i < n_out; i += 128) z[i] = make_float2(0.f, 0.f);
    __syncthreads();
    z[t] = y;
    if (t > 0) z[n_out - t] = make_float2(y.x, -y.y);  // Hermitian half
    __syncthreads();
    fft_small(z, n_out, log_out, +1);
}
__global__ void __launch_bounds__(128) k_shaper_os(const ShaperOsInst* __restrict__ insts, ChunkInfo ci) {
    __shared__ float2 z[1024];
    __shared__ float keep[4][512];  // up_{q-2} second half, up_{q-1} both halves, up_q first half
    __shared__ float dn_prev[128];
    const ShaperOsInst& p = insts[blockIdx.z];
    const int c = blockIdx.y;
    if (c >= p.ch) return;
    const int q = blockIdx.x;  // quantum inside the chunk
    const int t = threadIdx.x;
    const int fo = 128 * p.factor, n2 = 2 * fo, log2n = p.factor == 2 ? 9 : 10;
    const float* in = chan(p.in, c, ci);
    const float* hist = p.hist + 256 * c;
    int q_of[3] = {q - 2, q - 1, q};
    int since = 2;  // processed quanta since the resamplers were (re)built, before q (capped at 2; always 2 without rebuilds)
    if (p.prev) {  // silent quanta are not processed at all (block-uniform): the neighbours are the last processed quanta
        const int32_t* pv = p.prev;
        bool skip;
        if (p.rebuild) {
            pv = p.prev + 2;
            const int32_t info = pv[2 * (ci.nf / 128) + 2 + q];
            skip = !(info & OS_INFO_PROCESSED);
            if (!skip && c >= (info & 0x3f)) return;  // (no such channel in this quantum: unspecified)
            since = info >> OS_INFO_SINCE_SHIFT;
        } else {
            skip = buf_silent(p.in, p.ch, meta_qi(ci, q * 128));
        }
        if (skip) {
            chan(p.out, c, ci)[q * 128 + t] = 0.f;
            return;
        }
        q_of[0] = pv[2 * q + 1];
        q_of[1] = pv[2 * q];
    }
    // three up-transforms: quanta q-2, q-1, q
    for (int r = 0; r < 3; r++) {
        const int qq = q_of[r];
        float x;
        if (r < 2 - since) x = 0.f;  // older than the last rebuild
        else if (qq < 0) x = hist[(qq + 2) * 128 + t];
        else if (p.rebuild && buf_silent(p.in, p.ch, meta_qi(ci, qq * 128))) x = 0.f;  // a processed silent quantum: one zero channel
        else x = in[qq * 128 + t];
        z[t] = make_float2(x, 0.f);
        z[128 + t] = make_float2(0.f, 0.f);
        __syncthreads();
        os_resample(z, 256, 8, n2, log2n, p.f_up);
        for (int i = t; i < fo; i += 128) {
            if (r == 0) keep[0][i] = z[fo + i].x;
            if (r == 1) keep[1][i] = z[i].x, keep[2][i] = z[fo + i].x;
            if (r == 2) keep[3][i] = z[i].x;
        }
        __syncthreads();
    }
    // two down-transforms: u_{q-1} and u_q
    float result = 0.f;
    for (int r = 0; r < 2; r++) {
        for (int i = t; i < n2; i += 128) {
            float u = 0.f;
            if (i < fo) {
                u = r == 0 ? keep[1][i] + keep[0][i] : keep[3][i] + keep[2][i];
                u = p.n == 0 ? 0.f : shaper_apply(p.curve, p.n, u);
            }
            z[i] = make_float2(u, 0.f);
        }
        __syncthreads();
        os_resample(z, n2, log2n, 256, 8, p.f_dn);
        if (r == 0) dn_prev[t] = z[128 + t].x;
        else result = z[t].x;
        __syncthreads();
    }
    // (at a rebuild the fresh down-sampler's overlap is zero in the SHAPED domain: not the transform of curve(0))
    chan(p.out, c, ci)[q * 128 + t] = since > 0 ? result + dn_prev[t] : result;
}
// dynamic input layout: the processed quanta before every quantum of the chunk (ShaperOsInst::prev), one thread per instance
__global__ void __launch_bounds__(64) k_shaper_os_prev(const ShaperOsInst* __restrict__ insts, int n_inst, ChunkInfo ci) {
    const int ii = blockIdx.x * blockDim.x + threadIdx.x;
    if (ii >= n_inst) return;
    const ShaperOsInst& p = insts[ii];
    if (!p.prev) return;
    int last1 = -1, last2 = -2;
    const int nq = ci.nf / 128;
    if (p.rebuild) {  // + which quanta are processed, their counts, the rebuilds (waveshaper.rs:395-420)
        int32_t* pv = p.prev + 2;
        int built = p.prev[0] ? p.prev[0] : 1, since = p.prev[1];
        for (int q = 0; q < nq; q++) {
            pv[2 * q] = last1;
            pv[2 * q + 1] = last2;
            const int qi = meta_qi(ci, q * 128);
            const bool silent = buf_silent(p.in, p.ch, qi);
            int32_t info = 0;
            if (!silent || p.rebuild == 1) {
                const int count = silent ? 1 : buf_count(p.in, p.ch, qi);
                if (count != built) {
                    built = count;
                    since = 0;
                }
                info = OS_INFO_PROCESSED | count | since << OS_INFO_SINCE_SHIFT;
                since = since < 2 ? since + 1 : 2;
                last2 = last1;
                last1 = q;
            }
            pv[2 * nq + 2 + q] = info;
        }
        pv[2 * nq] = last1;
        pv[2 * nq + 1] = last2;
        p.prev[0] = built;
        p.prev[1] = since;
        return;
    }
    for (int q = 0; q < nq; q++) {
        p.prev[2 * q] = last1;
        p.prev[2 * q + 1] = last2;
        if (!buf_silent(p.in, p.ch, meta_qi(ci, q * 128))) {
            last2 = last1;
            last1 = q;
        }
    }
    p.prev[2 * nq] = last1;
    p.prev[2 * nq + 1] = last2;
}
// the two input quanta before the next chunk
__global__ void __launch_bounds__(256) k_shaper_os_hist(const ShaperOsInst* __restrict__ insts, ChunkInfo ci) {
    const ShaperOsInst& p = insts[blockIdx.x];
    const int t = threadIdx.x;
    for (int c = 0; c < p.ch; c++) {
        if (p.prev) {  // the two PROCESSED quanta before the next chunk: slot 1 (t >= 128) the latest, slot 0 the one before
            const int nq = ci.nf / 128;
            const int32_t* pv = p.rebuild ? p.prev + 2 : p.prev;
            const int qq = t >= 128 ? pv[2 * nq] : pv[2 * nq + 1];
            const int i = t & 127;
            float v;
            if (p.rebuild && (t >= 128 ? 1 : 2) > p.prev[1]) v = 0.f;  // older than the last rebuild
            else if (qq < 0) v = p.hist[256 * c + (qq + 2) * 128 + i];
            else if (p.rebuild && (!(pv[2 * nq + 2 + qq] & OS_INFO_PROCESSED) || c >= (pv[2 * nq + 2 + qq] & 0x3f) ||
                                   buf_silent(p.in, p.ch, meta_qi(ci, qq * 128))))
                v = 0.f;  // a processed silent quantum (one zero channel) / a channel the quantum does not have
            else v = chan(p.in, c, ci)[qq * 128 + i];
            __syncthreads();
            p.hist[256 * c + t] = v;
            __syncthreads();
            continue;
        }
        const int m = ci.nf - 256 + t;
        const float v = m >= 0 ? chan(p.in, c, ci)[m] : p.hist[256 * c + 128 + t - (128 - ci.nf)];  // nf == 128: shift by one quantum
        __syncthreads();
        p.hist[256 * c + t] = v;
        __syncthreads();
    }
}

// the 15 spatial params at frame n of the chunk; `first_of_quantum`: take the quantum's first value of every param
__device__ __forceinline__ void spatial_fetch(const SpatialTracks& t, int n, bool first_of_quantum, const ChunkInfo& ci, float v[15]) {
    const int pf = first_of_quantum ? (n & ~127) : n;
#pragma unroll
    for (int i = 0; i < 15; i++) v[i] = t.track[i].p ? chan(t.track[i], 0, ci)[pf] : t.value[i];
}
// panner.rs:833-841: all nine listener params single-valued in this quantum?
__device__ __forceinline__ bool listener_single_valued(const SpatialTracks& t, int n, const ChunkInfo& ci) {
    const int q0 = n & ~127;
    bool single = true;
#pragma unroll
    for (int i = 6; i < 15; i++)
        if (t.track[i].p && chan(t.track[i], 1, ci)[q0] == 0.f) single = false;
    return single;
}

// PannerRenderer equal-power branch with automated source / listener params (panner.rs:714-780, 833-897)
__global__ void __launch_bounds__(128) k_panner_dyn(const PanDynInst* __restrict__ insts, int n_inst, ChunkInfo ci) {
    for (int ii = blockIdx.y; ii < n_inst; ii += gridDim.y) {
        const PanDynInst& p = insts[ii];
        int n = blockIdx.x * blockDim.x + threadIdx.x;
        if (n >= ci.nf) continue;
        float v[15];
        spatial_fetch(p.sp, n, listener_single_valued(p.sp, n, ci), ci, v);
        const spatial::SpatialParams sp = spatial::spatial_params(p.model, v);
        int in_ch = p.in_ch;
        if (p.in.meta) {  // dynamic input layout (panner.rs:698-708,846,872)
            const int qi = meta_qi(ci, n);
            if (buf_silent(p.in, p.in_ch, qi)) {
                chan(p.out, 0, ci)[n] = 0.f;
                chan(p.out, 1, ci)[n] = 0.f;
                continue;
            }
            in_ch = buf_count(p.in, p.in_ch, qi);
        }
        float il = chan(p.in, 0, ci)[n], ir = in_ch == 2 ? chan(p.in, 1, ci)[n] : 0.f;
        float l, r;
        pan_eq_frame(sp, in_ch, il, ir, l, r);
        chan(p.out, 0, ci)[n] = l;
        chan(p.out, 1, ci)[n] = r;
    }
}

// HRTF panner with automated params: k-rate, first value of every quantum (panner.rs:781-802)
__global__ void __launch_bounds__(64) k_hrtf_sel(const HrtfSelInst* __restrict__ insts, ChunkInfo ci) {
    const HrtfSelInst& p = insts[blockIdx.y];
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q * 128 >= ci.nf) return;
    float v[15];
    spatial_fetch(p.sp, q * 128, true, ci, v);
    const spatial::SpatialParams sp = spatial::spatial_params(p.model, v);
    float proj[3];
    spatial::projected_source(sp, proj);
    const float dir[3] = {proj[0], proj[2], proj[1]};  // HrtfState::process swaps y / z (panner.rs:248-252)
    HrtfSel s{{0, 0, 0}, {0.f, 0.f, 0.f}, sp.cone_gain * sp.dist_gain, 0.f};
    spatial::hrir_locate(p.pos, p.tri, p.n_faces, dir, s.v, s.w);
    p.sel[(ci.sub >> 7) + q] = s;
}

// ---------------------------------------------------------------------------------------------------------
// HRTF panner: out[n] = gain * sum_k h[k] x[n-k] for the left and the right blended response (L taps, L = 512 for the
// reference's IRC_1003_C sphere).  One warp per render quantum, 4 consecutive frames x 2 ears per lane with the input window
// sliding through registers: per 4 taps 4 shared loads of x + 2 float4 broadcasts of h feed 32 FMAs.
// ---------------------------------------------------------------------------------------------------------
constexpr int HRTF_TILE = 1024;  // frames per CTA: 4 warps x 32 lanes x 8 frames = 8 render quanta
DEVI int hrtf_pad(int i) { return i + (i >> 3); }  // stride-8 lane access -> 32 distinct banks

DEVI float hrtf_input(const HrtfInst& p, int m, const ChunkInfo& ci) {
    int in_ch = p.in_ch;
    if (p.in.meta) {  // dynamic layout: the channels this quantum has; a (processed) silent quantum reads as zeros
        const int qi = meta_qi(ci, m);
        if (buf_silent(p.in, p.in_ch, qi)) return 0.f;
        in_ch = buf_count(p.in, p.in_ch, qi);
    }
    float v = chan(p.in, 0, ci)[m];
    if (in_ch == 2) v = 0.5f * (v + chan(p.in, 1, ci)[m]);  // output.mix(1, Speakers), quantum.rs 2 -> 1
    return v;
}
// frame mc of the PROCESSED sequence of this chunk (HrtfInst::cmap) -> chunk frame
DEVI int hrtf_unmap(const HrtfInst& p, int mc) { return p.dyn ? p.cmap[1 + (mc >> 7)] * 128 + (mc & 127) : mc; }
// dynamic input layout: which quanta of the chunk the node processes (panner.rs:697-711), its output layout track
__global__ void __launch_bounds__(64) k_hrtf_map(const HrtfInst* __restrict__ insts, int n_inst, ChunkInfo ci) {
    const int ii = blockIdx.x * blockDim.x + threadIdx.x;
    if (ii >= n_inst) return;
    const HrtfInst& p = insts[ii];
    if (!p.dyn) return;
    int64_t tail = *p.tail;
    int n_proc = 0;
    for (int q = 0; q < ci.nf / 128; q++) {
        const int qi = meta_qi(ci, q * 128);
        const bool silent = buf_silent(p.in, p.in_ch, qi);
        bool processed = true;
        if (silent) {
            processed = (int64_t)p.L > tail;
            if (processed) tail += 128;
        }
        if (processed) p.cmap[1 + n_proc++] = q;
        if (p.out.meta) meta_put_all(p.out, 2, qi, processed ? 2 : 1, !processed);
    }
    p.cmap[0] = n_proc;
    *p.tail = tail;
}
// quanta the node did not process: silent output, PCM zeroed
__global__ void __launch_bounds__(256) k_hrtf_fill(const HrtfInst* __restrict__ insts, int n_inst, ChunkInfo ci) {
    for (int ii = blockIdx.y; ii < n_inst; ii += gridDim.y) {
        const HrtfInst& p = insts[ii];
        const int n = blockIdx.x * blockDim.x + threadIdx.x;
        if (!p.dyn || !p.out.meta || n >= ci.nf) continue;
        if (p.out.meta[meta_qi(ci, n)] & WAE_META_SILENT) {
            chan(p.out, 0, ci)[n] = 0.f;
            chan(p.out, 1, ci)[n] = 0.f;
        }
    }
}

// One lane = 8 consecutive frames x 2 ears (16 accumulators); the input window slides through registers, so 4 taps cost
// 4 shared loads of x + 2 float4 loads of h for 64 FMAs.  A warp covers two render quanta (lanes 0-15 / 16-31), each with
// its own blended response (moving sources: the response changes per quantum).
__global__ void __launch_bounds__(128) k_hrtf_fir(const HrtfInst* __restrict__ insts, ChunkInfo ci) {
    extern __shared__ __align__(16) float hsm[];
    const HrtfInst p = insts[blockIdx.y];
    const int L = p.L, L4 = (L + 3) & ~3;
    const int tile0 = blockIdx.x * HRTF_TILE;
    const int nx = 4 + (L4 - 1) + HRTF_TILE;  // 4 leading slots keep the 4-tap unroll in range
    float* xs = hsm;                           // padded input window: xs[pad(4 + (L4-1) + n)] = x[tile0 + n]
    float* hs = hsm + ((hrtf_pad(nx) + 4) & ~3);  // [8 quanta][2][L4]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    // (dynamic layout: tile0 and every frame index below count PROCESSED quanta; hrtf_unmap gives the chunk frame)
    const int nf_proc = p.dyn ? p.cmap[0] * 128 : ci.nf;
    if (tile0 >= nf_proc) return;
    for (int i = tid; i < nx; i += 128) {
        int m = tile0 + i - 4 - (L4 - 1);  // chunk-relative frame
        float v = 0.f;
        if (m >= 0) {
            if (m < nf_proc) v = hrtf_input(p, hrtf_unmap(p, m), ci);
        } else if (m >= -(L - 1)) {
            v = p.hist[(L - 1) + m];
        }
        xs[hrtf_pad(i)] = v;
    }
    // blended responses: one per quantum of the tile for a moving source / listener (warp w blends quanta 2w and 2w + 1),
    // a single shared one for a static panner (each warp blends a quarter of it)
    const bool moving = p.sel != nullptr;
    for (int h = 0; h < 2; h++) {
        const int qi = moving ? warp * 2 + h : 0;
        const int q0c = tile0 + qi * 128;
        if (moving && q0c >= nf_proc) break;
        if (!moving && h == 1) break;
        const int q0 = hrtf_unmap(p, q0c);
        const HrtfSel sel = moving ? p.sel[(ci.sub + q0) >> 7] : p.static_sel;
        float* hl = hs + qi * 2 * L4;
        float* hr = hl + L4;
        const float* A = p.sphere_ir + (size_t)sel.v[0] * 2 * L;
        const float* B = p.sphere_ir + (size_t)sel.v[1] * 2 * L;
        const float* C = p.sphere_ir + (size_t)sel.v[2] * 2 * L;
        for (int k = moving ? lane : tid; k < L4; k += moving ? 32 : 128) {
            float l = 0.f, r = 0.f;
            if (k < L) {
                l = __fadd_rn(__fadd_rn(__fmul_rn(A[k], sel.w[0]), __fmul_rn(B[k], sel.w[1])), __fmul_rn(C[k], sel.w[2]));
                r = __fadd_rn(__fadd_rn(__fmul_rn(A[L + k], sel.w[0]), __fmul_rn(B[L + k], sel.w[1])), __fmul_rn(C[L + k], sel.w[2]));
            }
            hl[k] = l;
            hr[k] = r;
        }
    }
    __syncthreads();
    const int qi = warp * 2 + (lane >> 4);
    const int q0c = tile0 + qi * 128;
    if (q0c >= nf_proc) return;
    const int q0 = hrtf_unmap(p, q0c);
    const HrtfSel sel = moving ? p.sel[(ci.sub + q0) >> 7] : p.static_sel;
    const float* hl = hs + (moving ? qi : 0) * 2 * L4;
    const float* hr = hl + L4;
    const int nrel = warp * 256 + lane * 8;        // tile-relative first frame of this lane
    const int base = 4 + (L4 - 1) + nrel;          // xs index of x[n0]
    float w[8], al[8], ar[8];
#pragma unroll
    for (int j = 0; j < 8; j++) {
        w[j] = xs[hrtf_pad(base + j)];
        al[j] = 0.f;
        ar[j] = 0.f;
    }
#pragma unroll 1
    for (int k = 0; k < L4; k += 4) {
        const float4 a = *reinterpret_cast<const float4*>(hl + k);
        const float4 b = *reinterpret_cast<const float4*>(hr + k);
        const float m1 = xs[hrtf_pad(base - k - 1)], m2 = xs[hrtf_pad(base - k - 2)];
        const float m3 = xs[hrtf_pad(base - k - 3)], m4 = xs[hrtf_pad(base - k - 4)];
        // tap k: x[n0 - k + j] = w[j]
#pragma unroll
        for (int j = 0; j < 8; j++) {
            al[j] = fmaf(a.x, w[j], al[j]);
            ar[j] = fmaf(b.x, w[j], ar[j]);
        }
        // tap k + 1: (m1, w0 .. w6)
        al[0] = fmaf(a.y, m1, al[0]); ar[0] = fmaf(b.y, m1, ar[0]);
#pragma unroll
        for (int j = 1; j < 8; j++) {
            al[j] = fmaf(a.y, w[j - 1], al[j]);
            ar[j] = fmaf(b.y, w[j - 1], ar[j]);
        }
        // tap k + 2: (m2, m1, w0 .. w5)
        al[0] = fmaf(a.z, m2, al[0]); ar[0] = fmaf(b.z, m2, ar[0]);
        al[1] = fmaf(a.z, m1, al[1]); ar[1] = fmaf(b.z, m1, ar[1]);
#pragma unroll
        for (int j = 2; j < 8; j++) {
            al[j] = fmaf(a.z, w[j - 2], al[j]);
            ar[j] = fmaf(b.z, w[j - 2], ar[j]);
        }
        // tap k + 3: (m3, m2, m1, w0 .. w4)
        al[0] = fmaf(a.w, m3, al[0]); ar[0] = fmaf(b.w, m3, ar[0]);
        al[1] = fmaf(a.w, m2, al[1]); ar[1] = fmaf(b.w, m2, ar[1]);
        al[2] = fmaf(a.w, m1, al[2]); ar[2] = fmaf(b.w, m1, ar[2]);
#pragma unroll
        for (int j = 3; j < 8; j++) {
            al[j] = fmaf(a.w, w[j - 3], al[j]);
            ar[j] = fmaf(b.w, w[j - 3], ar[j]);
        }
        // next window: x[n0 - k - 4 + j]
        w[7] = w[3]; w[6] = w[2]; w[5] = w[1]; w[4] = w[0];
        w[3] = m1; w[2] = m2; w[1] = m3; w[0] = m4;
    }
    const int n = q0 + (nrel & 127);  // (8 frames of a lane never straddle a quantum)
    float* ol = chan(p.out, 0, ci);
    float* orr = chan(p.out, 1, ci);
    float c = p.correction;
    if (p.in.meta) {  // overall_gain_correction: 2 for a two-channel input quantum (panner.rs:805-812)
        const int mq = meta_qi(ci, q0);
        c = (!buf_silent(p.in, p.in_ch, mq) && buf_count(p.in, p.in_ch, mq) == 2) ? 2.f : 1.f;
    }
    const float g = sel.gain;
#pragma unroll
    for (int j = 0; j < 8; j++)
        if (n + j < ci.nf) {
            ol[n + j] = __fmul_rn(c, __fmul_rn(al[j], g));
            orr[n + j] = __fmul_rn(c, __fmul_rn(ar[j], g));
        }
}

// input history for the next chunk (runs after every k_hrtf_fir CTA of the chunk has read the old one)
__global__ void __launch_bounds__(128) k_hrtf_hist(const HrtfInst* __restrict__ insts, ChunkInfo ci) {
    extern __shared__ float hh[];
    const HrtfInst p = insts[blockIdx.x];
    const int H = p.L - 1;
    const int nf_proc = p.dyn ? p.cmap[0] * 128 : ci.nf;
    for (int i = threadIdx.x; i < H; i += blockDim.x) {
        int m = nf_proc - H + i;
        hh[i] = m >= 0 ? hrtf_input(p, hrtf_unmap(p, m), ci) : p.hist[H + m];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < H; i += blockDim.x) p.hist[i] = hh[i];
}

// channel merger / splitter (src/node/channel_merger.rs:146-171, channel_splitter.rs:183-208)
__global__ void __launch_bounds__(256) k_route(const RouteInst* __restrict__ insts, int n_inst, ChunkInfo ci) {
    for (int ii = blockIdx.y; ii < n_inst; ii += gridDim.y) {
        const RouteInst r = insts[ii];
        int n0 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
        if (n0 >= ci.nf) continue;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        bool zero = r.zero != 0;
        if (!zero && r.in.meta) {  // dynamic input layout: a channel the input does not have in this quantum (or a silent input) reads as zeros
            const int qi = meta_qi(ci, n0);
            zero = buf_silent(r.in, r.in_ch, qi) || r.in_channel >= buf_count(r.in, r.in_ch, qi);
        }
        if (!zero) v = *reinterpret_cast<const float4*>(chan(r.in, r.in_channel, ci) + n0);
        *reinterpret_cast<float4*>(chan(r.out, r.out_channel, ci) + n0) = v;
    }
}

// ---------------------------------------------------------------------------------------------------------
// Delay — DelayWriter/DelayReader (src/node/delay.rs:428-461, 515-743), constant delayTime, acyclic.
// The reference's ring-of-quanta index arithmetic reduces to out[n] = fmaf(1-k, x[n+fl], k*x[n+fl+1]) with
// fl = floor(-delay*sr), k = frac(-delay*sr); history older than the chunk comes from a persistent ring.
// ---------------------------------------------------------------------------------------------------------
DEVI float delay_fetch(const DelayInst& d, const float* in, const float* ring, int64_t m, const ChunkInfo& ci) {
    if (m < 0) return 0.f;
    if (d.in_cycle) return m >= ci.f0 ? 0.f : ring[m & (d.ring_len - 1)];
    if (m >= ci.f0) {
        int64_t r = m - ci.f0;
        if (r < ci.nf) return in[r];
        // "next" sample beyond the newest quantum: the reference reads the oldest ring entry here; it is
        // always multiplied by k == 0 in that situation (delay == 0)
        return 0.f;
    }
    return ring[m & (d.ring_len - 1)];
}
// Dynamic input layout (static channels <= 2).  Sample of frame m as the reference's ring holds it when the reader runs in quantum
// `q_read`: the ring stores the canonical two channels of every quantum (a one-channel quantum is stored twice); every time the
// writer sees a channel count different from the ring's it re-mixes the WHOLE ring (delay.rs:470-488, speakers rules: 2 -> 1 is
// 0.5 * (L + R), 1 -> 2 a copy), so a stereo sample has collapsed to its mono down-mix iff some quantum in (its own, q_read] had a
// one-channel input — mono_at[q_read] > quantum of m.  In a feedback cycle the reader runs before the writer: q_read is the quantum
// before.
DEVI void delay_fetch2(const DelayInst& d, int64_t m, const ChunkInfo& ci, int64_t mono_last, float& l, float& r) {
    l = r = 0.f;
    if (m < 0) return;
    const float* ring = d.ring;
    if (!d.in_cycle && m >= ci.f0) {
        const int64_t rr = m - ci.f0;
        if (rr >= ci.nf) return;
        const int qi = meta_qi(ci, (int)rr);
        if (buf_silent(d.in, d.ch, qi)) return;
        l = chan(d.in, 0, ci)[rr];
        r = buf_count(d.in, d.ch, qi) >= 2 ? chan(d.in, 1, ci)[rr] : l;
    } else {
        if (d.in_cycle && m >= ci.f0) return;
        l = ring[m & (d.ring_len - 1)];
        r = d.ch > 1 ? ring[(size_t)d.ring_len + (m & (d.ring_len - 1))] : l;
    }
    if (mono_last > (m >> 7)) l = r = 0.5f * (l + r);
}
__global__ void __launch_bounds__(256) k_delay_read(const DelayInst* __restrict__ insts, int n_inst, ChunkInfo ci) {
    __shared__ int s_live[2];
    for (int ii = blockIdx.y; ii < n_inst; ii += gridDim.y) {
        const DelayInst d = insts[ii];
        int n = blockIdx.x * blockDim.x + threadIdx.x;
        if (d.dyn) {  // whole quanta per block (256 threads = 2 quanta): every thread takes part in the silence vote
            if (threadIdx.x < 2) s_live[threadIdx.x] = 0;
            __syncthreads();
            const bool inside = n < ci.nf;
            int out_ch = 1;
            if (inside) {
                const int64_t q_abs = (ci.f0 + n) >> 7;
                const int64_t q_read = d.in_cycle ? q_abs - 1 : q_abs;  // newest quantum the ring has seen when the reader runs
                int64_t mono_last = -1;
                if (q_read >= 0) {
                    mono_last = d.mono_at[q_read & (d.mono_len - 1)];
                    out_ch = mono_last == q_read ? 1 : d.ch;  // ring[0].number_of_channels() (:532-533)
                }
                int64_t m = ci.f0 + n + d.fl;
                float k = d.k;
                if (d.delay_track.p) {
                    double delay = (double)chan(d.delay_track, 0, ci)[n];
                    const double sr = (double)d.sample_rate;
                    if (d.in_cycle) delay = fmax(delay, 128. / sr);
                    const int i = (int)((ci.f0 + n) & 127);
                    double position = (double)i - delay * sr;
                    double pf = floor(position);
                    m = (ci.f0 + n - i) + (int64_t)pf;
                    k = (float)(position - pf);
                }
                float pl, pr, nl, nr;
                delay_fetch2(d, m, ci, mono_last, pl, pr);
                delay_fetch2(d, m + 1, ci, mono_last, nl, nr);
                if (out_ch == 1) {  // a one-channel ring: every stereo sample in it has been mixed down
                    pl = pr = 0.5f * (pl + pr);
                    nl = nr = 0.5f * (nl + nr);
                }
                const float vl = fmaf(1.f - k, pl, k * nl), vr = fmaf(1.f - k, pr, k * nr);
                chan(d.out, 0, ci)[n] = vl;
                if (d.ch > 1) chan(d.out, 1, ci)[n] = vr;
                const float al = fabsf(vl), ar = fabsf(vr);
                const bool live = (al >= 1.17549435e-38f && al <= 3.40282347e+38f) || (out_ch > 1 && ar >= 1.17549435e-38f && ar <= 3.40282347e+38f);
                if (live) s_live[threadIdx.x >> 7] = 1;  // is_normal(value) (:654-664)
            }
            __syncthreads();
            if (inside && (threadIdx.x & 127) == 0 && d.out.meta)
                meta_put_all(d.out, d.ch, meta_qi(ci, n), s_live[threadIdx.x >> 7] ? out_ch : 1, !s_live[threadIdx.x >> 7]);
            __syncthreads();
            continue;
        }
        if (n >= ci.nf) continue;
        for (int c = 0; c < d.ch; c++) {
            const float* in = d.in_cycle ? nullptr : chan(d.in, c, ci);
            const float* ring = d.ring + (size_t)c * d.ring_len;
            int64_t m = ci.f0 + n + d.fl;
            float k = d.k;
            if (d.delay_track.p) {  // a-rate delayTime: get_playback_infos per frame (delay.rs:688-743)
                double delay = (double)chan(d.delay_track, 0, ci)[n];
                const double sr = (double)d.sample_rate;
                if (d.in_cycle) delay = fmax(delay, 128. / sr);
                const int i = (int)((ci.f0 + n) & 127);
                double position = (double)i - delay * sr;
                double pf = floor(position);
                m = (ci.f0 + n - i) + (int64_t)pf;
                k = (float)(position - pf);
            }
            float prev = delay_fetch(d, in, ring, m, ci);
            float next = delay_fetch(d, in, ring, m + 1, ci);
            chan(d.out, c, ci)[n] = fmaf(1.f - k, prev, k * next);
        }
    }
}
// the "last quantum whose input had one channel" track of a delay line for the quanta of this chunk (a running maximum: serial)
DEVI void delay_mono_scan(const DelayInst& d, const ChunkInfo& ci) {
    const int64_t q0 = ci.f0 >> 7;
    int64_t last = q0 > 0 ? d.mono_at[(q0 - 1) & (d.mono_len - 1)] : -1;
    for (int q = 0; q < ci.nf / 128; q++) {
        const int qi = meta_qi(ci, q * 128);
        if (buf_count(d.in, d.ch, qi) <= 1) last = q0 + q;  // (a silent quantum has one channel unless the port's count is explicit)
        d.mono_at[(q0 + q) & (d.mono_len - 1)] = last;
    }
}
__global__ void __launch_bounds__(64) k_delay_mono(const DelayInst* __restrict__ insts, int n_inst, ChunkInfo ci) {
    const int ii = blockIdx.x * blockDim.x + threadIdx.x;
    if (ii < n_inst && (insts[ii].dyn & 1)) delay_mono_scan(insts[ii], ci);
}
__global__ void __launch_bounds__(256) k_ring_write(const DelayInst* __restrict__ insts, int n_inst, ChunkInfo ci) {
    for (int ii = blockIdx.y; ii < n_inst; ii += gridDim.y) {
        const DelayInst d = insts[ii];
        int n = blockIdx.x * blockDim.x + threadIdx.x;
        if ((d.dyn & 2) && blockIdx.x == 0 && threadIdx.x == 0) delay_mono_scan(d, ci);  // feedback cycle: the writer runs after the reader
        if (n >= ci.nf || ci.nf - n > (int64_t)d.ring_len) continue;  // only the newest ring_len frames (no slot written twice)
        if (d.dyn) {  // canonical two channels: a one-channel quantum is stored twice, a silent one as zeros
            const int qi = meta_qi(ci, n);
            float l = 0.f, r = 0.f;
            if (!buf_silent(d.in, d.ch, qi)) {
                l = chan(d.in, 0, ci)[n];
                r = (d.ch > 1 && buf_count(d.in, d.ch, qi) >= 2) ? chan(d.in, 1, ci)[n] : l;
            }
            d.ring[(ci.f0 + n) & (d.ring_len - 1)] = l;
            if (d.ch > 1) d.ring[(size_t)d.ring_len + ((ci.f0 + n) & (d.ring_len - 1))] = r;
            continue;
        }
        for (int c = 0; c < d.ch; c++) d.ring[(size_t)c * d.ring_len + ((ci.f0 + n) & (d.ring_len - 1))] = chan(d.in, c, ci)[n];
    }
}

// ---------------------------------------------------------------------------------------------------------
// DynamicsCompressor — DynamicsCompressorRenderer::process (src/node/dynamics_compressor.rs:330-478).
// The branching peak detector is a non-linear serial recurrence: one thread per instance walks the chunk.
// ---------------------------------------------------------------------------------------------------------
DEVI float db_to_lin(float v) { return powf(10.0f, v / 20.f); }
DEVI float lin_to_db(float v) { return v == 0.f ? -1000.f : 20.f * log10f(v); }
// READOUTS: the instances declare reduction read-outs (wae_compressor_set_readouts), `ro` parallel to `insts`: at the end of each
// quantum the reduction is written to the rows of the read-outs at that frame (those at frame 0: at the start of the first chunk)
template <bool READOUTS>
__global__ void __launch_bounds__(32) k_compressor(const CompInst* __restrict__ insts, const CompReadoutInst* __restrict__ ro, int n_inst,
                                                   ChunkInfo ci) {
    int ii = blockIdx.x * blockDim.x + threadIdx.x;
    if (ii >= n_inst) return;
    const CompInst q = insts[ii];
    CompReadoutInst r{};
    int rk = 0;  // the next read-out: the first with frame > f0 (>= 0 in the first chunk)
    if (READOUTS) {
        r = ro[ii];
        const int64_t lo = ci.f0 == 0 ? -1 : ci.f0;
        int b = r.n;
        while (rk < b) {
            const int m = (rk + b) >> 1;
            if (r.frames[m] > lo) b = m;
            else rk = m + 1;
        }
        for (; rk < r.n && r.frames[rk] == 0; rk++) r.rows[rk] = 0.f;  // before the first quantum (the reference's initial value)
    }
    float thr = 0.f, half_knee = 0.f, knee_partial = 0.f, attack_tau = 0.f, release_tau = 0.f, makeup_gain = 0.f, ratio = 1.f;
    const bool automated = q.track[0].p || q.track[1].p || q.track[2].p || q.track[3].p || q.track[4].p;
    float prev = q.state[0];
    float reduction_gain = q.state[1];
    const uint32_t mask = q.ring_len - 1;
    // dynamic input layout: the look-ahead ring holds whole quanta WITH their layout (dynamics_compressor.rs:452-461): the output of
    // quantum q has the channel count / silence of input quantum q - D; the detector reads the channels the current input has
    const bool dyn = q.in.meta != nullptr || q.out.meta != nullptr;
    const int D = q.delay_frames / 128;
    int cur_ch = q.ch, out_ch = q.ch;
    bool cur_silent = false, out_silent = false;
    for (int n = 0; n < ci.nf; n++) {
        if (dyn && (n & 127) == 0) {
            const int qi = meta_qi(ci, n);
            const int64_t q_abs = (ci.f0 + n) >> 7;
            cur_silent = buf_silent(q.in, q.ch, qi);
            cur_ch = buf_count(q.in, q.ch, qi);
            q.meta_ring[q_abs & (COMP_META_RING - 1)] = (uint8_t)(cur_ch | (cur_silent ? WAE_META_SILENT : 0));
            uint8_t dm = (uint8_t)(1 | WAE_META_SILENT);  // the ring starts out as silent quanta (:340-349)
            if (q_abs - D >= 0) dm = q.meta_ring[(q_abs - D) & (COMP_META_RING - 1)];
            out_silent = (dm & WAE_META_SILENT) != 0;
            out_ch = out_silent ? 1 : (dm & 0x3f);
            if (q.out.meta) meta_put_all(q.out, q.ch, qi, out_ch, out_silent);
        }
        if (n == 0 || (automated && (n & 127) == 0)) {  // per-quantum constants (dynamics_compressor.rs:352-391), params are k-rate
            const float attack = q.track[0].p ? chan(q.track[0], 0, ci)[n] : q.attack;
            const float knee = q.track[1].p ? chan(q.track[1], 0, ci)[n] : q.knee;
            ratio = q.track[2].p ? chan(q.track[2], 0, ci)[n] : q.ratio;
            const float release = q.track[3].p ? chan(q.track[3], 0, ci)[n] : q.release;
            const float threshold = q.track[4].p ? chan(q.track[4], 0, ci)[n] : q.threshold;
            thr = knee > 0.f ? threshold + knee / 2.f : threshold;
            half_knee = knee / 2.f;
            knee_partial = (1.f / ratio - 1.f) / (2.f * knee);
            // correctly rounded, as the reference's f32 exp: at high rates 1 - tau is only a few hundred ulps, so expf's error of up
            // to one ulp would change the detector's attack / release rate by up to 1 %
            attack_tau = (float)exp((double)(-1.f / (attack * q.sample_rate)));
            release_tau = (float)exp((double)(-1.f / (release * q.sample_rate)));
            const float full_range_gain = thr + (-thr / ratio);
            const float full_range_makeup = 1.f / db_to_lin(full_range_gain);
            makeup_gain = lin_to_db(powf(full_range_makeup, 0.6f));
        }
        float mx = -3.40282347e+38f;
        for (int c = 0; c < cur_ch; c++) {
            float s = cur_silent ? 0.f : fabsf(chan(q.in, c, ci)[n]);
            if (s > mx) mx = s;
        }
        float sample_db = lin_to_db(mx);
        float att;
        if (sample_db <= thr - half_knee) {
            att = sample_db;
        } else if (sample_db <= thr + half_knee) {
            float t = sample_db - thr + half_knee;
            att = __fadd_rn(sample_db, __fmul_rn(__fmul_rn(t, t), knee_partial));
        } else {
            att = thr + (sample_db - thr) / ratio;
        }
        float attenuation = sample_db - att;
        float det;
        if (attenuation > prev)
            det = __fadd_rn(__fmul_rn(attack_tau, prev), __fmul_rn(1.f - attack_tau, attenuation));
        else
            det = __fadd_rn(__fmul_rn(release_tau, prev), __fmul_rn(1.f - release_tau, attenuation));
        const float red = -det + makeup_gain;
        float g = db_to_lin(red);
        if (ci.f0 + n < q.end) {  // past the graph's own end (a shorter graph of a longer group) the state stays as the render left it
            reduction_gain = red;
            prev = det;
        }
        if (READOUTS && (n & 127) == 127)
            for (; rk < r.n && r.frames[rk] == ci.f0 + n + 1; rk++) r.rows[rk] = reduction_gain;
        int64_t m = ci.f0 + n - q.delay_frames;
        for (int c = 0; c < q.ch; c++) {
            float x = 0.f;
            if (out_silent || c >= out_ch)
                x = 0.f;
            else if (m >= ci.f0)
                x = chan(q.in, c, ci)[m - ci.f0];
            else if (m >= 0)
                x = q.ring[(size_t)c * q.ring_len + (m & mask)];
            chan(q.out, c, ci)[n] = x * g;
        }
    }
    // history for the next chunk
    for (int n = max(0, ci.nf - q.delay_frames); n < ci.nf; n++)
        for (int c = 0; c < q.ch; c++) q.ring[(size_t)c * q.ring_len + ((ci.f0 + n) & mask)] = chan(q.in, c, ci)[n];
    q.state[0] = prev;
    q.state[1] = reduction_gain;
}

// The analyser's mono down-mix of input frame n of the chunk: mono.mix(1, Speakers) (analyser.rs:267-294)
__device__ __forceinline__ float analyser_mono(const BufRef& in, int ch, int n, const ChunkInfo& ci) {
    MixEdge e;
    e.src = in;
    e.src_ch = ch;
    if (in.meta) {  // dynamic input layout: the down-mix sees the channels this quantum has
        const int qi = meta_qi(ci, n);
        e.src_ch = buf_count(in, ch, qi);
        return buf_silent(in, ch, qi) ? 0.f : mixed_sample(e, 1, 0, 0, n, ci);
    }
    return mixed_sample(e, 1, 0, 0, n, ci);
}

// AnalyserRenderer (src/node/analyser.rs:267-294) + AnalyserRingBuffer::write (src/analysis.rs:96-112)
__global__ void __launch_bounds__(256) k_analyser(const AnalyserInst* __restrict__ insts, int n_inst, ChunkInfo ci) {
    const int RING = 32768 + 128;
    for (int ii = blockIdx.y; ii < n_inst; ii += gridDim.y) {
        const AnalyserInst a = insts[ii];
        // frames from the graph's own end on (a shorter graph of a longer group) are not part of its render: they are not recorded
        const int nf_end = (int)max((int64_t)0, min((int64_t)ci.nf, a.end - ci.f0));
        int n = blockIdx.x * blockDim.x + threadIdx.x;
        if (n >= ci.nf) continue;
        const bool record = n < nf_end && nf_end - n <= RING;  // (older than the ring: overwritten by this very chunk)
        if (!a.out.p && !record) continue;
        const float mono = analyser_mono(a.in, a.ch, n, ci);
        if (a.out.p)
            for (int c = 0; c < a.ch; c++) chan(a.out, c, ci)[n] = chan(a.in, c, ci)[n];
        if (record) a.ring[(ci.f0 + n) % RING] = mono;
    }
}

// ---------------------------------------------------------------------------------------------------------
// AudioParam automation — AudioParamProcessor::compute_buffer + mix_to_output (src/param.rs:739-797, 1038-1600).
// Lane 0 of a warp per param instance walks the chunk quantum by quantum through the (host-prepared) event timeline,
// exactly like the reference's per-quantum state machine (set_value / linear & exponential ramps / setTarget with
// snap-to-target / value curves / cancel_and_hold), adds the summed audio-rate input, maps NaN to the default and
// clamps to [min, max].  The output is the param's value for EVERY frame (k-rate and constant blocks are
// replicated), which is what the a-rate consumers read.
// ---------------------------------------------------------------------------------------------------------
constexpr int PARAM_WARPS = 4;
// One WARP per param instance: lane 0 walks the state machine of the quantum (wae_param_core.h, the code the host also runs), the 32
// lanes then add the audio-rate input, map NaN to the default, clamp and store the 128 frames with coalesced accesses.
__global__ void __launch_bounds__(32 * PARAM_WARPS) k_param(const ParamInst* __restrict__ insts, int n_inst, ChunkInfo ci) {
    __shared__ float s_buf[PARAM_WARPS][128];
    __shared__ int s_len[PARAM_WARPS];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ii = blockIdx.x * PARAM_WARPS + w;
    if (ii >= n_inst) return;  // whole warps leave; the loop below only uses warp-level synchronisation
    const ParamInst p = insts[ii];
    ParamState st{};
    if (lane == 0) {
        st = *p.state;
        if (!st.inited) {  // first quantum of this param in this run (start of the render, or of the segment that created it / changed its events)
            st.intrinsic = p.intrinsic0;
            st.head = 0;
            st.has_last = p.has_last0;
            st.last = p.last0;
            st.override_valid = 0;
            st.inited = 1;
        }
    }
    float* out = chan(p.out, 0, ci);
    float* single = chan(p.out, 1, ci);  // [first frame of a quantum] = 1: the reference's output buffer is single-valued
    const float* in = p.in.p ? chan(p.in, 0, ci) : nullptr;
    float* buf = s_buf[w];
    // ---- mix_to_output (param.rs:739-797): + input signal, NaN -> default, clamp
    auto fix = [&](float v) {
        if (v != v) return p.def;
        v = v > p.mn ? v : p.mn;
        return v < p.mx ? v : p.mx;
    };
    for (int q0 = 0; q0 < ci.nf; q0 += 128) {
        if (lane == 0) {
            const double block_time = (double)(ci.f0 + q0) / (double)p.sample_rate;
            s_len[w] = param_compute_buffer(p, st, block_time, buf);
        }
        __syncwarp();
        const int len = s_len[w];
        if (len == 1 || !p.a_rate) {
            const float value = buf[0];
            if (!in || !p.a_rate) {
                const float v = fix(value + (in ? in[q0] : 0.f));
#pragma unroll
                for (int i = lane; i < 128; i += 32) out[q0 + i] = v;
                if (lane == 0) single[q0] = 1.f;
            } else {
#pragma unroll
                for (int i = lane; i < 128; i += 32) out[q0 + i] = fix(in[q0 + i] + value);
                if (lane == 0) single[q0] = 0.f;
            }
        } else {
#pragma unroll
            for (int i = lane; i < 128; i += 32) out[q0 + i] = fix((in ? in[q0 + i] : 0.f) + buf[i]);
            if (lane == 0) single[q0] = 0.f;
        }
        __syncwarp();  // the quantum's values are consumed before lane 0 overwrites them
    }
    if (lane == 0) *p.state = st;
}

// WAE_OPT_PARAM_PARALLEL = 1 (0 selects k_param above, 2 = the default k_param_spec below): lane 0 only WALKS the events of the quantum
// (wae_param_walk.h, recording sink: constants are written, ramps / set-target / curves are recorded as fills), then the 32 lanes evaluate
// the recorded fills, 4 consecutive frames each, re-accumulating `time += dt` from the fill's first frame so that the frame times are the
// reference's running sum.  Bit-equal to k_param on hardware (tests/test_gpu_criterion_and_setters.py renders every automation scenario
// with both and compares the PCM exactly); the walker and the sink are also tested on the host against the reference's event semantics.
__global__ void __launch_bounds__(32 * PARAM_WARPS) k_param_parallel(const ParamInst* __restrict__ insts, int n_inst, ChunkInfo ci) {
    __shared__ float s_buf[PARAM_WARPS][128];
    __shared__ ParamFill s_fill[PARAM_WARPS][RecordSink::kMax];
    __shared__ int s_meta[PARAM_WARPS][3];  // frames written (1 or 128), recorded fills, frames to flush subnormals in
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ii = blockIdx.x * PARAM_WARPS + w;
    if (ii >= n_inst) return;
    const ParamInst p = insts[ii];
    ParamState st{};
    if (lane == 0) {
        st = *p.state;
        if (!st.inited) {
            st.intrinsic = p.intrinsic0;
            st.head = 0;
            st.has_last = p.has_last0;
            st.last = p.last0;
            st.override_valid = 0;
            st.inited = 1;
        }
    }
    float* out = chan(p.out, 0, ci);
    float* single = chan(p.out, 1, ci);
    const float* in = p.in.p ? chan(p.in, 0, ci) : nullptr;
    float* buf = s_buf[w];
    const double dt = 1. / (double)p.sample_rate;  // the walker's own expression
    auto fix = [&](float v) {
        if (v != v) return p.def;
        v = v > p.mn ? v : p.mn;
        return v < p.mx ? v : p.mx;
    };
    for (int q0 = 0; q0 < ci.nf; q0 += 128) {
        if (lane == 0) {
            RecordSink sink;
            sink.buf = buf;
            sink.dt = dt;
            const double block_time = (double)(ci.f0 + q0) / (double)p.sample_rate;
            s_meta[w][0] = param_walk(p, st, block_time, sink);
            for (int k = 0; k < sink.n; k++) s_fill[w][k] = sink.fills[k];
            s_meta[w][1] = sink.n;
            s_meta[w][2] = sink.flush;
        }
        __syncwarp();
        const int len = s_meta[w][0], n_fills = s_meta[w][1], flush = s_meta[w][2];
        for (int k = 0; k < n_fills; k++) {
            const ParamFill f = s_fill[w][k];
            const int from = f.first + 4 * lane, to = min(f.last, from + 4);  // a fill is at most 128 frames = 32 lanes x 4
            if (from < to) param_fill_range(f, from, to, dt, buf);
        }
        __syncwarp();
        for (int i = lane; i < flush; i += 32)
            if (buf[i] != 0.f && fabsf(buf[i]) < 1.17549435e-38f) buf[i] = 0.f;
        __syncwarp();
        if (len == 1 || !p.a_rate) {
            const float value = buf[0];
            if (!in || !p.a_rate) {
                const float v = fix(value + (in ? in[q0] : 0.f));
#pragma unroll
                for (int i = lane; i < 128; i += 32) out[q0 + i] = v;
                if (lane == 0) single[q0] = 1.f;
            } else {
#pragma unroll
                for (int i = lane; i < 128; i += 32) out[q0 + i] = fix(in[q0 + i] + value);
                if (lane == 0) single[q0] = 0.f;
            }
        } else {
#pragma unroll
            for (int i = lane; i < 128; i += 32) out[q0 + i] = fix((in ? in[q0 + i] : 0.f) + buf[i]);
            if (lane == 0) single[q0] = 0.f;
        }
        __syncwarp();
    }
    if (lane == 0) *p.state = st;
}

// The default AudioParam kernel (WAE_OPT_PARAM_PARALLEL = 2): one CTA per automated param, SPECULATIVE walks.  The event state machine
// is serial from quantum to quantum, but almost every quantum leaves it where it was: queue position, last event and override untouched,
// the intrinsic value a closed form of the event at the head of the queue (param_walk leaves par_linear / par_exp / par_target / par_curve
// at next_block_time behind, or nothing at all in a constant block).  So the 32 lanes of warp 0 each walk ONE of the next 32 quanta from a
// PREDICTED state (the current state with that closed form as intrinsic value), and every prediction is then checked against the state
// the walk of the quantum before it actually left: the verified prefix is kept (always at least one quantum, whose input is the real
// state), the rest is thrown away and speculated again from the last verified state.  A wrong prediction costs time, never correctness.
// The recorded fills of the kept quanta are evaluated by all warps.  k_param_parallel walked quantum after quantum with one lane per
// param: 3 - 25 us per quantum, a second of GPU time for two automated params on a 120 s render.
constexpr int PSPEC_WARPS = 8;
constexpr int PSPEC_Q = 32;
__global__ void __launch_bounds__(32 * PSPEC_WARPS) k_param_spec(const ParamInst* __restrict__ insts, int n_inst, ChunkInfo ci) {
    __shared__ float s_buf[PSPEC_Q][129];  // (129: the lanes of warp 0 write their rows at the same column)
    __shared__ ParamFill s_fill[PSPEC_Q][RecordSink::kMax];
    __shared__ int s_meta[PSPEC_Q][3];     // frames written (1 or 128), recorded fills, frames to flush subnormals in
    __shared__ ParamState s_after[PSPEC_Q];
    __shared__ ParamState s_state;
    __shared__ int s_m;
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ii = blockIdx.x;
    if (ii >= n_inst) return;
    const ParamInst p = insts[ii];
    if (threadIdx.x == 0) {
        ParamState st = *p.state;
        if (!st.inited) {
            st.intrinsic = p.intrinsic0;
            st.head = 0;
            st.has_last = p.has_last0;
            st.last = p.last0;
            st.override_valid = 0;
            st.inited = 1;
        }
        s_state = st;
    }
    __syncthreads();
    float* out = chan(p.out, 0, ci);
    float* single = chan(p.out, 1, ci);
    const float* in = p.in.p ? chan(p.in, 0, ci) : nullptr;
    const double dt = 1. / (double)p.sample_rate;  // the walker's own expression
    auto fix = [&](float v) {
        if (v != v) return p.def;
        v = v > p.mn ? v : p.mn;
        return v < p.mx ? v : p.mx;
    };
    for (int q0 = 0; q0 < ci.nf;) {
        const int nq = min(PSPEC_Q, (ci.nf - q0 + 127) / 128);
        if (w == 0) {
            ParamState st = s_state;
            const bool active = lane < nq;
            if (active && lane > 0) {
                const double prev_block_time = (double)(ci.f0 + q0 + 128 * (lane - 1)) / (double)p.sample_rate;
                st.intrinsic = param_predict_intrinsic(p, st, fma(dt, 128., prev_block_time));
            }
            const ParamState before = st;
            RecordSink sink;
            sink.buf = s_buf[lane];
            sink.dt = dt;
            int len = 0;
            if (active) {
                const double block_time = (double)(ci.f0 + q0 + 128 * lane) / (double)p.sample_rate;
                len = param_walk(p, st, block_time, sink);
                s_after[lane] = st;
            }
            __syncwarp();
            const bool ok = active && (lane == 0 || param_state_equal(s_after[lane - 1], before));
            const unsigned good = __ballot_sync(0xffffffffu, ok);
            const int m = __ffs(~good) - 1;  // verified prefix (>= 1: lane 0 walked the real state); 32 verified: ~good == 0 -> ffs 0 -> -1
            const int keep = m < 0 ? 32 : m;
            if (lane < keep) {
                for (int k = 0; k < sink.n; k++) s_fill[lane][k] = sink.fills[k];
                s_meta[lane][0] = len;
                s_meta[lane][1] = sink.n;
                s_meta[lane][2] = sink.flush;
            }
            if (lane == keep - 1) s_state = st;
            if (lane == 0) s_m = keep;
        }
        __syncthreads();
        const int m = s_m;
        for (int j = w; j < m; j += PSPEC_WARPS) {
            float* buf = s_buf[j];
            const int qf = q0 + 128 * j;
            const int len = s_meta[j][0], n_fills = s_meta[j][1], flush = s_meta[j][2];
            for (int k = 0; k < n_fills; k++) {
                const ParamFill f = s_fill[j][k];
                const int from = f.first + 4 * lane, to = min(f.last, from + 4);  // a fill is at most 128 frames = 32 lanes x 4
                if (from < to) param_fill_range(f, from, to, dt, buf);
            }
            __syncwarp();
            for (int i = lane; i < flush; i += 32)
                if (buf[i] != 0.f && fabsf(buf[i]) < 1.17549435e-38f) buf[i] = 0.f;
            __syncwarp();
            if (len == 1 || !p.a_rate) {
                const float value = buf[0];
                if (!in || !p.a_rate) {
                    const float v = fix(value + (in ? in[qf] : 0.f));
#pragma unroll
                    for (int i = lane; i < 128; i += 32) out[qf + i] = v;
                    if (lane == 0) single[qf] = 1.f;
                } else {
#pragma unroll
                    for (int i = lane; i < 128; i += 32) out[qf + i] = fix(in[qf + i] + value);
                    if (lane == 0) single[qf] = 0.f;
                }
            } else {
#pragma unroll
                for (int i = lane; i < 128; i += 32) out[qf + i] = fix((in ? in[qf + i] : 0.f) + buf[i]);
                if (lane == 0) single[qf] = 0.f;
            }
        }
        __syncthreads();
        q0 += 128 * m;
    }
    if (threadIdx.x == 0) *p.state = s_state;
}

// ---------------------------------------------------------------------------------------------------------
// Convolver — ConvolverRenderer (src/node/convolver.rs:343-490).  The reference runs fft-convolver's uniformly
// partitioned overlap-save with 1024-frame partitions because it must answer every 128 frames; an offline batch has no
// such deadline, so the same linear convolution is evaluated time-batched with B = 8192-frame partitions (FFT 16384):
// 8x fewer partitions => 8x less spectrum traffic and MAC work per output frame.  Per chunk:
//   k_conv_fft_in : X_j = FFT([block j-1 | block j])                         CTA per (input channel, block), smem FFT (DIF)
//   k_conv_mac    : Y_j = sum_i H_i * X_{j-i}  for CV_J output blocks at once  thread per bin, register tiled over j
//   k_conv_ifft   : out_j = IFFT(Y_j)[B..2B) / 2B                              CTA per (path, block), smem FFT (DIT)
// Real FFTs of 2B points are computed as complex FFTs of B points (packed even/odd) in shared memory (64 KB); spectra are kept in
// bit-reversed ("position") order end to end, see below.
// ---------------------------------------------------------------------------------------------------------
constexpr int CV_B = WAE_CONV_BLOCK;    // frames per partition
constexpr int CV_LOGB = 13;
static_assert((1 << CV_LOGB) == CV_B, "CV_LOGB");
constexpr int CV_BINS = CV_B;           // packed half spectrum: bin 0 = (DC, Nyquist), bins 1..B-1 complex
constexpr int CV_THREADS = 256;
constexpr int CV_ROWS = CV_B / 32;      // warp rows of a spectrum

__device__ float2 c_tw[CV_B];           // exp(-2*pi*i*k/(2B)), k < B
__constant__ float2 c_rowtw[CV_ROWS];   // c_tw[brev8(r)]: the warp-uniform factor of a bin's real-FFT twiddle when lanes walk POSITIONS (below)
static float2 h_tw[CV_B];               // host copy (wae_selftest_conv_fft)

#define WAE_HD __host__ __device__ __forceinline__
// the library is built with -fmad=false (the reference's arithmetic is unfused); the transforms are compared at a tolerance against a
// different FFT anyway (rustfft), so their complex multiply asks for the fused form explicitly: 4 instructions instead of 6
WAE_HD float2 cmul(float2 a, float2 b) { return make_float2(fmaf(a.x, b.x, -(a.y * b.y)), fmaf(a.x, b.y, a.y * b.x)); }
WAE_HD float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
WAE_HD float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }

// B-point (8192) complex FFTs in shared memory with the butterflies in registers: radix 8 x 8 x 8 x 16, 4 passes / 3 barriers instead of 13
// radix-2 stages.  Two flow graphs, so that no pass ever permutes:
//   forward  = decimation in frequency: natural order in, BIT-REVERSED order out (element k at position brev13(k));
//   inverse  = decimation in time:      bit-reversed order in, natural order out.
// Spectra therefore live in HBM in POSITION order (X[p] = bin brev13(p)) — the MAC between the two transforms is bin-wise and does not care,
// and the real-FFT split pairs position p with the position of bin B-k, which for 32 consecutive p is 32 consecutive positions in reverse:
// both shared-memory reads are conflict free and both HBM accesses coalesced (round 1 indexed bins in natural order through cv_pos(): a
// 16-way bank conflict on every read, twice the shared-memory wavefronts of the four FFT passes together).
// Storage is padded by one float2 per 16 so that the contiguous radix-16 pass is free of bank conflicts.  sign = -1 forward, +1 inverse.
constexpr int CV_SMEM_ELEMS = CV_B + CV_B / 16;
WAE_HD int cv_pad(int i) { return i + (i >> 4); }
WAE_HD int cv_brev(int k) {
#ifdef __CUDA_ARCH__
    return (int)(__brev((unsigned)k) >> (32 - CV_LOGB));
#else
    int r = 0;
    for (int b = 0; b < CV_LOGB; b++) r |= ((k >> b) & 1) << (CV_LOGB - 1 - b);
    return r;
#endif
}
// multiply by exp(sign * 2*pi*i * m / 16)
template <int M>
WAE_HD float2 rot16(float2 v, int sign) {
    constexpr float C1 = 0.92387953251128675613f, S1 = 0.38268343236508977173f, R = 0.70710678118654752440f;
    constexpr int m = M & 15;
    float c, sn;
    if (m == 0) return v;
    if (m == 4) return sign > 0 ? make_float2(-v.y, v.x) : make_float2(v.y, -v.x);
    if (m == 8) return make_float2(-v.x, -v.y);
    if (m == 12) return sign > 0 ? make_float2(v.y, -v.x) : make_float2(-v.y, v.x);
    // cos / sin of 2*pi*m/16
    if (m == 1) c = C1, sn = S1;
    else if (m == 2) c = R, sn = R;
    else if (m == 3) c = S1, sn = C1;
    else if (m == 5) c = -S1, sn = C1;
    else if (m == 6) c = -R, sn = R;
    else if (m == 7) c = -C1, sn = S1;
    else if (m == 9) c = -C1, sn = -S1;
    else if (m == 10) c = -R, sn = -R;
    else if (m == 11) c = -S1, sn = -C1;
    else if (m == 13) c = S1, sn = -C1;
    else if (m == 14) c = R, sn = -R;
    else c = C1, sn = -S1;
    if (sign < 0) sn = -sn;
    return make_float2(fmaf(v.x, c, -(v.y * sn)), fmaf(v.x, sn, v.y * c));
}
// radix-8 butterfly on elements base + m*q (radix-2 spans 4q, 2q, q) with t1 = exp(sign*2*pi*i*lo/(8q)); the twiddles of the two
// inner spans are its square and fourth power
WAE_HD void bf8_dif(float2 (&a)[8], float2 t1, int sign) {
    const float2 t2 = cmul(t1, t1), t3 = cmul(t2, t2);
    float2 u, v;
    u = cadd(a[0], a[4]); v = csub(a[0], a[4]); a[0] = u; a[4] = cmul(v, t1);
    u = cadd(a[1], a[5]); v = csub(a[1], a[5]); a[1] = u; a[5] = cmul(rot16<2>(v, sign), t1);
    u = cadd(a[2], a[6]); v = csub(a[2], a[6]); a[2] = u; a[6] = cmul(rot16<4>(v, sign), t1);
    u = cadd(a[3], a[7]); v = csub(a[3], a[7]); a[3] = u; a[7] = cmul(rot16<6>(v, sign), t1);
#pragma unroll
    for (int g = 0; g < 8; g += 4) {
        u = cadd(a[g], a[g + 2]); v = csub(a[g], a[g + 2]); a[g] = u; a[g + 2] = cmul(v, t2);
        u = cadd(a[g + 1], a[g + 3]); v = csub(a[g + 1], a[g + 3]); a[g + 1] = u; a[g + 3] = cmul(rot16<4>(v, sign), t2);
    }
#pragma unroll
    for (int m = 0; m < 8; m += 2) {
        u = cadd(a[m], a[m + 1]); v = csub(a[m], a[m + 1]); a[m] = u; a[m + 1] = cmul(v, t3);
    }
}
// the transposed flow graph: twiddle first, spans q, 2q, 4q
WAE_HD void bf8_dit(float2 (&a)[8], float2 t1, int sign) {
    const float2 t2 = cmul(t1, t1), t3 = cmul(t2, t2);
    float2 u, v;
#pragma unroll
    for (int m = 0; m < 8; m += 2) {
        v = cmul(a[m + 1], t3); u = a[m]; a[m] = cadd(u, v); a[m + 1] = csub(u, v);
    }
#pragma unroll
    for (int g = 0; g < 8; g += 4) {
        v = cmul(a[g + 2], t2); u = a[g]; a[g] = cadd(u, v); a[g + 2] = csub(u, v);
        v = rot16<4>(cmul(a[g + 3], t2), sign); u = a[g + 1]; a[g + 1] = cadd(u, v); a[g + 3] = csub(u, v);
    }
    v = cmul(a[4], t1); u = a[0]; a[0] = cadd(u, v); a[4] = csub(u, v);
    v = rot16<2>(cmul(a[5], t1), sign); u = a[1]; a[1] = cadd(u, v); a[5] = csub(u, v);
    v = rot16<4>(cmul(a[6], t1), sign); u = a[2]; a[2] = cadd(u, v); a[6] = csub(u, v);
    v = rot16<6>(cmul(a[7], t1), sign); u = a[3]; a[3] = cadd(u, v); a[7] = csub(u, v);
}
// four radix-2 stages on 16 contiguous elements: all twiddles are 16th roots of unity
WAE_HD void bf16_dif(float2 (&a)[16], int sign) {
    float2 u, v;
#define WAE_BF(i, j, M) u = cadd(a[i], a[j]); v = csub(a[i], a[j]); a[i] = u; a[j] = rot16<M>(v, sign);
    WAE_BF(0, 8, 0) WAE_BF(1, 9, 1) WAE_BF(2, 10, 2) WAE_BF(3, 11, 3) WAE_BF(4, 12, 4) WAE_BF(5, 13, 5) WAE_BF(6, 14, 6) WAE_BF(7, 15, 7)
#pragma unroll
    for (int g = 0; g < 16; g += 8) {
        WAE_BF(g, g + 4, 0) WAE_BF(g + 1, g + 5, 2) WAE_BF(g + 2, g + 6, 4) WAE_BF(g + 3, g + 7, 6)
    }
#pragma unroll
    for (int g = 0; g < 16; g += 4) {
        WAE_BF(g, g + 2, 0) WAE_BF(g + 1, g + 3, 4)
    }
#pragma unroll
    for (int g = 0; g < 16; g += 2) {
        WAE_BF(g, g + 1, 0)
    }
#undef WAE_BF
}
WAE_HD void bf16_dit(float2 (&a)[16], int sign) {
    float2 u, v;
#define WAE_BF(i, j, M) v = rot16<M>(a[j], sign); u = a[i]; a[i] = cadd(u, v); a[j] = csub(u, v);
#pragma unroll
    for (int g = 0; g < 16; g += 2) {
        WAE_BF(g, g + 1, 0)
    }
#pragma unroll
    for (int g = 0; g < 16; g += 4) {
        WAE_BF(g, g + 2, 0) WAE_BF(g + 1, g + 3, 4)
    }
#pragma unroll
    for (int g = 0; g < 16; g += 8) {
        WAE_BF(g, g + 4, 0) WAE_BF(g + 1, g + 5, 2) WAE_BF(g + 2, g + 6, 4) WAE_BF(g + 3, g + 7, 6)
    }
    WAE_BF(0, 8, 0) WAE_BF(1, 9, 1) WAE_BF(2, 10, 2) WAE_BF(3, 11, 3) WAE_BF(4, 12, 4) WAE_BF(5, 13, 5) WAE_BF(6, 14, 6) WAE_BF(7, 15, 7)
#undef WAE_BF
}
// Pass twiddles out of registers.  Thread t handles butterflies bf = t + 256*it of a radix-8 pass with span q; lo = bf & (q-1) is
//   q = 1024: t + 256*it -> exp(s*2*pi*i*t/8192) * exp(s*2*pi*i*it/32)      (one table value + a compile-time rotation per butterfly)
//   q = 128 : t & 127                                                         (one table value for the whole pass)
//   q = 16  : t & 15
// so a thread reads THREE table entries per transform, before its input loads, instead of one L2-latency gather per butterfly (the 64 KB
// table does not survive in an L1 that shares 256 KB with 3 x 68 KB of shared memory: long_scoreboard 6 - 7 per issue in round 1's profile).
struct FftTw { float2 w1, w2, w3; };
static_assert(CV_THREADS == 256 && CV_LOGB == 13, "FftTw assumes 4 radix-8 butterflies per thread and spans 1024 / 128 / 16");
WAE_HD FftTw fft_tw_of(const float2* tw, int t, int sign) {
    FftTw w;
    w.w1 = tw[t << 1];
    w.w2 = tw[(t & 127) << 4];
    w.w3 = tw[(t & 15) << 7];
    if (sign > 0) w.w1.y = -w.w1.y, w.w2.y = -w.w2.y, w.w3.y = -w.w3.y;
    return w;
}
WAE_HD float2 tw_it(float2 w1, int it, int sign) {  // w1 * exp(sign*2*pi*i*it/32)
    float c, s;
    if (it == 0) return w1;
    if (it == 1) c = 0.98078528040323044913f, s = 0.19509032201612826785f;
    else if (it == 2) c = 0.92387953251128675613f, s = 0.38268343236508977173f;
    else c = 0.83146961230254523708f, s = 0.55557023301960222474f;
    return cmul(w1, make_float2(c, sign > 0 ? s : -s));
}
template <int LOG_Q, bool DIT>
WAE_HD void fft_pass8_one(float2* s, int t, int it, const FftTw& w, int sign) {
    constexpr int q = 1 << LOG_Q;
    const int bf = t + it * CV_THREADS;
    const int lo = bf & (q - 1), hi = bf >> LOG_Q;
    const int base = (hi << (LOG_Q + 3)) + lo;
    float2 a[8];
#pragma unroll
    for (int m = 0; m < 8; m++) a[m] = s[cv_pad(base + m * q)];
    const float2 t1 = LOG_Q == 10 ? tw_it(w.w1, it, sign) : (LOG_Q == 7 ? w.w2 : w.w3);
    if (DIT) bf8_dit(a, t1, sign);
    else bf8_dif(a, t1, sign);
#pragma unroll
    for (int m = 0; m < 8; m++) s[cv_pad(base + m * q)] = a[m];
}
template <bool DIT>
WAE_HD void fft_pass16_one(float2* s, int t, int it, int sign) {
    float2 a[16];
    float2* p = s + cv_pad((t + it * CV_THREADS) * 16);  // 16 contiguous elements never straddle a pad slot
#pragma unroll
    for (int m = 0; m < 16; m++) a[m] = p[m];
    if (DIT) bf16_dit(a, sign);
    else bf16_dif(a, sign);
#pragma unroll
    for (int m = 0; m < 16; m++) p[m] = a[m];
}
#ifndef WAE_CV_UNROLL
#define WAE_CV_UNROLL 2   // radix-8 butterflies of one thread in flight (4 = all of a pass; registers decide)
#endif
template <int LOG_Q, bool DIT>
DEVI void fft_pass8(float2* s, const FftTw& w, int sign) {
#pragma unroll 1
    for (int i0 = 0; i0 < CV_B / 8 / CV_THREADS; i0 += WAE_CV_UNROLL) {
#pragma unroll
        for (int u = 0; u < WAE_CV_UNROLL; u++) fft_pass8_one<LOG_Q, DIT>(s, threadIdx.x, i0 + u, w, sign);
    }
}
template <bool DIT>
DEVI void fft_pass16(float2* s, int sign) {
#pragma unroll 1
    for (int it = 0; it < CV_B / 16 / CV_THREADS; it++) fft_pass16_one<DIT>(s, threadIdx.x, it, sign);
}
DEVI FftTw fft_tw_load(int sign) { return fft_tw_of(c_tw, threadIdx.x, sign); }
// natural order in -> position order out
DEVI void fft_dif_smem(float2* s, const FftTw& w) {
    fft_pass8<10, false>(s, w, -1);
    __syncthreads();
    fft_pass8<7, false>(s, w, -1);
    __syncthreads();
    fft_pass8<4, false>(s, w, -1);
    __syncthreads();
    fft_pass16<false>(s, -1);
    __syncthreads();
}
// position order in -> natural order out (unnormalised inverse)
DEVI void fft_dit_smem(float2* s, const FftTw& w) {
    fft_pass16<true>(s, +1);
    __syncthreads();
    fft_pass8<4, true>(s, w, +1);
    __syncthreads();
    fft_pass8<7, true>(s, w, +1);
    __syncthreads();
    fft_pass8<10, true>(s, w, +1);
    __syncthreads();
}
// exp(-2*pi*i*k/(2B)) for the bin at position p = lane + 32*row: k = brev13(p) = brev5(lane) << 8 | brev8(row), so the twiddle is the
// product of a per-lane value (loaded once per thread) and a per-row value that is uniform across the warp (constant cache broadcast)
DEVI float2 cv_lane_tw() { return c_tw[cv_brev(threadIdx.x & 31)]; }
DEVI float2 cv_bin_tw(float2 lane_tw, int p) { return cmul(lane_tw, c_rowtw[p >> 5]); }
// position of the mirror bin B - k of the bin at position p (p > 0)
WAE_HD int cv_mirror(int p) { return cv_brev(CV_B - cv_brev(p)); }
// one packed bin of the 2B-point real FFT from the B-point transform of (even, odd): X[k] = E[k] + w^k O[k], zm = Z[B - k], tw = w^k
WAE_HD float2 rfft_split(float2 zk, float2 zm, float2 tw) {
    const float2 zc = make_float2(zm.x, -zm.y);
    const float2 e = make_float2(0.5f * (zk.x + zc.x), 0.5f * (zk.y + zc.y));
    const float2 d = make_float2(zk.x - zc.x, zk.y - zc.y);
    const float2 o = make_float2(0.5f * d.y, -0.5f * d.x);
    const float2 r = cmul(tw, o);
    return make_float2(e.x + r.x, e.y + r.y);
}
// and back: the input element of the B-point inverse transform from Y[k], Y[B - k] (twice E + i O; the 1 / 2B scale comes at the end)
WAE_HD float2 irfft_merge(float2 yk, float2 ym, float2 tw) {
    const float2 yc = make_float2(ym.x, -ym.y);
    const float2 e = make_float2(yk.x + yc.x, yk.y + yc.y);
    const float2 d = make_float2(yk.x - yc.x, yk.y - yc.y);
    const float2 o = cmul(make_float2(tw.x, -tw.y), d);
    return make_float2(e.x - o.y, e.y + o.x);
}
// forward transform z (position order, padded) -> the B packed bins of the 2B-point real FFT in position order
DEVI void rfft_store(const float2* z, float2* __restrict__ X, float2 lane_tw) {
#pragma unroll 4
    for (int p = threadIdx.x; p < CV_B; p += CV_THREADS) {
        float2 r;
        if (p == 0) {
            const float2 z0 = z[0];
            r = make_float2(z0.x + z0.y, z0.x - z0.y);  // (DC, Nyquist)
        } else {
            r = rfft_split(z[cv_pad(p)], z[cv_pad(cv_mirror(p))], cv_bin_tw(lane_tw, p));
        }
        X[p] = r;
    }
}
// B reals (valid <= B of them readable at src, the rest zero; src == nullptr: all zero) -> B/2 packed complex (even, odd) at z[c0 ..)
// src2 != nullptr: the speakers down-mix of two channels, 0.5 * (a + b) (quantum.rs 2 -> 1; ConvInput::in_channel = -1)
DEVI void conv_load_half(float2* z, int c0, const float* __restrict__ src, int valid, const float* __restrict__ src2 = nullptr) {
    const int t = threadIdx.x;
    if (!src || valid <= 0) {
        for (int i = t; i < CV_B / 2; i += CV_THREADS) z[cv_pad(c0 + i)] = make_float2(0.f, 0.f);
    } else if (src2 && ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(src2)) & 15) == 0) {
#pragma unroll 8
        for (int i4 = t; i4 < CV_B / 4; i4 += CV_THREADS) {
            const int n = 4 * i4;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (n + 3 < valid) {
                const float4 a = *reinterpret_cast<const float4*>(src + n), c = *reinterpret_cast<const float4*>(src2 + n);
                v = make_float4(0.5f * (a.x + c.x), 0.5f * (a.y + c.y), 0.5f * (a.z + c.z), 0.5f * (a.w + c.w));
            } else if (n < valid) {
                v.x = 0.5f * (src[n] + src2[n]);
                if (n + 1 < valid) v.y = 0.5f * (src[n + 1] + src2[n + 1]);
                if (n + 2 < valid) v.z = 0.5f * (src[n + 2] + src2[n + 2]);
            }
            float2* d = z + cv_pad(c0 + 2 * i4);
            d[0] = make_float2(v.x, v.y);
            d[1] = make_float2(v.z, v.w);
        }
    } else if (src2) {
        for (int i = t; i < CV_B / 2; i += CV_THREADS) {
            const int n = 2 * i;
            z[cv_pad(c0 + i)] = make_float2(n < valid ? 0.5f * (src[n] + src2[n]) : 0.f, n + 1 < valid ? 0.5f * (src[n + 1] + src2[n + 1]) : 0.f);
        }
    } else if ((reinterpret_cast<uintptr_t>(src) & 15) == 0) {
#pragma unroll 8
        for (int i4 = t; i4 < CV_B / 4; i4 += CV_THREADS) {
            const int n = 4 * i4;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (n + 3 < valid) v = *reinterpret_cast<const float4*>(src + n);
            else if (n < valid) {
                v.x = src[n];
                if (n + 1 < valid) v.y = src[n + 1];
                if (n + 2 < valid) v.z = src[n + 2];
            }
            float2* d = z + cv_pad(c0 + 2 * i4);  // complex 2*i4 and 2*i4 + 1 share a 16-group (c0 is a multiple of 16)
            d[0] = make_float2(v.x, v.y);
            d[1] = make_float2(v.z, v.w);
        }
    } else {
        for (int i = t; i < CV_B / 2; i += CV_THREADS) {
            const int n = 2 * i;
            z[cv_pad(c0 + i)] = make_float2(n < valid ? src[n] : 0.f, n + 1 < valid ? src[n + 1] : 0.f);
        }
    }
}

// grid: (blocks in chunk, conv inputs).  Builds X_j for every new block of the chunk.
__global__ void __launch_bounds__(CV_THREADS, 3) k_conv_fft_in(const ConvInput* __restrict__ inputs, int n_inputs, ChunkInfo ci) {
    extern __shared__ float2 z[];
    const FftTw w = fft_tw_load(-1);  // table latency hides behind the input loads
    const float2 lane_tw = cv_lane_tw();
    const ConvInput ip = inputs[blockIdx.y];
    const int jb = blockIdx.x;                         // block within the chunk
    const int64_t jabs = ci.f0 / CV_B + jb;            // absolute block index
    // the graph's end (a graph shorter than its group): a block starting there is never read for a frame before it, and the input from
    // there on is zero, as in the graph's own render, whose last chunk ends there
    const int64_t to_end = ip.end - (ci.f0 + (int64_t)jb * CV_B);
    if (to_end <= 0) return;
    const bool mix = ip.in_channel < 0;
    const float* in = chan(ip.in, mix ? 0 : ip.in_channel, ci);
    const float* in2 = mix ? chan(ip.in, 1, ci) : nullptr;
    // frame = [previous block | current block]
    const int64_t left = min((int64_t)ci.nf - (int64_t)jb * CV_B, to_end);
    if (jb == 0) conv_load_half(z, 0, ip.prev, CV_B);  // (already mixed)
    else conv_load_half(z, 0, in + (size_t)(jb - 1) * CV_B, CV_B, mix ? in2 + (size_t)(jb - 1) * CV_B : nullptr);
    conv_load_half(z, CV_B / 2, in + (size_t)jb * CV_B, (int)(left < CV_B ? left : CV_B), mix ? in2 + (size_t)jb * CV_B : nullptr);
    __syncthreads();
    fft_dif_smem(z, w);
    rfft_store(z, ip.xring + (size_t)(jabs % ip.xring_blocks) * CV_BINS, lane_tw);
}

// saves the last block of the chunk as "previous block" for the next chunk.  grid: (B / 256, conv inputs)
__global__ void __launch_bounds__(256) k_conv_save_prev(const ConvInput* __restrict__ inputs, int n_inputs, ChunkInfo ci) {
    const ConvInput ip = inputs[blockIdx.y];
    const bool mix = ip.in_channel < 0;
    const float* in = chan(ip.in, mix ? 0 : ip.in_channel, ci);
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int nblocks = (ci.nf + CV_B - 1) / CV_B;
    const int64_t m = (int64_t)(nblocks - 1) * CV_B + i;
    float v = m < ci.nf ? in[m] : 0.f;
    if (mix && m < ci.nf) v = 0.5f * (v + chan(ip.in, 1, ci)[m]);
    ip.prev[i] = v;
}

// grid: (B / 256 * ceil(blocks in chunk / CV_J), paths), 256 threads, one bin per thread.  For CV_J consecutive output
// blocks j at once: Y_j = sum_i H_i X_{j-i}.  Register tiling over the block axis: the input blocks are walked in
// groups of CV_J; a group needs 2*CV_J-1 IR spectrum values and CV_J input spectrum values per bin for CV_J^2 complex
// MACs (0.36 loads per MAC instead of 2).  No shared memory => many resident warps hide the L2 latency of the loads.
// The products of a group are taken DIAGONAL by diagonal (d = jj - r selects one H_i, i = i_base + d): a diagonal outside 0 <= i < S is
// skipped by a warp-uniform branch, so the triangles at the head (i < 0) and at the tail (i >= S) of the walk cost nothing — S = 22
// used to pay 228 complex MACs per bin for 176.  The group's loads sit at compile-time offsets of two pointers (one ring / range test
// per group instead of three integer instructions per load: the kernel was bound by issue slots, ALU pipe above the FMA pipe).
constexpr int CV_J = 8;
constexpr int CV_MAC_THREADS = 256;
// PACKED: bin 0 holds (DC, Nyquist), two real bins that multiply component-wise.  FIRST: the head group (i_base = 0), only i = jj - r >= 0.
// The IR spectra are stored with WAE_CONV_H_PAD_LO zero partitions before H_0 and zero partitions behind H_{S-1} up to the end of the
// last group (plan_convolver): the loads of a group need no range tests at all — 23 loads and 256 FMAs per group, where the tests of
// the exact walk cost more issue slots than the multiplications with zero they saved (the ALU pipe, not the FMA pipe, was the busier one).
template <bool PACKED, bool FIRST>
DEVI void conv_mac_group(const float2* __restrict__ hp /* H_{i_base - (CV_J - 1)}[k] */, const float2 (&x)[CV_J], float2 acc[CV_J]) {
    float2 hw[2 * CV_J - 1];
#pragma unroll
    for (int u = FIRST ? CV_J - 1 : 0; u < 2 * CV_J - 1; u++) hw[u] = __ldg(hp + (size_t)u * CV_BINS);
#pragma unroll
    for (int r = 0; r < CV_J; r++) {
#pragma unroll
        for (int jj = FIRST ? r : 0; jj < CV_J; jj++) {
            const float2 h = hw[(CV_J - 1) + jj - r];
            if (PACKED) {
                acc[jj].x = fmaf(h.x, x[r].x, acc[jj].x);
                acc[jj].y = fmaf(h.y, x[r].y, acc[jj].y);
            } else {
                acc[jj].x = fmaf(h.x, x[r].x, fmaf(-h.y, x[r].y, acc[jj].x));
                acc[jj].y = fmaf(h.x, x[r].y, fmaf(h.y, x[r].x, acc[jj].y));
            }
        }
    }
}
template <bool PACKED>
DEVI void conv_mac_bin(const ConvPath& p, const ConvInput& ip, int k, int64_t jabs0, int64_t jabs_last, float2 acc[CV_J]) {
    const int groups = (p.S - 1 + CV_J - 1) / CV_J + 1;  // i runs up to S-1: i_base - (J-1) <= S-1
    const int ring = ip.xring_blocks;
    // ring slot of input block jabs0 (>= 0), walked backwards by CV_J per group without a division
    int slot0 = (int)(jabs0 % ring);
    const float2* hp = p.h + k - (ptrdiff_t)(CV_J - 1) * CV_BINS;  // (inside the zero partitions in front of H_0)
    const float2* __restrict__ xr = ip.xring + k;                  // (written by the previous launch: read-only here)
    int64_t b0 = jabs0;
#pragma unroll 1
    for (int g = 0; g < groups; g++) {
        float2 x[CV_J];
        if (slot0 + CV_J <= ring && b0 >= 0 && b0 + (CV_J - 1) <= jabs_last) {  // (uniform) eight produced blocks in eight consecutive slots
            const float2* xp = xr + (size_t)slot0 * CV_BINS;
#pragma unroll
            for (int r = 0; r < CV_J; r++) x[r] = __ldg(xp + (size_t)r * CV_BINS);
        } else {
#pragma unroll
            for (int r = 0; r < CV_J; r++) {
                const int64_t bb = b0 + r;
                int slot = slot0 + r;
                while (slot >= ring) slot -= ring;  // (rings shorter than CV_J blocks: tiny chunk option + one-partition IR)
                x[r] = (bb >= 0 && bb <= jabs_last) ? __ldg(xr + (size_t)slot * CV_BINS) : make_float2(0.f, 0.f);
            }
        }
        if (g == 0) conv_mac_group<PACKED, true>(hp, x, acc);
        else conv_mac_group<PACKED, false>(hp, x, acc);
        hp += (size_t)CV_J * CV_BINS;
        b0 -= CV_J;
        slot0 -= CV_J;
        while (slot0 < 0) slot0 += ring;  // only meaningful while b0 >= 0; older blocks are skipped by the range test
    }
}
#ifndef WAE_CV_MAC_MINB
#define WAE_CV_MAC_MINB 3
#endif
__global__ void __launch_bounds__(CV_MAC_THREADS, WAE_CV_MAC_MINB) k_conv_mac(const ConvPath* __restrict__ paths, const ConvInput* __restrict__ inputs, int n_paths,
                                                             ChunkInfo ci) {
    const ConvPath p = paths[blockIdx.y];
    if (p.S == 1) return;  // one partition: the product is formed by k_conv_ifft while it loads (Y never exists)
    const ConvInput ip = inputs[p.input];
    const int nb = (ci.nf + CV_B - 1) / CV_B;
    constexpr int TILES = CV_B / CV_MAC_THREADS;
    const int k = (blockIdx.x % TILES) * CV_MAC_THREADS + threadIdx.x;  // bin (position order: index 0 is still the packed DC / Nyquist pair)
    const int j0 = (blockIdx.x / TILES) * CV_J;                         // first output block of this CTA (chunk-relative)
    if (ci.f0 + (int64_t)j0 * CV_B >= p.end) return;                  // past the graph's end (a graph shorter than its group)
    const int64_t jabs0 = ci.f0 / CV_B + j0;
    const int64_t jabs_last = ci.f0 / CV_B + nb - 1;                    // newest input block transformed so far
    float2 acc[CV_J];
#pragma unroll
    for (int jj = 0; jj < CV_J; jj++) acc[jj] = make_float2(0.f, 0.f);
    if (k == 0) conv_mac_bin<true>(p, ip, k, jabs0, jabs_last, acc);
    else conv_mac_bin<false>(p, ip, k, jabs0, jabs_last, acc);
#pragma unroll
    for (int jj = 0; jj < CV_J; jj++)
        if (j0 + jj < nb) p.y[(size_t)(j0 + jj) * CV_BINS + k] = acc[jj];
}

// grid: (blocks in chunk, paths): out_j = IFFT(Y_j)[B..2B) / 2B
// A response of ONE partition (a static HRTF panner's: ~560 taps) needs no k_conv_mac pass: Y_j = H_0 X_j is formed here, from the
// input spectra ring, while the half spectrum is loaded (k_conv_mac skips such paths).
__global__ void __launch_bounds__(CV_THREADS, 3) k_conv_ifft(const ConvPath* __restrict__ paths, const ConvInput* __restrict__ inputs, int n_paths, ChunkInfo ci) {
    extern __shared__ float2 z[];
    const FftTw w = fft_tw_load(+1);
    const float2 lane_tw = cv_lane_tw();
    const ConvPath p = paths[blockIdx.y];
    const int jb = blockIdx.x;
    if (ci.f0 + (int64_t)jb * CV_B >= p.end) return;  // past the graph's end (a graph shorter than its group)
    const float2* __restrict__ Y = p.y + (size_t)jb * CV_BINS;
    const int t = threadIdx.x;
    if (p.S == 1) {
        const ConvInput ip = inputs[p.input];
        const int64_t jabs = ci.f0 / CV_B + jb;
        const float2* __restrict__ X = ip.xring + (size_t)(jabs % ip.xring_blocks) * CV_BINS;
        const float2* __restrict__ H = p.h;
        auto prod = [&](int q) {
            const float2 h = __ldg(H + q), x = __ldg(X + q);
            return make_float2(fmaf(h.x, x.x, __fmul_rn(-h.y, x.y)), fmaf(h.x, x.y, __fmul_rn(h.y, x.x)));
        };
#pragma unroll 4
        for (int q = t; q < CV_B; q += CV_THREADS) {
            float2 yk, ym;
            if (q == 0) {  // (DC, Nyquist): two real bins that multiply component-wise
                const float2 h = __ldg(H), x = __ldg(X);
                yk = make_float2(h.x * x.x, 0.f);
                ym = make_float2(h.y * x.y, 0.f);
            } else {
                yk = prod(q);
                ym = prod(cv_mirror(q));
            }
            z[cv_pad(q)] = irfft_merge(yk, ym, cv_bin_tw(lane_tw, q));
        }
    } else {
    // half spectrum (position order) -> packed complex input of the B-point inverse transform, same positions
#pragma unroll 4
    for (int q = t; q < CV_B; q += CV_THREADS) {
        float2 yk, ym;
        if (q == 0) {
            const float2 y0 = Y[0];
            yk = make_float2(y0.x, 0.f);
            ym = make_float2(y0.y, 0.f);
        } else {
            yk = Y[q];
            ym = Y[cv_mirror(q)];
        }
        z[cv_pad(q)] = irfft_merge(yk, ym, cv_bin_tw(lane_tw, q));
    }
    }
    __syncthreads();
    fft_dit_smem(z, w);
    const float scale = 1.f / (float)(2 * CV_B);
    float* out = chan(p.out, p.out_channel, ci) + (size_t)jb * CV_B;
    int64_t left = (int64_t)ci.nf - (int64_t)jb * CV_B;
    if (p.limit >= 0 && p.limit - (ci.f0 + (int64_t)jb * CV_B) < left) left = p.limit - (ci.f0 + (int64_t)jb * CV_B);
    const int valid = (int)(left < CV_B ? (left > 0 ? left : 0) : CV_B);
    // second half of the 2B frame: complex B/2 + i holds frames 2i, 2i+1 of the block (natural order after the DIT transform)
    if ((reinterpret_cast<uintptr_t>(out) & 15) == 0) {
#pragma unroll 4
        for (int i4 = t; i4 < CV_B / 4; i4 += CV_THREADS) {
            const int n = 4 * i4;
            const float2* c = z + cv_pad(CV_B / 2 + 2 * i4);
            float4 v = make_float4(c[0].x * scale, c[0].y * scale, c[1].x * scale, c[1].y * scale);
            if (n + 3 < valid) {
                float4* dst = reinterpret_cast<float4*>(out + n);
                if (p.accumulate) {
                    const float4 o = *dst;
                    v.x += o.x, v.y += o.y, v.z += o.z, v.w += o.w;
                }
                *dst = v;
            } else {
                const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
                for (int u = 0; u < 4; u++)
                    if (n + u < valid) out[n + u] = p.accumulate ? out[n + u] + vv[u] : vv[u];
            }
        }
    } else {
        for (int i = t; i < CV_B / 2; i += CV_THREADS) {
            const int n = 2 * i;
            const float2 c = z[cv_pad(CV_B / 2 + i)];
            if (n < valid) out[n] = p.accumulate ? out[n] + c.x * scale : c.x * scale;
            if (n + 1 < valid) out[n + 1] = p.accumulate ? out[n + 1] + c.y * scale : c.y * scale;
        }
    }
}

// ---- compacted second path of a mono-response convolver (ConvCmpInst, convolver.rs:378-400) -------------------------------------
// The stream is what the reference's convolvers[1] is fed: channel 1 of the chunk quanta that are not silent and have two channels.
// Stream frame s of the chunk's new frames (s - c0 = k) is chunk frame qmap[k / 128] * 128 + k % 128; the cursor c0 is a multiple of 128.
// Window frame w is stream frame (c0 / B - 1) * B + w: [last full block before c0 | partial block | new frames | zeros].  The grids are
// sized for the largest window (a chunk of nothing but two-channel quanta); CTAs past the chunk's own window exit.

// which chunk quanta convolvers[1] processes, and the stream cursor.  One warp per instance: 32 quanta per step, their positions in
// the list by a ballot and a population count.
__global__ void __launch_bounds__(128) k_conv_cmp_map(const ConvCmpInst* __restrict__ insts, int n_inst, ChunkInfo ci) {
    const int ii = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (ii >= n_inst) return;
    const int lane = threadIdx.x & 31;
    const ConvCmpInst& p = insts[ii];
    const int nq = ci.nf / 128;
    int n_proc = 0;
    for (int q0 = 0; q0 < nq; q0 += 32) {
        const int q = q0 + lane;
        bool fed = false;
        if (q < nq) {
            const int qi = meta_qi(ci, q * 128);
            fed = !buf_silent(p.in, p.in_ch, qi) && buf_count(p.in, p.in_ch, qi) >= 2;
        }
        const unsigned m = __ballot_sync(0xffffffffu, fed);
        if (fed) p.qmap[n_proc + __popc(m & ((1u << lane) - 1u))] = q;
        n_proc += __popc(m);
    }
    if (lane == 0) {
        const int64_t c0 = *p.cursor;
        p.wdesc[0] = c0;
        p.wdesc[1] = (int64_t)n_proc * 128;
        *p.cursor = c0 + (int64_t)n_proc * 128;
    }
}
// the stream window of the chunk.  grid: (window frames / 256, instances)
__global__ void __launch_bounds__(256) k_conv_cmp_gather(const ConvCmpInst* __restrict__ insts, ChunkInfo ci) {
    const ConvCmpInst& p = insts[blockIdx.y];
    const int64_t c0 = p.wdesc[0], n_new = p.wdesc[1];
    const int64_t w = (int64_t)blockIdx.x * 256 + threadIdx.x;
    const int64_t carried = CV_B + c0 % CV_B;  // last full block + partial block
    float v = 0.f;
    if (w < carried) {
        v = p.carry[w];
    } else if (w - carried < n_new) {
        const int k = (int)(w - carried);
        v = chan(p.in, 1, ci)[p.qmap[k >> 7] * 128 + (k & 127)];
    }
    p.win[w] = v;
}
// X_j of every stream block j the chunk's new frames reach (the partial one zero-padded), stored at the stream's absolute block index.
// grid: (window blocks, instances)
__global__ void __launch_bounds__(CV_THREADS, 3) k_conv_cmp_fft(const ConvCmpInst* __restrict__ insts, ChunkInfo ci) {
    extern __shared__ float2 z[];
    const ConvCmpInst& p = insts[blockIdx.y];
    const int64_t c0 = p.wdesc[0], c1 = c0 + p.wdesc[1];
    const int jb = blockIdx.x;
    const int64_t j = c0 / CV_B + jb;
    if (c1 == c0 || j * CV_B >= c1) return;
    const FftTw w = fft_tw_load(-1);
    const float2 lane_tw = cv_lane_tw();
    const float* win = p.win + (size_t)jb * CV_B;  // window block jb = stream block j - 1
    const int64_t left = c1 - j * CV_B;
    conv_load_half(z, 0, win, CV_B);
    conv_load_half(z, CV_B / 2, win + CV_B, (int)(left < CV_B ? left : CV_B));
    __syncthreads();
    fft_dif_smem(z, w);
    rfft_store(z, p.x.xring + (size_t)(j % p.x.xring_blocks) * CV_BINS, lane_tw);
}
// the last full stream block and the partial block for the next chunk's window.  grid: (2 B / 256, instances)
__global__ void __launch_bounds__(256) k_conv_cmp_carry(const ConvCmpInst* __restrict__ insts) {
    const ConvCmpInst& p = insts[blockIdx.y];
    const int64_t c0 = p.wdesc[0], c1 = c0 + p.wdesc[1];
    const int64_t first = (c1 / CV_B - c0 / CV_B) * CV_B;  // window frame of stream block c1 / B - 1
    const int i = blockIdx.x * 256 + threadIdx.x;
    p.carry[i] = p.win[first + i];
}
// Y_j = sum_i H_i X_{j-i} for the stream blocks of the window (conv_mac_bin of k_conv_mac).  grid: (B / 256 * groups of CV_J blocks, instances)
__global__ void __launch_bounds__(CV_MAC_THREADS, WAE_CV_MAC_MINB) k_conv_cmp_mac(const ConvCmpInst* __restrict__ insts, ChunkInfo ci) {
    const int64_t c0 = insts[blockIdx.y].wdesc[0], c1 = c0 + insts[blockIdx.y].wdesc[1];
    if (c1 == c0) return;
    const int64_t jfirst = c0 / CV_B, jlast = (c1 - 1) / CV_B;
    constexpr int TILES = CV_B / CV_MAC_THREADS;
    const int k = (blockIdx.x % TILES) * CV_MAC_THREADS + threadIdx.x;
    const int j0 = (blockIdx.x / TILES) * CV_J;  // first output block of this CTA, window-relative
    if (jfirst + j0 > jlast) return;
    const ConvPath path = insts[blockIdx.y].path;
    const ConvInput x = insts[blockIdx.y].x;
    float2 acc[CV_J];
#pragma unroll
    for (int jj = 0; jj < CV_J; jj++) acc[jj] = make_float2(0.f, 0.f);
    if (k == 0) conv_mac_bin<true>(path, x, k, jfirst + j0, jlast, acc);
    else conv_mac_bin<false>(path, x, k, jfirst + j0, jlast, acc);
#pragma unroll
    for (int jj = 0; jj < CV_J; jj++)
        if (jfirst + j0 + jj <= jlast) path.y[(size_t)(j0 + jj) * CV_BINS + k] = acc[jj];
}
// out_j = IFFT(Y_j)[B..2B) / 2B; the frames of the NEW stream frames go to channel 1 of the quanta they came from.  grid: (window blocks, instances)
__global__ void __launch_bounds__(CV_THREADS, 3) k_conv_cmp_ifft(const ConvCmpInst* __restrict__ insts, ChunkInfo ci) {
    extern __shared__ float2 z[];
    const ConvCmpInst& p = insts[blockIdx.y];
    const int64_t c0 = p.wdesc[0], c1 = c0 + p.wdesc[1];
    const int jb = blockIdx.x;
    const int64_t j = c0 / CV_B + jb;
    if (c1 == c0 || j * CV_B >= c1) return;
    const FftTw w = fft_tw_load(+1);
    const float2 lane_tw = cv_lane_tw();
    const float2* __restrict__ Y = p.path.y + (size_t)jb * CV_BINS;
    const int t = threadIdx.x;
#pragma unroll 4
    for (int q = t; q < CV_B; q += CV_THREADS) {
        float2 yk, ym;
        if (q == 0) {
            const float2 y0 = Y[0];
            yk = make_float2(y0.x, 0.f);
            ym = make_float2(y0.y, 0.f);
        } else {
            yk = Y[q];
            ym = Y[cv_mirror(q)];
        }
        z[cv_pad(q)] = irfft_merge(yk, ym, cv_bin_tw(lane_tw, q));
    }
    __syncthreads();
    fft_dit_smem(z, w);
    const float scale = 1.f / (float)(2 * CV_B);
    float* out = chan(p.path.out, p.path.out_channel, ci);
    const int64_t b0 = j * CV_B;
    const int lo = (int)((c0 > b0 ? c0 : b0) - b0), hi = (int)((c1 < b0 + CV_B ? c1 : b0 + CV_B) - b0);
    for (int i = lo + t; i < hi; i += CV_THREADS) {
        const float2 c = z[cv_pad(CV_B / 2 + (i >> 1))];
        const int k = (int)(b0 + i - c0);
        out[p.qmap[k >> 7] * 128 + (k & 127)] = ((i & 1) ? c.y : c.x) * scale;
    }
}

// IR segment spectra H_i (host uploads the scaled IR; one CTA per segment), position order like X.  grid: (S, ir channels)
__global__ void __launch_bounds__(CV_THREADS) k_conv_ir_fft(const float* __restrict__ ir, int64_t ir_len, int64_t ir_stride, float2* __restrict__ h,
                                                            int S) {
    extern __shared__ float2 z[];
    const FftTw w = fft_tw_load(-1);
    const float2 lane_tw = cv_lane_tw();
    const int seg = blockIdx.x, c = blockIdx.y;
    const float* src = ir + (size_t)c * ir_stride + (size_t)seg * CV_B;
    const int64_t left = ir_len - (int64_t)seg * CV_B;
    conv_load_half(z, 0, src, (int)(left < CV_B ? left : CV_B));  // segment in the first half, zeros in the second
    conv_load_half(z, CV_B / 2, nullptr, 0);
    __syncthreads();
    fft_dif_smem(z, w);
    rfft_store(z, h + ((size_t)c * (S + WAE_CONV_H_PAD) + WAE_CONV_H_PAD_LO + seg) * CV_BINS, lane_tw);  // (padding partitions stay zero)
}

// ---- wae_batch_bind_responses: the planner's normalisation, trimming and IR transform (plan_convolver), on the device --------------
// Three launches for all items of a bind: the power of the normalising items, the trimmed length of every (item, channel), the spectra.

// normalize_buffer (src/node/convolver.rs:16-53) with the planner's f32 operations in the planner's order, so that the scale is
// bit-equal to the one the host computes for an AudioBuffer of the same content: per channel a sequential sum of s * s, then the
// channels added in order.  One CTA per item; lane c of warp 0 runs channel c's dependent chain out of shared memory while the other
// warps load the next tile of every channel (coalesced, any alignment).  Items that do not normalise keep the scale 1.
constexpr int RB_TILE = 1024;
__global__ void __launch_bounds__(256) k_resp_power(RespBindItem* __restrict__ items) {
    __shared__ float buf[2][4][RB_TILE + 1];  // (+1: the four summing lanes read four different banks)
    __shared__ float part[4];
    RespBindItem& it = items[blockIdx.x];
    if (!it.normalize) return;
    const int ch = it.channels, t = threadIdx.x, warp = t >> 5;
    const int64_t len = it.len;
    const int64_t ntiles = (len + RB_TILE - 1) / RB_TILE;
    auto load = [&](int64_t tile, int b, int t0, int nt) {
        const int64_t f0 = tile * RB_TILE;
        const int cnt = (int)(len - f0 < RB_TILE ? len - f0 : RB_TILE);
        for (int k = t - t0; k < ch * RB_TILE; k += nt) {
            const int c = k / RB_TILE, i = k % RB_TILE;
            if (i < cnt) buf[b][c][i] = __ldcs(it.src + (int64_t)c * it.src_stride + f0 + i);
        }
    };
    load(0, 0, 0, blockDim.x);
    __syncthreads();
    float s = 0.f;
    for (int64_t tile = 0; tile < ntiles; tile++) {
        if (warp != 0) {
            if (tile + 1 < ntiles) load(tile + 1, (int)((tile + 1) & 1), 32, blockDim.x - 32);
        } else if (t < ch) {
            const float* __restrict__ x = buf[tile & 1][t];
            const int cnt = (int)(len - tile * RB_TILE < RB_TILE ? len - tile * RB_TILE : RB_TILE);
#pragma unroll 16
            for (int i = 0; i < cnt; i++) s = __fadd_rn(s, __fmul_rn(x[i], x[i]));
        }
        __syncthreads();
    }
    if (t < ch) part[t] = s;
    __syncthreads();
    if (t == 0) {
        float power = 0.f;
        for (int c = 0; c < ch; c++) power = __fadd_rn(power, part[c]);
        power = __fsqrt_rn(__fdiv_rn(power, (float)((uint64_t)ch * (uint64_t)len)));
        if (!isfinite(power) || power < 0.000125f) power = 0.000125f;
        float scale = __fdiv_rn(1.f, power);
        scale = __fmul_rn(scale, 0.00125f);
        scale = __fmul_rn(scale, __fdiv_rn(44100.f, it.sample_rate));
        if (ch == 4) scale = __fmul_rn(scale, 0.5f);
        it.scale = scale;
    }
}

// fft-convolver's init ignores the trailing samples below 1e-6: m = 1 + the last index whose scaled sample is not below it (the host's
// comparison, so NaN stops the trim), found as a max over the frames.  grid: (frame blocks, items, channels); it.m[c] is 0 on entry.
__global__ void __launch_bounds__(256) k_resp_trim(RespBindItem* __restrict__ items) {
    RespBindItem& it = items[blockIdx.y];
    const int c = blockIdx.z;
    if (c >= it.channels) return;
    const float* __restrict__ src = it.src + (int64_t)c * it.src_stride;
    const float scale = it.scale;
    int best = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < it.len; i += (int64_t)gridDim.x * blockDim.x)
        if (!(fabsf(__fmul_rn(__ldg(src + i), scale)) < 0.000001f)) best = (int)(i + 1);
    best = __reduce_max_sync(0xffffffffu, best);
    if ((threadIdx.x & 31) == 0 && best > 0) atomicMax(&it.m[c], best);
}

// The spectra of partition seg of channel c: the packed real FFT of x[i] * scale for i < m, zero after it — the values the planner
// uploads for an AudioBuffer, through k_conv_ir_fft's transform.  Every partition < S is written; the padding ones stay zero.
// grid: (partitions, channels, items)
__global__ void __launch_bounds__(CV_THREADS) k_resp_fft(const RespBindItem* __restrict__ items) {
    extern __shared__ float2 z[];
    const RespBindItem& it = items[blockIdx.z];
    const int seg = blockIdx.x, c = blockIdx.y;
    if (seg >= it.S || c >= it.channels) return;
    const FftTw w = fft_tw_load(-1);
    const float2 lane_tw = cv_lane_tw();
    const float* __restrict__ src = it.src + (int64_t)c * it.src_stride + (int64_t)seg * CV_B;
    const int64_t left = (int64_t)it.m[c] - (int64_t)seg * CV_B;
    const int valid = (int)(left < 0 ? 0 : left < CV_B ? left : CV_B);
    const float scale = it.scale;
    for (int i = threadIdx.x; i < CV_B / 2; i += CV_THREADS) {  // segment in the first half, zeros in the second
        const int n = 2 * i;
        z[cv_pad(i)] = make_float2(n < valid ? __fmul_rn(__ldg(src + n), scale) : 0.f, n + 1 < valid ? __fmul_rn(__ldg(src + n + 1), scale) : 0.f);
    }
    conv_load_half(z, CV_B / 2, nullptr, 0);
    __syncthreads();
    fft_dif_smem(z, w);
    rfft_store(z, it.h + ((size_t)c * (it.S + WAE_CONV_H_PAD) + WAE_CONV_H_PAD_LO + seg) * CV_BINS, lane_tw);
}

// ---- wae_batch_bind_curves: one CTA per declared WaveShaper curve ---------------------------------------------------------------
// Copies the caller's curve into the node's curve memory (128-bit stores; 128-bit loads where the source is 16 B aligned; the padding to
// a multiple of 4 floats is written as zeros), decides can_propagate_silence (waveshaper.rs:495-508) with the planner's f32 expression, and
// writes every record field that answer reaches.  Values are copied bit for bit (NaN payloads included).
__global__ void __launch_bounds__(256) k_bind_curves(const CurveBindItem* __restrict__ items) {
    __shared__ int keeps;
    const CurveBindItem it = items[blockIdx.x];
    const int n = it.n, n4 = (n + 3) >> 2;
    const bool aligned = (reinterpret_cast<uintptr_t>(it.src) & 15) == 0;
    for (int i = threadIdx.x; i < n4; i += blockDim.x) {
        float4 v;
        if (aligned && 4 * i + 4 <= n) {
            v = __ldcs(reinterpret_cast<const float4*>(it.src) + i);
        } else {
            const int k = 4 * i;
            v.x = __ldcs(it.src + k);
            v.y = k + 1 < n ? __ldcs(it.src + k + 1) : 0.f;
            v.z = k + 2 < n ? __ldcs(it.src + k + 2) : 0.f;
            v.w = k + 3 < n ? __ldcs(it.src + k + 3) : 0.f;
        }
        reinterpret_cast<float4*>(it.dst)[i] = v;
    }
    if (threadIdx.x == 0) {
        const float* c = it.src;
        keeps = n % 2 == 1 ? fabsf(c[n / 2]) < 1e-9f : fabsf(__fdiv_rn(__fadd_rn(c[n / 2 - 1], c[n / 2]), 2.f)) < 1e-9f;
    }
    __syncthreads();
    for (int k = threadIdx.x; k < it.n_patches; k += blockDim.x) {
        const CurvePatch p = it.patches[k];
        *p.dst = keeps ? p.keeps : p.other;
    }
}

// ---- wae_batch_bind_periodic_waves: the wavetables of declared custom oscillators -----------------------------------------------
// k_bind_waves: grid (tiles of WAVE_TILE table entries, items).  generate_wavetable (periodic_wave.rs:164-190) as
// wae_periodic_wave_table evaluates it: every thread owns one table entry and sums the harmonics j = 1 .. n-1 in the host's order with
// the host's f32 operations (the build has no FMA contraction); the CTA stages the coefficients through shared memory, so each one is
// a broadcast read.  sin / cos of the f32 phase are the f64 values rounded to f32, which agree with the host's sinf / cosf on nearly
// every argument (DESIGN.md §2).
constexpr int WAVE_TILE = 256;
__global__ void __launch_bounds__(WAVE_TILE) k_bind_waves(const WaveBindItem* __restrict__ items) {
    __shared__ float s_re[WAVE_TILE], s_im[WAVE_TILE];
    const WaveBindItem it = items[blockIdx.y];
    if ((int)blockIdx.x * WAVE_TILE >= it.len) return;  // (the whole CTA: shorter tables than the launch's longest)
    const int i = blockIdx.x * WAVE_TILE + threadIdx.x;
    const float pi_2 = 2.f * 3.14159265358979323846f;
    const float phase = __fdiv_rn(__fmul_rn(pi_2, (float)i), (float)it.len);
    float sample = 0.f;
    for (int c0 = 1; c0 < it.n; c0 += WAVE_TILE) {
        const int cn = min(WAVE_TILE, it.n - c0);
        __syncthreads();  // (the previous chunk is read)
        if (threadIdx.x < cn) {
            s_re[threadIdx.x] = it.re ? __ldg(it.re + c0 + threadIdx.x) : 0.f;
            s_im[threadIdx.x] = it.im ? __ldg(it.im + c0 + threadIdx.x) : 0.f;
        }
        __syncthreads();
        for (int k = 0; k < cn; k++) {
            const float rad = __fmul_rn(phase, (float)(c0 + k));
            double sd, cd;
            sincos((double)rad, &sd, &cd);
            sample = __fadd_rn(sample, __fadd_rn(__fmul_rn(s_re[k], (float)cd), __fmul_rn(s_im[k], (float)sd)));
        }
    }
    if (i < it.len) it.dst[i] = sample;
}

// k_wave_normalize: one CTA per item that normalises (periodic_wave.rs:192-209): the largest |x| (fmaxf ignores NaN as the host's `>`
// does; max is order-independent, so the result is the host's), then x *= 1 / max when max > 0
__global__ void __launch_bounds__(1024) k_wave_normalize(const WaveBindItem* __restrict__ items) {
    __shared__ float s_max[32];
    const WaveBindItem it = items[blockIdx.x];
    if (!it.normalize) return;
    float mx = 0.f;
    for (int i = threadIdx.x; i < it.len; i += blockDim.x) mx = fmaxf(mx, fabsf(it.dst[i]));
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = mx;
    __syncthreads();
    if (threadIdx.x < 32) {
        mx = threadIdx.x < (blockDim.x >> 5) ? s_max[threadIdx.x] : 0.f;
        for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        if (threadIdx.x == 0) s_max[0] = mx;
    }
    __syncthreads();
    mx = s_max[0];
    if (!(mx > 0.f)) return;
    const float norm = __fdiv_rn(1.f, mx);
    for (int i = threadIdx.x; i < it.len; i += blockDim.x) it.dst[i] = __fmul_rn(it.dst[i], norm);
}

// ---- wae_batch_bind_iir_coefficients: one CTA per declared IIRFilterNode -----------------------------------------------------------
// The shorter list padded with zeros to the longer one (and an order <= 2 filter to 3 on the chain path), every coefficient divided by
// feedback[0] (iir_filter.rs:282-309): the IEEE f64 quotients Planner::lower_iir computes, so that bound coefficients are bit-equal to a
// node constructed with them.  feedback[0] == 0, which the constructor refuses, writes zeros (the filter outputs silence).  Then every
// patch entry of the item: the IirInst coefficients of each render segment, or the chain's biquad and its scan constants.
__global__ void __launch_bounds__(32) k_bind_iir(const IirBindItem* __restrict__ items) {
    __shared__ double s_b[20], s_a[20];
    const IirBindItem it = items[blockIdx.x];
    const double a0 = it.fb[0];
    for (int i = threadIdx.x; i < 20; i += blockDim.x) {
        const double x = i < it.nff ? it.ff[i] : 0., y = i < it.nfb ? it.fb[i] : 0.;
        s_b[i] = a0 == 0. ? 0. : __ddiv_rn(x, a0);
        s_a[i] = a0 == 0. ? 0. : __ddiv_rn(y, a0);
    }
    __syncthreads();
    const int n = max(it.nff, it.nfb);
    for (int k = threadIdx.x; k < it.n_patches; k += blockDim.x) {
        const IirPatch p = it.patches[k];
        if (p.a) {
            for (int i = 0; i < n; i++) {
                p.b[i] = s_b[i];
                p.a[i] = s_a[i];
            }
        } else {
            p.b[0] = s_b[0]; p.b[1] = s_b[1]; p.b[2] = s_b[2]; p.b[3] = s_a[1]; p.b[4] = s_a[2];
            if (p.scan) make_scan_coef(s_b[1], s_b[2], s_a[1], s_a[2], *static_cast<ScanCoef*>(p.scan));
        }
    }
}

// ---- wae_batch_bind_value_curves: tiles of VC_TILE values (x) of each item (y), both grid-stride --------------------------------------
// The values are moved as 32-bit words, so they land bit for bit (NaN payloads included); nothing but k_param* reads them, so there is
// nothing to derive.  128-bit accesses where source and destination are both 16 B aligned (a tile starts a multiple of 16 B into both).
constexpr int VC_TILE = 1024;
__global__ void __launch_bounds__(256) k_bind_value_curves(const ValueCurveBindItem* __restrict__ items, int n_items) {
    for (int i = blockIdx.y; i < n_items; i += gridDim.y) {
        const ValueCurveBindItem it = items[i];
        for (int64_t t0 = (int64_t)blockIdx.x * VC_TILE; t0 < it.n; t0 += (int64_t)gridDim.x * VC_TILE) {
            const int m = (int)min((int64_t)VC_TILE, (int64_t)it.n - t0);
            const unsigned* src = reinterpret_cast<const unsigned*>(it.src) + t0;
            unsigned* dst = reinterpret_cast<unsigned*>(it.dst) + t0;
            int done = 0;
            if (((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0) {
                const int m4 = m >> 2;
                for (int k = threadIdx.x; k < m4; k += blockDim.x)
                    reinterpret_cast<uint4*>(dst)[k] = __ldcs(reinterpret_cast<const uint4*>(src) + k);
                done = 4 * m4;
            }
            for (int k = done + threadIdx.x; k < m; k += blockDim.x) dst[k] = __ldcs(src + k);
        }
    }
}

// ---- wae_batch_bind_schedules: one thread per item -----------------------------------------------------------------------------------
// The times are clamped to their windows, then every record field they reach is derived with the planner's functions (wae_kernels.h):
// f64 without transcendentals or contraction, so each field gets the bits a host-built plan of those times holds.  The frame walks are
// sequential (the slow track's start is sticky within almost_equal) and run once per bind.  A bound offset / duration of a buffer source
// is written raw: the render kernels derive the playhead from them on every run.
DEVI double sched_clamp(double v, double lo, double hi) { return v != v ? lo : (v < lo ? lo : (v > hi ? hi : v)); }
__global__ void __launch_bounds__(128) k_bind_schedules(const SchedBindItem* __restrict__ items, int n_items) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_items) return;
    const SchedBindItem it = items[i];
    const bool bind_stop = it.binds & SCHED_BIND_STOP, bind_offset = it.binds & SCHED_BIND_OFFSET, bind_duration = it.binds & SCHED_BIND_DURATION;
    int col = 0;  // the row holds only what was declared
    const double start = sched_clamp(it.times[col++], it.lo[0], it.hi[0]);
    const double bound_stop = bind_stop ? sched_clamp(it.times[col++], it.lo[1], it.hi[1]) : 0.;
    const double bound_offset = bind_offset ? sched_clamp(it.times[col++], it.lo[2], it.hi[2]) : 0.;
    const double bound_duration = bind_duration ? sched_clamp(it.times[col], it.lo[3], it.hi[3]) : 0.;
    for (int k = 0; k < it.n_patches; k++) {
        const SchedPatch p = it.patches[k];
        const double stop = bind_stop ? bound_stop : p.stop_time;
        const SchedClock clock(p.sample_rate);
        char* d = static_cast<char*>(p.dst);
        switch (p.kind) {
            case SCHED_OSC:
            case SCHED_OSC_AR:
            case SCHED_META_OSC: {
                // the phase increment is the record's own: planned, or re-derived by the oscillator's pitch bound from device memory
                // (PATCH_OSC), which reads the start written to start_out — either bind sees the other's current value
                OscInst* o = p.kind == SCHED_META_OSC ? nullptr
                             : p.kind == SCHED_OSC_AR ? &reinterpret_cast<OscArInst*>(d)->base
                                                      : reinterpret_cast<OscInst*>(d);
                const OscStart s = osc_start(clock, start, o ? o->incr : 0., o && o->outside_nyquist != 0);
                const int64_t n_stop = osc_stop_frame(clock, stop);
                if (!o) {
                    reinterpret_cast<MetaInst*>(d)->n_first = s.n_first;
                    reinterpret_cast<MetaInst*>(d)->n_stop = n_stop;
                    break;
                }
                o->n_first = s.n_first;
                o->n_stop = n_stop;
                o->phase0 = s.phase0;
                if (p.kind == SCHED_OSC_AR) reinterpret_cast<OscArInst*>(d)->start_ratio = s.start_ratio;
                if (p.start_out) *p.start_out = start;
                break;
            }
            case SCHED_CONST:
            case SCHED_META_CONST: {
                const int64_t n_first = clock.first_frame_at_or_after(start);
                const int64_t n_stop = stop < 1e300 ? clock.first_frame_at_or_after(stop) : SCHED_NEVER;
                if (p.kind == SCHED_META_CONST) {
                    reinterpret_cast<MetaInst*>(d)->n_first = n_first;
                    reinterpret_cast<MetaInst*>(d)->n_stop = n_stop;
                } else {
                    reinterpret_cast<ConstInst*>(d)->n_first = n_first;
                    reinterpret_cast<ConstInst*>(d)->n_stop = n_stop;
                }
                break;
            }
            case SCHED_ABSN_BOUND: {
                AbsnBoundInst* r = reinterpret_cast<AbsnBoundInst*>(d);
                const double offset = bind_offset ? bound_offset : p.offset;
                const int64_t q = absn_start_quantum(clock, start);
                const bool aligned = start <= clock.block_time(q) && offset == 0.;
                const AbsnStart st = absn_start(clock, start, stop);
                r->s.n_first = st.n_first;
                r->s.n_stop = st.n_stop;
                r->start_delta = st.t_first - st.start;
                r->n_start = q * 128;
                r->fast_end = absn_fast_end(clock, p.lq, q * 128, p.duration);
                r->fast_ok = aligned && p.flag && stop > 1e300;  // (flag is 0 for a declared duration: it is finite)
                if (bind_offset) r->offset = bound_offset;
                if (bind_duration) r->s.duration = bound_duration;
                break;
            }
            case SCHED_ABSN_SERIAL: {
                AbsnSerialInst* r = reinterpret_cast<AbsnSerialInst*>(d);
                r->start_time = start;
                r->stop_time = stop;
                if (bind_offset) r->offset = bound_offset;
                if (bind_duration) r->duration = bound_duration;
                break;
            }
        }
    }
}

// ---- wae_batch_bind_loops: one thread per item -----------------------------------------------------------------------------------------
// The loop points are clamped to their windows, then clamp_loop_boundaries and the actual-loop-points rule are applied with the planner's
// function (absn_loop_points).  A bound slow-track record takes the actual loop points; its table is derived by k_absn_loop_schedule,
// launched right after this kernel.
__global__ void __launch_bounds__(128) k_bind_loops(const LoopBindItem* __restrict__ items, int n_items) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_items) return;
    const LoopBindItem it = items[i];
    const double ls = sched_clamp(it.points[0], it.lo[0], it.hi[0]);
    const double le = sched_clamp(it.points[1], it.lo[1], it.hi[1]);
    for (int k = 0; k < it.n_patches; k++) {
        const LoopPatch p = it.patches[k];
        const AbsnLoopPoints lp = absn_loop_points(ls, le, p.buffer_duration);
        if (p.kind == LOOP_BOUND) {
            AbsnBoundInst* r = static_cast<AbsnBoundInst*>(p.dst);
            r->s.loop_start = lp.actual_start;
            r->s.loop_end = lp.actual_end;
        } else {
            AbsnSerialInst* r = static_cast<AbsnSerialInst*>(p.dst);
            r->loop_start = lp.start;
            r->loop_end = lp.end;
        }
    }
}

// ---- The playhead tables of looping bound slow-track records: one thread per record.  step / offset0 from the record's (bound or
// planned) rate, detune, start, offset and duration exactly as absn_bound_tiles derives them, then the planner's walk
// (absn_loop_segments) into the record's table.  A walk that needs more than the planned capacity is a planner defect: the table keeps
// its first `cap` segments and *overflow is set, which wae_batch_sync reports.
__global__ void __launch_bounds__(128) k_absn_loop_schedule(const LoopWalk* __restrict__ walks, int n, int* overflow) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const LoopWalk w = walks[i];
    AbsnBoundInst& r = *w.rec;
    const AbsnSlowInst& o = r.s;
    const double computed_rate = (double)r.rate * exp2((double)r.detune / 1200.);
    const AbsnSlowDerived d = absn_slow_derive(r.dt, computed_rate, r.offset, r.start_delta, o.buffer_duration, o.duration, true, o.loop_end,
                                               o.n_first, o.n_stop);
    const int64_t n_end = o.n_stop < w.lq ? o.n_stop : w.lq;
    int32_t k = absn_loop_segments(o.loop_start, o.loop_end, d.step, o.n_first, n_end, d.offset0, const_cast<int64_t*>(o.seg_n),
                                   const_cast<double*>(o.seg_bt), w.cap);
    if (k < 0) {
        atomicExch(overflow, 1);
        k = w.cap;
    }
    r.s.n_seg = k;
}

// wae_batch_bind_output: every record field that points into the rendered PCM now points into `base` (the caller's memory or the batch's
// own buffer), at the same offset
__global__ void __launch_bounds__(128) k_bind_output(const OutPatch* __restrict__ entries, int n, float* base) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const OutPatch e = entries[i];
    *e.dst = base + e.off;
}

// wae_batch_bind_sources, inputs declared by reference: every record that plays one now reads the caller's memory (pointer and channel
// stride); no audio moves
__global__ void __launch_bounds__(128) k_bind_source_refs(const SrcRefBindItem* __restrict__ items, int n, const SrcRefPatch* __restrict__ entries) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const SrcRefBindItem it = items[i];
    const SrcRefPatch e = entries[it.entry];
    *e.buf = it.pcm;
    *e.stride = it.stride;
}

// Host emulation of the transforms above with the SAME butterfly, index and twiddle code (tests/test_conv_fft_host.py pins them against
// numpy on a machine without a GPU).  mode 0: complex forward, natural -> position order; 1: complex inverse, position -> natural order
// (unnormalised); 2: 2B reals -> B packed bins in position order; 3: B packed bins -> 2B reals (scaled by 1 / 2B).  data: 2B floats in place.
static void host_twiddles() {
    if (h_tw[0].x == 1.f) return;
    for (int k = 0; k < CV_B; k++) {
        const double a = -2.0 * 3.14159265358979323846 * (double)k / (2.0 * CV_B);
        h_tw[k] = make_float2((float)std::cos(a), (float)std::sin(a));
    }
}
static int brev8(int r) {
    int o = 0;
    for (int b = 0; b < 8; b++) o |= ((r >> b) & 1) << (7 - b);
    return o;
}
template <int LOG_Q, bool DIT>
static void host_pass8(float2* s, int sign) {
    for (int t = 0; t < CV_THREADS; t++) {
        const FftTw w = fft_tw_of(h_tw, t, sign);
        for (int it = 0; it < CV_B / 8 / CV_THREADS; it++) fft_pass8_one<LOG_Q, DIT>(s, t, it, w, sign);
    }
}
template <bool DIT>
static void host_pass16(float2* s, int sign) {
    for (int t = 0; t < CV_THREADS; t++)
        for (int it = 0; it < CV_B / 16 / CV_THREADS; it++) fft_pass16_one<DIT>(s, t, it, sign);
}
static void host_fft(float2* s, bool inverse) {
    if (!inverse) {
        host_pass8<10, false>(s, -1), host_pass8<7, false>(s, -1), host_pass8<4, false>(s, -1), host_pass16<false>(s, -1);
    } else {
        host_pass16<true>(s, +1), host_pass8<4, true>(s, +1), host_pass8<7, true>(s, +1), host_pass8<10, true>(s, +1);
    }
}
void conv_fft_selftest(float* data, int mode) {
    host_twiddles();
    std::vector<float2> s(CV_SMEM_ELEMS), x(CV_B);
    float2* io = reinterpret_cast<float2*>(data);
    auto bin_tw = [](int p) { return cmul(h_tw[cv_brev(p & 31)], h_tw[brev8(p >> 5)]); };
    if (mode == 0 || mode == 1) {
        for (int i = 0; i < CV_B; i++) s[cv_pad(i)] = io[i];
        host_fft(s.data(), mode == 1);
        for (int i = 0; i < CV_B; i++) io[i] = s[cv_pad(i)];
    } else if (mode == 2) {
        for (int i = 0; i < CV_B; i++) s[cv_pad(i)] = io[i];  // (even, odd) packing is the memory layout of 2B reals
        host_fft(s.data(), false);
        for (int p = 0; p < CV_B; p++) {
            if (p == 0) io[0] = make_float2(s[0].x + s[0].y, s[0].x - s[0].y);
            else x[p] = rfft_split(s[cv_pad(p)], s[cv_pad(cv_mirror(p))], bin_tw(p));
        }
        for (int p = 1; p < CV_B; p++) io[p] = x[p];
    } else {
        for (int p = 0; p < CV_B; p++) {
            const float2 yk = p == 0 ? make_float2(io[0].x, 0.f) : io[p];
            const float2 ym = p == 0 ? make_float2(io[0].y, 0.f) : io[cv_mirror(p)];
            s[cv_pad(p)] = irfft_merge(yk, ym, bin_tw(p));
        }
        host_fft(s.data(), true);
        const float scale = 1.f / (float)(2 * CV_B);
        for (int i = 0; i < CV_B; i++) io[i] = make_float2(s[cv_pad(i)].x * scale, s[cv_pad(i)].y * scale);
    }
}
void upload_twiddles() {
    host_twiddles();
    float2 row[CV_ROWS];
    for (int r = 0; r < CV_ROWS; r++) row[r] = h_tw[brev8(r)];
    cudaMemcpyToSymbol(c_tw, h_tw, sizeof(float2) * CV_B);
    cudaMemcpyToSymbol(c_rowtw, row, sizeof(row));
}

// ---------------------------------------------------------------------------------------------------------
// Analyser frequency read-out — Analyser::compute_fft + get_float_frequency_data (src/analysis.rs:278-369): the most
// recent fftSize frames of the ring x Blackman window (alpha 0.16, :13-24) -> real FFT -> |X[k]| / N -> exponential
// smoothing with the previous read-out -> 20 log10.  One CTA per analyser, radix-2 complex FFT of fftSize/2 points in
// shared memory (fftSize up to 32768 -> 128 KB), the real-FFT split done on the fly.
// ---------------------------------------------------------------------------------------------------------
// Blackman window value of sample idx (analysis.rs:13-24)
__device__ __forceinline__ float analyser_blackman(int idx, int fft_size) {
    const float PI32 = 3.14159265358979323846f;
    return 0.42f - 0.5f * cosf(2.f * PI32 * (float)idx / (float)fft_size) + 0.08f * cosf(4.f * PI32 * (float)idx / (float)fft_size);
}
// Windowed samples 2i, 2i+1 -> bit-reversed slot of the complex FFT of fftSize / 2 points (`bits` = log2 of that)
__device__ __forceinline__ void analyser_store_pair(float2* zf, int i, int bits, float v0, float v1) {
    const int r = (int)(__brev((unsigned)i) >> (32 - bits));
    zf[bits == 0 ? 0 : r] = make_float2(v0, v1);
}
// In-place radix-2 transform of the n = fftSize / 2 points in zf (all threads of the CTA; the caller synchronises before)
__device__ __forceinline__ void analyser_fft_passes(float2* zf, int n) {
    const int t = threadIdx.x;
    for (int len = 2; len <= n; len <<= 1) {
        const int half = len >> 1;
        for (int b = t; b < n / 2; b += blockDim.x) {
            int grp = b / half, j = b % half;
            int i0 = grp * len + j, i1 = i0 + half;
            float sn, cs;
            sincospif(-2.f * (float)j / (float)len, &sn, &cs);
            float2 u = zf[i0], x = zf[i1];
            float2 v = make_float2(x.x * cs - x.y * sn, x.x * sn + x.y * cs);
            zf[i0] = make_float2(u.x + v.x, u.y + v.y);
            zf[i1] = make_float2(u.x - v.x, u.y - v.y);
        }
        __syncthreads();
    }
}
// |X[k]| / N of the real input from the transformed points (bins 0 .. N/2-1: the Nyquist bin is ignored, analysis.rs:303-333)
__device__ __forceinline__ float analyser_bin_magnitude(const float2* zf, int k, int n, int fft_size) {
    float2 X;
    if (k == 0) {
        X = make_float2(zf[0].x + zf[0].y, 0.f);
    } else {
        float2 zk = zf[k], zc = make_float2(zf[n - k].x, -zf[n - k].y);
        float2 e = make_float2(0.5f * (zk.x + zc.x), 0.5f * (zk.y + zc.y));
        float2 d = make_float2(zk.x - zc.x, zk.y - zc.y);
        float2 o = make_float2(0.5f * d.y, -0.5f * d.x);
        float sn, cs;
        sincospif(-2.f * (float)k / (float)fft_size, &sn, &cs);
        X = make_float2(e.x + (o.x * cs - o.y * sn), e.y + (o.x * sn + o.y * cs));
    }
    return hypotf(X.x, X.y) * (1.f / (float)fft_size);
}
// get_float_frequency_data's smoothing with the previous read-out (analysis.rs:335-345): the new state (its dB: 20 log10)
__device__ __forceinline__ float analyser_smooth(float smoothing, float last, float mag) {
    float value = smoothing * last + (1.f - smoothing) * mag;
    if (!isfinite(value)) value = 0.f;
    return value;
}

__global__ void __launch_bounds__(256) k_analyser_fft(const float* __restrict__ ring, uint32_t write_index, int fft_size, float smoothing,
                                                      float* __restrict__ last_fft, float* __restrict__ out_db) {
    extern __shared__ float2 zf[];
    const int RING = 32768 + 128;
    const int n = fft_size / 2;
    const int t = threadIdx.x;
    int bits = 0;
    while ((1 << bits) < n) bits++;
    for (int i = t; i < n; i += blockDim.x) {
        float v[2];
        for (int h = 0; h < 2; h++) {
            int idx = 2 * i + h;
            float x = ring[(RING + write_index - fft_size + idx) % RING];
            v[h] = x * analyser_blackman(idx, fft_size);
        }
        analyser_store_pair(zf, i, bits, v[0], v[1]);
    }
    __syncthreads();
    analyser_fft_passes(zf, n);
    for (int k = t; k < n; k += blockDim.x) {
        float mag = analyser_bin_magnitude(zf, k, n, fft_size);
        float value = analyser_smooth(smoothing, last_fft[k], mag);
        last_fft[k] = value;
        out_db[k] = 20.f * log10f(value);
    }
}

// ---------------------------------------------------------------------------------------------------------
// Declared analyser read-outs (wae_analyser_set_readouts), taken in the analyser's stage of the chunk (f0, f0 + nf] that holds their
// frame F, before k_analyser writes the chunk into the ring: a chunk longer than the ring overwrites slots an earlier read-out of the
// same chunk still needs.  Sample idx of the window is frame F - fftSize + idx: zero before the render, the ring before f0, the
// analyser's own down-mix of the input from f0 on.
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float readout_sample(const ReadoutInst& r, int idx, const ChunkInfo& ci) {
    const int RING = 32768 + 128;
    const int64_t m = r.frame - r.fft_size + idx;
    if (m < 0) return 0.f;
    if (m < ci.f0) return r.ring[m % RING];
    return analyser_mono(r.in, r.ch, (int)(m - ci.f0), ci);
}

// One CTA per read-out of the chunk: the window, Blackman, the transform of k_analyser_fft, linear magnitudes into the row
// (k_readout_smooth turns them into dB)
__global__ void __launch_bounds__(256) k_readout_fft(const ReadoutInst* __restrict__ insts, ChunkInfo ci) {
    extern __shared__ float2 zf[];
    const ReadoutInst r = insts[blockIdx.x];
    const int n = r.fft_size / 2;
    int bits = 0;
    while ((1 << bits) < n) bits++;
    for (int i = threadIdx.x; i < n; i += blockDim.x)
        analyser_store_pair(zf, i, bits, readout_sample(r, 2 * i, ci) * analyser_blackman(2 * i, r.fft_size),
                            readout_sample(r, 2 * i + 1, ci) * analyser_blackman(2 * i + 1, r.fft_size));
    __syncthreads();
    analyser_fft_passes(zf, n);
    for (int k = threadIdx.x; k < n; k += blockDim.x) r.row[k] = analyser_bin_magnitude(zf, k, n, r.fft_size);
}

// Analyser::get_byte_* (analysis.rs:266-276, 371-401): clamp(v, 0, 255) as u8 in f32 arithmetic; Rust's `as u8` maps NaN to 0
__device__ __forceinline__ uint8_t readout_byte(float v) {
    return (uint8_t)__float2uint_rz(!(v > 0.f) ? 0.f : fminf(v, 255.f));
}

// Time-domain read-outs: the window itself (get_float_time_domain_data, analysis.rs:261-264); its bytes 128 (1 + x) (:266-276)
__global__ void __launch_bounds__(256) k_readout_time(const ReadoutInst* __restrict__ insts, ChunkInfo ci) {
    const ReadoutInst r = insts[blockIdx.x];
    for (int i = blockIdx.y * blockDim.x + threadIdx.x; i < r.fft_size; i += gridDim.y * blockDim.x) {
        const float x = readout_sample(r, i, ci);
        r.row[i] = x;
        if (r.bytes) r.bytes[i] = readout_byte(__fmul_rn(128.f, __fadd_rn(1.f, x)));
    }
}

// One thread per (analyser, bin): the analyser's frequency read-outs of the chunk in time order, smoothed with the state the previous
// one left (analysis.rs:335-345); a read-out on the quantum of the one before repeats its row without smoothing again (last_fft_time,
// :347-361).  The state crosses chunks in last_fft; the last read-out's dB row is the analyser's post-render read-out.
__global__ void __launch_bounds__(256) k_readout_smooth(const ReadoutSmoothInst* __restrict__ insts, ChunkInfo ci) {
    const ReadoutSmoothInst s = insts[blockIdx.x];
    const int bin = blockIdx.y * blockDim.x + threadIdx.x;
    if (bin >= s.bins) return;
    // first read-out of the chunk: F > f0, or F >= 0 in the first chunk
    const int64_t lo = ci.f0 == 0 ? -1 : ci.f0, hi = ci.f0 + ci.nf;
    int a = 0, b = s.n;
    while (a < b) {
        const int m = (a + b) >> 1;
        if (s.frames[m] > lo) b = m;
        else a = m + 1;
    }
    if (a >= s.n || s.frames[a] > hi) return;
    float last = s.last_fft[bin], db = 0.f;
    // byte rows: 255 / (max - min) * (dB - min) (analysis.rs:390-398), rounded as numpy's f32 statement of it
    const float scale = s.bytes ? __fdiv_rn(255.f, __fsub_rn(s.max_db, s.min_db)) : 0.f;
    for (int k = a; k < s.n && s.frames[k] <= hi; k++) {
        float* row = s.rows + (size_t)k * s.bins;
        if (k > 0 && s.frames[k] == s.frames[k - 1]) db = row[(int64_t)-s.bins + bin];
        else db = 20.f * log10f(last = analyser_smooth(s.smoothing, last, row[bin]));
        row[bin] = db;
        if (s.bytes) s.bytes[(size_t)k * s.bins + bin] = readout_byte(__fmul_rn(scale, __fsub_rn(db, s.min_db)));
        if (k == s.n - 1) s.db[bin] = db;
    }
    s.last_fft[bin] = last;
}

// AudioBuffer::resample (src/buffer.rs:311-363): linear interpolation that keeps the first and the last frame
__global__ void __launch_bounds__(256) k_resample_linear(const float* __restrict__ in, int64_t len, float* __restrict__ out, int64_t target_len) {
    int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= target_len) return;
    double position = (double)i / (double)(target_len - 1);
    double playhead = position * (double)(len - 1);
    double fl = floor(playhead);
    int64_t prev = (int64_t)fl;
    int64_t next = prev + 1 < len - 1 ? prev + 1 : len - 1;
    float k = (float)(playhead - fl);
    out[i] = __fadd_rn(__fmul_rn(1.f - k, in[prev]), __fmul_rn(k, in[next]));
}

// wae_batch_bind_sources: copies caller device audio into device-input slots of the source slabs (HBM-bound).  blockIdx.y walks the
// items, blockIdx.z is the channel, x the slot's 16-byte vectors.  The whole slot is written, its zero padding [len, stride) included
// (the chain kernel's LDG.128 / cp.async.bulk reads run into it), with 128-bit stores; the loads are 128-bit where the source channel
// is 16 B aligned and scalar otherwise (torch views with odd lengths or storage offsets).
__global__ void __launch_bounds__(256) k_bind_sources(const BindItem* __restrict__ items, int n) {
    const int c = blockIdx.z;
    for (int i = blockIdx.y; i < n; i += gridDim.y) {
        const BindItem it = items[i];
        if (c >= it.channels) continue;
        const float* __restrict__ src = it.src + (int64_t)c * it.src_stride;
        float4* __restrict__ dst = reinterpret_cast<float4*>(it.dst + (int64_t)c * it.stride);
        const int64_t nvec = it.stride >> 2, full = it.len >> 2;
        const bool vec = (reinterpret_cast<uintptr_t>(src) & 15) == 0;
        for (int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; v < nvec; v += (int64_t)gridDim.x * blockDim.x) {
            float4 x;
            if (vec && v < full) {
                x = __ldcs(reinterpret_cast<const float4*>(src) + v);
            } else {
                const int64_t f = v * 4;
                x.x = f < it.len ? __ldcs(src + f) : 0.f;
                x.y = f + 1 < it.len ? __ldcs(src + f + 1) : 0.f;
                x.z = f + 2 < it.len ? __ldcs(src + f + 2) : 0.f;
                x.w = f + 3 < it.len ? __ldcs(src + f + 3) : 0.f;
            }
            dst[v] = x;
        }
    }
}

// wae_batch_bind_params, step 1: each item's float from the caller's device memory into its value slot, clamped to the declared range
// as AudioParam::set_value clamps (param.rs:407-413).  A non-finite value takes the param's default value, the reference's rule for a
// NaN computed value (param.rs:755-795): a device bind cannot panic as the reference's set_value does.
__global__ void __launch_bounds__(256) k_bind_params(const ParamBindItem* __restrict__ items, int n, const ParamSlotInfo* __restrict__ info,
                                                     float* __restrict__ values) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const ParamBindItem it = items[i];
    const ParamSlotInfo si = info[it.slot];
    float v = *it.src;
    if (!isfinite(v)) v = si.def;
    else v = fminf(fmaxf(v, si.lo), si.hi);
    values[it.slot] = v;
}

// step 2: every patch entry of the batch re-derived from the value slots and its planned constants, with the planner's own formulas
DEVI float patch_op(const ParamPatch& p, int i, const float* values) { return p.slot[i] >= 0 ? values[p.slot[i]] : p.val[i]; }
DEVI float patch_gain_product(const ParamPatch& p, const float* values) {
    float g = 1.f;
    for (int i = 0; i < p.n && i < PATCH_OPS; i++) {
        float f = patch_op(p, i, values);
        if (p.slot[i] >= 0) {  // gain.rs:153-169, as Planner::lower_gain applies it to a constant gain
            if (fabsf(f) <= 1e-6f) f = 0.f;
            else if (fabsf(1.f - f) <= 1e-6f) f = 1.f;
        }
        g *= f;
    }
    return g;
}
__global__ void __launch_bounds__(64) k_derive_params(const ParamPatch* __restrict__ patches, int n, const float* __restrict__ values) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const ParamPatch& p = patches[i];
    switch (p.kind) {
        case PATCH_GAIN: *static_cast<float*>(p.dst) = patch_gain_product(p, values); break;
        case PATCH_META: *static_cast<int32_t*>(p.dst) = patch_gain_product(p, values) == 0.f ? META_CONST : META_COPY; break;
        case PATCH_BIQUAD: {
            const float q = patch_op(p, 0, values), detune = patch_op(p, 1, values), freq = patch_op(p, 2, values), gain = patch_op(p, 3, values);
            const float computed = detune != 0.f ? freq * exp2f(detune / 1200.f) : freq;  // get_computed_freq, biquad_filter.rs:393-399
            const BqC c = bq_coefs(p.n, (double)p.sample_rate, (double)computed, (double)gain, (double)q);
            double* d = static_cast<double*>(p.dst);
            d[0] = c.b0; d[1] = c.b1; d[2] = c.b2; d[3] = c.a1; d[4] = c.a2;
            if (p.dst2) make_scan_coef(c.b1, c.b2, c.a1, c.a2, *static_cast<ScanCoef*>(p.dst2));
            break;
        }
        case PATCH_SPAN: {  // stereo_panner.rs:247-249,274-276 and get_stereo_gains (:74-79), as k_stereo_panner computes them
            const float pan = patch_op(p, 0, values), PI32 = 3.14159265358979323846f;
            const float x = p.n == 1 ? (pan + 1.f) * 0.5f : (pan <= 0.f ? pan + 1.f : pan);
            *static_cast<float*>(p.dst) = pan;
            *static_cast<float2*>(p.dst2) = make_float2(sinf((1.f - x) * PI32 / 2.f), sinf(x * PI32 / 2.f));
            break;
        }
        case PATCH_OSC: {  // Planner::lower_osc's f64 expressions (OscInst::fast stays the planner's: the declared range keeps it)
            const float freq = patch_op(p, 0, values), detune = patch_op(p, 1, values);
            const double sr = (double)p.sample_rate;
            const double computed_freq = (double)freq * exp2((double)detune / 1200.);  // oscillator.rs:30-32
            OscInst* o = static_cast<OscInst*>(p.dst);
            const double incr = computed_freq / sr;
            const bool outside = fabs(computed_freq) >= sr / 2.;
            o->incr = incr;
            o->inv_incr = incr != 0. ? 1. / incr : 0.;
            o->outside_nyquist = outside;
            const double start = *static_cast<const double*>(p.dst2);
            o->phase0 = start < 1e300 ? osc_start(SchedClock(p.sample_rate), start, incr, outside).phase0 : 0.;
            break;
        }
        default: *static_cast<float*>(p.dst) = patch_op(p, 0, values); break;
    }
}

// step 3 (batches with spatial entries): what a static panner derives from its 15 spatial params, with the functions the planner
// runs on the host (Planner::lower_panner, static_hrtf_sel) and k_hrtf_sel runs per quantum.  One thread per entry, as k_hrtf_sel.
__global__ void __launch_bounds__(64) k_derive_spatial(const SpatialPatch* __restrict__ patches, int n, const float* __restrict__ values) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const SpatialPatch& p = patches[i];
    float v[15];
    for (int k = 0; k < 15; k++) v[k] = p.slot[k] >= 0 ? values[p.slot[k]] : p.val[k];
    const spatial::SpatialParams sp = spatial::spatial_params(p.model, v);
    if (p.kind == SPATIAL_PAN) {
        PanInst* o = static_cast<PanInst*>(p.dst);
        o->azimuth = sp.azimuth;
        o->dist_gain = sp.dist_gain;
        o->cone_gain = sp.cone_gain;
        return;
    }
    float proj[3];
    spatial::projected_source(sp, proj);
    const float dir[3] = {proj[0], proj[2], proj[1]};  // HrtfState::process swaps y / z (panner.rs:248-252)
    HrtfSel s{{0, 0, 0}, {0.f, 0.f, 0.f}, sp.cone_gain * sp.dist_gain, 0.f};
    spatial::hrir_locate(p.pos, p.tri, p.n_faces, dir, s.v, s.w);  // no face: all-zero weights (silence)
    *static_cast<HrtfSel*>(p.dst) = s;
}

// step 4 (SPATIAL_RESP entries): the blended pair of panner_hrtf_conv, corr * (((A * w0 + B * w1) + C * w2) * gain) in its f32
// operations and order (no contraction).  grid: (tap blocks, entries)
__global__ void __launch_bounds__(256) k_spatial_blend(const SpatialPatch* __restrict__ patches) {
    const SpatialPatch& p = patches[blockIdx.y];
    if (p.kind != SPATIAL_RESP) return;
    const HrtfSel s = *static_cast<const HrtfSel*>(p.dst);
    const int taps = p.taps;
    const float* A = p.ir + (size_t)s.v[0] * 2 * taps;
    const float* B = p.ir + (size_t)s.v[1] * 2 * taps;
    const float* C = p.ir + (size_t)s.v[2] * 2 * taps;
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < 2 * taps; k += gridDim.x * blockDim.x) {  // (left taps, then right)
        const float x = __fadd_rn(__fadd_rn(__fmul_rn(__ldg(A + k), s.w[0]), __fmul_rn(__ldg(B + k), s.w[1])), __fmul_rn(__ldg(C + k), s.w[2]));
        p.resp[k] = __fmul_rn(p.correction, __fmul_rn(x, s.gain));
    }
}

// ---------------------------------------------------------------------------------------------------------
// launchers
// ---------------------------------------------------------------------------------------------------------
static int g_num_sms = 132;  // H100 SXM; wae_engine_create sets the device's own count
void set_num_sms(int n) {
    if (n > 0) g_num_sms = n;
}
static inline dim3 grid_tiles(int nf, int per_block, int n_inst) {
    return dim3((unsigned)((nf + per_block - 1) / per_block), (unsigned)(n_inst < 32768 ? n_inst : 32768));
}


void launch_oscillator(const OscInst* d, int n, ChunkInfo ci, cudaStream_t s) { k_oscillator<<<grid_tiles(ci.nf, 1024, n), 256, 0, s>>>(d, n, ci); }
void launch_constant(const ConstInst* d, int n, ChunkInfo ci, cudaStream_t s) { k_constant<<<grid_tiles(ci.nf, 1024, n), 256, 0, s>>>(d, n, ci); }
void launch_buffer_source(const AbsnInst* d, int n, ChunkInfo ci, cudaStream_t s) { k_buffer_source<<<grid_tiles(ci.nf, 1024, n), 256, 0, s>>>(d, n, ci); }
void launch_buffer_source_slow(const AbsnSlowInst* d, int n, ChunkInfo ci, cudaStream_t s) {
    k_buffer_source_slow<false><<<grid_tiles(ci.nf, 256, n), 256, 0, s>>>(d, n, ci);
}
void launch_buffer_source_bound(const AbsnBoundInst* d, int n, ChunkInfo ci, cudaStream_t s) {
    k_buffer_source_slow<true><<<grid_tiles(ci.nf, 256 * ABSN_BOUND_TILES, n), 256, 0, s>>>(d, n, ci);
}
void launch_mix(const MixInst* d, const MixEdge* e, int n, ChunkInfo ci, cudaStream_t s, int max_edges) {
    // few instances x few frames (one graph with a huge fan-in): one frame per thread keeps more loads in flight
    const long ctas4 = (long)((ci.nf + 1023) / 1024) * n;
    if (max_edges < 16) {  // no port of this stage is wide enough for the staged kernel
        if (ctas4 < 2 * g_num_sms) k_mix_narrow<1><<<grid_tiles(ci.nf, 256, n), 256, 0, s>>>(d, e, n, ci);
        else k_mix_narrow<4><<<grid_tiles(ci.nf, 1024, n), 256, 0, s>>>(d, e, n, ci);
        return;
    }
    if (ctas4 < 2 * g_num_sms) k_mix<1><<<grid_tiles(ci.nf, 256, n), 256, 0, s>>>(d, e, n, ci);
    else k_mix<4><<<grid_tiles(ci.nf, 1024, n), 256, 0, s>>>(d, e, n, ci);
}
void launch_mix_dyn(const MixDynInst* d, const MixEdge* e, int n, ChunkInfo ci, cudaStream_t s) { k_mix_dyn<<<grid_tiles(ci.nf, 512, n), 128, 0, s>>>(d, e, n, ci); }
void launch_meta(const MetaInst* d, int n, ChunkInfo ci, cudaStream_t s) { k_meta<<<(n + 63) / 64, 64, 0, s>>>(d, n, ci); }
void launch_biquad_serial(const BiquadInst* d, int n, int max_ch, ChunkInfo ci, cudaStream_t s) {
    int threads = n * max_ch;
    k_biquad_serial<<<(threads + 127) / 128, 128, 0, s>>>(d, n, max_ch, ci);
}
// ---- k_chain launch geometry ---------------------------------------------------------------------------------------
static int g_chain_tma = -1, g_chain_waves = -1, g_chain_prepass = -1;
void chain_set_prepass(int on) { g_chain_prepass = on != 0; }
static void chain_env() {
    if (g_chain_tma < 0) {
        const char* e = getenv("WAE_CHAIN_TMA");
        g_chain_tma = e ? (atoi(e) != 0) : 0;  // default: the cp.async path (WAE_CHAIN_TMA=1 selects the bulk copies)
        e = getenv("WAE_CHAIN_WAVES");
        g_chain_waves = e ? atoi(e) : 20;
        if (g_chain_waves < 0) g_chain_waves = 0;
    }
}
void chain_set_tuning(int tma, int waves) {
    chain_env();
    if (tma >= 0) g_chain_tma = tma != 0;
    if (waves >= 0) g_chain_waves = waves;
}
// Time slabs of one launch: enough work items for `waves` waves of resident CTAs (SMs x 6), at least 8 tiles each.  Filtered
// chains are only cut when the launch has enough (instance, channel) pairs to fill half the machine without it: the slabs of one
// pair run one after the other (the state is handed over), so with few pairs more slabs would only add waiting CTAs.
void chain_plan_slabs(int n, int max_ch, int nf, int nb, int* n_slabs, int* tiles_per_slab, int* pre_log2) {
    chain_env();
    const long ctas = (long)n * max_ch, tiles = (nf + CH_THREADS * CH_K - 1) / (CH_THREADS * CH_K);
    const long slots = (long)g_num_sms * (WAE_CH_MINB * 128 / CH_THREADS);
    if (pre_log2) *pre_log2 = -1;
    // Few (instance, channel) pairs and a long render (64 files of two minutes instead of 1000 of ten seconds): the pairs alone leave
    // the machine empty and the slabs of one pair would wait for each other — unless every slab first finds out what it hands on
    // (k_chain PRE).  One filter only: with two, the second one's input history is a rounded function of the first one's state.
    if (g_chain_prepass < 0) {
        const char* e = getenv("WAE_CHAIN_PREPASS");
        g_chain_prepass = (!e || atoi(e) != 0) ? 1 : 0;
    }
    if (pre_log2 && g_chain_prepass && nb == 1 && 2 * ctas < slots && tiles >= 2 * WAE_CHAIN_PRE_TILES) {
        long tps = WAE_CHAIN_PRE_TILES;
        int j = 0;
        while ((tiles + tps - 1) / tps > CHAIN_MAX_PRE_SLABS) tps *= 2, j++;
        *n_slabs = (int)((tiles + tps - 1) / tps);
        *tiles_per_slab = (int)tps;
        *pre_log2 = j;
        return;
    }
    const long min_tiles = std::max(1L, 16384L / (CH_THREADS * CH_K));  // a slab is at least 16384 frames
    long slabs = 1;
    if (nb == 0) {
        slabs = (slots * 2 / 3 + ctas - 1) / ctas;  // stateless chain: split along time until the launch fills the machine
        if (g_chain_waves > 0 && ctas * slabs < (long)g_chain_waves * slots) slabs = ((long)g_chain_waves * slots + ctas - 1) / ctas;
        if (slabs > std::max(1L, tiles / std::max(1L, min_tiles / 4))) slabs = std::max(1L, tiles / std::max(1L, min_tiles / 4));
    } else if (g_chain_waves > 0 && 2 * ctas >= slots) {
        slabs = ((long)g_chain_waves * slots + ctas - 1) / ctas;
        if (slabs > tiles / min_tiles) slabs = tiles / min_tiles;
    }
    if (slabs > CHAIN_MAX_SLABS) slabs = CHAIN_MAX_SLABS;
    if (slabs < 1) slabs = 1;
    long tps = (tiles + slabs - 1) / slabs;
    if (tps < 1) tps = 1;
    slabs = (tiles + tps - 1) / tps;
    if (slabs < 1) slabs = 1;
    *n_slabs = (int)slabs;
    *tiles_per_slab = (int)tps;
}
template <int SRC, int NB>
static void launch_chain_v(bool shaper, const ChainInst* d, const ScanCoef* c, int n, int max_ch, ChunkInfo ci, cudaStream_t s, ChainAux aux) {
    ChainSched sc{};
    int pre_log2 = -1;
    chain_plan_slabs(n, max_ch, ci.nf, NB, &sc.n_slabs, &sc.tiles_per_slab, &pre_log2);
    if (NB > 0 && (sc.n_slabs > aux.slab_stride || !aux.ticket)) {  // no hand-off memory for that many slabs: one slab
        sc.n_slabs = 1;
        sc.tiles_per_slab = (ci.nf + CH_THREADS * CH_K - 1) / (CH_THREADS * CH_K);
        pre_log2 = -1;
    }
    sc.pre_log2 = sc.n_slabs > 1 ? pre_log2 : -1;
    sc.max_ch = max_ch;
    sc.slab_stride = aux.slab_stride > 0 ? aux.slab_stride : 1;
    sc.epoch = aux.epoch;
    sc.ticket = (NB > 0 && sc.n_slabs > 1) ? aux.ticket : nullptr;
    sc.handoff = aux.handoff;
    sc.flags = aux.flags;
    const unsigned grid = (unsigned)n * (unsigned)max_ch * (unsigned)sc.n_slabs;
    constexpr bool STREAMED = SRC == CHAIN_SRC_BUFFER || SRC == CHAIN_SRC_ABSN;
    // six CTAs of ~35 KB staging each only fit an SM with the shared-memory carve-out at its maximum
    static bool carved = false;
    if (!carved && !getenv("WAE_CHAIN_NO_CARVEOUT")) {
        carved = true;
        cudaFuncSetAttribute(k_chain<SRC, NB, true, false>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        cudaFuncSetAttribute(k_chain<SRC, NB, false, false>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        if constexpr (STREAMED) {
            cudaFuncSetAttribute(k_chain<SRC, NB, true, true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
            cudaFuncSetAttribute(k_chain<SRC, NB, false, true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        }
    }
    if constexpr (STREAMED) {
        if (g_chain_tma) {
            if (shaper) k_chain<SRC, NB, true, true><<<grid, CH_THREADS, 0, s>>>(d, c, n, ci, sc);
            else k_chain<SRC, NB, false, true><<<grid, CH_THREADS, 0, s>>>(d, c, n, ci, sc);
            return;
        }
    }
    if constexpr (NB == 1) {
        if (sc.pre_log2 >= 0) {
            static bool carved_pre = false;
            if (!carved_pre && !getenv("WAE_CHAIN_NO_CARVEOUT")) {
                carved_pre = true;
                cudaFuncSetAttribute(k_chain<SRC, NB, true, false, true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
                cudaFuncSetAttribute(k_chain<SRC, NB, false, false, true>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
            }
            if (shaper) k_chain<SRC, NB, true, false, true><<<grid, CH_THREADS, 0, s>>>(d, c, n, ci, sc);
            else k_chain<SRC, NB, false, false, true><<<grid, CH_THREADS, 0, s>>>(d, c, n, ci, sc);
            return;
        }
    }
    {
        if (shaper) k_chain<SRC, NB, true, false><<<grid, CH_THREADS, 0, s>>>(d, c, n, ci, sc);
        else k_chain<SRC, NB, false, false><<<grid, CH_THREADS, 0, s>>>(d, c, n, ci, sc);
    }
}
template <int SRC>
static void launch_chain_s(int nb, bool shaper, const ChainInst* d, const ScanCoef* c, int n, int max_ch, ChunkInfo ci, cudaStream_t s, ChainAux aux) {
    if (nb == 0) launch_chain_v<SRC, 0>(shaper, d, c, n, max_ch, ci, s, aux);
    else if (nb == 1) launch_chain_v<SRC, 1>(shaper, d, c, n, max_ch, ci, s, aux);
    else launch_chain_v<SRC, 2>(shaper, d, c, n, max_ch, ci, s, aux);
}
// variant = src_kind * 6 + n_biquad * 2 + has_shaper (all instances of one launch share the chain shape)
void launch_chain(int variant, const ChainInst* d, const ScanCoef* c, int n, int max_ch, ChunkInfo ci, cudaStream_t s, ChainAux aux) {
    const int src = variant / 6, nb = (variant % 6) / 2;
    const bool shaper = (variant & 1) != 0;
    switch (src) {
        case CHAIN_SRC_BUFFER: launch_chain_s<CHAIN_SRC_BUFFER>(nb, shaper, d, c, n, max_ch, ci, s, aux); break;
        case CHAIN_SRC_ABSN: launch_chain_s<CHAIN_SRC_ABSN>(nb, shaper, d, c, n, max_ch, ci, s, aux); break;
        case CHAIN_SRC_OSC: launch_chain_s<CHAIN_SRC_OSC>(nb, shaper, d, c, n, max_ch, ci, s, aux); break;
        default: launch_chain_s<CHAIN_SRC_CONST>(nb, shaper, d, c, n, max_ch, ci, s, aux); break;
    }
}
int voice_sum_slots() { return g_num_sms * (WAE_VS_MINB * 128 / CH_THREADS); }
void launch_voice_sum(int nb, const ChainInst* d, const ScanCoef* c, const VoiceGroup* g, int n_groups, ChunkInfo ci, cudaStream_t s, ChainAux aux) {
    ChainSched sc{};
    const int n_tiles = (ci.nf + CH_THREADS * CH_K - 1) / (CH_THREADS * CH_K);
    sc.n_slabs = n_tiles;
    sc.tiles_per_slab = 1;
    sc.max_ch = 1;
    sc.slab_stride = aux.slab_stride;  // progress counters per group (>= n_tiles: sized for a whole chunk)
    sc.epoch = aux.epoch;
    sc.pre_log2 = -1;
    sc.ticket = aux.ticket;
    sc.handoff = aux.handoff;
    sc.flags = aux.flags;
    const unsigned grid = (unsigned)n_tiles * (unsigned)n_groups;
    static bool carved = false;
    if (!carved) {
        carved = true;
        cudaFuncSetAttribute(k_voice_sum<0>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
        cudaFuncSetAttribute(k_voice_sum<1>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    }
    if (nb == 0) k_voice_sum<0><<<grid, CH_THREADS, 0, s>>>(d, c, g, n_groups, ci, sc);
    else k_voice_sum<1><<<grid, CH_THREADS, 0, s>>>(d, c, g, n_groups, ci, sc);
}
void launch_iir(const IirInst* d, int n, int max_ch, ChunkInfo ci, cudaStream_t s) {
    int threads = n * max_ch;
    k_iir_serial<<<(threads + 63) / 64, 64, 0, s>>>(d, n, max_ch, ci);
}
void launch_gain(const GainInst* d, int n, ChunkInfo ci, cudaStream_t s) { k_gain<<<grid_tiles(ci.nf, 1024, n), 256, 0, s>>>(d, n, ci); }
void launch_shaper(const ShaperInst* d, int n, ChunkInfo ci, cudaStream_t s) { k_shaper<<<grid_tiles(ci.nf, 1024, n), 256, 0, s>>>(d, n, ci); }
void launch_stereo_panner(const SPanInst* d, const float2* g, int n, ChunkInfo ci, cudaStream_t s) {
    k_stereo_panner<<<grid_tiles(ci.nf, 256, n), 256, 0, s>>>(d, g, n, ci);
}
void launch_buffer_source_serial(const AbsnSerialInst* d, int n, ChunkInfo ci, cudaStream_t s) {
    k_buffer_source_serial<<<(n + ABSN_SERIAL_WARPS - 1) / ABSN_SERIAL_WARPS, 32 * ABSN_SERIAL_WARPS, 0, s>>>(d, n, ci);
}
void launch_shaper_os(const ShaperOsInst* d, int n, int max_ch, ChunkInfo ci, cudaStream_t s) {
    k_shaper_os_prev<<<(n + 63) / 64, 64, 0, s>>>(d, n, ci);
    k_shaper_os<<<dim3((unsigned)(ci.nf / 128), (unsigned)max_ch, (unsigned)n), 128, 0, s>>>(d, ci);
    k_shaper_os_hist<<<n, 256, 0, s>>>(d, ci);
}
void launch_panner_dyn(const PanDynInst* d, int n, ChunkInfo ci, cudaStream_t s) { k_panner_dyn<<<grid_tiles(ci.nf, 128, n), 128, 0, s>>>(d, n, ci); }
void launch_hrtf(const HrtfInst* d, int n, const HrtfSelInst* sel, int n_sel, int max_taps, ChunkInfo ci, cudaStream_t s) {
    if (n_sel > 0) k_hrtf_sel<<<dim3((ci.nf / 128 + 63) / 64 + 1, n_sel), 64, 0, s>>>(sel, ci);
    const int L4 = (max_taps + 3) & ~3;
    const int nx = 4 + (L4 - 1) + HRTF_TILE;
    const int copies = n_sel > 0 ? 8 : 1;  // blended responses kept in shared memory: one per quantum only for moving sources
    const size_t smem = (size_t)(((nx + (nx >> 3) + 4) & ~3) + copies * 2 * L4) * sizeof(float);
    static size_t configured = 48 * 1024;
    if (smem > configured) {
        cudaFuncSetAttribute(k_hrtf_fir, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        configured = smem;
    }
    k_hrtf_map<<<(n + 63) / 64, 64, 0, s>>>(d, n, ci);
    k_hrtf_fir<<<dim3((ci.nf + HRTF_TILE - 1) / HRTF_TILE, n), 128, smem, s>>>(d, ci);
    k_hrtf_fill<<<grid_tiles(ci.nf, 256, n), 256, 0, s>>>(d, n, ci);
    k_hrtf_hist<<<n, 128, (size_t)max_taps * sizeof(float), s>>>(d, ci);
}
void launch_panner_eq(const PanInst* d, int n, ChunkInfo ci, cudaStream_t s) { k_panner_eq<<<grid_tiles(ci.nf, 256, n), 256, 0, s>>>(d, n, ci); }
void launch_route(const RouteInst* d, int n, ChunkInfo ci, cudaStream_t s) { k_route<<<grid_tiles(ci.nf, 1024, n), 256, 0, s>>>(d, n, ci); }
void launch_delay_read(const DelayInst* d, int n, ChunkInfo ci, cudaStream_t s) { k_delay_read<<<grid_tiles(ci.nf, 256, n), 256, 0, s>>>(d, n, ci); }
void launch_delay_mono(const DelayInst* d, int n, ChunkInfo ci, cudaStream_t s) { k_delay_mono<<<(n + 63) / 64, 64, 0, s>>>(d, n, ci); }
void launch_ring_write(const DelayInst* d, int n, ChunkInfo ci, cudaStream_t s) { k_ring_write<<<grid_tiles(ci.nf, 256, n), 256, 0, s>>>(d, n, ci); }
void launch_osc_arate(const OscArInst* d, int n, ChunkInfo ci, cudaStream_t s) { k_osc_arate<<<n, 256, 0, s>>>(d, n, ci); }
void launch_biquad_arate(const BiquadArInst* d, int n, int max_ch, ChunkInfo ci, cudaStream_t s) {
    k_biquad_coefs<<<grid_tiles(ci.nf, 256, n), 256, 0, s>>>(d, n, ci);
    const int warps = n * max_ch;
    k_biquad_arate<<<(warps + BQA_WARPS - 1) / BQA_WARPS, 32 * BQA_WARPS, 0, s>>>(d, n, max_ch, ci);
}
void launch_analyser_fft(const float* ring, uint32_t write_index, int fft_size, float smoothing, float* last_fft, float* out_db, cudaStream_t s) {
    static bool configured = false;
    if (!configured) {
        cudaFuncSetAttribute(k_analyser_fft, cudaFuncAttributeMaxDynamicSharedMemorySize, 16384 * (int)sizeof(float2));
        configured = true;
    }
    k_analyser_fft<<<1, 256, (size_t)(fft_size / 2) * sizeof(float2), s>>>(ring, write_index, fft_size, smoothing, last_fft, out_db);
}
void launch_readout_fft(const ReadoutInst* d, int n, int max_fft, ChunkInfo ci, cudaStream_t s) {
    static bool configured = false;
    if (!configured) {
        cudaFuncSetAttribute(k_readout_fft, cudaFuncAttributeMaxDynamicSharedMemorySize, 16384 * (int)sizeof(float2));
        configured = true;
    }
    k_readout_fft<<<n, 256, (size_t)(max_fft / 2) * sizeof(float2), s>>>(d, ci);
}
void launch_readout_time(const ReadoutInst* d, int n, int max_fft, ChunkInfo ci, cudaStream_t s) {
    k_readout_time<<<dim3(n, (max_fft + 255) / 256), 256, 0, s>>>(d, ci);
}
void launch_readout_smooth(const ReadoutSmoothInst* d, int n, int max_bins, ChunkInfo ci, cudaStream_t s) {
    k_readout_smooth<<<dim3(n, (max_bins + 255) / 256), 256, 0, s>>>(d, ci);
}
void launch_resample_linear(const float* in, int64_t len, float* out, int64_t target_len, cudaStream_t s) {
    k_resample_linear<<<(unsigned)((target_len + 255) / 256), 256, 0, s>>>(in, len, out, target_len);
}
void launch_param(const ParamInst* d, int n, ChunkInfo ci, cudaStream_t s, int mode) {
    if (mode >= 2) k_param_spec<<<n, 32 * PSPEC_WARPS, 0, s>>>(d, n, ci);
    else if (mode == 1) k_param_parallel<<<(n + PARAM_WARPS - 1) / PARAM_WARPS, 32 * PARAM_WARPS, 0, s>>>(d, n, ci);
    else k_param<<<(n + PARAM_WARPS - 1) / PARAM_WARPS, 32 * PARAM_WARPS, 0, s>>>(d, n, ci);
}
void launch_compressor(const CompInst* d, const CompReadoutInst* ro, int n, ChunkInfo ci, cudaStream_t s) {
    if (ro) k_compressor<true><<<(n + 31) / 32, 32, 0, s>>>(d, ro, n, ci);
    else k_compressor<false><<<(n + 31) / 32, 32, 0, s>>>(d, nullptr, n, ci);
}
void launch_analyser(const AnalyserInst* d, int n, ChunkInfo ci, cudaStream_t s) { k_analyser<<<grid_tiles(ci.nf, 256, n), 256, 0, s>>>(d, n, ci); }
static void conv_configure() {
    static bool configured = false;
    if (configured) return;
    const int smem = CV_SMEM_ELEMS * (int)sizeof(float2);
    cudaFuncSetAttribute(k_conv_fft_in, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    cudaFuncSetAttribute(k_conv_ifft, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    cudaFuncSetAttribute(k_conv_ir_fft, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    cudaFuncSetAttribute(k_resp_fft, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    cudaFuncSetAttribute(k_conv_cmp_fft, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    cudaFuncSetAttribute(k_conv_cmp_ifft, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    configured = true;
}
void launch_conv_fft_in(const ConvInput* d, int n, ChunkInfo ci, cudaStream_t s) {
    conv_configure();
    const int nb = (ci.nf + CV_B - 1) / CV_B;
    k_conv_fft_in<<<dim3((unsigned)nb, (unsigned)n), CV_THREADS, CV_SMEM_ELEMS * sizeof(float2), s>>>(d, n, ci);
    k_conv_save_prev<<<dim3(CV_B / 256, (unsigned)n), 256, 0, s>>>(d, n, ci);
}
void launch_conv_mac_ifft(const ConvPath* p, const ConvInput* in, int n, ChunkInfo ci, cudaStream_t s) {
    conv_configure();
    const int nb = (ci.nf + CV_B - 1) / CV_B;
    k_conv_mac<<<dim3((unsigned)((CV_B / CV_MAC_THREADS) * ((nb + CV_J - 1) / CV_J)), (unsigned)n), CV_MAC_THREADS, 0, s>>>(p, in, n, ci);
    k_conv_ifft<<<dim3((unsigned)nb, (unsigned)n), CV_THREADS, CV_SMEM_ELEMS * sizeof(float2), s>>>(p, in, n, ci);
}
void launch_conv_compact(const ConvCmpInst* d, int n, ChunkInfo ci, cudaStream_t s) {
    conv_configure();
    const int wb = (ci.nf + CV_B - 1) / CV_B + 1;  // stream blocks the chunk's new frames can reach (the partial block in front: one more)
    const size_t smem = CV_SMEM_ELEMS * sizeof(float2);
    k_conv_cmp_map<<<(n + 3) / 4, 128, 0, s>>>(d, n, ci);
    k_conv_cmp_gather<<<dim3((unsigned)((wb + 1) * (CV_B / 256)), (unsigned)n), 256, 0, s>>>(d, ci);
    k_conv_cmp_fft<<<dim3((unsigned)wb, (unsigned)n), CV_THREADS, smem, s>>>(d, ci);
    k_conv_cmp_carry<<<dim3(2 * CV_B / 256, (unsigned)n), 256, 0, s>>>(d);
    k_conv_cmp_mac<<<dim3((unsigned)((CV_B / CV_MAC_THREADS) * ((wb + CV_J - 1) / CV_J)), (unsigned)n), CV_MAC_THREADS, 0, s>>>(d, ci);
    k_conv_cmp_ifft<<<dim3((unsigned)wb, (unsigned)n), CV_THREADS, smem, s>>>(d, ci);
}
void launch_bind_sources(const BindItem* d, int n, int64_t max_vec, int max_ch, cudaStream_t s) {
    // about four vectors per thread along a channel; items beyond 65535 are walked by the grid-stride loop over blockIdx.y
    const int64_t bx = std::max<int64_t>(1, std::min<int64_t>((max_vec + 1023) / 1024, 65535));
    k_bind_sources<<<dim3((unsigned)bx, (unsigned)std::min(n, 65535), (unsigned)max_ch), 256, 0, s>>>(d, n);
}
void launch_bind_params(const ParamBindItem* d, int n, const ParamSlotInfo* info, float* values, const ParamPatch* patches, int n_patches,
                        cudaStream_t s) {
    k_bind_params<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(d, n, info, values);
    if (n_patches > 0) k_derive_params<<<(unsigned)((n_patches + 63) / 64), 64, 0, s>>>(patches, n_patches, values);
}
void launch_derive_spatial(const SpatialPatch* patches, int n, const float* values, const RespBindItem* resp, int n_resp, int max_taps,
                           int max_S, cudaStream_t s) {
    k_derive_spatial<<<(unsigned)((n + 63) / 64), 64, 0, s>>>(patches, n, values);
    if (n_resp == 0) return;
    conv_configure();
    const unsigned bx = (unsigned)std::max(1, std::min((2 * max_taps + 255) / 256, 64));
    for (int k = 0; k < n; k += 65535) k_spatial_blend<<<dim3(bx, (unsigned)std::min(n - k, 65535)), 256, 0, s>>>(patches + k);
    for (int k = 0; k < n_resp; k += 65535)  // (the transform of wae_batch_bind_responses: scale 1, untrimmed)
        k_resp_fft<<<dim3((unsigned)max_S, 2, (unsigned)std::min(n_resp - k, 65535)), CV_THREADS, CV_SMEM_ELEMS * sizeof(float2), s>>>(resp + k);
}
void launch_bind_responses(RespBindItem* d, int n, bool any_normalize, int64_t max_len, int max_S, int max_ch, cudaStream_t s) {
    conv_configure();
    if (any_normalize) k_resp_power<<<(unsigned)n, 256, 0, s>>>(d);
    // about eight frames per thread; items and their channels in y / z (n <= 65535: checked by the caller)
    const int64_t bx = std::max<int64_t>(1, std::min<int64_t>((max_len + 2047) / 2048, 65535));
    k_resp_trim<<<dim3((unsigned)bx, (unsigned)n, (unsigned)max_ch), 256, 0, s>>>(d);
    k_resp_fft<<<dim3((unsigned)max_S, (unsigned)max_ch, (unsigned)n), CV_THREADS, CV_SMEM_ELEMS * sizeof(float2), s>>>(d);
}
void launch_bind_curves(const CurveBindItem* d, int n, cudaStream_t s) { k_bind_curves<<<(unsigned)n, 256, 0, s>>>(d); }
void launch_bind_waves(const WaveBindItem* d, int n, int max_len, bool any_normalize, cudaStream_t s) {
    for (int k = 0; k < n; k += 65535)  // (grid.y is at most 65535)
        k_bind_waves<<<dim3((unsigned)((max_len + WAVE_TILE - 1) / WAVE_TILE), (unsigned)std::min(n - k, 65535)), WAVE_TILE, 0, s>>>(d + k);
    if (any_normalize) k_wave_normalize<<<(unsigned)n, 1024, 0, s>>>(d);
}
void launch_bind_iir(const IirBindItem* d, int n, cudaStream_t s) { k_bind_iir<<<(unsigned)n, 32, 0, s>>>(d); }
void launch_bind_value_curves(const ValueCurveBindItem* d, int n, int64_t max_len, cudaStream_t s) {
    const int64_t bx = std::max<int64_t>(1, std::min<int64_t>((max_len + VC_TILE - 1) / VC_TILE, 65535));
    k_bind_value_curves<<<dim3((unsigned)bx, (unsigned)std::min(n, 65535)), 256, 0, s>>>(d, n);
}
void launch_bind_schedules(const SchedBindItem* d, int n, cudaStream_t s) { k_bind_schedules<<<(unsigned)((n + 127) / 128), 128, 0, s>>>(d, n); }
void launch_bind_loops(const LoopBindItem* d, int n, cudaStream_t s) { k_bind_loops<<<(unsigned)((n + 127) / 128), 128, 0, s>>>(d, n); }
void launch_absn_loop_schedule(const LoopWalk* d, int n, int* overflow, cudaStream_t s) {
    k_absn_loop_schedule<<<(unsigned)((n + 127) / 128), 128, 0, s>>>(d, n, overflow);
}
void launch_bind_output(const OutPatch* d, int n, float* base, cudaStream_t s) {
    k_bind_output<<<(unsigned)((n + 127) / 128), 128, 0, s>>>(d, n, base);
}
void launch_bind_source_refs(const SrcRefBindItem* d, int n, const SrcRefPatch* entries, cudaStream_t s) {
    k_bind_source_refs<<<(unsigned)((n + 127) / 128), 128, 0, s>>>(d, n, entries);
}
void launch_conv_ir_fft(const float* ir, int64_t ir_len, int64_t ir_stride, float2* h, int S, int channels, cudaStream_t s) {
    conv_configure();
    k_conv_ir_fft<<<dim3((unsigned)S, (unsigned)channels), CV_THREADS, CV_SMEM_ELEMS * sizeof(float2), s>>>(ir, ir_len, ir_stride, h, S);
}

}  // namespace wae
