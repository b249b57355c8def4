// Host-side (control-plane) math of the engine: per-node constants that the reference computes once per
// quantum from k-rate values and that the GPU kernels take as inputs.  f64/f32 glibc math in the same
// expressions as the reference so the constants are bit-identical to the CPU renderer's.
#pragma once
#include <cmath>
#include <cstdint>
#include <limits>
#include <vector>

#include "wae_spatial.h"

namespace wae {
namespace hostmath {

static const double PI64 = 3.14159265358979323846;
static const float PI32 = 3.14159265358979323846f;
static const double F64_MAX = 1.7976931348623157e308;

struct BiquadCoefs {
    double b0, b1, b2, a1, a2;
};

inline BiquadCoefs norm(double b0, double b1, double b2, double a0, double a1, double a2) {
    double s = 1. / a0;  // normalize_coefs, src/node/biquad_filter.rs:28-40
    return BiquadCoefs{b0 * s, b1 * s, b2 * s, a1 * s, a2 * s};
}

// calculate_coefs, src/node/biquad_filter.rs:42-390 (WPT biquad-filters.js formulas)
inline BiquadCoefs biquad_coefs(int type, double sample_rate, double f0, double gain, double q) {
    const BiquadCoefs wire{1., 0., 0., 0., 0.}, zero{0., 0., 0., 0., 0.};
    double nyquist = sample_rate / 2.;
    double f = f0 / nyquist;
    f = f < 0. ? 0. : (f > 1. ? 1. : f);
    double w0 = PI64 * f, s = std::sin(w0), c = std::cos(w0);
    double A = std::pow(10., gain / 40.);
    switch (type) {
        case 0: {
            if (f == 1.) return wire;
            double a = s / (2. * std::pow(10., q / 20.)), beta = (1. - c) / 2.;
            return norm(beta, 2. * beta, beta, 1. + a, -2. * c, 1. - a);
        }
        case 1: {
            if (f == 1.) return zero;
            if (f == 0.) return wire;
            double a = s / (2. * std::pow(10., q / 20.)), beta = (1. + c) / 2.;
            return norm(beta, -2. * beta, beta, 1. + a, -2. * c, 1. - a);
        }
        case 2: {
            if (!(f > 0. && f < 1.)) return zero;
            if (!(q > 0.)) return wire;
            double a = s / (2. * q);
            return norm(a, 0., -a, 1. + a, -2. * c, 1. - a);
        }
        case 3: {
            if (!(f > 0. && f < 1.)) return wire;
            if (!(q > 0.)) return zero;
            double a = s / (2. * q);
            return norm(1., -2. * c, 1., 1. + a, -2. * c, 1. - a);
        }
        case 4: {
            if (!(f > 0. && f < 1.)) return wire;
            if (!(q > 0.)) return BiquadCoefs{-1., 0., 0., 0., 0.};
            double a = s / (2. * q);
            return norm(1. - a, -2. * c, 1. + a, 1. + a, -2. * c, 1. - a);
        }
        case 5: {
            if (!(f > 0. && f < 1.)) return wire;
            if (!(q > 0.)) return BiquadCoefs{A * A, 0., 0., 0., 0.};
            double a = s / (2. * q);
            return norm(1. + a * A, -2. * c, 1. - a * A, 1. + a / A, -2. * c, 1. - a / A);
        }
        case 6: {
            if (f == 1.) return BiquadCoefs{A * A, 0., 0., 0., 0.};
            if (f == 0.) return wire;
            double as = s / 2. * 1.41421356237309504880168872420969808;
            double t = 2. * as * std::sqrt(A), ap = A + 1., am = A - 1.;
            return norm(A * (ap - am * c + t), 2. * A * (am - ap * c), A * (ap - am * c - t), ap + am * c + t, -2. * (am + ap * c),
                        ap + am * c - t);
        }
        default: {
            if (f == 1.) return wire;
            if (!(f > 0.)) return BiquadCoefs{A * A, 0., 0., 0., 0.};
            double as = s / 2. * 1.41421356237309504880168872420969808;
            double t = 2. * as * std::sqrt(A), ap = A + 1., am = A - 1.;
            return norm(A * (ap + am * c + t), -2. * A * (am + ap * c), A * (ap + am * c - t), ap - am * c + t, 2. * (am - ap * c),
                        ap - am * c - t);
        }
    }
}

// get_computed_freq, src/node/biquad_filter.rs:393-399 (f32)
inline float biquad_computed_freq(float freq, float detune) { return detune != 0.f ? freq * exp2f(detune / 1200.f) : freq; }

// An OscillatorNode whose frequency and detune are bound from device memory: every computed frequency f * 2^(d / 1200)
// (oscillator.rs:30-32) that f in [f_lo, f_hi], d in [d_lo, d_hi] allow lies inside (0, sample_rate / 2).  Then every value renders on
// the path the planner picks from one of them (inside Nyquist, OscInst::fast the same).  The product is monotone in both once f > 0, so
// the corners decide.  The top keeps a relative margin of a few ulps below Nyquist: the device's exp2 may round its last bit the other
// way than glibc's.
inline bool osc_pitch_inside(double f_lo, double f_hi, double d_lo, double d_hi, double sample_rate) {
    const double lo = f_lo * std::exp2(d_lo / 1200.), hi = f_hi * std::exp2(d_hi / 1200.);
    return f_lo > 0. && lo > 0. && hi < sample_rate / 2. * (1. - 8. * std::numeric_limits<double>::epsilon());
}

// sine table, src/node/oscillator.rs:16-28
inline std::vector<float> sine_table() {
    std::vector<float> t(2048);
    for (int x = 0; x < 2048; x++) t[x] = sinf((float)x * 2.0f * PI32 * (1.f / 2048.f));
    return t;
}

// get_stereo_gains, src/node/stereo_panner.rs:74-79
inline void stereo_gains(float x, float& gl, float& gr) {
    gl = sinf((1.f - x) * PI32 / 2.f);
    gr = sinf(x * PI32 / 2.f);
}

// spatial helpers (src/spatial.rs:205-299) live in wae_spatial.h, shared with the device code
using namespace ::wae::spatial;

}  // namespace hostmath
}  // namespace wae
