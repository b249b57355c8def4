// ORACLE — TEST INFRASTRUCTURE ONLY (see wao_core.h).
//
// rubato::FftFixedInOut<f32> as used by the over-sampled WaveShaper (src/node/waveshaper.rs:236-348,409-480).  The crate
// (rubato = "0.16", Cargo.toml:46) is NOT in the reference source tree: this restates its PUBLISHED algorithm (synchronous FFT
// resampler): per chunk of fft_size_in frames
//     X = rFFT([chunk | zeros])                          (2 * fft_size_in points)
//     Y[k] = X[k] * F[k]   for k < min(fft_size_in, fft_size_out),  0 above
//     y = irFFT(Y)                                       (2 * fft_size_out points, unnormalised)
//     out = y[0 .. fft_size_out) + overlap;  overlap = y[fft_size_out ..)
// where F = rFFT of a Blackman-Harris^2 windowed sinc of fft_size_in taps (cutoff 0.4^(16 / fft_size_in), times
// fft_size_out / fft_size_in when down-sampling), normalised to unit sum and divided by 2 * fft_size_in.
// PARITY UNPINNED: the reference has no numeric test for the over-sampled paths (waveshaper.rs:586-760 only checks
// OverSampleType::None values); constants and bin bookkeeping follow the crate's documentation / source as remembered.
#pragma once
#include "wao_fft.h"

#include <cstddef>
#include <vector>

namespace wao {

std::vector<float> rubato_sinc_filter(size_t npoints, float f_cutoff);  // make_sincs(npoints, 1, cutoff, BlackmanHarris2)[0]

class FftFixedInOut {
  public:
    size_t fft_size_in = 0, fft_size_out = 0;
    FftFixedInOut() {}
    FftFixedInOut(size_t sample_rate_in, size_t sample_rate_out, size_t chunk_size_in, size_t channels);
    // in: [channels][fft_size_in] -> out: [channels][fft_size_out]
    void process(const std::vector<std::vector<float>>& in, std::vector<std::vector<float>>& out);

  private:
    RealFFT fft, ifft;
    std::vector<cf32> filter_f;
    std::vector<std::vector<float>> overlaps;
};

}  // namespace wao
