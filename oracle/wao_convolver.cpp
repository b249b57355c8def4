// ORACLE — TEST INFRASTRUCTURE ONLY (see wao_core.h).
//
// ConvolverNode: src/node/convolver.rs (normalize_buffer :16-53, set_buffer :259-317, process :343-490).
//
// The arithmetic lives in the third-party crate `fft-convolver = "0.3"` (Cargo.toml:24), which is NOT in
// the reference source tree (no vendored sources, no Cargo.lock).  FFTConvolver below restates that crate's
// published algorithm (a Rust port of HiFi-LoFi's FFTConvolver): uniformly partitioned overlap-add
// convolution, block = next_pow2(block_size), FFT = 2*block, the partially filled input block is
// re-transformed on every process() call, the products of all but the newest segment are cached in
// `pre_multiplied` when a block starts.  Parity anchor: the reference's call sites (convolver.rs:301-304
// init(1024, ir); :384-466 process(in128, out128)) and its own tests convolver.rs:550-991 (restated in
// tests/test_oracle_kat.py).  FFT rounding (rustfft) is NOT pinned: any correct f32 FFT agrees with it to
// ~1e-7 relative, far below the 1e-5 tolerance of this path.
#include "wao_nodes.h"

namespace wao {

static size_t next_pow2(size_t v) {
    size_t p = 1;
    while (p < v) p <<= 1;
    return p;
}

void FFTConvolver::init(size_t block_size_, const float* ir, size_t ir_len_) {
    segments.clear();
    segments_ir.clear();
    seg_count = 0;
    current = 0;
    input_buffer_fill = 0;
    // "Ignore zeros at the end of the impulse response because they only waste computation time"
    size_t n = ir_len_;
    while (n > 0 && std::fabs(ir[n - 1]) < 0.000001f) n--;
    ir_len = n;
    if (n == 0) return;
    block_size = next_pow2(block_size_);
    seg_size = 2 * block_size;
    seg_count = (ir_len + block_size - 1) / block_size;
    fft_complex_size = seg_size / 2 + 1;
    fft.init((int)seg_size);
    fft_buffer.assign(seg_size, 0.f);
    segments.assign(seg_count, std::vector<cf32>(fft_complex_size, cf32(0.f, 0.f)));
    segments_ir.assign(seg_count, std::vector<cf32>(fft_complex_size, cf32(0.f, 0.f)));
    for (size_t i = 0; i < seg_count; i++) {
        size_t remaining = ir_len - i * block_size;
        size_t size_copy = remaining >= block_size ? block_size : remaining;
        std::fill(fft_buffer.begin(), fft_buffer.end(), 0.f);
        std::memcpy(fft_buffer.data(), ir + i * block_size, size_copy * sizeof(float));
        fft.forward(fft_buffer.data(), segments_ir[i].data());
    }
    pre_multiplied.assign(fft_complex_size, cf32(0.f, 0.f));
    conv.assign(fft_complex_size, cf32(0.f, 0.f));
    overlap.assign(block_size, 0.f);
    input_buffer.assign(block_size, 0.f);
}

static inline void complex_multiply_accumulate(std::vector<cf32>& result, const std::vector<cf32>& a, const std::vector<cf32>& b) {
    size_t n = result.size();
    for (size_t i = 0; i < n; i++) {
        float ar = a[i].real(), ai = a[i].imag(), br = b[i].real(), bi = b[i].imag();
        result[i] = cf32(result[i].real() + (ar * br - ai * bi), result[i].imag() + (ar * bi + ai * br));
    }
}

void FFTConvolver::process(const float* input, float* output, size_t len) {
    if (seg_count == 0) {
        std::memset(output, 0, len * sizeof(float));
        return;
    }
    size_t processed = 0;
    while (processed < len) {
        bool input_buffer_was_empty = input_buffer_fill == 0;
        size_t processing = std::min(len - processed, block_size - input_buffer_fill);
        size_t input_buffer_pos = input_buffer_fill;
        std::memcpy(input_buffer.data() + input_buffer_pos, input + processed, processing * sizeof(float));
        // forward FFT of the (partially filled, zero padded) input block
        std::memcpy(fft_buffer.data(), input_buffer.data(), block_size * sizeof(float));
        std::fill(fft_buffer.begin() + block_size, fft_buffer.end(), 0.f);
        fft.forward(fft_buffer.data(), segments[current].data());
        // complex multiplication
        if (input_buffer_was_empty) {
            std::fill(pre_multiplied.begin(), pre_multiplied.end(), cf32(0.f, 0.f));
            for (size_t i = 1; i < seg_count; i++) {
                size_t index_ir = i;
                size_t index_audio = (current + i) % seg_count;
                complex_multiply_accumulate(pre_multiplied, segments_ir[index_ir], segments[index_audio]);
            }
        }
        conv = pre_multiplied;
        complex_multiply_accumulate(conv, segments[current], segments_ir[0]);
        // backward FFT (realfft is unnormalised: scale by 1/seg_size)
        fft.inverse(conv.data(), fft_buffer.data());
        float scale = 1.f / (float)seg_size;
        for (size_t i = 0; i < seg_size; i++) fft_buffer[i] *= scale;
        // add overlap
        for (size_t i = 0; i < processing; i++)
            output[processed + i] = fft_buffer[input_buffer_pos + i] + overlap[input_buffer_pos + i];
        // input buffer full => next block
        input_buffer_fill += processing;
        if (input_buffer_fill == block_size) {
            std::fill(input_buffer.begin(), input_buffer.end(), 0.f);
            input_buffer_fill = 0;
            std::memcpy(overlap.data(), fft_buffer.data() + block_size, block_size * sizeof(float));
            current = current > 0 ? current - 1 : seg_count - 1;
        }
        processed += processing;
    }
}

// convolver.rs:16-53
float convolver_normalize_buffer(const AudioBuffer& buffer) {
    float gain_calibration = 0.00125f;
    float gain_calibration_sample_rate = 44100.f;
    float min_power = 0.000125f;
    int number_of_channels = buffer.number_of_channels();
    size_t length = buffer.length();
    float sample_rate = buffer.sample_rate;
    float power = 0.f;
    for (auto& c : buffer.channels) {
        float s = 0.f;
        for (float v : c) s += v * v;
        power += s;
    }
    power = std::sqrt(power / (float)((size_t)number_of_channels * length));
    if (!std::isfinite(power) || std::isnan(power) || power < min_power) power = min_power;
    float scale = 1.f / power;
    scale *= gain_calibration;
    scale *= gain_calibration_sample_rate / sample_rate;
    if (number_of_channels == 4) scale *= 0.5f;
    return scale;
}

// convolver.rs:259-317
void ConvolverRenderer::set_buffer(const AudioBuffer& buffer, bool normalize) {
    float scale = normalize ? convolver_normalize_buffer(buffer) : 1.f;
    int number_of_channels = buffer.number_of_channels();
    size_t partition_size = RQ * 8;
    convolvers.clear();
    for (int index = 0; index < std::max(number_of_channels, 2); index++) {
        int channel = std::min(index, number_of_channels - 1);
        std::vector<float> scaled(buffer.length());
        for (size_t i = 0; i < scaled.size(); i++) scaled[i] = buffer.channels[channel][i] * scale;
        convolvers.emplace_back();
        convolvers.back().init(partition_size, scaled.data(), scaled.size());
    }
    has_convolvers = true;
    impulse_length = buffer.length();
    impulse_number_of_channels = number_of_channels;
}

// convolver.rs:343-490
bool ConvolverRenderer::process(std::vector<Quantum>& inputs, std::vector<Quantum>& outputs, const ParamValues&, const Scope&) {
    const Quantum& input = inputs[0];
    Quantum& output = outputs[0];
    if (input.is_silent()) {
        if (tail_count >= impulse_length) {
            output.make_silent();
            return false;
        }
        tail_count += RQ;
    } else {
        tail_count = 0;
    }
    if (!has_convolvers) {
        output = input;
        return !input.is_silent();
    }
    int in_ch = input.number_of_channels();
    int ir_ch = impulse_number_of_channels;
    auto run = [&](int conv, int in_channel, int out_channel) {
        Channel i = input.channel(in_channel);  // clone: output may share buffers with input
        float* o = output.channel_mut(out_channel).make_mut();
        convolvers[conv].process(i.data(), o, RQ);
    };
    if (in_ch == 1 && ir_ch == 1) {
        output.set_number_of_channels(1);
        run(0, 0, 0);
    } else if (in_ch == 1 && ir_ch == 2) {
        output.set_number_of_channels(2);
        run(0, 0, 0);
        run(1, 0, 1);
    } else if (in_ch == 2 && (ir_ch == 1 || ir_ch == 2)) {
        output.set_number_of_channels(2);
        run(0, 0, 0);
        run(1, 1, 1);
    } else if (ir_ch == 4 && (in_ch == 2 || in_ch == 1)) {
        output.set_number_of_channels(4);
        if (in_ch == 2) {
            run(0, 0, 0);
            run(1, 0, 1);
            run(2, 1, 2);
            run(3, 1, 3);
        } else {
            run(0, 0, 0);
            run(1, 0, 1);
            run(2, 0, 2);
            run(3, 0, 3);
        }
        Channel o2 = output.channel(2), o3 = output.channel(3);
        float* l = output.channel_mut(0).make_mut();
        for (int i = 0; i < RQ; i++) l[i] += o2.data()[i];
        float* r = output.channel_mut(1).make_mut();
        for (int i = 0; i < RQ; i++) r[i] += o3.data()[i];
        output.set_number_of_channels(2);
    }
    return true;
}

}  // namespace wao
