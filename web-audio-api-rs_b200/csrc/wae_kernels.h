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

void upload_twiddles();                          // convolver FFT tables (computed in wae_kernels.cu, f64 -> f32)
void conv_fft_selftest(float* data, int mode);   // host emulation of the convolver transforms (wae_selftest_conv_fft)
void launch_oscillator(const OscInst* d, int n, ChunkInfo ci, cudaStream_t s);
void launch_constant(const ConstInst* d, int n, ChunkInfo ci, cudaStream_t s);
void launch_buffer_source(const AbsnInst* d, int n, ChunkInfo ci, cudaStream_t s);
void launch_buffer_source_slow(const AbsnSlowInst* d, int n, ChunkInfo ci, cudaStream_t s);
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
void launch_compressor(const CompInst* d, int n, ChunkInfo ci, cudaStream_t s);
void launch_analyser(const AnalyserInst* d, int n, ChunkInfo ci, cudaStream_t s);
void launch_conv_fft_in(const ConvInput* d, int n, ChunkInfo ci, cudaStream_t s);
void launch_conv_mac_ifft(const ConvPath* p, const ConvInput* in, int n, ChunkInfo ci, cudaStream_t s);
void launch_conv_compact(const ConvCmpInst* d, int n, ChunkInfo ci, cudaStream_t s);
// one launch for all items of a bind call; max_vec = the largest slot stride / 4, max_ch = the most channels of an item
void launch_bind_sources(const BindItem* d, int n, int64_t max_vec, int max_ch, cudaStream_t s);
void launch_conv_ir_fft(const float* ir, int64_t ir_len, int64_t ir_stride, float2* h, int S, int channels, cudaStream_t s);

}  // namespace wae
