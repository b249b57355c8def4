// C ABI, graph-construction half (include/wae.h): OfflineAudioContext::new, create_*, connect, AudioParam
// events, start/stop.  Mirrors the control side of the reference (file:line cited per function); argument
// validation returns the reference's panic text through wae_last_error().
#include "wae_graph.h"
#include "wae_hostmath.h"
#include "wae_hrtf_host.h"
#include "wae_kernels.h"
#include "wae_param_core.h"
#include "wae_param_host.h"
#include "wae_param_walk.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <complex>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <unordered_map>

using namespace wae;

namespace wae {
static thread_local std::string g_err;
void set_error(const std::string& msg) { g_err = msg; }
int32_t fail(int32_t code, const std::string& msg) {
    g_err = msg;
    return code;
}

// ---- page-locked pool of AudioBuffer memory (see PcmBuffer) ---------------------------------------------------------------
// Slabs of cudaHostAlloc(Portable) memory, carved by bump allocation; freed blocks are recycled by exact (64 KiB-rounded) size,
// which is what a caller that builds the same kind of graphs again and again produces.  Page-locking costs ~0.3 ms per MiB and
// happens once per slab, at graph-construction time; the slabs live as long as the process.
namespace {
struct PinnedPool {
    std::mutex mu;
    struct Slab {
        char* base;
        size_t size, used;
    };
    std::vector<Slab> slabs;
    std::unordered_map<size_t, std::vector<void*>> free_by_size;
    bool disabled = false;  // no CUDA device / page-locking refused: stop trying
    static size_t round(size_t b) { return (b + 65535) / 65536 * 65536; }
    void* alloc(size_t bytes) {
        const size_t r = round(bytes);
        std::lock_guard<std::mutex> lk(mu);
        if (disabled) return nullptr;
        auto it = free_by_size.find(r);
        if (it != free_by_size.end() && !it->second.empty()) {
            void* p = it->second.back();
            it->second.pop_back();
            return p;
        }
        for (auto& s : slabs)
            if (s.size - s.used >= r) {
                void* p = s.base + s.used;
                s.used += r;
                return p;
            }
        const size_t slab_bytes = std::max<size_t>(r, (size_t)256 << 20);
        void* hp = nullptr;
        if (cudaHostAlloc(&hp, slab_bytes, cudaHostAllocPortable) != cudaSuccess) {
            cudaGetLastError();
            if (slab_bytes == r || cudaHostAlloc(&hp, r, cudaHostAllocPortable) != cudaSuccess) {
                cudaGetLastError();
                disabled = slabs.empty();
                return nullptr;
            }
            slabs.push_back(Slab{(char*)hp, r, r});
            return hp;
        }
        slabs.push_back(Slab{(char*)hp, slab_bytes, r});
        return hp;
    }
    void free(void* p, size_t bytes) {
        std::lock_guard<std::mutex> lk(mu);
        free_by_size[round(bytes)].push_back(p);
    }
};
PinnedPool& pinned_pool() {
    static PinnedPool* pool = new PinnedPool;  // never destroyed: buffers may outlive static destruction order
    return *pool;
}
}  // namespace

void* pcm_host_alloc(size_t bytes, bool want_pinned, bool* pinned) {
    *pinned = false;
    if (want_pinned && bytes >= ((size_t)256 << 10)) {
        if (void* p = pinned_pool().alloc(bytes)) {
            *pinned = true;
            return p;
        }
    }
    return std::malloc(bytes);
}
void pcm_host_free(void* p, size_t bytes, bool pinned) {
    if (pinned) pinned_pool().free(p, bytes);
    else std::free(p);
}

// AudioParamProcessor::handle_incoming_event for SetValue (src/param.rs:987-990) + mix_to_output clamp (:755-760)
bool Param::constant() const {
    for (auto& e : events)
        if (e.type != WAE_EVENT_SET_VALUE) return false;
    return true;
}
float Param::constant_value() const {
    float v = default_value;
    for (auto& e : events)
        if (e.type == WAE_EVENT_SET_VALUE) v = e.value;
    if (std::isnan(v)) return default_value;
    v = v > min_value ? v : min_value;
    v = v < max_value ? v : max_value;
    if (device_bound) {  // the placeholder a bound param is planned with
        v = v > device_lo ? v : device_lo;
        v = v < device_hi ? v : device_hi;
    }
    return v;
}
}  // namespace wae

static const float F32_MAX = 3.40282347e+38f;

// BaseAudioContext::create_audio_param, src/context/base.rs:320-337
uint32_t wae_graph::create_param(uint32_t owner, float def, float mn, float mx, bool a_rate, float initial, bool send_set_value,
                                 bool fixed_id, uint32_t id, bool constrained) {
    uint32_t pid = fixed_id ? id : next_id++;
    Node n;
    n.id = pid;
    n.kind = K_PARAM;
    n.out_id = pid;
    n.cfg = ChannelCfg{1, WAE_COUNT_MODE_EXPLICIT, WAE_INTERPRETATION_DISCRETE};  // src/param.rs:296-310
    n.param = Param{def, mn, mx, a_rate, constrained, {}};
    if (send_set_value) n.param.events.push_back(ParamEv{WAE_EVENT_SET_VALUE, initial, 0., 0., {}});
    nodes[pid] = std::move(n);
    pending_param_edges.push_back({pid, owner});
    return pid;
}

// tail of ConcreteBaseAudioContext::register (src/context/concrete_base.rs:232-270)
Node& wae_graph::finish_register(Node n) {
    uint32_t id = n.id;
    nodes[id] = std::move(n);
    for (auto& e : pending_param_edges)
        if (e.second == id) add_edge(e.first, 0, e.second, -1);
    pending_param_edges.erase(
        std::remove_if(pending_param_edges.begin(), pending_param_edges.end(), [&](auto& e) { return e.second == id; }),
        pending_param_edges.end());
    return nodes[id];
}

// ensure_audio_listener_present, src/context/concrete_base.rs:516-534 + AudioListenerNode::new (src/spatial.rs:117-170)
void wae_graph::ensure_listener() {
    if (listener_present) return;
    listener_present = true;
    static const float defaults[9] = {0.f, 0.f, 0.f, 0.f, 0.f, -1.f, 0.f, 1.f, 0.f};
    Node l;
    l.id = 1;
    l.kind = K_LISTENER;
    l.out_id = 1;
    l.n_inputs = 0;
    l.n_outputs = 9;
    l.cfg = ChannelCfg{1, WAE_COUNT_MODE_EXPLICIT, WAE_INTERPRETATION_DISCRETE};
    for (int i = 0; i < 9; i++) l.params.push_back(create_param(1, defaults[i], -F32_MAX, F32_MAX, true, defaults[i], false, true, 2 + i));
    finish_register(std::move(l));
    add_edge(1, 0, 0, -1);
}

static ChannelCfg resolve_cfg(const wae_channel_config& c, ChannelCfg def) {
    if (c.count == 0) return def;
    return ChannelCfg{(int)c.count, (int)c.count_mode, (int)c.interpretation};
}
// a caller-supplied ChannelConfig: assert_valid_number_of_channels (src/lib.rs:185-192) and the two enums of include/wae.h
static wae_status check_cfg(const wae_channel_config& c) {
    if (c.count == 0) return WAE_OK;  // "use the node's default"
    if (c.count > WAE_MAX_CHANNELS)
        return fail(WAE_NOT_SUPPORTED, "NotSupportedError - Invalid number of channels: " + std::to_string(c.count) + " is outside range [1, 32]");
    if (c.count_mode > WAE_COUNT_MODE_EXPLICIT) return fail(WAE_INVALID_ARGUMENT, "unknown channel count mode");
    if (c.interpretation > WAE_INTERPRETATION_DISCRETE) return fail(WAE_INVALID_ARGUMENT, "unknown channel interpretation");
    return WAE_OK;
}

// `pin`: the buffer will be DMA-ed to a device by a render call (AudioBufferSourceNode assets of a graph that has an engine)
static std::shared_ptr<PcmBuffer> copy_buffer(wae_graph* g, const wae_audio_buffer* b, bool pin) {
    // AudioBuffer::new (src/buffer.rs:96-115): assert_valid_number_of_channels / assert_valid_buffer_length
    if (b->number_of_channels < 1 || b->number_of_channels > WAE_MAX_CHANNELS || !b->channels) {
        fail(WAE_NOT_SUPPORTED, "NotSupportedError - Invalid number of channels: " + std::to_string(b->number_of_channels) + " is outside range [1, 32]");
        return nullptr;
    }
    if (b->length == 0) {
        fail(WAE_NOT_SUPPORTED, "NotSupportedError - Invalid length: 0 is less than or equal to minimum bound (0)");
        return nullptr;
    }
    // the same PCM again (same shape, same samples): share the copy the graph already holds.  PcmBuffers are never written after this
    // function; only shape-equal candidates are compared, newest first, and memcmp stops at the first difference — a graph with one
    // buffer (C2) pays nothing, one with a hundred different buffers a few cache lines per candidate
    auto& assets = g->assets[pin ? 1 : 0];
    {
        int looked = 0;
        for (size_t i = assets.size(); i-- > 0 && looked < 16;) {
            std::shared_ptr<PcmBuffer> have = assets[i].lock();
            if (!have || have->channels.size() != b->number_of_channels || have->length() != b->length || have->sample_rate != b->sample_rate) continue;
            looked++;
            bool same = true;
            for (uint32_t c = 0; c < b->number_of_channels && same; c++)
                same = std::memcmp(have->channels[c].data(), b->channels[c], (size_t)b->length * sizeof(float)) == 0;
            if (same) return have;
        }
    }
    auto p = std::make_shared<PcmBuffer>();
    p->sample_rate = b->sample_rate;
    bool want = pin && g->engine != nullptr;
    if (want && cudaSetDevice(engine_device(g->engine)) != cudaSuccess) {
        cudaGetLastError();
        want = false;
    }
    if (!p->allocate(b->number_of_channels, b->length, want)) {
        fail(WAE_OUT_OF_MEMORY, "out of host memory (AudioBuffer copy)");
        return nullptr;
    }
    for (uint32_t c = 0; c < b->number_of_channels; c++) std::memcpy(p->channels[c].data(), b->channels[c], (size_t)b->length * sizeof(float));
    if (assets.size() >= 64 && (assets.size() & (assets.size() - 1)) == 0) {  // at 64, 128, ...: drop the entries whose buffer is gone
        size_t w = 0;
        for (auto& a : assets)
            if (!a.expired()) assets[w++] = a;
        assets.resize(w);
    }
    assets.push_back(p);
    return p;
}

extern "C" {

WAE_API const char* wae_last_error(void) { return g_err.c_str(); }
WAE_API const char* wae_version(void) { return "wae-b200 0.1 (sm_90a)"; }

// OfflineAudioContext::new, src/context/offline.rs:78-105
WAE_API wae_status wae_graph_create(wae_engine* engine, uint32_t number_of_channels, uint64_t length, float sample_rate,
                                    wae_graph** out) {
    if (!out) return fail(WAE_INVALID_ARGUMENT, "null out pointer");  // a NULL engine is fine: planning and rendering name their own
    if (number_of_channels < 1 || number_of_channels > WAE_MAX_CHANNELS)
        return fail(WAE_NOT_SUPPORTED, "NotSupportedError - Invalid number of channels");
    if (length == 0) return fail(WAE_NOT_SUPPORTED, "NotSupportedError - Invalid length: 0");
    if (!(sample_rate >= 3000.f && sample_rate <= 768000.f)) return fail(WAE_NOT_SUPPORTED, "NotSupportedError - Invalid sample rate");
    auto* g = new wae_graph;
    g->engine = engine;
    g->channels = number_of_channels;
    g->length = length;
    g->sample_rate = sample_rate;
    Node d;  // AudioDestinationNode::new, src/node/destination.rs:100-117
    d.id = 0;
    d.kind = K_DEST;
    d.cfg = ChannelCfg{(int)number_of_channels, WAE_COUNT_MODE_EXPLICIT, WAE_INTERPRETATION_SPEAKERS};
    g->finish_register(std::move(d));
    *out = g;
    return WAE_OK;
}

WAE_API wae_status wae_graph_destroy(wae_graph* g) {
    delete g;
    return WAE_OK;
}

// OscillatorNode::new, src/node/oscillator.rs:211-275
WAE_API wae_status wae_create_oscillator(wae_graph* g, const wae_oscillator_options* o, wae_node_id* out) {
    if (!g || !o || !out) return fail(WAE_INVALID_ARGUMENT, "null graph / options / out pointer");
    if (o->type > WAE_OSC_CUSTOM) return fail(WAE_INVALID_ARGUMENT, "invalid oscillator type");
    if (o->type == WAE_OSC_CUSTOM && (!o->periodic_wave || o->periodic_wave_len == 0))
        return fail(WAE_INVALID_ARGUMENT, "custom oscillator needs a periodic wave table");
    Node n;
    n.id = g->next_id++;
    n.out_id = n.id;
    n.kind = K_OSC;
    n.n_inputs = 0;
    n.type = (int)o->type;
    float nyquist = g->sample_rate / 2.f;
    n.params.push_back(g->create_param(n.id, 440.f, -nyquist, nyquist, true, o->frequency));
    n.params.push_back(g->create_param(n.id, 0.f, -153600.f, 153600.f, true, o->detune));
    if (o->type == WAE_OSC_CUSTOM) n.table.assign(o->periodic_wave, o->periodic_wave + o->periodic_wave_len);
    *out = g->finish_register(std::move(n)).id;
    return WAE_OK;
}

// BiquadFilterNode::new, src/node/biquad_filter.rs:542-608
WAE_API wae_status wae_create_biquad_filter(wae_graph* g, const wae_biquad_options* o, wae_node_id* out) {
    if (!g || !o || !out) return fail(WAE_INVALID_ARGUMENT, "null graph / options / out pointer");
    if (o->type > 7) return fail(WAE_INVALID_ARGUMENT, "invalid biquad type");
    Node n;
    n.id = g->next_id++;
    n.out_id = n.id;
    n.kind = K_BIQUAD;
    n.type = (int)o->type;
    if (wae_status cs = check_cfg(o->channel_config)) return cs;
    n.cfg = resolve_cfg(o->channel_config, ChannelCfg());
    n.params.push_back(g->create_param(n.id, 1.f, -F32_MAX, F32_MAX, true, o->q));
    n.params.push_back(g->create_param(n.id, 0.f, -153600.f, 153600.f, true, o->detune));
    n.params.push_back(g->create_param(n.id, 350.f, 0.f, g->sample_rate / 2.f, true, o->frequency));
    n.params.push_back(g->create_param(n.id, 0.f, -F32_MAX, 40.f * log10f(F32_MAX), true, o->gain));
    *out = g->finish_register(std::move(n)).id;
    return WAE_OK;
}

// IIRFilterNode::new, src/node/iir_filter.rs:146-205
WAE_API wae_status wae_create_iir_filter(wae_graph* g, const wae_iir_options* o, wae_node_id* out) {
    if (!g || !o || !out) return fail(WAE_INVALID_ARGUMENT, "null graph / options / out pointer");
    if (o->feedforward_len == 0 || o->feedforward_len > 20) return fail(WAE_NOT_SUPPORTED, "NotSupportedError - invalid feedforward length");
    if (o->feedback_len == 0 || o->feedback_len > 20) return fail(WAE_NOT_SUPPORTED, "NotSupportedError - invalid feedback length");
    bool all_zero = true;
    for (uint32_t i = 0; i < o->feedforward_len; i++)
        if (o->feedforward[i] != 0.) all_zero = false;
    if (all_zero) return fail(WAE_INVALID_STATE, "InvalidStateError - all feedforward coefficients are zero");
    if (o->feedback[0] == 0.) return fail(WAE_INVALID_STATE, "InvalidStateError - first feedback coefficient is zero");
    Node n;
    n.id = g->next_id++;
    n.out_id = n.id;
    n.kind = K_IIR;
    if (wae_status cs = check_cfg(o->channel_config)) return cs;
    n.cfg = resolve_cfg(o->channel_config, ChannelCfg());
    n.feedforward.assign(o->feedforward, o->feedforward + o->feedforward_len);
    n.feedback.assign(o->feedback, o->feedback + o->feedback_len);
    *out = g->finish_register(std::move(n)).id;
    return WAE_OK;
}

// GainNode::new, src/node/gain.rs:86-117
WAE_API wae_status wae_create_gain(wae_graph* g, const wae_gain_options* o, wae_node_id* out) {
    if (!g || !o || !out) return fail(WAE_INVALID_ARGUMENT, "null graph / options / out pointer");
    Node n;
    n.id = g->next_id++;
    n.out_id = n.id;
    n.kind = K_GAIN;
    if (wae_status cs = check_cfg(o->channel_config)) return cs;
    n.cfg = resolve_cfg(o->channel_config, ChannelCfg());
    n.params.push_back(g->create_param(n.id, 1.f, -F32_MAX, F32_MAX, true, o->gain));
    *out = g->finish_register(std::move(n)).id;
    return WAE_OK;
}

// AudioBufferSourceNode::new, src/node/audio_buffer_source.rs:160-235
WAE_API wae_status wae_create_buffer_source(wae_graph* g, const wae_buffer_source_options* o, wae_node_id* out) {
    if (!g || !o || !out) return fail(WAE_INVALID_ARGUMENT, "null graph / options / out pointer");
    Node n;
    n.id = g->next_id++;
    n.out_id = n.id;
    n.kind = K_ABSN;
    n.n_inputs = 0;
    n.params.push_back(g->create_param(n.id, 0.f, -F32_MAX, F32_MAX, false, o->detune, true, false, 0, true));
    n.params.push_back(g->create_param(n.id, 1.f, -F32_MAX, F32_MAX, false, o->playback_rate, true, false, 0, true));
    n.loop = o->loop != 0;
    n.loop_start = o->loop_start;
    n.loop_end = o->loop_end;
    if (o->buffer && !(n.buffer = copy_buffer(g, o->buffer, true))) return WAE_NOT_SUPPORTED;
    *out = g->finish_register(std::move(n)).id;
    return WAE_OK;
}

// ConstantSourceNode::new, src/node/constant_source.rs:138-170
WAE_API wae_status wae_create_constant_source(wae_graph* g, const wae_constant_source_options* o, wae_node_id* out) {
    if (!g || !o || !out) return fail(WAE_INVALID_ARGUMENT, "null graph / options / out pointer");
    Node n;
    n.id = g->next_id++;
    n.out_id = n.id;
    n.kind = K_CONST;
    n.n_inputs = 0;
    n.params.push_back(g->create_param(n.id, 1.f, -F32_MAX, F32_MAX, true, o->offset));
    *out = g->finish_register(std::move(n)).id;
    return WAE_OK;
}

// ConvolverNode::new + set_buffer, src/node/convolver.rs:199-317
WAE_API wae_status wae_create_convolver(wae_graph* g, const wae_convolver_options* o, wae_node_id* out) {
    if (!g || !o || !out) return fail(WAE_INVALID_ARGUMENT, "null graph / options / out pointer");
    if (wae_status cs = check_cfg(o->channel_config)) return cs;
    ChannelCfg cfg = resolve_cfg(o->channel_config, ChannelCfg{2, WAE_COUNT_MODE_CLAMPED_MAX, WAE_INTERPRETATION_SPEAKERS});
    if (cfg.count > 2) return fail(WAE_NOT_SUPPORTED, "NotSupportedError - ConvolverNode channel count cannot be greater than two");
    if (cfg.mode == WAE_COUNT_MODE_MAX) return fail(WAE_NOT_SUPPORTED, "NotSupportedError - ConvolverNode channel count mode cannot be set to max");
    if (o->buffer) {
        if (o->buffer->sample_rate != g->sample_rate)
            return fail(WAE_NOT_SUPPORTED, "NotSupportedError - sample rate of the convolution buffer must match the audio context");
        uint32_t c = o->buffer->number_of_channels;
        if (!(c == 1 || c == 2 || c == 4))
            return fail(WAE_NOT_SUPPORTED, "NotSupportedError - the convolution buffer must consist of 1, 2 or 4 channels");
    }
    Node n;
    n.id = g->next_id++;
    n.out_id = n.id;
    n.kind = K_CONV;
    n.cfg = cfg;
    n.normalize = n.normalize_next = !o->disable_normalization;
    if (o->buffer && !(n.buffer = copy_buffer(g, o->buffer, false))) return WAE_NOT_SUPPORTED;
    *out = g->finish_register(std::move(n)).id;
    return WAE_OK;
}

// WaveShaperNode::new, src/node/waveshaper.rs:190-260
WAE_API wae_status wae_create_wave_shaper(wae_graph* g, const wae_wave_shaper_options* o, wae_node_id* out) {
    if (!g || !o || !out) return fail(WAE_INVALID_ARGUMENT, "null graph / options / out pointer");
    if (o->oversample > WAE_OVERSAMPLE_X4) return fail(WAE_INVALID_ARGUMENT, "unknown oversample type");
    Node n;
    n.id = g->next_id++;
    n.out_id = n.id;
    n.kind = K_SHAPER;
    n.oversample = (int)o->oversample;
    if (wae_status cs = check_cfg(o->channel_config)) return cs;
    n.cfg = resolve_cfg(o->channel_config, ChannelCfg());
    if (o->curve) {
        n.has_curve = true;
        n.table.assign(o->curve, o->curve + o->curve_len);
    }
    *out = g->finish_register(std::move(n)).id;
    return WAE_OK;
}

// DelayNode::new, src/node/delay.rs:283-368: writer N, reader N+1, delayTime N+2
WAE_API wae_status wae_create_delay(wae_graph* g, const wae_delay_options* o, wae_node_id* out) {
    if (!g || !o || !out) return fail(WAE_INVALID_ARGUMENT, "null graph / options / out pointer");
    if (!(o->max_delay_time > 0. && o->max_delay_time < 180.))
        return fail(WAE_NOT_SUPPORTED, "NotSupportedError - maxDelayTime MUST be greater than zero and less than three minutes");
    if (wae_status cs = check_cfg(o->channel_config)) return cs;
    ChannelCfg cfg = resolve_cfg(o->channel_config, ChannelCfg());
    uint32_t writer_id = g->next_id++;
    uint32_t reader_id = g->next_id++;
    Node r;
    r.id = reader_id;
    r.out_id = reader_id;
    r.kind = K_DELAY_R;
    r.cfg = cfg;
    r.max_delay_time = o->max_delay_time;
    r.delay_peer = writer_id;
    r.params.push_back(g->create_param(reader_id, 0.f, 0.f, (float)o->max_delay_time, true, (float)o->delay_time));
    uint32_t p = r.params[0];
    g->finish_register(std::move(r));
    Node w;
    w.id = writer_id;
    w.out_id = reader_id;
    w.kind = K_DELAY_W;
    w.cfg = cfg;
    w.max_delay_time = o->max_delay_time;
    w.delay_peer = reader_id;
    w.params.push_back(p);
    w.cycle_breaker = true;
    g->finish_register(std::move(w));
    g->add_edge(writer_id, 0, reader_id, 0);
    *out = writer_id;
    return WAE_OK;
}

// StereoPannerNode::new, src/node/stereo_panner.rs:163-200
WAE_API wae_status wae_create_stereo_panner(wae_graph* g, const wae_stereo_panner_options* o, wae_node_id* out) {
    if (!g || !o || !out) return fail(WAE_INVALID_ARGUMENT, "null graph / options / out pointer");
    if (wae_status cs = check_cfg(o->channel_config)) return cs;
    ChannelCfg cfg = resolve_cfg(o->channel_config, ChannelCfg{2, WAE_COUNT_MODE_CLAMPED_MAX, WAE_INTERPRETATION_SPEAKERS});
    if (cfg.mode == WAE_COUNT_MODE_MAX) return fail(WAE_NOT_SUPPORTED, "NotSupportedError - StereoPannerNode channel count mode cannot be set to max");
    if (cfg.count > 2) return fail(WAE_NOT_SUPPORTED, "NotSupportedError - StereoPannerNode channel count cannot be greater than two");
    Node n;
    n.id = g->next_id++;
    n.out_id = n.id;
    n.kind = K_SPANNER;
    n.cfg = cfg;
    n.params.push_back(g->create_param(n.id, 0.f, -1.f, 1.f, true, o->pan));
    *out = g->finish_register(std::move(n)).id;
    return WAE_OK;
}

// PannerNode::new, src/node/panner.rs:392-520
WAE_API wae_status wae_create_panner(wae_graph* g, const wae_panner_options* o, wae_node_id* out) {
    if (!g || !o || !out) return fail(WAE_INVALID_ARGUMENT, "null graph / options / out pointer");
    if (wae_status cs = check_cfg(o->channel_config)) return cs;
    ChannelCfg cfg = resolve_cfg(o->channel_config, ChannelCfg{2, WAE_COUNT_MODE_CLAMPED_MAX, WAE_INTERPRETATION_SPEAKERS});
    if (cfg.mode == WAE_COUNT_MODE_MAX) return fail(WAE_NOT_SUPPORTED, "NotSupportedError - PannerNode channel count mode cannot be set to max");
    if (cfg.count > 2) return fail(WAE_NOT_SUPPORTED, "NotSupportedError - PannerNode channel count cannot be greater than two");
    if (o->ref_distance < 0.) return fail(WAE_INVALID_ARGUMENT, "RangeError - refDistance cannot be negative");
    if (o->max_distance <= 0.) return fail(WAE_INVALID_ARGUMENT, "RangeError - maxDistance must be strictly positive");
    if (o->rolloff_factor < 0.) return fail(WAE_INVALID_ARGUMENT, "RangeError - rolloffFactor cannot be negative");
    if (o->cone_outer_gain < 0. || o->cone_outer_gain > 1.) return fail(WAE_INVALID_STATE, "InvalidStateError - coneOuterGain must be in the range [0, 1]");
    Node n;
    n.id = g->next_id++;
    n.out_id = n.id;
    n.kind = K_PANNER;
    n.cfg = cfg;
    n.panning_model = (int)o->panning_model;
    n.distance_model = (int)o->distance_model;
    n.ref_distance = o->ref_distance;
    n.max_distance = o->max_distance;
    n.rolloff_factor = o->rolloff_factor;
    n.cone_inner_angle = o->cone_inner_angle;
    n.cone_outer_angle = o->cone_outer_angle;
    n.cone_outer_gain = o->cone_outer_gain;
    g->ensure_listener();
    const float init[6] = {o->position_x, o->position_y, o->position_z, o->orientation_x, o->orientation_y, o->orientation_z};
    for (int i = 0; i < 6; i++) n.params.push_back(g->create_param(n.id, i == 3 ? 1.f : 0.f, -F32_MAX, F32_MAX, true, init[i]));
    uint32_t id = g->finish_register(std::move(n)).id;
    g->add_edge(1, 0, id, -1);  // connect_listener_to_panner, concrete_base.rs:511-513
    *out = id;
    return WAE_OK;
}

// AnalyserNode::new, src/node/analyser.rs:130-175 (asserts of src/analysis.rs:33-72)
WAE_API wae_status wae_create_analyser(wae_graph* g, const wae_analyser_options* o, wae_node_id* out) {
    if (!g || !o || !out) return fail(WAE_INVALID_ARGUMENT, "null graph / options / out pointer");
    uint32_t fft = o->fft_size ? o->fft_size : 2048;
    if ((fft & (fft - 1)) != 0) return fail(WAE_INVALID_ARGUMENT, "IndexSizeError - Invalid fft size: not a power of two");
    if (fft < 32 || fft > 32768) return fail(WAE_INVALID_ARGUMENT, "IndexSizeError - Invalid fft size: outside range [32, 32768]");
    double stc = o->fft_size ? o->smoothing_time_constant : 0.8;
    if (!(stc >= 0. && stc <= 1.)) return fail(WAE_INVALID_ARGUMENT, "IndexSizeError - Invalid smoothing time constant");
    double mn = o->fft_size ? o->min_decibels : -100., mx = o->fft_size ? o->max_decibels : -30.;
    if (!(mn < mx)) return fail(WAE_INVALID_ARGUMENT, "IndexSizeError - Invalid min decibels");
    Node n;
    n.id = g->next_id++;
    n.out_id = n.id;
    n.kind = K_ANALYSER;
    if (wae_status cs = check_cfg(o->channel_config)) return cs;
    n.cfg = resolve_cfg(o->channel_config, ChannelCfg());
    n.fft_size = fft;
    n.smoothing = stc;
    n.min_db = mn;
    n.max_db = mx;
    *out = g->finish_register(std::move(n)).id;
    return WAE_OK;
}

// DynamicsCompressorNode::new, src/node/dynamics_compressor.rs:130-260
WAE_API wae_status wae_create_dynamics_compressor(wae_graph* g, const wae_dynamics_compressor_options* o, wae_node_id* out) {
    if (!g || !o || !out) return fail(WAE_INVALID_ARGUMENT, "null graph / options / out pointer");
    if (wae_status cs = check_cfg(o->channel_config)) return cs;
    ChannelCfg cfg = resolve_cfg(o->channel_config, ChannelCfg{2, WAE_COUNT_MODE_CLAMPED_MAX, WAE_INTERPRETATION_SPEAKERS});
    if (cfg.count > 2) return fail(WAE_NOT_SUPPORTED, "NotSupportedError - DynamicsCompressorNode channel count cannot be greater than two");
    if (cfg.mode == WAE_COUNT_MODE_MAX) return fail(WAE_NOT_SUPPORTED, "NotSupportedError - DynamicsCompressorNode channel count mode cannot be set to max");
    Node n;
    n.id = g->next_id++;
    n.out_id = n.id;
    n.kind = K_COMP;
    n.cfg = cfg;
    n.params.push_back(g->create_param(n.id, 0.003f, 0.f, 1.f, false, o->attack, true, false, 0, true));
    n.params.push_back(g->create_param(n.id, 30.f, 0.f, 40.f, false, o->knee, true, false, 0, true));
    n.params.push_back(g->create_param(n.id, 12.f, 1.f, 20.f, false, o->ratio, true, false, 0, true));
    n.params.push_back(g->create_param(n.id, 0.25f, 0.f, 1.f, false, o->release, true, false, 0, true));
    n.params.push_back(g->create_param(n.id, -24.f, -100.f, 0.f, false, o->threshold, true, false, 0, true));
    *out = g->finish_register(std::move(n)).id;
    return WAE_OK;
}

// ChannelMergerNode::new, src/node/channel_merger.rs:120-140
WAE_API wae_status wae_create_channel_merger(wae_graph* g, const wae_channel_merger_options* o, wae_node_id* out) {
    if (!g || !o || !out) return fail(WAE_INVALID_ARGUMENT, "null graph / options / out pointer");
    uint32_t k = o->number_of_inputs ? o->number_of_inputs : 6;
    if (k < 1 || k > WAE_MAX_CHANNELS) return fail(WAE_INVALID_ARGUMENT, "IndexSizeError - Invalid number of inputs");
    Node n;
    n.id = g->next_id++;
    n.out_id = n.id;
    n.kind = K_MERGER;
    n.n_inputs = (int)k;
    n.cfg = ChannelCfg{1, WAE_COUNT_MODE_EXPLICIT, WAE_INTERPRETATION_SPEAKERS};
    *out = g->finish_register(std::move(n)).id;
    return WAE_OK;
}

// ChannelSplitterNode::new, src/node/channel_splitter.rs:140-180
WAE_API wae_status wae_create_channel_splitter(wae_graph* g, const wae_channel_splitter_options* o, wae_node_id* out) {
    if (!g || !o || !out) return fail(WAE_INVALID_ARGUMENT, "null graph / options / out pointer");
    uint32_t k = o->number_of_outputs ? o->number_of_outputs : 6;
    if (k < 1 || k > WAE_MAX_CHANNELS) return fail(WAE_INVALID_ARGUMENT, "IndexSizeError - Invalid number of outputs");
    Node n;
    n.id = g->next_id++;
    n.out_id = n.id;
    n.kind = K_SPLITTER;
    n.n_outputs = (int)k;
    n.cfg = ChannelCfg{(int)k, WAE_COUNT_MODE_EXPLICIT, WAE_INTERPRETATION_DISCRETE};
    *out = g->finish_register(std::move(n)).id;
    return WAE_OK;
}

// AudioNode::connect_from_output_to_input, src/node/audio_node.rs:259-289
WAE_API wae_status wae_connect(wae_graph* g, wae_node_id from, uint32_t output, wae_node_id to, uint32_t input) {
    auto fi = g->nodes.find(from), ti = g->nodes.find(to);
    if (fi == g->nodes.end() || ti == g->nodes.end() || fi->second.kind == K_PARAM || ti->second.kind == K_PARAM)
        return fail(WAE_INVALID_ARGUMENT, "InvalidAccessError - unknown node");
    if ((int)output >= fi->second.n_outputs)
        return fail(WAE_INVALID_ARGUMENT, "IndexSizeError - output port " + std::to_string(output) + " is out of bounds");
    if ((int)input >= ti->second.n_inputs)
        return fail(WAE_INVALID_ARGUMENT, "IndexSizeError - input port " + std::to_string(input) + " is out of bounds");
    g->add_edge(fi->second.out_id, (int)output, to, (int)input);
    return WAE_OK;
}

WAE_API wae_status wae_connect_param(wae_graph* g, wae_node_id from, uint32_t output, wae_node_id to, uint32_t param_index) {
    if (to == 1) g->ensure_listener();  // BaseAudioContext::listener() creates it on first access (context/mod.rs)
    auto fi = g->nodes.find(from), ti = g->nodes.find(to);
    if (fi == g->nodes.end() || ti == g->nodes.end()) return fail(WAE_INVALID_ARGUMENT, "InvalidAccessError - unknown node");
    if ((int)output >= fi->second.n_outputs) return fail(WAE_INVALID_ARGUMENT, "IndexSizeError - output port out of bounds");
    if (param_index >= ti->second.params.size()) return fail(WAE_INVALID_ARGUMENT, "IndexSizeError - param index out of bounds");
    if (g->nodes.at(ti->second.params[param_index]).param.device_bound)
        return fail(WAE_INVALID_STATE, "InvalidStateError - the param's value is bound from device memory (wae_param_set_device_value): "
                                       "it takes no audio-rate input");
    g->add_edge(fi->second.out_id, (int)output, ti->second.params[param_index], 0);
    return WAE_OK;
}

// Params whose value stays constant over the render, so that a per-run value can be re-derived into the planned records (a GainNode's
// gain, a BiquadFilterNode's four, a StereoPannerNode's pan, a DynamicsCompressorNode's five, an AudioBufferSourceNode's detune and
// playbackRate: the planner picks the source's playback path from the declared range; an OscillatorNode's frequency and detune, whose
// computed frequencies the range keeps inside (0, sampleRate / 2): see osc_pitch_allowed; a PannerNode's position and orientation and the
// AudioListener's position, forward and up: no lowering decision reads their values, and kSpatialBound keeps their arithmetic finite)
static bool device_value_supported(Kind kind, uint32_t param_index) {
    switch (kind) {
        case K_GAIN: return param_index == 0;
        case K_BIQUAD: return param_index < 4;
        case K_SPANNER: return param_index == 0;
        case K_COMP: return param_index < 5;
        case K_ABSN: return param_index < 2;
        case K_OSC: return param_index < 2;
        case K_PANNER: return param_index < 6;
        case K_LISTENER: return param_index < 9;
        default: return false;
    }
}

// An oscillator's frequency (index 0) or detune (1) declared over [lo, hi]: the computed frequencies it allows, with the other param's
// declared range or current value, must all lie inside (0, sampleRate / 2), so that the planner's choice of path holds for every bound
// value.  Not needed while the other param is automated or driven at audio rate: the a-rate kernel takes the bound value raw.  The
// planner checks the rule again when it lowers the node (the other param may change after this call).
static bool osc_pitch_allowed(const wae_graph* g, const Node& n, uint32_t param_index, float lo, float hi, std::string& range) {
    const Param& other = g->nodes.at(n.params[1 - param_index]).param;
    if (!other.constant()) return true;
    for (const auto& kv : g->nodes)
        for (const Edge& e : kv.second.outgoing)
            if (e.other_id == n.params[1 - param_index]) return true;
    const float olo = other.device_bound ? other.device_lo : other.constant_value();
    const float ohi = other.device_bound ? other.device_hi : other.constant_value();
    const float f_lo = param_index == 0 ? lo : olo, f_hi = param_index == 0 ? hi : ohi;
    const float d_lo = param_index == 1 ? lo : olo, d_hi = param_index == 1 ? hi : ohi;
    range = "frequency [" + std::to_string(f_lo) + ", " + std::to_string(f_hi) + "] Hz, detune [" + std::to_string(d_lo) + ", " +
            std::to_string(d_hi) + "] cents";
    return hostmath::osc_pitch_inside(f_lo, f_hi, d_lo, d_hi, (double)g->sample_rate);
}

// A spatial param (a PannerNode's position / orientation, the AudioListener's position / forward / up) bound from device memory must keep
// its values inside [-kSpatialBound, kSpatialBound].  The spatial math is f32 (wae_spatial.h): it squares source - listener differences
// (up to 2 x the bound per axis) and the cross product of forward and up (up to 2 x bound^2 per axis), and 12 x (1e9)^4 = 1.2e37 still lies
// below FLT_MAX; wider values overflow to inf and the direction and gains the bind derives turn into NaN.  Metres, or unit vectors: a scene
// never comes near it, and the default range (the whole f32 line) is refused.
constexpr float kSpatialBound = 1e9f;

WAE_API wae_status wae_param_set_device_value(wae_graph* g, wae_node_id node, uint32_t param_index, float lo, float hi) {
    if (!g) return fail(WAE_INVALID_ARGUMENT, "null graph");
    if (node == 1) g->ensure_listener();  // BaseAudioContext::listener() creates it on first access (context/mod.rs)
    Node* n = g->nodes.get(node);
    if (!n || n->kind == K_PARAM || param_index >= n->params.size()) return fail(WAE_INVALID_ARGUMENT, "unknown param");
    if (!std::isfinite(lo) || !std::isfinite(hi) || lo > hi)
        return fail(WAE_INVALID_ARGUMENT, "device value range [" + std::to_string(lo) + ", " + std::to_string(hi) + "] is not a finite range");
    if (!device_value_supported(n->kind, param_index))
        return fail(WAE_UNSUPPORTED, "param " + std::to_string(param_index) + " of node " + std::to_string(node) +
                                         " cannot be bound from device memory (GainNode gain, BiquadFilterNode q / detune / frequency / gain, "
                                         "StereoPannerNode pan, DynamicsCompressorNode params, AudioBufferSourceNode detune / "
                                         "playbackRate, OscillatorNode frequency / detune, PannerNode position / orientation (0..5) and "
                                         "AudioListener position / forward / up (node 1, 0..8) can)");
    const uint32_t pid = n->params[param_index];
    Param& p = g->nodes.at(pid).param;
    if (p.device_bound) return fail(WAE_INVALID_STATE, "InvalidStateError - the param is already bound from device memory");
    if (!g->epochs.empty())  // (the segments before the suspend point were planned with the value of their own graph copy)
        return fail(WAE_INVALID_STATE, "InvalidStateError - a param is bound from device memory before the first suspend point");
    if (!p.constant()) return fail(WAE_INVALID_STATE, "InvalidStateError - the param has automation events");
    for (const auto& kv : g->nodes)
        for (const Edge& e : kv.second.outgoing)
            if (e.other_id == pid) return fail(WAE_INVALID_STATE, "InvalidStateError - the param has an audio-rate input (connect_param)");
    const float l = std::max(lo, p.min_value), h = std::min(hi, p.max_value);
    if (l > h) return fail(WAE_INVALID_ARGUMENT, "device value range lies outside the param's [minValue, maxValue]");
    std::string range;
    if (n->kind == K_OSC && !osc_pitch_allowed(g, *n, param_index, l, h, range))
        return fail(WAE_UNSUPPORTED, "OscillatorNode " + std::to_string(node) + ": " + range + " allow computed frequencies outside (0, " +
                                         std::to_string(g->sample_rate / 2.f) + ") Hz; a pitch bound from device memory must stay inside "
                                         "it (bind a wider pitch as a value curve: wae_param_set_device_value_curve)");
    if ((n->kind == K_PANNER || n->kind == K_LISTENER) && (l < -kSpatialBound || h > kSpatialBound))
        return fail(WAE_UNSUPPORTED, std::string(n->kind == K_PANNER ? "PannerNode " + std::to_string(node) : std::string("AudioListener")) +
                                         " param " + std::to_string(param_index) + ": a spatial value bound from device memory must lie "
                                         "inside [-1e9, 1e9] (the f32 spatial math overflows beyond it); declare a narrower range");
    p.device_bound = true;
    p.device_lo = l;
    p.device_hi = h;
    g->device_params++;
    return WAE_OK;
}

// OfflineAudioContext::suspend_sync (src/context/offline.rs:330-387).  The binding runs the user's callback right after this
// call: every graph mutation issued from here on takes effect at the quantised suspend frame.
WAE_API wae_status wae_graph_suspend(wae_graph* g, double suspend_time) {
    if (!g) return fail(WAE_INVALID_ARGUMENT, "null graph");
    if (!(suspend_time >= 0.)) return fail(WAE_INVALID_STATE, "InvalidStateError - suspendTime cannot be negative");
    const uint64_t quantum = (uint64_t)std::ceil(suspend_time * (double)g->sample_rate / 128.);  // offline.rs:248-251
    const uint64_t total = (g->length + 127) / 128;
    const uint64_t last = g->epochs.empty() ? 0 : g->epochs.back().frame / 128;
    if (!g->epochs.empty() && quantum == last)
        return fail(WAE_INVALID_STATE, "InvalidStateError - cannot suspend multiple times at the same render quantum");
    if (!g->epochs.empty() && quantum < last)
        return fail(WAE_INVALID_STATE, "InvalidStateError - cannot suspend at a time that is not after the current time");
    if (quantum >= total) return fail(WAE_INVALID_STATE, "InvalidStateError - cannot suspend after the end of the rendering");
    if (g->device_schedules)  // (sources are planned per render segment from their start time)
        return fail(WAE_INVALID_STATE, "InvalidStateError - the graph has schedules bound from device memory (wae_source_set_device_schedule)");
    if (g->device_loops)  // (the reference allows loop changes after start, which suspend points do not lower)
        return fail(WAE_INVALID_STATE, "InvalidStateError - the graph has loop points bound from device memory (wae_buffer_source_set_device_loop)");
    if (g->analyser_readouts)  // (read-outs are taken on the GPU; suspend callbacks run on the host before the render)
        return fail(WAE_INVALID_STATE, "InvalidStateError - the graph has analyser read-outs declared (wae_analyser_set_readouts)");
    if (g->compressor_readouts)
        return fail(WAE_INVALID_STATE, "InvalidStateError - the graph has compressor read-outs declared (wae_compressor_set_readouts)");
    g->epochs.push_back(wae_graph::Epoch{quantum * 128, g->nodes});
    return WAE_OK;
}

WAE_API wae_status wae_disconnect(wae_graph* g, wae_node_id from) {
    auto fi = g->nodes.find(from);
    if (fi == g->nodes.end()) return fail(WAE_INVALID_ARGUMENT, "InvalidAccessError - unknown node");
    g->nodes.at(fi->second.out_id).outgoing.clear();
    return WAE_OK;
}

// AudioNode::disconnect_dest / disconnect_output / disconnect_dest_from_output / disconnect_dest_from_output_to_input
// (src/node/audio_node.rs:304-405) = ConcreteBaseAudioContext::disconnect(from, Option<output>, Option<to>, Option<input>)
// (src/context/concrete_base.rs:474-507): -1 / WAE_NODE_NONE stand for None.
static wae_status disconnect_matching(wae_graph* g, wae_node_id from, int32_t output, bool has_to, uint32_t to_id, int32_t input) {
    auto fi = g->nodes.find(from);
    if (fi == g->nodes.end() || fi->second.kind == K_PARAM) return fail(WAE_INVALID_ARGUMENT, "InvalidAccessError - unknown node");
    if (output >= fi->second.n_outputs)
        return fail(WAE_INVALID_ARGUMENT, "IndexSizeError - output port " + std::to_string(output) + " is out of bounds");
    std::vector<Edge>& out = g->nodes.at(fi->second.out_id).outgoing;
    const size_t before = out.size();
    out.erase(std::remove_if(out.begin(), out.end(),
                             [&](const Edge& e) {
                                 if (e.other_index < 0) return false;  // hidden edges (DelayWriter -> reader, listener -> panner) are not the user's
                                 return (output < 0 || e.self_index == output) && (!has_to || e.other_id == to_id) && (input < 0 || e.other_index == input);
                             }),
              out.end());
    if (has_to && out.size() == before) return fail(WAE_INVALID_ARGUMENT, "InvalidAccessError - attempting to disconnect unconnected nodes");
    return WAE_OK;
}

WAE_API wae_status wae_disconnect_from(wae_graph* g, wae_node_id from, int32_t output, wae_node_id to, int32_t input) {
    if (!g) return fail(WAE_INVALID_ARGUMENT, "null graph");
    if (to == WAE_NODE_NONE) return disconnect_matching(g, from, output, false, 0, input);
    auto ti = g->nodes.find(to);
    if (ti == g->nodes.end() || ti->second.kind == K_PARAM) return fail(WAE_INVALID_ARGUMENT, "InvalidAccessError - unknown node");
    if (input >= ti->second.n_inputs)
        return fail(WAE_INVALID_ARGUMENT, "IndexSizeError - input port " + std::to_string(input) + " is out of bounds");
    return disconnect_matching(g, from, output, true, to, input);
}

// the same towards an AudioParam of `to` (AudioParam is an AudioNode in the reference: node.disconnect_dest(param))
WAE_API wae_status wae_disconnect_param(wae_graph* g, wae_node_id from, int32_t output, wae_node_id to, uint32_t param_index) {
    if (!g) return fail(WAE_INVALID_ARGUMENT, "null graph");
    auto ti = g->nodes.find(to);
    if (ti == g->nodes.end()) return fail(WAE_INVALID_ARGUMENT, "InvalidAccessError - unknown node");
    if (param_index >= ti->second.params.size()) return fail(WAE_INVALID_ARGUMENT, "IndexSizeError - param index out of bounds");
    return disconnect_matching(g, from, output, true, ti->second.params[param_index], -1);
}

static wae_status push_event(Param& p, const wae_param_event* e) {
    if (p.device_bound)
        return fail(WAE_INVALID_STATE, "InvalidStateError - the param's value is bound from device memory (wae_param_set_device_value): "
                                       "it takes no events");
    if (p.device_curve)
        return fail(WAE_INVALID_STATE, "InvalidStateError - the param's value curve is bound from device memory "
                                       "(wae_param_set_device_value_curve): it takes no further events");
    auto finite = [](float v) { return std::isfinite(v); };
    auto valid_time = [](double t) { return std::isfinite(t) && t >= 0.; };
    ParamEv ev{(int)e->type, e->value, e->time, e->aux, {}};
    switch (e->type) {
        case WAE_EVENT_SET_VALUE:
            if (!finite(e->value)) return fail(WAE_INVALID_ARGUMENT, "TypeError - The provided value is non-finite.");
            ev.time = 0.;
            break;
        case WAE_EVENT_SET_VALUE_AT_TIME:
        case WAE_EVENT_LINEAR_RAMP_TO_VALUE_AT_TIME:
            if (!finite(e->value)) return fail(WAE_INVALID_ARGUMENT, "TypeError - The provided value is non-finite.");
            if (!valid_time(e->time)) return fail(WAE_INVALID_ARGUMENT, "RangeError - time should be positive");
            break;
        case WAE_EVENT_EXPONENTIAL_RAMP_TO_VALUE_AT_TIME:
            if (!finite(e->value)) return fail(WAE_INVALID_ARGUMENT, "TypeError - The provided value is non-finite.");
            if (e->value == 0.f) return fail(WAE_INVALID_ARGUMENT, "RangeError - value (0.0) should not be equal to zero");
            if (!valid_time(e->time)) return fail(WAE_INVALID_ARGUMENT, "RangeError - time should be positive");
            break;
        case WAE_EVENT_SET_TARGET_AT_TIME:
            if (!finite(e->value)) return fail(WAE_INVALID_ARGUMENT, "TypeError - The provided value is non-finite.");
            if (!valid_time(e->time) || !valid_time(e->aux)) return fail(WAE_INVALID_ARGUMENT, "RangeError - time should be positive");
            if (e->aux == 0.) ev.type = WAE_EVENT_SET_VALUE_AT_TIME;  // src/param.rs:529-538
            break;
        case WAE_EVENT_CANCEL_SCHEDULED_VALUES:
        case WAE_EVENT_CANCEL_AND_HOLD_AT_TIME:
            if (!valid_time(e->time)) return fail(WAE_INVALID_ARGUMENT, "RangeError - time should be positive");
            break;
        case WAE_EVENT_SET_VALUE_CURVE_AT_TIME:
            if (e->values_len < 2) return fail(WAE_INVALID_STATE, "InvalidStateError - sequence length should not be less than 2");
            if (!valid_time(e->time)) return fail(WAE_INVALID_ARGUMENT, "RangeError - time should be positive");
            if (!(std::isfinite(e->aux) && e->aux > 0.)) return fail(WAE_INVALID_ARGUMENT, "RangeError - duration should be strictly positive");
            ev.values.assign(e->values, e->values + e->values_len);
            break;
        default: return fail(WAE_INVALID_ARGUMENT, "unknown event type");
    }
    p.events.push_back(std::move(ev));
    return WAE_OK;
}

// ---- host-side simulation of ONE AudioParam (diagnostics / tests, no GPU): the event folding of wae_param_host.h and the
// state machine of wae_param_core.h — the very code the planner and the k_param kernel run — driven block by block like the
// reference's unit tests drive AudioParamProcessor (src/param.rs:1766-3545: handle_incoming_event + compute_intrinsic_values).
struct wae_param_sim {
    Param prm;
    size_t folded = 0;
    ParamTimeline tl;
    ParamState st{};
    bool started = false;
    uint32_t walker = 0;  // 0: param_compute_buffer (k_param); 1 / 2: param_walk with the serial / the recording sink (k_param_parallel);
                          // 3: the recording sink walked from PREDICTED states that are verified first, like k_param_spec does
    // walker 3: the speculation window of k_param_spec (its lane j walks quantum j from `base` with a predicted intrinsic value)
    ParamState spec_base{};
    int spec_j = 0;
    double spec_prev_block_time = 0.;
    uint32_t spec_prev_count = 0;
    uint64_t spec_tried = 0, spec_hits = 0;
};
WAE_API wae_status wae_param_sim_set_walker(wae_param_sim* s, uint32_t walker) {
    if (!s || walker > 3) return fail(WAE_INVALID_ARGUMENT, "unknown walker");
    s->walker = walker;
    return WAE_OK;
}
WAE_API wae_status wae_param_sim_create(uint32_t a_rate, float default_value, float min_value, float max_value, wae_param_sim** out) {
    auto* s = new wae_param_sim;
    s->prm.default_value = default_value;
    s->prm.min_value = min_value;
    s->prm.max_value = max_value;
    s->prm.a_rate = a_rate != 0;
    *out = s;
    return WAE_OK;
}
WAE_API wae_status wae_param_sim_destroy(wae_param_sim* s) {
    delete s;
    return WAE_OK;
}
WAE_API wae_status wae_param_sim_push(wae_param_sim* s, const wae_param_event* e) { return push_event(s->prm, e); }
WAE_API wae_status wae_param_sim_set_automation_rate(wae_param_sim* s, uint32_t a_rate) {
    s->prm.a_rate = a_rate != 0;
    return WAE_OK;
}
// out must hold `count` floats; *len = 1 (single-valued block) or count
WAE_API wae_status wae_param_sim_compute(wae_param_sim* s, double block_time, double dt, uint32_t count, float* out, uint32_t* len) {
    if (count == 0 || count > 128) return fail(WAE_INVALID_ARGUMENT, "count must be in [1, 128]");
    if (s->folded < s->prm.events.size()) {  // events that arrived since the last block: handle_incoming_event against the live state
        ParamTimeline next;
        if (!s->started) {
            next.intrinsic = s->prm.default_value;
        } else {
            next.curves = s->tl.curves;
            for (int i = s->st.head; i < (int)s->tl.events.size(); i++)
                next.events.push_back(i == s->st.head && s->st.override_valid ? s->st.override_ev : s->tl.events[i]);
            next.intrinsic = s->st.intrinsic;
            next.has_last = s->st.has_last != 0;
            next.last = s->st.last;
        }
        fold_param_events(next, s->prm.events.data() + s->folded, s->prm.events.size() - s->folded);
        if (!next.error.empty()) return fail(WAE_NOT_SUPPORTED, next.error);
        s->tl = std::move(next);
        s->folded = s->prm.events.size();
        s->st.intrinsic = s->tl.intrinsic;
        s->st.head = 0;
        s->st.override_valid = 0;
        s->st.has_last = s->tl.has_last ? 1 : 0;
        s->st.last = s->tl.last;
        s->started = true;
    } else if (!s->started) {
        s->st.intrinsic = s->prm.default_value;
        s->started = true;
    }
    ParamInst host{};
    host.events = s->tl.events.data();
    host.curves = s->tl.curves.data();
    host.n_events = (int32_t)s->tl.events.size();
    host.a_rate = s->prm.a_rate ? 1 : 0;
    host.sample_rate = (float)(1. / dt);
    float buf[128];
    int n;
    if (s->walker == 1) {
        SerialSink sink{buf, 1. / (double)host.sample_rate};
        n = param_walk(host, s->st, block_time, sink, (int)count);
    } else if (s->walker == 2) {
        RecordSink sink;
        sink.buf = buf;
        sink.dt = 1. / (double)host.sample_rate;
        n = param_walk(host, s->st, block_time, sink, (int)count);
        sink.finish();
    } else if (s->walker == 3) {
        // k_param_spec, one quantum per call: lane 0 of a window walks the real state; lane j > 0 walks `base` with the predicted
        // intrinsic value, and its result is only kept when the state the previous walk left equals that prediction
        const double sdt = 1. / (double)host.sample_rate;
        bool speculate = s->spec_j > 0 && s->spec_j < 32 && s->spec_prev_count == count;
        ParamState from = s->st;
        if (speculate) {
            ParamState pred = s->spec_base;
            pred.intrinsic = param_predict_intrinsic(host, pred, std::fma(sdt, (double)count, s->spec_prev_block_time));
            s->spec_tried++;
            if (param_state_equal(s->st, pred)) {
                s->spec_hits++;
                from = pred;  // (what the kernel keeps is the walk that started from the prediction)
            } else {
                speculate = false;
            }
        }
        if (!speculate) {
            s->spec_base = s->st;
            s->spec_j = 0;
        }
        RecordSink sink;
        sink.buf = buf;
        sink.dt = sdt;
        n = param_walk(host, from, block_time, sink, (int)count);
        sink.finish();
        s->st = from;
        s->spec_j++;
        s->spec_prev_block_time = block_time;
        s->spec_prev_count = count;
    } else {
        n = param_compute_buffer(host, s->st, block_time, buf, (int)count);
    }
    for (int i = 0; i < n; i++) out[i] = buf[i];
    *len = (uint32_t)n;
    return WAE_OK;
}

WAE_API wae_status wae_param_sim_speculation(wae_param_sim* s, uint64_t* tried, uint64_t* hits) {
    if (!s || !tried || !hits) return fail(WAE_INVALID_ARGUMENT, "null argument");
    *tried = s->spec_tried;
    *hits = s->spec_hits;
    return WAE_OK;
}

WAE_API wae_status wae_param_event_push(wae_graph* g, wae_node_id node, uint32_t param_index, const wae_param_event* e) {
    auto ni = g->nodes.find(node);
    if (ni == g->nodes.end() || param_index >= ni->second.params.size()) return fail(WAE_INVALID_ARGUMENT, "unknown param");
    return push_event(g->nodes.at(ni->second.params[param_index]).param, e);
}

// One SetValueCurveAtTime event of `length` values that wae_batch_bind_value_curves supplies per run, pushed in arrival order as
// wae_param_event_push pushes a host curve (with zero placeholders for the values): folding, sorting and overlap errors are the host's.
// The param takes no further events, so no planning decision ever reads the values.
WAE_API wae_status wae_param_set_device_value_curve(wae_graph* g, wae_node_id node, uint32_t param_index, uint32_t length,
                                                    double start_time, double duration) {
    if (!g) return fail(WAE_INVALID_ARGUMENT, "null graph");
    Node* n = g->nodes.get(node);
    if (!n || n->kind == K_PARAM || param_index >= n->params.size()) return fail(WAE_INVALID_ARGUMENT, "unknown param");
    if (n->kind == K_LISTENER) return fail(WAE_INVALID_ARGUMENT, "AudioListener params are not bound from device memory");
    if (length < 2) return fail(WAE_INVALID_STATE, "InvalidStateError - sequence length should not be less than 2");
    if (!(std::isfinite(start_time) && start_time >= 0.)) return fail(WAE_INVALID_ARGUMENT, "RangeError - time should be positive");
    if (!(std::isfinite(duration) && duration > 0.)) return fail(WAE_INVALID_ARGUMENT, "RangeError - duration should be strictly positive");
    Param& p = g->nodes.at(n->params[param_index]).param;
    if (p.device_bound)
        return fail(WAE_INVALID_STATE, "InvalidStateError - the param's value is bound from device memory (wae_param_set_device_value)");
    if (p.device_curve)
        return fail(WAE_INVALID_STATE, "InvalidStateError - the param's value curve is already bound from device memory "
                                       "(wae_param_set_device_value_curve)");
    if (!g->epochs.empty())  // (the segments before the suspend point were planned with the events of their own graph copy)
        return fail(WAE_INVALID_STATE, "InvalidStateError - a value curve is bound from device memory before the first suspend point");
    p.events.push_back(ParamEv{WAE_EVENT_SET_VALUE_CURVE_AT_TIME, 0.f, start_time, duration, std::vector<float>(length, 0.f)});
    p.device_curve = length;
    p.device_curve_node = node;
    p.device_curve_index = param_index;
    g->device_value_curves++;
    return WAE_OK;
}

WAE_API wae_status wae_listener_param_event_push(wae_graph* g, uint32_t param_index, const wae_param_event* e) {
    if (param_index >= 9) return fail(WAE_INVALID_ARGUMENT, "unknown listener param");
    g->ensure_listener();
    return push_event(g->nodes.at(2 + param_index).param, e);
}

WAE_API wae_status wae_param_set_automation_rate(wae_graph* g, wae_node_id node, uint32_t param_index, uint32_t rate) {
    auto ni = g->nodes.find(node);
    if (ni == g->nodes.end() || param_index >= ni->second.params.size()) return fail(WAE_INVALID_ARGUMENT, "unknown param");
    Param& p = g->nodes.at(ni->second.params[param_index]).param;
    bool want_a = rate == WAE_AUTOMATION_RATE_A;
    if (p.rate_constrained && want_a != p.a_rate)
        return fail(WAE_INVALID_STATE, "InvalidStateError - automation rate cannot be changed for this param");
    p.a_rate = want_a;
    return WAE_OK;
}

// AudioScheduledSourceNode::start_at / stop_at, AudioBufferSourceNode::start_at_with_offset_and_duration
WAE_API wae_status wae_source_start(wae_graph* g, wae_node_id node, double when, double offset, double duration) {
    auto ni = g->nodes.find(node);
    if (ni == g->nodes.end()) return fail(WAE_INVALID_ARGUMENT, "unknown node");
    Node& n = ni->second;
    if (!(n.kind == K_OSC || n.kind == K_ABSN || n.kind == K_CONST)) return fail(WAE_INVALID_ARGUMENT, "not a scheduled source node");
    if (!(std::isfinite(when) && when >= 0.)) return fail(WAE_INVALID_ARGUMENT, "RangeError - when should be positive");
    if (n.device_schedule)
        return fail(WAE_INVALID_STATE, "InvalidStateError - the start time is bound from device memory (wae_source_set_device_schedule)");
    if (n.has_start) return fail(WAE_INVALID_STATE, "InvalidStateError - Cannot call `start` twice");
    if (n.kind == K_ABSN && (!(offset >= 0.) || !(duration >= 0.))) return fail(WAE_INVALID_ARGUMENT, "RangeError - offset/duration should be positive");
    n.has_start = true;
    // issued from a suspend_sync callback: a start time in the past snaps to the quantum the render is suspended at, the first
    // one that sees the message (oscillator.rs `if !started && start_time < current_time`, audio_buffer_source.rs:519-523;
    // the reference's test_start_in_the_past for both nodes)
    if (!g->epochs.empty()) when = std::max(when, (double)g->epochs.back().frame / (double)g->sample_rate);
    n.start_time = when;
    if (n.kind == K_ABSN) {
        n.offset = offset;
        n.duration = duration >= 1e300 ? 1.7976931348623157e308 : duration;
    }
    return WAE_OK;
}

WAE_API wae_status wae_source_stop(wae_graph* g, wae_node_id node, double when) {
    auto ni = g->nodes.find(node);
    if (ni == g->nodes.end()) return fail(WAE_INVALID_ARGUMENT, "unknown node");
    Node& n = ni->second;
    if (!(n.kind == K_OSC || n.kind == K_ABSN || n.kind == K_CONST)) return fail(WAE_INVALID_ARGUMENT, "not a scheduled source node");
    if (!(std::isfinite(when) && when >= 0.)) return fail(WAE_INVALID_ARGUMENT, "RangeError - when should be positive");
    if (!n.has_start) return fail(WAE_INVALID_STATE, "InvalidStateError cannot stop before start");
    if (n.device_schedule)
        return fail(WAE_INVALID_STATE, "InvalidStateError - the schedule is bound from device memory (wae_source_set_device_schedule)");
    n.stop_time = when;
    return WAE_OK;
}

// The start time (and with bind_stop the stop time) becomes a placeholder, written per run by wae_batch_bind_schedules clamped to its
// window.  The plan is made with the windows' low ends and a gated output layout, so no planning decision depends on the bound times.
// Sources are planned per render segment from their start time, so a graph with suspend points takes no declaration (and the other way
// round: wae_graph_suspend refuses a graph with one).
WAE_API wae_status wae_source_set_device_schedule(wae_graph* g, wae_node_id node, double start_lo, double start_hi, int32_t bind_stop,
                                                  double stop_lo, double stop_hi) {
    if (!g) return fail(WAE_INVALID_ARGUMENT, "null graph");
    Node* n = g->nodes.get(node);
    if (!n || !(n->kind == K_OSC || n->kind == K_ABSN || n->kind == K_CONST)) return fail(WAE_INVALID_ARGUMENT, "not a scheduled source node");
    auto window = [](double lo, double hi) { return std::isfinite(lo) && std::isfinite(hi) && 0. <= lo && lo <= hi; };
    if (!window(start_lo, start_hi) || (bind_stop && !window(stop_lo, stop_hi)))
        return fail(WAE_INVALID_ARGUMENT, "RangeError - a schedule window must be finite with 0 <= lo <= hi");
    if (n->device_schedule)
        return fail(WAE_INVALID_STATE, "InvalidStateError - the schedule is already bound from device memory (wae_source_set_device_schedule)");
    if (!n->has_start) return fail(WAE_INVALID_STATE, "InvalidStateError - the source has not been started");
    if (!g->epochs.empty())
        return fail(WAE_INVALID_STATE, "InvalidStateError - a schedule is bound from device memory in a graph with a suspend point");
    n->device_schedule = true;
    n->sched_stop = bind_stop != 0;
    n->start_time = start_lo;
    n->sched_lo[0] = start_lo;
    n->sched_hi[0] = start_hi;
    if (bind_stop) {
        n->stop_time = stop_lo;
        n->sched_lo[1] = stop_lo;
        n->sched_hi[1] = stop_hi;
    }
    g->device_schedules++;
    return WAE_OK;
}

// AnalyserNode read-outs taken during the render at declared times, each quantised like suspend_sync (offline.rs:248-251).  The
// suspend points a graph with read-outs would need are exactly what it does without: a graph has one or the other.
static wae_status readout_quanta(const wae_graph* g, const double* times, uint32_t n, std::vector<uint64_t>& q) {
    if (n == 0 || !times) return fail(WAE_INVALID_ARGUMENT, "no read-out times");
    const uint64_t total = (g->length + 127) / 128;
    q.assign(n, 0);
    for (uint32_t k = 0; k < n; k++) {
        if (!std::isfinite(times[k]) || times[k] < 0.)
            return fail(WAE_INVALID_ARGUMENT, "RangeError - read-out time " + std::to_string(k) + " is negative or not finite");
        if (k > 0 && times[k] < times[k - 1])
            return fail(WAE_INVALID_ARGUMENT, "RangeError - read-out times must not decrease (time " + std::to_string(k) + ")");
        const double qd = std::ceil(times[k] * (double)g->sample_rate / 128.);
        if (qd > (double)total)
            return fail(WAE_INVALID_ARGUMENT, "RangeError - read-out time " + std::to_string(k) + " is after the end of the rendering");
        q[k] = (uint64_t)qd;
    }
    return WAE_OK;
}

WAE_API wae_status wae_analyser_set_readouts(wae_graph* g, wae_node_id node, const double* times, uint32_t n, uint32_t kinds) {
    if (!g) return fail(WAE_INVALID_ARGUMENT, "null graph");
    Node* a = g->nodes.get(node);
    if (!a || a->kind != K_ANALYSER) return fail(WAE_INVALID_ARGUMENT, "not an AnalyserNode");
    if (n == 0 || !times) return fail(WAE_INVALID_ARGUMENT, "no read-out times");
    if (kinds == 0 || (kinds & ~(uint32_t)(WAE_READOUT_FREQUENCY | WAE_READOUT_TIME_DOMAIN)))
        return fail(WAE_INVALID_ARGUMENT, "kinds must be a non-empty set of WAE_READOUT_FREQUENCY | WAE_READOUT_TIME_DOMAIN");
    std::vector<uint64_t> q;
    const wae_status st = readout_quanta(g, times, n, q);
    if (st != WAE_OK) return st;
    if (a->readout_kinds) return fail(WAE_INVALID_STATE, "InvalidStateError - the analyser already has read-outs declared");
    if (!g->epochs.empty()) return fail(WAE_INVALID_STATE, "InvalidStateError - analyser read-outs are declared in a graph with a suspend point");
    a->readout_q = std::move(q);
    a->readout_kinds = kinds;
    g->analyser_readouts++;
    return WAE_OK;
}

// The declared read-outs of `kinds` are also delivered as bytes (get_byte_frequency_data / get_byte_time_domain_data), at the same times
WAE_API wae_status wae_analyser_set_byte_readouts(wae_graph* g, wae_node_id node, uint32_t kinds) {
    if (!g) return fail(WAE_INVALID_ARGUMENT, "null graph");
    Node* a = g->nodes.get(node);
    if (!a || a->kind != K_ANALYSER) return fail(WAE_INVALID_ARGUMENT, "not an AnalyserNode");
    if (kinds == 0 || (kinds & ~(uint32_t)(WAE_READOUT_FREQUENCY | WAE_READOUT_TIME_DOMAIN)))
        return fail(WAE_INVALID_ARGUMENT, "kinds must be a non-empty set of WAE_READOUT_FREQUENCY | WAE_READOUT_TIME_DOMAIN");
    if (!g->epochs.empty()) return fail(WAE_INVALID_STATE, "InvalidStateError - analyser read-outs are declared in a graph with a suspend point");
    if (!a->readout_kinds)
        return fail(WAE_INVALID_STATE, "InvalidStateError - the analyser has no read-outs declared (wae_analyser_set_readouts)");
    if (a->byte_readout_kinds) return fail(WAE_INVALID_STATE, "InvalidStateError - the analyser already has byte read-outs declared");
    if (kinds & ~a->readout_kinds) return fail(WAE_INVALID_ARGUMENT, "byte read-outs of a kind the analyser's read-outs do not declare");
    a->byte_readout_kinds = kinds;
    return WAE_OK;
}

// DynamicsCompressorNode::reduction read at declared times, each quantised like suspend_sync (offline.rs:248-251)
WAE_API wae_status wae_compressor_set_readouts(wae_graph* g, wae_node_id node, const double* times, uint32_t n) {
    if (!g) return fail(WAE_INVALID_ARGUMENT, "null graph");
    Node* c = g->nodes.get(node);
    if (!c || c->kind != K_COMP) return fail(WAE_INVALID_ARGUMENT, "not a DynamicsCompressorNode");
    std::vector<uint64_t> q;
    const wae_status st = readout_quanta(g, times, n, q);
    if (st != WAE_OK) return st;
    if (!c->readout_q.empty()) return fail(WAE_INVALID_STATE, "InvalidStateError - the compressor already has read-outs declared");
    if (!g->epochs.empty()) return fail(WAE_INVALID_STATE, "InvalidStateError - compressor read-outs are declared in a graph with a suspend point");
    c->readout_q = std::move(q);
    g->compressor_readouts++;
    return WAE_OK;
}

// Extends the schedule declaration of an AudioBufferSourceNode with its offset (and with bind_duration its duration): placeholders
// written per run by wae_batch_bind_schedules, planned at the windows' low ends like the start time.  A declared schedule already takes
// the bound slow track or the serial kernel, whose records hold the offset and duration the bind rewrites.
WAE_API wae_status wae_buffer_source_set_device_offset(wae_graph* g, wae_node_id node, double offset_lo, double offset_hi, int32_t bind_duration,
                                                       double duration_lo, double duration_hi) {
    if (!g) return fail(WAE_INVALID_ARGUMENT, "null graph");
    Node* n = g->nodes.get(node);
    if (!n || n->kind != K_ABSN) return fail(WAE_INVALID_ARGUMENT, "not an AudioBufferSourceNode");
    auto window = [](double lo, double hi) { return std::isfinite(lo) && std::isfinite(hi) && 0. <= lo && lo <= hi; };
    if (!window(offset_lo, offset_hi) || (bind_duration && !window(duration_lo, duration_hi)))
        return fail(WAE_INVALID_ARGUMENT, "RangeError - an offset / duration window must be finite with 0 <= lo <= hi");
    if (!n->device_schedule)
        return fail(WAE_INVALID_STATE, "InvalidStateError - the start time is not bound from device memory (wae_source_set_device_schedule)");
    if (n->sched_offset)
        return fail(WAE_INVALID_STATE, "InvalidStateError - the offset is already bound from device memory (wae_buffer_source_set_device_offset)");
    n->sched_offset = true;
    n->sched_duration = bind_duration != 0;
    n->offset = offset_lo;
    n->sched_lo[2] = offset_lo;
    n->sched_hi[2] = offset_hi;
    if (bind_duration) {
        n->duration = duration_lo;
        n->sched_lo[3] = duration_lo;
        n->sched_hi[3] = duration_hi;
    }
    return WAE_OK;
}

// loopStart and loopEnd become placeholders (the windows' low ends), written per run by wae_batch_bind_loops clamped to their windows.
// The planner decides the playback path from the windows (and the declared rates), never from the bound values.
WAE_API wae_status wae_buffer_source_set_device_loop(wae_graph* g, wae_node_id node, double start_lo, double start_hi, double end_lo,
                                                     double end_hi) {
    if (!g) return fail(WAE_INVALID_ARGUMENT, "null graph");
    Node* n = g->nodes.get(node);
    if (!n || n->kind != K_ABSN) return fail(WAE_INVALID_ARGUMENT, "not an AudioBufferSourceNode");
    auto window = [](double lo, double hi) { return std::isfinite(lo) && std::isfinite(hi) && 0. <= lo && lo <= hi; };
    if (!window(start_lo, start_hi) || !window(end_lo, end_hi))
        return fail(WAE_INVALID_ARGUMENT, "RangeError - a loop window must be finite with 0 <= lo <= hi");
    if (!n->loop) return fail(WAE_INVALID_STATE, "InvalidStateError - the source does not loop (set_loop)");
    if (n->device_loop)
        return fail(WAE_INVALID_STATE, "InvalidStateError - the loop points are already bound from device memory (wae_buffer_source_set_device_loop)");
    if (!g->epochs.empty())
        return fail(WAE_INVALID_STATE, "InvalidStateError - loop points are bound from device memory in a graph with a suspend point");
    n->device_loop = true;
    n->loop_start = start_lo;
    n->loop_end = end_lo;
    n->loop_lo[0] = start_lo;
    n->loop_hi[0] = start_hi;
    n->loop_lo[1] = end_lo;
    n->loop_hi[1] = end_hi;
    g->device_loops++;
    return WAE_OK;
}

WAE_API wae_status wae_oscillator_set_type(wae_graph* g, wae_node_id node, uint32_t type) {
    auto ni = g->nodes.find(node);
    if (ni == g->nodes.end() || ni->second.kind != K_OSC) return fail(WAE_INVALID_ARGUMENT, "not an oscillator");
    if (type >= WAE_OSC_CUSTOM) return fail(WAE_INVALID_STATE, "InvalidStateError: Custom type cannot be set manually");
    if (ni->second.type == WAE_OSC_CUSTOM) return WAE_OK;
    ni->second.type = (int)type;
    return WAE_OK;
}

WAE_API wae_status wae_biquad_set_type(wae_graph* g, wae_node_id node, uint32_t type) {
    auto ni = g->nodes.find(node);
    if (ni == g->nodes.end() || ni->second.kind != K_BIQUAD || type > 7) return fail(WAE_INVALID_ARGUMENT, "not a biquad / bad type");
    ni->second.type = (int)type;
    return WAE_OK;
}

// PeriodicWave::new -> generate_wavetable + normalize (src/periodic_wave.rs:104-209): the wavetable an OscillatorNode of type Custom plays
// (wae_oscillator_options.periodic_wave / wae_oscillator_set_periodic_wave take it).  real / imag may be NULL (zeros); both NULL = sine.
WAE_API wae_status wae_periodic_wave_table(const float* real, const float* imag, uint32_t len, uint32_t disable_normalization, float* table,
                                           uint32_t table_len) {
    const bool has_r = real != nullptr, has_i = imag != nullptr;
    if ((has_r || has_i) && len < 2) return fail(WAE_INVALID_ARGUMENT, "IndexSizeError - `real` and `imag` length should at least 2");
    if (!table || table_len == 0) return fail(WAE_INVALID_ARGUMENT, "null table");
    static const float sine_r[2] = {0.f, 0.f}, sine_i[2] = {0.f, 1.f};  // no coefficients: the built-in sine (periodic_wave.rs:143-146)
    const uint32_t n = (has_r || has_i) ? len : 2;
    const float pi_2 = 2.f * 3.14159265358979323846f;
    for (uint32_t i = 0; i < table_len; i++) {
        float sample = 0.f;
        const float phase = pi_2 * (float)i / (float)table_len;
        for (uint32_t j = 1; j < n; j++) {
            const float re = has_r ? real[j] : ((has_r || has_i) ? 0.f : sine_r[j]);
            const float im = has_i ? imag[j] : ((has_r || has_i) ? 0.f : sine_i[j]);
            const float rad = phase * (float)j;
            const float contrib = re * std::cos(rad) + im * std::sin(rad);
            sample += contrib;
        }
        table[i] = sample;
    }
    if (!disable_normalization) {
        float mx = 0.f;
        for (uint32_t i = 0; i < table_len; i++) mx = std::fabs(table[i]) > mx ? std::fabs(table[i]) : mx;
        if (mx > 0.f) {
            const float norm = 1.f / mx;
            for (uint32_t i = 0; i < table_len; i++) table[i] *= norm;
        }
    }
    return WAE_OK;
}

// Test hook for the scheduling clock every AudioScheduledSourceNode is lowered with (csrc/wae_kernels.h SchedClock): the first frame
// whose time, accumulated the way the reference's renderers do (block time = frame / sample_rate, then `+= dt` per frame inside the
// quantum that contains `time`), is >= `time`; *frame_time = that accumulated time.
WAE_API wae_status wae_sched_first_frame_at_or_after(float sample_rate, double time, int64_t* frame, double* frame_time) {
    if (!frame || !frame_time || !(sample_rate > 0.f)) return fail(WAE_INVALID_ARGUMENT, "null / bad argument");
    SchedClock clock(sample_rate);
    *frame = clock.first_frame_at_or_after(time, frame_time);
    return WAE_OK;
}

// Test hook for the spatial math of PannerNode (csrc/wae_spatial.h, shared by the planner and the k_panner_dyn / k_hrtf_sel kernels):
// v = source position xyz, source orientation xyz, listener position xyz, forward xyz, up xyz; model6 = refDistance, maxDistance,
// rolloffFactor, coneInnerAngle, coneOuterAngle, coneOuterGain; out4 = distance gain, cone gain, azimuth, elevation (degrees)
WAE_API wae_status wae_spatial_params(uint32_t distance_model, const double* model6, const float* v15, float* out4) {
    if (!model6 || !v15 || !out4 || distance_model > 2) return fail(WAE_INVALID_ARGUMENT, "null / bad argument");
    spatial::PanModel m{};
    m.distance_model = (int32_t)distance_model;
    m.ref_distance = model6[0]; m.max_distance = model6[1]; m.rolloff_factor = model6[2];
    m.cone_inner_angle = model6[3]; m.cone_outer_angle = model6[4]; m.cone_outer_gain = model6[5];
    const spatial::SpatialParams p = spatial::spatial_params(m, v15);
    out4[0] = p.dist_gain; out4[1] = p.cone_gain; out4[2] = p.azimuth; out4[3] = p.elevation;
    return WAE_OK;
}

// Test hook: which sphere triangle a direction crosses and the barycentric weights of the hit (csrc/wae_spatial.h::hrir_locate, shared by
// the planner for static panners and k_hrtf_sel for moving ones); returns 1 when a face is hit.
WAE_API int32_t wae_hrtf_locate(const float* pos, const uint32_t* faces, uint32_t n_faces, const float* dir, uint32_t* idx, float* weights) {
    if (!pos || !faces || !dir || !idx || !weights) return 0;
    return spatial::hrir_locate(pos, faces, (int)n_faces, dir, idx, weights) ? 1 : 0;
}

// ---- node attributes set after construction (the reference posts a control message per setter) ------------------------------
namespace {
Node* node_of_kind(wae_graph* g, wae_node_id id, Kind kind) {
    if (!g) return nullptr;
    auto it = g->nodes.find(id);
    return it == g->nodes.end() || it->second.kind != kind ? nullptr : &it->second;
}
}  // namespace

// "if start called and buffer is null, should fire ended event and ignore any subsequent buffer assignment"
// (audio_buffer_source.rs:443-451): a source that was started before the last suspend point and has been rendered without a
// buffer since has ended for good
static void end_if_started_without_buffer(wae_graph* g, wae_node_id node, Node* n) {
    if (g->epochs.empty()) return;
    const auto& before = g->epochs.back().nodes;
    auto pi = before.find(node);
    if (pi != before.end() && pi->second.has_start && !pi->second.buffer) n->start_time = 1.7976931348623157e308;
}

// AudioBufferSourceNode::set_buffer (src/node/audio_buffer_source.rs:278-288): once
WAE_API wae_status wae_buffer_source_set_buffer(wae_graph* g, wae_node_id node, const wae_audio_buffer* buffer) {
    Node* n = node_of_kind(g, node, K_ABSN);
    if (!n || !buffer) return fail(WAE_INVALID_ARGUMENT, "not an AudioBufferSourceNode / null buffer");
    if (n->buffer) return fail(WAE_INVALID_STATE, "InvalidStateError - cannot assign buffer twice");
    if (!(n->buffer = copy_buffer(g, buffer, true))) return WAE_NOT_SUPPORTED;
    end_if_started_without_buffer(g, node, n);
    return WAE_OK;
}

// A device input counts as the node's buffer: the placeholder has the declared shape and rate and no host block.  It is not entered in
// g->assets, so content sharing never merges two device inputs; each gets its own slot in the group's source slab, or none when it is
// read by reference.
static wae_status declare_device_input(wae_graph* g, wae_node_id node, uint32_t number_of_channels, uint64_t length, float sample_rate,
                                       bool by_reference) {
    Node* n = node_of_kind(g, node, K_ABSN);
    if (!n) return fail(WAE_INVALID_ARGUMENT, "not an AudioBufferSourceNode");
    // AudioBuffer::new (src/buffer.rs:96-115), as copy_buffer checks it
    if (number_of_channels < 1 || number_of_channels > WAE_MAX_CHANNELS)
        return fail(WAE_NOT_SUPPORTED, "NotSupportedError - Invalid number of channels: " + std::to_string(number_of_channels) + " is outside range [1, 32]");
    if (length == 0) return fail(WAE_NOT_SUPPORTED, "NotSupportedError - Invalid length: 0 is less than or equal to minimum bound (0)");
    if (n->buffer) return fail(WAE_INVALID_STATE, "InvalidStateError - cannot assign buffer twice");
    auto p = std::make_shared<PcmBuffer>();
    p->sample_rate = sample_rate;
    p->device_input = true;
    p->by_reference = by_reference;
    p->stride = (size_t)(length + 3) / 4 * 4;
    p->channels.resize(number_of_channels);
    for (auto& c : p->channels) c.n = (size_t)length;
    n->buffer = std::move(p);
    g->device_inputs++;
    end_if_started_without_buffer(g, node, n);
    return WAE_OK;
}

WAE_API wae_status wae_buffer_source_set_device_input(wae_graph* g, wae_node_id node, uint32_t number_of_channels, uint64_t length,
                                                      float sample_rate) {
    return declare_device_input(g, node, number_of_channels, length, sample_rate, false);
}

WAE_API wae_status wae_buffer_source_set_device_input_by_reference(wae_graph* g, wae_node_id node, uint32_t number_of_channels,
                                                                   uint64_t length, float sample_rate) {
    return declare_device_input(g, node, number_of_channels, length, sample_rate, true);
}

// ConvolverNode::set_buffer (src/node/convolver.rs:259-317): may replace the response; the normalisation is decided now
WAE_API wae_status wae_convolver_set_buffer(wae_graph* g, wae_node_id node, const wae_audio_buffer* buffer) {
    Node* n = node_of_kind(g, node, K_CONV);
    if (!n || !buffer) return fail(WAE_INVALID_ARGUMENT, "not a ConvolverNode / null buffer");
    if (n->buffer && n->buffer->device_input)
        return fail(WAE_INVALID_STATE, "InvalidStateError - the response is bound from device memory (wae_convolver_set_device_response)");
    if (buffer->sample_rate != g->sample_rate)
        return fail(WAE_NOT_SUPPORTED, "NotSupportedError - sample rate of the convolution buffer must match the audio context");
    const uint32_t c = buffer->number_of_channels;
    if (!(c == 1 || c == 2 || c == 4)) return fail(WAE_NOT_SUPPORTED, "NotSupportedError - the convolution buffer must consist of 1, 2 or 4 channels");
    if (!g->epochs.empty() && n->buffer)  // the reference swaps in fresh convolvers (tail dropped): not lowered mid-render
        return fail(WAE_UNSUPPORTED, "replacing the impulse response of a ConvolverNode at a suspend point is not lowered to the GPU");
    auto fresh = copy_buffer(g, buffer, false);
    if (!fresh) return WAE_NOT_SUPPORTED;
    n->buffer = fresh;
    n->normalize = n->normalize_next;
    return WAE_OK;
}

// A declared response counts as the node's set_buffer: a placeholder of the declared shape and rate with no host block, never shared by
// content (not in g->assets).  The normalisation is decided now, as set_buffer decides it; the scale itself is computed in the bind.
WAE_API wae_status wae_convolver_set_device_response(wae_graph* g, wae_node_id node, uint32_t number_of_channels, uint64_t length,
                                                     float sample_rate) {
    Node* n = node_of_kind(g, node, K_CONV);
    if (!n) return fail(WAE_INVALID_ARGUMENT, "not a ConvolverNode");
    // set_buffer's checks, in its order, then AudioBuffer::new's for the length (src/buffer.rs:96-115)
    if (sample_rate != g->sample_rate)
        return fail(WAE_NOT_SUPPORTED, "NotSupportedError - sample rate of the convolution buffer must match the audio context");
    const uint32_t c = number_of_channels;
    if (!(c == 1 || c == 2 || c == 4)) return fail(WAE_NOT_SUPPORTED, "NotSupportedError - the convolution buffer must consist of 1, 2 or 4 channels");
    if (length == 0) return fail(WAE_NOT_SUPPORTED, "NotSupportedError - Invalid length: 0 is less than or equal to minimum bound (0)");
    if (n->buffer && n->buffer->device_input)
        return fail(WAE_INVALID_STATE, "InvalidStateError - the response is already bound from device memory (wae_convolver_set_device_response)");
    if (n->buffer) return fail(WAE_INVALID_STATE, "InvalidStateError - the ConvolverNode already has a response (set_buffer)");
    if (!g->epochs.empty())  // (the segments before the suspend point were planned with the graph copy of their own: no response)
        return fail(WAE_INVALID_STATE, "InvalidStateError - a response is bound from device memory before the first suspend point");
    auto p = std::make_shared<PcmBuffer>();
    p->sample_rate = sample_rate;
    p->device_input = true;
    p->stride = (size_t)length;
    p->channels.resize(number_of_channels);
    for (auto& ch : p->channels) ch.n = (size_t)length;
    n->buffer = std::move(p);
    n->normalize = n->normalize_next;
    g->device_responses++;
    return WAE_OK;
}

// WaveShaperNode::set_curve (src/node/waveshaper.rs:203-213): once
WAE_API wae_status wae_wave_shaper_set_curve(wae_graph* g, wae_node_id node, const float* curve, uint32_t len) {
    Node* n = node_of_kind(g, node, K_SHAPER);
    if (!n || (!curve && len)) return fail(WAE_INVALID_ARGUMENT, "not a WaveShaperNode / null curve");
    if (n->device_curve)
        return fail(WAE_INVALID_STATE, "InvalidStateError - the curve is bound from device memory (wae_wave_shaper_set_device_curve)");
    if (n->has_curve) return fail(WAE_INVALID_STATE, "InvalidStateError - cannot assign curve twice");
    n->has_curve = true;
    n->table.assign(curve, curve + len);
    return WAE_OK;
}

// A declared curve counts as the node's set_curve: the node has a curve of `length` points whose values only the bind supplies
WAE_API wae_status wae_wave_shaper_set_device_curve(wae_graph* g, wae_node_id node, uint32_t length) {
    Node* n = node_of_kind(g, node, K_SHAPER);
    if (!n) return fail(WAE_INVALID_ARGUMENT, "not a WaveShaperNode");
    if (length == 0) return fail(WAE_INVALID_ARGUMENT, "a curve bound from device memory has at least one point");
    if (n->device_curve)
        return fail(WAE_INVALID_STATE, "InvalidStateError - the curve is already bound from device memory (wae_wave_shaper_set_device_curve)");
    if (n->has_curve) return fail(WAE_INVALID_STATE, "InvalidStateError - the WaveShaperNode already has a curve (set_curve)");
    if (!g->epochs.empty())  // (the segments before the suspend point were planned with the graph copy of their own: no curve)
        return fail(WAE_INVALID_STATE, "InvalidStateError - a curve is bound from device memory before the first suspend point");
    n->has_curve = true;
    n->device_curve = length;
    g->device_curves++;
    return WAE_OK;
}

// OscillatorNode::set_periodic_wave (src/node/oscillator.rs:334-337): the type becomes Custom for good; `table` is the wavetable the
// binding generated (PeriodicWave::new, src/periodic_wave.rs:163-209)
WAE_API wae_status wae_oscillator_set_periodic_wave(wae_graph* g, wae_node_id node, const float* table, uint32_t len) {
    Node* n = node_of_kind(g, node, K_OSC);
    if (!n || !table || len == 0) return fail(WAE_INVALID_ARGUMENT, "not an OscillatorNode / empty wavetable");
    if (n->device_wave)
        return fail(WAE_INVALID_STATE,
                    "InvalidStateError - the periodic wave is bound from device memory (wae_oscillator_set_device_periodic_wave)");
    n->type = WAE_OSC_CUSTOM;
    n->table.assign(table, table + len);
    return WAE_OK;
}

// A declared wave counts as the node's set_periodic_wave: the type becomes Custom for good, and the oscillator plays a wavetable of
// `table_len` points that wae_batch_bind_periodic_waves synthesises from `coefficients` bound coefficients (PeriodicWave::new)
WAE_API wae_status wae_oscillator_set_device_periodic_wave(wae_graph* g, wae_node_id node, uint32_t coefficients, uint32_t table_len,
                                                           uint32_t disable_normalization) {
    Node* n = node_of_kind(g, node, K_OSC);
    if (!n) return fail(WAE_INVALID_ARGUMENT, "not an OscillatorNode");
    if (coefficients < 2) return fail(WAE_INVALID_ARGUMENT, "IndexSizeError - `real` and `imag` length should at least 2");
    if (table_len == 0) return fail(WAE_INVALID_ARGUMENT, "a periodic wave bound from device memory has a wavetable of at least one point");
    if (n->device_wave)
        return fail(WAE_INVALID_STATE,
                    "InvalidStateError - the periodic wave is already bound from device memory (wae_oscillator_set_device_periodic_wave)");
    if (!g->epochs.empty())  // (the segments before the suspend point were planned with the graph copy of their own: no wave)
        return fail(WAE_INVALID_STATE, "InvalidStateError - a periodic wave is bound from device memory before the first suspend point");
    n->type = WAE_OSC_CUSTOM;
    n->table.clear();  // (replaces an earlier host wave, as a second set_periodic_wave would)
    n->table.shrink_to_fit();
    n->device_wave = coefficients;
    n->device_wave_len = table_len;
    n->device_wave_normalize = disable_normalization == 0;
    g->device_waves++;
    return WAE_OK;
}

// A declared IIR filter keeps its coefficient counts; its coefficients are written per run by wae_batch_bind_iir_coefficients.  The
// planner picks the filter's path from the counts alone, so the constructed coefficients plan the node as bound ones would.
WAE_API wae_status wae_iir_filter_set_device_coefficients(wae_graph* g, wae_node_id node) {
    Node* n = node_of_kind(g, node, K_IIR);
    if (!n) return fail(WAE_INVALID_ARGUMENT, "not an IIRFilterNode");
    if (n->device_iir)
        return fail(WAE_INVALID_STATE,
                    "InvalidStateError - the coefficients are already bound from device memory (wae_iir_filter_set_device_coefficients)");
    if (!g->epochs.empty())  // (the segments before the suspend point were planned with the graph copy of their own: no declaration)
        return fail(WAE_INVALID_STATE, "InvalidStateError - IIR coefficients are bound from device memory before the first suspend point");
    n->device_iir = true;
    g->device_iirs++;
    return WAE_OK;
}

// the scalar setters of AudioBufferSourceNode (audio_buffer_source.rs:324-349), ConvolverNode (convolver.rs:325-328), WaveShaperNode
// (waveshaper.rs:226-229), PannerNode (panner.rs:545-657) and AnalyserNode (analyser.rs:148-222)
WAE_API wae_status wae_node_set_attribute(wae_graph* g, wae_node_id node, uint32_t attribute, double value) {
    if (!g) return fail(WAE_INVALID_ARGUMENT, "null graph");
    auto it = g->nodes.find(node);
    if (it == g->nodes.end()) return fail(WAE_INVALID_ARGUMENT, "InvalidAccessError - unknown node");
    Node& n = it->second;
    auto wrong = [&]() { return fail(WAE_INVALID_ARGUMENT, "this node has no such attribute"); };
    switch (attribute) {
        case WAE_ATTR_LOOP: case WAE_ATTR_LOOP_START: case WAE_ATTR_LOOP_END:
            if (n.kind != K_ABSN) return wrong();
            // the renderer keeps playing from its current playhead when the loop changes under it; the closed-form tracks of the
            // engine are planned per segment from the start time, so a change at a suspend point of a started source is refused
            if (!g->epochs.empty() && n.has_start)
                return fail(WAE_UNSUPPORTED, "changing the loop attributes of a started AudioBufferSourceNode at a suspend point is not lowered to the GPU");
            if (n.device_loop)
                return fail(WAE_INVALID_STATE, "InvalidStateError - the loop points are bound from device memory (wae_buffer_source_set_device_loop)");
            if (attribute == WAE_ATTR_LOOP) n.loop = value != 0.;
            else if (attribute == WAE_ATTR_LOOP_START) n.loop_start = value;
            else n.loop_end = value;
            return WAE_OK;
        case WAE_ATTR_NORMALIZE:
            if (n.kind != K_CONV) return wrong();
            n.normalize_next = value != 0.;
            return WAE_OK;
        case WAE_ATTR_OVERSAMPLE:
            if (n.kind != K_SHAPER) return wrong();
            if (!(value == 0. || value == 1. || value == 2.)) return fail(WAE_INVALID_ARGUMENT, "unknown oversample type");
            n.oversample = (int)value;
            return WAE_OK;
        case WAE_ATTR_PANNING_MODEL: case WAE_ATTR_DISTANCE_MODEL: case WAE_ATTR_REF_DISTANCE: case WAE_ATTR_MAX_DISTANCE:
        case WAE_ATTR_ROLLOFF_FACTOR: case WAE_ATTR_CONE_INNER_ANGLE: case WAE_ATTR_CONE_OUTER_ANGLE: case WAE_ATTR_CONE_OUTER_GAIN:
            if (n.kind != K_PANNER) return wrong();
            switch (attribute) {
                case WAE_ATTR_PANNING_MODEL:
                    if (!(value == 0. || value == 1.)) return fail(WAE_INVALID_ARGUMENT, "unknown panning model");
                    n.panning_model = (int)value;
                    break;
                case WAE_ATTR_DISTANCE_MODEL:
                    if (!(value == 0. || value == 1. || value == 2.)) return fail(WAE_INVALID_ARGUMENT, "unknown distance model");
                    n.distance_model = (int)value;
                    break;
                case WAE_ATTR_REF_DISTANCE:
                    if (!(value >= 0.)) return fail(WAE_INVALID_ARGUMENT, "RangeError - refDistance cannot be negative");
                    n.ref_distance = value;
                    break;
                case WAE_ATTR_MAX_DISTANCE:
                    if (!(value > 0.)) return fail(WAE_INVALID_ARGUMENT, "RangeError - maxDistance must be strictly positive");
                    n.max_distance = value;
                    break;
                case WAE_ATTR_ROLLOFF_FACTOR:
                    if (!(value >= 0.)) return fail(WAE_INVALID_ARGUMENT, "RangeError - rolloffFactor cannot be negative");
                    n.rolloff_factor = value;
                    break;
                case WAE_ATTR_CONE_INNER_ANGLE: n.cone_inner_angle = value; break;
                case WAE_ATTR_CONE_OUTER_ANGLE: n.cone_outer_angle = value; break;
                default:
                    if (!(value >= 0. && value <= 1.)) return fail(WAE_INVALID_STATE, "InvalidStateError - coneOuterGain must be in the range [0, 1]");
                    n.cone_outer_gain = value;
            }
            return WAE_OK;
        case WAE_ATTR_FFT_SIZE: {
            if (n.kind != K_ANALYSER) return wrong();
            const uint64_t f = (uint64_t)value;
            if (!((double)f == value && f >= 32 && f <= 32768 && (f & (f - 1)) == 0))
                return fail(WAE_INVALID_ARGUMENT, "IndexSizeError - Invalid fft size: must be a power of two in [32, 32768]");
            n.fft_size = (uint32_t)f;
            return WAE_OK;
        }
        case WAE_ATTR_SMOOTHING_TIME_CONSTANT:
            if (n.kind != K_ANALYSER) return wrong();
            if (!(value >= 0. && value <= 1.)) return fail(WAE_INVALID_ARGUMENT, "IndexSizeError - Invalid smoothing time constant: must be in [0, 1]");
            n.smoothing = value;
            return WAE_OK;
        case WAE_ATTR_MIN_DECIBELS:
            if (n.kind != K_ANALYSER) return wrong();
            if (!(value < n.max_db)) return fail(WAE_INVALID_ARGUMENT, "IndexSizeError - Invalid min decibels: must be less than max decibels");
            n.min_db = value;
            return WAE_OK;
        case WAE_ATTR_MAX_DECIBELS:
            if (n.kind != K_ANALYSER) return wrong();
            if (!(value > n.min_db)) return fail(WAE_INVALID_ARGUMENT, "IndexSizeError - Invalid max decibels: must be greater than min decibels");
            n.max_db = value;
            return WAE_OK;
        default: return fail(WAE_INVALID_ARGUMENT, "unknown attribute");
    }
}

// ---- AudioNode::set_channel_count / set_channel_count_mode / set_channel_interpretation -------------------------------------
// src/node/audio_node.rs:417-441 and the per-node overrides that narrow them.  `node` is the id create_* returned (a DelayNode
// is addressed by its writer, delay.rs:108-115, which is the half that has the mixed input).
namespace {
enum CfgField { F_COUNT, F_MODE, F_INTERP };
// returns "" when the value is allowed for this kind of node, else the reference's panic text
std::string channel_config_constraint(const wae_graph* g, const Node& n, CfgField f, uint32_t v) {
    switch (n.kind) {
        case K_PARAM:  // src/param.rs:325-333
            return f == F_COUNT ? "NotSupportedError - AudioParam has channel count constraints"
                 : f == F_MODE  ? "NotSupportedError - AudioParam has channel count mode constraints"
                                : "NotSupportedError - AudioParam has channel interpretation constraints";
        case K_LISTENER:  // src/spatial.rs:113-121
            return f == F_COUNT ? "NotSupportedError - AudioListenerNode has channel count constraints"
                 : f == F_MODE  ? "NotSupportedError - AudioListenerNode has channel count mode constraints"
                                : "NotSupportedError - AudioListenerNode has channel interpretation constraints";
        case K_DEST:  // src/node/destination.rs:55-96 (offline context)
            if (f == F_COUNT && v != g->channels) return "NotSupportedError - not allowed to change OfflineAudioContext destination channel count";
            if (f == F_MODE && v != WAE_COUNT_MODE_EXPLICIT) return "InvalidStateError - AudioDestinationNode has channel count mode constraints";
            return "";
        case K_MERGER:  // src/node/channel_merger.rs:39-62
            if (f == F_COUNT && v != 1) return "InvalidStateError - channel count of ChannelMergerNode must be equal to 1";
            if (f == F_MODE && v != WAE_COUNT_MODE_EXPLICIT) return "InvalidStateError - channel count of ChannelMergerNode must be set to Explicit";
            return "";
        case K_SPLITTER:  // src/node/channel_splitter.rs:36-78
            if (f == F_COUNT && v != (uint32_t)n.n_outputs) return "InvalidStateError - channel count of ChannelSplitterNode must be equal to number of outputs";
            if (f == F_MODE && v != WAE_COUNT_MODE_EXPLICIT) return "InvalidStateError - channel count mode of ChannelSplitterNode must be set to Explicit";
            if (f == F_INTERP && v != WAE_INTERPRETATION_DISCRETE) return "InvalidStateError - channel interpretation of ChannelSplitterNode must be set to Discrete";
            return "";
        case K_CONV: case K_COMP: case K_SPANNER: case K_PANNER: {  // convolver.rs:48-78, dynamics_compressor.rs:21-50, stereo_panner.rs:23-53, panner.rs
            const char* name = n.kind == K_CONV ? "ConvolverNode" : n.kind == K_COMP ? "DynamicsCompressorNode" : n.kind == K_SPANNER ? "StereoPannerNode" : "PannerNode";
            if (f == F_COUNT && v > 2) return std::string("NotSupportedError - ") + name + " channel count cannot be greater than two";
            if (f == F_MODE && v == WAE_COUNT_MODE_MAX) return std::string("NotSupportedError - ") + name + " channel count mode cannot be set to max";
            return "";
        }
        default:
            return "";
    }
}
wae_status set_channel_config_field(wae_graph* g, wae_node_id node, CfgField f, uint32_t v) {
    if (!g) return fail(WAE_INVALID_ARGUMENT, "null graph");
    auto ni = g->nodes.find(node);
    if (ni == g->nodes.end()) return fail(WAE_INVALID_ARGUMENT, "InvalidAccessError - unknown node");
    Node& n = ni->second;
    if (f == F_MODE && v > WAE_COUNT_MODE_EXPLICIT) return fail(WAE_INVALID_ARGUMENT, "unknown channel count mode");
    if (f == F_INTERP && v > WAE_INTERPRETATION_DISCRETE) return fail(WAE_INVALID_ARGUMENT, "unknown channel interpretation");
    std::string why = channel_config_constraint(g, n, f, v);
    if (!why.empty()) return fail(WAE_NOT_SUPPORTED, why);
    if (f == F_COUNT) {
        if (v < 1 || v > WAE_MAX_CHANNELS)  // assert_valid_number_of_channels, src/lib.rs:185-192
            return fail(WAE_NOT_SUPPORTED, "NotSupportedError - Invalid number of channels: " + std::to_string(v) + " is outside range [1, 32]");
        if (n.kind != K_MERGER && n.kind != K_SPLITTER) n.cfg.count = (int)v;  // those two only validate (channel_merger.rs:102-104)
    } else if (f == F_MODE) {
        n.cfg.mode = (int)v;
    } else {
        n.cfg.interp = (int)v;
    }
    return WAE_OK;
}
}  // namespace

WAE_API wae_status wae_node_set_channel_count(wae_graph* g, wae_node_id node, uint32_t count) { return set_channel_config_field(g, node, F_COUNT, count); }
WAE_API wae_status wae_node_set_channel_count_mode(wae_graph* g, wae_node_id node, uint32_t mode) { return set_channel_config_field(g, node, F_MODE, mode); }
WAE_API wae_status wae_node_set_channel_interpretation(wae_graph* g, wae_node_id node, uint32_t interpretation) {
    return set_channel_config_field(g, node, F_INTERP, interpretation);
}

// ---- control-side read-outs of the filter nodes (no device work) ---------------------------------------------------------
// calculate_coefs (src/node/biquad_filter.rs:42-390): the normalised coefficients the k_biquad / k_chain kernels are fed with
WAE_API void wae_biquad_coefs(uint32_t type, double sample_rate, double f0, double gain, double q, double* out5) {
    hostmath::BiquadCoefs c = hostmath::biquad_coefs((int)type, sample_rate, f0, gain, q);
    out5[0] = c.b0; out5[1] = c.b1; out5[2] = c.b2; out5[3] = c.a1; out5[4] = c.a2;
}
// BiquadFilterNode::get_frequency_response (src/node/biquad_filter.rs:657-735)
WAE_API void wae_biquad_frequency_response(uint32_t type, float sample_rate, float frequency, float detune, float q, float gain,
                                           const float* freq_hz, float* mag, float* phase, uint32_t n) {
    const float nyquist = sample_rate / 2.f;
    const float computed = hostmath::biquad_computed_freq(frequency, detune);
    const hostmath::BiquadCoefs c = hostmath::biquad_coefs((int)type, (double)sample_rate, (double)computed, (double)gain, (double)q);
    for (uint32_t i = 0; i < n; i++) {
        const float f = freq_hz[i];
        if (!(f >= 0.f && f <= nyquist)) {
            mag[i] = phase[i] = std::numeric_limits<float>::quiet_NaN();
            continue;
        }
        const double omega = -hostmath::PI64 * (double)(f / nyquist);
        const std::complex<double> z(std::cos(omega), std::sin(omega));
        const std::complex<double> h = (c.b0 + (c.b1 + c.b2 * z) * z) / (std::complex<double>(1., 0.) + (c.a1 + c.a2 * z) * z);
        mag[i] = (float)std::abs(h);
        phase[i] = (float)std::arg(h);
    }
}
// IIRFilterNode::get_frequency_response (src/node/iir_filter.rs:215-265)
WAE_API void wae_iir_frequency_response(const double* ff, uint32_t nff, const double* fb, uint32_t nfb, float sample_rate,
                                        const float* freq_hz, float* mag, float* phase, uint32_t n) {
    const float nyquist = sample_rate / 2.f;
    for (uint32_t i = 0; i < n; i++) {
        const float f = freq_hz[i];
        if (!(f >= 0.f && f <= nyquist)) {
            mag[i] = phase[i] = std::numeric_limits<float>::quiet_NaN();
            continue;
        }
        const double z = -2.0 * hostmath::PI64 * (double)f / (double)sample_rate;
        std::complex<double> num(0., 0.), den(0., 0.);
        for (uint32_t k = 0; k < nff; k++) num += std::polar(1.0, (double)k * z) * ff[k];  // Complex::from_polar(b, idx * z)
        for (uint32_t k = 0; k < nfb; k++) den += std::polar(1.0, (double)k * z) * fb[k];
        const std::complex<double> h = num / den;
        mag[i] = (float)std::abs(h);
        phase[i] = (float)std::arg(h);
    }
}

// One impulse response of the HRIR sphere resampled the way HrirSphere::new of the hrtf crate does when the context rate differs from the
// data's (csrc/wae_hrtf_host.h); the engine applies it to the whole sphere on first use of a rate.  Host work.
WAE_API wae_status wae_hrir_resample(const float* hrir, uint32_t len, double ratio, float* out, uint32_t cap, uint32_t* n) {
    if (!hrir || !n || !(ratio > 0.)) return fail(WAE_INVALID_ARGUMENT, "null argument / non-positive ratio");
    const SincBank bank(ratio >= 1.0 ? 0.95f : 0.95f * (float)ratio);
    const std::vector<float> r = hrir_resample(bank, hrir, len, ratio);
    *n = (uint32_t)r.size();
    for (uint32_t i = 0; i < *n && i < cap; i++) out[i] = r[i];
    return WAE_OK;
}

}  // extern "C"
