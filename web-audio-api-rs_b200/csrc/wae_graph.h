// Host-side graph description built through the C ABI (include/wae.h).
//
// This is the control half of the engine: what the reference keeps in its control-thread structs
// (XxxNode, AudioParam, ConcreteBaseAudioContext::connections — src/context/concrete_base.rs) and ships to
// the render thread as ControlMessages (src/message.rs:13-87).  Nothing here renders; wae_plan.cpp lowers a
// batch of these descriptions into GPU stages.
#pragma once
#include "../../include/wae.h"

#include <algorithm>
#include <cstdint>
#include <map>
#include <memory>
#include <stdexcept>
#include <type_traits>
#include <utility>
#include <string>
#include <vector>

namespace wae {

enum Kind : int {
    K_DEST = 0, K_PARAM, K_OSC, K_BIQUAD, K_IIR, K_GAIN, K_ABSN, K_CONST, K_CONV, K_SHAPER, K_DELAY_W, K_DELAY_R,
    K_SPANNER, K_PANNER, K_ANALYSER, K_COMP, K_MERGER, K_SPLITTER, K_LISTENER, K_KINDS
};

struct ChannelCfg {
    int count = 2, mode = WAE_COUNT_MODE_MAX, interp = WAE_INTERPRETATION_SPEAKERS;
};

// Host memory of AudioBuffer assets.  When the graph belongs to an engine the samples live in page-locked memory drawn from a
// process-wide pool (slabs of cudaHostAlloc memory, recycled by size), so that the render call can DMA them to the device at full
// PCIe speed straight from where `wae_create_buffer_source` / `set_buffer` put them — the counterpart of the reference moving the
// `Arc<AudioBuffer>` to its render thread (audio_buffer_source.rs:853-866).  Without an engine (CPU-only planning / validation) or
// when page-locking fails it is ordinary heap memory.
void* pcm_host_alloc(size_t bytes, bool want_pinned, bool* pinned);
void pcm_host_free(void* p, size_t bytes, bool pinned);

struct PcmChannel {  // one channel of a PcmBuffer: a view with the std::vector surface the planner uses
    float* p = nullptr;
    size_t n = 0;
    float* data() { return p; }
    const float* data() const { return p; }
    size_t size() const { return n; }
    float& operator[](size_t i) { return p[i]; }
    const float& operator[](size_t i) const { return p[i]; }
    float* begin() { return p; }
    float* end() { return p + n; }
    const float* begin() const { return p; }
    const float* end() const { return p + n; }
};

struct PcmBuffer {  // an AudioBuffer asset (src/buffer.rs:69-72), host copy: ONE block, planar [ch][stride], stride = len rounded up to 4
                    // floats with zeroed padding — the layout of the device copy (every channel starts 16 B aligned)
    std::vector<PcmChannel> channels;
    float sample_rate = 0.f;
    float* base = nullptr;
    size_t stride = 0, bytes = 0;
    bool pinned = false;
    // wae_buffer_source_set_device_input: a placeholder of the declared shape (channels[c].n = length) with no host block; its PCM is
    // written into the device slab by wae_batch_bind_sources, and nothing copies host memory over it.  The response of a ConvolverNode
    // declared with wae_convolver_set_device_response is such a placeholder too: its spectra are written by wae_batch_bind_responses
    bool device_input = false;
    // wae_buffer_source_set_device_input_by_reference: a device input read where the caller keeps it (no slab memory, nothing copied)
    bool by_reference = false;
    PcmBuffer() = default;
    PcmBuffer(const PcmBuffer&) = delete;
    PcmBuffer& operator=(const PcmBuffer&) = delete;
    ~PcmBuffer() {
        if (base) pcm_host_free(base, bytes, pinned);
    }
    bool allocate(size_t n_channels, size_t len, bool want_pinned) {
        stride = (len + 3) / 4 * 4;
        bytes = std::max<size_t>(n_channels * stride, 4) * sizeof(float);
        base = static_cast<float*>(pcm_host_alloc(bytes, want_pinned, &pinned));
        if (!base) return false;
        channels.resize(n_channels);
        for (size_t c = 0; c < n_channels; c++) {
            channels[c].p = base + c * stride;
            channels[c].n = len;
            for (size_t i = len; i < stride; i++) channels[c].p[i] = 0.f;
        }
        return true;
    }
    size_t length() const { return channels.empty() ? 0 : channels[0].size(); }
    double duration() const { return (double)length() / (double)sample_rate; }
};

struct ParamEv {
    int type = 0;
    float value = 0.f;
    double time = 0., aux = 0.;
    std::vector<float> values;
};

struct Param {  // AudioParam: its own graph node in the reference (src/context/base.rs:320-337)
    float default_value = 0.f, min_value = 0.f, max_value = 0.f;  // (initialised: every Node carries a Param, only K_PARAM nodes use it)
    bool a_rate = false;
    bool rate_constrained = false;
    std::vector<ParamEv> events;  // in arrival order
    // wae_param_set_device_value: the value is supplied per run from device memory (wae_batch_bind_params), clamped to
    // [device_lo, device_hi] (the declared range intersected with [min_value, max_value]); planned as constant_value()
    bool device_bound = false;
    float device_lo = 0.f, device_hi = 0.f;
    // wae_param_set_device_value_curve: the length of the SetValueCurveAtTime event whose values are written per run by
    // wae_batch_bind_value_curves.  That event is the last of `events` (its `values` are zero placeholders): the param takes no further
    // events, so the planner never replays its timeline on the host.  0: not declared
    uint32_t device_curve = 0;
    uint32_t device_curve_node = 0, device_curve_index = 0;  // the (node, param index) it was declared through: its name in binds
    // lowering helpers
    bool constant() const;        // only SetValue events: value is constant over the render
    float constant_value() const; // clamped like AudioParamProcessor::mix_to_output (src/param.rs:755-760)
};

struct Edge {
    int self_index;
    uint32_t other_id;
    int other_index;  // -1: hidden param port (usize::MAX in the reference)
};

struct Node {
    uint32_t id = 0;
    Kind kind = K_DEST;
    uint32_t out_id = 0;  // DelayNode: outputs come from the reader (src/node/delay.rs:128-159)
    int n_inputs = 1, n_outputs = 1;
    ChannelCfg cfg;
    std::vector<uint32_t> params;  // param node ids, creation order
    std::vector<Edge> outgoing;
    bool cycle_breaker = false;
    bool has_start = false;

    // per-kind options
    int type = 0;  // oscillator / biquad type
    std::vector<float> table;  // periodic wave / shaper curve
    bool has_curve = false;
    // wae_wave_shaper_set_device_curve: the curve's length (has_curve is set, `table` stays empty); its points are written by
    // wae_batch_bind_curves.  0: not declared
    uint32_t device_curve = 0;
    // wae_oscillator_set_device_periodic_wave: the coefficient count of the wave (type is Custom, `table` stays empty), the length of
    // the wavetable wae_batch_bind_periodic_waves synthesises from the bound coefficients, and whether it is normalised.  0: not declared
    uint32_t device_wave = 0;
    uint32_t device_wave_len = 0;
    bool device_wave_normalize = true;
    int oversample = 0;  // WaveShaper: WAE_OVERSAMPLE_*
    std::vector<double> feedforward, feedback;  // IIR
    // wae_iir_filter_set_device_coefficients: the coefficients are written per run by wae_batch_bind_iir_coefficients (as many as
    // `feedforward` / `feedback` hold: the plan is made with these constructed ones)
    bool device_iir = false;
    std::shared_ptr<PcmBuffer> buffer;          // ABSN buffer / convolver IR
    bool normalize = true;                      // convolver: the scale the CURRENT buffer was given (taken when the buffer is set)
    bool normalize_next = true;                 // ConvolverNode::set_normalize: applies to the next set_buffer (convolver.rs:325-328)
    double start_time = 1.7976931348623157e308, stop_time = 1.7976931348623157e308;
    double offset = 0., duration = 1.7976931348623157e308;
    // wae_source_set_device_schedule: the start time (and, with sched_stop, the stop time) is written per run by wae_batch_bind_schedules,
    // clamped to [sched_lo, sched_hi] (index 0: start, 1: stop).  start_time / stop_time hold the windows' low ends: the plan is made
    // with them, always with a gated output layout, so no planning decision depends on the bound times.
    // wae_buffer_source_set_device_offset extends the declaration of an AudioBufferSourceNode with its offset (index 2) and, with
    // sched_duration, its duration (index 3); offset / duration hold those windows' low ends.
    bool device_schedule = false;
    bool sched_stop = false, sched_offset = false, sched_duration = false;
    double sched_lo[4] = {0., 0., 0., 0.}, sched_hi[4] = {0., 0., 0., 0.};
    bool loop = false;
    double loop_start = 0., loop_end = 0.;
    // wae_buffer_source_set_device_loop: loop_start / loop_end are written per run by wae_batch_bind_loops, clamped to [loop_lo, loop_hi]
    // (index 0: start, 1: end); loop_start / loop_end hold the windows' low ends, which the plan is made with
    bool device_loop = false;
    double loop_lo[2] = {0., 0.}, loop_hi[2] = {0., 0.};
    double max_delay_time = 1.;
    uint32_t delay_peer = 0;  // writer <-> reader
    // panner
    int panning_model = 0, distance_model = 1;
    double ref_distance = 1., max_distance = 10000., rolloff_factor = 1., cone_inner_angle = 360., cone_outer_angle = 360.,
           cone_outer_gain = 0.;
    // analyser
    uint32_t fft_size = 2048;
    double smoothing = 0.8, min_db = -100., max_db = -30.;
    // wae_analyser_set_readouts / wae_compressor_set_readouts: the read-out quanta (non-decreasing).  Empty: not declared
    std::vector<uint64_t> readout_q;
    uint32_t readout_kinds = 0;       // analyser: WAE_READOUT_* kinds
    uint32_t byte_readout_kinds = 0;  // analyser: the kinds also delivered as bytes (wae_analyser_set_byte_readouts)
    Param param;  // K_PARAM only
};

// node id -> Node.  Ids are handed out densely (wae_graph::next_id), so this is a table indexed by id, not a tree: the planner walks all
// nodes of every graph several times per pass and looks them up per edge.  Surface of the std::map it replaces where the code uses it
// (iteration in id order yielding (id, node) pairs, find / at / operator[]); every node is its own allocation, so references to nodes
// stay valid while nodes are added (the graph-building calls hold some across create_param).
class NodeMap {
  public:
    using value_type = std::pair<const uint32_t, Node>;
    template <bool Const>
    class Iter {
        using Map = typename std::conditional<Const, const NodeMap, NodeMap>::type;
        using Ref = typename std::conditional<Const, const value_type, value_type>::type;
        Map* m = nullptr;
        size_t i = 0;
        void skip() {
            while (i < m->slots.size() && !m->slots[i]) i++;
        }
        friend class NodeMap;
        Iter(Map* map, size_t at) : m(map), i(at) { skip(); }

      public:
        Iter() = default;
        Ref& operator*() const { return *m->slots[i]; }
        Ref* operator->() const { return m->slots[i].get(); }
        Iter& operator++() {
            i++;
            skip();
            return *this;
        }
        bool operator==(const Iter& o) const { return i == o.i; }
        bool operator!=(const Iter& o) const { return i != o.i; }
    };
    using iterator = Iter<false>;
    using const_iterator = Iter<true>;
    NodeMap() = default;
    NodeMap(NodeMap&&) = default;
    NodeMap& operator=(NodeMap&&) = default;
    NodeMap(const NodeMap& o) : slots(o.slots.size()), count_(o.count_), max_id_(o.max_id_) {  // (suspend_sync keeps the graph as it was: a deep copy)
        for (size_t i = 0; i < o.slots.size(); i++)
            if (o.slots[i]) slots[i] = std::make_unique<value_type>(*o.slots[i]);
    }
    NodeMap& operator=(const NodeMap& o) {
        if (this != &o) {
            NodeMap c(o);
            *this = std::move(c);
        }
        return *this;
    }
    iterator begin() { return iterator(this, 0); }
    iterator end() { return iterator(this, slots.size()); }
    const_iterator begin() const { return const_iterator(this, 0); }
    const_iterator end() const { return const_iterator(this, slots.size()); }
    iterator find(uint32_t id) { return id < slots.size() && slots[id] ? iterator(this, id) : end(); }
    const_iterator find(uint32_t id) const { return id < slots.size() && slots[id] ? const_iterator(this, id) : end(); }
    Node* get(uint32_t id) { return id < slots.size() && slots[id] ? &slots[id]->second : nullptr; }
    const Node* get(uint32_t id) const { return id < slots.size() && slots[id] ? &slots[id]->second : nullptr; }
    Node& at(uint32_t id) {
        Node* n = get(id);
        if (!n) throw std::out_of_range("unknown node id");
        return *n;
    }
    const Node& at(uint32_t id) const {
        const Node* n = get(id);
        if (!n) throw std::out_of_range("unknown node id");
        return *n;
    }
    Node& operator[](uint32_t id) {
        if (id >= slots.size()) slots.resize(std::max<size_t>((size_t)id + 1, slots.size() * 2));
        if (!slots[id]) {
            slots[id] = std::make_unique<value_type>(id, Node{});
            count_++;
            if (id > max_id_ || count_ == 1) max_id_ = id;
        }
        return slots[id]->second;
    }
    size_t size() const { return count_; }
    bool empty() const { return count_ == 0; }
    uint32_t max_id() const { return max_id_; }  // (of a non-empty map)

  private:
    std::vector<std::unique_ptr<value_type>> slots;
    size_t count_ = 0;
    uint32_t max_id_ = 0;
};

}  // namespace wae

struct wae_graph {
    wae_engine* engine = nullptr;
    uint32_t channels = 0;
    uint64_t length = 0;
    float sample_rate = 0.f;
    uint32_t next_id = 11;  // src/context/mod.rs:24-40
    wae::NodeMap nodes;
    std::vector<std::pair<uint32_t, uint32_t>> pending_param_edges;
    bool listener_present = false;
    // OfflineAudioContext::suspend_sync (src/context/offline.rs:330-387): `epochs[k]` is the graph as it was before the k-th
    // suspend point, valid for the frames before `frame`; the live `nodes` describe the frames after the last suspend point
    struct Epoch {
        uint64_t frame;
        wae::NodeMap nodes;
    };
    std::vector<Epoch> epochs;
    // AudioBuffer assets of this graph, by pin mode: a buffer handed in again (the reference clones an Arc: one `AudioBuffer` played by
    // hundreds of grains, src/buffer.rs:69-72) shares ONE host copy — and so one copy in the device slab (Planner::buf_offsets)
    std::vector<std::weak_ptr<wae::PcmBuffer>> assets[2];
    uint32_t device_inputs = 0;  // AudioBufferSourceNodes declared with wae_buffer_source_set_device_input (never in `assets`)
    uint32_t device_params = 0;  // AudioParams declared with wae_param_set_device_value
    uint32_t device_responses = 0;  // ConvolverNodes declared with wae_convolver_set_device_response (never in `assets`)
    uint32_t device_curves = 0;     // WaveShaperNodes declared with wae_wave_shaper_set_device_curve
    uint32_t device_waves = 0;      // OscillatorNodes declared with wae_oscillator_set_device_periodic_wave
    uint32_t device_iirs = 0;       // IIRFilterNodes declared with wae_iir_filter_set_device_coefficients
    uint32_t device_value_curves = 0;  // AudioParams declared with wae_param_set_device_value_curve
    uint32_t device_schedules = 0;     // scheduled sources declared with wae_source_set_device_schedule
    uint32_t device_loops = 0;         // AudioBufferSourceNodes declared with wae_buffer_source_set_device_loop
    uint32_t analyser_readouts = 0;    // AnalyserNodes declared with wae_analyser_set_readouts
    uint32_t compressor_readouts = 0;  // DynamicsCompressorNodes declared with wae_compressor_set_readouts

    uint32_t create_param(uint32_t owner, float def, float mn, float mx, bool a_rate, float initial, bool send_set_value = true,
                          bool fixed_id = false, uint32_t id = 0, bool constrained = false);
    wae::Node& finish_register(wae::Node n);
    void ensure_listener();
    void add_edge(uint32_t src, int out, uint32_t dst, int in) { nodes.at(src).outgoing.push_back(wae::Edge{out, dst, in}); }
};

namespace wae {
int engine_device(const wae_engine* eng);  // CUDA device ordinal of an engine (wae_engine.cu)
void set_error(const std::string& msg);
int32_t fail(int32_t code, const std::string& msg);
}  // namespace wae
