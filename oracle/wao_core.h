// ORACLE — TEST INFRASTRUCTURE ONLY.  Not part of the product; never linked into libwae_b200.so.
//
// CPU restatement (C++17, single thread per context) of web-audio-api-rs's OfflineAudioContext render
// path: src/render/{quantum,graph,thread}.rs + the per-quantum processors of src/node/*.rs and
// src/param.rs.  Same operation order and precisions as the reference (f64 where it uses f64,
// fma/fmaf exactly where it uses mul_add, no contraction elsewhere: build with -ffp-contract=off,
// FTZ/DAZ set while rendering like src/render/thread.rs:373-380).
//
// Parity status: pinned against the reference's own known-answer tests (tests/test_oracle_kat.py lists
// each vector with its reference file:line).  Third-party arithmetic that is not in the reference source tree
// (fft-convolver 0.3, hrtf 0.8.1, rubato 0.16, realfft 3.3) is restated from the published algorithms;
// see the header of the respective file for what is and is not pinned.
#pragma once
#include <cstdint>
#include <cstddef>
#include <cstring>
#include <array>
#include <cmath>
#include <vector>
#include <memory>
#include <map>
#include <string>
#include <algorithm>

namespace wao {

constexpr int RQ = 128;           // RENDER_QUANTUM_SIZE, src/lib.rs:18
constexpr int MAX_CHANNELS = 32;  // src/lib.rs:21

// ---- src/render/quantum.rs:12-74: Alloc — pool of Rc<[f32;128]> + shared zero buffer -------------
struct Buf {
    float d[RQ];
    int rc;
};

struct Alloc {
    std::vector<Buf*> pool;
    Buf zeroes;
    Alloc() {
        std::memset(zeroes.d, 0, sizeof(zeroes.d));
        zeroes.rc = 1 << 30;  // never returned to the pool
    }
    ~Alloc() {
        for (Buf* b : pool) delete b;
    }
    Buf* allocate() {
        if (!pool.empty()) {
            Buf* b = pool.back();
            pool.pop_back();
            b->rc = 1;
            return b;
        }
        Buf* b = new Buf;
        std::memset(b->d, 0, sizeof(b->d));
        b->rc = 1;
        return b;
    }
    void release(Buf* b) {
        if (b == &zeroes) return;
        if (--b->rc == 0) pool.push_back(b);
    }
};

// ---- src/render/quantum.rs:90-131: AudioRenderQuantumChannel (copy-on-write Rc) -------------------
class Channel {
  public:
    Buf* b = nullptr;
    Alloc* a = nullptr;
    Channel() {}
    Channel(Buf* b_, Alloc* a_) : b(b_), a(a_) {}  // takes ownership of one reference
    Channel(const Channel& o) : b(o.b), a(o.a) {
        if (b && b != &a->zeroes) b->rc++;
    }
    Channel(Channel&& o) noexcept : b(o.b), a(o.a) { o.b = nullptr; }
    Channel& operator=(const Channel& o) {
        if (this != &o) {
            Buf* nb = o.b;
            if (nb && nb != &o.a->zeroes) nb->rc++;
            if (b) a->release(b);
            b = nb;
            a = o.a;
        }
        return *this;
    }
    Channel& operator=(Channel&& o) noexcept {
        if (this != &o) {
            if (b) a->release(b);
            b = o.b;
            a = o.a;
            o.b = nullptr;
        }
        return *this;
    }
    ~Channel() {
        if (b) a->release(b);
    }
    const float* data() const { return b->d; }
    // quantum.rs:96-104 make_mut: clone when shared
    float* make_mut() {
        if (b == &a->zeroes || b->rc != 1) {
            Buf* nb = a->allocate();
            std::memcpy(nb->d, b->d, sizeof(nb->d));
            a->release(b);
            b = nb;
        }
        return b->d;
    }
    // quantum.rs:109-111
    bool is_silent() const { return b == &a->zeroes; }
    // quantum.rs:114-120
    void add(const Channel& other) {
        if (is_silent()) {
            *this = other;
        } else if (!other.is_silent()) {
            float* d = make_mut();
            const float* s = other.data();
            for (int i = 0; i < RQ; i++) d[i] += s[i];
        }
    }
    Channel silence() const { return Channel(&a->zeroes, a); }
};

enum CountMode { MODE_MAX = 0, MODE_CLAMPED_MAX = 1, MODE_EXPLICIT = 2 };
enum Interp { SPEAKERS = 0, DISCRETE = 1 };
struct ChannelConfig {
    int count = 2;
    int mode = MODE_MAX;
    int interp = SPEAKERS;
};

// ---- src/render/quantum.rs:179-586: AudioRenderQuantum -------------------------------------------
class Quantum {
  public:
    std::vector<Channel> ch;  // 1..=32 channels
    bool single_valued = false;

    explicit Quantum(const Channel& c) {
        ch.reserve(8);
        ch.push_back(c);
    }
    int number_of_channels() const { return (int)ch.size(); }
    // quantum.rs:221-227
    void set_number_of_channels(int n) {
        for (int i = number_of_channels(); i < n; i++) ch.push_back(ch[0]);
        ch.resize(n, ch[0]);
    }
    const Channel& channel(int i) const { return ch[i]; }
    Channel& channel_mut(int i) { return ch[i]; }
    bool is_silent() const {
        for (auto& c : ch)
            if (!c.is_silent()) return false;
        return true;
    }
    void mix(int computed, int interp) {
        if (number_of_channels() == computed) return;
        mix_inner(computed, interp);
    }
    void mix_inner(int computed, int interp);
    // quantum.rs:512-517
    void make_silent() {
        Channel s = ch[0].silence();
        ch[0] = s;
        ch.resize(1, s);
    }
    void force_mono() { ch.resize(1, ch[0]); }
    void add(const Quantum& other, const ChannelConfig& cfg);
    bool all_channels_identical() const {
        for (size_t i = 1; i < ch.size(); i++)
            if (ch[i].b != ch[0].b) return false;
        return true;
    }
};

// ---- src/render/processor.rs:38-45 ---------------------------------------------------------------
struct Scope {
    uint64_t current_frame;
    double current_time;
    float sample_rate;
};

class Graph;
struct ParamSlice {
    const float* p;
    int len;  // 1 or 128
    float operator[](int i) const { return p[i]; }
};
// src/render/processor.rs:204-247 AudioParamValues::get
struct ParamValues {
    Graph* g;
    ParamSlice get(uint32_t param_id) const;
};

// ---- src/render/processor.rs:131-196 AudioProcessor ------------------------------------------------
struct Processor {
    virtual ~Processor() {}
    virtual bool process(std::vector<Quantum>& inputs, std::vector<Quantum>& outputs, const ParamValues& params,
                         const Scope& scope) = 0;
    virtual bool has_side_effects() const { return false; }
    virtual const char* name() const = 0;
};

struct Edge {
    int self_index;
    uint32_t other_id;
    int other_index;  // -1 == usize::MAX hidden param edge
};

struct Node {
    std::unique_ptr<Processor> processor;
    std::vector<Quantum> inputs, outputs;
    ChannelConfig cfg;
    std::vector<Edge> outgoing;
    bool cycle_breaker = false;
    bool has_inputs_connected = false;
};

// ---- src/render/graph.rs ---------------------------------------------------------------------------
class Graph {
  public:
    Alloc alloc;
    std::map<uint32_t, std::unique_ptr<Node>> nodes;  // NodeCollection: ascending id iteration
    std::vector<uint32_t> ordered, marked, marked_temp, in_cycle, cycle_breakers;

    void add_node(uint32_t id, std::unique_ptr<Processor> p, int n_in, int n_out, ChannelConfig cfg);
    void add_edge(uint32_t src, int out, uint32_t dst, int in);
    void remove_edges_from(uint32_t src);
    void mark_cycle_breaker(uint32_t id) { nodes.at(id)->cycle_breaker = true; }
    Node* get(uint32_t id) { return nodes.at(id).get(); }
    const Quantum& render(const Scope& scope);
    const std::vector<uint32_t>& order() {
        if (ordered.empty()) order_nodes();
        return ordered;
    }

  private:
    bool visit(uint32_t id);
    void order_nodes();
};

inline bool is_normal(double v) { return std::isnormal(v); }
inline bool is_normal(float v) { return std::isnormal(v); }

}  // namespace wao
