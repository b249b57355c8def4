// Engine + planner: lowers a batch of graph descriptions (wae_graph.h) into GPU stages (wae_device.h) and runs
// them chunk by chunk on one CUDA stream.  C ABI: wae_engine_*, wae_batch_*, wae_render_batch (include/wae.h).
//
// Reference functions replaced by this file:
//   RenderThread::render_audiobuffer_sync / render_offline_quantum   src/render/thread.rs:260-302,355-396
//   Graph::order_nodes / visit / render                              src/render/graph.rs:331-591
//   (the per-node arithmetic is in wae_kernels.cu)
#include "wae_graph.h"
#include "wae_hostmath.h"
#include "wae_hrtf_host.h"
#include "wae_resample_host.h"
#include "wae_kernels.h"
#include "wae_param_core.h"
#include "wae_param_host.h"

#include <cuda.h>  // (types of cuMemGetAddressRange only: it is reached through cudaGetDriverEntryPoint)
#include <cuda_runtime.h>
#include <emmintrin.h>

#include <algorithm>
#include <array>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdlib>
#include <deque>
#include <fstream>
#include <mutex>
#include <sched.h>
#include <sstream>
#include <thread>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <functional>
#include <limits>
#include <map>
#include <memory>
#include <set>
#include <tuple>
#include <unordered_map>
#include <unordered_set>

using namespace wae;
namespace hm = wae::hostmath;

#define CUDA_TRY(expr)                                                                                       \
    do {                                                                                                     \
        cudaError_t _e = (expr);                                                                             \
        if (_e != cudaSuccess) return fail(WAE_CUDA_ERROR, std::string(#expr) + ": " + cudaGetErrorString(_e)); \
    } while (0)

// host worker threads of an engine: planning of graph groups and the copy-out of rendered PCM to pageable caller memory
struct WorkerPool {
    std::vector<std::thread> threads;
    std::mutex mu;
    std::condition_variable cv;
    std::deque<std::function<void()>> q;
    bool stop = false;
    WorkerPool(int n, int device) {
        for (int i = 0; i < n; i++)
            threads.emplace_back([this, device] {
                cudaSetDevice(device);
                for (;;) {
                    std::function<void()> f;
                    {
                        std::unique_lock<std::mutex> lk(mu);
                        cv.wait(lk, [this] { return stop || !q.empty(); });
                        if (q.empty()) return;
                        f = std::move(q.front());
                        q.pop_front();
                    }
                    f();
                }
            });
    }
    ~WorkerPool() {
        {
            std::lock_guard<std::mutex> lk(mu);
            stop = true;
        }
        cv.notify_all();
        for (auto& t : threads) t.join();
    }
    void submit(std::function<void()> f) {
        {
            std::lock_guard<std::mutex> lk(mu);
            q.push_back(std::move(f));
        }
        cv.notify_one();
    }
    int size() const { return (int)threads.size(); }
    // fn(i) for i in [0, n), on the workers; returns when all are done
    void parallel_for(int n, const std::function<void(int)>& fn) {
        if (n <= 0) return;
        std::mutex dm;
        std::condition_variable dcv;
        int left = n;
        for (int i = 0; i < n; i++)
            submit([&, i] {
                fn(i);
                std::lock_guard<std::mutex> lk(dm);
                if (--left == 0) dcv.notify_all();
            });
        std::unique_lock<std::mutex> lk(dm);
        dcv.wait(lk, [&] { return left == 0; });
    }
};

struct wae_engine {
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaStream_t s_h2d = nullptr, s_d2h = nullptr;  // copy streams of the pipelined / one-shot paths
    int64_t chunk_frames = 0;  // 0 = auto
    bool fuse = true;
    int voice_sum = -1;  // WAE_OPT_VOICE_SUM: fused oscillator voices + ordered sum (k_voice_sum); -1: WAE_VOICE_SUM from the environment, default on
    bool serial_filters = false;
    int pipeline_groups = 0;  // 0 = auto
    int param_parallel = 2;  // WAE_OPT_PARAM_PARALLEL: 2 k_param_spec (CTA per param, speculative walks of 32 quanta), 1 k_param_parallel (warp per param), 0 k_param (lane 0 evaluates every frame)
    float* d_sine = nullptr;
    wae::HrirSphere* sphere = nullptr;  // wae_engine_set_hrir_sphere
    float* d_sphere_ir = nullptr;
    float* d_sphere_pos = nullptr;
    uint32_t* d_sphere_tri = nullptr;
    uint64_t sphere_gen = 0;  // counts the spheres wae_engine_set_hrir_sphere installed (a bind checks that its batch's is still there)
    struct RateSphere {  // the sphere's responses resampled to a context rate (HrirSphere::new of the crate), built on first use
        float* d_ir = nullptr;
        uint32_t taps = 0;
        std::vector<float> ir_host;  // [vertex][2][taps] (static panners: blended on the host into the response of a convolution)
    };
    std::map<uint32_t, RateSphere> sphere_rates;
    std::mutex sphere_mu;
    void drop_rate_spheres() {
        for (auto& kv : sphere_rates)
            if (kv.second.d_ir) cudaFree(kv.second.d_ir);
        sphere_rates.clear();
    }
    // ---- device memory of finished batches is kept and handed to the next batch (a render call that prepares, renders and drops
    // its batch would otherwise pay cudaMalloc / cudaFree — both synchronising — for gigabytes of PCM every time)
    std::mutex mem_mu;
    std::multimap<size_t, void*> dev_free;          // cached blocks by size
    std::unordered_map<void*, size_t> dev_size;     // every live block (handed out or cached)
    size_t dev_cached_bytes = 0;
    static size_t round_block(size_t b) {
        if (b < 512) return 512;
        if (b < ((size_t)1 << 16)) return (b + 511) / 512 * 512;
        if (b < ((size_t)2 << 20)) return (b + 65535) / 65536 * 65536;
        return (b + (((size_t)2 << 20) - 1)) / ((size_t)2 << 20) * ((size_t)2 << 20);
    }
    void* dev_alloc(size_t bytes, bool* fresh = nullptr) {
        const size_t r = round_block(bytes);
        {
            std::lock_guard<std::mutex> lk(mem_mu);
            auto it = dev_free.lower_bound(r);
            if (it != dev_free.end() && it->first <= r + std::max<size_t>(r / 8, 4096)) {
                void* p = it->second;
                dev_cached_bytes -= it->first;
                dev_free.erase(it);
                if (fresh) *fresh = false;
                return p;
            }
        }
        void* p = nullptr;
        if (cudaMalloc(&p, r) != cudaSuccess) {
            cudaGetLastError();
            dev_trim();  // give the cache back and try once more
            if (cudaMalloc(&p, r) != cudaSuccess) {
                cudaGetLastError();
                return nullptr;
            }
        }
        std::lock_guard<std::mutex> lk(mem_mu);
        dev_size[p] = r;
        if (fresh) *fresh = true;
        return p;
    }
    void dev_release(void* p) {
        std::lock_guard<std::mutex> lk(mem_mu);
        auto it = dev_size.find(p);
        if (it == dev_size.end()) return;
        dev_free.emplace(it->second, p);
        dev_cached_bytes += it->second;
    }
    void dev_trim() {
        std::lock_guard<std::mutex> lk(mem_mu);
        for (auto& kv : dev_free) {
            cudaFree(kv.second);
            dev_size.erase(kv.second);
        }
        dev_free.clear();
        dev_cached_bytes = 0;
    }
    // ---- host side of the one-shot render: worker threads, page-locked staging slots for pageable output buffers
    WorkerPool* pool = nullptr;
    int n_workers = 0;  // 0 = auto
    WorkerPool* workers() {
        if (!pool) {
            int n = n_workers;
            if (n <= 0) {
                const unsigned hw = std::thread::hardware_concurrency();
                n = (int)std::min<unsigned>(16u, std::max<unsigned>(2u, hw / 8u));
            }
            pool = new WorkerPool(n, device);
        }
        return pool;
    }
    static constexpr int kStageSlots = 4;
    float* h_stage[kStageSlots] = {nullptr, nullptr, nullptr, nullptr};
    size_t h_stage_bytes = 0;
    bool ensure_stage(size_t bytes) {
        if (h_stage_bytes >= bytes) return true;
        for (int i = 0; i < kStageSlots; i++) {
            if (h_stage[i]) cudaFreeHost(h_stage[i]);
            h_stage[i] = nullptr;
        }
        h_stage_bytes = 0;
        for (int i = 0; i < kStageSlots; i++)
            if (cudaHostAlloc((void**)&h_stage[i], bytes, cudaHostAllocDefault) != cudaSuccess) {
                cudaGetLastError();
                return false;
            }
        h_stage_bytes = bytes;
        return true;
    }
    // small ring of page-locked pieces for the copy-out to pageable caller memory (render_oneshot_host)
    char* h_ring = nullptr;
    size_t h_ring_bytes = 0;
    bool ensure_ring(size_t bytes) {
        if (h_ring_bytes >= bytes) return true;
        if (h_ring) cudaFreeHost(h_ring);
        h_ring = nullptr;
        h_ring_bytes = 0;
        if (cudaHostAlloc((void**)&h_ring, bytes, cudaHostAllocDefault) != cudaSuccess) {
            cudaGetLastError();
            return false;
        }
        h_ring_bytes = bytes;
        return true;
    }
    std::string numa_cpus;  // CPUs this engine's host threads were bound to (WAE_OPT_BIND_NUMA), for the record
};

namespace wae {
int engine_device(const wae_engine* eng) { return eng ? eng->device : 0; }
}  // namespace wae

namespace {

// (the order of the kinds is the launch order inside one level: mixes first; k_delay_mono before the delay reader that needs it)
enum StageKind : int {
    S_MIX = 0, S_MIX_DYN, S_OSC, S_CONST, S_ABSN, S_BIQUAD, S_IIR, S_GAIN, S_SHAPER, S_SPAN, S_PAN, S_ROUTE, S_DELAY_MONO, S_DELAY, S_DELAY_WRITE, S_COMP, S_ANALYSER,
    S_CONV_FFT, S_CONV_MAC, S_CONV_MAC_ACC, S_CHAIN, S_PARAM, S_OSC_AR, S_BIQUAD_AR, S_ABSN_SLOW, S_HRTF, S_PAN_DYN, S_ABSN_SERIAL, S_SHAPER_OS, S_META, S_VSUM, S_CONV_CMP, S_ABSN_BOUND,
    S_READOUT_FFT, S_READOUT_TIME, S_READOUT_SMOOTH, S_KINDS  // (launched before S_ANALYSER of their level: Planner::stage)
};
const char* kStageNames[S_KINDS] = {"k_mix", "k_mix_dyn", "k_oscillator", "k_constant", "k_buffer_source", "k_biquad_serial", "k_iir_serial", "k_gain",
                                    "k_shaper", "k_stereo_panner", "k_panner_eq", "k_route", "k_delay_mono", "k_delay_read", "k_ring_write", "k_compressor",
                                    "k_analyser", "k_conv_fft_in", "k_conv_mac_ifft", "k_conv_mac_ifft(acc)", "k_chain", "k_param", "k_osc_arate", "k_biquad_arate", "k_buffer_source_slow", "k_hrtf_fir", "k_panner_dyn", "k_buffer_source_serial", "k_shaper_os", "k_meta", "k_voice_sum", "k_conv_compact",
                                    "k_buffer_source_slow(bound)", "k_readout_fft", "k_readout_time", "k_readout_smooth"};

// Bind entries: what prepare uploads for the binds from device memory to rewrite planned records.  The planner records one Entry per
// device entry in the stage whose records it reaches.  Its payload is the device entry; the payload's pointers into the stage's records
// are named by references (table, record, offset into the record) until the tables are uploaded: merge_builds rebases the records,
// prep_plan_group writes each address into the payload field `field` bytes from its start.  Prepare uploads the entries of each kind
// in group, stage and planning order.
enum EntryKind : int32_t {
    E_PARAM,      // ParamPatch (d_patches): a param bound from device memory (wae_param_set_device_value); operands name their param by
                  // node id (slot) until prepare numbers the value slots
    E_SPATIAL,    // SpatialPatch (d_spatial): a static panner whose source or listener is bound from device memory, operands as E_PARAM
    E_CURVE,      // CurvePatch (d_curve_patches): the int32 field that takes `keeps` or `other` as a bound curve maps 0 to 0 or not
    E_IIR,        // IirPatch (d_iir_patches): the coefficients of an IirInst or a ChainBiquad, and that biquad's scan constants
    E_SCHED,      // SchedPatch (d_sched_patches): the fields of a source whose start and stop times are bound from device memory
    E_LOOP,       // LoopPatch (d_loop_patches): a record whose loop points are bound from device memory
    E_LOOP_WALK,  // LoopWalk (d_loop_walks): a looping S_ABSN_BOUND record whose playhead table is derived on the device
    E_OUT,        // OutPatch (d_out_patches): the BufRef::p of a destination writer (wae_batch_bind_output)
    E_SRC_REF,    // SrcRefPatch (d_src_refs): the PCM pointer and channel stride of a source declared by reference
    E_KINDS
};
constexpr size_t kEntryPayloadBytes[E_KINDS] = {sizeof(ParamPatch), sizeof(SpatialPatch), sizeof(CurvePatch), sizeof(IirPatch),
                                                sizeof(SchedPatch), sizeof(LoopPatch), sizeof(LoopWalk), sizeof(OutPatch), sizeof(SrcRefPatch)};
enum StageTable : int32_t { T_NONE = 0, T_A, T_B, T_C };  // Stage::d_a, d_b, d_c (see StageBuild::table)
struct FieldRef {
    int32_t table;   // StageTable
    int32_t rec;     // record of that table
    uint32_t off;    // bytes into the record
    uint32_t field;  // bytes into the payload of the pointer that takes the address
};
struct Entry {  // (trivially copyable, made zeroed by Planner::entry: its bytes are digested)
    int32_t kind;      // EntryKind
    uint32_t graph;    // batch position
    wae_node_id node;  // the declaration a node-level kind belongs to (E_CURVE, E_IIR, E_SCHED, E_LOOP, E_SRC_REF), else 0
    FieldRef ref[3];   // T_NONE: unused (addresses the planner sets itself are in the payload already)
    union Payload {
        ParamPatch param;
        SpatialPatch spatial;
        CurvePatch curve;
        IirPatch iir;
        SchedPatch sched;
        LoopPatch loop;
        LoopWalk walk;
        OutPatch out;
        SrcRefPatch src_ref;
    } p;
    float2* spec;  // SPATIAL_RESP: the spectra of `S` partitions its bind transforms the blended pair into
    int32_t S;
    void refer(int i, int t, int32_t rec, size_t off, size_t field) { ref[i] = FieldRef{t, rec, (uint32_t)off, (uint32_t)field}; }
};

// host-side accumulation of instances for one (level, kind) stage
struct StageBuild {
    int cls = 0;
    int level = 0;
    int kind = 0;
    int variant = 0;
    std::vector<OscInst> osc;
    std::vector<ConstInst> cst;
    std::vector<AbsnInst> absn;
    std::vector<BiquadInst> biquad;
    std::vector<ChainInst> chain;
    std::vector<ParamInst> param;
    std::vector<OscArInst> osc_ar;
    std::vector<BiquadArInst> biquad_ar;
    std::vector<AbsnSlowInst> absn_slow;
    std::vector<ScanCoef> scan_coef;
    size_t n_scan_coef = 0;  // sets appended (the sizing pass counts them without building them)
    // one set of scan constants per biquad of a chain instance, in instance order; returns its index
    template <typename MakeFn>
    int32_t add_scan_coef(bool build, MakeFn&& make) {
        if (build) scan_coef.push_back(make());
        return (int32_t)n_scan_coef++;
    }
    std::vector<IirInst> iir;
    std::vector<GainInst> gain;
    std::vector<ShaperInst> shaper;
    std::vector<SPanInst> span;
    std::vector<float2> span_gains;
    std::vector<PanInst> pan;
    std::vector<HrtfInst> hrtf;
    std::vector<HrtfSelInst> hrtf_sel;
    std::vector<PanDynInst> pan_dyn;
    std::vector<AbsnSerialInst> absn_serial;
    std::vector<AbsnBoundInst> absn_bound;  // S_ABSN_BOUND
    std::vector<ShaperOsInst> shaper_os;
    std::vector<RouteInst> route;
    std::vector<DelayInst> delay;
    std::vector<CompInst> comp;
    std::vector<CompReadoutInst> comp_ro;           // S_COMP variant 1 (declared reduction read-outs): parallel to comp
    std::vector<AnalyserInst> analyser;
    std::vector<ReadoutInst> readout;                // S_READOUT_FFT / S_READOUT_TIME
    std::vector<ReadoutSmoothInst> readout_smooth;  // S_READOUT_SMOOTH
    std::vector<MixInst> mix;
    std::vector<MixEdge> mix_edges;
    std::vector<MixDynInst> mix_dyn;
    std::vector<MetaInst> meta;
    std::vector<ConvInput> conv_in;
    std::vector<ConvPath> conv_path;
    std::vector<ConvCmpInst> conv_cmp;  // S_CONV_CMP: compacted second path of a mono-response convolver
    std::vector<VoiceGroup> vgroups;  // S_VSUM: groups of consecutive `chain` records
    int max_ch = 1;
    std::vector<Entry> entries;  // the bind entries of this stage's records, every kind in one list
    // The stage's tables as prep_plan_group uploads them: T_A (Stage::d_a) holds the instances; T_B (d_b) the mix edges (S_MIX,
    // S_MIX_DYN), scan constants (S_CHAIN, S_VSUM; the sizing pass counts them without building them), stereo gains (S_SPAN), selection
    // records of moving panners (S_HRTF) or read-outs (S_COMP); T_C (d_c) the voice groups (S_VSUM).  Rows and bytes of one row.
    struct Shape {
        size_t n = 0, bytes = 0;
    };
    template <typename T>
    static Shape shape(const std::vector<T>& v) { return {v.size(), sizeof(T)}; }
    Shape table(int t) const {
        if (t == T_B) switch (kind) {
            case S_MIX: case S_MIX_DYN: return shape(mix_edges);
            case S_CHAIN: case S_VSUM: return {n_scan_coef, sizeof(ScanCoef)};
            case S_SPAN: return shape(span_gains);
            case S_HRTF: return shape(hrtf_sel);
            case S_COMP: return shape(comp_ro);
            default: return {};  // (S_CONV_MAC, S_CONV_MAC_ACC: the conv inputs of their level's S_CONV_FFT stage)
        }
        if (t == T_C) return kind == S_VSUM ? shape(vgroups) : Shape{};
        switch (kind) {
            case S_MIX: return shape(mix);
            case S_MIX_DYN: return shape(mix_dyn);
            case S_META: return shape(meta);
            case S_OSC: return shape(osc);
            case S_CONST: return shape(cst);
            case S_ABSN: return shape(absn);
            case S_BIQUAD: return shape(biquad);
            case S_CHAIN: case S_VSUM: return shape(chain);
            case S_PARAM: return shape(param);
            case S_OSC_AR: return shape(osc_ar);
            case S_BIQUAD_AR: return shape(biquad_ar);
            case S_ABSN_SLOW: return shape(absn_slow);
            case S_IIR: return shape(iir);
            case S_GAIN: return shape(gain);
            case S_SHAPER: return shape(shaper);
            case S_SPAN: return shape(span);
            case S_PAN: return shape(pan);
            case S_HRTF: return shape(hrtf);
            case S_PAN_DYN: return shape(pan_dyn);
            case S_ABSN_SERIAL: return shape(absn_serial);
            case S_ABSN_BOUND: return shape(absn_bound);
            case S_SHAPER_OS: return shape(shaper_os);
            case S_ROUTE: return shape(route);
            case S_DELAY_MONO: case S_DELAY: case S_DELAY_WRITE: return shape(delay);
            case S_COMP: return shape(comp);
            case S_ANALYSER: return shape(analyser);
            case S_CONV_FFT: return shape(conv_in);
            case S_CONV_CMP: return shape(conv_cmp);
            case S_CONV_MAC: case S_CONV_MAC_ACC: return shape(conv_path);
            default: return {};  // (S_READOUT_*: uploaded sorted by frame, no entry points into them)
        }
    }
    size_t records(int t = T_A) const { return table(t).n; }
    size_t record_bytes(int t) const { return table(t).bytes; }
    // records entry `e` for the last record of table `t`, its reference 0 `off` bytes into it (filling the payload field `field`)
    void add_entry(Entry e, size_t off, size_t field, int t = T_A) {
        e.refer(0, t, (int32_t)records(t) - 1, off, field);
        entries.push_back(e);
    }
};

struct Stage {
    int cls = 0;  // see Planner::stage()
    int seg = 0;  // render segment (between two suspend points) this stage belongs to
    int kind = 0;
    int variant = 0;
    int group = 0;
    int n = 0;
    int n_b = 0;
    int max_ch = 1;
    void* d_a = nullptr;  // instances
    void* d_b = nullptr;  // auxiliary table (mix edges, scan coefficients, conv inputs, panner gains)
    void* d_c = nullptr;  // S_VSUM: voice groups
    std::vector<int64_t> frames;  // S_READOUT_FFT / S_READOUT_TIME: the records' frames (sorted); a chunk launches those it holds
    float ms = 0.f;       // accumulated device time of the last run (when timing is enabled)
    ChainAux chain;       // S_CHAIN with biquads: ticket counter + slab hand-off slots (k_chain)
};

struct AnalyserRec {
    uint32_t graph_index;
    uint32_t node;
    float* d_ring;
    uint32_t fft_size;
    double smoothing;
    float* d_last_fft;  // last_fft_output (analysis.rs:168), zeroed per run
    float* d_db;        // read-out scratch
    bool computed;      // frequency data already computed for the end-of-render time (analysis.rs:353-361)
    double min_db, max_db;
    int64_t lq;         // frames the graph renders (its own length padded to whole quanta): the ring's write index after the render
    bool end_readout = false;  // its last declared frequency read-out is at lq: each run leaves that row in d_db, computed
};

// The rows of the declared read-outs of one node (and kind) over the batch: one allocation, graphs in the caller's order, each [k][row]
// (wae_analyser_set_readouts: float rows, wae_analyser_set_byte_readouts: byte rows; wae_compressor_set_readouts: row = 1 float)
template <typename T>
struct ReadoutRows {
    T* d = nullptr;
    uint64_t count = 0;         // elements in all
    std::vector<uint64_t> off;  // [batch position] first element of the graph's rows, or UINT64_MAX: not declared there
    std::vector<uint64_t> len;  // [batch position] elements of the graph's rows
    void add(uint32_t n_graphs, uint32_t j, uint64_t elems) {
        if (off.empty()) {
            off.assign(n_graphs, UINT64_MAX);
            len.assign(n_graphs, 0);
        }
        off[j] = count;
        len[j] = elems;
        count += elems;
    }
};
using ReadoutOut = ReadoutRows<float>;

// One kind of input a prepared batch takes from device memory, as messages name it
struct BindKind {
    const char* noun;     // one declaration, in the messages of runs that wait for it
    const char* plural;   // a graph's declarations, in the refusals of one-shot renders
    const char* declare;  // the call that declares one
    const char* bind;     // the call that binds them
    uint32_t wae_graph::*count;  // the graph's number of declarations
};
enum { BK_SOURCES, BK_PARAMS, BK_RESPONSES, BK_CURVES, BK_WAVES, BK_IIRS, BK_VALUE_CURVES, BK_SCHEDULES, BK_LOOPS, BK_COUNT };
const BindKind kBindKinds[BK_COUNT] = {
    {"device input", "device inputs", "wae_buffer_source_set_device_input", "wae_batch_bind_sources", &wae_graph::device_inputs},
    {"param bound from device memory", "params bound from device memory", "wae_param_set_device_value", "wae_batch_bind_params",
     &wae_graph::device_params},
    {"response bound from device memory", "convolver responses bound from device memory", "wae_convolver_set_device_response",
     "wae_batch_bind_responses", &wae_graph::device_responses},
    {"curve bound from device memory", "WaveShaper curves bound from device memory", "wae_wave_shaper_set_device_curve",
     "wae_batch_bind_curves", &wae_graph::device_curves},
    {"periodic wave bound from device memory", "periodic waves bound from device memory", "wae_oscillator_set_device_periodic_wave",
     "wae_batch_bind_periodic_waves", &wae_graph::device_waves},
    {"IIR coefficients bound from device memory", "IIR coefficients bound from device memory", "wae_iir_filter_set_device_coefficients",
     "wae_batch_bind_iir_coefficients", &wae_graph::device_iirs},
    {"value curve bound from device memory", "value curves bound from device memory", "wae_param_set_device_value_curve",
     "wae_batch_bind_value_curves", &wae_graph::device_value_curves},
    {"schedule bound from device memory", "schedules bound from device memory", "wae_source_set_device_schedule", "wae_batch_bind_schedules",
     &wae_graph::device_schedules},
    {"loop points bound from device memory", "loop points bound from device memory", "wae_buffer_source_set_device_loop",
     "wae_batch_bind_loops", &wae_graph::device_loops},
};

// The name of a declaration: (batch position, node, param index); kinds declared on a node take kNodeLevel as param index
constexpr uint32_t kNodeLevel = UINT32_MAX;
struct BindKey {
    uint32_t graph;
    wae_node_id node;
    uint32_t param;
    bool operator<(const BindKey& o) const { return std::tie(graph, node, param) < std::tie(o.graph, o.node, o.param); }
};

// The declarations of one kind, whatever each holds.  A declaration is bound once a bind has named it; runs wait for the unbound ones.
struct BindTable {
    const BindKind* kind;
    std::vector<BindKey> keys;  // [declaration]
    std::vector<char> bound;
    std::map<BindKey, size_t> index;  // key -> declaration
    size_t unbound = 0;
    static constexpr size_t npos = SIZE_MAX;
    explicit BindTable(const BindKind& k) : kind(&k) {}
    size_t find(const BindKey& key) const {
        auto it = index.find(key);
        return it == index.end() ? npos : it->second;
    }
    void set_bound(size_t k, bool is_bound) {
        if (bound[k] == (char)is_bound) return;
        bound[k] = is_bound;
        if (is_bound) unbound--;
        else unbound++;
    }
};

// The declarations of one kind with what a bind writes for each (`D`: slot pointers, spectra, curve or wavetable memory, a range of
// patch entries, windows).  The planner adds the ones it gives memory, under wae_batch::mu; seal() then puts them in key order and
// appends the declared ones the planner never reached.  Those are bound from the start: binding one is validated and writes nothing,
// and runs do not wait for it.
template <typename D>
struct Bindings : BindTable {
    std::vector<D> data;  // [declaration]
    using BindTable::BindTable;
    void add(const BindKey& key, const D& d, bool is_bound = false) {
        index[key] = keys.size();
        keys.push_back(key);
        data.push_back(d);
        bound.push_back(is_bound);
        unbound += is_bound ? 0 : 1;
    }
    // `visit(j, nodes, node, declare)` calls declare(key, d) for each declaration of `node` (of `nodes`: graph j's own nodes or an
    // epoch's copy of them), declare(key, d, false) for one runs wait for whether or not the planner reached it
    template <typename Visit>
    void seal(wae_graph* const* graphs, uint32_t n_graphs, Visit&& visit) {
        std::vector<size_t> perm(keys.size());
        for (size_t k = 0; k < perm.size(); k++) perm[k] = k;
        std::sort(perm.begin(), perm.end(), [&](size_t x, size_t y) { return keys[x] < keys[y]; });
        Bindings sorted(*kind);
        for (size_t k : perm) sorted.add(keys[k], data[k], bound[k]);
        *this = std::move(sorted);
        auto declare = [&](const BindKey& key, const D& d, bool is_bound = true) {
            if (!index.count(key)) add(key, d, is_bound);
        };
        for (uint32_t j = 0; j < n_graphs; j++) {
            if (!(graphs[j]->*kind->count)) continue;
            for (const auto& kv : graphs[j]->nodes) visit(j, graphs[j]->nodes, kv.second, declare);
            for (const auto& ep : graphs[j]->epochs)
                for (const auto& kv : ep.nodes) visit(j, ep.nodes, kv.second, declare);
        }
    }
};

// What the binds write, per kind
struct DevInput {  // wae_buffer_source_set_device_input: the slot in its group's slab
    float* slot;   // [channels][stride]
    uint32_t channels;
    uint64_t length, stride;
    // wae_buffer_source_set_device_input_by_reference (no slot): the entries of every record that plays it, in d_src_refs, and the
    // caller's memory its last bind named (the extent bind_output must not overlap)
    bool by_reference = false;
    int32_t p0 = 0, p1 = 0;
    const float* pcm = nullptr;
    uint64_t pcm_stride = 0;
    uint64_t extent_bytes() const { return ((uint64_t)(channels - 1) * pcm_stride + length) * sizeof(float); }
};
struct DevResponse {  // wae_convolver_set_device_response: the spectra the planner made
    float2* h;        // [channels][S + WAE_CONV_H_PAD][WAE_CONV_SPEC]
    uint32_t channels;
    uint64_t length;
    int S;
    bool normalize;
    float sample_rate;
};
struct DevCurve {  // wae_wave_shaper_set_device_curve: the curve memory the planner made (zeroed, never in the upload slabs)
    float* d;      // [length rounded up to 4]
    uint32_t length;
    int32_t p0, p1;  // its entries in d_curve_patches
};
struct DevWave {  // wae_oscillator_set_device_periodic_wave: the wavetable memory the planner made (zeroed, never in the upload slabs)
    float* d;     // [table_len]
    uint32_t coefficients, table_len;
    bool normalize;
};
struct DevIir {  // wae_iir_filter_set_device_coefficients: the entries of every record its coefficients reach
    uint32_t nff, nfb;
    int32_t p0, p1;  // in d_iir_patches
};
struct DevSchedule {  // wae_source_set_device_schedule (+ wae_buffer_source_set_device_offset): the windows and the entries of every
    int32_t binds;    // record the values reach; SchedBinds
    double lo[4], hi[4];
    int32_t p0, p1;  // in d_sched_patches
};
struct DevLoop {         // wae_buffer_source_set_device_loop: the windows and the entries of every record the loop points reach
    double lo[2], hi[2];
    int32_t p0, p1;  // in d_loop_patches
};
struct DevValueCurve {  // wae_param_set_device_value_curve: the param's curve pool (ParamInst::curves, made by the planner) and where
    float* pool;        // the declared values lie in it
    int32_t values_off;
    uint32_t length;
};
struct DevParam {  // wae_param_set_device_value: the value slot is the declaration's index
    uint32_t pid;  // the param's node id
    ParamSlotInfo info;
};

}  // namespace

struct wae_batch {
    wae_engine* engine = nullptr;
    uint32_t n_graphs = 0, channels = 0;
    uint64_t length = 0;   // frames requested (the longest graph's when the graphs differ in shape)
    int64_t lq = 0;        // frames rendered: whole quanta (src/render/thread.rs:273); the longest group's
    int64_t chunk = 0;     // frames per chunk
    std::vector<void*> allocs;
    std::vector<Stage> stages;
    float* d_out = nullptr;  // packed: graph i (batch order) is [channels_i][length_i] at out_off[i]
    std::vector<size_t> out_off;  // [n_graphs + 1] floats
    // Graphs of different shapes (wae_batch_prepare_many / wae_render_many): the batch holds them sorted into groups, `order` maps
    // the batch position to the caller's index and `pos` back.  Both are empty for a batch of one shape, which keeps the caller's order.
    bool mixed = false;
    std::vector<uint32_t> order, pos;
    uint64_t needed_quanta = 0;  // sum over graphs of ceil(length / 128)
    std::vector<std::pair<uint32_t, uint64_t>> shape;  // per graph (batch order): number_of_channels, length
    uint32_t batch_pos(uint32_t caller_index) const { return pos.empty() ? caller_index : pos[caller_index]; }
    // state that must be reset before every run
    std::vector<std::pair<void*, size_t>> zero_on_run;
    std::vector<AnalyserRec> analysers;
    std::map<std::pair<wae_node_id, uint32_t>, ReadoutOut> readout_outs;  // (node, WAE_READOUT_*) -> rows
    std::map<std::pair<wae_node_id, uint32_t>, ReadoutRows<uint8_t>> byte_readout_outs;  // (node, WAE_READOUT_*) -> byte rows
    std::map<wae_node_id, ReadoutOut> comp_readout_outs;  // compressor node -> reduction rows
    struct CompRec { uint32_t graph; wae_node_id node; const float* d_state; };
    std::vector<CompRec> compressors;
    // source PCM assets: device destination <- host source (re-uploadable: wae_batch_upload)
    // Graph groups: the batch is cut into contiguous groups of graphs; a group's source PCM lives in one device slab
    // mirrored by one pinned host slab, so that H2D(group k+1), render(group k) and D2H(group k-1) overlap on three
    // streams (wae_batch_run_pipelined).  All groups share the arena-sizing chunk.
    struct Group {
        uint32_t g0 = 0, g1 = 0;        // graphs [g0, g1)
        int64_t lq = 0;                 // frames the group renders: its longest graph's length in whole quanta
        size_t stage0 = 0, stage1 = 0;  // stages [stage0, stage1) of `stages` (all segments)
        std::vector<std::pair<size_t, size_t>> seg_stages;  // per render segment: its stages
        std::vector<int64_t> seg_bounds;                    // 0 = b0 < b1 < ... < lq: the suspend frames of this group's graphs
        std::vector<std::pair<size_t, size_t>> out_zero;    // (offset, floats) of the output no stage writes: zeroed when it is bound
        float* d_src = nullptr;         // device slab of source PCM
        float* h_src = nullptr;         // pinned host mirror, built on first use (wae_batch_upload / wae_batch_run_pipelined)
        struct SrcCopy {                // the PCM of one AudioBufferSourceNode inside the slab: planar [ch][stride], as PcmBuffer holds it
            std::shared_ptr<PcmBuffer> buf;
            size_t offset, floats;      // floats
            uint32_t graph;             // (batch position) and node of its first user: names a device input (buf->device_input)
            wae_node_id node;
        };
        std::vector<SrcCopy> src_copies;  // device inputs included: every path that copies host PCM skips them
        bool has_device_inputs = false;
        std::vector<size_t> graph_src_base;  // groups without suspend points: the slab cursor each graph starts at (split planning)
        size_t src_floats = 0;
        cudaEvent_t ev_h2d = nullptr, ev_done = nullptr;
    };
    std::vector<Group> groups;
    // the declarations of the inputs bound from device memory, one table per kind
    Bindings<DevInput> sources{kBindKinds[BK_SOURCES]};
    Bindings<DevParam> params{kBindKinds[BK_PARAMS]};
    Bindings<DevResponse> responses{kBindKinds[BK_RESPONSES]};
    Bindings<DevCurve> curves{kBindKinds[BK_CURVES]};
    Bindings<DevWave> waves{kBindKinds[BK_WAVES]};
    Bindings<DevIir> iirs{kBindKinds[BK_IIRS]};
    Bindings<DevValueCurve> value_curves{kBindKinds[BK_VALUE_CURVES]};
    Bindings<DevSchedule> schedules{kBindKinds[BK_SCHEDULES]};
    Bindings<DevLoop> loops{kBindKinds[BK_LOOPS]};
    // The item table of a bind is staged in page-locked memory (a copy from pageable memory would wait for the engine stream first) and
    // copied to d_bind, which the next bind may overwrite at once (its copy is queued behind this bind's kernel on the same stream).  A
    // staging buffer is reused once its copy has run (its event has completed); while all are in flight a new one is made, so a bind
    // does not wait on the host for runs queued before it (up to kMaxBindStages staging buffers; then the bind waits for the first one that fits).
    struct BindStage {
        void* h;
        size_t cap;      // bytes
        cudaEvent_t ev;  // the copy out of `h`
    };
    static constexpr size_t kMaxBindStages = 8;
    std::vector<BindStage> bind_stages;
    void* d_bind = nullptr;
    size_t bind_cap = 0;  // bytes
    // wae_batch_bind_params: the value of each slot and the patch entries of every record a bound value reaches (re-derived by
    // k_derive_params after each bind)
    ParamSlotInfo* d_slot_info = nullptr;
    float* d_values = nullptr;
    ParamPatch* d_patches = nullptr;
    int n_patches = 0;
    // and the spatial entries of its static panners (re-derived by k_derive_spatial after k_derive_params), with the transform items of
    // those lowered to a convolver (k_resp_fft).  Entries with HRTF read the engine's sphere of generation sphere_gen.
    SpatialPatch* d_spatial = nullptr;
    int n_spatial = 0;
    RespBindItem* d_spatial_resp = nullptr;
    int n_spatial_resp = 0, spatial_max_taps = 0, spatial_max_S = 0;
    bool spatial_sphere = false;
    uint64_t sphere_gen = 0;
    // the patch entries of declared curves, IIR filters and schedules, each declaration's a contiguous range
    CurvePatch* d_curve_patches = nullptr;
    IirPatch* d_iir_patches = nullptr;
    SchedPatch* d_sched_patches = nullptr;
    LoopPatch* d_loop_patches = nullptr;
    SrcRefPatch* d_src_refs = nullptr;  // and of the device inputs declared by reference
    // the looping bound slow-track records whose playhead tables k_absn_loop_schedule derives after every bind of loop points, params or
    // schedules (their inputs); d_loop_overflow: set by a walk that outgrew its table (reported by wae_batch_sync)
    LoopWalk* d_loop_walks = nullptr;
    int n_loop_walks = 0;
    int* d_loop_overflow = nullptr;
    cudaEvent_t ev_bind = nullptr;  // orders a bind after the caller's stream
    // wae_batch_bind_output: the output entries of every group and the caller's memory the runs write instead of d_out (nullptr: d_out).
    // dest_reader: a graph (batch position) whose destination feeds another node, -1: none; its output cannot be bound.
    OutPatch* d_out_patches = nullptr;
    int n_out_patches = 0;
    float* bound_out = nullptr;
    int64_t dest_reader = -1;
    float* out_ptr() const { return bound_out ? bound_out : d_out; }
    // OfflineAudioContext::suspend_sync: a group's render is cut at the suspend frames of its graphs (graphs with different
    // suspend points are put in different groups); every segment has its own plan, node state is shared between the plans
    // through `state_map` (graph, node, allocation sequence, salt)
    struct StateKey {
        uint32_t graph, node, seq;
        uint64_t salt;
        bool operator<(const StateKey& o) const { return std::tie(graph, node, seq, salt) < std::tie(o.graph, o.node, o.seq, o.salt); }
    };
    std::map<StateKey, std::pair<void*, size_t>> state_map;
    std::vector<void*> pinned;
    cudaStream_t s_h2d = nullptr, s_d2h = nullptr;  // the engine's copy streams
    std::recursive_mutex mu;  // groups are planned on worker threads: allocation, state map, read-out records
    struct Timed {
        size_t stage, e0, e1;
    };
    std::vector<Timed> timed;
    wae_batch_stats stats{};
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    std::vector<cudaEvent_t> stage_events;
    bool time_stages = false;
    size_t timed_events_used = 0;
    std::atomic<uint64_t> arena_bytes{0}, asset_bytes{0};
    uint64_t n_cuda_malloc = 0;  // prepare-time diagnostics (WAE_PREPARE_PROFILE=1): blocks that were not served from the engine's cache

    // small per-node state that is zeroed before every run lives in slabs: one memset per slab, not per node
    char* slab = nullptr;
    size_t slab_used = 0, slab_cap = 0;
    void* slab_alloc(size_t bytes) {
        bytes = (bytes + 255) / 256 * 256;
        if (bytes > (1u << 20)) return nullptr;
        if (!slab || slab_used + bytes > slab_cap) {
            slab_cap = 8u << 20;
            bool fresh = false;
            void* p = engine->dev_alloc(slab_cap, &fresh);
            if (!p) return nullptr;
            n_cuda_malloc += fresh ? 1 : 0;
            allocs.push_back(p);
            cudaMemsetAsync(p, 0, slab_cap, engine->stream);
            zero_on_run.push_back({p, slab_cap});
            slab = (char*)p;
            slab_used = 0;
        }
        void* r = slab + slab_used;
        slab_used += bytes;
        return r;
    }
    // small uploads / tables share slabs too (one device block per 4 MiB instead of one per table)
    char* tslab = nullptr;
    size_t tslab_used = 0, tslab_cap = 0;
    void* table_alloc(size_t bytes) {
        bytes = (bytes + 255) / 256 * 256;
        if (bytes > (512u << 10)) return nullptr;
        if (!tslab || tslab_used + bytes > tslab_cap) {
            tslab_cap = 4u << 20;
            bool fresh = false;
            void* p = engine->dev_alloc(tslab_cap, &fresh);
            if (!p) return nullptr;
            n_cuda_malloc += fresh ? 1 : 0;
            allocs.push_back(p);
            tslab = (char*)p;
            tslab_used = 0;
        }
        void* r = tslab + tslab_used;
        tslab_used += bytes;
        return r;
    }
    template <typename T>
    T* dalloc(size_t count, bool zero = false, bool rezero_on_run = false) {
        std::lock_guard<std::recursive_mutex> lk(mu);
        if (rezero_on_run && count * sizeof(T) <= (1u << 20)) {
            void* r = slab_alloc(count * sizeof(T));
            if (r) return (T*)r;
        }
        size_t bytes = count * sizeof(T);
        if (bytes == 0) bytes = 16;
        if (!rezero_on_run) {
            void* r = table_alloc(bytes);
            if (r) {
                if (zero) cudaMemsetAsync(r, 0, bytes, engine->stream);
                return (T*)r;
            }
        }
        bool fresh = false;
        void* p = engine->dev_alloc(bytes, &fresh);
        if (!p) return nullptr;
        n_cuda_malloc += fresh ? 1 : 0;
        allocs.push_back(p);
        if (zero || rezero_on_run) cudaMemsetAsync(p, 0, bytes, engine->stream);
        if (rezero_on_run) zero_on_run.push_back({p, bytes});
        return (T*)p;
    }
    // Small uploads (instance tables, AudioParam timelines) have 4 MiB slabs of their own, are written into a host shadow of the slab and
    // sent with ONE copy per slab: flush_uploads(), at the end of a group's planning — before its first launch, on the stream the
    // launches go to.  (One cudaMemcpyAsync per table before: a plan with thousands of automated params issued thousands of them, each
    // a driver call that syncs the stream first because the source is pageable.)  Ranges are flushed once; tables of a group that is
    // still being planned by another worker may travel with this group's flush — they are complete (written under `mu`) and their
    // group flushes whatever it adds later.
    char* uslab = nullptr;
    std::vector<char> uslab_host;
    size_t uslab_used = 0, uslab_cap = 0, uslab_flushed = 0;
    void flush_uploads() {
        std::lock_guard<std::recursive_mutex> lk(mu);
        if (uslab && uslab_used > uslab_flushed) {
            cudaMemcpyAsync(uslab + uslab_flushed, uslab_host.data() + uslab_flushed, uslab_used - uslab_flushed, cudaMemcpyHostToDevice, engine->stream);
            uslab_flushed = uslab_used;
        }
    }
    void* upload_alloc(size_t bytes) {  // (under `mu`)
        bytes = (bytes + 255) / 256 * 256;
        if (bytes > (512u << 10)) return nullptr;
        if (!uslab || uslab_used + bytes > uslab_cap) {
            flush_uploads();  // what is left of the slab that is full
            bool fresh = false;
            void* p = engine->dev_alloc(4u << 20, &fresh);
            if (!p) return nullptr;
            n_cuda_malloc += fresh ? 1 : 0;
            allocs.push_back(p);
            uslab = (char*)p;
            uslab_cap = 4u << 20;
            uslab_used = uslab_flushed = 0;
            if (uslab_host.size() != uslab_cap) uslab_host.assign(uslab_cap, 0);  // (one shadow: the copy above has left it when cudaMemcpyAsync returns)
        }
        void* r = uslab + uslab_used;
        uslab_used += bytes;
        return r;
    }
    template <typename T>
    T* dupload(const std::vector<T>& v) {
        std::lock_guard<std::recursive_mutex> lk(mu);
        const size_t bytes = v.size() * sizeof(T);
        if (bytes > 0)
            if (void* r = upload_alloc(bytes)) {
                std::memcpy(uslab_host.data() + ((char*)r - uslab), v.data(), bytes);
                return (T*)r;
            }
        return dupload_now(v);
    }
    // ... and the direct form, for large tables and for data a kernel launched by the planner itself reads (the response of a convolver)
    template <typename T>
    T* dupload_now(const std::vector<T>& v) {
        std::lock_guard<std::recursive_mutex> lk(mu);
        T* p = dalloc<T>(v.size());
        if (p && !v.empty()) cudaMemcpyAsync(p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, engine->stream);
        return p;
    }
};

struct PrepState;  // wae_batch_prepare's state (below): what the planners of a batch share

namespace {

// ---- topological order: Graph::order_nodes / visit (src/render/graph.rs:331-487) ---------------------------
// node id -> outgoing edges (ids are dense: a vector with presence flags; iteration in id order like the std::map it replaces).  The lists
// are the graph's own (no copies); a cycle breaker's list is replaced by the empty one.
struct EdgeTable {
    std::vector<const std::vector<Edge>*> v;
    std::vector<char> has;
    static const std::vector<Edge>& none() {
        static const std::vector<Edge> e;
        return e;
    }
    void reset(uint32_t max_id) {
        v.assign((size_t)max_id + 1, &none());
        has.assign((size_t)max_id + 1, 0);
    }
    void set(uint32_t id, const std::vector<Edge>* edges) {
        if (id >= v.size()) {
            v.resize((size_t)id + 1, &none());
            has.resize((size_t)id + 1, 0);
        }
        has[id] = 1;
        v[id] = edges;
    }
    void clear(uint32_t id) { set(id, &none()); }
    bool count(uint32_t id) const { return id < v.size() && has[id]; }
    const std::vector<Edge>* find(uint32_t id) const { return count(id) ? v[id] : nullptr; }
    const std::vector<Edge>& at(uint32_t id) const {
        if (!count(id)) throw std::out_of_range("orderer: unknown node id");
        return *v[id];
    }
};

struct Orderer {
    wae_graph* g;
    EdgeTable edges;  // working copy: cycle breakers clear a DelayWriter's edges
    std::vector<uint32_t> ordered, marked, marked_temp, in_cycle, cycle_breakers, broken;
    static bool contains(const std::vector<uint32_t>& v, uint32_t x) { return std::find(v.begin(), v.end(), x) != v.end(); }
    // returns true when a cycle breaker was applied (the ordering is then restarted), graph.rs:331-403.  Same visiting order
    // as the reference; membership tests use flag vectors indexed by node id instead of its linear `contains` (O(n^2) on 10^4-node graphs).
    struct IdSet {
        std::vector<char> f;
        void reset(size_t n) { f.assign(n, 0); }
        bool count(uint32_t id) const { return id < f.size() && f[id]; }
        bool insert(uint32_t id) {  // true: newly inserted
            if (id >= f.size()) f.resize((size_t)id + 1, 0);
            const bool fresh = !f[id];
            f[id] = 1;
            return fresh;
        }
        void erase(uint32_t id) { if (id < f.size()) f[id] = 0; }
    };
    IdSet marked_set, temp_set;
    bool visit(uint32_t id) {
        if (temp_set.count(id)) {
            auto it = std::find(marked_temp.begin(), marked_temp.end(), id);
            for (auto jt = it; jt != marked_temp.end(); ++jt)
                if (g->nodes.at(*jt).cycle_breaker) {
                    cycle_breakers.push_back(*jt);
                    return true;
                }
            in_cycle.insert(in_cycle.end(), it, marked_temp.end());  // no DelayNode in the cycle: its nodes are muted
            return false;
        }
        if (!marked_set.insert(id)) return false;
        marked_temp.push_back(id);
        temp_set.insert(id);
        const std::vector<Edge>& out = edges.at(id);
        for (size_t i = 0; i < out.size(); i++)
            if (edges.count(out[i].other_id) && visit(out[i].other_id)) return true;  // (every node of the graph has an entry)
        ordered.push_back(id);
        // `id` is the innermost node still being visited: it is the last entry of the stack unless an unbroken cycle was
        // recorded below it, in which case the reference's `retain` removes it wherever it is
        if (!marked_temp.empty() && marked_temp.back() == id) marked_temp.pop_back();
        else marked_temp.erase(std::remove(marked_temp.begin(), marked_temp.end(), id), marked_temp.end());
        temp_set.erase(id);
        return false;
    }
    void run() {  // graph.rs:418-487
        edges.reset(g->nodes.empty() ? 0 : g->nodes.max_id());
        for (auto& kv : g->nodes) edges.set(kv.first, &kv.second.outgoing);
        ordered.reserve(g->nodes.size());
        for (;;) {
            ordered.clear(); marked.clear(); marked_temp.clear(); in_cycle.clear(); cycle_breakers.clear();
            marked_set.reset(edges.v.size()); temp_set.reset(edges.v.size());
            bool applied = false;
            for (auto& kv : g->nodes) {
                applied = visit(kv.first);
                if (applied) break;
            }
            if (!applied) break;
            for (uint32_t id : cycle_breakers) {
                edges.clear(id);
                if (!contains(broken, id)) broken.push_back(id);
            }
        }
        if (!in_cycle.empty()) {
            std::unordered_set<uint32_t> muted(in_cycle.begin(), in_cycle.end());
            ordered.erase(std::remove_if(ordered.begin(), ordered.end(), [&](uint32_t o) { return muted.count(o) != 0; }), ordered.end());
        }
        std::reverse(ordered.begin(), ordered.end());
    }
};

struct PortRef {
    uint32_t node;
    int port;
};

// What the planner can say about a buffer's layout over the render (see BufRef::meta): the range of its channel count over all quanta
// (a silent quantum has one channel, quantum.rs:512-517, unless it sits in a port with an explicit count), the range over the quanta
// that are not silent, and whether it can be silent at all.  A layout that is provably constant needs no track and keeps every
// kernel on its static path; sources that run from frame 0 to the end of the render (every BASELINE config) are.
struct Lay {
    uint8_t lo = 1, hi = 1, nlo = 1, nhi = 1;
    bool may_silent = false;
    bool dyn() const { return lo != hi || may_silent; }
    static Lay fixed(int ch) { return Lay{(uint8_t)ch, (uint8_t)ch, (uint8_t)ch, (uint8_t)ch, false}; }
    static Lay gated(int ch) { return Lay{1, (uint8_t)ch, (uint8_t)ch, (uint8_t)ch, true}; }  // `ch` channels or silent
};

struct PNode {
    Node* n = nullptr;
    int level = 0;
    std::vector<std::vector<PortRef>> in_edges;  // per input port, reference summation order
    std::vector<int> in_ch;
    std::vector<BufRef> in_buf;
    std::vector<Lay> in_lay;
    std::vector<int> out_ch;
    std::vector<BufRef> out_buf;
    std::vector<Lay> out_lay;  // empty: constant (out_ch channels, never silent)
    bool wrote_dest = false;   // out_buf[0] IS the graph's rendered PCM (a convolver that is the destination's only input)
    Lay lay_out(int port) const { return port < (int)out_lay.size() ? out_lay[port] : Lay::fixed(out_ch[port]); }
};

// node id -> PNode; ids are handed out densely (wae_graph::next_id), so this is a vector, not a tree (the planner looks nodes up
// several times per edge).  One table per Planner, reset from graph to graph: the per-node vectors keep their capacity, so the graphs
// of a batch after the first are planned without allocating them again (seven vectors per node).
struct NodeTable {
    std::vector<PNode> v;
    std::vector<char> has;
    void reset(uint32_t max_id) {
        if (v.size() < (size_t)max_id + 1) v.resize((size_t)max_id + 1);
        has.assign(v.size(), 0);
    }
    PNode& put(uint32_t id, Node* n) {
        if (id >= v.size()) {
            v.resize((size_t)id + 1);
            has.resize((size_t)id + 1, 0);
        }
        PNode& p = v[id];
        p.n = n;
        p.level = 0;
        p.in_edges.resize((size_t)n->n_inputs);
        for (auto& port : p.in_edges) port.clear();
        p.in_ch.clear();
        p.in_buf.clear();
        p.in_lay.clear();
        p.out_ch.clear();
        p.out_buf.clear();
        p.out_lay.clear();
        p.wrote_dest = false;
        has[id] = 1;
        return p;
    }
    PNode* find(uint32_t id) { return id < v.size() && has[id] ? &v[id] : nullptr; }
    bool count(uint32_t id) const { return id < v.size() && has[id]; }
    PNode& at(uint32_t id) {
        if (!(id < v.size() && has[id])) throw std::out_of_range("planner: unknown node id");
        return v[id];
    }
};

struct Planner {
    wae_batch* b;
    wae_engine* eng;
    // a planner of group `grp`: its sizing pass when `sizing_copies` is given (the copies of the AudioBuffers into the group's source slab
    // are recorded there), else its planning pass proper, which draws from the slab and shares the batch's IR spectra
    Planner(wae_batch* b, const wae_batch::Group& grp, PrepState& ps, std::vector<wae_batch::Group::SrcCopy>* sizing_copies);
    std::map<std::pair<int, int>, StageBuild> builds;  // (level, kind * 64 + variant)
    std::string error;
    int error_code = 0;
    uint64_t algorithmic_bytes = 0;
    // IR spectra cache: content hash -> device spectra (shared by the planners of all groups of a batch, guarded by b->mu)
    struct IrSpectra {
        float2* h;
        int S;
        int channels;
    };
    std::unordered_map<uint64_t, IrSpectra> own_ir_cache;
    std::unordered_map<uint64_t, IrSpectra>* ir_cache = &own_ir_cache;
    std::map<int, std::pair<const float2*, const float2*>> os_filters;  // over-sampled shaper: factor -> (up, down) filter bins

    bool has_feedback = false;            // some graph has a cycle broken by a DelayNode
    std::map<std::pair<uint32_t, uint32_t>, int>* delay_ch_hint = nullptr;  // (graph, reader id) -> channels of an in-cycle delay
    std::map<std::pair<uint32_t, uint32_t>, int> delay_ch_seen;
    struct DelayRing {
        float* ring;
        uint32_t ring_len;
        int ch;
        int64_t* mono_at;
        int32_t mono_len;
    };
    std::map<std::pair<uint32_t, uint32_t>, DelayRing> delay_rings;       // (graph, writer id)
    std::map<std::pair<uint32_t, uint32_t>, int> conv_paths_seen;        // (graph, convolver id) -> 1: compacted second path, 2: ordinary one (all segments)
    bool dry = false;                     // sizing pass: count arena floats per frame, touch no device memory
    int group_graphs = 1;                 // graphs of the group being planned (k_voice_sum: are there enough work items?)
    // 0 off (default: measured slower than k_chain + k_mix on north_star), 1 when the launch is large enough,
    // 2 whenever the port has the shape (tests).  WAE_OPT_VOICE_SUM, else WAE_VOICE_SUM from the environment (read per plan).
    int vs_mode = -1;
    int voice_sum_mode() {
        if (eng->voice_sum >= 0) return eng->voice_sum;
        if (vs_mode < 0) {
            const char* e = getenv("WAE_VOICE_SUM");
            vs_mode = e ? std::max(0, std::min(2, atoi(e))) : 0;
        }
        return vs_mode;
    }
    uint64_t arena_floats_per_frame = 0;
    // source PCM slab of the group being planned (device pointer, pinned host mirror, cursor in floats)
    float* d_src = nullptr;
    std::vector<wae_batch::Group::SrcCopy>* src_copies = nullptr;
    size_t src_cursor = 0;
    struct PendingChain {
        ChainInst inst;
        hm::BiquadCoefs coefs[CHAIN_MAX_BIQUADS] = {};  // of inst.bq[k]: the scan constants (1.3 KB a set) are derived when the chain is emitted
        int ch = 1;
        int phase = 0;  // 0: before biquad A, 1: after A, 3: after B, 5: after the shaper (canonical chain order)
        int cls = 0;    // scheduling class of the node that opened the chain (see stage())
        Lay lay;        // layout of the chain's output over time (the kernel writes the track when it is not constant)
        // the bind entries of the chain's record: their T_A references take the record's index when the chain is emitted, their T_B
        // references name biquad k until then and its scan constants after; and per gain slot the param entry of the factors folded into
        // it since the first bound one (gain_fold[s].p.param.n == 0: the slot has none)
        std::vector<Entry> entries;
        Entry gain_fold[4] = {};
        // entry `e` with reference 0 `off` bytes into the chain's record (filling the payload field `field`)
        void add_entry(Entry e, size_t off, size_t field) {
            e.refer(0, T_A, -1, off, field);
            entries.push_back(e);
        }
    };

    // Node state is allocated through a key (graph, node, n-th allocation of that node, salt): the plans of consecutive
    // render segments (suspend_sync) find the state of a node that lives on, new nodes get fresh (zeroed) state.
    uint32_t key_graph = 0, key_node = 0, key_seq = 0;
    // Sizing pass: every node-state and arena buffer gets its own placeholder address, numbered by (graph, n-th call in plan_graph), so
    // that the plan digest sees which buffer feeds which instance.  16 MB apart: offsets into one (a splitter's channel aliases, a layout
    // track) never reach the next.  Per graph, not per planner: the split sizing pass must number a graph as the serial one does.
    uint64_t dry_gi = 0, dry_seq = 0;
    uintptr_t dry_addr() { return (uintptr_t)256 + ((dry_gi + 1) << 44) + (dry_seq++ << 24); }
    uint64_t key_salt = 0;
    template <typename T>
    T* alloc(size_t count, bool zero = false, bool rezero_on_run = false) {
        if (dry) return reinterpret_cast<T*>(dry_addr());
        if (seg_start == 0 && seg_end >= lq) return b->dalloc<T>(count, zero, rezero_on_run);  // no suspend point: no later plan looks it up
        const wae_batch::StateKey key{key_graph, key_node, key_seq++, key_salt};
        const size_t bytes = count * sizeof(T);
        std::lock_guard<std::recursive_mutex> lk(b->mu);
        auto it = b->state_map.find(key);
        if (it != b->state_map.end() && it->second.second == bytes) return (T*)it->second.first;
        T* p = b->dalloc<T>(count, zero, rezero_on_run);
        if (p) b->state_map[key] = {(void*)p, bytes};
        return p;
    }
    // arena buffers are chunk-local scratch: every segment's plan draws from the same pool
    std::map<int, std::vector<float*>> arena_pool;
    std::map<int, size_t> arena_used;
    std::map<std::pair<uint32_t, uint32_t>, size_t> src_offsets;  // (graph, buffer source node) -> offset in the group's PCM slab
    std::unordered_map<const PcmBuffer*, size_t> buf_offsets;       // one copy per AudioBuffer in the slab, whatever number of nodes play it
    // render-side view of every AudioParam: the event queue it (re)started with at `init_frame`.  When a suspend callback
    // pushed more events, the state machine is replayed on the host up to the suspend frame and the new events are folded
    // into what is left of the queue — handle_incoming_event against the live state, like the reference's render thread.
    struct ParamRecord {
        size_t n_source_events = 0;  // arrival-order events of the Param already folded in
        ParamTimeline tl;
        int64_t init_frame = 0;
    };
    std::unordered_map<uint64_t, ParamRecord> param_records;  // (graph << 32 | param id); element addresses survive rehashing
    const ParamTimeline* param_timeline(uint32_t gi, uint32_t pid, const Param& prm, float sample_rate) {
        const uint64_t rec_key = (uint64_t)gi << 32 | pid;
        auto it = param_records.find(rec_key);
        if (it == param_records.end()) {
            ParamRecord r;
            r.tl = build_param_timeline(prm);
            r.n_source_events = prm.events.size();
            r.init_frame = seg_start;
            return &param_records.emplace(rec_key, std::move(r)).first->second.tl;
        }
        ParamRecord& r = it->second;
        if (r.n_source_events == prm.events.size() || !r.tl.error.empty()) return &r.tl;
        // replay compute_buffer from the record's start to this segment's start
        ParamInst host{};
        host.events = r.tl.events.data();
        host.curves = r.tl.curves.data();
        host.n_events = (int32_t)r.tl.events.size();
        host.a_rate = prm.a_rate ? 1 : 0;
        host.sample_rate = sample_rate;
        ParamState st{};
        st.intrinsic = r.tl.intrinsic;
        st.has_last = r.tl.has_last ? 1 : 0;
        st.last = r.tl.last;
        st.inited = 1;
        float buf[128];
        for (int64_t f = r.init_frame; f < seg_start; f += 128) param_compute_buffer(host, st, (double)f / (double)sample_rate, buf);
        ParamTimeline next;
        next.curves = r.tl.curves;
        for (int i = st.head; i < host.n_events; i++) next.events.push_back(i == st.head && st.override_valid ? st.override_ev : r.tl.events[i]);
        next.intrinsic = st.intrinsic;
        next.has_last = st.has_last != 0;
        next.last = st.last;
        fold_param_events(next, prm.events.data() + r.n_source_events, prm.events.size() - r.n_source_events);
        r.tl = std::move(next);
        r.n_source_events = prm.events.size();
        r.init_frame = seg_start;
        return &r.tl;
    }
    int64_t seg_start = 0, seg_end = 0;
    // frames the group renders (every kernel runs to here; buffers and tables are sized for it) and frames the graph being planned
    // renders (its own length in whole quanta): a graph shorter than its group decides what depends on the end of ITS render
    int64_t lq = 0, glq = 0;
    // the graph's rendered PCM in the packed output: [channels][length], frames from `length` on are not written (limit)
    BufRef dest_ref() const { return BufRef{b->d_out + b->out_off[gi], (uint32_t)g->length, 1}; }
    // the output entry of the last record of table `t` of `s` (a destination writer), whose BufRef `off` bytes into it is dest_ref()
    void add_out(StageBuild& s, size_t off, int t = T_A) const {
        Entry e = entry(E_OUT);
        e.p.out.off = (uint64_t)b->out_off[gi];
        s.add_entry(e, off + offsetof(BufRef, p), offsetof(OutPatch, dst), t);
    }
    // a graph planned so far feeds its destination's output to another node, which reads the rendered PCM through a record the output
    // entries do not cover: batch position, -1: none
    int64_t dest_reader = -1;
    void begin_segment(int64_t f0, int64_t f1) {
        seg_start = f0;
        seg_end = f1;
        builds.clear();
        arena_used.clear();
        arena_floats_per_frame = 0;
    }
    template <typename T>
    T* upload(const std::vector<T>& v) {
        if (dry) return reinterpret_cast<T*>(uintptr_t(256));
        return b->dupload(v);
    }

    bool bail(int code, const std::string& msg) {
        if (!error_code) {
            error_code = code;
            error = msg;
        }
        return false;
    }
    bool no_arena() { return bail(WAE_OUT_OF_MEMORY, "out of device memory (arena)"); }

    // Scheduling class of a stage.  Graphs without DelayNode feedback: 0 (whole chunks).  Graphs with feedback: 0 = strictly
    // upstream of every cycle (whole chunks, rendered first: sources, a reverb feeding an echo loop), 1 = on a path from a
    // cycle to a cycle-breaking DelayWriter, i.e. inside a feedback cycle or between two of them (replayed quantum by quantum
    // inside the chunk, like the reference's render loop), 2 = the rest: downstream of the cycles only (whole chunks again,
    // e.g. a reverb after an echo loop).
    int cur_cls = 0;  // class of the node being planned
    StageBuild& stage(int level, int kind, int variant = 0) {
        const int cls = cur_cls;
        // the read-out stages run right before k_analyser of their level, which then writes the chunk into the ring
        const int order = kind >= S_READOUT_FFT ? S_ANALYSER * 64 - 3 + (kind - S_READOUT_FFT) : kind * 64 + variant;
        StageBuild& s = builds[{cls * 1000000 + level, order}];
        s.cls = cls;
        s.level = level;
        s.kind = kind;
        s.variant = variant;
        return s;
    }

    // `with_meta`: the buffer's layout is not provably constant: it carries a per-quantum layout track (BufRef::meta), one row per
    // static channel, stored behind the PCM
    BufRef arena_buf(int ch, bool with_meta = false) {
        arena_floats_per_frame += (uint64_t)ch;
        const uint32_t mstride = (uint32_t)((b->chunk / 128 + 16) / 16 * 16);
        BufRef r{dry ? reinterpret_cast<float*>(dry_addr()) : nullptr, (uint32_t)b->chunk, 0, nullptr, 0, 0};
        if (!dry) {
            std::vector<float*>& pool = arena_pool[ch];
            size_t& used = arena_used[ch];
            if (used < pool.size()) {
                r.p = pool[used++];
            } else {
                const size_t floats = (size_t)ch * (size_t)b->chunk;
                float* p = b->dalloc<float>(floats + ((size_t)ch * mstride + 3) / 4);
                b->arena_bytes += floats * 4;
                if (p) {
                    pool.push_back(p);
                    used++;
                }
                r.p = p;
            }
        }
        if (with_meta && r.p) {
            r.meta = reinterpret_cast<uint8_t*>(r.p + (size_t)ch * (size_t)b->chunk);
            r.meta_stride = mstride;
        }
        return r;
    }
    // layout track of a node output from its input's (k_meta)
    void meta_stage(int L, int mode, const BufRef& in, int in_ch, const BufRef& out, int out_ch, int count = 0, int aux = 0) {
        MetaInst m{};
        m.in = in;
        m.out = out;
        m.mode = mode;
        m.in_ch = in_ch;
        m.out_ch = out_ch;
        m.count = count;
        m.aux = aux;
        stage(L, S_META).meta.push_back(m);
    }

    // ---- the graph being planned (plan_graph), reset from graph to graph
    wae_graph* g = nullptr;
    uint32_t gi = 0;
    Orderer ord{};
    NodeTable node_table;  // (the per-node vectors keep their capacity)
    SchedClock clock{48000.f};
    bool want_scan_coefs = false;  // (the sizing pass needs their number only)
    // ---- chain fusion (WAE_OPT_FUSE): sources and biquad/gain/shaper nodes are not emitted one stage each; a node
    // with exactly one consumer stays PENDING, the consumer either extends the chain (same channel count, single
    // edge) or forces it to be materialised into an arena buffer.  A chain that ends at a destination whose only
    // input it is writes the final PCM directly.
    std::map<uint32_t, PendingChain> pending;
    // what the lowering of one node knows about it once its inputs are planned
    struct NodeCtx {
        uint32_t id;
        Node& n;
        PNode& p;
        int level = 0, L = 1;  // L: the stage level of its kernels, after the mixes of its level
        Lay in0;               // layout of input 0
        bool dyn_params = false, fuse_n = false;
        bool extend = false, dest_direct = false;  // it extends / the destination takes the pending chain of `fuse_src`
        uint32_t fuse_src = 0;
    };
    struct PRef {
        bool dyn = false;  // automated / audio-rate driven: one value per frame in `track`
        float v = 0.f;
        BufRef track{nullptr, 0, 0};
        int32_t bound = -1;      // bound from device memory: the param's id (`v` is the placeholder), -1: not bound
        float lo = 0.f, hi = 0.f;  // bound: the range its values are clamped to
    };
    PRef param_ref(uint32_t pid);
    // a bind entry of this graph, of declaration `node` (see Entry::node)
    Entry entry(int kind, wae_node_id node = 0) const {
        Entry e;
        std::memset(&e, 0, sizeof e);
        e.kind = kind;
        e.graph = gi;
        e.node = node;
        return e;
    }
    // a param entry of this graph; operand i of `r` is `pr` (its id when bound, else its planned value)
    Entry patch(int kind, int n) const {
        Entry r = entry(E_PARAM);
        r.p.param.kind = kind;
        r.p.param.n = n;
        for (int i = 0; i < PATCH_OPS; i++) r.p.param.slot[i] = -1;
        return r;
    }
    static void operand(Entry& r, int i, const PRef& pr, float planned) {
        r.p.param.slot[i] = pr.bound;
        r.p.param.val[i] = planned;
    }
    // records param entry `r` for the last record of table `t` of stage `s`, its field `off` bytes into it
    static void add_patch(StageBuild& s, const Entry& r, size_t off, int t = T_A) { s.add_entry(r, off, offsetof(ParamPatch, dst), t); }
    // the spatial entry of a static panner of this graph; operand i is pr[i] (its id when bound, else its planned value)
    Entry spatial_entry(int kind, const PRef* pr, const spatial::PanModel& model) const {
        Entry r = entry(E_SPATIAL);
        r.p.spatial.kind = kind;
        r.p.spatial.model = model;
        for (int i = 0; i < 15; i++) {
            r.p.spatial.slot[i] = pr[i].bound;
            r.p.spatial.val[i] = pr[i].v;
        }
        return r;
    }
    // a moving panner: its bound params are taken raw, PATCH_RAW into SpatialTracks::value of the last record of table `t` of `s`, `off`
    // bytes into it
    void raw_spatial_patches(StageBuild& s, const PRef* pr, size_t off, int t = T_A) const {
        for (int i = 0; i < 15; i++)
            if (pr[i].bound >= 0) {
                Entry r = patch(PATCH_RAW, 1);
                operand(r, 0, pr[i], pr[i].v);
                add_patch(s, r, off + offsetof(SpatialTracks, value) + (size_t)i * sizeof(float), t);
            }
    }
    // a chain's bind entries for its record at index `rec` of stage `s` (emit_chain, sum_voices)
    static void chain_entries(StageBuild& s, const PendingChain& pc, int32_t rec) {
        auto emit = [&](Entry e) {
            for (FieldRef& r : e.ref)
                if (r.table == T_A) r.rec = rec;
                else if (r.table == T_B) r.rec = pc.inst.bq[r.rec].coef;
            s.entries.push_back(e);
        };
        for (const Entry& e : pc.entries) emit(e);
        for (const Entry& f : pc.gain_fold)  // (the gain slots' entries after the others)
            if (f.p.param.n > 0) emit(f);
    }
    static bool chain_has_entries(const PendingChain& pc) {
        bool any = !pc.entries.empty();
        for (const auto& f : pc.gain_fold) any = any || f.p.param.n > 0;
        return any;
    }
    bool plan_graph(wae_graph* graph, uint32_t graph_index);
    // ir_override: the response of a STATIC HRTF panner (blended, gain folded in): no normalisation, no trimming of small trailing taps;
    // a two-channel input is mixed down to mono by the forward transform's loads (ConvInput::in_channel = -1)
    bool plan_convolver(PNode& pn, int level, const BufRef* dest = nullptr, int64_t dest_limit = -1, const PcmBuffer* ir_override = nullptr,
                        const IrSpectra* fixed = nullptr);
    bool ir_spectra(const PcmBuffer& ir, float scale, const std::vector<std::vector<float>>& scaled, int Smax, IrSpectra& spec);
    bool device_response_spectra(const Node& n, int S, IrSpectra& spec);
    bool bound_panner_spectra(const Node& n, int S, IrSpectra& spec);
    const float* device_curve(const Node& n);
    float* device_wave(const Node& n);
    float* device_value_curve(const Param& prm, const ParamTimeline& tl);
    // an entry of the declared curve of node `n`, for the int32 field a reference names
    Entry curve_patch(const Node& n, int32_t keeps, int32_t other) const {
        Entry e = entry(E_CURVE, n.id);
        e.p.curve.keeps = keeps;
        e.p.curve.other = other;
        return e;
    }
    bool conv_compact_path(PNode& pn, int level, int in_ch, const IrSpectra& spec, int Smax, int blocks_per_chunk);
    // chain fusion
    int consumers(uint32_t id) {
        int k = 0;
        for (auto& e : ord.edges.at(id))
            if (e.other_index >= 0) k++;
        return k;
    }
    StageBuild& emit_chain(PendingChain& pc, int L);  // (returns the stage the chain's record went to)
    bool materialize(uint32_t nid, bool may_alias = false);
    // can a node of this kind still be appended to the canonical chain gain, A, gain, B, gain, shaper, gain?
    static bool chain_accepts(const PendingChain& pc, Kind kind) {
        if (kind == K_GAIN) return true;
        if (kind == K_BIQUAD) return pc.phase <= 1;
        if (kind == K_SHAPER) return pc.phase < 5;
        return false;
    }
    // registers this node as the tail of a chain: pending while exactly one consumer may still fuse with it
    bool finish_chain(NodeCtx& nc, PendingChain&& pc) {
        nc.p.out_ch = {pc.ch};
        nc.p.out_buf = {BufRef{nullptr, 0, 0}};
        nc.p.out_lay = {pc.lay};
        pending[nc.id] = std::move(pc);
        if (!(eng->fuse && consumers(nc.n.id) == 1)) return materialize(nc.id);
        return true;
    }
    PendingChain source_chain(int kind, int ch) {
        PendingChain pc;
        std::memset(&pc.inst, 0, sizeof(pc.inst));
        pc.inst.src_kind = kind;
        pc.inst.ch = ch;
        pc.inst.limit = -1;
        pc.inst.end = glq;
        for (int i = 0; i < 4; i++) pc.inst.g[i] = 1.f;
        pc.ch = ch;
        pc.cls = cur_cls;
        pc.lay = Lay::fixed(ch);
        return pc;
    }
    // chain that this biquad / gain / shaper node joins: its producer's pending chain, or a new one reading in_buf
    PendingChain open_chain(NodeCtx& nc) {
        if (nc.extend) {
            PendingChain pc = std::move(pending.at(nc.fuse_src));
            pending.erase(nc.fuse_src);
            return pc;
        }
        PendingChain pc = source_chain(CHAIN_SRC_BUFFER, nc.p.in_ch[0]);
        pc.inst.in = nc.p.in_buf[0];
        pc.lay = nc.in0;
        return pc;
    }
    // a biquad (or an IIR filter of order <= 2, which opens a chain of its own with a constant layout) appended to the chain it joins
    // `bound`: the patch entry of a biquad with params bound from device memory; `iir_bound`: an IIR filter whose coefficients are bound
    // from device memory
    bool append_biquad(NodeCtx& nc, double* state, const hm::BiquadCoefs& c, const Entry* bound = nullptr, bool iir_bound = false) {
        PendingChain pc = open_chain(nc);
        const int k = pc.inst.n_biquad++;
        ChainBiquad& st = pc.inst.bq[k];
        st.state = state;
        st.b0 = c.b0; st.b1 = c.b1; st.b2 = c.b2; st.a1 = c.a1; st.a2 = c.a2;
        pc.coefs[k] = c;
        const size_t coefs = offsetof(ChainInst, bq) + (size_t)k * sizeof(ChainBiquad) + offsetof(ChainBiquad, b0);
        if (bound) {  // (and the biquad's scan constants)
            Entry e = *bound;
            e.refer(1, T_B, k, 0, offsetof(ParamPatch, dst2));
            pc.add_entry(e, coefs, offsetof(ParamPatch, dst));
        }
        if (iir_bound) {
            Entry e = entry(E_IIR, nc.n.id);
            e.refer(1, T_B, k, 0, offsetof(IirPatch, scan));
            pc.add_entry(e, coefs, offsetof(IirPatch, b));
        }
        pc.phase = pc.phase == 0 ? 1 : 3;
        pc.lay = filter_lay(pc.lay);
        return finish_chain(nc, std::move(pc));
    }
    // a node's output buffer and layout
    bool need_out(NodeCtx& nc, int ch) {
        nc.p.out_ch = {ch};
        nc.p.out_buf = {arena_buf(ch)};
        return nc.p.out_buf[0].p != nullptr || no_arena();
    }
    // the node's (single) output has a layout that is not constant: give its buffer a layout track
    void out_dynamic(NodeCtx& nc, const Lay& l) {
        PNode& p = nc.p;
        p.out_lay = {l};
        if (l.dyn() && !p.out_buf.empty() && p.out_buf[0].p && !p.out_buf[0].absolute) {
            p.out_buf[0].meta = dry ? reinterpret_cast<uint8_t*>(uintptr_t(256)) : reinterpret_cast<uint8_t*>(p.out_buf[0].p + (size_t)p.out_ch[0] * (size_t)b->chunk);
            p.out_buf[0].meta_stride = (uint32_t)((b->chunk / 128 + 16) / 16 * 16);
        }
    }
    // a scheduled source: `ch` channels inside [n_first, n_stop), one silent channel outside (never silent when it covers the render; a
    // schedule bound from device memory is always gated)
    Lay source_lay(int64_t n_first, int64_t n_stop, int ch, bool declared = false) const {
        return (!declared && n_first <= 0 && n_stop >= glq) ? Lay::fixed(ch) : Lay::gated(ch);
    }
    void source_meta(NodeCtx& nc, int64_t n_first, int64_t n_stop, int ch) {
        MetaInst m{};
        m.out = nc.p.out_buf[0];
        m.mode = META_SOURCE;
        m.out_ch = ch;
        m.count = ch;
        m.n_first = n_first;
        m.n_stop = n_stop;
        stage(nc.L, S_META).meta.push_back(m);
    }
    // a scheduled source's output buffer: its layout, and the layout track (k_meta) where that is not constant.  `sched`: the patch entry
    // of a schedule bound from device memory, for the track's record
    BufRef source_out(NodeCtx& nc, int64_t n_first, int64_t n_stop, int ch, const SchedPatch* sched = nullptr) {
        out_dynamic(nc, source_lay(n_first, n_stop, ch, sched != nullptr));
        if (nc.p.out_lay[0].dyn()) {
            source_meta(nc, n_first, n_stop, ch);
            if (sched) add_sched_patch(stage(nc.L, S_META), nc.n, *sched);
        }
        return nc.p.out_buf[0];
    }
    // biquad / IIR (biquad_filter.rs:778-815): silent once the input is and the tail has rung out; keeps the channels of the last
    // input that was not silent
    static Lay filter_lay(const Lay& l) { return Lay{(uint8_t)(l.may_silent ? 1 : l.lo), l.hi, l.nlo, l.nhi, l.may_silent}; }
    // a serial filter behind an input whose layout changes follows the channel count of its last sounding input quantum
    bool filter_dyn_len(NodeCtx& nc, int ch, int32_t*& dyn_len) {
        if (!nc.in0.dyn()) return true;
        dyn_len = alloc<int32_t>((size_t)ch, true, true);
        if (!dyn_len) return bail(WAE_OUT_OF_MEMORY, "out of device memory (state)");
        out_dynamic(nc, filter_lay(nc.in0));
        return true;
    }
    // output with the input's layout and channel count: share the input's layout track
    void out_like_input(NodeCtx& nc) {
        PNode& p = nc.p;
        p.out_lay = {nc.in0};
        if (nc.in0.dyn() && !p.out_buf.empty() && p.out_buf[0].p) {
            p.out_buf[0].meta = p.in_buf[0].meta;
            p.out_buf[0].meta_stride = p.in_buf[0].meta_stride;
        }
    }
    // inputs
    bool mix(int level, const std::vector<PortRef>& edges, int ch, const ChannelCfg& cfg, bool to_dest, bool dyn, bool with_meta, BufRef& out);
    bool lower_param(uint32_t id, Node& n, PNode& p);
    bool plan_inputs(NodeCtx& nc);
    std::vector<int> voice_sum_ports(const NodeCtx& nc);
    bool plan_port(NodeCtx& nc, int port, int vsum_nb);
    bool sum_voices(NodeCtx& nc, int port, int ch, int nb);
    // one method per node kind
    bool lower_dest(NodeCtx& nc);
    bool lower_osc(NodeCtx& nc);
    bool lower_const(NodeCtx& nc);
    struct AbsnPlay {  // what every playback path of an AudioBufferSourceNode reads
        const PcmBuffer* pb;
        float* buf;  // its PCM in the group's slab (a device input declared by reference: a placeholder its bind replaces)
        size_t len, stride;
        int ch;
        double duration, ls, le, computed_rate;  // ls / le: the clamped loop boundaries
        bool by_ref;
    };
    // the source-reference entry of a record that plays declared source `n`, its PCM pointer and channel stride `buf` and `stride` bytes
    // into record `rec` (-1 in a pending chain)
    Entry src_ref(const Node& n, int32_t rec, size_t buf, size_t stride) const {
        Entry e = entry(E_SRC_REF, n.id);
        e.refer(0, T_A, rec, buf, offsetof(SrcRefPatch, buf));
        e.refer(1, T_A, rec, stride, offsetof(SrcRefPatch, stride));
        return e;
    }
    void add_src_ref(StageBuild& s, const Node& n, size_t buf, size_t stride) { s.entries.push_back(src_ref(n, (int32_t)s.records() - 1, buf, stride)); }
    // an entry of the schedule of declared source `n` (wae_source_set_device_schedule); add_sched_patch: for the last record of stage
    // `s`, its fields `off` bytes into it
    Entry sched_patch(const Node& n, const SchedPatch& p) const {
        Entry e = entry(E_SCHED, n.id);
        e.p.sched = p;
        return e;
    }
    void add_sched_patch(StageBuild& s, const Node& n, const SchedPatch& p, size_t off = 0) {
        s.add_entry(sched_patch(n, p), off, offsetof(SchedPatch, dst));
    }
    SchedPatch sched_entry(const Node& n, int32_t kind) const {
        SchedPatch p{};
        p.kind = kind;
        p.sample_rate = g->sample_rate;
        p.stop_time = n.stop_time;
        p.lq = lq;
        return p;
    }
    bool lower_absn(NodeCtx& nc);
    bool absn_silent(NodeCtx& nc);
    bool absn_serial(NodeCtx& nc, const AbsnPlay& s, const PRef& pdet, const PRef& prate);
    bool absn_slow(NodeCtx& nc, const AbsnPlay& s);
    bool absn_bound(NodeCtx& nc, const AbsnPlay& s, const PRef& pdet, const PRef& prate, int64_t q, bool aligned, double rate_hi,
                    int32_t loop_cap);
    bool absn_fast(NodeCtx& nc, const AbsnPlay& s, int64_t q, bool fused);
    bool lower_biquad(NodeCtx& nc);
    bool lower_iir(NodeCtx& nc);
    bool lower_gain(NodeCtx& nc);
    bool lower_shaper(NodeCtx& nc);
    bool lower_stereo_panner(NodeCtx& nc);
    struct HrirAtRate {  // the HRIR sphere at the context's rate
        uint32_t sr, taps;
        const float* d_ir;
        const float* h_ir;  // [vertex][2][taps] on the host
    };
    bool lower_panner(NodeCtx& nc);
    bool hrir_at_rate(HrirAtRate& hr);
    HrtfSel static_hrtf_sel(const spatial::SpatialParams& sp0) const;
    bool panner_hrtf_conv(NodeCtx& nc, const spatial::SpatialParams& sp0, const HrirAtRate& hr, const PRef* pr, const spatial::PanModel& model);
    bool panner_hrtf_fir(NodeCtx& nc, const spatial::SpatialParams& sp0, const HrirAtRate& hr, bool moving, const SpatialTracks& tr,
                         const spatial::PanModel& model, const PRef* pr);
    bool lower_delay_writer(NodeCtx& nc);
    bool lower_delay_reader(NodeCtx& nc);
    bool lower_compressor(NodeCtx& nc);
    bool lower_analyser(NodeCtx& nc);
    bool lower_readouts(NodeCtx& nc, const AnalyserInst& a, float* last, float* db);
    bool lower_merger(NodeCtx& nc);
    bool lower_splitter(NodeCtx& nc);
    bool lower_convolver(NodeCtx& nc);
};

static uint64_t fnv1a(const void* data, size_t bytes, uint64_t h = 1469598103934665603ull) {
    const uint8_t* p = (const uint8_t*)data;
    // 8 bytes at a time is enough for a cache key
    size_t n8 = bytes / 8;
    const uint64_t* q = (const uint64_t*)p;
    for (size_t i = 0; i < n8; i++) {
        h ^= q[i];
        h *= 1099511628211ull;
    }
    for (size_t i = n8 * 8; i < bytes; i++) {
        h ^= p[i];
        h *= 1099511628211ull;
    }
    return h;
}

// computedNumberOfChannels for one input port (src/render/quantum.rs:543-547), static channel counts
// Developer check of planner refactorings (WAE_PLAN_DIGEST=1, wae_batch_plan only): a hash over every instance record the sizing pass
// builds (records are value-initialised, device pointers are the dry pass's placeholders), printed per group — equal digests before and
// after a change of the planner's data structures mean the same tables would be uploaded.
static bool plan_digest_wanted() {
    static const bool on = [] { const char* e = getenv("WAE_PLAN_DIGEST"); return e && atoi(e) != 0; }();
    return on;
}
template <typename T>
static uint64_t digest_vec(const std::vector<T>& v, uint64_t h) {
    const uint64_t n = v.size();
    h = fnv1a(&n, sizeof n, h);
    if (v.empty()) return h;
    static const bool dump = [] { const char* e = getenv("WAE_PLAN_DIGEST"); return e && atoi(e) >= 2; }();
    if (dump) {  // which 8-byte word of which record type differs between two runs
        std::fprintf(stderr, "  [%s] n %zu size %zu:", __PRETTY_FUNCTION__, v.size(), sizeof(T));
        const uint64_t* q = (const uint64_t*)v.data();
        for (size_t i = 0; i < sizeof(T) / 8 && i < 400; i++) std::fprintf(stderr, " %llx", (unsigned long long)q[i]);
        std::fprintf(stderr, "\n");
    }
    return fnv1a(v.data(), v.size() * sizeof(T), h);
}
// The records that carry a graph's end frame (`end`: k_chain, the convolver kernels, k_analyser, k_compressor) are digested without it,
// so that the plan of a batch of one shape (where it is the render length) digests as it did before the field existed.  `skip`: the
// offsets of the 8-byte fields left out of each record.
template <typename T>
static uint64_t digest_vec_skipping(const std::vector<T>& v, std::initializer_list<size_t> skip, uint64_t h) {
    const uint64_t n = v.size();
    h = fnv1a(&n, sizeof n, h);
    if (v.empty()) return h;
    std::vector<uint8_t> bytes;
    bytes.reserve(v.size() * sizeof(T));
    for (const T& x : v) {
        const uint8_t* p = reinterpret_cast<const uint8_t*>(&x);
        size_t at = 0;
        for (size_t off : skip) {
            bytes.insert(bytes.end(), p + at, p + off);
            at = off + sizeof(int64_t);
        }
        bytes.insert(bytes.end(), p + at, p + sizeof(T));
    }
    return fnv1a(bytes.data(), bytes.size(), h);
}
template <typename T>
static uint64_t digest_vec_without_end(const std::vector<T>& v, uint64_t h) { return digest_vec_skipping(v, {offsetof(T, end)}, h); }

using Builds = std::map<std::pair<int, int>, StageBuild>;
// The bind entries are not part of any record: the split sizing's self-check compares them on their own, and WAE_PLAN_DIGEST prints them
// on a line of their own (a graph with declarations and its twin with host values plan the same records, but only the first has
// entries).  Canonical form, in the order prepare uploads them (kind, stage, planning order): kind, graph, node, each reference's table,
// record and offset, and the payload with the addresses the references fill zeroed.  `count`: the entries digested.
static uint64_t digest_entries(const Builds& builds, uint64_t h, size_t& count) {
    std::vector<uint8_t> bytes;  // (hashed from the heap: fnv1a reads 8-byte words)
    for (int kind = 0; kind < E_KINDS; kind++)
        for (auto& kv : builds)
            for (Entry e : kv.second.entries) {
                if (e.kind != kind) continue;
                int32_t head[12] = {e.kind, (int32_t)e.graph, (int32_t)e.node};
                for (int i = 0; i < 3; i++) {
                    const FieldRef& r = e.ref[i];
                    head[3 + 3 * i] = r.table;
                    head[4 + 3 * i] = r.rec;
                    head[5 + 3 * i] = (int32_t)r.off;
                    if (r.table != T_NONE) std::memset(reinterpret_cast<char*>(&e.p) + r.field, 0, sizeof(void*));
                }
                const uint8_t* p = reinterpret_cast<const uint8_t*>(head);
                bytes.insert(bytes.end(), p, p + sizeof head);
                p = reinterpret_cast<const uint8_t*>(&e.p);
                bytes.insert(bytes.end(), p, p + kEntryPayloadBytes[kind]);
                count++;
            }
    return fnv1a(bytes.data(), bytes.size(), h);
}
static uint64_t digest_builds(const Builds& builds, uint64_t h) {
    for (auto& kv : builds) {
        const StageBuild& s = kv.second;
        const int key[6] = {kv.first.first, kv.first.second, s.cls, s.level, s.kind * 64 + s.variant, s.max_ch};
        h = fnv1a(key, sizeof key, h);
        h = digest_vec(s.osc, h); h = digest_vec(s.cst, h); h = digest_vec(s.absn, h); h = digest_vec(s.biquad, h); h = digest_vec_without_end(s.chain, h);
        h = digest_vec(s.param, h); h = digest_vec(s.osc_ar, h); h = digest_vec(s.biquad_ar, h); h = digest_vec(s.absn_slow, h);
        h = digest_vec(s.scan_coef, h); h = digest_vec(s.iir, h); h = digest_vec(s.gain, h); h = digest_vec(s.shaper, h); h = digest_vec(s.span, h);
        h = digest_vec(s.span_gains, h); h = digest_vec(s.pan, h); h = digest_vec(s.hrtf, h); h = digest_vec(s.hrtf_sel, h); h = digest_vec(s.pan_dyn, h);
        h = digest_vec(s.absn_serial, h); h = digest_vec(s.shaper_os, h); h = digest_vec(s.route, h); h = digest_vec(s.delay, h); h = digest_vec_without_end(s.comp, h);
        h = digest_vec_without_end(s.analyser, h); h = digest_vec(s.mix, h); h = digest_vec(s.mix_edges, h); h = digest_vec(s.mix_dyn, h); h = digest_vec(s.meta, h);
        h = digest_vec_without_end(s.conv_in, h); h = digest_vec_without_end(s.conv_path, h); h = digest_vec(s.vgroups, h);
        if (!s.conv_cmp.empty())
            h = digest_vec_skipping(s.conv_cmp, {offsetof(ConvCmpInst, x) + offsetof(ConvInput, end), offsetof(ConvCmpInst, path) + offsetof(ConvPath, end)}, h);  // (only where it exists: the digests of plans without it stay comparable)
        if (!s.absn_bound.empty()) h = digest_vec(s.absn_bound, h);  // (the same)
        if (!s.readout.empty()) h = digest_vec(s.readout, h);
        if (!s.readout_smooth.empty()) h = digest_vec(s.readout_smooth, h);
        if (!s.comp_ro.empty()) h = digest_vec(s.comp_ro, h);
    }
    return h;
}

// Split planning (a group of few, large graphs planned by several workers, each with its own Planner over a contiguous run of the
// group's graphs): the runs' stage builds are appended to one another in graph order, which is the order a single planner would have
// produced.  Records that index a sibling table of their stage are rebased: mix instances -> mix edges, chain biquads -> scan constants,
// voice groups -> chain records, convolver paths -> the conv-input table of the forward-transform stage of their level; and so are the
// references of the bind entries.
template <typename T>
static void append_vec(std::vector<T>& d, std::vector<T>& s) {
    if (d.empty()) d = std::move(s);
    else d.insert(d.end(), s.begin(), s.end());
}
static void merge_builds(Builds& dst, Builds& src) {
    using Base = std::array<size_t, 4>;  // per StageTable
    std::map<std::pair<int, int>, Base> base;  // table sizes of `dst` before anything of `src` is appended
    for (auto& kv : src) {
        auto it = dst.find(kv.first);
        Base& bs = base[kv.first];
        for (int t = T_NONE; t <= T_C; t++) bs[t] = it != dst.end() && t != T_NONE ? it->second.records(t) : 0;
    }
    for (auto& kv : src) {
        StageBuild& s = kv.second;
        const Base bs = base[kv.first];
        for (Entry& e : s.entries)
            for (FieldRef& r : e.ref) r.rec += (int32_t)bs[r.table];
        for (auto& m : s.mix) m.edge_offset += (uint32_t)bs[T_B];
        for (auto& m : s.mix_dyn) m.edge_offset += (uint32_t)bs[T_B];
        for (auto& c : s.chain)
            for (int k = 0; k < c.n_biquad; k++) c.bq[k].coef += (int32_t)bs[T_B];
        for (auto& v : s.vgroups) v.first += (int32_t)bs[T_A];
        if (s.kind == S_CONV_MAC || s.kind == S_CONV_MAC_ACC) {
            const std::pair<int, int> fft_key{kv.first.first, S_CONV_FFT * 64};
            size_t off = 0;
            auto bi = base.find(fft_key);
            if (bi != base.end()) off = bi->second[T_A];
            else if (dst.count(fft_key)) off = dst[fft_key].conv_in.size();
            for (auto& cp : s.conv_path) cp.input += (int32_t)off;
        }
        auto it = dst.find(kv.first);
        if (it == dst.end()) {
            dst.emplace(kv.first, std::move(s));
            continue;
        }
        StageBuild& d = it->second;
        append_vec(d.osc, s.osc); append_vec(d.cst, s.cst); append_vec(d.absn, s.absn); append_vec(d.biquad, s.biquad); append_vec(d.chain, s.chain);
        append_vec(d.param, s.param); append_vec(d.osc_ar, s.osc_ar); append_vec(d.biquad_ar, s.biquad_ar); append_vec(d.absn_slow, s.absn_slow);
        append_vec(d.scan_coef, s.scan_coef); append_vec(d.iir, s.iir); append_vec(d.gain, s.gain); append_vec(d.shaper, s.shaper); append_vec(d.span, s.span);
        append_vec(d.span_gains, s.span_gains); append_vec(d.pan, s.pan); append_vec(d.hrtf, s.hrtf); append_vec(d.hrtf_sel, s.hrtf_sel);
        append_vec(d.pan_dyn, s.pan_dyn); append_vec(d.absn_serial, s.absn_serial); append_vec(d.shaper_os, s.shaper_os); append_vec(d.route, s.route);
        append_vec(d.delay, s.delay); append_vec(d.comp, s.comp); append_vec(d.analyser, s.analyser); append_vec(d.mix, s.mix);
        append_vec(d.mix_edges, s.mix_edges); append_vec(d.mix_dyn, s.mix_dyn); append_vec(d.meta, s.meta); append_vec(d.conv_in, s.conv_in);
        append_vec(d.conv_path, s.conv_path); append_vec(d.vgroups, s.vgroups); append_vec(d.conv_cmp, s.conv_cmp);
        append_vec(d.absn_bound, s.absn_bound);
        append_vec(d.readout, s.readout); append_vec(d.readout_smooth, s.readout_smooth); append_vec(d.comp_ro, s.comp_ro);
        append_vec(d.entries, s.entries);
        d.n_scan_coef += s.n_scan_coef;
        d.max_ch = std::max(d.max_ch, s.max_ch);
    }
}

static int computed_channels(const ChannelCfg& cfg, int max_in) {
    switch (cfg.mode) {
        case WAE_COUNT_MODE_MAX: return max_in;
        case WAE_COUNT_MODE_EXPLICIT: return cfg.count;
        default: return std::min(max_in, cfg.count);
    }
}

static uint32_t next_pow2(uint64_t v) {
    uint32_t p = 1;
    while (p < v) p <<= 1;
    return p;
}

// constants of the time-parallel biquad recurrence (see ScanCoef in wae_kernels.h), f64 on the host
static ScanCoef make_scan_coef(const hm::BiquadCoefs& c) {
    ScanCoef sc{};
    make_scan_coef(c.b1, c.b2, c.a1, c.a2, sc);
    return sc;
}

bool Planner::plan_convolver(PNode& pn, int level, const BufRef* dest, int64_t dest_limit, const PcmBuffer* ir_override, const IrSpectra* fixed) {
    Node& n = *pn.n;
    int in_ch = pn.in_ch[0];
    const bool mono_mix = ir_override && in_ch == 2;
    if (mono_mix) in_ch = 1;
    if ((n.buffer || ir_override) && cur_cls == 1)  // (the class is a property of the graph: the sizing pass already knows it)
        return bail(WAE_UNSUPPORTED, "a ConvolverNode inside a DelayNode feedback cycle is not lowered to the GPU (before or after the cycle it is)");
    const Lay in_lay = pn.in_lay.empty() ? Lay::fixed(in_ch) : pn.in_lay[0];
    if (!n.buffer && !ir_override) {  // no buffer: pass-through (convolver.rs:368-375)
        pn.out_ch = {in_ch};
        pn.out_buf = {pn.in_buf[0]};
        pn.out_lay = {in_lay};
        return true;
    }
    const PcmBuffer& ir = ir_override ? *ir_override : *n.buffer;
    int ir_ch = (int)ir.channels.size();
    size_t ir_len = ir.length();
    // a response bound from device memory (wae_convolver_set_device_response): planned as an untrimmed response of the declared length;
    // the bind normalises, trims and transforms it on the device
    const bool declared = !ir_override && ir.device_input;
    // `fixed`: spectra made by the caller (an HRTF panner whose position is bound from device memory), of fixed->S partitions whatever
    // the response holds; the bind writes them
    // normalize_buffer, src/node/convolver.rs:16-53 (f32, channel by channel)
    float scale = 1.f;
    if (n.normalize && !ir_override && !declared) {
        float power = 0.f;
        for (auto& c : ir.channels) {
            float s = 0.f;
            for (float v : c) s += v * v;
            power += s;
        }
        power = std::sqrt(power / (float)((size_t)ir_ch * ir_len));
        if (!std::isfinite(power) || power < 0.000125f) power = 0.000125f;
        scale = 1.f / power;
        scale *= 0.00125f;
        scale *= 44100.f / ir.sample_rate;
        if (ir_ch == 4) scale *= 0.5f;
    }
    // convolvers: one per IR channel, a mono IR is duplicated (convolver.rs:289-293)
    int n_conv = std::max(ir_ch, 2);
    // trailing samples below 1e-6 are ignored by fft-convolver's init
    std::vector<std::vector<float>> scaled(declared || fixed ? 0 : ir_ch);
    size_t trimmed_len = declared ? ir_len : 0;
    for (int c = 0; c < (declared || fixed ? 0 : ir_ch); c++) {
        scaled[c].resize(ir_len);
        for (size_t i = 0; i < ir_len; i++) scaled[c][i] = ir.channels[c][i] * scale;
    }
    // per-channel trimmed length (each FFTConvolver trims its own IR); use per channel S
    std::vector<int> S(ir_ch, declared ? (int)((ir_len + WAE_CONV_BLOCK - 1) / WAE_CONV_BLOCK) : fixed ? fixed->S : 0);
    for (int c = 0; c < (declared || fixed ? 0 : ir_ch); c++) {
        size_t m = ir_len;
        while (!ir_override && m > 0 && std::fabs(scaled[c][m - 1]) < 0.000001f) m--;
        while (ir_override && m > 0 && scaled[c][m - 1] == 0.f) m--;  // (exact zeros only)
        S[c] = (int)((m + WAE_CONV_BLOCK - 1) / WAE_CONV_BLOCK);
        trimmed_len = std::max(trimmed_len, m);
        // zero the ignored tail so that a shared segment count reproduces the per-convolver trimming
        for (size_t i = m; i < ir_len; i++) scaled[c][i] = 0.f;
    }
    int Smax = *std::max_element(S.begin(), S.end());
    pn.out_ch = {ir_ch == 1 && in_ch == 1 ? 1 : 2};
    // a mono response behind an input that switches between one and two channels: the reference feeds its second convolver the
    // two-channel quanta only (convolver.rs:378-400), so input R -> output 1 runs as a compacted path of its own (ConvCmpInst)
    const bool compact = in_lay.dyn() && ir_ch == 1 && in_lay.hi >= 2;
    if (compact && in_ch != 2) return bail(WAE_UNSUPPORTED, "unsupported convolver channel routing");
    if (ir_ch == 1 && in_ch == 2 && !ir_override) {
        // the second convolver's history lives in the compacted path's stream state or in the ordinary path's input ring, not in both:
        // a node whose input turns from a changing layout to a constant two-channel one (or back) at a suspend point cannot hand it on
        int& seen = conv_paths_seen[{key_graph, key_node}];
        seen |= compact ? 1 : 2;
        if (seen == 3)
            return bail(WAE_UNSUPPORTED, "a ConvolverNode with a mono response whose input changes between a constant two-channel layout and a "
                                         "changing one at a suspend point is not lowered to the GPU (its second convolver's history would not "
                                         "carry over, convolver.rs:378-400)");
    }
    // node state is keyed by its role, not by the order of the allocations: which of them happen depends on the input's layout, and that
    // can change at a suspend point (a tone alone, then a stereo source added from the callback) while the history has to carry over
    const uint32_t key_base = key_seq;
    auto role = [&](uint32_t r) { key_seq = key_base + r; };
    // silent once the input has been silent for the length of the response (convolver.rs:357-366); channels from the routing table (:378-487)
    const bool conv_dyn = in_lay.dyn();
    // the destination's only input, same channel count, constant layout: the inverse transforms write the rendered PCM themselves
    const bool direct = dest && !conv_dyn && Smax > 0 && pn.out_ch[0] == (int)g->channels;
    pn.out_buf = {direct ? *dest : arena_buf(pn.out_ch[0], conv_dyn && Smax > 0)};
    pn.wrote_dest = direct;
    if (conv_dyn && Smax > 0) {
        const int oc = pn.out_ch[0];
        pn.out_lay = {Lay{(uint8_t)(in_lay.may_silent ? 1 : oc), (uint8_t)oc, (uint8_t)oc, (uint8_t)oc, in_lay.may_silent}};
        if (compact)  // (a mono response: one output channel wherever the input has one)
            pn.out_lay = {Lay{(uint8_t)(in_lay.may_silent || in_lay.lo < 2 ? 1 : 2), 2,
                              // (a silent input quantum while the tail runs: a SOUNDING one-channel output)
                              (uint8_t)(in_lay.may_silent || in_lay.nlo < 2 ? 1 : 2), 2, in_lay.may_silent}};
        MetaInst m{};
        m.in = pn.in_buf[0];
        m.out = pn.out_buf[0];
        m.mode = META_CONV;
        m.in_ch = in_ch;
        m.out_ch = oc;
        m.aux = ir_ch;
        m.tail_len = (int64_t)ir_len;
        role(0);
        m.state = alloc<int64_t>(1, true, true);
        if (!m.state) return bail(WAE_OUT_OF_MEMORY, "out of device memory (convolver tail counter)");
        stage(level, S_META).meta.push_back(m);
    }
    if (Smax == 0) {  // all-zero IR: output zeros -> a mix with no edges
        StageBuild& ms = stage(level, S_MIX);
        ms.mix.push_back(MixInst{pn.out_buf[0], pn.out_ch[0], 0, 0, (uint32_t)ms.mix_edges.size(), -1});
        return true;
    }
    IrSpectra spec;
    if (fixed) spec = *fixed;
    else if (!(declared ? device_response_spectra(n, Smax, spec) : ir_spectra(ir, scale, scaled, Smax, spec))) return false;
    // inputs: one spectra ring per input channel
    StageBuild& fs = stage(level, S_CONV_FFT);
    int blocks_per_chunk = (int)((b->chunk + WAE_CONV_BLOCK - 1) / WAE_CONV_BLOCK);
    int ring_blocks = Smax + blocks_per_chunk;
    int in_base = (int)fs.conv_in.size();
    for (int c = 0; c < (compact ? 1 : in_ch); c++) {
        ConvInput ci;
        ci.in = pn.in_buf[0];
        ci.in_channel = mono_mix ? -1 : c;
        role(1 + 2 * (uint32_t)c);
        ci.prev = alloc<float>(WAE_CONV_BLOCK, true, true);
        ci.xring = alloc<float2>((size_t)ring_blocks * WAE_CONV_SPEC);
        ci.xring_blocks = ring_blocks;
        ci.end = glq;
        if (!ci.prev || !ci.xring) return bail(WAE_OUT_OF_MEMORY, "out of device memory (convolver input spectra)");
        b->arena_bytes += (size_t)ring_blocks * WAE_CONV_SPEC * 8;
        fs.conv_in.push_back(ci);
    }
    // paths: channel routing table of convolver.rs:378-487
    struct R {
        int in, ir, out, acc;
    };
    std::vector<R> routes;
    if (compact) routes = {{0, 0, 0, 0}};  // (+ the compacted path below)
    else if (in_ch == 1 && ir_ch == 1) routes = {{0, 0, 0, 0}};
    else if (in_ch == 1 && ir_ch == 2) routes = {{0, 0, 0, 0}, {0, 1, 1, 0}};
    else if (in_ch == 2 && ir_ch == 1) routes = {{0, 0, 0, 0}, {1, 0, 1, 0}};
    else if (in_ch == 2 && ir_ch == 2) routes = {{0, 0, 0, 0}, {1, 1, 1, 0}};
    else if (in_ch == 2 && ir_ch == 4) routes = {{0, 0, 0, 0}, {0, 1, 1, 0}, {1, 2, 0, 1}, {1, 3, 1, 1}};
    else if (in_ch == 1 && ir_ch == 4) routes = {{0, 0, 0, 0}, {0, 1, 1, 0}, {0, 2, 0, 1}, {0, 3, 1, 1}};
    else return bail(WAE_UNSUPPORTED, "unsupported convolver channel routing");
    (void)n_conv;
    for (auto& r : routes) {
        role(12 + (uint32_t)(&r - routes.data()));
        ConvPath p;
        p.out = pn.out_buf[0];
        p.h = spec.h + ((size_t)r.ir * (Smax + WAE_CONV_H_PAD) + WAE_CONV_H_PAD_LO) * WAE_CONV_SPEC;
        p.input = in_base + r.in;
        p.S = Smax;
        p.out_channel = r.out;
        p.accumulate = r.acc;
        p.limit = direct ? dest_limit : -1;
        p.end = glq;
        p.y = nullptr;
        if (Smax > 1) {  // (one partition: k_conv_ifft forms the product itself, there are no output spectra)
            p.y = alloc<float2>((size_t)blocks_per_chunk * WAE_CONV_SPEC);
            if (!p.y) return bail(WAE_OUT_OF_MEMORY, "out of device memory (convolver output spectra)");
            b->arena_bytes += (size_t)blocks_per_chunk * WAE_CONV_SPEC * 8;
        }
        StageBuild& cs = stage(level, r.acc ? S_CONV_MAC_ACC : S_CONV_MAC);
        cs.conv_path.push_back(p);
        if (direct) add_out(cs, offsetof(ConvPath, out));
    }
    if (compact) {
        role(16);  // (16 .. 22, in this order)
        if (!conv_compact_path(pn, level, in_ch, spec, Smax, blocks_per_chunk)) return false;
    }
    // SURVEY §8(d): S*1025*8 B of input-history spectra per convolver-block of 1024 frames
    // (the reference's 1024-frame partitioning defines the algorithmic figure, whatever block size the kernels use)
    role(32);  // (whatever the caller allocates next)
    if (!ir_override) algorithmic_bytes += (uint64_t)(routes.size() + (compact ? 1 : 0)) * (uint64_t)((trimmed_len + 1023) / 1024) * 1025ull * 8ull * (uint64_t)((lq + 1023) / 1024);
    return true;
}

// IR spectra (deduplicated across the batch by content)
bool Planner::ir_spectra(const PcmBuffer& ir, float scale, const std::vector<std::vector<float>>& scaled, int Smax, IrSpectra& spec) {
    const int ir_ch = (int)ir.channels.size();
    const size_t ir_len = ir.length();
    uint64_t key = fnv1a(&scale, sizeof(scale));
    for (int c = 0; c < ir_ch; c++) key = fnv1a(ir.channels[c].data(), ir_len * sizeof(float), key);
    key = fnv1a(&ir_len, sizeof(ir_len), key);
    std::unique_lock<std::recursive_mutex> ir_lock(b->mu);
    auto it = ir_cache->find(key);
    if (it != ir_cache->end()) {
        spec = it->second;
    } else {
        std::vector<float> flat((size_t)ir_ch * ir_len);
        for (int c = 0; c < ir_ch; c++) std::memcpy(flat.data() + (size_t)c * ir_len, scaled[c].data(), ir_len * sizeof(float));
        float* d_ir = dry ? upload(flat) : b->dupload_now(flat);  // (read by launch_conv_ir_fft below: not through the deferred upload slabs)
        if (!dry) cudaStreamSynchronize(eng->stream);  // `flat` is about to go out of scope
        spec.S = Smax;
        spec.channels = ir_ch;
        // (zeroed: the padding partitions of every channel).  An asset shared by content, not node state: not drawn through the node's
        // state keys, whose sequence would otherwise depend on whether this segment's plan found the spectra in the cache
        spec.h = dry ? reinterpret_cast<float2*>(uintptr_t(256)) : b->dalloc<float2>((size_t)ir_ch * (Smax + WAE_CONV_H_PAD) * WAE_CONV_SPEC, true);
        if (!d_ir || !spec.h) return bail(WAE_OUT_OF_MEMORY, "out of device memory (IR spectra)");
        if (!dry) launch_conv_ir_fft(d_ir, (int64_t)ir_len, (int64_t)ir_len, spec.h, Smax, ir_ch, eng->stream);
        b->asset_bytes += (size_t)ir_ch * (Smax + WAE_CONV_H_PAD) * WAE_CONV_SPEC * 8;
        (*ir_cache)[key] = spec;
    }
    return true;
}

// The spectra of a response bound from device memory: one zeroed [ch][S + WAE_CONV_H_PAD][WAE_CONV_SPEC] allocation per (batch graph,
// node), never shared by content, that wae_batch_bind_responses rewrites in full on every bind (the padding partitions stay zero).  It is
// keyed in the cache by (graph, node), so every suspend segment and both paths of a mono response read the same memory, and entered in
// the batch's response table when it is made.
bool Planner::device_response_spectra(const Node& n, int S, IrSpectra& spec) {
    const PcmBuffer& ir = *n.buffer;
    const int ir_ch = (int)ir.channels.size();
    const uint64_t tag[3] = {0x646576696365ull /* "device" */, key_graph, n.id};
    const uint64_t key = fnv1a(tag, sizeof(tag));
    std::unique_lock<std::recursive_mutex> ir_lock(b->mu);
    auto it = ir_cache->find(key);
    if (it != ir_cache->end()) {
        spec = it->second;
        return true;
    }
    spec.S = S;
    spec.channels = ir_ch;
    spec.h = dry ? reinterpret_cast<float2*>(uintptr_t(256)) : b->dalloc<float2>((size_t)ir_ch * (S + WAE_CONV_H_PAD) * WAE_CONV_SPEC, true);
    if (!spec.h) return bail(WAE_OUT_OF_MEMORY, "out of device memory (IR spectra)");
    b->asset_bytes += (size_t)ir_ch * (S + WAE_CONV_H_PAD) * WAE_CONV_SPEC * 8;
    (*ir_cache)[key] = spec;
    if (!dry)
        b->responses.add({key_graph, n.id, kNodeLevel}, DevResponse{spec.h, (uint32_t)ir_ch, (uint64_t)ir.length(), S, n.normalize, ir.sample_rate});
    return true;
}

// The spectra of an HRTF panner lowered to a convolver whose source or listener is bound from device memory: one zeroed
// [2][S + WAE_CONV_H_PAD][WAE_CONV_SPEC] allocation per (batch graph, node), never shared by content, that wae_batch_bind_params rewrites
// in full on every bind (the padding partitions stay zero)
bool Planner::bound_panner_spectra(const Node& n, int S, IrSpectra& spec) {
    const uint64_t tag[3] = {0x70616e6e6572ull /* "panner" */, key_graph, n.id};
    const uint64_t key = fnv1a(tag, sizeof(tag));
    std::unique_lock<std::recursive_mutex> ir_lock(b->mu);
    auto it = ir_cache->find(key);
    if (it != ir_cache->end()) {
        spec = it->second;
        return true;
    }
    spec.S = S;
    spec.channels = 2;
    spec.h = dry ? reinterpret_cast<float2*>(uintptr_t(256)) : b->dalloc<float2>((size_t)2 * (S + WAE_CONV_H_PAD) * WAE_CONV_SPEC, true);
    if (!spec.h) return bail(WAE_OUT_OF_MEMORY, "out of device memory (HRTF spectra)");
    b->asset_bytes += (size_t)2 * (S + WAE_CONV_H_PAD) * WAE_CONV_SPEC * 8;
    (*ir_cache)[key] = spec;
    return true;
}

// The curve memory of a curve bound from device memory: one zeroed allocation per (batch graph, node), outside the upload slabs (nothing
// but wae_batch_bind_curves writes it), shared by every suspend segment and lowering path of the node.  The sizing pass gets the
// placeholder an uploaded curve gets, so that plan digests stay comparable.
const float* Planner::device_curve(const Node& n) {
    if (dry) return reinterpret_cast<const float*>(uintptr_t(256));
    std::lock_guard<std::recursive_mutex> lk(b->mu);
    const size_t k = b->curves.find({gi, n.id, kNodeLevel});
    if (k != BindTable::npos) return b->curves.data[k].d;
    float* d = b->dalloc<float>((size_t)(n.device_curve + 3) / 4 * 4, true);
    if (!d) {
        bail(WAE_OUT_OF_MEMORY, "out of device memory (WaveShaper curve)");
        return nullptr;
    }
    b->asset_bytes += (size_t)(n.device_curve + 3) / 4 * 16;
    b->curves.add({gi, n.id, kNodeLevel}, DevCurve{d, n.device_curve, 0, 0});
    return d;
}

// The wavetable memory of a periodic wave bound from device memory: one zeroed allocation per (batch graph, node), outside the upload
// slabs (nothing but wae_batch_bind_periodic_waves writes it), shared by every suspend segment and lowering path of the node.  The sizing
// pass gets the placeholder an uploaded wavetable gets, so that plan digests stay comparable.
float* Planner::device_wave(const Node& n) {
    if (dry) return reinterpret_cast<float*>(uintptr_t(256));
    std::lock_guard<std::recursive_mutex> lk(b->mu);
    const size_t k = b->waves.find({gi, n.id, kNodeLevel});
    if (k != BindTable::npos) return b->waves.data[k].d;
    float* d = b->dalloc<float>((size_t)n.device_wave_len, true);
    if (!d) {
        bail(WAE_OUT_OF_MEMORY, "out of device memory (periodic wave)");
        return nullptr;
    }
    b->asset_bytes += (size_t)n.device_wave_len * sizeof(float);
    b->waves.add({gi, n.id, kNodeLevel}, DevWave{d, n.device_wave, n.device_wave_len, n.device_wave_normalize});
    return d;
}

// The curve pool of a param with a value curve bound from device memory: one zeroed allocation per (batch graph, param), outside the
// upload slabs (nothing but wae_batch_bind_value_curves writes the declared values), shared by every suspend segment.  The declared event
// is the param's last, so its values are the last `device_curve` of the pool; the param's other curves are copied in once.  The sizing
// pass gets the placeholder an uploaded pool gets, so that plan digests stay comparable.  The pool is found by the (node, param index) the
// param was declared through.
float* Planner::device_value_curve(const Param& prm, const ParamTimeline& tl) {
    if (dry) return reinterpret_cast<float*>(uintptr_t(256));
    std::lock_guard<std::recursive_mutex> lk(b->mu);
    const BindKey key{gi, prm.device_curve_node, prm.device_curve_index};
    const size_t k = b->value_curves.find(key);
    if (k != BindTable::npos) return b->value_curves.data[k].pool;
    const size_t host_part = tl.curves.size() - prm.device_curve;
    float* d = b->dalloc<float>((tl.curves.size() + 3) / 4 * 4, true);
    if (!d || (host_part && cudaMemcpyAsync(d, tl.curves.data(), host_part * sizeof(float), cudaMemcpyHostToDevice, b->engine->stream) !=
                                cudaSuccess)) {
        bail(WAE_OUT_OF_MEMORY, "out of device memory (value curve)");
        return nullptr;
    }
    b->asset_bytes += (tl.curves.size() + 3) / 4 * 16;
    b->value_curves.add(key, DevValueCurve{d, (int32_t)host_part, prm.device_curve});
    return d;
}

// the second convolver of a mono response behind an input that switches between one and two channels: input R -> output 1, fed the
// two-channel quanta only (ConvCmpInst)
bool Planner::conv_compact_path(PNode& pn, int level, int in_ch, const IrSpectra& spec, int Smax, int blocks_per_chunk) {
    // stream frames of a chunk: at most the chunk's; with the partial block in front they touch one block more
    const int wblocks = blocks_per_chunk + 1;
    ConvCmpInst cc{};
    cc.in = pn.in_buf[0];
    cc.in_ch = in_ch;
    cc.x.xring_blocks = Smax + wblocks;
    cc.x.xring = alloc<float2>((size_t)cc.x.xring_blocks * WAE_CONV_SPEC, true);  // (finite: the MAC multiplies stale slots by zero partitions)
    cc.path.out = pn.out_buf[0];
    cc.path.h = spec.h + (size_t)WAE_CONV_H_PAD_LO * WAE_CONV_SPEC;
    cc.path.S = Smax;
    cc.path.out_channel = 1;
    cc.path.limit = -1;
    cc.path.y = alloc<float2>((size_t)wblocks * WAE_CONV_SPEC);
    cc.cursor = alloc<int64_t>(1, true, true);
    cc.carry = alloc<float>(2 * WAE_CONV_BLOCK, true, true);
    cc.win = alloc<float>((size_t)(wblocks + 1) * WAE_CONV_BLOCK);
    cc.qmap = alloc<int32_t>((size_t)(b->chunk / 128 + 1));
    cc.wdesc = alloc<int64_t>(2);
    if (!cc.x.xring || !cc.path.y || !cc.cursor || !cc.carry || !cc.win || !cc.qmap || !cc.wdesc)
        return bail(WAE_OUT_OF_MEMORY, "out of device memory (convolver, compacted path)");
    b->arena_bytes += ((size_t)cc.x.xring_blocks + wblocks) * WAE_CONV_SPEC * 8 + (size_t)(wblocks + 1) * WAE_CONV_BLOCK * 4;
    stage(level, S_CONV_CMP).conv_cmp.push_back(cc);
    return true;
}

Planner::PRef Planner::param_ref(uint32_t pid) {
    PRef r;
    PNode* it = node_table.find(pid);
    const Param& prm = (it ? *it->n : g->nodes.at(pid)).param;
    r.v = prm.constant_value();
    if (prm.device_bound) {
        r.bound = (int32_t)pid;
        r.lo = prm.device_lo;
        r.hi = prm.device_hi;
    }
    if (it && !it->out_buf.empty()) {
        r.dyn = true;
        r.track = it->out_buf[0];
    }
    return r;
}

// ---- chain fusion ---------------------------------------------------------------------------------------------------------
StageBuild& Planner::emit_chain(PendingChain& pc, int L) {
    const int variant = pc.inst.src_kind * 6 + pc.inst.n_biquad * 2 + (pc.inst.has_shaper ? 1 : 0);
    const int consumer_cls = cur_cls;  // a chain is emitted while its consumer is planned, but runs with its own nodes' class
    cur_cls = pc.cls;
    StageBuild& cs = stage(L, S_CHAIN, variant);
    cur_cls = consumer_cls;
    for (int k = 0; k < pc.inst.n_biquad; k++) {
        pc.inst.bq[k].coef = cs.add_scan_coef(want_scan_coefs, [&] { return make_scan_coef(pc.coefs[k]); });
    }
    cs.max_ch = std::max(cs.max_ch, pc.ch);
    chain_entries(cs, pc, (int32_t)cs.chain.size());
    cs.chain.push_back(pc.inst);
    return cs;
}

// may_alias: the consumer reads its input through chan() with any alignment (the convolver's forward transform): a pending chain that
// is nothing but an AudioBufferSourceNode playing its buffer 1:1 from frame 0, the buffer covering the whole (quantum-padded) render,
// IS that buffer — no copy into the arena.  Not a device input read by reference: the consumer's BufRef would bake the placeholder, and
// its readers (chain_load_source<CHAIN_SRC_BUFFER>) load 16 B aligned, zero-padded channels, which caller memory need not be.
bool Planner::materialize(uint32_t nid, bool may_alias) {
    auto it = pending.find(nid);
    if (it == pending.end()) return true;
    PNode& sp = node_table.at(nid);
    {
        const ChainInst& ci = it->second.inst;
        const AbsnInst& a = ci.absn;
        bool unit = true;
        for (int i = 0; i < 4; i++) unit = unit && ci.g[i] == 1.f;
        if (may_alias && ci.src_kind == CHAIN_SRC_ABSN && ci.n_biquad == 0 && !ci.has_shaper && unit && !chain_has_entries(it->second) && it->second.phase == 0 &&
            !it->second.lay.dyn() && a.n_start == 0 && !a.loop && a.buf_offset == 0 && a.buf_len >= lq && a.buf_stride <= 0xffffffffll &&
            seg_start == 0 && seg_end >= lq) {
            sp.out_buf = {BufRef{const_cast<float*>(a.buf), (uint32_t)a.buf_stride, 1}};
            pending.erase(it);
            return true;
        }
    }
    BufRef buf = arena_buf(it->second.ch, it->second.lay.dyn());  // (k_chain writes the layout track itself)
    if (!buf.p) return no_arena();
    it->second.inst.out = buf;
    it->second.inst.limit = -1;
    it->second.inst.out_dup = 0;
    emit_chain(it->second, 2 * sp.level + 1);
    sp.out_buf = {buf};
    pending.erase(it);
    return true;
}

// ---- inputs ---------------------------------------------------------------------------------------------------------------
// AudioRenderQuantum::add of `edges` into `ch` channels under `cfg` (k_mix, or k_mix_dyn when `dyn`), written to the graph's rendered PCM
// (`to_dest`) or to a new arena buffer (`with_meta`: with a layout track): `out`
bool Planner::mix(int level, const std::vector<PortRef>& edges, int ch, const ChannelCfg& cfg, bool to_dest, bool dyn, bool with_meta, BufRef& out) {
    StageBuild& ms = stage(level, dyn ? S_MIX_DYN : S_MIX);
    if (to_dest) {
        if (g->length > 0xffffffffull) return bail(WAE_UNSUPPORTED, "render length above 2^32 frames");
        out = dest_ref();
    } else {
        out = arena_buf(ch, with_meta);
        if (!out.p) return no_arena();
    }
    const uint32_t edge_offset = (uint32_t)ms.mix_edges.size();
    for (auto& r : edges) {
        PNode& s = node_table.at(r.node);
        ms.mix_edges.push_back(MixEdge{s.out_buf[r.port], s.out_ch[r.port], 0});
    }
    const int64_t limit = to_dest ? (int64_t)g->length : -1;
    if (dyn) {
        MixDynInst m{};
        m.out = out;
        m.out_ch = ch;
        m.interp = cfg.interp;
        m.mode = cfg.mode;
        m.cfg_count = cfg.count;
        m.n_edges = (int)edges.size();
        m.edge_offset = edge_offset;
        m.limit = limit;
        ms.mix_dyn.push_back(m);
        if (to_dest) add_out(ms, offsetof(MixDynInst, out));
    } else {
        MixInst m{};
        m.out = out;
        m.out_ch = ch;
        m.interp = cfg.interp;
        m.n_edges = (int)edges.size();
        m.edge_offset = edge_offset;
        m.limit = limit;
        ms.mix.push_back(m);
        if (to_dest) add_out(ms, offsetof(MixInst, out));
    }
    return true;
}

// AudioParamProcessor (param.rs:685-797): only params with automation events or audio-rate inputs become
// GPU work; a constant param is a scalar in its owner's instance
bool Planner::lower_param(uint32_t id, Node& n, PNode& p) {
    auto& edges = p.in_edges[0];
    // (a render without suspend points never replays a timeline: a constant param needs no record at all — most params are)
    if (seg_start == 0 && seg_end >= lq && edges.empty() && n.param.constant()) return true;
    const ParamTimeline* tlp = param_timeline(gi, id, n.param, g->sample_rate);
    if (n.param.constant() && edges.empty()) return true;
    int level = 0;
    for (auto& r : edges) level = std::max(level, node_table.at(r.node).level + 1);
    p.level = level;
    for (auto& r : edges)
        if (!materialize(r.node)) return false;
    const ParamTimeline& tl = *tlp;
    if (!tl.error.empty()) return bail(WAE_NOT_SUPPORTED, tl.error);
    ParamInst pi{};
    if (!edges.empty()) {  // sum of the connected signals, first channel each (1 / explicit / discrete, param.rs:296-310)
        bool any_dyn = false;
        for (auto& r : edges) any_dyn = any_dyn || node_table.at(r.node).lay_out(r.port).dyn();
        // edges whose layout changes: folded per quantum; a silent sum reads as zeros, which is what the param adds then
        const ChannelCfg first_channel{1, WAE_COUNT_MODE_EXPLICIT, WAE_INTERPRETATION_DISCRETE};
        if (!mix(2 * level, edges, 1, first_channel, false, any_dyn, false, pi.in)) return false;
    }
    pi.events = tl.events.empty() ? nullptr : upload(tl.events);
    // (a value curve bound from device memory: the pool of its own the bind writes into)
    if (n.param.device_curve) {
        if (!(pi.curves = device_value_curve(n.param, tl))) return false;
    } else {
        pi.curves = tl.curves.empty() ? nullptr : upload(tl.curves);
    }
    pi.state = alloc<ParamState>(1, true, true);
    pi.out = arena_buf(2);  // channel 0: value per frame, channel 1: single-valued flag per quantum
    if (!pi.state || !pi.out.p) return bail(WAE_OUT_OF_MEMORY, "out of device memory (param)");
    pi.def = n.param.default_value;
    pi.mn = n.param.min_value;
    pi.mx = n.param.max_value;
    pi.intrinsic0 = tl.intrinsic;
    pi.has_last0 = tl.has_last ? 1 : 0;
    pi.last0 = tl.last;
    pi.sample_rate = g->sample_rate;
    pi.n_events = (int32_t)tl.events.size();
    pi.a_rate = n.param.a_rate ? 1 : 0;
    stage(2 * level + 1, S_PARAM).param.push_back(pi);
    p.out_ch = {1};
    p.out_buf = {pi.out};
    return true;
}

// ---- inputs: static channel count + mix stage where needed
bool Planner::plan_inputs(NodeCtx& nc) {
    Node& n = nc.n; PNode& p = nc.p;
    NodeTable& pn = node_table;
    int level = 0;
    for (auto& port : p.in_edges)
        for (auto& r : port) level = std::max(level, pn.at(r.node).level + 1);
    bool dyn_params = false;
    for (uint32_t pid : n.params) {
        PNode& pp = pn.at(pid);
        if (!pp.out_buf.empty()) {
            dyn_params = true;
            level = std::max(level, pp.level + 1);
        }
    }
    if (n.kind == K_PANNER)
        for (uint32_t pid = 2; pid <= 10; pid++)
            if (pn.count(pid) && !pn.at(pid).out_buf.empty()) level = std::max(level, pn.at(pid).level + 1);
    p.level = level;
    nc.level = level;
    nc.L = 2 * level + 1;  // node kernels run after the mixes of their level
    nc.dyn_params = dyn_params;
    const bool fuse = eng->fuse;
    nc.fuse_n = fuse && !dyn_params;  // nodes with automated params run their own a-rate kernels
    // does this node extend the pending chain of its only producer / take it as the destination's only input?
    const bool chain_kind = !dyn_params && ((n.kind == K_BIQUAD && !eng->serial_filters) || (fuse && (n.kind == K_GAIN || (n.kind == K_SHAPER && !(n.oversample && n.has_curve)))));
    if (fuse && n.n_inputs == 1 && p.in_edges[0].size() == 1 && p.in_edges[0][0].port == 0) {
        auto it = pending.find(p.in_edges[0][0].node);
        if (it != pending.end()) {
            int sch = pn.at(it->first).out_ch[0];
            if (chain_kind && computed_channels(n.cfg, sch) == sch && chain_accepts(it->second, n.kind)) {
                nc.extend = true;
                nc.fuse_src = it->first;
            } else if (n.kind == K_DEST && g->length <= 0xffffffffull &&
                       (sch == (int)g->channels || (sch == 1 && g->channels == 2 && n.cfg.interp == WAE_INTERPRETATION_SPEAKERS))) {
                nc.dest_direct = true;
                nc.fuse_src = it->first;
            }
        }
    }
    const std::vector<int> vsum_nb = voice_sum_ports(nc);
    for (size_t pi = 0; pi < p.in_edges.size(); pi++) {
        if (vsum_nb[pi] >= 0) continue;
        auto& port = p.in_edges[pi];
        for (auto& r : port)
            if (!((nc.extend || nc.dest_direct) && r.node == nc.fuse_src))
                if (!materialize(r.node, n.kind == K_CONV && n.buffer && port.size() == 1)) return false;
    }
    p.in_ch.assign(n.n_inputs, 1);
    p.in_buf.assign(n.n_inputs, BufRef{nullptr, 0, 0});
    p.in_lay.assign(n.n_inputs, Lay::fixed(1));
    for (int port = 0; port < n.n_inputs; port++)
        if (!plan_port(nc, port, vsum_nb[port])) return false;
    nc.in0 = p.in_lay.empty() ? Lay::fixed(1) : p.in_lay[0];
    return true;
}

// ---- k_voice_sum (WAE_OPT_VOICE_SUM): a port fed by many oscillator -> [biquad] -> gain voices, all of them still pending chains
// (mono, constant layout, one consumer): the voices are not materialised, one kernel renders them and keeps the running sum in
// registers, in the port's edge order.  Only when the launch has enough (2048-frame tile, port) work items to fill the machine
// about twice: one graph with thousands of voices and a short render (configs[2]) is better served by k_chain + k_mix, which
// take their parallelism from the voices.
// Per input port: the biquads of each of its voices when it is rendered that way, else -1.
std::vector<int> Planner::voice_sum_ports(const NodeCtx& nc) {
    const Node& n = nc.n;
    std::vector<int> port_vsum_nb(nc.p.in_edges.size(), -1);
    if (!(eng->fuse && voice_sum_mode() != 0 && !nc.extend && !nc.dest_direct && cur_cls == 0 && n.kind != K_DELAY_R)) return port_vsum_nb;
    for (size_t pi = 0; pi < nc.p.in_edges.size() && (int)pi < n.n_inputs; pi++) {
        const auto& edges = nc.p.in_edges[pi];
        if ((int)edges.size() < 8) continue;
        const int ch = computed_channels(n.cfg, 1);
        if (!(ch == 1 || (ch == 2 && n.cfg.interp == WAE_INTERPRETATION_SPEAKERS))) continue;
        if (n.kind == K_DEST && g->length > 0xffffffffull) continue;
        const int64_t tiles = (seg_end - seg_start + 2047) / 2048;
        if (voice_sum_mode() < 2 && tiles * (int64_t)group_graphs < 2 * (int64_t)voice_sum_slots()) continue;
        int nb = -1;
        bool ok = true;
        std::set<uint32_t> seen_nodes;
        for (auto& r : edges) {
            auto it = pending.find(r.node);
            if (r.port != 0 || it == pending.end()) { ok = false; break; }
            const PendingChain& pc = it->second;
            if (pc.inst.src_kind != CHAIN_SRC_OSC || pc.ch != 1 || pc.inst.has_shaper || pc.inst.n_biquad > 1 || pc.lay.dyn() || pc.cls != cur_cls ||
                (nb >= 0 && nb != pc.inst.n_biquad) || !seen_nodes.insert(r.node).second) { ok = false; break; }
            nb = pc.inst.n_biquad;
        }
        if (!ok) continue;
        port_vsum_nb[pi] = nb;
    }
    return port_vsum_nb;
}

// one input port: its channel count, layout and buffer (`vsum_nb` >= 0: its voices and their sum in one kernel, see voice_sum_ports)
bool Planner::plan_port(NodeCtx& nc, int port, int vsum_nb) {
    Node& n = nc.n; PNode& p = nc.p;
    NodeTable& pn = node_table;
    auto& edges = p.in_edges[port];
    int max_in = 1;
    for (auto& r : edges) max_in = std::max(max_in, pn.at(r.node).out_ch[r.port]);
    int ch = computed_channels(n.cfg, max_in);
    if (n.kind == K_DELAY_R) {  // the reader's only input is the hidden writer edge: take the writer's layout
        ch = max_in;
    }
    p.in_ch[port] = ch;
    p.in_lay[port] = Lay::fixed(ch);
    bool is_dest = n.kind == K_DEST;
    if (nc.extend || nc.dest_direct) {  // the producer's chain is consumed in registers / written directly
        if (nc.extend) p.in_lay[port] = pending.at(nc.fuse_src).lay;
        return true;
    }
    if (vsum_nb >= 0) return sum_voices(nc, port, ch, vsum_nb);
    if (is_dest && edges.size() == 1 && pn.at(edges[0].node).wrote_dest) {  // the producer already wrote the rendered PCM
        p.in_buf[port] = pn.at(edges[0].node).out_buf[edges[0].port];
        return true;
    }
    // ---- the port's layout over time: AudioRenderQuantum::add folded over the edges (quantum.rs:532-569)
    bool any_dyn = false;
    Lay pl = Lay::fixed(ch);
    if (!edges.empty()) {
        int lo = 1, hi = 1, on_nlo = 0, min_nlo = 255;
        bool all_may_silent = true;
        for (auto& r : edges) {
            const Lay el = pn.at(r.node).lay_out(r.port);
            any_dyn = any_dyn || el.dyn();
            lo = std::max<int>(lo, el.lo);
            hi = std::max<int>(hi, el.hi);
            if (!el.may_silent) on_nlo = std::max<int>(on_nlo, el.nlo);
            min_nlo = std::min<int>(min_nlo, el.nlo);
            all_may_silent = all_may_silent && el.may_silent;
        }
        const int nlo = std::max(on_nlo, min_nlo);
        pl.lo = (uint8_t)computed_channels(n.cfg, lo);
        pl.hi = (uint8_t)computed_channels(n.cfg, hi);
        pl.nlo = (uint8_t)computed_channels(n.cfg, nlo);
        pl.nhi = pl.hi;
        pl.may_silent = all_may_silent;
        if (n.kind == K_DELAY_R) pl = pn.at(edges[0].node).lay_out(edges[0].port);
    }
    // more than two layouts meeting in a port wider than stereo: the order of the up-mixes matters (mono, stereo, 5.1: the
    // reference goes 1 -> 2 -> 6): fold edge by edge like it does
    bool needs_fold = false;
    if (ch > 2 && n.cfg.mode != WAE_COUNT_MODE_EXPLICIT)
        for (auto& r : edges) needs_fold = needs_fold || pn.at(r.node).out_ch[r.port] != ch;
    if (!is_dest && edges.size() == 1 && pn.at(edges[0].node).out_ch[edges[0].port] == ch) {
        const Lay el = pn.at(edges[0].node).lay_out(edges[0].port);
        // a single edge IS the port when computedNumberOfChannels leaves every count it can have alone
        const bool identity = !el.dyn() || n.kind == K_DELAY_R || n.cfg.mode == WAE_COUNT_MODE_MAX ||
                              (n.cfg.mode == WAE_COUNT_MODE_CLAMPED_MAX && el.hi <= n.cfg.count);
        // the time-batched convolver reads all static channels of every quantum: it needs the canonical PCM k_mix_dyn writes
        const bool canonical_needed = el.dyn() && n.kind == K_CONV;
        if (identity && !canonical_needed) {
            p.in_buf[port] = pn.at(edges[0].node).out_buf[edges[0].port];  // alias, no copy
            p.in_lay[port] = el;
            return true;
        }
    }
    const bool dyn = any_dyn || needs_fold;
    if (!mix(2 * nc.level, edges, ch, n.cfg, is_dest, dyn, dyn && pl.dyn(), p.in_buf[port])) return false;
    if (dyn) p.in_lay[port] = pl;
    return true;
}

// the voices of this port and their sum in one kernel
bool Planner::sum_voices(NodeCtx& nc, int port, int ch, int nb) {
    auto& edges = nc.p.in_edges[port];
    StageBuild& vs = stage(2 * nc.level, S_VSUM, nb);
    VoiceGroup vg{};
    vg.first = (int32_t)vs.chain.size();
    vg.n_voices = (int32_t)edges.size();
    vg.out_dup = ch;
    vg.limit = -1;
    if (nc.n.kind == K_DEST) {
        vg.out = dest_ref();
        vg.limit = (int64_t)g->length;
    } else {
        vg.out = arena_buf(ch);
        if (!vg.out.p) return no_arena();
    }
    for (auto& r : edges) {
        PendingChain pc = std::move(pending.at(r.node));
        pending.erase(r.node);
        // (k_voice_sum prefetches the constants of voice k as coefficient set k: one set per voice, in voice order)
        if (pc.inst.n_biquad == 1 && vs.n_scan_coef != vs.chain.size()) return bail(WAE_UNSUPPORTED, "internal: voice-sum coefficient table out of step");
        for (int k = 0; k < pc.inst.n_biquad; k++)
            pc.inst.bq[k].coef = vs.add_scan_coef(want_scan_coefs, [&] { return make_scan_coef(pc.coefs[k]); });
        pc.inst.limit = -1;
        pc.inst.out_dup = 0;
        chain_entries(vs, pc, (int32_t)vs.chain.size());
        vs.chain.push_back(pc.inst);
    }
    vs.vgroups.push_back(vg);
    if (nc.n.kind == K_DEST) add_out(vs, offsetof(VoiceGroup, out), T_C);
    nc.p.in_buf[port] = vg.out;
    return true;
}

// ---- one lowering per node kind -------------------------------------------------------------------------------------------
bool Planner::lower_dest(NodeCtx& nc) {
    PNode& p = nc.p;
    p.out_ch = {(int)g->channels};
    if (nc.dest_direct) {  // the chain writes the rendered PCM itself (speaker up-mix 1->2 = copy, quantum.rs:301-305)
        PendingChain pc = std::move(pending.at(nc.fuse_src));
        pending.erase(nc.fuse_src);
        const BufRef fin = dest_ref();
        pc.inst.out = fin;
        pc.inst.limit = (int64_t)g->length;
        pc.inst.out_dup = (pc.ch == 1 && g->channels == 2) ? 2 : 0;
        add_out(emit_chain(pc, nc.L), offsetof(ChainInst, out));
        node_table.at(nc.fuse_src).out_buf = {fin};
        p.in_buf[0] = fin;
    }
    p.out_buf = {p.in_buf[0]};
    if (const std::vector<Edge>* outs = ord.edges.find(nc.id))
        for (auto& e : *outs)
            if (e.other_index >= 0 && dest_reader < 0) dest_reader = gi;
    algorithmic_bytes += (uint64_t)g->channels * g->length * 4;  // destination write, SURVEY §8(d)
    return true;
}

bool Planner::lower_osc(NodeCtx& nc) {
    Node& n = nc.n; PNode& p = nc.p;
    const double sr = (double)g->sample_rate;
    PRef pf = param_ref(n.params[0]), pd = param_ref(n.params[1]);
    float freq = pf.v, detune = pd.v;
    if (!nc.fuse_n && !need_out(nc, 1)) return false;
    OscInst o{};
    double start_ratio = 0.;
    if (!nc.fuse_n) o.out = p.out_buf[0];
    o.type = n.type;
    double computed_freq = (double)freq * std::exp2((double)detune / 1200.);  // oscillator.rs:30-32
    o.incr = computed_freq / sr;
    o.inv_incr = o.incr != 0. ? 1. / o.incr : 0.;
    o.outside_nyquist = std::fabs(computed_freq) >= sr / 2.;
    o.n_first = std::numeric_limits<int64_t>::max();
    o.n_stop = std::numeric_limits<int64_t>::max();
    o.phase0 = 0.;
    if (n.start_time < 1e300) {
        const OscStart st = osc_start(clock, n.start_time, o.incr, o.outside_nyquist);
        o.n_first = st.n_first;
        o.phase0 = st.phase0;
        start_ratio = st.start_ratio;
        o.n_stop = osc_stop_frame(clock, n.stop_time);
    }
    // a schedule bound from device memory: the fields the times reach are re-derived by the bind (planned with the windows' low ends)
    SchedPatch sched{};
    if (n.device_schedule) sched = sched_entry(n, nc.dyn_params ? SCHED_OSC_AR : SCHED_OSC);
    SchedPatch meta_sched = sched;
    meta_sched.kind = SCHED_META_OSC;
    const SchedPatch* track_sched = n.device_schedule ? &meta_sched : nullptr;
    // frequency / detune bound from device memory, planned with their placeholders.  With the other param automated the a-rate kernel
    // takes the bound value raw (PATCH_RAW into f_val / d_val).  Otherwise the declared ranges keep every computed frequency inside
    // (0, Nyquist), so the path and OscInst::fast hold for every value, and a PATCH_OSC entry re-derives the phase fields per bind: from
    // the planned start time, or from the slot a bound schedule writes its start into.
    const bool pitch_bound = pf.bound >= 0 || pd.bound >= 0;
    Entry pitch = patch(PATCH_OSC, 2);
    if (pitch_bound && !nc.dyn_params) {
        const double f_lo = pf.bound >= 0 ? pf.lo : freq, f_hi = pf.bound >= 0 ? pf.hi : freq;
        const double d_lo = pd.bound >= 0 ? pd.lo : detune, d_hi = pd.bound >= 0 ? pd.hi : detune;
        if (!hm::osc_pitch_inside(f_lo, f_hi, d_lo, d_hi, sr)) {
            const uint32_t caller = b->order.empty() ? gi : b->order[gi];
            return bail(WAE_UNSUPPORTED, "graph " + std::to_string(caller) + ", OscillatorNode " + std::to_string(n.id) +
                                             ": the pitch bound from device memory allows computed frequencies outside (0, sampleRate / 2) "
                                             "with frequency [" + std::to_string(f_lo) + ", " + std::to_string(f_hi) + "] Hz and detune [" +
                                             std::to_string(d_lo) + ", " + std::to_string(d_hi) +
                                             "] cents (bind a wider pitch as a value curve: wae_param_set_device_value_curve)");
        }
        operand(pitch, 0, pf, freq);
        operand(pitch, 1, pd, detune);
        pitch.p.param.sample_rate = g->sample_rate;
        double* start = upload(std::vector<double>{n.start_time});
        if (!start) return bail(WAE_OUT_OF_MEMORY, "out of device memory (oscillator start time)");
        pitch.p.param.dst2 = start;
        if (n.device_schedule) sched.start_out = start;
    }
    if (n.type == WAE_OSC_CUSTOM && n.device_wave) {  // a wave bound from device memory: planned as a host wave of its length
        o.table = device_wave(n);
        o.table_len = (int)n.device_wave_len;
        if (!o.table) return false;
    } else if (n.type == WAE_OSC_CUSTOM) {
        float* d = upload(n.table);
        o.table = d;
        o.table_len = (int)n.table.size();
    } else {
        o.table = eng->d_sine;
        o.table_len = 2048;
    }
    o.fast = (!o.outside_nyquist && o.incr > 0. && o.incr < 0.5 && (o.table_len == 2048 || (o.type != WAE_OSC_SINE && o.type != WAE_OSC_CUSTOM))) ? 1 : 0;
    if (nc.dyn_params) {  // automated / audio-rate frequency or detune: running-sum phase
        OscArInst oa{};
        oa.base = o;
        oa.freq = pf.dyn ? pf.track : BufRef{nullptr, 0, 0};
        oa.detune = pd.dyn ? pd.track : BufRef{nullptr, 0, 0};
        oa.f_val = freq;
        oa.d_val = detune;
        oa.start_ratio = start_ratio;
        oa.phase = alloc<double>(1, true, true);
        oa.sample_rate = g->sample_rate;
        if (!oa.phase) return bail(WAE_OUT_OF_MEMORY, "out of device memory (state)");
        oa.base.out = source_out(nc, o.n_first, o.n_stop, 1, track_sched);
        StageBuild& sb = stage(nc.L, S_OSC_AR);
        sb.osc_ar.push_back(oa);
        if (n.device_schedule) add_sched_patch(sb, n, sched);
        const PRef* refs[2] = {&pf, &pd};
        const size_t offs[2] = {offsetof(OscArInst, f_val), offsetof(OscArInst, d_val)};
        for (int i = 0; i < 2; i++)
            if (refs[i]->bound >= 0) {
                Entry r = patch(PATCH_RAW, 1);
                operand(r, 0, *refs[i], refs[i]->v);
                add_patch(sb, r, offs[i]);
            }
    } else if (nc.fuse_n) {
        PendingChain pc = source_chain(CHAIN_SRC_OSC, 1);
        pc.inst.osc = o;
        pc.lay = source_lay(o.n_first, o.n_stop, 1, n.device_schedule);
        if (n.device_schedule) pc.add_entry(sched_patch(n, sched), offsetof(ChainInst, osc), offsetof(SchedPatch, dst));
        if (pitch_bound) pc.add_entry(pitch, offsetof(ChainInst, osc), offsetof(ParamPatch, dst));
        return finish_chain(nc, std::move(pc));
    } else {
        o.out = source_out(nc, o.n_first, o.n_stop, 1, track_sched);
        StageBuild& sb = stage(nc.L, S_OSC);
        sb.osc.push_back(o);
        if (n.device_schedule) add_sched_patch(sb, n, sched);
        if (pitch_bound) add_patch(sb, pitch, 0);
    }
    return true;
}

bool Planner::lower_const(NodeCtx& nc) {
    Node& n = nc.n; PNode& p = nc.p;
    PRef po = param_ref(n.params[0]);
    float v = po.v;
    if (!nc.fuse_n && !need_out(nc, 1)) return false;
    ConstInst c{};
    if (!nc.fuse_n) c.out = p.out_buf[0];
    if (po.dyn) c.track = po.track;
    c.value = v;
    c.n_first = std::numeric_limits<int64_t>::max();
    c.n_stop = std::numeric_limits<int64_t>::max();
    if (n.start_time < 1e300) {
        // constant_source.rs:203-246
        c.n_first = clock.first_frame_at_or_after(n.start_time);
        if (n.stop_time < 1e300) c.n_stop = clock.first_frame_at_or_after(n.stop_time);
    }
    // a schedule bound from device memory: the fields the times reach are re-derived by the bind (planned with the windows' low ends)
    const SchedPatch sched = sched_entry(n, SCHED_CONST);
    SchedPatch meta_sched = sched;
    meta_sched.kind = SCHED_META_CONST;
    if (nc.fuse_n) {
        PendingChain pc = source_chain(CHAIN_SRC_CONST, 1);
        pc.inst.cst = c;
        pc.lay = source_lay(c.n_first, c.n_stop, 1, n.device_schedule);
        if (n.device_schedule) pc.add_entry(sched_patch(n, sched), offsetof(ChainInst, cst), offsetof(SchedPatch, dst));
        return finish_chain(nc, std::move(pc));
    }
    c.out = source_out(nc, c.n_first, c.n_stop, 1, n.device_schedule ? &meta_sched : nullptr);
    StageBuild& sb = stage(nc.L, S_CONST);
    sb.cst.push_back(c);
    if (n.device_schedule) add_sched_patch(sb, n, sched);
    return true;
}

// A looping source whose loop points are bound from device memory, on the bound slow track: the capacity of its playhead table (segments),
// or 0 when its windows and computed rates [rate_lo, rate_hi] do not allow the track.  Decided from the declared ranges only.
//  - The shortest actual loop the windows allow is min(end_lo, duration) - min(start_hi, duration) (clamp_loop_boundaries); it must be
//    longer than four output frames at the top rate (the host rule of a built loop), so no frame wraps twice.  Overlapping windows fail.
//  - A step at the lowest rate wider than two snap zones (almost::equal around a loop point: < 3e-8 (1 + duration)) lets at most one
//    frame per pass be snapped without a wrap.
//  - Over `frames` frames the playhead advances at most frames * dt * rate_hi; each wrap takes back at least the shortest loop, so it
//    wraps at most W = floor(frames * dt * rate_hi / shortest) + 1 times.  Every segment is a wrap or a snap, and a snap without a wrap
//    happens once, on the way into the loop: at most W + 2 segments with the first.  The capacity is 2 (W + 1) + 4, which also covers the
//    rounding of the device's exp2 and the snaps' own displacement of the playhead.
constexpr int32_t kLoopSegmentsMax = 1 << 16;  // per record: 1 MiB of table
static int32_t absn_loop_capacity(const Node& n, double duration, double dt, double rate_lo, double rate_hi, int64_t frames) {
    const double max_start = std::min(n.loop_hi[0], duration);
    const double min_end = n.loop_lo[1] > duration ? duration : n.loop_lo[1];
    const double shortest = min_end - max_start;
    if (!(shortest > 4. * dt * rate_hi)) return 0;
    if (!(dt * rate_lo > 6.0e-8 * (1. + duration))) return 0;
    const double wraps = std::floor((double)frames * dt * rate_hi / shortest) + 1.;
    const double cap = 2. * (wraps + 1.) + 4.;
    return cap > (double)kLoopSegmentsMax ? 0 : (int32_t)cap;
}

bool Planner::lower_absn(NodeCtx& nc) {
    Node& n = nc.n;
    const double sr = (double)g->sample_rate;
    PRef pdet = param_ref(n.params[0]), prate = param_ref(n.params[1]);
    const float detune = pdet.v, rate = prate.v;
    const bool rate_automated = pdet.dyn || prate.dyn;
    const bool rate_bound = pdet.bound >= 0 || prate.bound >= 0;
    int ch = n.buffer ? (int)n.buffer->channels.size() : 1;
    if (!n.buffer || n.start_time >= 1e300 || ch == 0) return absn_silent(nc);  // never plays: silence
    PcmBuffer& pb = *n.buffer;
    double computed_rate = (double)rate * std::exp2((double)detune / 1200.);
    double duration = pb.duration();
    double ls = n.loop_start, le = n.loop_end;  // clamp_loop_boundaries, audio_buffer_source.rs:400-417
    if (ls < 0.) ls = 0.; else if (ls > duration) ls = duration;
    if (le <= 0. || le > duration) le = duration;
    const int64_t q = absn_start_quantum(clock, n.start_time);
    bool aligned = (n.start_time <= clock.block_time(q)) && n.offset == 0.;  // start in the past snaps to the block
    // (a schedule bound from device memory: the start may fall anywhere, the bound slow track or the serial kernel plays it)
    bool fast = !rate_automated && !rate_bound && !n.device_schedule && !n.device_loop && aligned && (double)pb.sample_rate / sr == 1. && computed_rate == 1. &&
                ls == 0. && le == duration && n.duration > 1e300 && n.stop_time > 1e300;
    // everything the closed-form tracks do not cover runs the renderer's own frame loop (one warp per source)
    bool serial = rate_automated || (!fast && !(computed_rate > 0.)) || (n.device_schedule && n.loop);
    // playbackRate / detune bound from device memory: the path follows from the computed rates their declared ranges allow (the low
    // corner's exp2 underflows to 0 far enough below 0 cents), never from the value.  A non-looping source whose rates are all positive
    // takes the bound slow track; the serial kernel is right for every other value.
    double rate_lo = computed_rate, rate_hi = computed_rate;
    if (rate_bound) {
        const bool br = prate.bound >= 0, bd = pdet.bound >= 0;
        rate_lo = (double)(br ? prate.lo : rate) * std::exp2((double)(bd ? pdet.lo : detune) / 1200.);
        rate_hi = (double)(br ? prate.hi : rate) * std::exp2((double)(bd ? pdet.hi : detune) / 1200.);
        serial = rate_automated || n.loop || !(rate_lo > 0.);
    }
    // loop points bound from device memory: the bound slow track when the windows and the rates allow a playhead table of bounded size
    // (absn_loop_capacity), else the serial kernel
    int32_t loop_cap = 0;
    if (n.device_loop) {
        loop_cap = rate_automated || !(rate_lo > 0.) ? 0 : absn_loop_capacity(n, duration, clock.dt, rate_lo, rate_hi, lq);
        serial = loop_cap == 0;
    }
    if (!fast && !serial && n.loop && !n.device_loop) {
        const bool custom = ls >= 0. && le > 0. && ls < le;
        const double loop_len = custom ? le - ls : duration;
        if (!(loop_len > 4. * clock.dt * computed_rate)) serial = true;  // loop shorter than four output frames
    }
    const bool fused = nc.fuse_n && fast;
    if (!fused && !need_out(nc, ch)) return false;
    size_t len = pb.length();
    size_t stride = (len + 3) / 4 * 4;  // every channel starts 16 B aligned (LDG.128)
    // a device input read by reference has no slab memory: its records get a placeholder pointer and the slab's stride (the plan sizes as
    // its copy-declared twin's does), and an entry each that its bind rewrites with the caller's pointer and stride
    float* d_buf = reinterpret_cast<float*>(uintptr_t(256));
    if (!pb.by_reference) {
        // one copy of the PCM per AudioBuffer in the group's slab (the grains of a granular patch all play the same one: the graph
        // holds it once, wae_abi_graph.cpp copy_buffer), shared by the plans of all render segments
        auto so = src_offsets.find({gi, nc.id});
        bool first_use = so == src_offsets.end();
        if (first_use) {
            auto bo = buf_offsets.find(n.buffer.get());
            if (bo != buf_offsets.end()) first_use = false;  // (already in the slab for another node)
            else bo = buf_offsets.emplace(n.buffer.get(), src_cursor).first;
            so = src_offsets.emplace(std::make_pair(gi, nc.id), bo->second).first;
        }
        d_buf = d_src + so->second;
        if (first_use) {
            if (src_copies)  // recorded by the sizing pass: uploaded straight from the graph's buffer, planar [ch][stride] like the slab
                src_copies->push_back(wae_batch::Group::SrcCopy{n.buffer, src_cursor, (size_t)ch * stride, gi, nc.id});
            src_cursor += (size_t)ch * stride;
            b->asset_bytes += (size_t)ch * len * 4;
        }
    }
    const AbsnPlay s{&pb, d_buf, len, stride, ch, duration, ls, le, computed_rate, pb.by_reference};
    if (serial) return absn_serial(nc, s, pdet, prate);
    if (rate_bound || n.device_schedule || n.device_loop) return absn_bound(nc, s, pdet, prate, q, aligned, rate_hi, loop_cap);
    if (!fast) return absn_slow(nc, s);
    return absn_fast(nc, s, q, fused);
}

bool Planner::absn_silent(NodeCtx& nc) {
    if (!need_out(nc, 1)) return false;
    StageBuild& ms = stage(nc.L, S_MIX);
    ms.mix.push_back(MixInst{nc.p.out_buf[0], 1, 0, 0, (uint32_t)ms.mix_edges.size(), -1});
    out_dynamic(nc, Lay{1, 1, 1, 1, true});  // silent for good
    if (nc.p.out_buf[0].meta) source_meta(nc, 0, 0, 1);
    return true;
}

bool Planner::absn_serial(NodeCtx& nc, const AbsnPlay& s, const PRef& pdet, const PRef& prate) {
    Node& n = nc.n;
    AbsnSerialInst a{};
    a.out = nc.p.out_buf[0];
    a.buf = s.buf;
    a.buf_len = (int64_t)s.len;
    a.buf_stride = (int64_t)s.stride;
    a.start_time = n.start_time;
    a.stop_time = n.stop_time;
    a.offset = n.offset;
    a.duration = n.duration;
    a.loop_start = s.ls;
    a.loop_end = s.le;
    a.buffer_duration = s.duration;
    a.buffer_sample_rate = (double)s.pb->sample_rate;
    a.sample_rate = (double)g->sample_rate;
    const BufRef none{nullptr, 0, 0};
    a.rate_track = prate.dyn ? prate.track : none;
    a.detune_track = pdet.dyn ? pdet.track : none;
    a.rate = prate.v;
    a.detune = pdet.v;
    a.ch = s.ch;
    a.loop = n.loop ? 1 : 0;
    a.state = alloc<AbsnSerialState>(1, true, true);
    if (!a.state) return bail(WAE_OUT_OF_MEMORY, "out of device memory (buffer source state)");
    out_dynamic(nc, Lay::gated(s.ch));  // when it plays depends on the automated rate: the kernel writes the layout track
    a.out = nc.p.out_buf[0];
    StageBuild& sb = stage(nc.L, S_ABSN_SERIAL);
    sb.absn_serial.push_back(a);
    if (s.by_ref) add_src_ref(sb, n, offsetof(AbsnSerialInst, buf), offsetof(AbsnSerialInst, buf_stride));
    const PRef* refs[2] = {&pdet, &prate};
    const size_t offs[2] = {offsetof(AbsnSerialInst, detune), offsetof(AbsnSerialInst, rate)};
    for (int i = 0; i < 2; i++)
        if (refs[i]->bound >= 0) {  // bound from device memory (the kernel takes the raw values)
            Entry r = patch(PATCH_RAW, 1);
            operand(r, 0, *refs[i], refs[i]->v);
            add_patch(sb, r, offs[i]);
        }
    if (n.device_schedule) add_sched_patch(sb, n, sched_entry(n, SCHED_ABSN_SERIAL));  // (the raw start / stop times)
    if (n.device_loop) {  // (the loop points after clamp_loop_boundaries)
        Entry e = entry(E_LOOP, n.id);
        e.p.loop = LoopPatch{nullptr, LOOP_SERIAL, 0, s.duration};
        sb.add_entry(e, 0, offsetof(LoopPatch, dst));
    }
    algorithmic_bytes += (uint64_t)s.ch * 4ull * (uint64_t)std::min<int64_t>(lq, (int64_t)s.len);
    return true;
}

// ---- slow track (audio_buffer_source.rs:625-823): fractional playhead
bool Planner::absn_slow(NodeCtx& nc, const AbsnPlay& s) {
    Node& n = nc.n;
    const double sr = (double)g->sample_rate;
    const double duration = s.duration, computed_rate = s.computed_rate;
    AbsnSlowInst a{};
    a.out = nc.p.out_buf[0];
    a.buf = s.buf;
    a.buf_len = (int64_t)s.len;
    a.buf_stride = (int64_t)s.stride;
    a.ch = s.ch;
    a.loop = n.loop ? 1 : 0;
    a.sample_rate = sr;
    a.buffer_duration = duration;
    a.pos_scale = ((double)s.pb->sample_rate / sr) * sr;  // position = buffer_time * sampling_ratio; playhead = position * sr
    a.duration = n.duration;
    // actual loop points (:627-636)
    if (n.loop && s.ls >= 0. && s.le > 0. && s.ls < s.le) {
        a.loop_start = s.ls;
        a.loop_end = s.le;
    } else {
        a.loop_start = 0.;
        a.loop_end = duration;
    }
    const AbsnStart st = absn_start(clock, n.start_time, n.stop_time);
    const int64_t n_first = st.n_first;
    a.n_first = n_first;
    a.n_stop = st.n_stop;
    const AbsnSlowDerived d = absn_slow_derive(clock.dt, computed_rate, n.offset, st.t_first - st.start, duration, n.duration, n.loop, a.loop_end,
                                               n_first, a.n_stop);
    a.step = d.step;
    a.offset0 = d.offset0;
    a.elapsed0 = d.elapsed0;
    std::vector<int64_t> seg_n(64);
    std::vector<double> seg_bt(64);
    int32_t n_seg = 1;
    seg_n[0] = n_first;
    seg_bt[0] = d.offset0;
    const int64_t n_end = std::min<int64_t>(lq, a.n_stop);
    while (n.loop && (n_seg = absn_loop_segments(a.loop_start, a.loop_end, d.step, n_first, n_end, d.offset0, seg_n.data(), seg_bt.data(),
                                                 (int32_t)seg_n.size())) < 0) {
        seg_n.resize(seg_n.size() * 4);
        seg_bt.resize(seg_bt.size() * 4);
    }
    seg_n.resize(n_seg);
    seg_bt.resize(n_seg);
    a.n_seg = n_seg;
    a.seg_n = upload(seg_n);
    a.seg_bt = upload(seg_bt);
    // layout: silent before the quantum of the first playing frame and after the quantum in which the source ends
    // (stop time, explicit duration, or — not looping — the end of the buffer; audio_buffer_source.rs:826-838)
    a.out = source_out(nc, n_first, d.n_end, s.ch);
    StageBuild& sb = stage(nc.L, S_ABSN_SLOW);
    sb.absn_slow.push_back(a);
    if (s.by_ref) add_src_ref(sb, n, offsetof(AbsnSlowInst, buf), offsetof(AbsnSlowInst, buf_stride));
    algorithmic_bytes += (uint64_t)s.ch * 4ull * (uint64_t)std::min<int64_t>(lq, (int64_t)s.len);
    return true;
}

// ---- playbackRate / detune bound from device memory, a non-looping source whose declared rates are all positive: the slow track's
// constants that do not depend on the rate, and the bound values (PATCH_RAW); k_buffer_source_slow<true> derives the rest per run
bool Planner::absn_bound(NodeCtx& nc, const AbsnPlay& s, const PRef& pdet, const PRef& prate, int64_t q, bool aligned, double rate_hi,
                         int32_t loop_cap) {
    Node& n = nc.n;
    const double sr = (double)g->sample_rate;
    AbsnBoundInst r{};
    AbsnSlowInst& a = r.s;
    a.buf = s.buf;
    a.buf_len = (int64_t)s.len;
    a.buf_stride = (int64_t)s.stride;
    a.ch = s.ch;
    a.sample_rate = sr;
    a.buffer_duration = s.duration;
    a.pos_scale = ((double)s.pb->sample_rate / sr) * sr;
    a.duration = n.duration;
    a.loop_end = s.duration;
    const AbsnStart st = absn_start(clock, n.start_time, n.stop_time);
    a.n_first = st.n_first;
    a.n_stop = st.n_stop;
    r.dt = clock.dt;
    r.offset = n.offset;
    r.start_delta = st.t_first - st.start;
    r.n_start = q * 128;
    r.fast_end = absn_fast_end(clock, lq, r.n_start, s.duration);
    const bool fast_shape = (double)s.pb->sample_rate / sr == 1. && s.ls == 0. && s.le == s.duration && n.duration > 1e300 && !n.device_loop;
    r.fast_ok = aligned && fast_shape && n.stop_time > 1e300;
    if (n.device_loop) {  // the placeholders' actual loop points and a table of loop_cap segments, both rewritten by the binds
        const AbsnLoopPoints lp = absn_loop_points(n.loop_start, n.loop_end, s.duration);
        a.loop = 1;
        a.loop_start = lp.actual_start;
        a.loop_end = lp.actual_end;
        a.n_seg = 1;
        if (dry) {
            a.seg_n = reinterpret_cast<const int64_t*>(uintptr_t(256));
            a.seg_bt = reinterpret_cast<const double*>(uintptr_t(256));
        } else {
            a.seg_n = b->dalloc<int64_t>((size_t)loop_cap, true);
            a.seg_bt = b->dalloc<double>((size_t)loop_cap, true);
            if (!a.seg_n || !a.seg_bt) return bail(WAE_OUT_OF_MEMORY, "out of device memory (loop playhead table)");
            b->asset_bytes += (size_t)loop_cap * (sizeof(int64_t) + sizeof(double));
        }
    }
    r.rate = prate.v;
    r.detune = pdet.v;
    // The one decision the range drives: a constant layout only when the source plays to the end of the render at every rate it allows.
    // It ends first at the highest rate; a quantum of margin covers the device's exp2 rounding its last bit the other way.
    const AbsnSlowDerived top = absn_slow_derive(clock.dt, rate_hi, n.offset, r.start_delta, s.duration, n.duration, false, s.duration, a.n_first,
                                                 a.n_stop);
    const int64_t margin = (pdet.bound >= 0 || pdet.v != 0.f) ? 128 : 0;
    // (a schedule bound from device memory is always gated; a looping source never reaches the end of its buffer, so it plays to the
    // end of the render unless it stops or has a duration)
    const bool fixed = n.device_loop ? !n.device_schedule && a.n_first <= 0 && n.stop_time > 1e300 && n.duration > 1e300
                                     : !n.device_schedule && a.n_first <= 0 && top.n_end >= glq + margin && !(r.fast_ok && r.fast_end < glq);
    out_dynamic(nc, fixed ? Lay::fixed(s.ch) : Lay::gated(s.ch));  // (gated: the kernel writes the layout track)
    a.out = nc.p.out_buf[0];
    StageBuild& sb = stage(nc.L, S_ABSN_BOUND);
    sb.absn_bound.push_back(r);
    if (s.by_ref)
        add_src_ref(sb, n, offsetof(AbsnBoundInst, s) + offsetof(AbsnSlowInst, buf), offsetof(AbsnBoundInst, s) + offsetof(AbsnSlowInst, buf_stride));
    if (n.device_schedule) {  // the start-dependent fields, re-derived by the bind; the kernel derives the rest per run as before
        SchedPatch sp = sched_entry(n, SCHED_ABSN_BOUND);
        sp.flag = fast_shape;
        sp.offset = n.offset;
        sp.duration = s.duration;
        add_sched_patch(sb, n, sp);
    }
    if (n.device_loop) {
        Entry e = entry(E_LOOP, n.id), w = entry(E_LOOP_WALK);
        e.p.loop = LoopPatch{nullptr, LOOP_BOUND, 0, s.duration};
        w.p.walk = LoopWalk{nullptr, lq, loop_cap, 0};
        sb.add_entry(e, 0, offsetof(LoopPatch, dst));
        sb.add_entry(w, 0, offsetof(LoopWalk, rec));
    }
    const PRef* refs[2] = {&pdet, &prate};
    const size_t offs[2] = {offsetof(AbsnBoundInst, detune), offsetof(AbsnBoundInst, rate)};
    for (int i = 0; i < 2; i++)
        if (refs[i]->bound >= 0) {
            Entry pr = patch(PATCH_RAW, 1);
            operand(pr, 0, *refs[i], refs[i]->v);
            add_patch(sb, pr, offs[i]);
        }
    algorithmic_bytes += (uint64_t)s.ch * 4ull * (uint64_t)std::min<int64_t>(lq, (int64_t)s.len);
    return true;
}

// fast track: the buffer played 1:1 from a block boundary (a chain source when it fuses)
bool Planner::absn_fast(NodeCtx& nc, const AbsnPlay& s, int64_t q, bool fused) {
    Node& n = nc.n; PNode& p = nc.p;
    AbsnInst a{};
    if (!fused) a.out = p.out_buf[0];
    a.buf = s.buf;
    a.buf_len = (int64_t)s.len;
    a.buf_stride = (int64_t)s.stride;
    a.n_start = q * 128;
    a.n_stop = std::numeric_limits<int64_t>::max();
    a.buf_offset = 0;
    a.ch = s.ch;
    a.loop = n.loop ? 1 : 0;
    if (!n.loop) a.n_stop = absn_fast_end(clock, lq, a.n_start, s.duration);
    if (fused) {
        PendingChain pc = source_chain(CHAIN_SRC_ABSN, s.ch);
        pc.inst.absn = a;
        pc.lay = source_lay(a.n_start, a.n_stop, s.ch);
        if (s.by_ref)
            pc.entries.push_back(src_ref(n, -1, offsetof(ChainInst, absn) + offsetof(AbsnInst, buf), offsetof(ChainInst, absn) + offsetof(AbsnInst, buf_stride)));
        if (!finish_chain(nc, std::move(pc))) return false;
    } else {
        a.out = source_out(nc, a.n_start, a.n_stop, s.ch);
        StageBuild& sb = stage(nc.L, S_ABSN);
        sb.absn.push_back(a);
        if (s.by_ref) add_src_ref(sb, n, offsetof(AbsnInst, buf), offsetof(AbsnInst, buf_stride));
    }
    // compulsory read of the source PCM that is actually played
    algorithmic_bytes += (uint64_t)s.ch * 4ull * (uint64_t)std::max<int64_t>(0, std::min<int64_t>(lq - a.n_start, n.loop ? lq : (int64_t)s.len));
    return true;
}

bool Planner::lower_biquad(NodeCtx& nc) {
    Node& n = nc.n; PNode& p = nc.p; const Lay& in0 = nc.in0;
    PRef pq = param_ref(n.params[0]), pdt = param_ref(n.params[1]), pfr = param_ref(n.params[2]), pg = param_ref(n.params[3]);
    float q = pq.v, detune = pdt.v, freq = pfr.v, gain = pg.v;
    int ch = p.in_ch[0];
    if (nc.dyn_params) {  // per-frame coefficients (biquad_filter.rs:837-855): serial a-rate kernel
        if (!need_out(nc, ch)) return false;
        BiquadArInst ba{};
        ba.in = p.in_buf[0];
        ba.out = p.out_buf[0];
        const BufRef none{nullptr, 0, 0};
        ba.q = pq.dyn ? pq.track : none;
        ba.detune = pdt.dyn ? pdt.track : none;
        ba.freq = pfr.dyn ? pfr.track : none;
        ba.gain = pg.dyn ? pg.track : none;
        ba.q_val = q; ba.detune_val = detune; ba.freq_val = freq; ba.gain_val = gain;
        ba.state = alloc<double>((size_t)ch * 4, true, true);
        if (!ba.state) return bail(WAE_OUT_OF_MEMORY, "out of device memory (state)");
        if (!filter_dyn_len(nc, ch, ba.dyn_len)) return false;
        ba.out = p.out_buf[0];
        {
            // five planes of f64 coefficients per frame of the chunk (an arena buffer of 10 float channels read as doubles)
            BufRef cb = arena_buf(10);
            if (!cb.p) return no_arena();
            cb.stride = (uint32_t)b->chunk;  // in DOUBLES: plane k starts at double index k * chunk
            ba.coefs = cb;
        }
        ba.sample_rate = g->sample_rate;
        ba.type = n.type;
        ba.ch = ch;
        StageBuild& sb = stage(nc.L, S_BIQUAD_AR);
        sb.max_ch = std::max(sb.max_ch, ch);
        sb.biquad_ar.push_back(ba);
        // params bound from device memory next to automated ones: the constant operands of k_biquad_coefs
        const PRef* refs[4] = {&pq, &pdt, &pfr, &pg};
        const size_t offs[4] = {offsetof(BiquadArInst, q_val), offsetof(BiquadArInst, detune_val), offsetof(BiquadArInst, freq_val),
                                offsetof(BiquadArInst, gain_val)};
        for (int i = 0; i < 4; i++)
            if (refs[i]->bound >= 0) {
                Entry r = patch(PATCH_RAW, 1);
                operand(r, 0, *refs[i], refs[i]->v);
                add_patch(sb, r, offs[i]);
            }
        return true;
    }
    float cf = hm::biquad_computed_freq(freq, detune);
    hm::BiquadCoefs c = hm::biquad_coefs(n.type, (double)g->sample_rate, (double)cf, (double)gain, (double)q);
    // coefficients that depend on params bound from device memory: re-derived per bind
    const bool bound = pq.bound >= 0 || pdt.bound >= 0 || pfr.bound >= 0 || pg.bound >= 0;
    Entry bp = patch(PATCH_BIQUAD, n.type);
    bp.p.param.sample_rate = g->sample_rate;
    operand(bp, 0, pq, q);
    operand(bp, 1, pdt, detune);
    operand(bp, 2, pfr, freq);
    operand(bp, 3, pg, gain);
    double* state = alloc<double>((size_t)ch * 4, true, true);
    if (!state) return bail(WAE_OUT_OF_MEMORY, "out of device memory (state)");
    // An input whose channel COUNT changes while it sounds resets / drops channels of the filter mid-render
    // (biquad_filter.rs:798-815): the serial kernel follows it quantum by quantum; the scan keeps one state per channel
    const bool count_varies = !nc.extend && in0.dyn() && !(in0.nlo == in0.nhi && in0.nhi == ch);
    if (!eng->serial_filters && !count_varies) return append_biquad(nc, state, c, bound ? &bp : nullptr);
    // bit-faithful serial recurrence, one stage per biquad
    if (!need_out(nc, ch)) return false;
    BiquadInst bi{};
    if (!filter_dyn_len(nc, ch, bi.dyn_len)) return false;
    bi.in = p.in_buf[0];
    bi.out = p.out_buf[0];
    bi.b0 = c.b0; bi.b1 = c.b1; bi.b2 = c.b2; bi.a1 = c.a1; bi.a2 = c.a2;
    bi.ch = ch;
    bi.state = state;
    StageBuild& s = stage(nc.L, S_BIQUAD);
    s.max_ch = std::max(s.max_ch, ch);
    s.biquad.push_back(bi);
    if (bound) add_patch(s, bp, offsetof(BiquadInst, b0));
    return true;
}

bool Planner::lower_iir(NodeCtx& nc) {
    Node& n = nc.n; PNode& p = nc.p; const Lay& in0 = nc.in0;
    int ch = p.in_ch[0];
    std::vector<double> ff = n.feedforward, fb = n.feedback;  // iir_filter.rs:282-309
    if (ff.size() < fb.size()) ff.resize(fb.size(), 0.);
    if (ff.size() > fb.size()) fb.resize(ff.size(), 0.);
    if (ff.size() <= 3 && !eng->serial_filters && !in0.dyn() && seg_start == 0 && seg_end >= lq) {
        // Order <= 2 with a constant input layout: the same transfer function as a biquad — rendered by the time-parallel scan
        // of k_chain (direct form I there, transposed direct form II in iir_filter.rs:386-407: the outputs differ in the last
        // bits of the f64 arithmetic only) instead of one serial thread per channel.  With an input that can fall silent the
        // serial kernel stays: its tail test looks at the reference's own state variables.  Same for a render cut by suspend
        // points: the two forms keep different state (x / y history here, the reference's 20 accumulators there) and a later
        // segment may see a layout that needs the serial kernel — the filter memory must survive the cut (fuzz seeds 31, 33).
        ff.resize(3, 0.);
        fb.resize(3, 0.);
        const double a0 = fb[0];
        hm::BiquadCoefs c{ff[0] / a0, ff[1] / a0, ff[2] / a0, fb[1] / a0, fb[2] / a0};
        double* state = alloc<double>((size_t)ch * 4, true, true);
        if (!state) return bail(WAE_OUT_OF_MEMORY, "out of device memory (state)");
        return append_biquad(nc, state, c, nullptr, n.device_iir);
    }
    if (!need_out(nc, ch)) return false;
    IirInst ii{};
    ii.in = p.in_buf[0];
    ii.out = p.out_buf[0];
    ii.n = (int)ff.size();
    ii.ch = ch;
    double a0 = fb[0];
    for (size_t i = 0; i < ff.size(); i++) {
        ii.b[i] = ff[i] / a0;
        ii.a[i] = fb[i] / a0;
    }
    ii.state = alloc<double>((size_t)ch * 20, true, true);
    if (!ii.state) return bail(WAE_OUT_OF_MEMORY, "out of device memory (state)");
    if (!filter_dyn_len(nc, ch, ii.dyn_len)) return false;
    ii.out = p.out_buf[0];
    StageBuild& s = stage(nc.L, S_IIR);
    s.max_ch = std::max(s.max_ch, ch);
    s.iir.push_back(ii);
    // coefficients bound from device memory (wae_iir_filter_set_device_coefficients): the bind rewrites b[0..n) and a[0..n) of this
    // segment's record
    if (n.device_iir) {
        Entry e = entry(E_IIR, n.id);
        e.refer(1, T_A, (int32_t)s.records() - 1, offsetof(IirInst, a), offsetof(IirPatch, a));
        s.add_entry(e, offsetof(IirInst, b), offsetof(IirPatch, b));
    }
    return true;
}

bool Planner::lower_gain(NodeCtx& nc) {
    PNode& p = nc.p;
    PRef pgn = param_ref(nc.n.params[0]);
    float gv = pgn.v;
    int ch = p.in_ch[0];
    if (pgn.dyn) {  // a-rate gain (gain.rs:189-197)
        if (!need_out(nc, ch)) return false;
        out_like_input(nc);  // silent in -> silent out (gain.rs:155-158); the ~0 / ~1 shortcuts only exist for single values
        stage(nc.L, S_GAIN).gain.push_back(GainInst{p.in_buf[0], p.out_buf[0], gv, ch, pgn.track});
        return true;
    }
    // gain.rs:153-169: |g| <= 1e-6 -> silence, |1-g| <= 1e-6 -> pass-through (quanta >= 1; quantum 0 takes
    // the multiply path, a difference of at most 1e-6 * |x| that is below the parity tolerance)
    if (std::fabs(gv) <= 1e-6f) gv = 0.f;
    else if (std::fabs(1.f - gv) <= 1e-6f) gv = 1.f;
    // A gain bound from device memory is planned as this constant.  Whether it answers with silence depends on the value: when its
    // range does not exclude |g| <= 1e-6 its output is planned as the input's layout OR silence, and the bind decides
    const bool bound = pgn.bound >= 0;
    const bool may_zero = bound && !(pgn.lo > 1e-6f || pgn.hi < -1e-6f);
    const Lay or_silent{1, nc.in0.hi, nc.in0.nlo, nc.in0.nhi, true};
    if (nc.fuse_n) {
        PendingChain pc = open_chain(nc);
        // consecutive gains of one slot are folded (differs from two f32 multiplies by <= 1 ulp)
        const int slot = pc.phase == 0 ? 0 : (pc.phase == 1 ? 1 : (pc.phase == 3 ? 2 : 3));
        Entry& fold = pc.gain_fold[slot];
        if (bound || fold.p.param.n > 0) {  // the slot's factors in node order, from the first bound one on (the constant product before it first)
            if (fold.p.param.n == 0) {
                fold = patch(PATCH_GAIN, 1);
                fold.p.param.val[0] = pc.inst.g[slot];
                fold.refer(0, T_A, -1, offsetof(ChainInst, g) + (size_t)slot * sizeof(float), offsetof(ParamPatch, dst));
            }
            if (fold.p.param.n >= PATCH_OPS) return bail(WAE_UNSUPPORTED, "too many gains folded into one chain slot behind a gain bound from device memory");
            operand(fold, fold.p.param.n++, pgn, gv);
        }
        pc.inst.g[slot] *= gv;
        if (may_zero) pc.lay = Lay{1, pc.lay.hi, pc.lay.nlo, pc.lay.nhi, true};  // (k_chain reports a zero slot on its track rows)
        else if (gv == 0.f && !bound) pc.lay = Lay{1, 1, 1, 1, true};  // a gain of (about) zero answers with silence (gain.rs:160-163)
        return finish_chain(nc, std::move(pc));
    }
    if (!need_out(nc, ch)) return false;
    Entry gp = patch(PATCH_GAIN, 1);
    operand(gp, 0, pgn, gv);
    if (may_zero) {
        out_dynamic(nc, or_silent);
        if (p.out_buf[0].meta) {  // META_COPY, or silent (META_CONST with count 1 and the silent flag) while the bound gain is about zero
            meta_stage(nc.L, META_COPY, p.in_buf[0], ch, p.out_buf[0], ch, 1, 1);
            Entry mp = gp;
            mp.p.param.kind = PATCH_META;
            add_patch(stage(nc.L, S_META), mp, offsetof(MetaInst, mode));
        }
    } else if (gv == 0.f && !bound) {
        out_dynamic(nc, Lay{1, 1, 1, 1, true});
        if (p.out_buf[0].meta) source_meta(nc, 0, 0, 1);
    } else {
        out_like_input(nc);
    }
    StageBuild& s = stage(nc.L, S_GAIN);
    s.gain.push_back(GainInst{p.in_buf[0], p.out_buf[0], gv, ch, BufRef{nullptr, 0, 0}});
    if (bound) add_patch(s, gp, offsetof(GainInst, gain));
    return true;
}

bool Planner::lower_shaper(NodeCtx& nc) {
    Node& n = nc.n; PNode& p = nc.p; const Lay& in0 = nc.in0;
    int ch = p.in_ch[0];
    // A curve bound from device memory (wae_wave_shaper_set_device_curve): whether it maps 0 to 0 is known only once it is bound.  Behind
    // an input that is never silent that answer changes no layout, and the node is planned as a curve that maps 0 to 0.  Otherwise the
    // plan covers both answers (the output gets a layout track of its own), and the bind patches every field the answer decides:
    // ChainInst::shaper_keeps_silence, the MetaInst::mode of the output track (META_COPY / META_SHAPER), ShaperOsInst::rebuild (2 / 1).
    const bool declared = n.device_curve != 0;
    const int curve_n = declared ? (int)n.device_curve : (int)n.table.size();
    const float* curve = declared ? device_curve(n) : n.has_curve ? upload(n.table) : nullptr;
    if (declared && !curve) return false;
    // can_propagate_silence (waveshaper.rs:480-503): the curve maps 0 to 0
    bool keeps_silence = true;
    if (n.has_curve && !declared && !n.table.empty()) {
        const size_t cn = n.table.size();
        keeps_silence = cn % 2 == 1 ? std::fabs(n.table[cn / 2]) < 1e-9f : std::fabs((n.table[cn / 2 - 1] + n.table[cn / 2]) / 2.f) < 1e-9f;
    }
    // a silent input that still produces sound does so on the ONE channel a silent quantum has (waveshaper.rs:395-400)
    auto shaper_lay = [keeps_silence, declared](const Lay& l) {
        if (declared && l.may_silent) return Lay{1, l.hi, 1, l.nhi, true};  // (either answer)
        if (keeps_silence || !l.may_silent) return l;
        return Lay{1, l.hi, 1, l.nhi, false};
    };
    // the output track of a declared curve behind an input that may be silent: k_meta, its mode patched by the bind
    auto declared_meta = [&]() {
        out_dynamic(nc, shaper_lay(in0));
        if (!p.out_buf[0].meta) return;
        meta_stage(nc.L, META_COPY, p.in_buf[0], ch, p.out_buf[0], ch);
        stage(nc.L, S_META).add_entry(curve_patch(n, META_COPY, META_SHAPER), offsetof(MetaInst, mode), offsetof(CurvePatch, dst));
    };
    if (n.oversample && n.has_curve) {  // waveshaper.rs:409-480: up-sample, shape, down-sample
        // input that can fall silent: a curve that maps 0 to 0 makes the node return early WITHOUT feeding its resamplers
        // (frozen state: the kernel then works on the last processed quanta); a curve that does not keeps processing — on the
        // one channel of a silent quantum, which rebuilds the resamplers of a wider node (waveshaper.rs:395-420)
        bool freeze = in0.dyn() && keeps_silence && in0.nlo == in0.nhi && in0.nhi == ch;
        bool as_static = !in0.dyn() || (!keeps_silence && ch == 1 && in0.hi == 1);
        // a declared curve behind a dynamic input always rebuilds: which of freeze / as_static applies depends on the curve.  From zero
        // state rebuild 2 renders what freeze renders (both count only the processed quanta).  Rebuild 1 behind a mono input never
        // changes the count, and differs from as_static in the first quantum only: as_static adds the down-sampled curve(0) of its zero
        // history there, rebuild starts from zero resamplers as the reference does (waveshaper.rs:409-420)
        if (declared) {
            freeze = false;
            as_static = !in0.dyn();
        }
        // every other dynamic input: the count of the processed quanta changes, and the resamplers are rebuilt with it
        const bool rebuild = !freeze && !as_static;
        if (!need_out(nc, ch)) return false;
        if (rebuild && declared && in0.may_silent) {
            declared_meta();
        } else if (freeze || (rebuild && keeps_silence)) {
            out_like_input(nc);
        } else if (rebuild) {  // silent quanta processed: a sounding output with the input's count (one channel when silent)
            out_dynamic(nc, shaper_lay(in0));
            if (p.out_buf[0].meta) meta_stage(nc.L, META_SHAPER, p.in_buf[0], ch, p.out_buf[0], ch);
        }
        const int factor = n.oversample == WAE_OVERSAMPLE_X2 ? 2 : 4;
        auto& filt = os_filters[factor];
        if (!filt.first) {
            const std::vector<float2> fu = resampler_filter_bins(128, 128 * factor, 128);
            const std::vector<float2> fd = resampler_filter_bins(128 * factor, 128, 128);
            filt.first = upload(fu);
            filt.second = upload(fd);
            if (!dry) cudaStreamSynchronize(eng->stream);  // the host vectors go out of scope
        }
        ShaperOsInst so{};
        so.in = p.in_buf[0];
        so.out = p.out_buf[0];
        so.curve = curve;
        so.n = curve_n;
        so.ch = ch;
        so.factor = factor;
        so.f_up = filt.first;
        so.f_dn = filt.second;
        so.hist = alloc<float>((size_t)256 * ch, true, true);
        if (!so.hist || !so.f_up || !so.f_dn) return bail(WAE_OUT_OF_MEMORY, "out of device memory (over-sampled shaper)");
        if (freeze) {
            so.prev = alloc<int32_t>((size_t)(2 * (b->chunk / 128) + 2));
            if (!so.prev) return bail(WAE_OUT_OF_MEMORY, "out of device memory (over-sampled shaper)");
        }
        if (rebuild) {  // (the two words in front carry the resamplers' state across chunks and segments)
            so.rebuild = keeps_silence ? 2 : 1;
            so.prev = alloc<int32_t>((size_t)(2 + 3 * (b->chunk / 128) + 2), true, true);
            if (!so.prev) return bail(WAE_OUT_OF_MEMORY, "out of device memory (over-sampled shaper)");
        }
        StageBuild& os = stage(nc.L, S_SHAPER_OS);
        os.max_ch = std::max(os.max_ch, ch);
        os.shaper_os.push_back(so);
        if (declared && rebuild) os.add_entry(curve_patch(n, 2, 1), offsetof(ShaperOsInst, rebuild), offsetof(CurvePatch, dst));
        return true;
    }
    if (nc.fuse_n) {
        PendingChain pc = open_chain(nc);
        pc.inst.has_shaper = 1;
        pc.inst.curve = curve;
        pc.inst.shaper_n = curve_n;
        pc.inst.shaper_keeps_silence = keeps_silence ? 1 : 0;
        if (declared) pc.add_entry(curve_patch(n, 1, 0), offsetof(ChainInst, shaper_keeps_silence), offsetof(CurvePatch, dst));
        pc.lay = shaper_lay(pc.lay);
        pc.phase = 5;
        return finish_chain(nc, std::move(pc));
    }
    if (!need_out(nc, ch)) return false;
    ShaperInst sh{};
    if (declared && in0.may_silent) {
        declared_meta();
    } else if (in0.dyn() && !keeps_silence && n.has_curve) {
        out_dynamic(nc, shaper_lay(in0));
        if (p.out_buf[0].meta) meta_stage(nc.L, META_SHAPER, p.in_buf[0], ch, p.out_buf[0], ch);
    } else {
        out_like_input(nc);
    }
    sh.in = p.in_buf[0];
    sh.out = p.out_buf[0];
    sh.ch = ch;
    sh.n = curve_n;
    sh.curve = curve;
    stage(nc.L, S_SHAPER).shaper.push_back(sh);
    return true;
}

bool Planner::lower_stereo_panner(NodeCtx& nc) {
    PNode& p = nc.p;
    PRef ppan = param_ref(nc.n.params[0]);
    float pan = ppan.v;
    int ch = p.in_ch[0];
    if (!need_out(nc, 2)) return false;
    // silent in -> silent out, else two channels (stereo_panner.rs:230-235); the kernel picks the mono / stereo law per quantum
    out_dynamic(nc, nc.in0.may_silent ? Lay{1, 2, 2, 2, true} : Lay::fixed(2));
    if (p.out_buf[0].meta) meta_stage(nc.L, META_PAN, p.in_buf[0], ch, p.out_buf[0], 2);
    float x = ch == 1 ? (pan + 1.f) * 0.5f : (pan <= 0.f ? pan + 1.f : pan);  // stereo_panner.rs:247-249,274-276
    float gl, gr;
    hm::stereo_gains(x, gl, gr);
    StageBuild& s = stage(nc.L, S_SPAN);
    s.span.push_back(SPanInst{p.in_buf[0], p.out_buf[0], pan, ch, ppan.dyn ? ppan.track : BufRef{nullptr, 0, 0}});
    s.span_gains.push_back(make_float2(gl, gr));
    if (ppan.bound >= 0) {
        Entry r = patch(PATCH_SPAN, ch);
        operand(r, 0, ppan, pan);
        r.refer(1, T_B, (int32_t)s.records(T_B) - 1, 0, offsetof(ParamPatch, dst2));  // (and its stereo gains)
        add_patch(s, r, offsetof(SPanInst, pan));
    }
    return true;
}

bool Planner::lower_panner(NodeCtx& nc) {
    Node& n = nc.n; PNode& p = nc.p; const Lay& in0 = nc.in0;
    // the 15 spatial params (panner.rs:714-780): 6 of the node, 9 of the AudioListener (graph ids 2..10)
    // Params bound from device memory (source position / orientation, listener pose) are planned with their placeholders: no lowering
    // decision reads a value.  A moving panner takes them raw (PATCH_RAW), a static one gets a spatial entry that re-derives what the
    // values decide (SpatialPatch).
    PRef pr[15];
    bool moving = false, bound = false;
    for (int i = 0; i < 15; i++) {
        pr[i] = param_ref(i < 6 ? n.params[i] : (uint32_t)(2 + i - 6));
        moving = moving || pr[i].dyn;
        bound = bound || pr[i].bound >= 0;
    }
    int ch = p.in_ch[0];
    // (a static HRTF panner with a constant-layout input is lowered to the convolver kernels, which take their own output buffer)
    static const bool hrtf_fft_on = [] { const char* e = getenv("WAE_HRTF_FFT"); return !e || atoi(e) != 0; }();
    const bool hrtf_as_conv = n.panning_model == WAE_PANNING_HRTF && hrtf_fft_on && eng->sphere && !moving && !in0.dyn() && cur_cls != 1 &&
                              seg_start == 0 && seg_end >= lq && (ch == 1 || ch == 2);
    if (!hrtf_as_conv && !need_out(nc, 2)) return false;
    if (hrtf_as_conv) p.out_lay = {Lay::fixed(2)};
    else out_dynamic(nc, in0.may_silent ? Lay{1, 2, 2, 2, true} : Lay::fixed(2));  // panner.rs:698-708
    // (the HRTF panner keeps its own tail budget: its layout track is written by k_hrtf_map)
    if (!hrtf_as_conv && p.out_buf[0].meta && n.panning_model != WAE_PANNING_HRTF) meta_stage(nc.L, META_PAN, p.in_buf[0], ch, p.out_buf[0], 2);
    spatial::PanModel model{};
    model.distance_model = n.distance_model;
    model.ref_distance = n.ref_distance;
    model.max_distance = n.max_distance;
    model.rolloff_factor = n.rolloff_factor;
    model.cone_inner_angle = n.cone_inner_angle;
    model.cone_outer_angle = n.cone_outer_angle;
    model.cone_outer_gain = n.cone_outer_gain;
    SpatialTracks tr{};
    float v[15];
    for (int i = 0; i < 15; i++) {
        v[i] = tr.value[i] = pr[i].v;
        tr.track[i] = pr[i].dyn ? pr[i].track : BufRef{nullptr, 0, 0};
    }
    const spatial::SpatialParams sp0 = spatial::spatial_params(model, v);  // static source and listener
    if (n.panning_model == WAE_PANNING_HRTF) {  // panner.rs:781-830
        HrirAtRate hr;
        if (!hrir_at_rate(hr)) return false;
        if (hrtf_as_conv) return panner_hrtf_conv(nc, sp0, hr, bound ? pr : nullptr, model);
        return panner_hrtf_fir(nc, sp0, hr, moving, tr, model, bound ? pr : nullptr);
    }
    if (moving) {
        PanDynInst d{};
        d.in = p.in_buf[0];
        d.out = p.out_buf[0];
        d.sp = tr;
        d.model = model;
        d.in_ch = ch;
        StageBuild& ds = stage(nc.L, S_PAN_DYN);
        ds.pan_dyn.push_back(d);
        if (bound) raw_spatial_patches(ds, pr, offsetof(PanDynInst, sp));
        return true;
    }
    PanInst pi{};
    pi.in = p.in_buf[0];
    pi.out = p.out_buf[0];
    pi.in_ch = ch;
    pi.azimuth = sp0.azimuth;
    pi.dist_gain = sp0.dist_gain;
    pi.cone_gain = sp0.cone_gain;
    StageBuild& ps = stage(nc.L, S_PAN);
    ps.pan.push_back(pi);
    if (bound) ps.add_entry(spatial_entry(SPATIAL_PAN, pr, model), 0, offsetof(SpatialPatch, dst));
    return true;
}

// the HRIR sphere at the context's rate (panner.rs:46: at least 27 kHz)
bool Planner::hrir_at_rate(HrirAtRate& hr) {
    const HrirSphere* sph = eng->sphere;
    if (!sph) return bail(WAE_UNSUPPORTED, "HRTF panning needs an HRIR sphere: call wae_engine_set_hrir_sphere first");
    uint32_t sr = (uint32_t)g->sample_rate;
    if (sr < 27000) sr = 27000;  // panner.rs:46
    uint32_t taps = sph->taps;
    const float* d_ir = eng->d_sphere_ir;
    const float* h_ir = sph->ir.data();  // [vertex][2][taps] on the host
    if (sr != sph->sample_rate) {  // the crate resamples the responses to the context rate once (wae_hrtf_host.h)
        std::lock_guard<std::mutex> slk(eng->sphere_mu);
        auto it = eng->sphere_rates.find(sr);
        if (it == eng->sphere_rates.end()) {
            const HrirSphere rs = sph->at_rate(sr);
            wae_engine::RateSphere r;
            r.taps = rs.taps;
            if (r.taps < 2) return bail(WAE_UNSUPPORTED, "HRTF panning: the HRIR sphere is too short to be resampled to the context rate");
            if (cudaMalloc(&r.d_ir, rs.ir.size() * sizeof(float)) != cudaSuccess) return bail(WAE_OUT_OF_MEMORY, "out of device memory (resampled HRIR sphere)");
            cudaMemcpy(r.d_ir, rs.ir.data(), rs.ir.size() * sizeof(float), cudaMemcpyHostToDevice);
            r.ir_host = rs.ir;
            it = eng->sphere_rates.emplace(sr, r).first;
        }
        taps = it->second.taps;
        d_ir = it->second.d_ir;
        h_ir = it->second.ir_host.data();  // (map nodes are stable; entries are only dropped with the sphere)
    }
    hr = HrirAtRate{sr, taps, d_ir, h_ir};
    return true;
}

// the three sphere vertices and their weights of a static source and listener, with the distance and cone gains
HrtfSel Planner::static_hrtf_sel(const spatial::SpatialParams& sp0) const {
    float proj[3];
    spatial::projected_source(sp0, proj);
    const float dir[3] = {proj[0], proj[2], proj[1]};  // HrtfState::process swaps y / z (panner.rs:248-252)
    HrtfSel sel{{0, 0, 0}, {0.f, 0.f, 0.f}, sp0.cone_gain * sp0.dist_gain, 0.f};
    eng->sphere->locate(dir, sel.v, sel.w);  // no face: all-zero weights (silence)
    return sel;
}

// A static source heard by a static listener through a constant-layout input is ONE fixed pair of impulse responses:
// out_ear = gain * (h_ear * mono(in)).  The crate evaluates that by FFT overlap-save per 128-frame block (hrtf 0.8.1
// process_samples); here it is handed to the time-batched convolver kernels as a ConvolverNode-shaped problem —
// response = the blended pair with the gain (and the reference's correction of 2 for a two-channel input,
// panner.rs:805-812) folded in; a two-channel input is mixed down to mono by the forward transform's loads; one
// partition, so the product is formed inside the inverse transform — instead of 2 x taps multiply-adds per output
// frame in k_hrtf_fir.  WAE_HRTF_FFT=0: keep the FIR kernel.
// `pr` (source or listener bound from device memory): planned with ceil(taps / WAE_CONV_BLOCK) partitions whatever the placeholder's
// response holds, into spectra of the node's own; a SPATIAL_RESP entry re-derives the triangle, blends the pair into a [2][taps]
// scratch of its own and transforms it on every bind.
bool Planner::panner_hrtf_conv(NodeCtx& nc, const spatial::SpatialParams& sp0, const HrirAtRate& hr, const PRef* pr,
                               const spatial::PanModel& model) {
    const uint32_t taps = hr.taps;
    const int ch = nc.p.in_ch[0];
    PcmBuffer resp;
    if (!resp.allocate(2, taps, false)) return bail(WAE_OUT_OF_MEMORY, "out of host memory (hrtf response)");
    const float corr = ch == 2 ? 2.f : 1.f;  // overall_gain_correction of a two-channel input (panner.rs:805-812)
    resp.sample_rate = (float)hr.sr;
    if (pr) {
        IrSpectra spec;
        const int S = (int)((taps + WAE_CONV_BLOCK - 1) / WAE_CONV_BLOCK);
        if (!bound_panner_spectra(nc.n, S, spec) || !plan_convolver(nc.p, nc.L, nullptr, -1, &resp, &spec)) return false;
        if (dry) return true;
        Entry r = spatial_entry(SPATIAL_RESP, pr, model);
        r.p.spatial.pos = eng->d_sphere_pos;
        r.p.spatial.tri = eng->d_sphere_tri;
        r.p.spatial.n_faces = (int32_t)(eng->sphere->tri.size() / 3);
        r.p.spatial.ir = hr.d_ir;
        r.p.spatial.taps = (int32_t)taps;
        r.p.spatial.correction = corr;
        const size_t sel_floats = sizeof(HrtfSel) / sizeof(float);
        std::lock_guard<std::recursive_mutex> lk(b->mu);  // (groups are planned on worker threads)
        float* scratch = b->dalloc<float>((size_t)2 * taps + sel_floats, true);  // the pair, then the selection
        if (!scratch) return bail(WAE_OUT_OF_MEMORY, "out of device memory (hrtf response)");
        b->asset_bytes += ((size_t)2 * taps + sel_floats) * sizeof(float);
        r.p.spatial.resp = scratch;
        r.p.spatial.dst = scratch + (size_t)2 * taps;
        r.spec = spec.h;
        r.S = S;
        stage(nc.L, S_CONV_FFT).entries.push_back(r);
        return true;
    }
    const HrtfSel sel = static_hrtf_sel(sp0);
    const float* A = hr.h_ir + (size_t)sel.v[0] * 2 * taps;
    const float* B = hr.h_ir + (size_t)sel.v[1] * 2 * taps;
    const float* C = hr.h_ir + (size_t)sel.v[2] * 2 * taps;
    for (uint32_t k = 0; k < taps; k++) {  // (the blend k_hrtf_fir does, same f32 operations)
        const float l = (A[k] * sel.w[0] + B[k] * sel.w[1]) + C[k] * sel.w[2];
        const float r = (A[taps + k] * sel.w[0] + B[taps + k] * sel.w[1]) + C[taps + k] * sel.w[2];
        resp.channels[0].p[k] = corr * (l * sel.gain);
        resp.channels[1].p[k] = corr * (r * sel.gain);
    }
    return plan_convolver(nc.p, nc.L, nullptr, -1, &resp);
}

bool Planner::panner_hrtf_fir(NodeCtx& nc, const spatial::SpatialParams& sp0, const HrirAtRate& hr, bool moving, const SpatialTracks& tr,
                              const spatial::PanModel& model, const PRef* pr) {
    PNode& p = nc.p;
    const HrirSphere* sph = eng->sphere;
    const int ch = p.in_ch[0];
    HrtfInst h{};
    h.in = p.in_buf[0];
    h.out = p.out_buf[0];
    h.in_ch = ch;
    h.L = (int)hr.taps;
    h.sphere_ir = hr.d_ir;
    h.sel = nullptr;
    h.correction = ch == 2 ? 2.f : 1.f;
    h.hist = alloc<float>(hr.taps, true, true);
    if (!h.hist) return bail(WAE_OUT_OF_MEMORY, "out of device memory (hrtf history)");
    if (nc.in0.dyn()) {  // the node stops processing (and freezes) once its tail budget is used up: panner.rs:697-711
        h.dyn = 1;
        h.cmap = alloc<int32_t>((size_t)(b->chunk / 128 + 2));
        h.tail = alloc<int64_t>(1, true, true);
        if (!h.cmap || !h.tail) return bail(WAE_OUT_OF_MEMORY, "out of device memory (hrtf layout)");
    }
    StageBuild& hs = stage(nc.L, S_HRTF);
    if (moving) {
        HrtfSelInst si{};
        si.sp = tr;
        si.model = model;
        si.pos = eng->d_sphere_pos;
        si.tri = eng->d_sphere_tri;
        si.n_faces = (int)(sph->tri.size() / 3);
        si.sel = alloc<HrtfSel>((size_t)(b->chunk / 128 + 1));
        if (!si.sel) return bail(WAE_OUT_OF_MEMORY, "out of device memory (hrtf selection)");
        h.sel = si.sel;
        hs.hrtf_sel.push_back(si);
        if (pr) raw_spatial_patches(hs, pr, offsetof(HrtfSelInst, sp), T_B);
    } else {
        h.static_sel = static_hrtf_sel(sp0);
    }
    hs.hrtf.push_back(h);
    if (pr && !moving) {  // (the sphere operands: the ones a moving panner's HrtfSelInst holds)
        Entry r = spatial_entry(SPATIAL_SEL, pr, model);
        r.p.spatial.pos = eng->d_sphere_pos;
        r.p.spatial.tri = eng->d_sphere_tri;
        r.p.spatial.n_faces = (int32_t)(sph->tri.size() / 3);
        hs.add_entry(r, offsetof(HrtfInst, static_sel), offsetof(SpatialPatch, dst));
    }
    return true;
}

bool Planner::lower_delay_writer(NodeCtx& nc) {
    PNode& p = nc.p;
    p.out_ch = {p.in_ch[0]};
    p.out_buf = {p.in_buf[0]};
    p.out_lay = {nc.in0};
    if (!Orderer::contains(ord.broken, nc.id)) return true;
    // cycle breaker applied (graph.rs:458-466): the hidden writer->reader edge is gone, the reader ran
    // earlier in this quantum from the ring; record this quantum's input now
    delay_ch_seen[{gi, nc.n.delay_peer}] = p.in_ch[0];
    auto it = delay_rings.find({gi, nc.id});
    if (it == delay_rings.end()) return bail(WAE_UNSUPPORTED, "DelayNode writer processed before its reader inside a cycle");
    if (it->second.ch != p.in_ch[0]) {
        if (!dry) return bail(WAE_UNSUPPORTED, "channel layout of a DelayNode in a feedback cycle did not converge");
        return true;  // sizing pass: the hint is corrected and the pass repeated
    }
    DelayInst d{};
    d.in = p.in_buf[0];
    d.ch = it->second.ch;
    d.ring = it->second.ring;
    d.ring_len = it->second.ring_len;
    d.mono_at = it->second.mono_at;
    d.mono_len = it->second.mono_len;
    d.dyn = it->second.mono_at ? 3 : 0;  // inside a cycle the writer runs after the reader: it extends the one-channel track
    stage(nc.L, S_DELAY_WRITE).delay.push_back(d);
    return true;
}

bool Planner::lower_delay_reader(NodeCtx& nc) {
    Node& n = nc.n; PNode& p = nc.p;
    const double sr = (double)g->sample_rate;
    PRef pdl = param_ref(n.params[0]);
    float dt = pdl.v;
    const bool in_cycle = Orderer::contains(ord.broken, n.delay_peer);
    int ch = p.in_ch[0];
    if (in_cycle) {
        ch = 1;
        if (delay_ch_hint) {
            auto it = delay_ch_hint->find({gi, nc.id});
            if (it != delay_ch_hint->end()) ch = it->second;
        }
    }
    if (!need_out(nc, ch)) return false;
    DelayInst d{};
    d.in = p.in_buf[0];
    d.out = p.out_buf[0];
    d.ch = ch;
    d.in_cycle = in_cycle ? 1 : 0;
    if (pdl.dyn) d.delay_track = pdl.track;
    d.sample_rate = g->sample_rate;
    double delay = (double)dt;
    if (in_cycle) delay = std::max(delay, 128. / sr);  // delay.rs:699-703: at least one quantum inside a cycle
    double num_samples = delay * sr;               // delay.rs:706
    double position = 0. - num_samples;            // sample_index 0
    double pf = std::floor(position);
    d.fl = (int64_t)pf;
    d.k = (float)(position - pf);
    uint64_t max_frames = (uint64_t)std::ceil(std::max(n.max_delay_time, 128. / sr) * sr) + 2;
    d.ring_len = next_pow2(max_frames + 128);
    d.ring = alloc<float>((size_t)ch * d.ring_len, true, true);
    if (!d.ring) return bail(WAE_OUT_OF_MEMORY, "out of device memory (delay ring)");
    b->arena_bytes += (size_t)ch * d.ring_len * 4;
    if (ch <= 2) {
        // The reader reports a quantum without any normal sample as silent (delay.rs:654-664) and the ring follows the
        // channel count of the writer's input (:470-488): its output layout is never constant.  (Wider than stereo: the
        // static layout is kept, the re-mix of the ring is not followed.)
        d.dyn = 1;
        d.mono_len = (int32_t)next_pow2((uint64_t)(b->chunk / 128 + 2));
        d.mono_at = alloc<int64_t>((size_t)d.mono_len, true, true);
        if (!d.mono_at) return bail(WAE_OUT_OF_MEMORY, "out of device memory (delay layout track)");
        const Lay wl = in_cycle ? Lay{1, (uint8_t)ch, 1, (uint8_t)ch, true} : nc.in0;
        out_dynamic(nc, Lay{1, (uint8_t)ch, (uint8_t)(wl.dyn() ? 1 : ch), (uint8_t)ch, true});
        d.out = p.out_buf[0];
        if (!in_cycle) stage(nc.L, S_DELAY_MONO).delay.push_back(d);
    }
    stage(nc.L, S_DELAY).delay.push_back(d);
    if (in_cycle) delay_rings[{gi, n.delay_peer}] = DelayRing{d.ring, d.ring_len, ch, d.mono_at, d.mono_len};
    else stage(nc.L, S_DELAY_WRITE).delay.push_back(d);  // acyclic: history is recorded right after the read
    return true;
}

bool Planner::lower_compressor(NodeCtx& nc) {
    PNode& p = nc.p; const Lay& in0 = nc.in0;
    PRef cp[5];
    for (int i = 0; i < 5; i++) cp[i] = param_ref(nc.n.params[i]);
    const float at = cp[0].v, kn = cp[1].v, ra = cp[2].v, re = cp[3].v, th = cp[4].v;
    int ch = p.in_ch[0];
    if (!need_out(nc, ch)) return false;
    CompInst c{};
    c.in = p.in_buf[0];
    c.out = p.out_buf[0];
    c.ch = ch;
    int ring_size = (int)std::ceil(g->sample_rate * 0.006f / 128.f) + 1;  // dynamics_compressor.rs:250-255
    c.delay_frames = (ring_size - 1) * 128;
    // (the layout ring holds the look-ahead's quanta and the one being written: 38 slots at the highest sample rate the ABI takes)
    if (ring_size > COMP_META_RING) return bail(WAE_UNSUPPORTED, "compressor look-ahead longer than its layout ring");
    c.ring_len = next_pow2((uint64_t)c.delay_frames + 128);
    c.ring = alloc<float>((size_t)ch * c.ring_len, true, true);
    c.state = alloc<float>(2, true, true);
    c.meta_ring = alloc<uint8_t>(COMP_META_RING, true, true);
    if (!c.ring || !c.state || !c.meta_ring) return bail(WAE_OUT_OF_MEMORY, "out of device memory (compressor)");
    // the look-ahead ring starts out silent and hands on the layout of the quantum it delays (dynamics_compressor.rs:340-349,452-468)
    out_dynamic(nc, Lay{1, in0.hi, in0.nlo, in0.nhi, true});
    c.out = p.out_buf[0];
    c.threshold = th; c.knee = kn; c.ratio = ra; c.attack = at; c.release = re;
    for (int i = 0; i < 5; i++) c.track[i] = cp[i].dyn ? cp[i].track : BufRef{nullptr, 0, 0};
    c.sample_rate = g->sample_rate;
    c.end = glq;
    // declared reduction read-outs (wae_compressor_set_readouts): a stage of its own, whose records carry them in a parallel table
    const bool readouts = !nc.n.readout_q.empty();
    StageBuild& s = stage(nc.L, S_COMP, readouts ? 1 : 0);
    s.comp.push_back(c);
    if (readouts) {
        float* rows = nullptr;
        if (dry) rows = reinterpret_cast<float*>(dry_addr());
        else {
            auto it = b->comp_readout_outs.find(nc.id);
            if (it != b->comp_readout_outs.end() && it->second.d) rows = it->second.d + it->second.off[gi];
        }
        if (!rows) return bail(WAE_INVALID_STATE, "compressor read-out rows missing");
        std::vector<int64_t> frames(nc.n.readout_q.size());
        for (size_t k = 0; k < frames.size(); k++) frames[k] = (int64_t)nc.n.readout_q[k] * 128;
        const int64_t* d_frames = upload(frames);
        if (!d_frames) return bail(WAE_OUT_OF_MEMORY, "out of device memory (read-out frames)");
        s.comp_ro.push_back(CompReadoutInst{d_frames, rows, (int32_t)frames.size(), 0});
    }
    const size_t offs[5] = {offsetof(CompInst, attack), offsetof(CompInst, knee), offsetof(CompInst, ratio), offsetof(CompInst, release),
                            offsetof(CompInst, threshold)};
    for (int i = 0; i < 5; i++)
        if (cp[i].bound >= 0) {  // (the kernel takes the raw values)
            Entry r = patch(PATCH_RAW, 1);
            operand(r, 0, cp[i], cp[i].v);
            add_patch(s, r, offs[i]);
        }
    if (!dry) {
        std::lock_guard<std::recursive_mutex> lk(b->mu);  // (groups are planned on worker threads)
        bool known = false;
        for (auto& r : b->compressors) known = known || (r.graph == gi && r.node == nc.id);
        if (!known) b->compressors.push_back(wae_batch::CompRec{gi, nc.id, c.state});
    }
    return true;
}

bool Planner::lower_analyser(NodeCtx& nc) {
    Node& n = nc.n; PNode& p = nc.p;
    int ch = p.in_ch[0];
    // pass-through (analyser.rs:267-294): the output IS the input buffer (nobody writes an edge buffer after its
    // producer), only the ring is written
    p.out_ch = {ch};
    p.out_buf = {p.in_buf[0]};
    p.out_lay = {nc.in0};
    AnalyserInst a{};
    a.in = p.in_buf[0];
    a.out = BufRef{nullptr, 0, 0};
    a.ch = ch;
    a.end = glq;
    a.ring = alloc<float>(32768 + 128, true, true);
    if (!a.ring) return bail(WAE_OUT_OF_MEMORY, "out of device memory (analyser ring)");
    stage(nc.L, S_ANALYSER).analyser.push_back(a);
    float* last = alloc<float>(16384, true, true);
    float* db = alloc<float>(16384);
    if (!last || !db) return bail(WAE_OUT_OF_MEMORY, "out of device memory (analyser)");
    const bool freq = (n.readout_kinds & WAE_READOUT_FREQUENCY) != 0;
    if (!dry) {
        std::lock_guard<std::recursive_mutex> lk(b->mu);
        bool known = false;
        for (auto& r : b->analysers) known = known || (r.graph_index == gi && r.node == nc.id);
        if (!known) {
            b->analysers.push_back(AnalyserRec{gi, nc.id, a.ring, n.fft_size, n.smoothing, last, db, false, n.min_db, n.max_db, glq});
            b->analysers.back().end_readout = freq && (int64_t)n.readout_q.back() * 128 == glq;
        }
    }
    algorithmic_bytes += (uint64_t)lq * 4;  // ring write, SURVEY §8(d)
    if (n.readout_kinds) return lower_readouts(nc, a, last, db);
    return true;
}

// The declared read-outs of an analyser (wae_analyser_set_readouts): one record per distinct frequency read-out frame (a read-out on
// the quantum of the one before repeats its row: k_readout_smooth copies it), one per time-domain read-out, and the analyser's
// smoothing walk.  Their rows are the batch's ReadoutOut of (node, kind).
bool Planner::lower_readouts(NodeCtx& nc, const AnalyserInst& a, float* last, float* db) {
    const Node& n = nc.n;
    const std::vector<uint64_t>& q = n.readout_q;
    const int K = (int)q.size();
    std::vector<int64_t> frames(K);
    for (int k = 0; k < K; k++) frames[k] = (int64_t)q[k] * 128;
    auto rows = [&](uint32_t kind) -> float* {
        if (dry) return reinterpret_cast<float*>(dry_addr());
        auto it = b->readout_outs.find({nc.id, kind});
        return it == b->readout_outs.end() || !it->second.d ? nullptr : it->second.d + it->second.off[gi];
    };
    auto byte_rows = [&](uint32_t kind) -> uint8_t* {
        if (!(n.byte_readout_kinds & kind)) return nullptr;
        if (dry) return reinterpret_cast<uint8_t*>(dry_addr());
        auto it = b->byte_readout_outs.find({nc.id, kind});
        return it == b->byte_readout_outs.end() || !it->second.d ? nullptr : it->second.d + it->second.off[gi];
    };
    for (uint32_t kind : {(uint32_t)WAE_READOUT_FREQUENCY, (uint32_t)WAE_READOUT_TIME_DOMAIN}) {
        if (!(n.readout_kinds & kind)) continue;
        float* base = rows(kind);
        uint8_t* bytes = byte_rows(kind);
        if (!base || (!bytes && (n.byte_readout_kinds & kind))) return bail(WAE_INVALID_STATE, "analyser read-out rows missing");
        const bool f = kind == WAE_READOUT_FREQUENCY;
        const uint32_t row = f ? n.fft_size / 2 : n.fft_size;
        StageBuild& sb = stage(nc.L, f ? S_READOUT_FFT : S_READOUT_TIME);
        for (int k = 0; k < K; k++) {
            if (f && k > 0 && frames[k] == frames[k - 1]) continue;
            sb.readout.push_back(ReadoutInst{a.in, a.ring, base + (size_t)k * row, frames[k], a.ch, (int32_t)n.fft_size,
                                             f || !bytes ? nullptr : bytes + (size_t)k * row});
        }
        if (f) {
            const int64_t* d_frames = upload(frames);
            if (!d_frames) return bail(WAE_OUT_OF_MEMORY, "out of device memory (read-out frames)");
            stage(nc.L, S_READOUT_SMOOTH).readout_smooth.push_back(ReadoutSmoothInst{d_frames, base, last, db, K, (int32_t)row, (float)n.smoothing, 0,
                                                                                      bytes, (float)n.min_db, (float)n.max_db});
        }
    }
    return true;
}

bool Planner::lower_merger(NodeCtx& nc) {
    PNode& p = nc.p;
    int k = nc.n.n_inputs;
    if (!need_out(nc, k)) return false;
    {
        // `k` channels as soon as one input is not silent, else silent (channel_merger.rs:160-168)
        bool some_always_on = false, any_dyn = false;
        for (int i = 0; i < k; i++) {
            some_always_on = some_always_on || !p.in_lay[i].may_silent;
            any_dyn = any_dyn || p.in_lay[i].dyn();
        }
        if (any_dyn && !some_always_on) {
            out_dynamic(nc, Lay{1, (uint8_t)k, (uint8_t)k, (uint8_t)k, true});
            if (p.out_buf[0].meta) {
                MetaInst m{};
                m.out = p.out_buf[0];
                m.mode = META_MERGE;
                m.out_ch = k;
                m.count = k;
                m.n_more = k;
                m.more = upload(p.in_buf);
                if (!m.more) return bail(WAE_OUT_OF_MEMORY, "out of device memory (merger inputs)");
                stage(nc.L, S_META).meta.push_back(m);
            }
        }
    }
    for (int i = 0; i < k; i++) stage(nc.L, S_ROUTE).route.push_back(RouteInst{p.in_buf[i], p.out_buf[0], 0, i, 0, 1});
    return true;
}

bool Planner::lower_splitter(NodeCtx& nc) {
    PNode& p = nc.p;
    int k = nc.n.n_outputs;
    p.out_ch.assign(k, 1);
    p.out_buf.resize(k);
    p.out_lay.assign(k, Lay::fixed(1));
    for (int i = 0; i < k; i++) {
        if (i < p.in_ch[0] && nc.in0.dyn()) {  // channel i exists only in some quanta: copy it, zeros elsewhere, own layout track
            p.out_buf[i] = arena_buf(1, true);
            if (!p.out_buf[i].p) return no_arena();
            p.out_lay[i] = Lay{1, 1, 1, 1, true};
            stage(nc.L, S_ROUTE).route.push_back(RouteInst{p.in_buf[0], p.out_buf[i], i, 0, 0, p.in_ch[0]});
            meta_stage(nc.L, META_SPLIT, p.in_buf[0], p.in_ch[0], p.out_buf[i], 1, 0, i);
        } else if (i < p.in_ch[0]) {  // alias channel i of the input
            BufRef r = p.in_buf[0];
            r.p += (size_t)i * r.stride;
            p.out_buf[i] = r;
        } else {
            p.out_buf[i] = arena_buf(1);
            stage(nc.L, S_ROUTE).route.push_back(RouteInst{p.in_buf[0], p.out_buf[i], 0, 0, 1, 0});
        }
    }
    return true;
}

bool Planner::lower_convolver(NodeCtx& nc) {
    Node& n = nc.n;
    // the destination's only input (and this node's only consumer): the inverse transforms write the rendered PCM
    const BufRef* dest = nullptr;
    const BufRef fin = dest_ref();
    if (eng->fuse && cur_cls == 0 && g->length <= 0xffffffffull) {
        int n_out = 0;
        uint32_t to = 0;
        int to_port = -1;
        for (auto& e : ord.edges.at(nc.id))
            if (e.other_index >= 0) n_out++, to = e.other_id, to_port = e.other_index;
        if (n_out == 1 && to_port == 0 && g->nodes.at(to).kind == K_DEST && node_table.at(to).in_edges[0].size() == 1 &&
            computed_channels(g->nodes.at(to).cfg, (n.buffer && n.buffer->channels.size() == 1 && nc.p.in_ch[0] == 1) ? 1 : 2) == (int)g->channels)
            dest = &fin;
    }
    return plan_convolver(nc.p, nc.L, dest, (int64_t)g->length);
}

bool Planner::plan_graph(wae_graph* graph, uint32_t graph_index) {
    g = graph;
    gi = graph_index;
    glq = (int64_t)((g->length + 127) / 128 * 128);
    dry_gi = gi;
    dry_seq = 0;
    ord = Orderer{g};
    ord.run();
    if (!ord.broken.empty()) has_feedback = true;  // feedback through a DelayNode: its levels are replayed quantum by quantum
    // nodes from which a broken DelayWriter is reachable (reverse reachability over the ordered graph's edges, AudioParam ->
    // owner edges included): they have to be rendered quantum by quantum
    std::set<uint32_t> feeds_cycle;
    if (!ord.broken.empty()) {
        std::map<uint32_t, std::vector<uint32_t>> rev;
        for (uint32_t src = 0; src < (uint32_t)ord.edges.v.size(); src++)
            if (ord.edges.has[src])
                for (auto& e : *ord.edges.v[src]) rev[e.other_id].push_back(src);
        std::vector<uint32_t> todo(ord.broken.begin(), ord.broken.end());
        while (!todo.empty()) {
            uint32_t x = todo.back();
            todo.pop_back();
            if (!feeds_cycle.insert(x).second) continue;
            for (uint32_t y : rev[x]) todo.push_back(y);
        }
    }
    // ... and of those, the ones a cycle feeds (descendants of the readers of the broken delays): only they depend on
    // audio that is produced quantum by quantum
    std::set<uint32_t> fed_by_cycle;
    if (!ord.broken.empty()) {
        std::vector<uint32_t> todo;
        for (uint32_t w : ord.broken) todo.push_back(g->nodes.at(w).delay_peer);
        while (!todo.empty()) {
            uint32_t x = todo.back();
            todo.pop_back();
            if (!fed_by_cycle.insert(x).second) continue;
            const std::vector<Edge>* it = ord.edges.find(x);
            if (!it) continue;
            for (auto& e : *it) todo.push_back(e.other_id);
        }
    }
    auto node_class = [&](uint32_t id) {
        if (ord.broken.empty() || !feeds_cycle.count(id)) return ord.broken.empty() ? 0 : 2;
        return fed_by_cycle.count(id) ? 1 : 0;
    };
    NodeTable& pn = node_table;
    pn.reset(g->nodes.empty() ? 0 : g->nodes.max_id());
    for (auto& kv : g->nodes) pn.put(kv.first, &kv.second);
    // Graph::render (graph.rs:500-535): walk the order, append each audio edge to its destination port
    for (uint32_t id : ord.ordered) {
        for (auto& e : ord.edges.at(id)) {
            if (e.other_index < 0) continue;
            PNode* it = pn.find(e.other_id);
            if (!it) continue;
            it->in_edges[e.other_index].push_back(PortRef{id, e.self_index});
        }
    }
    clock = SchedClock(g->sample_rate);
    want_scan_coefs = !dry || plan_digest_wanted();
    pending.clear();
    for (uint32_t id : ord.ordered) {
        Node& n = g->nodes.at(id);
        if (n.kind == K_LISTENER) continue;
        PNode& p = pn.at(id);
        cur_cls = node_class(id);
        key_graph = gi;
        key_node = id;
        key_seq = 0;
        key_salt = n.kind == K_PARAM ? (uint64_t)n.param.events.size() : 0;  // a param whose event list grew restarts its timeline
        if (n.kind == K_PARAM) {
            if (!lower_param(id, n, p)) return false;
            continue;
        }
        NodeCtx nc{id, n, p};
        if (!plan_inputs(nc)) return false;
        bool ok = false;
        switch (n.kind) {
            case K_DEST: ok = lower_dest(nc); break;
            case K_OSC: ok = lower_osc(nc); break;
            case K_CONST: ok = lower_const(nc); break;
            case K_ABSN: ok = lower_absn(nc); break;
            case K_BIQUAD: ok = lower_biquad(nc); break;
            case K_IIR: ok = lower_iir(nc); break;
            case K_GAIN: ok = lower_gain(nc); break;
            case K_SHAPER: ok = lower_shaper(nc); break;
            case K_SPANNER: ok = lower_stereo_panner(nc); break;
            case K_PANNER: ok = lower_panner(nc); break;
            case K_DELAY_W: ok = lower_delay_writer(nc); break;
            case K_DELAY_R: ok = lower_delay_reader(nc); break;
            case K_COMP: ok = lower_compressor(nc); break;
            case K_ANALYSER: ok = lower_analyser(nc); break;
            case K_MERGER: ok = lower_merger(nc); break;
            case K_SPLITTER: ok = lower_splitter(nc); break;
            case K_CONV: ok = lower_convolver(nc); break;
            default: return bail(WAE_UNSUPPORTED, "node kind not lowered to the GPU");
        }
        if (!ok) return false;
    }
    // chains whose single consumer never showed up as an audio input (e.g. it feeds an AudioParam): materialise
    while (!pending.empty())
        if (!materialize(pending.begin()->first)) return false;
    return true;
}

template <typename T>
static void* up(wae_batch* b, const std::vector<T>& v) {
    return (void*)b->dupload(v);
}

// While alive, `g->nodes` is the graph description that is valid at `frame` (the snapshot taken at the first suspend point
// after it, or the live graph when none follows): the planner reads g->nodes without knowing about suspend points.
struct EpochView {
    wae_graph* g;
    size_t e;
    EpochView(wae_graph* g_, int64_t frame) : g(g_), e(0) {
        while (e < g->epochs.size() && (int64_t)g->epochs[e].frame <= frame) e++;
        if (e < g->epochs.size()) std::swap(g->nodes, g->epochs[e].nodes);
    }
    ~EpochView() {
        if (e < g->epochs.size()) std::swap(g->nodes, g->epochs[e].nodes);
    }
    EpochView(const EpochView&) = delete;
    EpochView& operator=(const EpochView&) = delete;
};

// WAE_OPT_BIND_NUMA / WAE_BIND_NUMA=1: restrict the calling thread (and the engine's workers, which inherit the mask) to the CPUs
// next to this engine's GPU (/sys/bus/pci/devices/<bus id>/local_cpulist), so that page-locked staging memory is allocated and
// touched on that socket: on a two-socket host the H2D / D2H copies of eight ranks otherwise share one socket's memory
// controllers and the inter-socket link.
static bool bind_to_device_numa_node(wae_engine* eng) {
    char bus[64] = {0};
    if (cudaDeviceGetPCIBusId(bus, sizeof bus, eng->device) != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    for (char* c = bus; *c; c++) *c = (char)std::tolower((unsigned char)*c);
    std::ifstream f(std::string("/sys/bus/pci/devices/") + bus + "/local_cpulist");
    std::string list;
    if (!f || !std::getline(f, list) || list.empty()) return false;
    cpu_set_t set;
    CPU_ZERO(&set);
    std::stringstream ss(list);
    std::string part;
    int n = 0;
    while (std::getline(ss, part, ',')) {
        int a = 0, b2 = 0;
        if (std::sscanf(part.c_str(), "%d-%d", &a, &b2) == 2) {
            for (int c = a; c <= b2 && c < CPU_SETSIZE; c++, n++) CPU_SET(c, &set);
        } else if (std::sscanf(part.c_str(), "%d", &a) == 1 && a < CPU_SETSIZE) {
            CPU_SET(a, &set);
            n++;
        }
    }
    if (n == 0 || sched_setaffinity(0, sizeof set, &set) != 0) return false;
    eng->numa_cpus = list;
    return true;
}

}  // namespace

extern "C" {

WAE_API wae_status wae_engine_create(int32_t device_ordinal, wae_engine** out) {
    if (!out) return fail(WAE_INVALID_ARGUMENT, "null out pointer");
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0)
        return fail(WAE_NO_DEVICE, std::string("no CUDA device usable (") + cudaGetErrorString(e) + "): this library has no CPU fallback");
    if (device_ordinal < 0 || device_ordinal >= count) return fail(WAE_NO_DEVICE, "device ordinal out of range");
    CUDA_TRY(cudaSetDevice(device_ordinal));
    cudaDeviceProp prop;
    CUDA_TRY(cudaGetDeviceProperties(&prop, device_ordinal));
    if (prop.major != 9 || prop.minor != 0) return fail(WAE_NO_DEVICE, "the kernels are built for sm_90a (H100) only");
    set_num_sms(prop.multiProcessorCount);
    auto* eng = new wae_engine;
    eng->device = device_ordinal;
    CUDA_TRY(cudaStreamCreateWithFlags(&eng->stream, cudaStreamNonBlocking));
    CUDA_TRY(cudaStreamCreateWithFlags(&eng->s_h2d, cudaStreamNonBlocking));
    CUDA_TRY(cudaStreamCreateWithFlags(&eng->s_d2h, cudaStreamNonBlocking));
    if (const char* e = getenv("WAE_BIND_NUMA"))
        if (atoi(e) != 0) bind_to_device_numa_node(eng);
    std::vector<float> sine = hm::sine_table();
    CUDA_TRY(cudaMalloc(&eng->d_sine, sine.size() * sizeof(float)));
    CUDA_TRY(cudaMemcpy(eng->d_sine, sine.data(), sine.size() * sizeof(float), cudaMemcpyHostToDevice));
    upload_twiddles();
    CUDA_TRY(cudaDeviceSynchronize());
    *out = eng;
    return WAE_OK;
}

WAE_API wae_status wae_engine_destroy(wae_engine* eng) {
    if (!eng) return WAE_OK;
    cudaSetDevice(eng->device);
    if (eng->d_sine) cudaFree(eng->d_sine);
    if (eng->d_sphere_ir) cudaFree(eng->d_sphere_ir);
    if (eng->d_sphere_pos) cudaFree(eng->d_sphere_pos);
    if (eng->d_sphere_tri) cudaFree(eng->d_sphere_tri);
    eng->drop_rate_spheres();
    delete eng->sphere;
    delete eng->pool;  // joins the workers
    eng->dev_trim();
    for (int i = 0; i < wae_engine::kStageSlots; i++)
        if (eng->h_stage[i]) cudaFreeHost(eng->h_stage[i]);
    if (eng->h_ring) cudaFreeHost(eng->h_ring);
    if (eng->stream) cudaStreamDestroy(eng->stream);
    if (eng->s_h2d) cudaStreamDestroy(eng->s_h2d);
    if (eng->s_d2h) cudaStreamDestroy(eng->s_d2h);
    delete eng;
    return WAE_OK;
}

// load_hrtf_processor (src/node/panner.rs:39-68): the reference embeds resources/IRC_1003_C.bin; the binding hands the same
// bytes to the engine once.  Batches prepared afterwards may contain PanningModelType::HRTF panners.
WAE_API wae_status wae_engine_set_hrir_sphere(wae_engine* eng, const void* data, uint64_t len) {
    if (!eng) return fail(WAE_INVALID_ARGUMENT, "null engine");
    auto* sp = new HrirSphere();
    std::string err;
    if (!sp->parse(static_cast<const uint8_t*>(data), len, err)) {
        delete sp;
        return fail(WAE_INVALID_ARGUMENT, err.c_str());
    }
    CUDA_TRY(cudaSetDevice(eng->device));
    float* d = nullptr;
    if (cudaMalloc(&d, sp->ir.size() * sizeof(float)) != cudaSuccess) {
        delete sp;
        return fail(WAE_OUT_OF_MEMORY, "out of device memory (HRIR sphere)");
    }
    float* dpos = nullptr;
    uint32_t* dtri = nullptr;
    if (cudaMalloc(&dpos, sp->pos.size() * sizeof(float)) != cudaSuccess || cudaMalloc(&dtri, sp->tri.size() * sizeof(uint32_t)) != cudaSuccess) {
        cudaFree(d);
        if (dpos) cudaFree(dpos);
        delete sp;
        return fail(WAE_OUT_OF_MEMORY, "out of device memory (HRIR sphere)");
    }
    cudaMemcpy(d, sp->ir.data(), sp->ir.size() * sizeof(float), cudaMemcpyHostToDevice);
    cudaMemcpy(dpos, sp->pos.data(), sp->pos.size() * sizeof(float), cudaMemcpyHostToDevice);
    cudaMemcpy(dtri, sp->tri.data(), sp->tri.size() * sizeof(uint32_t), cudaMemcpyHostToDevice);
    CUDA_TRY(cudaStreamSynchronize(eng->stream));  // batches in flight may still read the previous sphere
    if (eng->d_sphere_ir) cudaFree(eng->d_sphere_ir);
    if (eng->d_sphere_pos) cudaFree(eng->d_sphere_pos);
    if (eng->d_sphere_tri) cudaFree(eng->d_sphere_tri);
    eng->drop_rate_spheres();
    eng->d_sphere_pos = dpos;
    eng->d_sphere_tri = dtri;
    delete eng->sphere;
    eng->sphere = sp;
    eng->d_sphere_ir = d;
    eng->sphere_gen++;
    return WAE_OK;
}

// the CUDA stream every kernel of this engine is launched on (for callers that time with their own events)
WAE_API wae_status wae_engine_stream(wae_engine* eng, void** out_stream) {
    *out_stream = (void*)eng->stream;
    return WAE_OK;
}

WAE_API wae_status wae_engine_set_option(wae_engine* eng, uint32_t option, int64_t value) {
    switch (option) {
        case WAE_OPT_CHUNK_FRAMES:
            if (value < 0 || value % 128 != 0) return fail(WAE_INVALID_ARGUMENT, "chunk frames must be a multiple of 128");
            eng->chunk_frames = value;
            return WAE_OK;
        case WAE_OPT_FUSE: eng->fuse = value != 0; return WAE_OK;
        case WAE_OPT_VOICE_SUM: eng->voice_sum = value < 0 ? 0 : (value > 2 ? 2 : (int)value); return WAE_OK;
        case WAE_OPT_SERIAL_FILTERS: eng->serial_filters = value != 0; return WAE_OK;
        case WAE_OPT_PIPELINE_GROUPS:
            if (value < 0 || value > 1024) return fail(WAE_INVALID_ARGUMENT, "pipeline groups must be in [0, 1024]");
            eng->pipeline_groups = (int)value;
            return WAE_OK;
        case WAE_OPT_PARAM_PARALLEL: eng->param_parallel = value > 2 ? 2 : (int)value; return WAE_OK;
        case WAE_OPT_BIND_NUMA:
            if (value != 0 && eng->pool) return fail(WAE_INVALID_STATE, "bind the engine to its NUMA node before its first render (worker threads already run)");
            if (value != 0 && !bind_to_device_numa_node(eng)) return fail(WAE_UNSUPPORTED, "could not read / apply the CPU list of the GPU's NUMA node");
            return WAE_OK;
        case WAE_OPT_HOST_WORKERS:
            if (value < 0 || value > 256) return fail(WAE_INVALID_ARGUMENT, "host workers must be in [0, 256]");
            if (eng->pool) return fail(WAE_INVALID_STATE, "the worker threads already run");
            eng->n_workers = (int)value;
            return WAE_OK;
        case WAE_OPT_CHAIN_TMA: chain_set_tuning(value != 0 ? 1 : 0, -1); return WAE_OK;
        case WAE_OPT_CHAIN_WAVES:
            if (value < 0 || value > 1024) return fail(WAE_INVALID_ARGUMENT, "chain waves must be in [0, 1024]");
            chain_set_tuning(-1, (int)value);
            return WAE_OK;
        case WAE_OPT_CHAIN_PREPASS: chain_set_prepass(value != 0 ? 1 : 0); return WAE_OK;
        default: return fail(WAE_INVALID_ARGUMENT, "unknown option");
    }
}

WAE_API wae_status wae_batch_destroy(wae_batch* b) {
    if (!b) return WAE_OK;
    cudaSetDevice(b->engine->device);
    if (b->engine->stream) {  // (a plan-only batch has no streams)
        cudaStreamSynchronize(b->engine->stream);
        cudaStreamSynchronize(b->engine->s_h2d);
        cudaStreamSynchronize(b->engine->s_d2h);
    }
    for (void* h : b->pinned) cudaFreeHost(h);
    for (auto& g : b->groups) {
        if (g.ev_h2d) cudaEventDestroy(g.ev_h2d);
        if (g.ev_done) cudaEventDestroy(g.ev_done);
    }
    for (void* p : b->allocs) b->engine->dev_release(p);  // kept by the engine for the next batch (wae_engine::dev_alloc)
    if (b->ev0) cudaEventDestroy(b->ev0);
    if (b->ev1) cudaEventDestroy(b->ev1);
    if (b->ev_bind) cudaEventDestroy(b->ev_bind);
    for (auto& bs : b->bind_stages) cudaEventDestroy(bs.ev);  // (the staging memory is in `pinned`)
    for (auto e : b->stage_events) cudaEventDestroy(e);
    delete b;
    return WAE_OK;
}

// Graph::order_nodes as the planner runs it (host only): lets the CPU tests pin the ordering against the reference's tests
WAE_API wae_status wae_graph_render_order(wae_graph* g, wae_node_id* ids, uint32_t cap, uint32_t* n) {
    if (!g || !n || (cap && !ids)) return fail(WAE_INVALID_ARGUMENT, "null argument");
    Orderer o;
    o.g = g;
    o.run();
    *n = (uint32_t)o.ordered.size();
    for (uint32_t i = 0; i < *n && i < cap; i++) ids[i] = o.ordered[i];
    return WAE_OK;
}

// ---- wae_batch_prepare in phases ------------------------------------------------------------------------------------------
// A (prep_begin): validation, graph groups, the sizing pass of the planner (no device memory touched; groups in parallel on the
//   engine's worker threads), chunk size.  B (prep_plan_group): the real plan of ONE group — allocation of its node state / arena,
//   upload of its instance tables — safe to run for several groups at once (shared structures are guarded by wae_batch::mu).
//   C (prep_append_group / prep_finish): the groups' stages joined in group order, statistics.
// wae_batch_prepare runs A, B for every group, C.  The one-shot render (wae_render_batch with a host buffer) runs A, starts the
// H2D copies of the source PCM, and then overlaps B of group k+1.. with the copies and the render of group k.
struct PrepState {
    std::map<std::pair<uint32_t, uint32_t>, int> delay_ch_hint;
    std::unordered_map<uint64_t, Planner::IrSpectra> ir_cache;
    uint64_t algorithmic_bytes = 0;
    std::chrono::steady_clock::time_point t0, t1;
};
Planner::Planner(wae_batch* b_, const wae_batch::Group& grp, PrepState& ps, std::vector<wae_batch::Group::SrcCopy>* sizing_copies)
    : b(b_), eng(b_->engine), delay_ch_hint(&ps.delay_ch_hint), dry(sizing_copies != nullptr), group_graphs((int)(grp.g1 - grp.g0)),
      d_src(dry ? reinterpret_cast<float*>(uintptr_t(256)) : grp.d_src), src_copies(sizing_copies), lq(grp.lq) {
    if (!dry) ir_cache = &ps.ir_cache;
}
struct GroupPlan {  // result of phase B for one group
    std::vector<Stage> stages;
    std::vector<std::pair<size_t, size_t>> seg_ranges;  // per segment: [first, last) into `stages`
    uint64_t algorithmic_bytes = 0;
    int code = WAE_OK;
    std::string error;
    std::vector<Entry> entries;                        // device addresses set (operands of E_PARAM / E_SPATIAL still param ids)
    std::vector<std::pair<size_t, size_t>> out_zero;   // (offset, floats) of the output no stage writes
    int64_t dest_reader = -1;                          // see Planner::dest_reader
};

static int64_t padded_length(const wae_graph* g) { return (int64_t)((g->length + 127) / 128 * 128); }

// the suspend frames of a graph inside its own render
static std::vector<int64_t> graph_cuts(const wae_graph* g) {
    const int64_t lq = padded_length(g);
    std::vector<int64_t> cuts;
    for (auto& ep : g->epochs)
        if ((int64_t)ep.frame > 0 && (int64_t)ep.frame < lq) cuts.push_back((int64_t)ep.frame);
    return cuts;
}

// A group renders every graph to the group's longest padded length; a shorter graph's extra frames are dropped (the destination's
// `limit`) or land in the arena, and the kernels whose state is read after the render stop at the graph's own end.  A group is at most
// 4/3 of its shortest graph long: the shortest graph of a group is at least 3/4 of the longest.
constexpr int64_t kGroupPadNum = 3, kGroupPadDen = 4;
static bool fits_group(int64_t longest, int64_t lq) { return lq * kGroupPadDen >= longest * kGroupPadNum; }

// Graph groups for the H2D / render / D2H pipeline: contiguous runs of graphs with the same suspend frames, the same sample rate and
// lengths within the padding bound (in a batch of one shape only the suspend frames differ), cut further into about n_groups pieces.
static std::vector<wae_batch::Group> form_groups(const wae_engine* eng, wae_graph* const* graphs, uint32_t n_graphs,
                                                  const std::vector<std::vector<int64_t>>& cuts) {
    int n_groups = eng->pipeline_groups;
    if (n_groups == 0) n_groups = n_graphs >= 512 ? 32 : (n_graphs >= 64 ? 8 : 1);  // more groups = shorter fill / drain of the 3-stage pipeline
    if (eng->pipeline_groups == 0 && n_graphs >= 512) {  // (tuning: WAE_AUTO_GROUPS overrides the automatic choice for large batches)
        static const int env_groups = [] { const char* e = getenv("WAE_AUTO_GROUPS"); return e ? atoi(e) : 0; }();
        if (env_groups > 0) n_groups = env_groups;
    }
    n_groups = std::max(1, std::min<int>(n_groups, (int)n_graphs));
    const uint32_t target = (n_graphs + (uint32_t)n_groups - 1) / (uint32_t)n_groups;
    std::vector<wae_batch::Group> groups;
    uint32_t g0 = 0;
    for (uint32_t i = 1; i <= n_graphs; i++)
        if (i == n_graphs || cuts[i] != cuts[g0] || i - g0 >= target || graphs[i]->sample_rate != graphs[g0]->sample_rate ||
            !fits_group(padded_length(graphs[g0]), padded_length(graphs[i]))) {
            wae_batch::Group grp;
            grp.g0 = g0;
            grp.g1 = i;
            for (uint32_t j = g0; j < i; j++) grp.lq = std::max(grp.lq, padded_length(graphs[j]));
            grp.seg_bounds.push_back(0);
            for (int64_t f : cuts[g0]) grp.seg_bounds.push_back(f);
            grp.seg_bounds.push_back(grp.lq);
            groups.push_back(std::move(grp));
            g0 = i;
        }
    return groups;
}

// The batch order of graphs of different shapes: by sample rate, suspend frames, then longest first (the caller's order among equals),
// so that the groups form_groups cuts are contiguous runs.  Empty when all graphs share one shape: that batch keeps the caller's order
// and plans exactly as wae_batch_prepare plans it.
static wae_status many_order(wae_graph* const* graphs, uint32_t n_graphs, std::vector<uint32_t>& order) {
    order.clear();
    if (!graphs || n_graphs == 0) return fail(WAE_INVALID_ARGUMENT, "null / empty batch");
    bool uniform = true;
    for (uint32_t i = 0; i < n_graphs; i++) {
        if (!graphs[i]) return fail(WAE_INVALID_ARGUMENT, "null graph in the batch");
        uniform = uniform && graphs[i]->channels == graphs[0]->channels && graphs[i]->length == graphs[0]->length &&
                  graphs[i]->sample_rate == graphs[0]->sample_rate;
    }
    if (uniform) return WAE_OK;
    std::vector<std::vector<int64_t>> cuts(n_graphs);
    for (uint32_t i = 0; i < n_graphs; i++) cuts[i] = graph_cuts(graphs[i]);
    order.resize(n_graphs);
    for (uint32_t i = 0; i < n_graphs; i++) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](uint32_t x, uint32_t y) {
        if (graphs[x]->sample_rate != graphs[y]->sample_rate) return graphs[x]->sample_rate < graphs[y]->sample_rate;
        if (cuts[x] != cuts[y]) return cuts[x] < cuts[y];
        return padded_length(graphs[x]) > padded_length(graphs[y]);
    });
    return WAE_OK;
}

// `order` != nullptr: the graphs differ in shape and are given in the batch order many_order made (`order` maps it to the caller's)
static wae_status prep_begin(wae_engine* eng, wae_graph* const* graphs, uint32_t n_graphs, wae_plan_info* plan, wae_batch** out_b, PrepState& ps,
                             bool want_d_out, const std::vector<uint32_t>* order = nullptr) {
    if (!eng || !graphs || n_graphs == 0) return fail(WAE_INVALID_ARGUMENT, "null / empty batch");
    if (!plan) CUDA_TRY(cudaSetDevice(eng->device));
    for (uint32_t i = 0; i < n_graphs; i++) {
        if (!graphs[i]) return fail(WAE_INVALID_ARGUMENT, "null graph in the batch");
        if (!order && (graphs[i]->channels != graphs[0]->channels || graphs[i]->length != graphs[0]->length ||
                       graphs[i]->sample_rate != graphs[0]->sample_rate))
            return fail(WAE_INVALID_ARGUMENT, "all graphs of a batch must share number_of_channels, length and sample_rate");
    }
    ps.t0 = std::chrono::steady_clock::now();
    auto* b = new wae_batch;
    b->engine = eng;
    b->s_h2d = eng->s_h2d;
    b->s_d2h = eng->s_d2h;
    b->n_graphs = n_graphs;
    b->channels = graphs[0]->channels;
    b->out_off.assign(n_graphs + 1, 0);
    for (uint32_t i = 0; i < n_graphs; i++) {
        b->length = std::max(b->length, graphs[i]->length);
        b->out_off[i + 1] = b->out_off[i] + (size_t)graphs[i]->channels * graphs[i]->length;
        b->shape.push_back({graphs[i]->channels, graphs[i]->length});
    }
    b->lq = (int64_t)((b->length + 127) / 128 * 128);
    for (uint32_t i = 0; i < n_graphs; i++) b->needed_quanta += (uint64_t)(padded_length(graphs[i]) / 128);
    if (order) {
        b->mixed = true;
        b->order = *order;
        b->pos.assign(n_graphs, 0);
        for (uint32_t i = 0; i < n_graphs; i++) b->pos[b->order[i]] = i;
    }
    bool has_conv = false, has_hrtf = false;
    std::vector<char> graph_has_conv(n_graphs, 0);
    std::vector<std::vector<int64_t>> cuts(n_graphs);  // per graph: its suspend frames inside the render
    for (uint32_t i = 0; i < n_graphs; i++) {
        for (auto& kv : graphs[i]->nodes) {
            if (kv.second.kind == K_CONV && kv.second.buffer) graph_has_conv[i] = 1;
            if (kv.second.kind == K_PANNER && kv.second.panning_model == WAE_PANNING_HRTF) has_hrtf = true;  // (static ones ride the convolver kernels)
        }
        cuts[i] = graph_cuts(graphs[i]);
        for (auto& ep : graphs[i]->epochs)
            for (auto& kv : ep.nodes)
                if (kv.second.kind == K_CONV && kv.second.buffer) graph_has_conv[i] = 1;
        has_conv = has_conv || graph_has_conv[i];
    }
    size_t out_floats = b->out_off[n_graphs];
    if (!plan && want_d_out) {
        b->d_out = b->dalloc<float>(out_floats, true);
        if (!b->d_out) {
            wae_batch_destroy(b);
            return fail(WAE_OUT_OF_MEMORY, "out of device memory (output PCM)");
        }
    }
    b->groups = form_groups(eng, graphs, n_graphs, cuts);
    int n_groups = (int)b->groups.size();
    // the convolver kernels work on whole partitions: a chunk (and so a render segment) has to start on one
    for (auto& grp : b->groups) {
        bool conv = false;
        for (uint32_t i = grp.g0; i < grp.g1; i++) conv = conv || graph_has_conv[i];
        if (!conv) continue;
        for (int64_t f : grp.seg_bounds)
            if (f != grp.lq && f % WAE_CONV_BLOCK != 0) {
                wae_batch_destroy(b);
                return fail(WAE_UNSUPPORTED, "a suspend point that is not a multiple of the convolver partition (8192 frames) in a graph with a ConvolverNode is not lowered to the GPU");
            }
    }
    // Sizing pass (no device memory touched): arena floats per frame of the largest group and the source-PCM slab of
    // every group.  Chunk size: explicit option, else chosen so that a group's arena stays around 1 GiB.  A plan without any
    // arena buffer (fully fused source->...->destination chains) renders the whole length in one launch per group.
    // Convolvers work on whole 8192-frame blocks and prefer long chunks (their spectra ring, not the arena, is the traffic
    // that matters).
    b->chunk = 2048;
    uint64_t fpf = 0;
    bool has_feedback = false;
    std::vector<std::vector<int>> plan_stage_lists;  // plan-only: stage kinds per (group, segment) of the last iteration
    struct SizeOut {
        uint64_t fpf = 0;
        bool has_feedback = false;
        std::map<std::pair<uint32_t, uint32_t>, int> delay_ch_seen;
        std::vector<std::vector<int>> stage_lists;
        uint64_t digest = 1469598103934665603ull, entries_digest = 1469598103934665603ull;
        size_t n_entries = 0;
        int code = WAE_OK;
        std::string error;
    };
    WorkerPool* pool = (!plan && n_groups > 1 && n_graphs >= 64) ? eng->workers() : nullptr;
    bool converged = false;
    for (int iter = 0; iter < 8; iter++) {  // repeated only while the channel layout of in-cycle delays changes
        bool hints_changed = false;
        fpf = 0;
        plan_stage_lists.clear();
        std::vector<SizeOut> so(n_groups);
        // A group without suspend points whose graphs are large is sized by several workers, each with its own dry planner over a
        // contiguous run of the group's graphs: the graphs of a group share nothing in this pass but the running totals — arena floats per
        // frame (summed) and the cursor into the source-PCM slab (the copies are recorded relative to the run and rebased in graph order,
        // which is the order the planning pass walks).  WAE_PLAN_PARALLEL=1 lets wae_batch_plan (no engine, no GPU) size every group
        // both ways and compare — the check of this path in the CPU suite.
        struct RangeOut {
            uint64_t fpf = 0;
            size_t src_floats = 0;
            bool has_feedback = false;
            std::map<std::pair<uint32_t, uint32_t>, int> delay_ch_seen;
            std::vector<wae_batch::Group::SrcCopy> copies;
            std::vector<size_t> graph_base;  // slab cursor before each graph (relative to the run, rebased by the merge)
            Builds builds;                   // kept for the self-check only
            int code = WAE_OK;
            std::string error;
        };
        // `cursor0`: where the run starts in the slab — 0 while that is not known yet (the sizing pass proper: rebased by the merge), the
        // recorded base of graph i0 once it is (the planning pass and the self-check of the merged stage builds)
        auto size_range = [&](int k, uint32_t i0, uint32_t i1, RangeOut& ro, size_t cursor0) {  // single-segment groups only
            Planner sizing(b, b->groups[k], ps, &ro.copies);
            sizing.src_cursor = cursor0;
            sizing.begin_segment(0, b->groups[k].lq);
            for (uint32_t i = i0; i < i1; i++) {
                EpochView view(graphs[i], 0);
                ro.graph_base.push_back(sizing.src_cursor);
                if (!sizing.plan_graph(graphs[i], i)) {
                    ro.code = sizing.error_code;
                    ro.error = sizing.error;
                    return;
                }
            }
            if (plan) ro.builds = std::move(sizing.builds);
            ro.fpf = sizing.arena_floats_per_frame;
            ro.src_floats = sizing.src_cursor - cursor0;
            ro.has_feedback = sizing.has_feedback;
            ro.delay_ch_seen = std::move(sizing.delay_ch_seen);
        };
        // (RangeOut of the whole group) from `parts` runs sized on `wp`; false: a run failed (first failing graph's error in `out`)
        auto size_group_split = [&](int k, WorkerPool* wp, int parts, RangeOut& out, const std::vector<size_t>* known_base = nullptr) {
            const uint32_t g0 = b->groups[k].g0, n = b->groups[k].g1 - g0;
            std::vector<RangeOut> ro((size_t)parts);
            auto run = [&](int t) {
                const uint32_t i0 = (uint32_t)((uint64_t)n * t / parts), i1 = (uint32_t)((uint64_t)n * (t + 1) / parts);
                size_range(k, g0 + i0, g0 + i1, ro[t], known_base ? (*known_base)[i0] : 0);
            };
            if (wp) wp->parallel_for(parts, run);
            else
                for (int t = 0; t < parts; t++) run(t);
            for (auto& r : ro) {
                if (r.code != WAE_OK) {
                    out.code = r.code;
                    out.error = r.error;
                    return false;
                }
                const size_t rebase = known_base ? 0 : out.src_floats;
                for (auto& c : r.copies) out.copies.push_back(wae_batch::Group::SrcCopy{c.buf, c.offset + rebase, c.floats, c.graph, c.node});
                for (size_t gb : r.graph_base) out.graph_base.push_back(gb + rebase);
                if (plan) merge_builds(out.builds, r.builds);
                out.fpf += r.fpf;
                out.src_floats += r.src_floats;
                out.has_feedback = out.has_feedback || r.has_feedback;
                for (auto& kv : r.delay_ch_seen) out.delay_ch_seen[kv.first] = kv.second;
            }
            return true;
        };
        auto group_nodes = [&](int k) {
            size_t nn = 0;
            for (uint32_t i = b->groups[k].g0; i < b->groups[k].g1; i++) nn += graphs[i]->nodes.size();
            return nn;
        };
        static const bool check_split = [] { const char* e = getenv("WAE_PLAN_PARALLEL"); return e && atoi(e) != 0; }();
        auto size_group = [&](int k) {
            const uint32_t n_in_group = b->groups[k].g1 - b->groups[k].g0;
            const bool one_segment = b->groups[k].seg_bounds.size() == 2;
            // groups are sized one after the other on this thread (no group-level pool): its workers are free for the runs of a group
            if (!plan && !pool && one_segment && n_in_group >= 2 && group_nodes(k) >= 4096) {
                WorkerPool* wp = eng->workers();
                RangeOut out;
                if (!size_group_split(k, wp, (int)std::min<uint32_t>(n_in_group, (uint32_t)wp->size()), out)) {
                    so[k].code = out.code;
                    so[k].error = out.error;
                    return;
                }
                b->groups[k].src_copies = std::move(out.copies);
                b->groups[k].graph_src_base = std::move(out.graph_base);
                b->groups[k].src_floats = out.src_floats;
                so[k].fpf = out.fpf;
                so[k].has_feedback = out.has_feedback;
                so[k].delay_ch_seen = std::move(out.delay_ch_seen);
                return;
            }
            b->groups[k].src_copies.clear();
            b->groups[k].graph_src_base.clear();
            Planner sizing(b, b->groups[k], ps, &b->groups[k].src_copies);
            const std::vector<int64_t>& bounds = b->groups[k].seg_bounds;
            uint64_t serial_digest = 0, serial_entries = 0;
            size_t unused = 0;
            for (size_t sg = 0; sg + 1 < bounds.size(); sg++) {
                sizing.begin_segment(bounds[sg], bounds[sg + 1]);
                for (uint32_t i = b->groups[k].g0; i < b->groups[k].g1; i++) {
                    EpochView view(graphs[i], bounds[sg]);
                    if (one_segment) b->groups[k].graph_src_base.push_back(sizing.src_cursor);
                    if (!sizing.plan_graph(graphs[i], i)) {
                        so[k].code = sizing.error_code;
                        so[k].error = sizing.error;
                        return;
                    }
                }
                so[k].fpf = std::max(so[k].fpf, sizing.arena_floats_per_frame);
                if (plan) {  // the stages (= kernel launches per chunk) this segment of this group lowers to
                    std::vector<int> kinds;
                    for (auto& kv : sizing.builds) kinds.push_back(kv.second.kind);
                    so[k].stage_lists.push_back(std::move(kinds));
                    if (plan_digest_wanted()) {
                        so[k].digest = digest_builds(sizing.builds, so[k].digest);
                        so[k].entries_digest = digest_entries(sizing.builds, so[k].entries_digest, so[k].n_entries);
                    }
                    if (check_split && one_segment) {
                        serial_digest = digest_builds(sizing.builds, 1469598103934665603ull);
                        serial_entries = digest_entries(sizing.builds, 1469598103934665603ull, unused);
                    }
                }
            }
            b->groups[k].src_floats = sizing.src_cursor;
            so[k].has_feedback = sizing.has_feedback;
            so[k].delay_ch_seen = std::move(sizing.delay_ch_seen);
            if (plan && check_split && one_segment && n_in_group >= 2) {  // the split sizing of the same group must say the same
                RangeOut out;
                // (WAE_PLAN_PARALLEL=2: the runs on real worker threads, as the one-shot render sizes them — for the sanitizers)
                static const bool threaded = [] { const char* e = getenv("WAE_PLAN_PARALLEL"); return e && atoi(e) >= 2; }();
                std::unique_ptr<WorkerPool> tmp_pool(threaded ? new WorkerPool(3, 0) : nullptr);
                const bool ok = size_group_split(k, tmp_pool.get(), (int)std::min<uint32_t>(n_in_group, 3u), out);
                bool same = ok && out.fpf == so[k].fpf && out.src_floats == b->groups[k].src_floats && out.has_feedback == so[k].has_feedback &&
                            out.delay_ch_seen == so[k].delay_ch_seen && out.copies.size() == b->groups[k].src_copies.size() &&
                            out.graph_base == b->groups[k].graph_src_base;
                if (same) {  // with the runs started at their place in the slab the merged stage builds ARE the serial ones
                    RangeOut abs_out;
                    same = size_group_split(k, nullptr, (int)std::min<uint32_t>(n_in_group, 3u), abs_out, &b->groups[k].graph_src_base) &&
                           abs_out.graph_base == b->groups[k].graph_src_base && digest_builds(abs_out.builds, 1469598103934665603ull) == serial_digest &&
                           digest_entries(abs_out.builds, 1469598103934665603ull, unused) == serial_entries;
                }
                for (size_t c = 0; same && c < out.copies.size(); c++) {
                    const auto& x = out.copies[c];
                    const auto& y = b->groups[k].src_copies[c];
                    same = x.buf == y.buf && x.offset == y.offset && x.floats == y.floats;
                }
                if (!same) {
                    so[k].code = WAE_INVALID_STATE;
                    so[k].error = "internal: the split sizing pass disagrees with the serial one";
                }
            }
        };
        if (pool) pool->parallel_for(n_groups, size_group);
        else
            for (int k = 0; k < n_groups; k++) size_group(k);
        for (int k = 0; k < n_groups; k++) {
            if (so[k].code != WAE_OK) {
                int code = so[k].code;
                std::string msg = so[k].error;
                wae_batch_destroy(b);
                return fail(code, msg);
            }
            fpf = std::max(fpf, so[k].fpf);
            has_feedback = has_feedback || so[k].has_feedback;
            for (auto& l : so[k].stage_lists) plan_stage_lists.push_back(std::move(l));
            if (plan && plan_digest_wanted()) {
                std::fprintf(stderr, "[wae plan digest] group %d fpf %llu src %zu: %016llx\n", k, (unsigned long long)so[k].fpf, b->groups[k].src_floats, (unsigned long long)so[k].digest);
                std::fprintf(stderr, "[wae plan entries] group %d entries %zu: %016llx\n", k, so[k].n_entries, (unsigned long long)so[k].entries_digest);
            }
            for (auto& kv : so[k].delay_ch_seen) {
                auto it = ps.delay_ch_hint.find(kv.first);
                int cur = it == ps.delay_ch_hint.end() ? 1 : it->second;
                if (cur != kv.second) {
                    ps.delay_ch_hint[kv.first] = kv.second;
                    hints_changed = true;
                }
            }
        }
        if (!hints_changed) {
            converged = true;
            break;
        }
    }
    if (!converged) {
        wae_batch_destroy(b);
        return fail(WAE_UNSUPPORTED, "the channel layout of DelayNodes inside feedback cycles did not settle (graph not lowered to the GPU)");
    }
    ps.t1 = std::chrono::steady_clock::now();  // sizing pass done
    b->arena_bytes = 0;
    b->asset_bytes = 0;
    int64_t chunk = eng->chunk_frames;
    if (chunk == 0) {
        if (fpf == 0) {
            chunk = b->lq;
        } else {
            chunk = (int64_t)(1024.0 * 1024 * 1024 / (4.0 * (double)fpf));  // arena budget 1 GiB
            chunk = std::max<int64_t>(8192, std::min<int64_t>(chunk, 1 << 20));  // >= 8192: keeps per-chunk launches and serial tails amortised
            chunk = chunk / 2048 * 2048;
        }
        if (has_conv || has_hrtf) chunk = std::max<int64_t>(chunk, 8 * WAE_CONV_BLOCK);  // k_conv_mac tiles 8 output blocks
    }
    // feedback through a DelayNode: the stages up to the cycle are replayed one render quantum at a time INSIDE each chunk
    // (run_group), so the chunk size does not depend on it
    (void)has_feedback;
    if (has_conv || has_hrtf) chunk = (chunk + WAE_CONV_BLOCK - 1) / WAE_CONV_BLOCK * WAE_CONV_BLOCK;
    if (chunk > b->lq) chunk = (has_conv || has_hrtf) ? (b->lq + WAE_CONV_BLOCK - 1) / WAE_CONV_BLOCK * WAE_CONV_BLOCK : b->lq;
    b->chunk = chunk;
    if (plan) {
        std::memset(plan, 0, sizeof *plan);
        plan->groups = (uint32_t)n_groups;
        plan->chunk_frames = (uint64_t)chunk;
        plan->chunks = (uint64_t)((b->lq + chunk - 1) / chunk);
        plan->arena_floats_per_frame = fpf;
        plan->has_feedback = has_feedback ? 1u : 0u;
        uint32_t per_kind[S_KINDS] = {0};
        for (auto& grp : b->groups) {
            plan->source_floats += grp.src_floats;
            plan->segments += (uint32_t)grp.seg_bounds.size() - 1;
        }
        for (auto& kinds : plan_stage_lists) {
            plan->stages += (uint32_t)kinds.size();
            for (int k : kinds) per_kind[k]++;
        }
        std::string txt;  // "k_chain x 1, k_mix x 1": stages by kernel, summed over groups and segments
        for (int k = 0; k < S_KINDS; k++)
            if (per_kind[k]) txt += (txt.empty() ? "" : ", ") + std::string(kStageNames[k]) + " x " + std::to_string(per_kind[k]);
        std::snprintf(plan->stage_kinds, sizeof plan->stage_kinds, "%s", txt.c_str());
        delete b;  // nothing was allocated on the device
        *out_b = nullptr;
        return WAE_OK;
    }
    for (auto& grp : b->groups) {
        if (cudaEventCreateWithFlags(&grp.ev_h2d, cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&grp.ev_done, cudaEventDisableTiming) != cudaSuccess) {
            const std::string msg = std::string("prepare: cudaEventCreate: ") + cudaGetErrorString(cudaGetLastError());
            wae_batch_destroy(b);
            return fail(WAE_CUDA_ERROR, msg);
        }
        if (grp.src_floats) {
            // (not zeroed: every float of the slab is covered by a source copy, channel paddings included)
            grp.d_src = b->dalloc<float>(grp.src_floats, false);
            if (!grp.d_src) {
                wae_batch_destroy(b);
                return fail(WAE_OUT_OF_MEMORY, "out of device memory (source PCM slab)");
            }
        }
    }
    *out_b = b;
    return WAE_OK;
}

// phase B: plans group k (all its segments) and uploads its tables.  Thread-safe against other groups of the same batch.
static void prep_plan_group(wae_batch* b, wae_graph* const* graphs, int k, PrepState& ps, GroupPlan& gp) {
    wae_engine* eng = b->engine;
    wae_batch::Group& grp = b->groups[k];
    Planner pl(b, grp, ps, nullptr);  // (the source copies are recorded by the sizing pass)
    auto oom = [&](const char* what) {
        gp.code = WAE_OUT_OF_MEMORY;
        gp.error = std::string("out of device memory (") + what + ")";
    };
    // The only group of a batch of few, large graphs, no suspend points (north_star: 8 graphs of 3000 nodes): planned by several workers,
    // one Planner per contiguous run of graphs starting at the slab cursor the sizing pass recorded for its first graph; the runs' stage
    // builds are merged in graph order (merge_builds) — the tables a single planner would have built (wae_batch_plan checks that on the
    // CPU under WAE_PLAN_PARALLEL=1).  This function may itself run on a worker (one-shot render), which then waits for the others: only
    // with one group in the batch, and never with fewer than two workers left.
    int split_parts = 0;
    {
        static const bool split_on = [] { const char* e = getenv("WAE_PLAN_SPLIT"); return !e || atoi(e) != 0; }();
        const uint32_t n_in_group = grp.g1 - grp.g0;
        size_t nn = 0;
        for (uint32_t i = grp.g0; i < grp.g1; i++) nn += graphs[i]->nodes.size();
        if (split_on && b->groups.size() == 1 && grp.seg_bounds.size() == 2 && n_in_group >= 2 && nn >= 4096 && grp.graph_src_base.size() == n_in_group) {
            const int free_workers = eng->workers()->size() - 1;
            if (free_workers >= 2) split_parts = (int)std::min<uint32_t>(n_in_group, (uint32_t)free_workers);
        }
    }
    for (int sg = 0; sg + 1 < (int)grp.seg_bounds.size(); sg++) {
        pl.begin_segment(grp.seg_bounds[sg], grp.seg_bounds[sg + 1]);
        const uint64_t alg_before = pl.algorithmic_bytes;
        if (split_parts >= 2) {
            struct Run {
                Builds builds;
                uint64_t algorithmic_bytes = 0;
                int64_t dest_reader = -1;
                int code = WAE_OK;
                std::string error;
            };
            std::vector<Run> runs((size_t)split_parts);
            const uint32_t n = grp.g1 - grp.g0;
            eng->workers()->parallel_for(split_parts, [&](int t) {
                const uint32_t i0 = (uint32_t)((uint64_t)n * t / split_parts), i1 = (uint32_t)((uint64_t)n * (t + 1) / split_parts);
                Planner rp(b, grp, ps, nullptr);
                rp.src_cursor = grp.graph_src_base[i0];
                rp.begin_segment(grp.seg_bounds[sg], grp.seg_bounds[sg + 1]);
                for (uint32_t i = grp.g0 + i0; i < grp.g0 + i1; i++) {
                    EpochView view(graphs[i], grp.seg_bounds[sg]);
                    if (!rp.plan_graph(graphs[i], i)) {
                        runs[t].code = rp.error_code;
                        runs[t].error = rp.error;
                        return;
                    }
                }
                runs[t].builds = std::move(rp.builds);
                runs[t].algorithmic_bytes = rp.algorithmic_bytes;
                runs[t].dest_reader = rp.dest_reader;
            });
            for (auto& r : runs) {
                if (r.code != WAE_OK) {
                    gp.code = r.code;
                    gp.error = r.error;
                    return;
                }
                merge_builds(pl.builds, r.builds);
                pl.algorithmic_bytes += r.algorithmic_bytes;
                if (pl.dest_reader < 0) pl.dest_reader = r.dest_reader;
            }
        } else
        for (uint32_t i = grp.g0; i < grp.g1; i++) {
            EpochView view(graphs[i], grp.seg_bounds[sg]);
            if (!pl.plan_graph(graphs[i], i)) {
                gp.code = pl.error_code;
                gp.error = pl.error;
                return;
            }
        }
        // the per-node byte counts assume the whole render: scale to this segment's share of it
        gp.algorithmic_bytes += (uint64_t)((double)(pl.algorithmic_bytes - alg_before) * (double)(pl.seg_end - pl.seg_start) / (double)grp.lq);
        // materialise the segment's stages in (class, level, kind) order
        const size_t seg_stage0 = gp.stages.size();
        void* last_conv_inputs = nullptr;
        for (auto& kv : pl.builds) {
            StageBuild& s = kv.second;
            Stage st;
            st.seg = sg;
            st.cls = s.cls;
            st.kind = s.kind;
            st.variant = s.variant;
            st.group = k;
            st.max_ch = s.max_ch;
            switch (s.kind) {
                case S_MIX: {
                    for (auto& m : s.mix) {  // classify: vector fast path of k_mix
                        bool simple = true, all_mono = m.n_edges > 0;
                        for (int e = 0; e < m.n_edges; e++) {
                            const MixEdge& ed = s.mix_edges[m.edge_offset + e];
                            bool same = ed.src_ch == m.out_ch;
                            bool dup = ed.src_ch == 1 && m.out_ch == 2 && m.interp == WAE_INTERPRETATION_SPEAKERS;
                            if (!(same || dup)) simple = false;
                            if (ed.src_ch != 1) all_mono = false;
                            // sources must allow 16-byte loads: arena buffers do; asset / output aliases may not
                            if (ed.src.absolute || (ed.src.stride & 3) != 0 || (reinterpret_cast<uintptr_t>(ed.src.p) & 15) != 0) simple = false;
                        }
                        m.simple = simple ? 1 : 0;
                        m.all_mono = (simple && all_mono && (m.out_ch == 1 || (m.out_ch == 2 && m.interp == WAE_INTERPRETATION_SPEAKERS))) ? 1 : 0;
                    }
                    st.n = (int)s.mix.size(); st.d_a = up(b, s.mix); st.d_b = up(b, s.mix_edges);
                    for (auto& m : s.mix) st.n_b = std::max(st.n_b, (int)m.n_edges);  // widest port: picks the mixer kernel
                    break;
                }
                case S_MIX_DYN: {
                    for (auto& m : s.mix_dyn) {  // classify: the four-frames-per-thread path of k_mix_dyn
                        bool ok = m.out_ch <= 2;
                        for (int e = 0; e < m.n_edges && ok; e++) {
                            const MixEdge& ed = s.mix_edges[m.edge_offset + e];
                            if (ed.src_ch > 2 || ed.src.absolute || (ed.src.stride & 3) != 0 || (reinterpret_cast<uintptr_t>(ed.src.p) & 15) != 0) ok = false;
                        }
                        m.stereo4 = ok ? 1 : 0;
                    }
                    st.n = (int)s.mix_dyn.size(); st.d_a = up(b, s.mix_dyn); st.d_b = up(b, s.mix_edges);
                    break;
                }
                case S_META: st.n = (int)s.meta.size(); st.d_a = up(b, s.meta); break;
                case S_OSC: st.n = (int)s.osc.size(); st.d_a = up(b, s.osc); break;
                case S_CONST: st.n = (int)s.cst.size(); st.d_a = up(b, s.cst); break;
                case S_ABSN: st.n = (int)s.absn.size(); st.d_a = up(b, s.absn); break;
                case S_BIQUAD: st.n = (int)s.biquad.size(); st.d_a = up(b, s.biquad); break;
                case S_CHAIN: {
                    st.n = (int)s.chain.size(); st.d_a = up(b, s.chain); st.d_b = up(b, s.scan_coef);
                    const int nb = (s.variant % 6) / 2;
                    int slabs = 1, tps = 1;
                    int pre_log2 = -1;
                    if (nb > 0) chain_plan_slabs(st.n, st.max_ch, (int)std::min<int64_t>(b->chunk, pl.seg_end - pl.seg_start), nb, &slabs, &tps, &pre_log2);
                    if (slabs > 1) {  // time slabs of filtered chains hand their state over through device memory
                        const size_t slots = (size_t)st.n * st.max_ch * slabs;
                        st.chain.slab_stride = slabs;
                        st.chain.ticket = b->dalloc<unsigned>(1, true);
                        st.chain.flags = b->dalloc<unsigned>(slots, true);
                        st.chain.handoff = b->dalloc<double>(slots * CHAIN_MAX_BIQUADS * 4);
                        if (!st.chain.ticket || !st.chain.flags || !st.chain.handoff) return oom("chain hand-off");
                    }
                    break;
                }
                case S_VSUM: {
                    st.n = (int)s.vgroups.size(); st.d_a = up(b, s.chain); st.d_b = up(b, s.scan_coef); st.d_c = up(b, s.vgroups);
                    const int64_t nf_max = std::min<int64_t>(b->chunk, pl.seg_end - pl.seg_start);
                    const int tiles = (int)((nf_max + 2047) / 2048);
                    st.chain.slab_stride = tiles;  // progress counters per group
                    st.chain.ticket = b->dalloc<unsigned>(1, true);
                    st.chain.flags = b->dalloc<unsigned>((size_t)st.n * tiles, true);
                    st.chain.handoff = b->dalloc<double>(s.chain.size() * 2 * 4);
                    if (!st.chain.ticket || !st.chain.flags || !st.chain.handoff) return oom("voice-sum hand-off");
                    break;
                }
                case S_PARAM: st.n = (int)s.param.size(); st.d_a = up(b, s.param); break;
                case S_OSC_AR: st.n = (int)s.osc_ar.size(); st.d_a = up(b, s.osc_ar); break;
                case S_BIQUAD_AR: st.n = (int)s.biquad_ar.size(); st.d_a = up(b, s.biquad_ar); break;
                case S_ABSN_SLOW: st.n = (int)s.absn_slow.size(); st.d_a = up(b, s.absn_slow); break;
                case S_IIR: st.n = (int)s.iir.size(); st.d_a = up(b, s.iir); break;
                case S_GAIN: st.n = (int)s.gain.size(); st.d_a = up(b, s.gain); break;
                case S_SHAPER: st.n = (int)s.shaper.size(); st.d_a = up(b, s.shaper); break;
                case S_SPAN: st.n = (int)s.span.size(); st.d_a = up(b, s.span); st.d_b = up(b, s.span_gains); break;
                case S_PAN: st.n = (int)s.pan.size(); st.d_a = up(b, s.pan); break;
                case S_HRTF: st.n = (int)s.hrtf.size(); st.d_a = up(b, s.hrtf); st.max_ch = s.hrtf.empty() ? 0 : s.hrtf[0].L;
                    st.n_b = (int)s.hrtf_sel.size(); st.d_b = up(b, s.hrtf_sel); break;
                case S_PAN_DYN: st.n = (int)s.pan_dyn.size(); st.d_a = up(b, s.pan_dyn); break;
                case S_ABSN_SERIAL: st.n = (int)s.absn_serial.size(); st.d_a = up(b, s.absn_serial); break;
                case S_ABSN_BOUND: st.n = (int)s.absn_bound.size(); st.d_a = up(b, s.absn_bound); break;
                case S_SHAPER_OS: st.n = (int)s.shaper_os.size(); st.d_a = up(b, s.shaper_os); break;
                case S_ROUTE: st.n = (int)s.route.size(); st.d_a = up(b, s.route); break;
                case S_DELAY_MONO:
                case S_DELAY:
                case S_DELAY_WRITE: st.n = (int)s.delay.size(); st.d_a = up(b, s.delay); break;
                case S_COMP:  // (d_b stays null without read-outs: undeclared compressors run k_compressor<false>)
                    st.n = (int)s.comp.size(); st.d_a = up(b, s.comp);
                    if (!s.comp_ro.empty() && !(st.d_b = up(b, s.comp_ro))) return oom("compressor read-outs");
                    break;
                case S_ANALYSER: st.n = (int)s.analyser.size(); st.d_a = up(b, s.analyser); break;
                case S_READOUT_FFT:
                case S_READOUT_TIME: {
                    std::vector<ReadoutInst> r = s.readout;
                    std::stable_sort(r.begin(), r.end(), [](const ReadoutInst& x, const ReadoutInst& y) { return x.frame < y.frame; });
                    st.n = (int)r.size();
                    st.d_a = up(b, r);
                    for (const ReadoutInst& x : r) {
                        st.frames.push_back(x.frame);
                        st.n_b = std::max(st.n_b, (int)x.fft_size);
                    }
                    break;
                }
                case S_READOUT_SMOOTH:
                    st.n = (int)s.readout_smooth.size();
                    st.d_a = up(b, s.readout_smooth);
                    for (const ReadoutSmoothInst& x : s.readout_smooth) st.n_b = std::max(st.n_b, (int)x.bins);
                    break;
                case S_CONV_FFT: st.n = (int)s.conv_in.size(); st.d_a = up(b, s.conv_in); last_conv_inputs = st.d_a; break;
                case S_CONV_CMP: st.n = (int)s.conv_cmp.size(); st.d_a = up(b, s.conv_cmp); break;
                case S_CONV_MAC:
                case S_CONV_MAC_ACC:
                    st.n = (int)s.conv_path.size();
                    st.d_a = up(b, s.conv_path);
                    st.d_b = last_conv_inputs;  // conv-input table of the same level (kinds are ordered FFT < MAC < MAC_ACC)
                    break;
            }
            if (st.n > 0) {
                if (!st.d_a) return oom("stage tables");
                gp.stages.push_back(st);
            }
            if (st.n > 0) {  // bind entries: the device addresses of the record fields their references name (this pass builds the
                             // scan constants of every chain biquad, which the T_B references of its entries name)
                char* const tables[4] = {nullptr, static_cast<char*>(st.d_a), static_cast<char*>(st.d_b), static_cast<char*>(st.d_c)};
                for (Entry e : s.entries) {
                    for (const FieldRef& r : e.ref)
                        if (r.table != T_NONE) {
                            char* const at = tables[r.table] + (size_t)r.rec * s.record_bytes(r.table) + r.off;
                            std::memcpy(reinterpret_cast<char*>(&e.p) + r.field, &at, sizeof at);
                        }
                    gp.entries.push_back(e);
                }
            }
        }
        // the frames of this segment of the graphs no stage writes: zeroed by every run into a bound output (the batch's own buffer
        // keeps the zeros it was allocated with)
        std::vector<char> written(grp.g1 - grp.g0, 0);
        for (auto& kv : pl.builds)
            for (const Entry& e : kv.second.entries)
                if (e.kind == E_OUT) written[e.graph - grp.g0] = 1;
        for (uint32_t j = grp.g0; j < grp.g1; j++) {
            const int64_t len = (int64_t)b->shape[j].second, f1 = std::min<int64_t>(pl.seg_end, len);
            if (written[j - grp.g0] || f1 <= pl.seg_start) continue;
            for (uint32_t c = 0; c < b->shape[j].first; c++)
                gp.out_zero.push_back({b->out_off[j] + (size_t)c * (size_t)len + (size_t)pl.seg_start, (size_t)(f1 - pl.seg_start)});
        }
        gp.seg_ranges.push_back({seg_stage0, gp.stages.size()});
    }  // segments
    gp.dest_reader = pl.dest_reader;
    b->flush_uploads();  // the group's tables, before anything of it is launched
}

static void prep_append_group(wae_batch* b, int k, PrepState& ps, GroupPlan& gp) {
    wae_batch::Group& grp = b->groups[k];
    grp.stage0 = b->stages.size();
    for (auto& r : gp.seg_ranges) grp.seg_stages.push_back({grp.stage0 + r.first, grp.stage0 + r.second});
    for (auto& st : gp.stages) b->stages.push_back(st);
    grp.stage1 = b->stages.size();
    grp.out_zero = std::move(gp.out_zero);
    if (b->dest_reader < 0 && gp.dest_reader >= 0) b->dest_reader = gp.dest_reader;
    ps.algorithmic_bytes += gp.algorithmic_bytes;
}

// H2D of a group's source PCM, one copy per AudioBufferSourceNode, straight from the buffers the graphs own
// (device inputs have no host PCM: their slots are written by wae_batch_bind_sources only)
static wae_status enqueue_source_copies(wae_batch* b, wae_batch::Group& grp, cudaStream_t s) {
    for (auto& sc : grp.src_copies)
        if (!sc.buf->device_input)
            CUDA_TRY(cudaMemcpyAsync(grp.d_src + sc.offset, sc.buf->base, sc.floats * sizeof(float), cudaMemcpyHostToDevice, s));
    return WAE_OK;
}

// The device inputs of the batch (`graphs` in batch order): the slots of the planned groups, then the declared ones the planner gave no
// slot (a source that is never started renders silence without reading its buffer, and an input read by reference has none), which
// behave like a node given an AudioBuffer of that shape.  Runs wait for an input read by reference once record_declarations has found
// entries for it.
static void record_device_inputs(wae_batch* b, wae_graph* const* graphs, uint32_t n_graphs) {
    for (auto& grp : b->groups)
        for (auto& sc : grp.src_copies)
            if (sc.buf->device_input) {
                grp.has_device_inputs = true;
                b->sources.add({sc.graph, sc.node, kNodeLevel}, DevInput{grp.d_src + sc.offset, (uint32_t)sc.buf->channels.size(),
                                                                         (uint64_t)sc.buf->length(), (uint64_t)sc.buf->stride});
            }
    b->sources.seal(graphs, n_graphs, [](uint32_t j, const NodeMap&, const Node& nd, auto& declare) {
        if (nd.kind == K_ABSN && nd.buffer && nd.buffer->device_input)
            declare({j, nd.id, kNodeLevel}, DevInput{nullptr, (uint32_t)nd.buffer->channels.size(), (uint64_t)nd.buffer->length(),
                                                     (uint64_t)nd.buffer->stride, nd.buffer->by_reference});
    });
}

// The entries of kind `kind` of the planned groups (their `payload`) gathered per declaration of `t`, each declaration's range [p0, p1)
// set, and uploaded to *d (from `patches`, which the caller keeps alive until the stream has been synchronised).  Runs wait for a
// declaration with entries.
extern "C++" {
template <typename D, typename P>
static wae_status gather_patches(wae_batch* b, Bindings<D>& t, const std::vector<GroupPlan>& gps, int kind, P Entry::Payload::*payload,
                                 std::vector<P>& patches, P** d) {
    std::vector<std::vector<P>> per(t.keys.size());
    for (const auto& gp : gps)
        for (const Entry& e : gp.entries)
            if (e.kind == kind) per[t.index.at({e.graph, e.node, kNodeLevel})].push_back(e.p.*payload);
    for (size_t k = 0; k < per.size(); k++) {
        t.data[k].p0 = (int32_t)patches.size();
        patches.insert(patches.end(), per[k].begin(), per[k].end());
        t.data[k].p1 = (int32_t)patches.size();
        if (!per[k].empty()) t.set_bound(k, false);
    }
    if (!patches.empty() && !(*d = b->dupload_now(patches)))
        return fail(WAE_OUT_OF_MEMORY, std::string("out of device memory (patch entries of ") + t.kind->bind + ")");
    return WAE_OK;
}
}  // extern "C++"

// The declared responses, curves, periodic waves, IIR filters, schedules and value curves of the batch (`graphs` in batch order), after
// planning, and the entries of the device inputs read by reference.  Runs wait for the ones the planner gave memory or patch entries;
// the patch entries are uploaded from the vectors passed, which the caller keeps alive until the stream has been synchronised.
static wae_status record_declarations(wae_batch* b, wae_graph* const* graphs, uint32_t n_graphs, const std::vector<GroupPlan>& gps,
                                      std::vector<CurvePatch>& curve_patches, std::vector<IirPatch>& iir_patches,
                                      std::vector<SchedPatch>& sched_patches, std::vector<LoopPatch>& loop_patches,
                                      std::vector<LoopWalk>& loop_walks, std::vector<SrcRefPatch>& src_refs) {
    b->responses.seal(graphs, n_graphs, [](uint32_t j, const NodeMap&, const Node& nd, auto& declare) {
        if (nd.kind == K_CONV && nd.buffer && nd.buffer->device_input)
            declare({j, nd.id, kNodeLevel}, DevResponse{nullptr, (uint32_t)nd.buffer->channels.size(), (uint64_t)nd.buffer->length(), 0,
                                                        nd.normalize, nd.buffer->sample_rate});
    });
    b->curves.seal(graphs, n_graphs, [](uint32_t j, const NodeMap&, const Node& nd, auto& declare) {
        if (nd.kind == K_SHAPER && nd.device_curve) declare({j, nd.id, kNodeLevel}, DevCurve{nullptr, nd.device_curve, 0, 0});
    });
    b->waves.seal(graphs, n_graphs, [](uint32_t j, const NodeMap&, const Node& nd, auto& declare) {
        if (nd.kind == K_OSC && nd.device_wave)
            declare({j, nd.id, kNodeLevel}, DevWave{nullptr, nd.device_wave, nd.device_wave_len, nd.device_wave_normalize});
    });
    b->iirs.seal(graphs, n_graphs, [](uint32_t j, const NodeMap&, const Node& nd, auto& declare) {
        if (nd.kind == K_IIR && nd.device_iir)
            declare({j, nd.id, kNodeLevel}, DevIir{(uint32_t)nd.feedforward.size(), (uint32_t)nd.feedback.size(), 0, 0});
    });
    b->schedules.seal(graphs, n_graphs, [](uint32_t j, const NodeMap&, const Node& nd, auto& declare) {
        if (nd.device_schedule) {
            DevSchedule d{(nd.sched_stop ? SCHED_BIND_STOP : 0) | (nd.sched_offset ? SCHED_BIND_OFFSET : 0) |
                              (nd.sched_duration ? SCHED_BIND_DURATION : 0),
                          {}, {}, 0, 0};
            std::copy(nd.sched_lo, nd.sched_lo + 4, d.lo);
            std::copy(nd.sched_hi, nd.sched_hi + 4, d.hi);
            declare({j, nd.id, kNodeLevel}, d);
        }
    });
    b->value_curves.seal(graphs, n_graphs, [](uint32_t j, const NodeMap&, const Node& nd, auto& declare) {
        if (nd.kind == K_PARAM && nd.param.device_curve)
            declare({j, nd.param.device_curve_node, nd.param.device_curve_index}, DevValueCurve{nullptr, 0, nd.param.device_curve});
    });
    b->loops.seal(graphs, n_graphs, [](uint32_t j, const NodeMap&, const Node& nd, auto& declare) {
        if (nd.kind == K_ABSN && nd.device_loop)
            declare({j, nd.id, kNodeLevel}, DevLoop{{nd.loop_lo[0], nd.loop_lo[1]}, {nd.loop_hi[0], nd.loop_hi[1]}, 0, 0});
    });
    wae_status st = gather_patches(b, b->curves, gps, E_CURVE, &Entry::Payload::curve, curve_patches, &b->d_curve_patches);
    if (st == WAE_OK) st = gather_patches(b, b->iirs, gps, E_IIR, &Entry::Payload::iir, iir_patches, &b->d_iir_patches);
    if (st == WAE_OK) st = gather_patches(b, b->schedules, gps, E_SCHED, &Entry::Payload::sched, sched_patches, &b->d_sched_patches);
    if (st == WAE_OK) st = gather_patches(b, b->loops, gps, E_LOOP, &Entry::Payload::loop, loop_patches, &b->d_loop_patches);
    if (st == WAE_OK) st = gather_patches(b, b->sources, gps, E_SRC_REF, &Entry::Payload::src_ref, src_refs, &b->d_src_refs);
    for (const auto& gp : gps)
        for (const Entry& e : gp.entries)
            if (e.kind == E_LOOP_WALK) loop_walks.push_back(e.p.walk);
    if (st == WAE_OK && !loop_walks.empty()) {
        b->n_loop_walks = (int)loop_walks.size();
        b->d_loop_walks = b->dupload_now(loop_walks);
        b->d_loop_overflow = b->dalloc<int>(1, true);
        if (!b->d_loop_walks || !b->d_loop_overflow) st = fail(WAE_OUT_OF_MEMORY, "out of device memory (loop playhead tables)");
    }
    return st;
}

// runs of a batch need every declaration they read bound once; the first unbound one is named, kind by kind in this order
static wae_status check_bound(wae_batch* b) {
    if (!b) return fail(WAE_INVALID_ARGUMENT, "null batch");
    const BindTable* const kinds[] = {&b->loops, &b->schedules, &b->value_curves, &b->iirs, &b->waves, &b->curves, &b->responses, &b->sources, &b->params};
    for (const BindTable* t : kinds)
        for (size_t k = 0; t->unbound && k < t->keys.size(); k++)
            if (!t->bound[k]) {
                const BindKey& key = t->keys[k];
                const uint32_t caller = b->order.empty() ? key.graph : b->order[key.graph];
                return fail(WAE_INVALID_STATE, std::string(t->kind->noun) + " never bound: graph " + std::to_string(caller) + ", node " +
                                                   std::to_string(key.node) + (key.param == kNodeLevel ? "" : ", param " + std::to_string(key.param)) +
                                                   " (" + t->kind->bind + ")");
            }
    return WAE_OK;
}

// The value slots of the params declared with wae_param_set_device_value (`graphs` in batch order: one slot per param, in graph, node and
// param order; runs wait for every one, reached by the planner or not) and the patch entries of the planned groups, their operands
// renumbered from param ids to slots; both uploaded (from `info` and `patches`, which the caller keeps alive until the stream has been
// synchronised).  The spatial entries and their transform items likewise (`spatial`, `resp`).
static wae_status record_params(wae_batch* b, wae_graph* const* graphs, uint32_t n_graphs, std::vector<GroupPlan>& gps,
                                std::vector<ParamSlotInfo>& info, std::vector<ParamPatch>& patches, std::vector<SpatialPatch>& spatial,
                                std::vector<RespBindItem>& resp) {
    b->params.seal(graphs, n_graphs, [](uint32_t j, const NodeMap& nodes, const Node& nd, auto& declare) {
        if (nd.kind == K_PARAM) return;
        for (uint32_t i = 0; i < nd.params.size(); i++) {
            const Param& prm = nodes.at(nd.params[i]).param;
            if (!prm.device_bound) continue;
            // a non-finite value takes the default value; an oscillator's pitch takes it clamped to the range, which keeps the bound
            // pitch inside the range its plan was checked for
            const float def = nd.kind == K_OSC ? std::min(std::max(prm.default_value, prm.device_lo), prm.device_hi) : prm.default_value;
            declare({j, nd.id, i}, DevParam{nd.params[i], ParamSlotInfo{prm.device_lo, prm.device_hi, def, 0}}, false);
        }
    });
    if (b->params.keys.empty()) return WAE_OK;
    std::unordered_map<uint64_t, int32_t> slot_of;  // (batch position << 32 | param id) -> slot
    for (size_t k = 0; k < b->params.keys.size(); k++) {
        slot_of[(uint64_t)b->params.keys[k].graph << 32 | b->params.data[k].pid] = (int32_t)k;
        info.push_back(b->params.data[k].info);
    }
    for (auto& gp : gps)
        for (const Entry& e : gp.entries) {
            if (e.kind != E_PARAM) continue;
            ParamPatch p = e.p.param;
            for (int i = 0; i < PATCH_OPS; i++)
                if (p.slot[i] >= 0) p.slot[i] = slot_of.at((uint64_t)e.graph << 32 | (uint32_t)p.slot[i]);
            patches.push_back(p);
        }
    for (auto& gp : gps)
        for (const Entry& sr : gp.entries) {
            if (sr.kind != E_SPATIAL) continue;
            SpatialPatch p = sr.p.spatial;
            for (int i = 0; i < 15; i++)
                if (p.slot[i] >= 0) p.slot[i] = slot_of.at((uint64_t)sr.graph << 32 | (uint32_t)p.slot[i]);
            spatial.push_back(p);
            b->spatial_sphere = b->spatial_sphere || p.kind != SPATIAL_PAN;
            if (p.kind != SPATIAL_RESP) continue;
            RespBindItem it{};  // the blended pair, untrimmed, scale 1: the transform panner_hrtf_conv's host path runs
            it.src = p.resp;
            it.h = sr.spec;
            it.src_stride = it.len = p.taps;
            it.channels = 2;
            it.S = sr.S;
            it.scale = 1.f;
            it.m[0] = it.m[1] = p.taps;
            resp.push_back(it);
            b->spatial_max_taps = std::max(b->spatial_max_taps, p.taps);
            b->spatial_max_S = std::max(b->spatial_max_S, sr.S);
        }
    b->sphere_gen = b->engine->sphere_gen;
    b->n_spatial = (int)spatial.size();
    b->n_spatial_resp = (int)resp.size();
    b->d_spatial = spatial.empty() ? nullptr : b->dupload_now(spatial);
    b->d_spatial_resp = resp.empty() ? nullptr : b->dupload_now(resp);
    if ((!spatial.empty() && !b->d_spatial) || (!resp.empty() && !b->d_spatial_resp))
        return fail(WAE_OUT_OF_MEMORY, "out of device memory (spatial entries)");
    b->d_slot_info = b->dupload_now(info);
    b->d_values = b->dalloc<float>(info.size(), true);
    b->n_patches = (int)patches.size();
    b->d_patches = patches.empty() ? nullptr : b->dupload_now(patches);
    if (!b->d_slot_info || !b->d_values || (!patches.empty() && !b->d_patches)) return fail(WAE_OUT_OF_MEMORY, "out of device memory (bound params)");
    return WAE_OK;
}

static wae_status prep_finish(wae_batch* b, PrepState& ps) {
    CUDA_TRY(cudaEventCreate(&b->ev0));
    CUDA_TRY(cudaEventCreate(&b->ev1));
    int64_t n_chunks = 0;
    for (auto& grp : b->groups)  // the largest number of chunks any group renders
    {
        int64_t c = 0;
        for (size_t sg = 0; sg + 1 < grp.seg_bounds.size(); sg++) c += (grp.seg_bounds[sg + 1] - grp.seg_bounds[sg] + b->chunk - 1) / b->chunk;
        n_chunks = std::max(n_chunks, c);
    }
    uint64_t launches = 0;
    for (auto& st : b->stages) {
        const uint64_t k = (st.kind == S_CONV_FFT || st.kind == S_CONV_MAC || st.kind == S_CONV_MAC_ACC || st.kind == S_SHAPER_OS) ? 2
                           : st.kind == S_HRTF ? (st.n_b > 0 ? 3 : 2) : st.kind == S_CONV_CMP ? 6 : 1;
        // per-quantum stages (class 1) launch once per render quantum of their segment, the others once per chunk of it
        const std::vector<int64_t>& sb = b->groups[st.group].seg_bounds;
        const int64_t seg_len = sb[st.seg + 1] - sb[st.seg];
        launches += st.cls == 1 ? k * (uint64_t)(seg_len / 128) : k * (uint64_t)((seg_len + b->chunk - 1) / b->chunk);
    }
    std::memset(&b->stats, 0, sizeof(b->stats));
    b->stats.kernel_launches_per_run = launches;
    b->stats.stages = b->stages.size();
    b->stats.chunks = (uint64_t)n_chunks;
    b->stats.arena_bytes = b->arena_bytes;
    b->stats.asset_bytes = b->asset_bytes;
    b->stats.algorithmic_bytes = ps.algorithmic_bytes;
    b->stats.graph_quanta = b->needed_quanta;
    return WAE_OK;
}

// The rows of every declared analyser and compressor read-out (wae_analyser_set_readouts, wae_analyser_set_byte_readouts,
// wae_compressor_set_readouts), before planning: the planner points the records at them.
// `graphs` in batch order; the rows of one (node, kind) are laid out in the caller's order.
static wae_status alloc_readout_rows(wae_batch* b, wae_graph* const* graphs, uint32_t n_graphs) {
    for (uint32_t c = 0; c < n_graphs; c++) {
        const uint32_t j = b->batch_pos(c);
        if (!graphs[j]->analyser_readouts && !graphs[j]->compressor_readouts) continue;
        for (const auto& kv : graphs[j]->nodes) {
            const Node& n = kv.second;
            if (n.kind == K_COMP && !n.readout_q.empty()) b->comp_readout_outs[kv.first].add(n_graphs, j, n.readout_q.size());
            if (n.kind != K_ANALYSER || !n.readout_kinds) continue;
            for (uint32_t kind : {(uint32_t)WAE_READOUT_FREQUENCY, (uint32_t)WAE_READOUT_TIME_DOMAIN}) {
                if (!(n.readout_kinds & kind)) continue;
                const uint64_t elems = (uint64_t)n.readout_q.size() * (kind == WAE_READOUT_FREQUENCY ? n.fft_size / 2 : n.fft_size);
                b->readout_outs[{kv.first, kind}].add(n_graphs, j, elems);
                if (n.byte_readout_kinds & kind) b->byte_readout_outs[{kv.first, kind}].add(n_graphs, j, elems);
            }
        }
    }
    for (auto& kv : b->readout_outs)
        if (!(kv.second.d = b->dalloc<float>(kv.second.count))) return fail(WAE_OUT_OF_MEMORY, "out of device memory (analyser read-outs)");
    for (auto& kv : b->byte_readout_outs)
        if (!(kv.second.d = b->dalloc<uint8_t>(kv.second.count))) return fail(WAE_OUT_OF_MEMORY, "out of device memory (analyser read-outs)");
    for (auto& kv : b->comp_readout_outs)
        if (!(kv.second.d = b->dalloc<float>(kv.second.count, true))) return fail(WAE_OUT_OF_MEMORY, "out of device memory (compressor read-outs)");
    return WAE_OK;
}

// `plan` != nullptr: planning only — grouping, the sizing pass of the planner (which touches no device memory) and the chunk choice,
// reported through *plan; nothing is allocated and no CUDA call is made (wae_batch_plan: runs without a GPU).
static wae_status prepare_impl(wae_engine* eng, wae_graph* const* graphs, uint32_t n_graphs, wae_batch** out, wae_plan_info* plan,
                               const std::vector<uint32_t>* order = nullptr) {
    if (!out && !plan) return fail(WAE_INVALID_ARGUMENT, "null out pointer");
    PrepState ps;
    wae_batch* b = nullptr;
    wae_status st = prep_begin(eng, graphs, n_graphs, plan, &b, ps, true, order);
    if (st != WAE_OK || plan) return st;
    record_device_inputs(b, graphs, n_graphs);
    st = alloc_readout_rows(b, graphs, n_graphs);
    if (st != WAE_OK) {
        wae_batch_destroy(b);
        return st;
    }
    const int n_groups = (int)b->groups.size();
    std::vector<GroupPlan> gps(n_groups);
    WorkerPool* pool = (n_groups > 1 && n_graphs >= 64) ? eng->workers() : nullptr;
    if (pool) pool->parallel_for(n_groups, [&](int k) { prep_plan_group(b, graphs, k, ps, gps[k]); });
    else
        for (int k = 0; k < n_groups; k++) prep_plan_group(b, graphs, k, ps, gps[k]);
    for (int k = 0; k < n_groups; k++) {
        if (gps[k].code != WAE_OK) {
            int code = gps[k].code;
            std::string msg = gps[k].error;
            wae_batch_destroy(b);
            return fail(code, msg);
        }
        prep_append_group(b, k, ps, gps[k]);
        // first upload of the group's source PCM, straight from the graphs' buffers (page-locked when the graphs have an engine)
        wae_status cs = enqueue_source_copies(b, b->groups[k], eng->stream);
        if (cs != WAE_OK) {
            wae_batch_destroy(b);
            return cs;
        }
    }
    std::vector<CurvePatch> curve_patches;
    std::vector<IirPatch> iir_patches;
    std::vector<SchedPatch> sched_patches;
    std::vector<LoopPatch> loop_patches;
    std::vector<LoopWalk> loop_walks;
    std::vector<SrcRefPatch> src_refs;
    std::vector<ParamSlotInfo> slot_info;
    std::vector<ParamPatch> patches;
    std::vector<SpatialPatch> spatial;
    std::vector<RespBindItem> spatial_resp;
    std::vector<OutPatch> out_patches;
    for (const auto& gp : gps)
        for (const Entry& e : gp.entries)
            if (e.kind == E_OUT) out_patches.push_back(e.p.out);
    b->n_out_patches = (int)out_patches.size();
    if (!out_patches.empty() && !(b->d_out_patches = b->dupload_now(out_patches))) st = fail(WAE_OUT_OF_MEMORY, "out of device memory (output entries)");
    if (st == WAE_OK) st = record_declarations(b, graphs, n_graphs, gps, curve_patches, iir_patches, sched_patches, loop_patches, loop_walks, src_refs);
    if (st == WAE_OK) st = record_params(b, graphs, n_graphs, gps, slot_info, patches, spatial, spatial_resp);
    if (st != WAE_OK) {
        wae_batch_destroy(b);
        return st;
    }
    const auto t_prep2 = std::chrono::steady_clock::now();  // planned, allocated, uploads enqueued
    st = prep_finish(b, ps);
    if (st == WAE_OK && cudaStreamSynchronize(eng->stream) != cudaSuccess) st = fail(WAE_CUDA_ERROR, "prepare: stream synchronisation failed");
    if (st != WAE_OK) {
        wae_batch_destroy(b);
        return st;
    }
    if (getenv("WAE_PREPARE_PROFILE")) {
        const auto t_prep3 = std::chrono::steady_clock::now();
        auto ms = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point c) { return std::chrono::duration<double, std::milli>(c - a).count(); };
        std::fprintf(stderr, "[wae prepare] sizing %.1f ms, plan+alloc+upload %.1f ms, sync %.1f ms, fresh device blocks %llu, stages %zu\n", ms(ps.t0, ps.t1),
                     ms(ps.t1, t_prep2), ms(t_prep2, t_prep3), (unsigned long long)b->n_cuda_malloc, b->stages.size());
    }
    cudaError_t le = cudaGetLastError();
    if (le != cudaSuccess) {
        wae_batch_destroy(b);
        return fail(WAE_CUDA_ERROR, std::string("prepare: ") + cudaGetErrorString(le));
    }
    *out = b;
    return WAE_OK;
}

WAE_API wae_status wae_batch_prepare(wae_engine* eng, wae_graph* const* graphs, uint32_t n_graphs, wae_batch** out) {
    if (!out) return fail(WAE_INVALID_ARGUMENT, "null out pointer");
    return prepare_impl(eng, graphs, n_graphs, out, nullptr);
}

// What wae_batch_prepare would lower the graphs to, without a device: the planner's sizing pass under the default engine options.
WAE_API wae_status wae_batch_plan(wae_graph* const* graphs, uint32_t n_graphs, wae_plan_info* info) {
    if (!info) return fail(WAE_INVALID_ARGUMENT, "null info pointer");
    wae_engine host_only;  // default options; no stream, no sphere: HRTF panners answer WAE_UNSUPPORTED ("needs an HRIR sphere")
    return prepare_impl(&host_only, graphs, n_graphs, nullptr, info);
}

// Graphs of different shapes: the batch order (many_order) and the graphs in it.  A batch of one shape keeps the caller's array.
struct ManyOrder {
    std::vector<uint32_t> order;
    std::vector<wae_graph*> sorted;
    wae_graph* const* graphs = nullptr;  // what the planner walks
    const std::vector<uint32_t>* order_ptr() const { return order.empty() ? nullptr : &order; }
};
static wae_status many_batch(wae_graph* const* graphs, uint32_t n_graphs, ManyOrder& mo) {
    wae_status st = many_order(graphs, n_graphs, mo.order);
    if (st != WAE_OK) return st;
    mo.graphs = graphs;
    if (!mo.order.empty()) {
        for (uint32_t i : mo.order) mo.sorted.push_back(graphs[i]);
        mo.graphs = mo.sorted.data();
    }
    return WAE_OK;
}

WAE_API wae_status wae_batch_prepare_many(wae_engine* eng, wae_graph* const* graphs, uint32_t n_graphs, wae_batch** out) {
    if (!out) return fail(WAE_INVALID_ARGUMENT, "null out pointer");
    ManyOrder mo;
    wae_status st = many_batch(graphs, n_graphs, mo);
    if (st != WAE_OK) return st;
    return prepare_impl(eng, mo.graphs, n_graphs, out, nullptr, mo.order_ptr());
}

WAE_API wae_status wae_batch_plan_many(wae_graph* const* graphs, uint32_t n_graphs, wae_plan_info* info) {
    if (!info) return fail(WAE_INVALID_ARGUMENT, "null info pointer");
    ManyOrder mo;
    wae_status st = many_batch(graphs, n_graphs, mo);
    if (st != WAE_OK) return st;
    wae_engine host_only;
    return prepare_impl(&host_only, mo.graphs, n_graphs, nullptr, info, mo.order_ptr());
}

WAE_API wae_status wae_batch_plan_quanta(wae_graph* const* graphs, uint32_t n_graphs, uint32_t* group_of, uint64_t* rendered, uint64_t* needed) {
    if (!rendered || !needed) return fail(WAE_INVALID_ARGUMENT, "null argument");
    ManyOrder mo;
    wae_status st = many_batch(graphs, n_graphs, mo);
    if (st != WAE_OK) return st;
    wae_engine host_only;
    std::vector<std::vector<int64_t>> cuts(n_graphs);
    for (uint32_t i = 0; i < n_graphs; i++) cuts[i] = graph_cuts(mo.graphs[i]);
    const std::vector<wae_batch::Group> groups = form_groups(&host_only, mo.graphs, n_graphs, cuts);
    *rendered = *needed = 0;
    for (size_t k = 0; k < groups.size(); k++)
        for (uint32_t j = groups[k].g0; j < groups[k].g1; j++) {
            *rendered += (uint64_t)(groups[k].lq / 128);
            *needed += (uint64_t)(padded_length(mo.graphs[j]) / 128);
            if (group_of) group_of[mo.order.empty() ? j : mo.order[j]] = (uint32_t)k;
        }
    return WAE_OK;
}

static void launch_stage(wae_batch* b, Stage& st, ChunkInfo ci) {
    cudaStream_t s = b->engine->stream;
    switch (st.kind) {
        case S_MIX: launch_mix((MixInst*)st.d_a, (MixEdge*)st.d_b, st.n, ci, s, st.n_b); break;
        case S_MIX_DYN: launch_mix_dyn((MixDynInst*)st.d_a, (MixEdge*)st.d_b, st.n, ci, s); break;
        case S_META: launch_meta((MetaInst*)st.d_a, st.n, ci, s); break;
        case S_DELAY_MONO: launch_delay_mono((DelayInst*)st.d_a, st.n, ci, s); break;
        case S_OSC: launch_oscillator((OscInst*)st.d_a, st.n, ci, s); break;
        case S_CONST: launch_constant((ConstInst*)st.d_a, st.n, ci, s); break;
        case S_ABSN: launch_buffer_source((AbsnInst*)st.d_a, st.n, ci, s); break;
        case S_BIQUAD:
            launch_biquad_serial((BiquadInst*)st.d_a, st.n, st.max_ch, ci, s);
            break;
        case S_PARAM: launch_param((ParamInst*)st.d_a, st.n, ci, s, b->engine->param_parallel); break;
        case S_OSC_AR: launch_osc_arate((OscArInst*)st.d_a, st.n, ci, s); break;
        case S_ABSN_SLOW: launch_buffer_source_slow((AbsnSlowInst*)st.d_a, st.n, ci, s); break;
        case S_BIQUAD_AR: launch_biquad_arate((BiquadArInst*)st.d_a, st.n, st.max_ch, ci, s); break;
        case S_CHAIN:
            st.chain.epoch++;  // hand-off flags of this launch carry its number (never reset, never reused)
            launch_chain(st.variant, (ChainInst*)st.d_a, (ScanCoef*)st.d_b, st.n, st.max_ch, ci, s, st.chain);
            break;
        case S_VSUM:
            st.chain.epoch++;  // (progress counters carry the launch number)
            launch_voice_sum(st.variant, (ChainInst*)st.d_a, (ScanCoef*)st.d_b, (VoiceGroup*)st.d_c, st.n, ci, s, st.chain);
            break;
        case S_IIR: launch_iir((IirInst*)st.d_a, st.n, st.max_ch, ci, s); break;
        case S_GAIN: launch_gain((GainInst*)st.d_a, st.n, ci, s); break;
        case S_SHAPER: launch_shaper((ShaperInst*)st.d_a, st.n, ci, s); break;
        case S_SPAN: launch_stereo_panner((SPanInst*)st.d_a, (float2*)st.d_b, st.n, ci, s); break;
        case S_PAN: launch_panner_eq((PanInst*)st.d_a, st.n, ci, s); break;
        case S_HRTF: launch_hrtf((HrtfInst*)st.d_a, st.n, (HrtfSelInst*)st.d_b, st.n_b, st.max_ch, ci, s); break;
        case S_PAN_DYN: launch_panner_dyn((PanDynInst*)st.d_a, st.n, ci, s); break;
        case S_ABSN_SERIAL: launch_buffer_source_serial((AbsnSerialInst*)st.d_a, st.n, ci, s); break;
        case S_ABSN_BOUND: launch_buffer_source_bound((AbsnBoundInst*)st.d_a, st.n, ci, s); break;
        case S_SHAPER_OS: launch_shaper_os((ShaperOsInst*)st.d_a, st.n, st.max_ch, ci, s); break;
        case S_ROUTE: launch_route((RouteInst*)st.d_a, st.n, ci, s); break;
        case S_DELAY: launch_delay_read((DelayInst*)st.d_a, st.n, ci, s); break;
        case S_DELAY_WRITE: launch_ring_write((DelayInst*)st.d_a, st.n, ci, s); break;
        case S_COMP: launch_compressor((CompInst*)st.d_a, (const CompReadoutInst*)st.d_b, st.n, ci, s); break;
        case S_ANALYSER: launch_analyser((AnalyserInst*)st.d_a, st.n, ci, s); break;
        case S_READOUT_FFT:
        case S_READOUT_TIME: {  // the records with f0 < frame <= f0 + nf (frame 0: the first chunk)
            const int64_t lo = ci.f0 == 0 ? -1 : ci.f0;
            const size_t r0 = std::upper_bound(st.frames.begin(), st.frames.end(), lo) - st.frames.begin();
            const size_t r1 = std::upper_bound(st.frames.begin(), st.frames.end(), ci.f0 + ci.nf) - st.frames.begin();
            if (r1 <= r0) break;
            const ReadoutInst* d = (const ReadoutInst*)st.d_a + r0;
            if (st.kind == S_READOUT_FFT) launch_readout_fft(d, (int)(r1 - r0), st.n_b, ci, s);
            else launch_readout_time(d, (int)(r1 - r0), st.n_b, ci, s);
            break;
        }
        case S_READOUT_SMOOTH: launch_readout_smooth((ReadoutSmoothInst*)st.d_a, st.n, st.n_b, ci, s); break;
        case S_CONV_FFT: launch_conv_fft_in((ConvInput*)st.d_a, st.n, ci, s); break;
        case S_CONV_MAC:
        case S_CONV_MAC_ACC: launch_conv_mac_ifft((ConvPath*)st.d_a, (ConvInput*)st.d_b, st.n, ci, s); break;
        case S_CONV_CMP: launch_conv_compact((ConvCmpInst*)st.d_a, st.n, ci, s); break;
    }
}

// Groups whose source PCM is not all page-locked (graphs built without an engine, buffers below the pinning threshold) get a pinned
// mirror of their slab, built once, when the PCM is uploaded a second time; page-locked buffers are copied from where they are.
// Device inputs take no part: they have no host PCM, and their slots keep the bound audio.
static bool group_sources_pinned(const wae_batch::Group& g) {
    for (auto& sc : g.src_copies)
        if (!sc.buf->device_input && !sc.buf->pinned) return false;
    return true;
}
static wae_status ensure_host_mirror(wae_batch* b) {
    for (auto& g : b->groups) {
        if (!g.src_floats || g.h_src || group_sources_pinned(g)) continue;
        void* hp = nullptr;
        if (cudaHostAlloc(&hp, g.src_floats * sizeof(float), cudaHostAllocDefault) != cudaSuccess) {
            cudaGetLastError();
            return fail(WAE_OUT_OF_MEMORY, "out of memory (pinned mirror of the source PCM)");
        }
        b->pinned.push_back(hp);
        g.h_src = (float*)hp;
        for (auto& sc : g.src_copies)
            if (!sc.buf->device_input) std::memcpy(g.h_src + sc.offset, sc.buf->base, sc.floats * sizeof(float));
    }
    return WAE_OK;
}
static wae_status resend_group_sources(wae_batch* b, wae_batch::Group& g, cudaStream_t s) {
    if (!g.src_floats) return WAE_OK;
    if (g.h_src && !g.has_device_inputs) {
        CUDA_TRY(cudaMemcpyAsync(g.d_src, g.h_src, g.src_floats * sizeof(float), cudaMemcpyHostToDevice, s));
        return WAE_OK;
    }
    if (g.h_src) {  // only the host ranges of the mirror: one copy per run of consecutive host-PCM copies, device-input slots left out
        size_t i = 0;
        const auto& cs = g.src_copies;
        while (i < cs.size()) {
            if (cs[i].buf->device_input) {
                i++;
                continue;
            }
            size_t j = i + 1, end = cs[i].offset + cs[i].floats;
            while (j < cs.size() && !cs[j].buf->device_input && cs[j].offset == end) end += cs[j++].floats;
            CUDA_TRY(cudaMemcpyAsync(g.d_src + cs[i].offset, g.h_src + cs[i].offset, (end - cs[i].offset) * sizeof(float), cudaMemcpyHostToDevice, s));
            i = j;
        }
        return WAE_OK;
    }
    return enqueue_source_copies(b, g, s);
}

// re-upload the source PCM of every AudioBufferSourceNode (page-locked buffers / pinned mirror)
WAE_API wae_status wae_batch_upload(wae_batch* b) {
    CUDA_TRY(cudaSetDevice(b->engine->device));
    wae_status ms = ensure_host_mirror(b);
    if (ms != WAE_OK) return ms;
    for (auto& g : b->groups) {
        ms = resend_group_sources(b, g, b->engine->stream);
        if (ms != WAE_OK) return ms;
    }
    return WAE_OK;
}

WAE_API wae_status wae_batch_set_timing(wae_batch* b, uint32_t per_stage) {
    b->time_stages = per_stage != 0;
    return WAE_OK;
}

// renders one group (all its chunks, all its stages) on the engine stream
static wae_status run_group(wae_batch* b, const wae_batch::Group& g) {
    cudaStream_t s = b->engine->stream;
    // each run writes every float of a bound output: what no stage writes is zeroed first
    if (b->bound_out)
        for (const auto& z : g.out_zero) CUDA_TRY(cudaMemsetAsync(b->bound_out + z.first, 0, z.second * sizeof(float), s));
    // per-stage device time: one event between consecutive launches, recorded on the launching stream and read back in
    // wae_batch_sync (no host synchronisation inside the run)
    size_t e_prev = (size_t)-1;
    auto next_event = [&]() -> size_t {
        if (b->timed_events_used == b->stage_events.size()) {
            cudaEvent_t e;
            if (cudaEventCreate(&e) != cudaSuccess) return (size_t)-1;
            b->stage_events.push_back(e);
        }
        return b->timed_events_used++;
    };
    auto run = [&](size_t i, const ChunkInfo& ci) -> bool {
        launch_stage(b, b->stages[i], ci);
        if (b->time_stages) {
            size_t e = next_event();
            if (e == (size_t)-1) return false;
            if (cudaEventRecord(b->stage_events[e], s) != cudaSuccess) return false;
            b->timed.push_back({i, e_prev, e});
            e_prev = e;
        }
        return true;
    };
    for (size_t sg = 0; sg + 1 < g.seg_bounds.size(); sg++) {  // render segments between suspend points (usually one)
        const size_t s0 = g.seg_stages[sg].first, s1 = g.seg_stages[sg].second;
        // stages are sorted by class: [whole-chunk stages of feedback-free graphs | per-quantum stages | whole-chunk stages after cycles]
        size_t c1 = s0, c2 = s0;
        while (c1 < s1 && b->stages[c1].cls == 0) c1++;
        c2 = c1;
        while (c2 < s1 && b->stages[c2].cls == 1) c2++;
        const int64_t seg_end = g.seg_bounds[sg + 1];
        for (int64_t f0 = g.seg_bounds[sg]; f0 < seg_end; f0 += b->chunk) {
            const ChunkInfo ci{f0, (int32_t)std::min<int64_t>(b->chunk, seg_end - f0), 0};
            if (b->time_stages) {
                e_prev = next_event();
                if (e_prev == (size_t)-1) return fail(WAE_CUDA_ERROR, "cudaEventCreate failed");
                CUDA_TRY(cudaEventRecord(b->stage_events[e_prev], s));
            }
            for (size_t i = s0; i < c1; i++)
                if (!run(i, ci)) return fail(WAE_CUDA_ERROR, "cudaEventRecord failed");
            if (c2 > c1)
                for (int32_t sub = 0; sub < ci.nf; sub += 128) {  // the reference's render loop, for the cyclic part only
                    const ChunkInfo cq{f0 + sub, 128, sub};
                    for (size_t i = c1; i < c2; i++)
                        if (!run(i, cq)) return fail(WAE_CUDA_ERROR, "cudaEventRecord failed");
                }
            for (size_t i = c2; i < s1; i++)
                if (!run(i, ci)) return fail(WAE_CUDA_ERROR, "cudaEventRecord failed");
        }
    }
    return WAE_OK;
}

static wae_status begin_run(wae_batch* b) {
    CUDA_TRY(cudaSetDevice(b->engine->device));
    cudaStream_t s = b->engine->stream;
    for (auto& z : b->zero_on_run) CUDA_TRY(cudaMemsetAsync(z.first, 0, z.second, s));
    b->timed.clear();
    b->timed_events_used = 0;
    for (auto& a : b->analysers) a.computed = a.end_readout;
    CUDA_TRY(cudaEventRecord(b->ev0, s));
    return WAE_OK;
}

WAE_API wae_status wae_batch_run(wae_batch* b) {
    wae_status st = check_bound(b);
    if (st != WAE_OK) return st;
    st = begin_run(b);
    if (st != WAE_OK) return st;
    for (auto& g : b->groups) {
        st = run_group(b, g);
        if (st != WAE_OK) return st;
    }
    CUDA_TRY(cudaEventRecord(b->ev1, b->engine->stream));
    cudaError_t le = cudaGetLastError();
    if (le != cudaSuccess) return fail(WAE_CUDA_ERROR, std::string("run: ") + cudaGetErrorString(le));
    return WAE_OK;
}

WAE_API wae_status wae_batch_group_count(wae_batch* b, uint32_t* n_groups) {
    if (!b || !n_groups) return fail(WAE_INVALID_ARGUMENT, "null argument");
    *n_groups = (uint32_t)b->groups.size();
    return WAE_OK;
}
WAE_API wae_status wae_batch_group_range(wae_batch* b, uint32_t group, uint32_t* first_graph, uint32_t* last_graph) {
    if (!b || !first_graph || !last_graph || group >= b->groups.size()) return fail(WAE_INVALID_ARGUMENT, "null argument / group out of range");
    *first_graph = b->groups[group].g0;
    *last_graph = b->groups[group].g1;
    return WAE_OK;
}
WAE_API wae_status wae_batch_run_group(wae_batch* b, uint32_t group) {
    if (!b || group >= b->groups.size()) return fail(WAE_INVALID_ARGUMENT, "null batch / group out of range");
    wae_status st = check_bound(b);
    if (st != WAE_OK) return st;
    if (group == 0) st = begin_run(b);
    else CUDA_TRY(cudaSetDevice(b->engine->device));
    if (st != WAE_OK) return st;
    st = run_group(b, b->groups[group]);
    if (st != WAE_OK) return st;
    if (group + 1 == b->groups.size()) CUDA_TRY(cudaEventRecord(b->ev1, b->engine->stream));
    cudaError_t le = cudaGetLastError();
    if (le != cudaSuccess) return fail(WAE_CUDA_ERROR, std::string("run_group: ") + cudaGetErrorString(le));
    return WAE_OK;
}

// End-to-end render with HOST buffers: for every group, H2D of its source PCM (pinned mirror), render, D2H of its
// rendered PCM into `host_out` ([n_graphs][channels][length] f32; pinned memory gives full PCIe speed) — on three
// streams, so the copies of neighbouring groups overlap the render.  Synchronous: returns when host_out is complete.
static wae_status run_pipelined(wae_batch* b, float* host_out, bool resend_sources) {
    wae_status st = resend_sources ? ensure_host_mirror(b) : WAE_OK;
    if (st != WAE_OK) return st;
    st = begin_run(b);
    if (st != WAE_OK) return st;
    cudaStream_t s = b->engine->stream;
    const size_t per_graph = (size_t)b->channels * b->length;
    for (auto& g : b->groups) {
        if (g.src_floats && resend_sources) {
            st = resend_group_sources(b, g, b->s_h2d);
            if (st != WAE_OK) return st;
            CUDA_TRY(cudaEventRecord(g.ev_h2d, b->s_h2d));
            CUDA_TRY(cudaStreamWaitEvent(s, g.ev_h2d, 0));
        }
        st = run_group(b, g);
        if (st != WAE_OK) return st;
        CUDA_TRY(cudaEventRecord(g.ev_done, s));
        CUDA_TRY(cudaStreamWaitEvent(b->s_d2h, g.ev_done, 0));
        CUDA_TRY(cudaMemcpyAsync(host_out + (size_t)g.g0 * per_graph, b->d_out + (size_t)g.g0 * per_graph,
                                 (size_t)(g.g1 - g.g0) * per_graph * sizeof(float), cudaMemcpyDeviceToHost, b->s_d2h));
    }
    CUDA_TRY(cudaEventRecord(b->ev1, s));
    CUDA_TRY(cudaStreamSynchronize(b->s_d2h));
    CUDA_TRY(cudaStreamSynchronize(s));
    cudaError_t le = cudaGetLastError();
    if (le != cudaSuccess) return fail(WAE_CUDA_ERROR, std::string("run_pipelined: ") + cudaGetErrorString(le));
    return WAE_OK;
}

static const char* kMixedPacked = "the graphs of this batch differ in shape: there is no [n][channels][length] host layout, copy each graph with "
                                  "wae_batch_fetch_graph (or render with wae_render_many)";
WAE_API wae_status wae_batch_run_pipelined(wae_batch* b, float* host_out) {
    if (b && b->mixed) return fail(WAE_INVALID_STATE, kMixedPacked);
    if (b && b->bound_out)
        return fail(WAE_INVALID_STATE, "wae_batch_run_pipelined streams the batch's own output buffer to host memory, and an output is bound "
                                       "(wae_batch_bind_output): unbind it with a null output first, or run and fetch");
    wae_status st = check_bound(b);
    if (st != WAE_OK) return st;
    return run_pipelined(b, host_out, true);
}

// The caller's pointers must be device (or managed) memory of the engine's GPU and each extent must lie in ONE allocation: checked on the
// host before anything is enqueued, so that a bad pointer never reaches a kernel.  cuMemGetAddressRange is reached through the runtime's
// driver entry point (no link dependency on libcuda).  One checker serves one bind call: the allocations it has looked up are remembered,
// so items that point into one allocation (the rows of one tensor) cost one pair of driver calls, not one per item.
struct BindExtents {
    int device;
    std::map<uintptr_t, size_t> known;  // base -> bytes of allocations of the engine's GPU looked up so far
    // `what`: the pointer's name in the messages; `align`: the alignment the bind kernel's loads need; `overrun`: the message when the
    // extent runs past the end of its allocation
    wae_status check(const void* ptr, size_t align, uint64_t bytes, const char* what, const char* overrun) {
        const uintptr_t p = (uintptr_t)ptr;
        if (!ptr) return fail(WAE_INVALID_ARGUMENT, std::string("bind: null ") + what);
        if (p % align) return fail(WAE_INVALID_ARGUMENT, std::string("bind: ") + what + " is not " + std::to_string(align) + "-byte aligned");
        auto it = known.upper_bound(p);
        if (it != known.begin() && p - std::prev(it)->first < std::prev(it)->second) {
            --it;
            return fits(p - it->first, it->second, bytes, overrun);
        }
        using MemRange = CUresult(CUDAAPI*)(CUdeviceptr*, size_t*, CUdeviceptr);
        static MemRange mem_range = [] {
            void* fn = nullptr;
            cudaDriverEntryPointQueryResult q = cudaDriverEntryPointSymbolNotFound;
            if (cudaGetDriverEntryPoint("cuMemGetAddressRange", &fn, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) {
                cudaGetLastError();
                fn = nullptr;
            }
            return reinterpret_cast<MemRange>(fn);
        }();
        cudaPointerAttributes a{};
        if (cudaPointerGetAttributes(&a, ptr) != cudaSuccess) {
            cudaGetLastError();
            return fail(WAE_INVALID_ARGUMENT, std::string("bind: ") + what + " is not device memory");
        }
        if (!(a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) || a.device != device)
            return fail(WAE_INVALID_ARGUMENT, std::string("bind: ") + what + " is not device (or managed) memory of the engine's GPU");
        if (!mem_range) return fail(WAE_CUDA_ERROR, "bind: cuMemGetAddressRange is not available");
        CUdeviceptr base = 0;
        size_t size = 0;
        if (mem_range(&base, &size, (CUdeviceptr)p) != CUDA_SUCCESS)
            return fail(WAE_INVALID_ARGUMENT, std::string("bind: ") + what + " lies in no device allocation");
        known[(uintptr_t)base] = size;
        return fits(p - (uintptr_t)base, size, bytes, overrun);
    }
    static wae_status fits(uint64_t at, uint64_t size, uint64_t bytes, const char* overrun) {
        if (bytes > size || at > size - bytes) return fail(WAE_INVALID_ARGUMENT, std::string("bind: ") + overrun);
        return WAE_OK;
    }
};

// A bind runs on the engine stream after the work already queued on the caller's `stream`: any stream of the engine's device,
// cudaStreamLegacy (the legacy default stream, which a non-blocking engine stream does not wait for by itself) or cudaStreamPerThread
static wae_status bind_after(wae_batch* b, void* stream) {
    cudaStream_t s = b->engine->stream;
    if (stream && (cudaStream_t)stream != s) {
        if (!b->ev_bind) CUDA_TRY(cudaEventCreateWithFlags(&b->ev_bind, cudaEventDisableTiming));
        CUDA_TRY(cudaEventRecord(b->ev_bind, (cudaStream_t)stream));
        CUDA_TRY(cudaStreamWaitEvent(s, b->ev_bind, 0));
    }
    return WAE_OK;
}

// The item table of a bind -> b->d_bind on the engine stream, through a page-locked staging buffer whose last copy has run
static wae_status stage_bind_table(wae_batch* b, const void* table, size_t bytes) {
    cudaStream_t s = b->engine->stream;
    wae_batch::BindStage* stage = nullptr;
    for (auto& bs : b->bind_stages) {  // a staging buffer whose copy has run
        if (bs.cap < bytes) continue;
        const cudaError_t q = cudaEventQuery(bs.ev);
        if (q == cudaSuccess) {
            stage = &bs;
            break;
        }
        if (q != cudaErrorNotReady) return fail(WAE_CUDA_ERROR, std::string("bind: ") + cudaGetErrorString(q));
        cudaGetLastError();  // (not ready is no error)
    }
    if (!stage && b->bind_stages.size() >= wae_batch::kMaxBindStages) {  // all in flight: wait for the first one that fits
        for (auto& bs : b->bind_stages)
            if (bs.cap >= bytes) {
                CUDA_TRY(cudaEventSynchronize(bs.ev));
                stage = &bs;
                break;
            }
    }
    if (!stage) {
        const size_t cap = std::max<size_t>(bytes, 64 * sizeof(BindItem));
        void* hp = nullptr;
        cudaEvent_t ev = nullptr;
        if (cudaHostAlloc(&hp, cap, cudaHostAllocDefault) != cudaSuccess) {
            cudaGetLastError();
            return fail(WAE_OUT_OF_MEMORY, "out of memory (bind table staging)");
        }
        b->pinned.push_back(hp);
        CUDA_TRY(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
        b->bind_stages.push_back(wae_batch::BindStage{hp, cap, ev});
        stage = &b->bind_stages.back();
    }
    if (bytes > b->bind_cap) {
        void* t = b->dalloc<char>(bytes);
        if (!t) return fail(WAE_OUT_OF_MEMORY, "out of device memory (bind table)");
        b->d_bind = t;
        b->bind_cap = bytes;
    }
    std::memcpy(stage->h, table, bytes);
    CUDA_TRY(cudaMemcpyAsync(b->d_bind, stage->h, bytes, cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaEventRecord(stage->ev, s));
    return WAE_OK;
}

// The playhead tables of the batch's looping bound slow-track records, from the values the binds have written so far.  Every bind that
// writes one of their inputs (loop points, params, schedules) ends with it on the engine stream, so every later run reads tables that
// follow the latest binds, with no work per run and no host synchronisation.
static void derive_loop_tables(wae_batch* b) {
    if (b->n_loop_walks > 0) launch_absn_loop_schedule(b->d_loop_walks, b->n_loop_walks, b->d_loop_overflow, b->engine->stream);
}

extern "C++" {
// The rows of one bind call, staged as one table (Row: the kind's device item)
template <typename Row>
struct BindRows : std::vector<Row> {
    wae_status stage(wae_batch* b) const { return stage_bind_table(b, this->data(), this->size() * sizeof(Row)); }
};
// wae_batch_bind_sources: the copied items (k_bind_sources), then one row per entry of the items read by reference (k_bind_source_refs)
template <>
struct BindRows<BindItem> {
    std::vector<BindItem> copies;
    std::vector<SrcRefBindItem> refs;
    bool empty() const { return copies.empty() && refs.empty(); }
    wae_status stage(wae_batch* b) const {
        const size_t nc = copies.size() * sizeof(BindItem), nr = refs.size() * sizeof(SrcRefBindItem);
        std::vector<char> t(nc + nr);
        if (nc) std::memcpy(t.data(), copies.data(), nc);
        if (nr) std::memcpy(t.data() + nc, refs.data(), nr);
        return stage_bind_table(b, t.data(), t.size());
    }
};

template <typename Item>
static uint32_t param_of(const Item&) { return kNodeLevel; }
static uint32_t param_of(const wae_param_binding& it) { return it.param_index; }
static uint32_t param_of(const wae_value_curve_binding& it) { return it.param_index; }

// The steps every wae_batch_bind_* shares.  Every item is validated before anything is enqueued: its graph index, its declaration in
// `table`, then `check(it, d, k, extents, rows)`, which checks the kind's pointers against declaration k (`d`) and appends the device
// item, or nothing for a declaration the planner never reached.  `launch(rows_on_device, rows)` enqueues the kind's kernel.
template <typename Row, typename Item, typename D, typename Check, typename Launch>
static wae_status bind_items(wae_batch* b, Bindings<D> wae_batch::*table, const Item* items, uint32_t n, void* stream, Check&& check,
                             Launch&& launch) {
    if (!b || (n && !items)) return fail(WAE_INVALID_ARGUMENT, "null batch / items");
    if (n == 0) return WAE_OK;
    CUDA_TRY(cudaSetDevice(b->engine->device));
    Bindings<D>& t = b->*table;
    BindRows<Row> rows;
    std::vector<char> named(t.keys.size(), 0);
    BindExtents extents{b->engine->device, {}};
    for (uint32_t i = 0; i < n; i++) {
        const Item& it = items[i];
        if (it.graph_index >= b->n_graphs)
            return fail(WAE_INVALID_STATE, "bind: graph index " + std::to_string(it.graph_index) + " is out of range");
        const BindKey key{b->batch_pos(it.graph_index), it.node, param_of(it)};
        auto name = [&] {
            return (key.param == kNodeLevel ? std::string() : "param " + std::to_string(key.param) + " of ") + "node " +
                   std::to_string(it.node) + " of graph " + std::to_string(it.graph_index);
        };
        const size_t k = t.find(key);
        if (k == BindTable::npos) return fail(WAE_INVALID_STATE, "bind: " + name() + " was not declared with " + t.kind->declare);
        if (named[k]++)  // (two items of one launch writing one declaration's memory: which one lands would be undefined)
            return fail(WAE_INVALID_ARGUMENT, "bind: " + name() + " is named twice in one call");
        wae_status st = check(it, t.data[k], k, extents, rows);
        if (st != WAE_OK) return st;
    }
    if (!rows.empty()) {
        wae_status st = bind_after(b, stream);
        if (st == WAE_OK) st = rows.stage(b);
        if (st != WAE_OK) return st;
        launch(static_cast<Row*>(b->d_bind), rows);
        cudaError_t le = cudaGetLastError();
        if (le != cudaSuccess) return fail(WAE_CUDA_ERROR, std::string("bind: ") + cudaGetErrorString(le));
    }
    for (size_t k = 0; t.unbound && k < named.size(); k++)
        if (named[k]) t.set_bound(k, true);
    return WAE_OK;
}
}  // extern "C++"

static bool overlaps(const void* p, uint64_t p_bytes, const void* q, uint64_t q_bytes) {
    return (uintptr_t)p < (uintptr_t)q + q_bytes && (uintptr_t)q < (uintptr_t)p + p_bytes;
}

// Copied items are copied into their slots (k_bind_sources); items read by reference have their pointer and stride written into the
// records that play them (k_bind_source_refs), after the copies, from the same staged table
WAE_API wae_status wae_batch_bind_sources(wae_batch* b, const wae_source_binding* items, uint32_t n, void* stream) {
    wae_status bs = bind_items<BindItem>(
        b, &wae_batch::sources, items, n, stream,
        [b](const wae_source_binding& it, const DevInput& d, size_t, BindExtents& extents, auto& rows) -> wae_status {
            if (it.channel_stride < d.length)
                return fail(WAE_INVALID_ARGUMENT, "bind: channel_stride " + std::to_string(it.channel_stride) + " is below the declared length " +
                                                      std::to_string(d.length));
            if (it.channel_stride > (UINT64_MAX / 4 - d.length) / WAE_MAX_CHANNELS)
                return fail(WAE_INVALID_ARGUMENT, "bind: channel_stride runs past the end of its allocation");
            const uint64_t bytes = ((uint64_t)(d.channels - 1) * it.channel_stride + d.length) * sizeof(float);
            wae_status st = extents.check(it.pcm, alignof(float), bytes, "pcm",
                                          "[pcm, pcm + (channels - 1) * channel_stride + length) runs past the end of its allocation");
            if (st != WAE_OK) return st;
            if (d.by_reference) {  // (the runs would read what they write)
                const uint64_t out_bytes = (uint64_t)b->out_off[b->n_graphs] * sizeof(float);
                if (overlaps(it.pcm, bytes, b->d_out, out_bytes) || (b->bound_out && overlaps(it.pcm, bytes, b->bound_out, out_bytes)))
                    return fail(WAE_INVALID_ARGUMENT, "bind: the pcm of node " + std::to_string(it.node) + " of graph " +
                                                          std::to_string(it.graph_index) + ", read by reference, overlaps the batch's output");
                for (int32_t e = d.p0; e < d.p1; e++) rows.refs.push_back(SrcRefBindItem{it.pcm, (int64_t)it.channel_stride, e, 0});
            } else if (d.slot) {
                rows.copies.push_back(BindItem{d.slot, it.pcm, (int64_t)d.stride, (int64_t)it.channel_stride, (int64_t)d.length, (int32_t)d.channels, 0});
            }
            return WAE_OK;
        },
        [b](const BindItem* dev, const BindRows<BindItem>& rows) {
            int64_t max_vec = 0;
            int max_ch = 0;
            for (const BindItem& r : rows.copies) {
                max_vec = std::max<int64_t>(max_vec, r.stride / 4);
                max_ch = std::max<int>(max_ch, r.channels);
            }
            if (!rows.copies.empty()) launch_bind_sources(dev, (int)rows.copies.size(), max_vec, max_ch, b->engine->stream);
            if (!rows.refs.empty())
                launch_bind_source_refs(reinterpret_cast<const SrcRefBindItem*>(dev + rows.copies.size()), (int)rows.refs.size(), b->d_src_refs,
                                        b->engine->stream);
        });
    if (bs != WAE_OK) return bs;
    for (uint32_t i = 0; i < n; i++) {  // the memory each input read by reference now reads (bind_output must not overlap it)
        DevInput& d = b->sources.data[b->sources.find({b->batch_pos(items[i].graph_index), items[i].node, kNodeLevel})];
        if (d.by_reference) {
            d.pcm = items[i].pcm;
            d.pcm_stride = items[i].channel_stride;
        }
    }
    return WAE_OK;
}

WAE_API wae_status wae_batch_bind_params(wae_batch* b, const wae_param_binding* items, uint32_t n, void* stream) {
    if (b && n && b->spatial_sphere && b->sphere_gen != b->engine->sphere_gen)  // (its records point into the freed sphere)
        return fail(WAE_INVALID_STATE, "bind: the batch's HRTF panners were prepared with an HRIR sphere that wae_engine_set_hrir_sphere has "
                                       "since replaced; prepare the batch again");
    return bind_items<ParamBindItem>(
        b, &wae_batch::params, items, n, stream,
        [](const wae_param_binding& it, const DevParam&, size_t slot, BindExtents& extents, auto& rows) -> wae_status {
            wae_status st = extents.check(it.value, alignof(float), sizeof(float), "value", "the value's 4 bytes run past the end of its allocation");
            if (st == WAE_OK) rows.push_back(ParamBindItem{it.value, (int32_t)slot, 0});
            return st;
        },
        [b](const ParamBindItem* dev, const std::vector<ParamBindItem>& rows) {
            launch_bind_params(dev, (int)rows.size(), b->d_slot_info, b->d_values, b->d_patches, b->n_patches, b->engine->stream);
            if (b->n_spatial > 0)
                launch_derive_spatial(b->d_spatial, b->n_spatial, b->d_values, b->d_spatial_resp, b->n_spatial_resp, b->spatial_max_taps,
                                      b->spatial_max_S, b->engine->stream);
            derive_loop_tables(b);  // (a bound playbackRate / detune moves the loop wraps)
        });
}

// The spectra are rewritten in full on the engine stream: runs queued before the bind have read the previous ones by then.
WAE_API wae_status wae_batch_bind_responses(wae_batch* b, const wae_response_binding* items, uint32_t n, void* stream) {
    return bind_items<RespBindItem>(
        b, &wae_batch::responses, items, n, stream,
        [](const wae_response_binding& it, const DevResponse& d, size_t, BindExtents& extents, auto& rows) -> wae_status {
            if (it.channel_stride < d.length)
                return fail(WAE_INVALID_ARGUMENT, "bind: channel_stride " + std::to_string(it.channel_stride) + " is below the declared length " +
                                                      std::to_string(d.length));
            if (it.channel_stride > (UINT64_MAX / 4 - d.length) / 4)
                return fail(WAE_INVALID_ARGUMENT, "bind: channel_stride runs past the end of its allocation");
            wae_status st = extents.check(it.pcm, alignof(float), ((uint64_t)(d.channels - 1) * it.channel_stride + d.length) * sizeof(float), "pcm",
                                          "[pcm, pcm + (channels - 1) * channel_stride + length) runs past the end of its allocation");
            if (st != WAE_OK || !d.h) return st;
            if (rows.size() == 65535)  // (the launch's grid)
                return fail(WAE_INVALID_ARGUMENT, "bind: more than 65535 responses in one call");
            RespBindItem r{};
            r.src = it.pcm;
            r.h = d.h;
            r.src_stride = (int64_t)it.channel_stride;
            r.len = (int64_t)d.length;
            r.sample_rate = d.sample_rate;
            r.channels = (int32_t)d.channels;
            r.S = d.S;
            r.normalize = d.normalize ? 1 : 0;
            r.scale = 1.f;
            rows.push_back(r);
            return WAE_OK;
        },
        [b](RespBindItem* dev, const std::vector<RespBindItem>& rows) {
            int64_t max_len = 0;
            int max_S = 0, max_ch = 0;
            bool any_normalize = false;
            for (const RespBindItem& r : rows) {
                max_len = std::max<int64_t>(max_len, r.len);
                max_S = std::max(max_S, r.S);
                max_ch = std::max(max_ch, (int)r.channels);
                any_normalize |= r.normalize != 0;
            }
            launch_bind_responses(dev, (int)rows.size(), any_normalize, max_len, max_S, max_ch, b->engine->stream);
        });
}

// The curve memory and the patched fields are rewritten on the engine stream: runs queued before the bind have read the previous ones.
WAE_API wae_status wae_batch_bind_curves(wae_batch* b, const wae_curve_binding* items, uint32_t n, void* stream) {
    return bind_items<CurveBindItem>(
        b, &wae_batch::curves, items, n, stream,
        [b](const wae_curve_binding& it, const DevCurve& d, size_t, BindExtents& extents, auto& rows) -> wae_status {
            wae_status st = extents.check(it.curve, alignof(float), (uint64_t)d.length * sizeof(float), "curve",
                                          "[curve, curve + length) runs past the end of its allocation");
            if (st == WAE_OK && d.d) rows.push_back(CurveBindItem{it.curve, d.d, b->d_curve_patches + d.p0, (int32_t)d.length, d.p1 - d.p0});
            return st;
        },
        [b](const CurveBindItem* dev, const std::vector<CurveBindItem>& rows) { launch_bind_curves(dev, (int)rows.size(), b->engine->stream); });
}

// The wavetables are rewritten on the engine stream: runs queued before the bind have read the previous ones.
WAE_API wae_status wae_batch_bind_periodic_waves(wae_batch* b, const wae_periodic_wave_binding* items, uint32_t n, void* stream) {
    return bind_items<WaveBindItem>(
        b, &wae_batch::waves, items, n, stream,
        [](const wae_periodic_wave_binding& it, const DevWave& d, size_t, BindExtents& extents, auto& rows) -> wae_status {
            if (!it.real && !it.imag) return fail(WAE_INVALID_ARGUMENT, "bind: null real and imag");
            const uint64_t bytes = (uint64_t)d.coefficients * sizeof(float);
            for (const float* p : {it.real, it.imag}) {
                if (!p) continue;
                wae_status st = extents.check(p, alignof(float), bytes, p == it.real ? "real" : "imag",
                                              "[coefficients, coefficients + count) runs past the end of its allocation");
                if (st != WAE_OK) return st;
            }
            if (d.d) rows.push_back(WaveBindItem{it.real, it.imag, d.d, (int32_t)d.coefficients, (int32_t)d.table_len, d.normalize ? 1 : 0, 0});
            return WAE_OK;
        },
        [b](const WaveBindItem* dev, const std::vector<WaveBindItem>& rows) {
            int max_len = 0;
            bool any_normalize = false;
            for (const WaveBindItem& r : rows) {
                max_len = std::max(max_len, (int)r.len);
                any_normalize = any_normalize || r.normalize != 0;
            }
            launch_bind_waves(dev, (int)rows.size(), max_len, any_normalize, b->engine->stream);
        });
}

// The coefficient fields are rewritten on the engine stream: runs queued before the bind have read the previous ones.
WAE_API wae_status wae_batch_bind_iir_coefficients(wae_batch* b, const wae_iir_binding* items, uint32_t n, void* stream) {
    return bind_items<IirBindItem>(
        b, &wae_batch::iirs, items, n, stream,
        [b](const wae_iir_binding& it, const DevIir& d, size_t, BindExtents& extents, auto& rows) -> wae_status {
            wae_status st = extents.check(it.feedforward, alignof(double), (uint64_t)d.nff * sizeof(double), "feedforward",
                                          "[feedforward, feedforward + count) runs past the end of its allocation");
            if (st == WAE_OK)
                st = extents.check(it.feedback, alignof(double), (uint64_t)d.nfb * sizeof(double), "feedback",
                                   "[feedback, feedback + count) runs past the end of its allocation");
            if (st == WAE_OK && d.p0 != d.p1)
                rows.push_back(IirBindItem{it.feedforward, it.feedback, b->d_iir_patches + d.p0, (int32_t)d.nff, (int32_t)d.nfb, d.p1 - d.p0, 0});
            return st;
        },
        [b](const IirBindItem* dev, const std::vector<IirBindItem>& rows) { launch_bind_iir(dev, (int)rows.size(), b->engine->stream); });
}

// The schedule fields are rewritten on the engine stream: runs queued before the bind have read the previous ones.
WAE_API wae_status wae_batch_bind_schedules(wae_batch* b, const wae_schedule_binding* items, uint32_t n, void* stream) {
    return bind_items<SchedBindItem>(
        b, &wae_batch::schedules, items, n, stream,
        [b](const wae_schedule_binding& it, const DevSchedule& d, size_t, BindExtents& extents, auto& rows) -> wae_status {
            const int count = 1 + __builtin_popcount((unsigned)d.binds);
            wae_status st = extents.check(it.times, alignof(double), count * sizeof(double), "times",
                                          "[times, times + count) runs past the end of its allocation");
            if (st == WAE_OK && d.p0 != d.p1) {
                SchedBindItem r{it.times, b->d_sched_patches + d.p0, {}, {}, d.p1 - d.p0, d.binds};
                std::copy(d.lo, d.lo + 4, r.lo);
                std::copy(d.hi, d.hi + 4, r.hi);
                rows.push_back(r);
            }
            return st;
        },
        [b](const SchedBindItem* dev, const std::vector<SchedBindItem>& rows) {
            launch_bind_schedules(dev, (int)rows.size(), b->engine->stream);
            derive_loop_tables(b);  // (a bound start, offset, stop or duration moves the loop wraps)
        });
}

// The loop points are rewritten on the engine stream: runs queued before the bind have read the previous ones.
WAE_API wae_status wae_batch_bind_loops(wae_batch* b, const wae_loop_binding* items, uint32_t n, void* stream) {
    return bind_items<LoopBindItem>(
        b, &wae_batch::loops, items, n, stream,
        [b](const wae_loop_binding& it, const DevLoop& d, size_t, BindExtents& extents, auto& rows) -> wae_status {
            wae_status st = extents.check(it.points, alignof(double), 2 * sizeof(double), "points",
                                          "[points, points + 2) runs past the end of its allocation");
            if (st == WAE_OK && d.p0 != d.p1)
                rows.push_back(LoopBindItem{it.points, b->d_loop_patches + d.p0, {d.lo[0], d.lo[1]}, {d.hi[0], d.hi[1]}, d.p1 - d.p0, 0});
            return st;
        },
        [b](const LoopBindItem* dev, const std::vector<LoopBindItem>& rows) {
            launch_bind_loops(dev, (int)rows.size(), b->engine->stream);
            derive_loop_tables(b);
        });
}

// The declared values are rewritten on the engine stream: runs queued before the bind have read the previous ones.
WAE_API wae_status wae_batch_bind_value_curves(wae_batch* b, const wae_value_curve_binding* items, uint32_t n, void* stream) {
    return bind_items<ValueCurveBindItem>(
        b, &wae_batch::value_curves, items, n, stream,
        [](const wae_value_curve_binding& it, const DevValueCurve& d, size_t, BindExtents& extents, auto& rows) -> wae_status {
            wae_status st = extents.check(it.values, alignof(float), (uint64_t)d.length * sizeof(float), "values",
                                          "[values, values + length) runs past the end of its allocation");
            if (st == WAE_OK && d.pool) rows.push_back(ValueCurveBindItem{it.values, d.pool + d.values_off, (int32_t)d.length, 0});
            return st;
        },
        [b](const ValueCurveBindItem* dev, const std::vector<ValueCurveBindItem>& rows) {
            int64_t max_len = 0;
            for (const ValueCurveBindItem& r : rows) max_len = std::max<int64_t>(max_len, r.n);
            launch_bind_value_curves(dev, (int)rows.size(), max_len, b->engine->stream);
        });
}

WAE_API wae_status wae_batch_sync(wae_batch* b) {
    CUDA_TRY(cudaSetDevice(b->engine->device));
    CUDA_TRY(cudaStreamSynchronize(b->engine->stream));
    if (b->d_loop_overflow) {
        int overflow = 0;
        CUDA_TRY(cudaMemcpy(&overflow, b->d_loop_overflow, sizeof overflow, cudaMemcpyDeviceToHost));
        if (overflow)
            return fail(WAE_CUDA_ERROR, "a loop playhead table derived on the device needed more segments than were planned for it (a defect)");
    }
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, b->ev0, b->ev1) == cudaSuccess) b->stats.last_run_ms = ms;
    else cudaGetLastError();
    if (!b->timed.empty()) {
        for (auto& st : b->stages) st.ms = 0.f;
        for (auto& t : b->timed) {
            float v = 0.f;
            if (cudaEventElapsedTime(&v, b->stage_events[t.e0], b->stage_events[t.e1]) == cudaSuccess) b->stages[t.stage].ms += v;
            else cudaGetLastError();
        }
        int best = -1;
        for (size_t i = 0; i < b->stages.size(); i++)
            if (best < 0 || b->stages[i].ms > b->stages[best].ms) best = (int)i;
        if (best >= 0) {
            b->stats.dominant_kernel_ms = b->stages[best].ms;
            const char* nm = kStageNames[b->stages[best].kind];
            std::snprintf(b->stats.dominant_kernel, sizeof(b->stats.dominant_kernel), "%s", nm);
        }
    }
    return WAE_OK;
}

WAE_API wae_status wae_batch_output_device_ptr(wae_batch* b, float** out_dev, uint64_t* out_floats) {
    *out_dev = b->out_ptr();
    *out_floats = (uint64_t)b->out_off[b->n_graphs];
    return WAE_OK;
}

WAE_API wae_status wae_batch_graph_output(wae_batch* b, uint32_t graph_index, uint64_t* offset_floats, uint32_t* channels, uint64_t* length) {
    if (!b || !offset_floats || !channels || !length) return fail(WAE_INVALID_ARGUMENT, "null argument");
    if (graph_index >= b->n_graphs) return fail(WAE_INVALID_ARGUMENT, "graph index out of range");
    const uint32_t j = b->batch_pos(graph_index);
    *offset_floats = b->out_off[j];
    *channels = b->shape[j].first;
    *length = b->shape[j].second;
    return WAE_OK;
}

WAE_API wae_status wae_batch_fetch_graph(wae_batch* b, uint32_t graph_index, float* out) {
    if (!b || !out) return fail(WAE_INVALID_ARGUMENT, "null argument");
    if (graph_index >= b->n_graphs) return fail(WAE_INVALID_ARGUMENT, "graph index out of range");
    const uint32_t j = b->batch_pos(graph_index);
    CUDA_TRY(cudaSetDevice(b->engine->device));
    const size_t bytes = (b->out_off[j + 1] - b->out_off[j]) * sizeof(float);
    if (bytes) CUDA_TRY(cudaMemcpyAsync(out, b->out_ptr() + b->out_off[j], bytes, cudaMemcpyDeviceToHost, b->engine->stream));
    CUDA_TRY(cudaStreamSynchronize(b->engine->stream));
    return WAE_OK;
}

WAE_API wae_status wae_batch_fetch(wae_batch* b, float* host_out) {
    if (b && b->mixed) return fail(WAE_INVALID_STATE, kMixedPacked);
    CUDA_TRY(cudaSetDevice(b->engine->device));
    size_t bytes = (size_t)b->n_graphs * b->channels * b->length * sizeof(float);
    CUDA_TRY(cudaMemcpyAsync(host_out, b->out_ptr(), bytes, cudaMemcpyDeviceToHost, b->engine->stream));
    CUDA_TRY(cudaStreamSynchronize(b->engine->stream));
    return WAE_OK;
}

// Later runs write `out` ([out_floats] in the layout of the batch's own buffer) instead of that buffer: every output entry is rewritten on
// the engine stream, after the work queued on `stream`.  A null `out` with 0 floats returns the batch to its own buffer.
WAE_API wae_status wae_batch_bind_output(wae_batch* b, float* out, uint64_t floats, void* stream) {
    if (!b) return fail(WAE_INVALID_ARGUMENT, "null batch");
    const uint64_t n = (uint64_t)b->out_off[b->n_graphs];
    CUDA_TRY(cudaSetDevice(b->engine->device));
    if (!out) {
        if (floats != 0) return fail(WAE_INVALID_ARGUMENT, "bind_output: a null output (unbind) takes 0 floats, not " + std::to_string(floats));
    } else {
        if (b->dest_reader >= 0)
            return fail(WAE_INVALID_STATE, "bind_output: the destination of graph " +
                                               std::to_string(b->order.empty() ? b->dest_reader : b->order[b->dest_reader]) +
                                               " feeds another node, which reads the batch's own output buffer: its output cannot be bound");
        if (floats != n)
            return fail(WAE_INVALID_ARGUMENT, "bind_output: " + std::to_string(floats) + " floats given, the batch renders " + std::to_string(n));
        // (256 bytes, as cudaMalloc aligns the batch's own buffer: the alignment every writer found at its graph's offset holds)
        BindExtents extents{b->engine->device, {}};
        wae_status st = extents.check(out, 256, n * sizeof(float), "output", "the output runs past the end of its allocation");
        if (st != WAE_OK) return st;
        for (size_t k = 0; k < b->sources.keys.size(); k++) {  // (the runs would write what they read)
            const DevInput& d = b->sources.data[k];
            if (d.by_reference && d.pcm && overlaps(out, n * sizeof(float), d.pcm, d.extent_bytes()))
                return fail(WAE_INVALID_ARGUMENT, "bind_output: the output overlaps the memory node " + std::to_string(b->sources.keys[k].node) +
                                                      " of graph " + std::to_string(b->order.empty() ? b->sources.keys[k].graph : b->order[b->sources.keys[k].graph]) +
                                                      " reads by reference");
        }
    }
    wae_status st = bind_after(b, stream);
    if (st != WAE_OK) return st;
    if (b->n_out_patches > 0) launch_bind_output(b->d_out_patches, b->n_out_patches, out ? out : b->d_out, b->engine->stream);
    cudaError_t le = cudaGetLastError();
    if (le != cudaSuccess) return fail(WAE_CUDA_ERROR, std::string("bind_output: ") + cudaGetErrorString(le));
    b->bound_out = out;
    return WAE_OK;
}

WAE_API wae_status wae_batch_stage_time(wae_batch* b, uint32_t index, char* name64, float* ms, uint32_t* n_instances) {
    if (index >= b->stages.size()) return fail(WAE_INVALID_ARGUMENT, "stage index out of range");
    const Stage& st = b->stages[index];
    const char* nm = kStageNames[st.kind];
    std::snprintf(name64, 64, "%s", nm);
    *ms = st.ms;
    *n_instances = (uint32_t)st.n;
    return WAE_OK;
}

WAE_API wae_status wae_batch_get_stats(wae_batch* b, wae_batch_stats* out) {
    *out = b->stats;
    return WAE_OK;
}

// ---- one-shot render into a HOST buffer: what `OfflineAudioContext::start_rendering_sync` (src/context/offline.rs:157-185) is for
// a batch of contexts.  Everything a render needs happens inside this call, overlapped:
//   sizing pass (workers, all groups at once)
//   -> H2D of every group's source PCM (copy stream; straight from the graphs' page-locked AudioBuffer memory)
//   -> per group, in order: plan (workers, running ahead) | render (engine stream, waits for the group's PCM) | D2H (copy stream)
//   -> D2H lands in `out` directly when `out` is page-locked, else in one of four page-locked staging slots that worker threads
//      copy out to `out` while the next groups are in flight.
// Device memory comes from the engine's cache (wae_engine::dev_alloc): after the first call of a given shape no cudaMalloc / cudaFree.
// copy with non-temporal stores: the destination (the caller's pageable buffer) is written once and not read here, so its lines are
// not fetched first (a plain memcpy of a few MB stays below glibc's non-temporal threshold and pays a read for every line it writes)
static void copy_streaming(void* dst, const void* src, size_t n) {
    char* d = static_cast<char*>(dst);
    const char* sp = static_cast<const char*>(src);
    const size_t head = std::min(n, (size_t)((64 - (reinterpret_cast<uintptr_t>(d) & 63)) & 63));
    if (head) std::memcpy(d, sp, head);
    d += head; sp += head; n -= head;
    if ((reinterpret_cast<uintptr_t>(sp) & 15) == 0) {
        for (; n >= 64; n -= 64, d += 64, sp += 64) {
            const __m128i a = _mm_load_si128(reinterpret_cast<const __m128i*>(sp)), b2 = _mm_load_si128(reinterpret_cast<const __m128i*>(sp + 16));
            const __m128i c = _mm_load_si128(reinterpret_cast<const __m128i*>(sp + 32)), e = _mm_load_si128(reinterpret_cast<const __m128i*>(sp + 48));
            _mm_stream_si128(reinterpret_cast<__m128i*>(d), a);
            _mm_stream_si128(reinterpret_cast<__m128i*>(d + 16), b2);
            _mm_stream_si128(reinterpret_cast<__m128i*>(d + 32), c);
            _mm_stream_si128(reinterpret_cast<__m128i*>(d + 48), e);
        }
    } else {
        for (; n >= 64; n -= 64, d += 64, sp += 64) {
            const __m128i a = _mm_loadu_si128(reinterpret_cast<const __m128i*>(sp)), b2 = _mm_loadu_si128(reinterpret_cast<const __m128i*>(sp + 16));
            const __m128i c = _mm_loadu_si128(reinterpret_cast<const __m128i*>(sp + 32)), e = _mm_loadu_si128(reinterpret_cast<const __m128i*>(sp + 48));
            _mm_stream_si128(reinterpret_cast<__m128i*>(d), a);
            _mm_stream_si128(reinterpret_cast<__m128i*>(d + 16), b2);
            _mm_stream_si128(reinterpret_cast<__m128i*>(d + 32), c);
            _mm_stream_si128(reinterpret_cast<__m128i*>(d + 48), e);
        }
    }
    _mm_sfence();
    if (n) std::memcpy(d, sp, n);
}

// `outs` != nullptr (wae_render_many): one host buffer per graph, outs[i] = [channels_i][length_i] of the caller's graph i; `out` unused.
// `graphs` is then in the batch order of `order` (many_order) when that is given.
static wae_status render_oneshot_host(wae_engine* eng, wae_graph* const* graphs, uint32_t n_graphs, float* out, float* const* outs = nullptr,
                                      const std::vector<uint32_t>* order = nullptr) {
    if (!out && !outs) return fail(WAE_INVALID_ARGUMENT, "null output buffer");
    if (outs)
        for (uint32_t i = 0; i < n_graphs; i++)
            if (!outs[i]) return fail(WAE_INVALID_ARGUMENT, "null output buffer");
    PrepState ps;
    wae_batch* b = nullptr;
    wae_status st = prep_begin(eng, graphs, n_graphs, nullptr, &b, ps, true, order);
    if (st != WAE_OK) return st;
    const int n_groups = (int)b->groups.size();
    // the packed rendered PCM of group k: floats [out_off[g0], out_off[g1])
    auto group_off = [&](const wae_batch::Group& grp) { return b->out_off[grp.g0]; };
    auto group_bytes = [&](const wae_batch::Group& grp) { return (b->out_off[grp.g1] - b->out_off[grp.g0]) * sizeof(float); };
    // outs: the caller's buffer of the graph at batch position j, and whether it is page-locked (its own D2H) or not (staging slot)
    auto graph_out = [&](uint32_t j) { return outs[order ? (*order)[j] : j]; };
    std::vector<char> graph_pinned(outs ? n_graphs : 0, 0);
    cudaStream_t s = eng->stream;
    WorkerPool* pool = eng->workers();
    // ---- everything below must run to its end before the batch can be destroyed: `pending` counts worker tasks in flight
    std::mutex mu;
    std::condition_variable cv;
    int pending = 0;
    std::vector<char> planned(n_groups, 0);
    std::vector<GroupPlan> gps(n_groups);
    auto task_done = [&] {
        std::lock_guard<std::mutex> lk(mu);
        pending--;
        cv.notify_all();
    };
    auto drain = [&] {
        std::unique_lock<std::mutex> lk(mu);
        cv.wait(lk, [&] { return pending == 0; });
    };
    wae_status result = WAE_OK;
    std::string result_msg;
    auto set_fail = [&](wae_status code, const std::string& msg) {
        if (result == WAE_OK) {
            result = code;
            result_msg = msg;
        }
    };
    // 1. the source PCM of all groups, in group order, on the H2D stream
    for (int k = 0; k < n_groups && result == WAE_OK; k++) {
        wae_batch::Group& grp = b->groups[k];
        if (!grp.src_floats) continue;
        if (enqueue_source_copies(b, grp, eng->s_h2d) != WAE_OK || cudaEventRecord(grp.ev_h2d, eng->s_h2d) != cudaSuccess)
            set_fail(WAE_CUDA_ERROR, std::string("one-shot render: H2D of the source PCM failed: ") + wae_last_error());
    }
    // 2. plans, running ahead of the render on the workers
    if (result == WAE_OK) {
        std::lock_guard<std::mutex> lk(mu);
        pending += n_groups;
    }
    if (result == WAE_OK)
        for (int k = 0; k < n_groups; k++)
            pool->submit([&, k] {
                prep_plan_group(b, graphs, k, ps, gps[k]);
                {
                    std::lock_guard<std::mutex> lk(mu);
                    planned[k] = 1;
                }
                task_done();
            });
    // 3. where the rendered PCM lands
    auto is_pinned = [](const void* p) {
        cudaPointerAttributes attr;
        if (cudaPointerGetAttributes(&attr, p) == cudaSuccess) return attr.type == cudaMemoryTypeHost;
        cudaGetLastError();
        return false;
    };
    const bool out_pinned = !outs && is_pinned(out);
    for (uint32_t j = 0; outs && j < n_graphs; j++) graph_pinned[j] = is_pinned(graph_out(j)) ? 1 : 0;
    // (outs: a group whose buffers are all page-locked needs no staging slot)
    auto group_staged = [&](const wae_batch::Group& grp) {
        if (!outs) return !out_pinned;
        for (uint32_t j = grp.g0; j < grp.g1; j++)
            if (!graph_pinned[j] && b->out_off[j + 1] > b->out_off[j]) return true;
        return false;
    };
    size_t max_group_bytes = 0;
    for (auto& grp : b->groups)
        if (group_staged(grp)) max_group_bytes = std::max(max_group_bytes, group_bytes(grp));
    // Pageable `out`, default: whole-group page-locked staging slots, copied out in parts by the workers (below).  WAE_STAGE_RING=1 (an
    // experiment that lost, kept for the record): the PCM comes down in PIECES of a couple of MB through a small
    // ring of page-locked slots meant to stay in the last-level cache (inbound DMA writes allocate there), each piece copied out as soon
    // as it has landed.  Two ranks on one socket: 414 - 1117 ms per call against 184 ms with the group slots — a piece pays a blocking
    // event wait and two thread wake-ups, and 2 MB is not enough work to hide them.
    static const bool use_ring = [] { const char* e = getenv("WAE_STAGE_RING"); return e && atoi(e) != 0; }();
    static const size_t piece_bytes = [] { const char* e = getenv("WAE_STAGE_PIECE_KB"); long kb = e ? atol(e) : 2048; return (size_t)std::max(64l, std::min(65536l, kb)) * 1024; }();
    static const int ring_slots = [] { const char* e = getenv("WAE_STAGE_SLOTS"); int n = e ? atoi(e) : 8; return std::max(2, std::min(64, n)); }();
    const bool ring = !outs && !out_pinned && use_ring;
    if (result == WAE_OK && ring && !eng->ensure_ring(piece_bytes * (size_t)ring_slots)) set_fail(WAE_OUT_OF_MEMORY, "out of memory (page-locked staging ring of the rendered PCM)");
    if (result == WAE_OK && max_group_bytes && !ring && !eng->ensure_stage(max_group_bytes)) set_fail(WAE_OUT_OF_MEMORY, "out of memory (page-locked staging of the rendered PCM)");
    // ring state (guarded by `mu`): slot i is free again once its copy-out is done; groups are handed to the pump thread in order
    std::vector<char> ring_busy(ring ? ring_slots : 0, 0);
    std::vector<cudaEvent_t> ring_ev(ring ? ring_slots : 0, nullptr);
    for (auto& e : ring_ev)
        if (result == WAE_OK && cudaEventCreateWithFlags(&e, cudaEventDisableTiming | cudaEventBlockingSync) != cudaSuccess) set_fail(WAE_CUDA_ERROR, "cudaEventCreate failed");
    int issued_groups = 0;       // groups whose render has been launched and whose ev_done is recorded
    bool pump_abort = false;     // the main thread gave up: no more groups will come
    std::string pump_error;
    std::thread pump;
    if (result == WAE_OK && ring)
        pump = std::thread([&] {
            cudaSetDevice(eng->device);
            size_t piece_no = 0;
            for (int k = 0; k < n_groups; k++) {
                {
                    std::unique_lock<std::mutex> lk(mu);
                    cv.wait(lk, [&] { return issued_groups > k || pump_abort; });
                    if (issued_groups <= k) return;
                }
                wae_batch::Group& grp = b->groups[k];
                if (cudaStreamWaitEvent(eng->s_d2h, grp.ev_done, 0) != cudaSuccess) {
                    std::lock_guard<std::mutex> lk(mu);
                    pump_error = "cudaStreamWaitEvent failed";
                    return;
                }
                const size_t off = group_off(grp) * sizeof(float), bytes = group_bytes(grp);
                for (size_t a0 = 0; a0 < bytes; a0 += piece_bytes, piece_no++) {
                    const size_t nb = std::min(piece_bytes, bytes - a0);
                    const int slot = (int)(piece_no % (size_t)ring_slots);
                    {
                        std::unique_lock<std::mutex> lk(mu);
                        cv.wait(lk, [&] { return !ring_busy[slot]; });
                        ring_busy[slot] = 1;
                        pending++;
                    }
                    char* stage = eng->h_ring + (size_t)slot * piece_bytes;
                    if (cudaMemcpyAsync(stage, (const char*)b->d_out + off + a0, nb, cudaMemcpyDeviceToHost, eng->s_d2h) != cudaSuccess ||
                        cudaEventRecord(ring_ev[slot], eng->s_d2h) != cudaSuccess) {
                        std::lock_guard<std::mutex> lk(mu);
                        pump_error = "D2H failed";
                        ring_busy[slot] = 0;
                        pending--;
                        cv.notify_all();
                        return;
                    }
                    char* dst = (char*)out + off + a0;
                    pool->submit([&, slot, stage, dst, nb] {
                        cudaEventSynchronize(ring_ev[slot]);
                        copy_streaming(dst, stage, nb);
                        {
                            std::lock_guard<std::mutex> lk(mu);
                            ring_busy[slot] = 0;
                        }
                        task_done();  // (notifies: the pump may be waiting for this slot)
                    });
                }
            }
        });
    constexpr int SLOTS = wae_engine::kStageSlots;
    bool slot_busy[SLOTS] = {false, false, false, false};
    std::vector<cudaEvent_t> ev_copy((out_pinned || ring) ? 0 : n_groups, nullptr);
    std::vector<std::unique_ptr<std::atomic<int>>> parts_left;
    for (auto& e : ev_copy)
        if (result == WAE_OK && cudaEventCreateWithFlags(&e, cudaEventDisableTiming | cudaEventBlockingSync) != cudaSuccess)
            set_fail(WAE_CUDA_ERROR, "cudaEventCreate failed");
    static const int env_parts = [] { const char* e = getenv("WAE_COPY_PARTS"); return e ? atoi(e) : 0; }();  // (tuning)
    const int copy_parts = env_parts > 0 ? std::min(env_parts, 32) : std::max(1, std::min(8, pool->size() / 2));
    if (result == WAE_OK) {
        if (cudaEventCreate(&b->ev0) != cudaSuccess || cudaEventCreate(&b->ev1) != cudaSuccess || cudaEventRecord(b->ev0, s) != cudaSuccess)
            set_fail(WAE_CUDA_ERROR, "cudaEventCreate failed");
    }
    // 4. group by group: wait for its plan, render, copy back
    for (int k = 0; k < n_groups && result == WAE_OK; k++) {
        {
            std::unique_lock<std::mutex> lk(mu);
            cv.wait(lk, [&] { return planned[k] != 0; });
        }
        if (gps[k].code != WAE_OK) {
            set_fail(gps[k].code, gps[k].error);
            break;
        }
        prep_append_group(b, k, ps, gps[k]);
        wae_batch::Group& grp = b->groups[k];
        if (grp.src_floats && cudaStreamWaitEvent(s, grp.ev_h2d, 0) != cudaSuccess) {
            set_fail(WAE_CUDA_ERROR, "cudaStreamWaitEvent failed");
            break;
        }
        if (run_group(b, grp) != WAE_OK) {
            set_fail(WAE_CUDA_ERROR, wae_last_error());
            break;
        }
        const size_t off = group_off(grp), bytes = group_bytes(grp);
        // (ring: the pump thread makes the copy stream wait, in group order — a wait queued from here could land between the pieces of
        // the group before)
        if (cudaEventRecord(grp.ev_done, s) != cudaSuccess || (!ring && cudaStreamWaitEvent(eng->s_d2h, grp.ev_done, 0) != cudaSuccess)) {
            set_fail(WAE_CUDA_ERROR, "event record / wait failed");
            break;
        }
        if (out_pinned) {
            if (cudaMemcpyAsync(out + off, b->d_out + off, bytes, cudaMemcpyDeviceToHost, eng->s_d2h) != cudaSuccess) set_fail(WAE_CUDA_ERROR, "D2H failed");
            continue;
        }
        for (uint32_t j = grp.g0; outs && j < grp.g1; j++)  // page-locked outs[i]: a copy of its own
            if (graph_pinned[j] && b->out_off[j + 1] > b->out_off[j] &&
                cudaMemcpyAsync(graph_out(j), b->d_out + b->out_off[j], (b->out_off[j + 1] - b->out_off[j]) * sizeof(float), cudaMemcpyDeviceToHost,
                                eng->s_d2h) != cudaSuccess)
                set_fail(WAE_CUDA_ERROR, "D2H failed");
        if (result != WAE_OK) break;
        if (!group_staged(grp)) continue;
        if (ring) {  // the pump thread brings this group down piece by piece
            std::lock_guard<std::mutex> lk(mu);
            issued_groups = k + 1;
            cv.notify_all();
            continue;
        }
        const int slot = k % SLOTS;
        {
            std::unique_lock<std::mutex> lk(mu);
            cv.wait(lk, [&] { return !slot_busy[slot]; });
            slot_busy[slot] = true;
            pending += copy_parts;
        }
        // (outs: only the runs of graphs with pageable buffers come down into the slot, at their place in the group's packed PCM; the
        // page-locked ones already have their own copy)
        auto stage_group = [&]() -> cudaError_t {
            if (!outs) return cudaMemcpyAsync(eng->h_stage[slot], b->d_out + off, bytes, cudaMemcpyDeviceToHost, eng->s_d2h);
            for (uint32_t j = grp.g0; j < grp.g1;) {
                if (graph_pinned[j]) { j++; continue; }
                uint32_t j1 = j + 1;
                while (j1 < grp.g1 && !graph_pinned[j1]) j1++;
                const size_t n = (b->out_off[j1] - b->out_off[j]) * sizeof(float);
                if (n) {
                    const cudaError_t e = cudaMemcpyAsync((char*)eng->h_stage[slot] + (b->out_off[j] - off) * sizeof(float), b->d_out + b->out_off[j], n,
                                                          cudaMemcpyDeviceToHost, eng->s_d2h);
                    if (e != cudaSuccess) return e;
                }
                j = j1;
            }
            return cudaSuccess;
        };
        if (stage_group() != cudaSuccess || cudaEventRecord(ev_copy[k], eng->s_d2h) != cudaSuccess) {
            set_fail(WAE_CUDA_ERROR, "D2H failed");
            std::lock_guard<std::mutex> lk(mu);
            pending -= copy_parts;
            slot_busy[slot] = false;
            break;
        }
        parts_left.emplace_back(new std::atomic<int>(copy_parts));
        std::atomic<int>* left = parts_left.back().get();
        for (int part = 0; part < copy_parts; part++)
            pool->submit([&, k, slot, part, left, off, bytes] {
                cudaEventSynchronize(ev_copy[k]);
                const size_t chunk = (bytes / copy_parts + 63) / 64 * 64;
                const size_t a0 = std::min(bytes, (size_t)part * chunk), a1 = std::min(bytes, a0 + chunk);
                // (non-temporal stores: a 15 MB part is far below glibc's non-temporal threshold — 3/4 of a 260 MB L3 — and a plain memcpy
                // would fetch every destination line before overwriting it; WAE_STAGE_NT=0: memcpy)
                static const bool nt = [] { const char* e = getenv("WAE_STAGE_NT"); return !e || atoi(e) != 0; }();
                auto put = [&](char* dst, size_t x0, size_t x1) {  // bytes [x0, x1) of the group's staged PCM
                    if (nt) copy_streaming(dst, (const char*)eng->h_stage[slot] + x0, x1 - x0);
                    else std::memcpy(dst, (const char*)eng->h_stage[slot] + x0, x1 - x0);
                };
                if (a1 > a0 && !outs) put((char*)(out + off) + a0, a0, a1);
                const wae_batch::Group& grp_k = b->groups[k];
                for (uint32_t j = grp_k.g0; a1 > a0 && outs && j < grp_k.g1; j++) {  // the pageable outs[i] this part overlaps
                    const size_t j0 = (b->out_off[j] - off) * sizeof(float), j1 = (b->out_off[j + 1] - off) * sizeof(float);
                    const size_t x0 = std::max(a0, j0), x1 = std::min(a1, j1);
                    if (!graph_pinned[j] && x1 > x0) put((char*)graph_out(j) + (x0 - j0), x0, x1);
                }
                if (left->fetch_sub(1) == 1) {
                    std::lock_guard<std::mutex> lk(mu);
                    slot_busy[slot] = false;
                }
                task_done();
            });
    }
    if (result == WAE_OK && cudaEventRecord(b->ev1, s) != cudaSuccess) set_fail(WAE_CUDA_ERROR, "cudaEventRecord failed");
    if (pump.joinable()) {
        {
            std::lock_guard<std::mutex> lk(mu);
            if (issued_groups < n_groups) pump_abort = true;  // (a failure above: the groups that were launched are still brought down)
            cv.notify_all();
        }
        pump.join();
        if (!pump_error.empty()) set_fail(WAE_CUDA_ERROR, "one-shot render: " + pump_error);
    }
    drain();  // plans and copy-outs
    if (cudaStreamSynchronize(eng->s_d2h) != cudaSuccess || cudaStreamSynchronize(s) != cudaSuccess || cudaStreamSynchronize(eng->s_h2d) != cudaSuccess)
        set_fail(WAE_CUDA_ERROR, std::string("one-shot render: ") + cudaGetErrorString(cudaGetLastError()));
    cudaError_t le = cudaGetLastError();
    if (le != cudaSuccess) set_fail(WAE_CUDA_ERROR, std::string("one-shot render: ") + cudaGetErrorString(le));
    for (auto& e : ev_copy)
        if (e) cudaEventDestroy(e);
    for (auto& e : ring_ev)
        if (e) cudaEventDestroy(e);
    wae_batch_destroy(b);
    if (result != WAE_OK) return fail(result, result_msg);
    return WAE_OK;
}

// Page-locked host memory for callers that keep their output (or input) buffers around: D2H lands in such a buffer directly instead of
// going through the staging slots.  wae_host_register page-locks memory the caller allocated itself (it must stay allocated until
// wae_host_unregister); both are thin wrappers so that a binding needs no CUDA of its own.
WAE_API wae_status wae_host_alloc(wae_engine* eng, uint64_t bytes, void** out) {
    if (!eng || !out || bytes == 0) return fail(WAE_INVALID_ARGUMENT, "null engine / out pointer or zero size");
    CUDA_TRY(cudaSetDevice(eng->device));
    if (cudaHostAlloc(out, bytes, cudaHostAllocPortable) != cudaSuccess) {
        cudaGetLastError();
        return fail(WAE_OUT_OF_MEMORY, "out of page-locked host memory");
    }
    return WAE_OK;
}
WAE_API wae_status wae_host_free(wae_engine* eng, void* p) {
    if (!eng) return fail(WAE_INVALID_ARGUMENT, "null engine");
    if (p) CUDA_TRY(cudaFreeHost(p));
    return WAE_OK;
}
WAE_API wae_status wae_host_register(wae_engine* eng, void* p, uint64_t bytes) {
    if (!eng || !p || bytes == 0) return fail(WAE_INVALID_ARGUMENT, "null engine / pointer or zero size");
    CUDA_TRY(cudaSetDevice(eng->device));
    if (cudaHostRegister(p, bytes, cudaHostRegisterPortable) != cudaSuccess) {
        const std::string msg = std::string("cudaHostRegister: ") + cudaGetErrorString(cudaGetLastError());
        return fail(WAE_CUDA_ERROR, msg);
    }
    return WAE_OK;
}
WAE_API wae_status wae_host_unregister(wae_engine* eng, void* p) {
    if (!eng || !p) return fail(WAE_INVALID_ARGUMENT, "null engine / pointer");
    CUDA_TRY(cudaHostUnregister(p));
    return WAE_OK;
}

WAE_API wae_status wae_selftest_conv_fft(float* data, uint32_t mode) {
    if (!data || mode > 3) return fail(WAE_INVALID_ARGUMENT, "wae_selftest_conv_fft: null data or mode > 3");
    conv_fft_selftest(data, (int)mode);
    return WAE_OK;
}

// a one-shot call renders the graphs before a caller could bind anything to their declarations
static wae_status refuse_device_inputs(wae_graph* const* graphs, uint32_t n_graphs) {
    for (uint32_t i = 0; graphs && i < n_graphs; i++) {
        for (const BindKind& kind : kBindKinds)
            if (graphs[i] && graphs[i]->*kind.count)
                return fail(WAE_INVALID_STATE, "graph " + std::to_string(i) + " has " + kind.plural + ": render it with wae_batch_prepare " +
                                                   "(or _prepare_many), " + kind.bind + " and wae_batch_run");
        if (graphs[i] && graphs[i]->analyser_readouts)  // (a one-shot render returns no read-outs)
            return fail(WAE_INVALID_STATE, "graph " + std::to_string(i) + " has analyser read-outs declared: render it with wae_batch_prepare " +
                                               "(or _prepare_many) and wae_batch_run, and read them with wae_batch_fetch_analyser_readouts");
        if (graphs[i] && graphs[i]->compressor_readouts)
            return fail(WAE_INVALID_STATE, "graph " + std::to_string(i) + " has compressor read-outs declared: render it with wae_batch_prepare " +
                                               "(or _prepare_many) and wae_batch_run, and read them with wae_batch_fetch_compressor_readouts");
    }
    return WAE_OK;
}

WAE_API wae_status wae_render_many(wae_engine* eng, wae_graph* const* graphs, uint32_t n_graphs, float* const* outs) {
    if (!outs) return fail(WAE_INVALID_ARGUMENT, "null output buffers");
    if (wae_status ds = refuse_device_inputs(graphs, n_graphs)) return ds;
    ManyOrder mo;
    wae_status st = many_batch(graphs, n_graphs, mo);
    if (st != WAE_OK) return st;
    return render_oneshot_host(eng, mo.graphs, n_graphs, nullptr, outs, mo.order_ptr());
}

WAE_API wae_status wae_render_batch(wae_engine* eng, wae_graph* const* graphs, uint32_t n_graphs, float* out, uint32_t flags) {
    if (wae_status ds = refuse_device_inputs(graphs, n_graphs)) return ds;
    if (!(flags & WAE_RENDER_OUT_DEVICE)) return render_oneshot_host(eng, graphs, n_graphs, out);
    wae_batch* b = nullptr;
    wae_status st = wae_batch_prepare(eng, graphs, n_graphs, &b);
    if (st != WAE_OK) return st;
    st = wae_batch_run(b);
    if (st == WAE_OK) st = wae_batch_sync(b);
    if (st == WAE_OK) {
        size_t bytes = (size_t)b->n_graphs * b->channels * b->length * sizeof(float);
        cudaError_t e = cudaMemcpyAsync(out, b->d_out, bytes, cudaMemcpyDeviceToDevice, eng->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(eng->stream);
        if (e != cudaSuccess) st = fail(WAE_CUDA_ERROR, cudaGetErrorString(e));
    }
    std::string saved = wae_last_error();
    wae_batch_destroy(b);
    if (st != WAE_OK) set_error(saved);
    return st;
}

// AnalyserNode read-out: get_float_time_domain_data (src/analysis.rs:261-264, ring read :114-127)
static const AnalyserRec* find_analyser(wae_batch* b, uint32_t graph_index, wae_node_id node) {
    if (!b || graph_index >= b->n_graphs) return nullptr;
    const uint32_t gi = b->batch_pos(graph_index);
    for (auto& a : b->analysers)
        if (a.graph_index == gi && a.node == node) return &a;
    return nullptr;
}

WAE_API wae_status wae_analyser_get_float_time_domain_data(wae_batch* b, uint32_t graph_index, wae_node_id node, float* out, uint32_t len) {
    const AnalyserRec* a = find_analyser(b, graph_index, node);
    if (!a) return fail(WAE_INVALID_ARGUMENT, "not an analyser of this batch");
    const uint32_t RING = 32768 + 128;
    std::vector<float> ring(RING);
    CUDA_TRY(cudaSetDevice(b->engine->device));
    CUDA_TRY(cudaMemcpy(ring.data(), a->d_ring, RING * sizeof(float), cudaMemcpyDeviceToHost));
    uint32_t n = std::min(len, a->fft_size);
    uint64_t write_index = (uint64_t)a->lq % RING;
    for (uint32_t i = 0; i < n; i++) out[i] = ring[(RING + write_index - n + i) % RING];
    return WAE_OK;
}

WAE_API wae_status wae_analyser_get_float_frequency_data(wae_batch* b, uint32_t graph_index, wae_node_id node, float* out, uint32_t len) {
    AnalyserRec* a = const_cast<AnalyserRec*>(find_analyser(b, graph_index, node));
    if (!a) return fail(WAE_INVALID_ARGUMENT, "not an analyser of this batch");
    CUDA_TRY(cudaSetDevice(b->engine->device));
    const uint32_t RING = 32768 + 128;
    const uint32_t bins = a->fft_size / 2;
    if (!a->computed) {  // one FFT per distinct current_time (analysis.rs:353-361): the read-out happens after the render
        launch_analyser_fft(a->d_ring, (uint32_t)((uint64_t)a->lq % RING), (int)a->fft_size, (float)a->smoothing, a->d_last_fft, a->d_db,
                            b->engine->stream);
        a->computed = true;
    }
    uint32_t n = std::min(len, bins);
    CUDA_TRY(cudaMemcpyAsync(out, a->d_db, n * sizeof(float), cudaMemcpyDeviceToHost, b->engine->stream));
    CUDA_TRY(cudaStreamSynchronize(b->engine->stream));
    return WAE_OK;
}

// The rows of the declared read-outs over the batch (wae_analyser_set_readouts, wae_analyser_set_byte_readouts, wae_compressor_set_readouts)
extern "C++" {  // (templates inside the C ABI's extern "C" block)
template <typename K, typename T>
static const ReadoutRows<T>* find_rows(wae_batch* b, std::map<K, ReadoutRows<T>> wae_batch::*m, const K& key) {
    if (!b) return nullptr;
    auto it = (b->*m).find(key);
    return it == (b->*m).end() ? nullptr : &it->second;
}
static bool readout_kind_ok(uint32_t kind) { return kind == WAE_READOUT_FREQUENCY || kind == WAE_READOUT_TIME_DOMAIN; }
// one graph's rows to the host; `what`: the declaration, as the refusal names it
template <typename T>
static wae_status fetch_rows(wae_batch* b, const ReadoutRows<T>* r, uint32_t graph_index, T* host_out, uint64_t count, const char* what,
                             const char* unit) {
    if (!host_out) return fail(WAE_INVALID_ARGUMENT, "null output");
    if (!r || graph_index >= b->n_graphs || r->off[b->batch_pos(graph_index)] == UINT64_MAX)
        return fail(WAE_INVALID_ARGUMENT, "graph " + std::to_string(graph_index) + " declares no " + what);
    const uint32_t j = b->batch_pos(graph_index);
    if (count != r->len[j]) return fail(WAE_INVALID_ARGUMENT, "the graph's read-outs are " + std::to_string(r->len[j]) + " " + unit);
    CUDA_TRY(cudaSetDevice(b->engine->device));
    CUDA_TRY(cudaMemcpyAsync(host_out, r->d + r->off[j], count * sizeof(T), cudaMemcpyDeviceToHost, b->engine->stream));
    CUDA_TRY(cudaStreamSynchronize(b->engine->stream));
    return WAE_OK;
}
}  // extern "C++"
WAE_API wae_status wae_batch_analyser_readouts_device_ptr(wae_batch* b, wae_node_id node, uint32_t kind, float** ptr, uint64_t* floats) {
    if (!ptr || !floats) return fail(WAE_INVALID_ARGUMENT, "null argument");
    const ReadoutOut* r = readout_kind_ok(kind) ? find_rows(b, &wae_batch::readout_outs, {node, kind}) : nullptr;
    if (!r) return fail(WAE_INVALID_ARGUMENT, "no graph of this batch declares read-outs of that kind on that node");
    *ptr = r->d;
    *floats = r->count;
    return WAE_OK;
}
WAE_API wae_status wae_batch_fetch_analyser_readouts(wae_batch* b, uint32_t graph_index, wae_node_id node, uint32_t kind, float* host_out,
                                                     uint64_t floats) {
    if (!host_out) return fail(WAE_INVALID_ARGUMENT, "null output");
    const ReadoutOut* r = readout_kind_ok(kind) ? find_rows(b, &wae_batch::readout_outs, {node, kind}) : nullptr;
    return fetch_rows(b, r, graph_index, host_out, floats, "read-outs of that kind on that node", "floats");
}
WAE_API wae_status wae_batch_analyser_byte_readouts_device_ptr(wae_batch* b, wae_node_id node, uint32_t kind, uint8_t** ptr,
                                                               uint64_t* bytes) {
    if (!ptr || !bytes) return fail(WAE_INVALID_ARGUMENT, "null argument");
    const ReadoutRows<uint8_t>* r = readout_kind_ok(kind) ? find_rows(b, &wae_batch::byte_readout_outs, {node, kind}) : nullptr;
    if (!r) return fail(WAE_INVALID_ARGUMENT, "no graph of this batch declares byte read-outs of that kind on that node");
    *ptr = r->d;
    *bytes = r->count;
    return WAE_OK;
}
WAE_API wae_status wae_batch_fetch_analyser_byte_readouts(wae_batch* b, uint32_t graph_index, wae_node_id node, uint32_t kind,
                                                          uint8_t* host_out, uint64_t bytes) {
    if (!host_out) return fail(WAE_INVALID_ARGUMENT, "null output");
    const ReadoutRows<uint8_t>* r = readout_kind_ok(kind) ? find_rows(b, &wae_batch::byte_readout_outs, {node, kind}) : nullptr;
    return fetch_rows(b, r, graph_index, host_out, bytes, "byte read-outs of that kind on that node", "bytes");
}
WAE_API wae_status wae_batch_compressor_readouts_device_ptr(wae_batch* b, wae_node_id node, float** ptr, uint64_t* floats) {
    if (!ptr || !floats) return fail(WAE_INVALID_ARGUMENT, "null argument");
    const ReadoutOut* r = find_rows(b, &wae_batch::comp_readout_outs, node);
    if (!r) return fail(WAE_INVALID_ARGUMENT, "no graph of this batch declares compressor read-outs on that node");
    *ptr = r->d;
    *floats = r->count;
    return WAE_OK;
}
WAE_API wae_status wae_batch_fetch_compressor_readouts(wae_batch* b, uint32_t graph_index, wae_node_id node, float* host_out,
                                                       uint64_t floats) {
    if (!host_out) return fail(WAE_INVALID_ARGUMENT, "null output");
    return fetch_rows(b, find_rows(b, &wae_batch::comp_readout_outs, node), graph_index, host_out, floats, "compressor read-outs on that node", "floats");
}

// Analyser::get_byte_time_domain_data (src/analysis.rs:266-276): 128 (1 + x) clamped to a byte
WAE_API wae_status wae_analyser_get_byte_time_domain_data(wae_batch* b, uint32_t graph_index, wae_node_id node, uint8_t* out, uint32_t len) {
    std::vector<float> tmp(len, 0.f);
    wae_status st = wae_analyser_get_float_time_domain_data(b, graph_index, node, tmp.data(), len);
    if (st != WAE_OK) return st;
    const AnalyserRec* a = find_analyser(b, graph_index, node);
    const uint32_t n = std::min(len, a->fft_size);
    for (uint32_t i = 0; i < n; i++) {
        float scaled = 128.f * (1.f + tmp[i]);
        scaled = scaled < 0.f ? 0.f : (scaled > 255.f ? 255.f : scaled);
        out[i] = (uint8_t)scaled;
    }
    return WAE_OK;
}

// Analyser::get_byte_frequency_data (src/analysis.rs:371-401): dB scaled into [minDecibels, maxDecibels] -> 0..255
WAE_API wae_status wae_analyser_get_byte_frequency_data(wae_batch* b, uint32_t graph_index, wae_node_id node, uint8_t* out, uint32_t len) {
    const AnalyserRec* a = find_analyser(b, graph_index, node);
    if (!a) return fail(WAE_INVALID_ARGUMENT, "not an analyser of this batch");
    const uint32_t n = std::min(len, a->fft_size / 2);
    std::vector<float> db(n, 0.f);
    wae_status st = wae_analyser_get_float_frequency_data(b, graph_index, node, db.data(), n);
    if (st != WAE_OK) return st;
    const float mn = (float)a->min_db, mx = (float)a->max_db;
    for (uint32_t i = 0; i < n; i++) {
        float scaled = 255.f / (mx - mn) * (db[i] - mn);
        scaled = !(scaled > 0.f) ? 0.f : (scaled > 255.f ? 255.f : scaled);  // -inf dB (silence) and NaN -> 0
        out[i] = (uint8_t)scaled;
    }
    return WAE_OK;
}

// DynamicsCompressorNode::reduction (src/node/dynamics_compressor.rs:204-206,448): the reduction (dB) of the last frame
WAE_API wae_status wae_compressor_reduction(wae_batch* b, uint32_t graph_index, wae_node_id node, float* out) {
    if (!b || !out) return fail(WAE_INVALID_ARGUMENT, "null argument");
    if (graph_index >= b->n_graphs) return fail(WAE_INVALID_ARGUMENT, "not a dynamics compressor of this batch");
    for (auto& c : b->compressors)
        if (c.graph == b->batch_pos(graph_index) && c.node == node) {
            CUDA_TRY(cudaSetDevice(b->engine->device));
            CUDA_TRY(cudaMemcpyAsync(out, c.d_state + 1, sizeof(float), cudaMemcpyDeviceToHost, b->engine->stream));
            CUDA_TRY(cudaStreamSynchronize(b->engine->stream));
            return WAE_OK;
        }
    return fail(WAE_INVALID_ARGUMENT, "not a dynamics compressor of this batch");
}

// AudioBuffer::resample on the GPU (src/buffer.rs:311-363): `in` / `out` are host pointers, out_cap >= ceil(len * to/from)
WAE_API wae_status wae_resample_linear(wae_engine* eng, const float* in, uint64_t len, float from_rate, float to_rate, float* out,
                                       uint64_t out_cap, uint64_t* out_len) {
    if (!eng || !in || !out || !out_len) return fail(WAE_INVALID_ARGUMENT, "null argument");
    if (std::fabs(from_rate - to_rate) <= 0.1f || len == 0) {  // "very similar sample rate: do not resample"
        if (out_cap < len) return fail(WAE_INVALID_ARGUMENT, "output capacity too small");
        std::memcpy(out, in, len * sizeof(float));
        *out_len = len;
        return WAE_OK;
    }
    uint64_t target = (uint64_t)std::ceil((double)len * ((double)to_rate / (double)from_rate));
    if (out_cap < target) return fail(WAE_INVALID_ARGUMENT, "output capacity too small");
    CUDA_TRY(cudaSetDevice(eng->device));
    float *d_in = nullptr, *d_out = nullptr;
    CUDA_TRY(cudaMalloc(&d_in, len * sizeof(float)));
    if (cudaMalloc(&d_out, target * sizeof(float)) != cudaSuccess) {
        cudaFree(d_in);
        return fail(WAE_OUT_OF_MEMORY, "out of device memory (resample)");
    }
    cudaMemcpyAsync(d_in, in, len * sizeof(float), cudaMemcpyHostToDevice, eng->stream);
    launch_resample_linear(d_in, (int64_t)len, d_out, (int64_t)target, eng->stream);
    cudaMemcpyAsync(out, d_out, target * sizeof(float), cudaMemcpyDeviceToHost, eng->stream);
    cudaError_t e = cudaStreamSynchronize(eng->stream);
    cudaFree(d_in);
    cudaFree(d_out);
    if (e != cudaSuccess) return fail(WAE_CUDA_ERROR, cudaGetErrorString(e));
    *out_len = target;
    return WAE_OK;
}

}  // extern "C"
