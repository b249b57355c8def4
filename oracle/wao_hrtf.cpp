// ORACLE — TEST INFRASTRUCTURE ONLY (see wao_core.h).
//
// HRTF panning.  The reference delegates to the third-party crate `hrtf = "0.8.1"` (Cargo.toml:41; call sites
// src/node/panner.rs:39-68 load_hrtf_processor, :239-271 HrtfState::process) whose source is NOT in the reference source tree.
// This file restates that crate's PUBLISHED algorithm as used by those call sites (interpolation_steps = 1,
// block_len = 128):
//   * HrirSphere::new parses the "HRIR" container (magic, sample rate, HRIR length L, vertex count, index count,
//     triangle indices, then per vertex: position xyz + left[L] + right[L], all little-endian u32 / f32) — the format
//     of resources/IRC_1003_C.bin (44.1 kHz, L = 512, 187 vertices, 370 faces);
//   * per block, the ray from the origin along the source direction selects the sphere triangle it crosses, the three
//     vertex responses are blended with the barycentric coordinates of the hit point (the crate blends the spectra;
//     the blend is linear, so blending the impulse responses is the same function);
//   * the block is convolved with the blended left / right response by overlap-save with L-1 samples of input
//     history (the crate: complex FFT of L+127 points, scaled by distance_gain / pad_length), i.e. a plain L-tap FIR:
//         out[n] = distance_gain * sum_k h[k] * x[n - k]
//     evaluated here in the time domain with f64 accumulation.
// When the context rate differs from the sphere's (the embedded sphere is 44.1 kHz data, contexts are usually 48 kHz) the
// crate resamples every impulse response once, at load time, with rubato's asynchronous sinc resampler (SincFixedIn, one
// `process` call over the whole response, parameters sinc_len 256 / f_cutoff 0.95 / oversampling 160 / cubic / BlackmanHarris2).
// resample_hrir() below restates that algorithm from rubato's published description (windowed-sinc bank, 4 neighbouring sinc
// phases, cubic polynomial between them, start index -sinc_len/2, stop at chunk - sinc_len - 1).  Neither crate is in
// the reference source tree, so the tap values of a resampled sphere are unpinned like the rest of this file.
// Degenerate rays (through a mesh vertex / edge) pick the face with the largest minimum barycentric coordinate instead of
// the crate's first-hit order.
// PARITY UNPINNED: the only reference test (panner.rs:1225-1269) asserts "output != input" and "tail is non-zero"
// (both checked in tests/test_oracle_kat.py when the sphere is present); there are no golden vectors for this path.
#include "wao_panner.h"

#include <cstring>
#include <mutex>

namespace wao {

struct HrirSphereData {
    uint32_t sample_rate = 0, length = 0;
    std::vector<float> pos;             // [v][3]
    std::vector<float> left, right;     // [v][length]
    std::vector<uint32_t> faces;        // [f][3]
};

static std::mutex g_sphere_mutex;
static std::shared_ptr<const HrirSphereData> g_sphere;

// HrirSphere::new (hrtf 0.8.1) — container parsing only
bool hrtf_set_sphere(const void* data, uint64_t len, std::string& err) {
    const uint8_t* p = static_cast<const uint8_t*>(data);
    auto u32 = [&](uint64_t off) {
        uint32_t v;
        std::memcpy(&v, p + off, 4);
        return v;
    };
    if (!p || len < 20 || std::memcmp(p, "HRIR", 4) != 0) {
        err = "invalid HRIR sphere: bad magic";
        return false;
    }
    auto s = std::make_shared<HrirSphereData>();
    s->sample_rate = u32(4);
    s->length = u32(8);
    uint32_t vcount = u32(12), icount = u32(16);
    if (s->length == 0 || vcount == 0 || icount % 3 != 0) {
        err = "invalid HRIR sphere: bad header";
        return false;
    }
    uint64_t need = 20 + 4ull * icount + (uint64_t)vcount * (12 + 8ull * s->length);
    if (len < need) {
        err = "invalid HRIR sphere: truncated";
        return false;
    }
    s->faces.resize(icount);
    std::memcpy(s->faces.data(), p + 20, 4ull * icount);
    for (uint32_t i : s->faces)
        if (i >= vcount) {
            err = "invalid HRIR sphere: face index out of range";
            return false;
        }
    uint64_t off = 20 + 4ull * icount;
    s->pos.resize(3ull * vcount);
    s->left.resize((size_t)vcount * s->length);
    s->right.resize((size_t)vcount * s->length);
    for (uint32_t v = 0; v < vcount; v++) {
        std::memcpy(&s->pos[3 * v], p + off, 12);
        off += 12;
        std::memcpy(&s->left[(size_t)v * s->length], p + off, 4ull * s->length);
        off += 4ull * s->length;
        std::memcpy(&s->right[(size_t)v * s->length], p + off, 4ull * s->length);
        off += 4ull * s->length;
    }
    std::lock_guard<std::mutex> lk(g_sphere_mutex);
    g_sphere = s;
    return true;
}

static std::shared_ptr<const HrirSphereData> current_sphere() {
    std::lock_guard<std::mutex> lk(g_sphere_mutex);
    return g_sphere;
}

// ---- rubato (asynchronous sinc resampler), as hrtf 0.8.1 drives it over one impulse response -----------------------------
namespace {
const float kPi = 3.14159265358979323846f;

float sinc_pi(float x) { return x == 0.f ? 1.f : std::sin(x * kPi) / (x * kPi); }

// make_sincs(npoints, factor, f_cutoff, BlackmanHarris2): `factor` phase-shifted copies of a windowed sinc, each `npoints` long
std::vector<std::vector<float>> make_sinc_bank(size_t npoints, size_t factor, float f_cutoff) {
    const size_t tot = npoints * factor;
    std::vector<float> y(tot);
    const float np_f = (float)tot;
    float sum = 0.f;
    for (size_t x = 0; x < tot; x++) {
        const float xf = (float)x;
        const float bh = 0.35875f - 0.48829f * std::cos(2.f * kPi * xf / np_f) + 0.14128f * std::cos(4.f * kPi * xf / np_f) -
                         0.01168f * std::cos(6.f * kPi * xf / np_f);
        const float val = bh * bh * sinc_pi((xf - (float)(tot / 2)) * f_cutoff / (float)factor);
        sum += val;
        y[x] = val;
    }
    sum /= (float)factor;
    std::vector<std::vector<float>> bank(factor, std::vector<float>(npoints));
    for (size_t p = 0; p < npoints; p++)
        for (size_t n = 0; n < factor; n++) bank[factor - n - 1][p] = y[factor * p + n] / sum;
    return bank;
}

float cubic(float x, const float y[4]) {
    const float a0 = y[1];
    const float a1 = -(1.f / 3.f) * y[0] - 0.5f * y[1] + y[2] - (1.f / 6.f) * y[3];
    const float a2 = 0.5f * (y[0] + y[2]) - y[1];
    const float a3 = 0.5f * (y[1] - y[2]) + (1.f / 6.f) * (y[3] - y[0]);
    const float x2 = x * x;
    return a0 + a1 * x + a2 * x2 + a3 * x2 * x;
}
}  // namespace

std::vector<float> resample_hrir(const std::vector<float>& hrir, double ratio) {
    const size_t sinc_len = 256, factor = 160, chunk = hrir.size();
    const float cutoff = ratio >= 1.0 ? 0.95f : 0.95f * (float)ratio;
    const std::vector<std::vector<float>> bank = make_sinc_bank(sinc_len, factor, cutoff);
    std::vector<float> buf(chunk + 2 * sinc_len, 0.f);  // [2 * sinc_len zeros of history | the response]
    std::memcpy(buf.data() + 2 * sinc_len, hrir.data(), chunk * sizeof(float));
    const double t_ratio = 1.0 / ratio;
    const double end_idx = (double)((ptrdiff_t)chunk - (ptrdiff_t)(sinc_len + 1));
    double idx = -(double)(sinc_len / 2);
    std::vector<float> out;
    while (idx < end_idx) {
        idx += t_ratio;
        const double fl = std::floor(idx);
        ptrdiff_t index = (ptrdiff_t)fl;
        ptrdiff_t sub = (ptrdiff_t)std::floor((idx - fl) * (double)factor);
        const double scaled = idx * (double)factor;
        const float frac = (float)(scaled - std::floor(scaled));
        float pts[4];
        for (int k = 0; k < 4; k++) {
            ptrdiff_t i = index, s2 = sub - 1 + k;
            if (s2 < 0) { s2 += (ptrdiff_t)factor; i -= 1; }
            else if (s2 >= (ptrdiff_t)factor) { s2 -= (ptrdiff_t)factor; i += 1; }
            const float* w = buf.data() + (i + 2 * (ptrdiff_t)sinc_len);
            const float* sc = bank[(size_t)s2].data();
            float acc = 0.f;
            for (size_t j = 0; j < sinc_len; j++) acc += w[j] * sc[j];
            pts[k] = acc;
        }
        out.push_back(cubic(frac, pts));
    }
    return out;
}

static std::mutex g_resampled_mutex;
static std::vector<std::pair<std::pair<const HrirSphereData*, uint32_t>, std::shared_ptr<const HrirSphereData>>> g_resampled;

// HrirSphere::new(reader, sample_rate): every response of the sphere at the context's rate
static std::shared_ptr<const HrirSphereData> sphere_at_rate(const std::shared_ptr<const HrirSphereData>& sp, uint32_t rate) {
    if (rate == sp->sample_rate) return sp;
    std::lock_guard<std::mutex> lk(g_resampled_mutex);
    for (auto& e : g_resampled)
        if (e.first.first == sp.get() && e.first.second == rate) return e.second;
    auto r = std::make_shared<HrirSphereData>();
    r->sample_rate = rate;
    r->pos = sp->pos;
    r->faces = sp->faces;
    const double ratio = (double)rate / (double)sp->sample_rate;
    const size_t nv = sp->pos.size() / 3, L = sp->length;
    for (size_t v = 0; v < nv; v++) {
        for (int ear = 0; ear < 2; ear++) {
            const std::vector<float>& src = ear ? sp->right : sp->left;
            std::vector<float> one(src.begin() + v * L, src.begin() + (v + 1) * L);
            std::vector<float> res = resample_hrir(one, ratio);
            if (v == 0 && ear == 0) r->length = (uint32_t)res.size();
            res.resize(r->length, 0.f);
            std::vector<float>& dst = ear ? r->right : r->left;
            dst.insert(dst.end(), res.begin(), res.end());
        }
    }
    if (g_resampled.size() > 8) g_resampled.erase(g_resampled.begin());
    g_resampled.push_back({{sp.get(), rate}, r});
    return r;
}

struct HrtfState {
    std::shared_ptr<const HrirSphereData> sphere;
    size_t len = 0;
    std::vector<float> prev;   // L-1 input samples before the current block (prev_left_samples == prev_right_samples)
    std::vector<float> hl, hr; // blended responses of the current block
};

bool hrtf_sphere_available(std::string& why) {
    if (current_sphere()) return true;
    why = "HRTF panning needs an HRIR sphere: call set_hrir_sphere with the bytes of resources/IRC_1003_C.bin first";
    return false;
}
size_t hrtf_tail_time_samples(const HrtfState& s) { return s.len; }

std::shared_ptr<HrtfState> hrtf_state_new(float sample_rate) {
    auto sp = current_sphere();
    if (!sp) return nullptr;
    // load_hrtf_processor clamps the rate to >= 27 kHz (panner.rs:46); HrirSphere::new resamples when it differs
    uint32_t sr = (uint32_t)sample_rate;
    if (sr < 27000) sr = 27000;
    sp = sphere_at_rate(sp, sr);
    if (sp->length < 2) return nullptr;
    auto st = std::make_shared<HrtfState>();
    st->sphere = sp;
    st->len = sp->length;
    st->prev.assign(sp->length - 1, 0.f);
    st->hl.assign(sp->length, 0.f);
    st->hr.assign(sp->length, 0.f);
    return st;
}

// Triangle crossed by the ray origin -> 10 * dir and the barycentric coordinates (ka, kb, kc) of the hit point
// (hrtf 0.8.1: ray_triangle_intersection + get_barycentric_coords, f32 arithmetic).
bool hrtf_locate(const float* pos, const uint32_t* faces, size_t n_faces, const float dir_in[3], uint32_t idx[3], float k[3]) {
    const float dir[3] = {dir_in[0] * 10.f, dir_in[1] * 10.f, dir_in[2] * 10.f};
    float best = -3.0e38f;
    bool found = false;
    for (size_t f = 0; f < n_faces; f++) {
        const float* a = pos + 3 * faces[3 * f];
        const float* b = pos + 3 * faces[3 * f + 1];
        const float* c = pos + 3 * faces[3 * f + 2];
        float ba[3] = {b[0] - a[0], b[1] - a[1], b[2] - a[2]};
        float ca[3] = {c[0] - a[0], c[1] - a[1], c[2] - a[2]};
        float nrm[3] = {ba[1] * ca[2] - ba[2] * ca[1], ba[2] * ca[0] - ba[0] * ca[2], ba[0] * ca[1] - ba[1] * ca[0]};
        float d = -(a[0] * nrm[0] + a[1] * nrm[1] + a[2] * nrm[2]);
        float denom = dir[0] * nrm[0] + dir[1] * nrm[1] + dir[2] * nrm[2];
        if (denom == 0.f) continue;
        float t = -d / denom;  // origin = 0
        if (!(t >= 0.f && t <= 1.f)) continue;
        float pt[3] = {dir[0] * t, dir[1] * t, dir[2] * t};
        float v2[3] = {pt[0] - a[0], pt[1] - a[1], pt[2] - a[2]};
        float d00 = ba[0] * ba[0] + ba[1] * ba[1] + ba[2] * ba[2];
        float d01 = ba[0] * ca[0] + ba[1] * ca[1] + ba[2] * ca[2];
        float d11 = ca[0] * ca[0] + ca[1] * ca[1] + ca[2] * ca[2];
        float d20 = v2[0] * ba[0] + v2[1] * ba[1] + v2[2] * ba[2];
        float d21 = v2[0] * ca[0] + v2[1] * ca[1] + v2[2] * ca[2];
        float den = d00 * d11 - d01 * d01;
        if (den == 0.f) continue;
        float v = (d11 * d20 - d01 * d21) / den;
        float w = (d00 * d21 - d01 * d20) / den;
        float u = 1.f - v - w;
        float m = std::fmin(u, std::fmin(v, w));
        if (m > best) {
            best = m;
            found = true;
            idx[0] = faces[3 * f];
            idx[1] = faces[3 * f + 1];
            idx[2] = faces[3 * f + 2];
            k[0] = u;
            k[1] = v;
            k[2] = w;
        }
    }
    return found;
}

// HrtfProcessor::process_samples (hrtf 0.8.1) with interpolation_steps = 1 (panner.rs:60-62)
void hrtf_process(HrtfState& st, const float* source, float new_distance_gain, const float projected_source[3], float* out_lr) {
    const HrirSphereData& sp = *st.sphere;
    const size_t L = sp.length;
    // HrtfState::process swaps y and z into the crate's Vec3 (panner.rs:248-252)
    const float dir[3] = {projected_source[0], projected_source[2], projected_source[1]};
    uint32_t idx[3];
    float k[3];
    if (hrtf_locate(sp.pos.data(), sp.faces.data(), sp.faces.size() / 3, dir, idx, k)) {
        for (size_t i = 0; i < L; i++) {
            st.hl[i] = sp.left[idx[0] * L + i] * k[0] + sp.left[idx[1] * L + i] * k[1] + sp.left[idx[2] * L + i] * k[2];
            st.hr[i] = sp.right[idx[0] * L + i] * k[0] + sp.right[idx[1] * L + i] * k[1] + sp.right[idx[2] * L + i] * k[2];
        }
    }  // else: the previous responses stay (sample_bilinear leaves its outputs untouched)
    std::vector<float> x(L - 1 + RQ);
    std::memcpy(x.data(), st.prev.data(), (L - 1) * sizeof(float));
    std::memcpy(x.data() + (L - 1), source, RQ * sizeof(float));
    for (int n = 0; n < RQ; n++) {
        double al = 0., ar = 0.;
        const float* xn = x.data() + (L - 1) + n;
        for (size_t j = 0; j < L; j++) {
            al += (double)st.hl[j] * (double)xn[-(ptrdiff_t)j];
            ar += (double)st.hr[j] * (double)xn[-(ptrdiff_t)j];
        }
        out_lr[2 * n] = (float)al * new_distance_gain;
        out_lr[2 * n + 1] = (float)ar * new_distance_gain;
    }
    std::memcpy(st.prev.data(), x.data() + RQ, (L - 1) * sizeof(float));
}

}  // namespace wao
