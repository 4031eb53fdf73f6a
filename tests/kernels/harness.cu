// harness.cu - runs ONE plane-convolution launch or ONE layer's weight gradient, given as text in the format
// wun_debug_launches writes (engine.cu export_launch / conv_wgrad), through the product's own planner and launchers; and
// ONE launch of the step's other kernels (first layer, output layer, upsampling backward, sigmoid, Adam, window gather /
// scatter) on buffers the caller passes.
// Test infrastructure (tests/test_kernels_gpu.py, tests/test_step_kernels_gpu.py): linked with the product's kernel sources into
// libwun_kernels.so, never loaded by the product.
//
// Addresses in a description are offsets from the fake bases of the dry run (workspace 1 << 40, parameters 1 << 41, mix
// 1 << 42; -1 = null); the harness moves them onto the device buffers the caller passes.  The wgrad lines' dW / db are
// element offsets into the caller's gradient buffer.  Host-only entry points (wkh_plan_*) keep the fake addresses, so the
// planner sees the same alignments as in the dry run.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <exception>
#include <map>
#include <sstream>
#include <string>
#include <vector>

#include "kernels.h"
#include "kernels_umma.h"

using namespace wun;

namespace {

const long long kWsBase = 1LL << 40, kParBase = 1LL << 41, kMixBase = 1LL << 42, kSlack = 1LL << 38;

struct Bufs {
    long long ws, par, mix;   // device addresses (or the fake bases themselves: plan only)
};
const Bufs kFake = {kWsBase, kParBase, kMixBase};

template <class T>
T* map_addr(long long a, const Bufs& B) {
    if (a == -1) return nullptr;
    long long base = B.ws, off = a - kWsBase;
    if (a >= kMixBase - kSlack) { base = B.mix; off = a - kMixBase; }
    else if (a >= kParBase - kSlack) { base = B.par; off = a - kParBase; }
    return reinterpret_cast<T*>((uintptr_t)(base + off));
}

typedef std::map<std::string, long long> KV;
struct Line {
    std::string kind;
    KV kv;
};

bool parse(const char* text, std::vector<Line>* out) {
    std::istringstream in(text ? text : "");
    std::string ln;
    while (std::getline(in, ln)) {
        std::istringstream ls(ln);
        Line L;
        if (!(ls >> L.kind)) continue;
        std::string tok;
        while (ls >> tok) {
            const size_t eq = tok.find('=');
            if (eq == std::string::npos) return false;
            L.kv[tok.substr(0, eq)] = std::stoll(tok.substr(eq + 1));
        }
        out->push_back(L);
    }
    return true;
}

long long get(const KV& kv, const char* k) {
    auto it = kv.find(k);
    if (it == kv.end()) throw std::string("missing field ") + k;
    return it->second;
}

PlaneView plane_from(const KV& kv, const Bufs& B) {
    PlaneView p;
    memset(&p, 0, sizeof(p));
    p.base = map_addr<const float>(get(kv, "base"), B);
    p.bstride = get(kv, "bstride"); p.rstride = (int)get(kv, "rstride");
    p.r_lo = (int)get(kv, "r_lo"); p.r_hi = (int)get(kv, "r_hi"); p.C = (int)get(kv, "C");
    p.kind = (int)get(kv, "kind"); p.mid_mode = (int)get(kv, "mid_mode"); p.xrows = (int)get(kv, "xrows");
    p.blend = map_addr<const float>(get(kv, "blend"), B);
    return p;
}

// launch / plane / cls / term lines -> ConvLaunch (what conv_forward / conv_dgrad hand to launch_conv)
bool conv_from(const char* text, const Bufs& B, ConvLaunch* L) {
    std::vector<Line> lines;
    if (!parse(text, &lines) || lines.empty() || lines[0].kind != "launch") return false;
    memset(L, 0, sizeof(*L));
    const KV& h = lines[0].kv;
    L->N = (int)get(h, "N"); L->pairC = (int)get(h, "pairC"); L->w_sk = (int)get(h, "w_sk"); L->w_sn = (int)get(h, "w_sn");
    L->W = map_addr<const float>(get(h, "W"), B); L->bias = map_addr<const float>(get(h, "bias"), B);
    L->epilogue = (int)get(h, "epilogue"); L->batch = (int)get(h, "batch");
    L->nplanes = (int)get(h, "nplanes"); L->ncls = (int)get(h, "ncls");
    if (L->nplanes < 1 || L->nplanes > kMaxPlanes || L->ncls < 1 || L->ncls > kMaxClasses) return false;
    int np = 0, nc = 0, nt = 0;
    for (size_t i = 1; i < lines.size(); ++i) {
        const KV& kv = lines[i].kv;
        if (lines[i].kind == "plane") {
            if (np >= L->nplanes) return false;
            L->planes[np++] = plane_from(kv, B);
        } else if (lines[i].kind == "cls") {
            if (nc >= L->ncls) return false;
            OutView& o = L->cls[nc++];
            o.base = map_addr<float>(get(kv, "base"), B); o.bstride = get(kv, "bstride"); o.rstride = (int)get(kv, "rstride");
            o.m_lo = (int)get(kv, "m_lo"); o.m_hi = (int)get(kv, "m_hi"); o.saved = map_addr<const float>(get(kv, "saved"), B);
            o.acc_lo = (int)get(kv, "acc_lo"); o.acc_hi = (int)get(kv, "acc_hi");
            o.term_begin = (int)get(kv, "term_begin"); o.term_end = (int)get(kv, "term_end");
            o.pairC = (int)get(kv, "pairC");
            if (o.pairC) {
                o.base2 = map_addr<float>(get(kv, "base2"), B); o.bstride2 = get(kv, "bstride2"); o.rstride2 = (int)get(kv, "rstride2");
                o.saved2 = map_addr<const float>(get(kv, "saved2"), B);
                o.acc_lo2 = (int)get(kv, "acc_lo2"); o.acc_hi2 = (int)get(kv, "acc_hi2");
                o.lo_h[0] = (int)get(kv, "lo0"); o.hi_h[0] = (int)get(kv, "hi0"); o.lo_h[1] = (int)get(kv, "lo1"); o.hi_h[1] = (int)get(kv, "hi1");
            }
            L->max_rows = std::max(L->max_rows, o.m_hi - o.m_lo);
        } else if (lines[i].kind == "term") {
            if (nt >= kMaxTerms) return false;
            Term& t = L->terms[nt++];
            t.plane = (int)get(kv, "plane"); t.d = (int)get(kv, "d"); t.woff = (int)get(kv, "woff"); t.woff2 = (int)get(kv, "woff2");
        } else {
            return false;
        }
    }
    return np == L->nplanes && nc == L->ncls;
}

// wgrad / wplane / wdpre / wterm lines of one layer -> the groups conv_wgrad builds (WgradLaunch), the layer's class-gradient
// views in order of appearance, and the bias-gradient offset
struct WgradDesc {
    std::vector<WgradLaunch> groups;
    std::vector<PlaneView> class_dpre;
    long long dW = 0, db = 0;
};

bool wgrad_from(const char* text, const Bufs& B, float* grads, float scale, WgradDesc* D) {
    std::vector<Line> lines;
    if (!parse(text, &lines) || lines.empty()) return false;
    for (const Line& l : lines) {
        const KV& kv = l.kv;
        if (l.kind == "wgrad") {
            WgradLaunch W;
            memset(&W, 0, sizeof(W));
            W.N = (int)get(kv, "N"); W.w_sk = (int)get(kv, "w_sk"); W.w_sn = (int)get(kv, "w_sn");
            W.m_lo = (int)get(kv, "m_lo"); W.m_hi = (int)get(kv, "m_hi"); W.batch = (int)get(kv, "batch");
            D->dW = get(kv, "dW"); D->db = get(kv, "db");
            W.dW = grads ? grads + D->dW : nullptr;
            W.scale = scale;
            D->groups.push_back(W);
        } else if (D->groups.empty()) {
            return false;
        } else if (l.kind == "wplane") {
            D->groups.back().plane = plane_from(kv, B);
        } else if (l.kind == "wdpre") {
            const PlaneView v = plane_from(kv, B);
            D->groups.back().dpre = v;
            bool seen = false;
            for (const auto& c : D->class_dpre) seen = seen || memcmp(&c, &v, sizeof(PlaneView)) == 0;
            if (!seen) D->class_dpre.push_back(v);
        } else if (l.kind == "wterm") {
            WgradLaunch& W = D->groups.back();
            if (W.nterms >= 16) return false;
            W.d[W.nterms] = (int)get(kv, "d"); W.woff[W.nterms] = (int)get(kv, "woff");
            ++W.nterms;
        } else {
            return false;
        }
    }
    return true;
}

// the tensor-core form of a layer's groups (conv_wgrad); false = not eligible
bool umma_from(const WgradDesc& D, float* grads, float scale, UmmaWgradLaunch* U) {
    if (D.groups.empty() || D.groups.size() > (size_t)kWgMaxGroups) return false;
    memset(U, 0, sizeof(*U));
    U->ngroups = (int)D.groups.size(); U->batch = D.groups[0].batch; U->dW = D.groups[0].dW;
    U->w_sp = D.groups[0].w_sk; U->w_sg = D.groups[0].w_sn; U->scale = scale;
    for (size_t g = 0; g < D.groups.size(); ++g) {
        WgGroup& G = U->grp[g];
        const WgradLaunch& W = D.groups[g];
        if (W.nterms > kWgMaxTaps) return false;
        G.P = W.plane; G.G = W.dpre; G.m_lo = W.m_lo; G.m_hi = W.m_hi; G.ntaps = W.nterms;
        for (int t = 0; t < W.nterms; ++t) { G.d[t] = W.d[t]; G.woff[t] = W.woff[t]; }
    }
    (void)grads;
    return umma_plan_wgrad(U);
}

std::string g_err;

}  // namespace

extern "C" {

const char* wkh_last_error() { return g_err.c_str(); }

// out[0..8): eligible, NPAD, nsplit, MT, rows_alloc, TB, nbs, pack_bytes.  Returns 0, or -1 for a malformed description.
int wkh_plan_conv(const char* desc, long long* out) {
    try {
        ConvLaunch L;
        if (!conv_from(desc, kFake, &L)) { g_err = "malformed conv description"; return -1; }
        UmmaChoice ch;
        const bool ok = umma_plan_from_conv(L, &ch);
        const long long v[8] = {ok ? 1 : 0, ch.NPAD, ch.nsplit, ch.MT, ch.rows_alloc, ch.TB, ch.nbs, (long long)ch.pack_bytes};
        memcpy(out, v, sizeof(v));
        return 0;
    } catch (const std::string& e) { g_err = e; return -1; } catch (const std::exception& e) { g_err = e.what(); return -1; }
}

// The K-loop steps the tensor-core conv walks (kernels_umma.h next_step) for every (class, row tile) of a launch, from the
// product's planner and umma_build (on a fake pack arena: only block indices are used).  out: TB, nbs, ncls; per class:
// ngroups, ntiles; per tile: nsteps, then (g, c, t0, nt, blk) per step.  Returns the number of values written, or -1 (malformed,
// not eligible, or more than cap values).
int wkh_conv_steps(const char* desc, long long* out, long long cap) {
    try {
        ConvLaunch L;
        if (!conv_from(desc, kFake, &L)) { g_err = "malformed conv description"; return -1; }
        UmmaChoice ch;
        if (!umma_plan_from_conv(L, &ch)) { g_err = "launch not eligible for the tensor-core conv"; return -1; }
        UmmaLaunch U;
        UmmaPackLaunch PL;
        if (umma_build(L, ch, reinterpret_cast<uint8_t*>((uintptr_t)256), &U, &PL) != cudaSuccess) { g_err = "umma_build failed"; return -1; }
        std::vector<long long> v = {U.TB, U.nbs, U.ncls};
        for (int q = 0; q < U.ncls; ++q) {
            const UmmaClass& K = U.cls[q];
            const int ntiles = std::max(0, (K.out.m_hi - K.out.m_lo + 127) / 128);
            v.push_back(K.ngroups);
            v.push_back(ntiles);
            for (int x = 0; x < ntiles; ++x) {
                const size_t at = v.size();
                v.push_back(0);
                ConvStep s = {-1, 0, 0, 0, 0};
                while (next_step(U, K, K.out.m_lo + 128 * x, s)) {
                    v.insert(v.end(), {s.g, s.c, s.t0, s.nt, s.blk});
                    ++v[at];
                }
            }
        }
        if ((long long)v.size() > cap) { g_err = "output too small"; return -1; }
        std::copy(v.begin(), v.end(), out);
        return (int)v.size();
    } catch (const std::string& e) { g_err = e; return -1; } catch (const std::exception& e) { g_err = e.what(); return -1; }
}

// out[0..10): eligible, bulk split fits (umma_plan_wgrad_split > 0), split bytes, partial bytes, ngroups, grid x/y/z, nstages,
// arena bytes wkh_run_wgrad needs for the bulk modes; then per group 10 values: swap, NT, n_mtiles, n_ntiles, taps_per_cta,
// n_tapsets, chunks_per_batch, chunks_per_cta, n_ctas_x, slot0.
int wkh_plan_wgrad(const char* desc, long long* out, int cap) {
    try {
        WgradDesc D;
        if (!wgrad_from(desc, kFake, nullptr, 1.f, &D)) { g_err = "malformed wgrad description"; return -1; }
        if (cap < 10 + 10 * kWgMaxGroups) { g_err = "output too small"; return -1; }
        memset(out, 0, sizeof(long long) * cap);
        UmmaWgradLaunch U;
        const bool ok = umma_from(D, nullptr, 1.f, &U);
        out[0] = ok ? 1 : 0;
        out[4] = (long long)D.groups.size();
        if (!ok) return 0;
        const int batch = U.batch;
        const size_t split = umma_plan_wgrad_split(U, batch, nullptr, nullptr, nullptr);
        out[1] = split > 0; out[2] = (long long)split; out[3] = (long long)umma_wgrad_partial_bytes(U);
        out[5] = U.grid_x; out[6] = U.grid_y; out[7] = U.grid_z; out[8] = U.nstages;
        out[9] = (long long)((split + 255) / 256 * 256 + umma_wgrad_partial_bytes(U) + 256);
        for (int g = 0; g < U.ngroups; ++g) {
            const WgGroup& G = U.grp[g];
            long long* o = out + 10 + 10 * g;
            o[0] = G.swap; o[1] = G.NT; o[2] = G.n_mtiles; o[3] = G.n_ntiles; o[4] = G.taps_per_cta; o[5] = G.n_tapsets;
            o[6] = G.chunks_per_batch; o[7] = G.chunks_per_cta; o[8] = G.n_ctas_x; o[9] = G.slot0;
        }
        return 0;
    } catch (const std::string& e) { g_err = e; return -1; } catch (const std::exception& e) { g_err = e.what(); return -1; }
}

// kernel 0: the tensor-core conv (umma_plan_from_conv + umma_run_conv: weight pack, then the conv); 1: the CUDA-core conv.
// Returns a cudaError_t, or -1 (malformed / not eligible / arena too small).
int wkh_run_conv(const char* desc, void* ws, void* par, void* mix, int kernel, void* arena, long long arena_bytes, void* stream) {
    try {
        const Bufs B = {(long long)(uintptr_t)ws, (long long)(uintptr_t)par, (long long)(uintptr_t)mix};
        ConvLaunch L;
        if (!conv_from(desc, B, &L)) { g_err = "malformed conv description"; return -1; }
        cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
        if (kernel == 1) {
            launch_plane_conv_simt(L, s);
            return (int)cudaGetLastError();
        }
        UmmaChoice ch;
        if (!umma_plan_from_conv(L, &ch)) { g_err = "launch not eligible for the tensor-core conv"; return -1; }
        if ((long long)ch.pack_bytes > arena_bytes || (reinterpret_cast<uintptr_t>(arena) & 255)) { g_err = "pack arena too small"; return -1; }
        return (int)umma_run_conv(L, ch, reinterpret_cast<uint8_t*>(arena), s);
    } catch (const std::string& e) { g_err = e; return -1; } catch (const std::exception& e) { g_err = e.what(); return -1; }
}

// One layer's weight and bias gradient into grads (+=), the way conv_wgrad runs it.  mode 0: split pass with fused bias
// column sums -> bulk-fed wgrad -> fixed-order reduction; 1: the same with the bias by launch_colsum; 2: converter-fed wgrad
// (float atomics) + launch_colsum; 3: CUDA-core wgrad + launch_colsum.  Returns a cudaError_t, or -1.
int wkh_run_wgrad(const char* desc, void* ws, void* par, void* mix, float* grads, float scale, int mode, void* arena,
                  long long arena_bytes, void* stream) {
    try {
        const Bufs B = {(long long)(uintptr_t)ws, (long long)(uintptr_t)par, (long long)(uintptr_t)mix};
        WgradDesc D;
        if (!wgrad_from(desc, B, grads, scale, &D)) { g_err = "malformed wgrad description"; return -1; }
        cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
        float* db = grads + D.db;
        const int batch = D.groups[0].batch;
        auto colsums = [&]() {
            for (const auto& dp : D.class_dpre) launch_colsum(dp, batch, scale, db, s);
        };
        if (mode == 3) {
            colsums();
            for (const auto& W : D.groups) launch_plane_wgrad_simt(W, s);
            return (int)cudaGetLastError();
        }
        UmmaWgradLaunch U;
        if (!umma_from(D, grads, scale, &U)) { g_err = "layer not eligible for the tensor-core wgrad"; return -1; }
        if (mode == 2) {
            colsums();
            return (int)launch_wgrad_umma(U, s);
        }
        const size_t split = umma_plan_wgrad_split(U, batch, nullptr, nullptr, nullptr);
        if (split == 0) { g_err = "the layer's views do not fit one split pass"; return -1; }
        const long long need = (long long)((split + 255) / 256 * 256 + umma_wgrad_partial_bytes(U));
        if (need > arena_bytes || (reinterpret_cast<uintptr_t>(arena) & 255)) { g_err = "split arena too small"; return -1; }
        WgSplit S;
        SplitJobs J;
        if (!umma_wgrad_bulk_setup(&U, batch, reinterpret_cast<uint8_t*>(arena), D.class_dpre.data(), (int)D.class_dpre.size(),
                                   mode == 0 ? db : nullptr, scale, &S, &J)) {
            g_err = "class gradient view not among the split jobs";
            return -1;
        }
        if (mode == 1) colsums();
        cudaError_t e = launch_split_views(J, s);
        if (e == cudaSuccess) e = launch_wgrad_umma_bulk(U, S, s);
        if (e == cudaSuccess) e = launch_wgrad_reduce(U, J, s);
        return (int)e;
    } catch (const std::string& e) { g_err = e; return -1; } catch (const std::exception& e) { g_err = e.what(); return -1; }
}

// ---- the step's other launches (kernels_first.cu, kernels_simt.cu): each through the product's own launcher ----------------------
// Geometry comes as an array of integers (the fields of the engine's `first` / `output` / `upsample` export lines), buffers as
// device pointers; partial-sum arenas must be at least as long as the product's own size functions say.

long long wkh_first_partial_bytes(int batch) { return (long long)first_wgrad_partial_bytes(batch); }
int wkh_first_supported(int C, int N, int k) { return first_layer_supported(C, N, k) ? 1 : 0; }

// g: C, N, k, pad_left, batch, x_bstride, T, dec_bstride, Td, odd_bstride, mo_lo, mo_hi
static bool first_from(const long long* g, const float* x, float* dec, float* odd, const float* W, const float* bias, FirstLayer* F,
                       int* C, int* N) {
    memset(F, 0, sizeof(*F));
    *C = (int)g[0]; *N = (int)g[1];
    F->k = (int)g[2]; F->pad_left = (int)g[3]; F->batch = (int)g[4];
    F->x = x; F->x_bstride = g[5]; F->T = (int)g[6];
    F->dec = dec; F->dec_bstride = g[7]; F->Td = (int)g[8];
    F->odd = odd; F->odd_bstride = g[9]; F->mo_lo = (int)g[10]; F->mo_hi = (int)g[11];
    F->W = W; F->bias = bias;
    if (!first_layer_supported(*C, *N, F->k)) { g_err = "first layer shape not supported"; return false; }
    return true;
}

int wkh_first_fwd(const long long* g, const float* x, float* dec, float* odd, const float* W, const float* bias, void* stream) {
    FirstLayer F;
    int C, N;
    if (!first_from(g, x, dec, odd, W, bias, &F, &C, &N)) return -1;
    launch_first_fwd(F, C, N, reinterpret_cast<cudaStream_t>(stream));
    return (int)cudaGetLastError();
}

int wkh_first_wgrad(const long long* g, const float* x, float* gdec, float* godd, float* dW, float* db, float scale, float* part,
                    long long part_bytes, void* stream) {
    FirstWgrad P;
    memset(&P, 0, sizeof(P));
    int C, N;
    if (!first_from(g, x, gdec, godd, nullptr, nullptr, &P.L, &C, &N)) return -1;
    if (part_bytes < (long long)first_wgrad_partial_bytes(P.L.batch)) { g_err = "first-layer partial arena too small"; return -1; }
    P.dW = dW; P.db = db; P.scale = scale; P.part = part;
    launch_first_wgrad(P, C, N, reinterpret_cast<cudaStream_t>(stream));
    return (int)cudaGetLastError();
}

// g: batch, T_in, Tf, T_out, C, F, nconv, K, ofs, pad_left, crop_feat, crop_out, output_type, activation, training, then w_off[8],
// b_off[8] (flat parameter offsets)
static void output_from(const long long* g, float inv_count, const float* params, const float* mix, const float* feat, OutputLaunch* O) {
    memset(O, 0, sizeof(*O));
    O->batch = (int)g[0]; O->T_in = (int)g[1]; O->Tf = (int)g[2]; O->T_out = (int)g[3]; O->C = (int)g[4]; O->F = (int)g[5];
    O->nconv = (int)g[6]; O->K = (int)g[7]; O->ofs = (int)g[8]; O->pad_left = (int)g[9]; O->crop_feat = (int)g[10];
    O->crop_out = (int)g[11]; O->output_type = (int)g[12]; O->activation = (int)g[13]; O->training = (int)g[14];
    for (int s = 0; s < 8; ++s) { O->w_off[s] = g[15 + s]; O->b_off[s] = g[23 + s]; }
    O->inv_count = inv_count; O->params = params; O->mix = mix; O->feat = feat;
}

// out[0]: output_wgrad_partial_bytes, out[1]: output_loss_partial_bytes
int wkh_output_partial_bytes(const long long* g, long long* out) {
    OutputLaunch O;
    output_from(g, 1.f, nullptr, nullptr, nullptr, &O);
    out[0] = (long long)output_wgrad_partial_bytes(O);
    out[1] = (long long)output_loss_partial_bytes(O.batch, O.T_out);
    return 0;
}

// loss_count: the CTA counter of the loss sum (0 before; the launch leaves it 0)
int wkh_output_fwd(const long long* g, float inv_count, const float* params, const float* mix, const float* feat, const float* targets,
                   float* outputs, float* dpre, float* loss, float* loss_part, long long part_bytes, unsigned* loss_count, void* stream) {
    OutputLaunch O;
    output_from(g, inv_count, params, mix, feat, &O);
    if (O.nconv * O.C > WUN_MAX_OUT_COLS) { g_err = "nconv * C above WUN_MAX_OUT_COLS"; return -1; }
    if (targets && loss && (!loss_count || part_bytes < (long long)output_loss_partial_bytes(O.batch, O.T_out))) { g_err = "loss needs a counter and a partial arena"; return -1; }
    O.targets = targets; O.outputs = outputs; O.dpre = dpre; O.loss = loss; O.loss_part = loss_part; O.loss_count = loss_count;
    launch_output_fwd(O, reinterpret_cast<cudaStream_t>(stream));
    return (int)cudaGetLastError();
}

int wkh_output_dgrad(const long long* g, const float* params, const float* feat, float* dpre, float* gfeat, void* stream) {
    OutputLaunch O;
    output_from(g, 1.f, params, nullptr, feat, &O);
    O.dpre = dpre;
    launch_output_dgrad(O, gfeat, reinterpret_cast<cudaStream_t>(stream));
    return (int)cudaGetLastError();
}

int wkh_output_wgrad(const long long* g, const float* params, const float* mix, const float* feat, float* dpre, float* grads, float scale,
                     float* part, long long part_bytes, void* stream) {
    OutputLaunch O;
    output_from(g, 1.f, params, mix, feat, &O);
    O.dpre = dpre;
    if (part_bytes < (long long)output_wgrad_partial_bytes(O)) { g_err = "output partial arena too small"; return -1; }
    launch_output_wgrad(O, grads, part, scale, reinterpret_cast<cudaStream_t>(stream));
    return (int)cudaGetLastError();
}

long long wkh_upsample_partial_bytes(int batch, int C) { return (long long)upsample_dvar_partial_bytes(batch, C); }

// g: batch, N, nmid, C, mid_mode; count: the CTA counter of the interp-gradient sum (0 before; the launch leaves it 0)
int wkh_upsample_bwd(const long long* g, const float* due, const float* dmid, const float* x, float* gx, const float* blend, float* dvar,
                     float scale, float* part, long long part_bytes, unsigned* count, void* stream) {
    UpsampleBwdLaunch U;
    memset(&U, 0, sizeof(U));
    U.batch = (int)g[0]; U.N = (int)g[1]; U.nmid = (int)g[2]; U.C = (int)g[3]; U.mid_mode = (int)g[4];
    U.due = due; U.dmid = dmid; U.x = x; U.gx = gx; U.blend = blend; U.dvar = dvar; U.scale = scale; U.part = part; U.count = count;
    if (dvar && (!blend || !count || part_bytes < (long long)upsample_dvar_partial_bytes(U.batch, U.C))) { g_err = "dvar needs blend, a counter and a partial arena"; return -1; }
    launch_upsample_bwd(U, reinterpret_cast<cudaStream_t>(stream));
    return (int)cudaGetLastError();
}

int wkh_sigmoid(const float* x, float* y, int n, void* stream) {
    launch_sigmoid(x, y, n, reinterpret_cast<cudaStream_t>(stream));
    return (int)cudaGetLastError();
}

// state == null: lr_t as given (folded on the host); else lr_t = lr * sqrt(1 - state[1]) / (1 - state[0]) on the device, then advanced
int wkh_adam(float* p, const float* g, float* m, float* v, long long n, float lr, float b1, float b2, float eps, float* state, void* stream) {
    launch_adam(p, g, m, v, n, lr, b1, b2, eps, state, reinterpret_cast<cudaStream_t>(stream));
    return (int)cudaGetLastError();
}

int wkh_gather_windows(const float* padded, long long n_padded, const long long* starts, int n_windows, int T_in, int C, float* out,
                       void* stream) {
    launch_gather_windows(padded, n_padded, starts, n_windows, T_in, C, out, reinterpret_cast<cudaStream_t>(stream));
    return (int)cudaGetLastError();
}

int wkh_scatter_windows(const float* outs, const long long* starts, int n_windows, int n_sources, int T_out, int C, float* preds,
                        long long n_frames, void* stream) {
    launch_scatter_windows(outs, starts, n_windows, n_sources, T_out, C, preds, n_frames, reinterpret_cast<cudaStream_t>(stream));
    return (int)cudaGetLastError();
}

}  // extern "C"
