// engine.cu - C ABI (include/wun.h) of the Wave-U-Net engine (H100, sm_90a): turns the host plan into kernel launches.
//
// Forward  = get_output             /root/reference/Models/UnetAudioSeparator.py:85-144
// Backward = what tf.gradients builds for AdamOptimizer.minimize, /root/reference/Training.py:77
// (the reference has no backward source; the derivation is in DESIGN.md "Backward").
#include <cuda_runtime.h>
#include <math.h>
#include <stdarg.h>
#include <stdlib.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <map>
#include <string>
#include <vector>

#include "../../include/wun.h"
#include "kernels.h"
#include "launch.h"
#include "plan.h"
#include "kernels_umma.h"

using namespace wun;

static thread_local std::string g_err;
static int set_err(int code, const std::string& m) { g_err = m; return code; }
// the spectrogram engine (spec.cu) reports through the same wun_last_error()
int wun::set_last_error(int code, const char* msg) { return set_err(code, msg); }

#define WUN_CUDA_OK(expr)                                                                  \
    do {                                                                                   \
        cudaError_t e__ = (expr);                                                          \
        if (e__ != cudaSuccess)                                                            \
            return set_err(WUN_E_CUDA, std::string(#expr) + ": " + cudaGetErrorString(e__)); \
    } while (0)

namespace {

struct DgradClass {
    int plane;            // forward plane whose gradient this class produces
    int r_lo, r_hi;       // rows written
    int acc_lo, acc_hi;   // rows accumulated into an earlier write
};

struct OpBackward {
    std::vector<DgradClass> dgrad;   // empty: no input gradient needed (down0)
};

// The A/B switches (DESIGN.md section 9), read from the environment once per handle, when it is created (read_options)
struct Options {
    bool umma_enabled = true;            // tensor-core path on (WUN_DISABLE_UMMA=1 turns it off, for A/B tests)
    bool umma_pass[3] = {true, true, true};   // per pass (fwd, dgrad, wgrad): WUN_UMMA_FWD=0 / WUN_UMMA_DGRAD=0 / WUN_UMMA_WGRAD=0
    bool use_side = true;                // WUN_SIDE_STREAM=0 disables
    bool first_fast = true;              // dedicated first-layer kernels (kernels_first.cu); WUN_FIRST_LAYER=0 = generic path
    bool bulk_wgrad = true;              // split pass + bulk-copy-fed tensor-core wgrad; WUN_BULK_WGRAD=0 = converter-fed kernel
    bool dgrad_par = true;               // WUN_DGRAD_PAR=0: a dgrad's second launch stays on the caller's stream
    // split passes run one layer AHEAD of the wgrad kernels, on their own stream, into a double-buffered arena: the split pass is
    // DRAM-bound, the wgrad kernel L2 / tensor bound, so they overlap well (WUN_SPLIT_AHEAD=0: same stream, one arena half)
    bool split_ahead = true;
    bool first_tail = true;              // first-layer weight gradient on the split stream (build_wgrad); WUN_FIRST_TAIL=0 disables
    // weight packs are hoisted off the critical path: a training step enqueues every pack kernel on the side stream first (they
    // only depend on the parameters), then everything else; inference and the debug hooks pack inline.  WUN_PACK_EVENTS=0: the
    // forward convs wait for all packs instead of each for its own
    bool pack_events_on = true;
    bool pair_fwd = true;                // pair-merged forward classes of the up blocks; WUN_PAIR_FWD=0 disables
    int pair_dgrad = 4;                  // pair-merged dgrad classes (launch.h OutView::pairC); WUN_PAIR_DGRAD=0 off, 1 all, 2 down blocks only,
                                         // 3 up blocks only, 4 (default) down blocks whose merged width still takes the fused-N MMAs (2C <= 64)
    int pair_min_ctas = 120;             // WUN_PAIR_MIN_CTAS
    // output layer in the last up block's conv epilogue (kernels_umma.h OutputFuse).  WUN_OUT_FUSE: 0 = separate kernels, 1 (default) =
    // estimates + loss + dL/dpre + the gradient w.r.t. the features fused, the output convs' weight gradient as its own launch on
    // the wgrad stream (off the critical path), 2 = the weight gradient in the epilogue too (measured slower: it serialises
    // ~650 shuffle-reduction instructions per row tile on the four epilogue warps)
    int out_fuse_mode = 1;
    int split_colsum = 1;                // bias column sums in the split pass (build_wgrad); WUN_SPLIT_COLSUM=0 separate launches, 2 few-row layers only
};

static Options read_options() {
    auto on = [](const char* name) { const char* v = getenv(name); return !(v && v[0] == '0'); };   // off only for "0..."
    auto num = [](const char* name, int def) { const char* v = getenv(name); return v ? atoi(v) : def; };
    Options o;
    const char* dis = getenv("WUN_DISABLE_UMMA");
    o.umma_enabled = !(dis && dis[0] == '1');
    o.umma_pass[0] = on("WUN_UMMA_FWD"); o.umma_pass[1] = on("WUN_UMMA_DGRAD"); o.umma_pass[2] = on("WUN_UMMA_WGRAD");
    o.use_side = on("WUN_SIDE_STREAM");
    o.first_fast = on("WUN_FIRST_LAYER");
    o.bulk_wgrad = on("WUN_BULK_WGRAD");
    o.dgrad_par = on("WUN_DGRAD_PAR");
    o.split_ahead = on("WUN_SPLIT_AHEAD");
    o.first_tail = on("WUN_FIRST_TAIL");
    o.pack_events_on = on("WUN_PACK_EVENTS");
    o.pair_fwd = on("WUN_PAIR_FWD");
    o.pair_dgrad = num("WUN_PAIR_DGRAD", 4);
    o.pair_min_ctas = num("WUN_PAIR_MIN_CTAS", 120);
    o.out_fuse_mode = num("WUN_OUT_FUSE", 1);
    o.split_colsum = num("WUN_SPLIT_COLSUM", 1);
    return o;
}

// Where one call's regions lie in its workspace, in this order: the activations (float offsets per tensor from the base; -1 = not
// allocated in this kind of call), the weight packs, then the training scratch: the split arena (two halves; bulk-fed wgrad only),
// the per-CTA sums of the first layer's and of the output layer's weight gradients, the CTA counters of the loss and interp-gradient
// sums ([0] loss, [1] interp; zeroed at the start of every training step's output layer), the per-CTA loss sums and the per-CTA
// interp-gradient sums (each added up in a fixed order).  Byte offsets from the base; `end` = the bytes a call needs.
struct WsMap {
    std::vector<int64_t> act;
    int64_t packs = 0, split[2] = {0, 0}, first_part = 0, out_part = 0, counters = 0, loss_part = 0, dvar_part = 0, end = 0;
};

// One engine call's inputs: the caller's buffers and stream, the batch and the workspace map.  The calls that only build a launch
// list (counts, descriptions, the create-time sizes) have null or fake buffers and no stream.
struct Call {
    const float* params = nullptr;
    const float* mix = nullptr;
    float* ws = nullptr;
    cudaStream_t stream = nullptr;
    int batch = 0;
    WsMap map;
};

}  // namespace

// The streams a launch record goes to: the caller's; ST_SIDE: weight-gradient kernels (and a training step's weight packs) run
// on an internal side stream, concurrently with the dgrad chain on the caller's stream; ST_SPLIT: the split passes (see
// Options::split_ahead); ST_HELPER: a dgrad with two launches (the up blocks: skip pair and upsampled pair have different
// widths) runs the second one on this helper stream, concurrently with the first: both read the same gradient planes and write
// different tensors, and in the deep layers neither fills the GPU (WUN_DGRAD_PAR=0 disables)
enum StreamRole : uint8_t { ST_CALLER, ST_SIDE, ST_SPLIT, ST_HELPER };
// Event pools.  EV_PAR: fork / join pairs, one pair per use inside a call (graph capture needs distinct events); EV_PACK: one
// event per FORWARD weight pack, so that forward conv i waits for pack i only instead of for all ~60 packs of the step (the
// backward convs still wait for the single EV_PACKS event; WUN_PACK_EVENTS=0 disables); EV_FIRST_DONE: first-layer weight
// gradient on the split stream; EV_BUCKET: bucket k is recorded once every gradient of the bucket is final
enum EventPool : uint8_t { EV_NONE, EV_FORK, EV_PAR, EV_SPLIT_DONE, EV_WG_DONE, EV_PACK, EV_JOIN, EV_PACKS, EV_FIRST_DONE, EV_BUCKET,
                           kEventPools };

enum OpKind : uint8_t {
    OP_SIGMOID, OP_FIRST_FWD, OP_CONV, OP_PACK, OP_UMMA_CONV, OP_COUNTERS, OP_OUTPUT_FWD, OP_OUTPUT_WGRAD, OP_OUTPUT_DGRAD,
    OP_UPSAMPLE_BWD, OP_FIRST_WGRAD, OP_COLSUM, OP_WGRAD, OP_WGRAD_UMMA, OP_SPLIT, OP_WGRAD_BULK, OP_WGRAD_REDUCE,   // kernels + memset
    OP_RECORD, OP_WAIT,          // event record / stream wait
    OP_MAKE                      // create a stream (+ the side stream's join / packs events) or pool events, if missing
};

// One runtime operation of an engine call, with the by-value block its launcher takes.
struct Op {
    OpKind kind;
    StreamRole stream;
    EventPool pool;
    bool early;                  // a training step's weight packs and their events: issued before everything else
    int index;                   // RECORD / WAIT: event in the pool; MAKE: events the pool must hold; WGRAD: group of the layer
    int layer, pass;             // pass 0 forward, 1 dgrad, 2 wgrad
    union {
        struct { const float* x; float* y; int n; } sig;
        FirstLayer first;
        ConvLaunch conv;
        UmmaPackLaunch pack;
        struct { UmmaLaunch U; ConvLaunch L; UmmaChoice ch; OutputFuse fuse; bool fused; } umma;
        unsigned* counters;
        struct { OutputLaunch O; float* grads; float* part; float scale; float* gfeat; } out;
        UpsampleBwdLaunch up;
        FirstWgrad fw;
        struct { PlaneView V; int batch; float scale; float* out; } colsum;
        WgradLaunch wg;
        struct { UmmaWgradLaunch U; WgSplit S; SplitJobs J; } wgu;   // WGRAD_UMMA: U; SPLIT: J; WGRAD_BULK: U, S; WGRAD_REDUCE: U, J
    };
    Op() {}
};

struct WunHandle {
    Plan plan;
    std::vector<OpBackward> bwd_down, bwd_up;
    OpBackward bwd_bottleneck;
    Options opt;
    std::vector<std::string> kernel_used;   // [layer*3 + pass] -> "simt" | "umma" (from the launch list built at create time)
    cudaStream_t streams[4] = {};        // by StreamRole, created where a call first needs them (ST_CALLER: unused)
    std::vector<cudaEvent_t> events[kEventPools];   // by EventPool, created where a call first needs them
    // sizes from the batch-1 training launch list built at create time
    size_t split_item_bytes = 0;         // per batch item: largest split arena any layer's wgrad needs
    size_t wg_partial_bytes = 0;         // largest partial-tile scratch of a layer's wgrad (any batch)
    size_t out_part_bytes = 0;           // the output layer's per-CTA weight-gradient sums (any batch)
    size_t arena_sum = 0;                // total pack bytes of one forward+backward
    // data-parallel overlap: gradient buckets in PRODUCTION order (output layer first, down0 last); bucket k = flat offsets
    // >= bucket_first[k] (and below bucket k-1's)
    std::vector<int64_t> bucket_first;
    std::vector<Op> ops;                 // storage of the calls' launch lists, kept from call to call: no allocation per call
};

// ------------------------------------------------------------------------------------------------
// planning helpers
// ------------------------------------------------------------------------------------------------
static void touched_range(const ConvOp& op, int plane, int* lo, int* hi) {
    int l = 1 << 30, h = -(1 << 30);
    for (const auto& c : op.classes) {
        if (c.m_hi <= c.m_lo) continue;
        for (const auto& t : c.terms)
            if (t.plane == plane) {
                l = std::min(l, c.m_lo + t.d);
                h = std::max(h, c.m_hi - 1 + t.d + 1);
            }
    }
    const ViewSpec& v = op.planes[plane];
    l = std::max(l, v.r_lo);
    h = std::min(h, v.r_hi);
    if (h < l) h = l;
    *lo = l; *hi = h;
}

static inline int ceil_div_floor(int a, int s) {   // ceil(a / s) for s > 0, any sign of a
    return (a >= 0) ? (a + s - 1) / s : -((-a) / s);
}

static void plan_backward(WunHandle* h) {
    Plan& P = h->plan;
    const int L = P.cfg.num_layers;
    std::map<int, std::pair<int, int>> written;   // grad tensor -> tensor-row range written so far
    auto plan_op = [&](const ConvOp& op, OpBackward* ob, bool is_up) {
        for (size_t p = 0; p < op.planes.size(); ++p) {
            const int gt = op.plane_grad_tensor[p];
            if (gt == -2) continue;
            const ViewSpec& v = op.planes[p];
            DgradClass dc;
            dc.plane = (int)p;
            if (is_up && p == 0) touched_range(op, 0, &dc.r_lo, &dc.r_hi);
            else { dc.r_lo = v.r_lo; dc.r_hi = v.r_hi; }
            dc.acc_lo = dc.acc_hi = 0;
            auto it = written.find(gt);
            if (it != written.end() && gt != P.t_gue && gt != P.t_gmid) {
                const int wlo = it->second.first, whi = it->second.second;
                dc.acc_lo = ceil_div_floor(wlo - v.row_offset, v.row_step);
                dc.acc_hi = ceil_div_floor(whi - v.row_offset, v.row_step);
            }
            ob->dgrad.push_back(dc);
        }
        // record writes after the whole op (both parities of one tensor belong to the same op)
        for (const auto& dc : ob->dgrad) {
            const ViewSpec& v = op.planes[dc.plane];
            const int gt = op.plane_grad_tensor[dc.plane];
            if (dc.r_hi <= dc.r_lo) continue;
            int lo = v.row_offset + dc.r_lo * v.row_step;
            int hi = v.row_offset + (dc.r_hi - 1) * v.row_step + 1;
            auto it = written.find(gt);
            if (it == written.end()) written[gt] = {lo, hi};
            else it->second = {std::min(it->second.first, lo), std::max(it->second.second, hi)};
        }
    };
    h->bwd_up.assign(L, OpBackward());
    h->bwd_down.assign(L, OpBackward());
    for (int i = L - 1; i >= 0; --i) plan_op(P.up[i], &h->bwd_up[i], true);
    plan_op(P.bottleneck, &h->bwd_bottleneck, false);
    for (int i = L - 1; i >= 0; --i) plan_op(P.down[i], &h->bwd_down[i], false);
}

constexpr int64_t kCounterBytes = 256;     // the CTA counters of the loss and interp-gradient sums

static WsMap ws_map(const WunHandle* h, int64_t B, bool training) {
    const Plan& P = h->plan;
    WsMap m;
    m.act.assign(P.tensors.size(), -1);
    int64_t cur = 0;
    for (size_t i = 0; i < P.tensors.size(); ++i) {
        const TensorSpec& t = P.tensors[i];
        if (t.training_only && !training) continue;
        int64_t n = t.rows * t.C * (t.per_batch ? B : 1);
        m.act[i] = cur;
        cur += (n + 63) / 64 * 64;
    }
    m.packs = (cur + 64) * (int64_t)sizeof(float);
    m.end = m.packs + (int64_t)h->arena_sum;
    auto region = [&](int64_t bytes) { const int64_t at = m.end; if (training) m.end += bytes; return at; };   // inference: none
    // split arena: each half holds the split arrays of one layer's wgrad, then its partial tiles, from a 256-byte boundary
    const int64_t half = (int64_t)h->split_item_bytes * B + 256 * (kSplitMaxJobs + 1) + (int64_t)h->wg_partial_bytes + 256;
    const int64_t split = region((h->opt.bulk_wgrad && h->split_item_bytes) ? 2 * half : 0);
    m.split[0] = (split + 255) / 256 * 256;
    m.split[1] = (split + half + 255) / 256 * 256;
    m.first_part = region((int64_t)first_wgrad_partial_bytes((int)B));
    m.out_part = region((int64_t)h->out_part_bytes);
    m.counters = region(kCounterBytes);
    m.loss_part = region((int64_t)output_loss_partial_bytes((int)B, (int)P.T_out));
    int C = 0;      // interp gradients: one level at a time, all on the caller's stream (none without learned upsampling)
    for (int i = 0; i < P.cfg.num_layers; ++i)
        if (P.ups[i].interp_param >= 0) C = std::max(C, P.ups[i].C);
    m.dvar_part = region(C ? (int64_t)upsample_dvar_partial_bytes((int)B, C) : 0);
    return m;
}

// ------------------------------------------------------------------------------------------------
// materialisation of launch blocks
// ------------------------------------------------------------------------------------------------
static const float* tensor_ptr(const Call& call, int tensor) {
    if (tensor == TENSOR_MIX) return call.mix;
    return call.ws + call.map.act[tensor];
}

static uint8_t* ws_at(const Call& call, int64_t offset) { return reinterpret_cast<uint8_t*>(call.ws) + offset; }

static void tensor_geom(const WunHandle* h, int tensor, int64_t* rows, int* C, bool* per_batch) {
    if (tensor == TENSOR_MIX) { *rows = h->plan.T_in; *C = h->plan.cfg.num_channels; *per_batch = true; return; }
    const TensorSpec& t = h->plan.tensors[tensor];
    *rows = t.rows; *C = t.C; *per_batch = t.per_batch;
}

static PlaneView make_plane(const WunHandle* h, const Call& call, const ViewSpec& v) {
    PlaneView p;
    memset(&p, 0, sizeof(p));
    int64_t rows; int C; bool pb;
    tensor_geom(h, v.tensor, &rows, &C, &pb);
    p.base = tensor_ptr(call, v.tensor) + (long long)v.row_offset * C;
    p.bstride = pb ? rows * C : 0;
    p.rstride = v.row_step * C;
    p.r_lo = v.r_lo; p.r_hi = v.r_hi; p.C = v.C;
    p.kind = v.kind; p.mid_mode = v.mid_mode; p.xrows = v.xrows;
    p.blend = (v.blend_tensor >= 0) ? tensor_ptr(call, v.blend_tensor) : nullptr;
    return p;
}

// the same geometry as `v`, but on another tensor (gradient twin / scratch) with explicit batch stride
static PlaneView make_plane_on(const Call& call, const ViewSpec& v, int tensor, long long bstride, int r_lo, int r_hi) {
    PlaneView p;
    memset(&p, 0, sizeof(p));
    p.base = tensor_ptr(call, tensor) + (long long)v.row_offset * v.C;
    p.bstride = bstride;
    p.rstride = v.row_step * v.C;
    p.r_lo = r_lo; p.r_hi = r_hi; p.C = v.C;
    p.kind = PLANE_DIRECT;
    return p;
}

static long long view_bstride(const WunHandle* h, const ViewSpec& v) {
    int64_t rows; int C; bool pb;
    tensor_geom(h, v.tensor, &rows, &C, &pb);
    return rows * C;
}

// ------------------------------------------------------------------------------------------------
// launch list: build_* turn one engine call into records without any CUDA call, issue() makes the runtime calls
// ------------------------------------------------------------------------------------------------
struct Build {                   // the walk over the plan that appends one call's records
    const WunHandle* h;
    const Call& call;
    std::vector<Op>& ops;
    bool train = false;          // a training step: the CTA counters of the loss sums are zeroed
    bool hoist = false;          // weight packs on the side stream ahead of the step (training, side stream, tensor cores)
    bool dgrad_fork = false;     // a dgrad's second launch may go to the helper stream
    StreamRole ws = ST_CALLER;   // stream of the weight-gradient launches
    float* grads = nullptr;      // training: gradient buffer / scale, known to the forward pass for the fused epilogue
    float scale = 1.f;
    const OutputFuse* fuse = nullptr;   // around the last up block's forward conv
    bool out_fused = false;      // that conv carried the output layer: no output_fwd / output_dgrad / output_wgrad launches
    int layer = -1, pass = -1;
    int pack_idx = 0, fork_used = 0, par_used = 0, wg_index = 0, bucket_next = 0;
    bool packs_pending = false;  // the caller's stream has not yet waited for the hoisted packs
    bool first_pending = false;  // the first-layer weight gradient runs on the split stream
    // sizes the workspace needs for these launches (pack_sum: also the bump pointer into the pack arena)
    size_t pack_sum = 0, split_item = 0, wg_partial = 0, out_part = 0;
};

static Op& add(Build& b, OpKind kind, StreamRole stream = ST_CALLER, EventPool pool = EV_NONE, int index = 0) {
    b.ops.emplace_back();
    Op& o = b.ops.back();
    o.kind = kind; o.stream = stream; o.pool = pool; o.early = false; o.index = index; o.layer = b.layer; o.pass = b.pass;
    return o;
}

// Every plane convolution goes through here: tensor cores (wgmma) when the launch is eligible, CUDA cores otherwise.
// It reserves at least `pack_floor` pack bytes: the pair-merge decision depends on the batch (folded or not) but the arena is
// sized by a batch-1 list, so both forms' bytes count.
static int add_conv(Build& b, const ConvLaunch& L, StreamRole s, size_t pack_floor) {
    const WunHandle* h = b.h;
    UmmaChoice ch;
    if (!(h->opt.umma_enabled && h->opt.umma_pass[b.pass] && umma_plan_from_conv(L, &ch))) {
        add(b, OP_CONV, s).conv = L;
        return WUN_OK;
    }
    const size_t bytes = std::max(ch.pack_bytes, pack_floor);
    uint8_t* arena = ws_at(b.call, b.call.map.packs + b.pack_sum);
    b.pack_sum += bytes;
    UmmaLaunch U;
    Op& pk = add(b, OP_PACK, b.hoist ? ST_SIDE : s);
    pk.early = b.hoist;
    if (umma_build(L, ch, arena, &U, &pk.pack) != cudaSuccess) return set_err(WUN_E_CUDA, "tensor-core conv launch: too many pack jobs");
    if (h->opt.pack_events_on && b.pass == 0 && b.hoist) {     // forward conv i waits for pack i only
        const int idx = b.pack_idx++;
        add(b, OP_MAKE, ST_SIDE, EV_PACK, idx + 1).early = true;
        add(b, OP_RECORD, ST_SIDE, EV_PACK, idx).early = true;
        add(b, OP_WAIT, s, EV_PACK, idx);
    } else if (b.packs_pending) {   // first conv that needs ALL hoisted packs (with per-pack events: the first dgrad)
        add(b, OP_WAIT, s, EV_PACKS);
        b.packs_pending = false;
    }
    Op& o = add(b, OP_UMMA_CONV, s);
    o.umma.U = U; o.umma.L = L; o.umma.ch = ch;
    o.umma.fused = b.fuse && umma_output_fusable(L, ch, b.fuse->O);
    if (o.umma.fused) { o.umma.fuse = *b.fuse; b.out_fused = true; }
    return WUN_OK;
}

// The first down block in the form kernels_first.cu wants, if the op has exactly the shape plan.cpp builds for it: input =
// the caller's mix in two parity planes, class 0 = even full-rate rows -> dec0, class 1 = odd rows of the skip window -> odd0.
static bool first_layer_desc(const WunHandle* h, const Call& call, const ConvOp& op, FirstLayer* F) {
    if (!h->opt.first_fast || op.planes.size() != 2 || op.classes.size() != 2) return false;
    const ViewSpec& p0 = op.planes[0];
    const ViewSpec& p1 = op.planes[1];
    if (p0.tensor != TENSOR_MIX || p1.tensor != TENSOR_MIX || p0.row_step != 2 || p1.row_step != 2 || p0.row_offset != 0 ||
        p1.row_offset != 1 || p0.kind != PLANE_DIRECT || p1.kind != PLANE_DIRECT) return false;
    const int C = h->plan.cfg.num_channels;
    if (op.cin_tot != C || !first_layer_supported(C, op.cout, op.k)) return false;
    const ClassSpec& c0 = op.classes[0];
    const ClassSpec& c1 = op.classes[1];
    if (c0.out.row_step != 1 || c1.out.row_step != 1 || c0.out.row_offset != 0 || c1.out.row_offset != -c1.m_lo || c0.m_lo != 0) return false;
    if ((int)c0.terms.size() != op.k || (int)c1.terms.size() != op.k) return false;
    // tap j of class q reads full-rate x row 2m + q + j - pad:  2*d + plane = q + j - pad
    int pad = 0;
    for (const auto& t : c0.terms) if (t.tap == 0) pad = -(2 * t.d + t.plane);
    for (int q = 0; q < 2; ++q)
        for (const auto& t : op.classes[q].terms)
            if (2 * t.d + t.plane != q + t.tap - pad || t.coff != 0) return false;
    memset(F, 0, sizeof(*F));
    F->x = call.mix; F->x_bstride = (long long)h->plan.T_in * C; F->T = (int)h->plan.T_in;
    F->k = op.k; F->pad_left = pad;
    F->dec = const_cast<float*>(tensor_ptr(call, c0.out.tensor)); F->dec_bstride = view_bstride(h, c0.out); F->Td = c0.m_hi;
    F->odd = const_cast<float*>(tensor_ptr(call, c1.out.tensor)); F->odd_bstride = view_bstride(h, c1.out);
    F->mo_lo = c1.m_lo; F->mo_hi = c1.m_hi;
    F->W = call.params + h->plan.params[op.w_param].offset;
    F->bias = call.params + h->plan.params[op.b_param].offset;
    F->batch = call.batch;
    return true;
}

// Two classes of equal width -> one pair-merged class (launch.h OutView::pairC), or false if the pair does not qualify.
static bool merge_pair(const ConvLaunch& S, ConvLaunch* out) {
    if (S.ncls != 2 || S.N % 4 != 0 || 2 * S.N > 256) return false;
    const OutView& A = S.cls[0];
    const OutView& B = S.cls[1];
    if (A.m_hi <= A.m_lo || B.m_hi <= B.m_lo) return false;
    // worthwhile only when most rows exist in both classes (the union is what gets computed)
    const int lo = std::min(A.m_lo, B.m_lo), hi = std::max(A.m_hi, B.m_hi);
    if ((long long)(hi - lo) * 4 > 3LL * ((A.m_hi - A.m_lo) + (B.m_hi - B.m_lo))) return false;
    ConvLaunch M = S;
    M.ncls = 1; M.N = 2 * S.N; M.pairC = S.N; M.max_rows = hi - lo;
    OutView& O = M.cls[0];
    O = A;
    O.m_lo = lo; O.m_hi = hi;
    O.pairC = S.N;
    O.base2 = B.base; O.bstride2 = B.bstride; O.rstride2 = B.rstride; O.saved2 = B.saved;
    O.acc_lo2 = B.acc_lo; O.acc_hi2 = B.acc_hi;
    O.lo_h[0] = A.m_lo; O.hi_h[0] = A.m_hi; O.lo_h[1] = B.m_lo; O.hi_h[1] = B.m_hi;
    // union of the two classes' (plane, shift) terms
    int nt = 0;
    Term merged[kMaxTerms];
    for (int t = A.term_begin; t < A.term_end; ++t) { merged[nt] = S.terms[t]; merged[nt].woff2 = -1; ++nt; }
    for (int t = B.term_begin; t < B.term_end; ++t) {
        int f = -1;
        for (int u = 0; u < nt; ++u) if (merged[u].plane == S.terms[t].plane && merged[u].d == S.terms[t].d) f = u;
        if (f < 0) {
            if (nt >= kMaxTerms) return false;
            merged[nt] = S.terms[t]; merged[nt].woff = -1; merged[nt].woff2 = S.terms[t].woff; ++nt;
        } else {
            merged[f].woff2 = S.terms[t].woff;
        }
    }
    std::stable_sort(merged, merged + nt, [](const Term& a, const Term& b) {
        if (a.plane != b.plane) return a.plane < b.plane;
        return a.d < b.d;
    });
    for (int t = 0; t < nt; ++t) M.terms[t] = merged[t];
    O.term_begin = 0; O.term_end = nt;
    *out = M;
    return true;
}

// Measured (M4 batch 16, same box A/B): merged launches that fill the GPU win (up8..up11 forward 78/66/95/115 -> 56/58/67/83 us),
// a merged launch with far fewer CTAs than SMs loses to the two-class form (up7 forward 64 -> 72 us at 80 CTAs).
static bool pair_worthwhile(const WunHandle* h, const ConvLaunch& M, const UmmaChoice& ch) {
    long long ctas = 0;
    for (int q = 0; q < M.ncls; ++q)
        ctas += (long long)((M.cls[q].m_hi - M.cls[q].m_lo + ch.MT * 128 - 1) / (ch.MT * 128)) * ch.nsplit * M.batch;
    return ctas >= h->opt.pair_min_ctas;
}

static int build_conv_forward(Build& b, const ConvOp& op, int layer_index) {
    const WunHandle* h = b.h;
    const Call& call = b.call;
    b.layer = layer_index; b.pass = 0;
    if (layer_index == 0) {
        FirstLayer F;
        if (first_layer_desc(h, call, op, &F)) {
            add(b, OP_FIRST_FWD).first = F;
            return WUN_OK;
        }
    }
    ConvLaunch L;
    memset(&L, 0, sizeof(L));
    L.nplanes = (int)op.planes.size();
    for (int p = 0; p < L.nplanes; ++p) L.planes[p] = make_plane(h, call, op.planes[p]);
    L.ncls = (int)op.classes.size();
    int nt = 0, max_rows = 0;
    for (int q = 0; q < L.ncls; ++q) {
        const ClassSpec& c = op.classes[q];
        OutView& o = L.cls[q];
        PlaneView ov = make_plane(h, call, c.out);
        o.base = const_cast<float*>(ov.base); o.bstride = ov.bstride; o.rstride = ov.rstride;
        o.m_lo = c.m_lo; o.m_hi = c.m_hi; o.saved = nullptr; o.acc_lo = o.acc_hi = 0;
        o.term_begin = nt;
        for (const auto& t : c.terms) {
            if (nt >= kMaxTerms) return set_err(WUN_E_INVALID, "too many conv terms");
            L.terms[nt++] = {t.plane, t.d, (t.tap * op.cin_tot + t.coff) * op.cout};
        }
        o.term_end = nt;
        max_rows = std::max(max_rows, c.m_hi - c.m_lo);
    }
    L.N = op.cout; L.w_sk = op.cout; L.w_sn = 1;
    L.W = call.params + h->plan.params[op.w_param].offset;
    L.bias = call.params + h->plan.params[op.b_param].offset;
    L.epilogue = EPI_BIAS_LRELU; L.batch = call.batch; L.max_rows = max_rows;
    // the even / odd output rows of an up block (and of the bottleneck) read the same planes at the same shifts: one
    // pair-merged class of 2*cout columns (out tensor viewed as [B, rows/2, 2*cout]) - 6+6 taps instead of 2 x (5+5)
    ConvLaunch M;
    size_t pack_floor = 0;
    if (h->opt.pair_fwd && L.ncls == 2 && h->opt.umma_enabled && h->opt.umma_pass[0] && merge_pair(L, &M)) {
        UmmaChoice ch0, ch;
        const bool ok0 = umma_plan_from_conv(L, &ch0), ok1 = umma_plan_from_conv(M, &ch);
        if (ok0 && ok1) {
            pack_floor = std::max(ch0.pack_bytes, ch.pack_bytes);
            if (pair_worthwhile(h, M, ch)) L = M;
        }
    }
    return add_conv(b, L, ST_CALLER, pack_floor);
}

// dgrad: one class per forward input plane that needs a gradient; the forward classes' gradient
// tensors become the input planes.
static int build_dgrad(Build& b, const ConvOp& op, const OpBackward& ob, int layer_index) {
    if (ob.dgrad.empty()) return WUN_OK;
    const WunHandle* h = b.h;
    const Call& call = b.call;
    b.layer = layer_index; b.pass = 1;
    const Plan& P = h->plan;
    ConvLaunch L;
    memset(&L, 0, sizeof(L));
    L.nplanes = (int)op.classes.size();
    for (int q = 0; q < L.nplanes; ++q) {
        const ClassSpec& c = op.classes[q];
        L.planes[q] = make_plane_on(call, c.out, P.grad_twin[c.out.tensor], view_bstride(h, c.out), c.m_lo, c.m_hi);
    }
    L.ncls = (int)ob.dgrad.size();
    int nt = 0, max_rows = 0;
    for (int k = 0; k < L.ncls; ++k) {
        const DgradClass& dc = ob.dgrad[k];
        const ViewSpec& v = op.planes[dc.plane];
        const int gt = op.plane_grad_tensor[dc.plane];
        long long bs = view_bstride(h, v);
        if (gt == P.t_gmid) bs = (long long)(v.r_hi - v.r_lo) * v.C;   // [B, nmid, C]
        PlaneView ov = make_plane_on(call, v, gt, bs, dc.r_lo, dc.r_hi);
        OutView& o = L.cls[k];
        o.base = const_cast<float*>(ov.base); o.bstride = ov.bstride; o.rstride = ov.rstride;
        o.m_lo = dc.r_lo; o.m_hi = dc.r_hi;
        o.saved = op.plane_slope[dc.plane] ? make_plane(h, call, v).base : nullptr;
        o.acc_lo = dc.acc_lo; o.acc_hi = dc.acc_hi;
        o.term_begin = nt;
        for (int q = 0; q < (int)op.classes.size(); ++q)
            for (const auto& t : op.classes[q].terms)
                if (t.plane == dc.plane) {
                    if (nt >= kMaxTerms) return set_err(WUN_E_INVALID, "too many dgrad terms");
                    L.terms[nt++] = {q, -t.d, (t.tap * op.cin_tot + t.coff) * op.cout};
                }
        // sort by (plane, d)
        std::stable_sort(L.terms + o.term_begin, L.terms + nt, [](const Term& a, const Term& b) {
            if (a.plane != b.plane) return a.plane < b.plane;
            return a.d < b.d;
        });
        o.term_end = nt;
        max_rows = std::max(max_rows, dc.r_hi - dc.r_lo);
        L.N = v.C;   // all classes of one op's dgrad have... (checked below)
    }
    // classes may differ in channel count (skip vs upsampled planes): launch per distinct N
    std::vector<int> done(L.ncls, 0);
    int n_launched = 0;
    // recorded on the caller's stream before the first launch (see `par` below)
    const bool fork = b.dgrad_fork && !b.packs_pending && L.ncls > 2;
    const int ev_fork = b.par_used;
    if (fork) {
        add(b, OP_MAKE, ST_CALLER, EV_PAR, b.par_used + 2);
        add(b, OP_RECORD, ST_CALLER, EV_PAR, ev_fork);
    }
    for (int k = 0; k < L.ncls; ++k) {
        if (done[k]) continue;
        const int N = op.planes[ob.dgrad[k].plane].C;
        ConvLaunch S = L;
        S.ncls = 0; S.max_rows = 0;
        for (int k2 = k; k2 < L.ncls; ++k2)
            if (!done[k2] && op.planes[ob.dgrad[k2].plane].C == N) {
                S.cls[S.ncls++] = L.cls[k2];
                S.max_rows = std::max(S.max_rows, L.cls[k2].m_hi - L.cls[k2].m_lo);
                done[k2] = 1;
            }
        S.N = N; S.w_sk = 1; S.w_sn = op.cout;
        S.W = call.params + P.params[op.w_param].offset;
        S.bias = nullptr;
        // slope is per class (saved != null); classes without saved use EPI_PLAIN semantics via null check
        S.epilogue = EPI_SLOPE;
        S.batch = call.batch;
        if (S.max_rows <= 0) continue;
        // Pair merge: two classes of the same width (the even / odd input rows of a down block; the skip-even / skip-odd or
        // the copied / interpolated inputs of an up block) read the same gradient planes with the same row shifts.  As ONE
        // class of N = 2C columns every slab is staged once instead of twice and a tap costs one MMA instead of two (for
        // N <= 64 an MMA costs the same ~46 cycles whatever N is) - launch.h OutView::pairC.
        ConvLaunch M;
        // Measured (M4 batch 16, same-box A/B): down1 (2C = 48, fused-N MMAs) 368 -> 332 us; wider pairs lose the fused-N form and
        // got slower (down2 276 -> 317, down3 216 -> 250, down4 156 -> 183, up11 194 -> 215 us): their dgrad is bound by the
        // epilogue's slope / accumulate read-backs, not by slab fills or MMAs.
        const bool pair_on = h->opt.pair_dgrad == 1 || (h->opt.pair_dgrad == 2 && op.planes.size() == 2) || (h->opt.pair_dgrad == 3 && op.planes.size() == 4) ||
                             (h->opt.pair_dgrad == 4 && op.planes.size() == 2 && 2 * S.N <= 64);
        size_t pack_floor = 0;
        if (h->opt.pair_dgrad != 0 && S.ncls == 2 && h->opt.umma_enabled && h->opt.umma_pass[1] && merge_pair(S, &M)) {
            UmmaChoice ch0, ch;
            const bool ok0 = umma_plan_from_conv(S, &ch0), ok1 = umma_plan_from_conv(M, &ch);
            if (ok0 && ok1) {
                pack_floor = std::max(ch0.pack_bytes, ch.pack_bytes);
                if (pair_on && pair_worthwhile(h, M, ch)) S = M;
            }
        }
        // second (third ...) launch of this dgrad: on the helper stream, forked from the point the first launch was enqueued at
        const bool par = fork && n_launched > 0;
        if (par) {
            add(b, OP_MAKE, ST_HELPER);
            add(b, OP_MAKE, ST_HELPER, EV_PAR, b.par_used + 2);
            add(b, OP_WAIT, ST_HELPER, EV_PAR, ev_fork);
        }
        const int rc = add_conv(b, S, par ? ST_HELPER : ST_CALLER, pack_floor);
        if (rc != WUN_OK) return rc;
        if (par) {
            add(b, OP_RECORD, ST_HELPER, EV_PAR, b.par_used + 1);
            add(b, OP_WAIT, ST_CALLER, EV_PAR, b.par_used + 1);
            b.par_used += 2;
        }
        ++n_launched;
    }
    return WUN_OK;
}

static int build_wgrad(Build& b, const ConvOp& op, float* grads, float scale, int layer_index) {
    const WunHandle* h = b.h;
    const Call& call = b.call;
    const Plan& P = h->plan;
    b.layer = layer_index; b.pass = 2;
    // split passes ahead on their own stream (see Options::split_ahead)
    const bool ahead = h->opt.split_ahead && b.ws != ST_CALLER;
    if (layer_index == 0) {
        FirstWgrad FW;
        if (first_layer_desc(h, call, op, &FW.L)) {    // one launcher call: dW and db of both classes (per-CTA sums + their total)
            FW.part = reinterpret_cast<float*>(ws_at(call, call.map.first_part));
            FW.L.dec = const_cast<float*>(tensor_ptr(call, P.grad_twin[op.classes[0].out.tensor]));
            FW.L.odd = const_cast<float*>(tensor_ptr(call, P.grad_twin[op.classes[1].out.tensor]));
            FW.dW = grads + P.params[op.w_param].offset;
            FW.db = grads + P.params[op.b_param].offset;
            FW.scale = scale; FW.rows_per_cta = 0;
            // the CUDA-core first-layer gradient is the tail of the step: on the split stream it runs next to the second
            // block's tensor-core wgrad instead of behind it (joined at the end of build_backward)
            const bool tail_par = h->opt.first_tail && ahead;
            add(b, OP_FIRST_WGRAD, tail_par ? ST_SPLIT : b.ws).fw = FW;
            if (tail_par) {
                add(b, OP_MAKE, ST_SPLIT, EV_FIRST_DONE, 1);
                add(b, OP_RECORD, ST_SPLIT, EV_FIRST_DONE);
                b.first_pending = true;
            }
            return WUN_OK;
        }
    }
    // collect (class, plane) groups
    std::vector<WgradLaunch> groups;
    std::vector<PlaneView> class_dpre;
    for (const auto& c : op.classes) {
        if (c.m_hi <= c.m_lo) continue;
        PlaneView dpre = make_plane_on(call, c.out, P.grad_twin[c.out.tensor], view_bstride(h, c.out), c.m_lo, c.m_hi);
        class_dpre.push_back(dpre);                            // bias gradient = its column sums (fused into the split pass below)
        size_t i = 0;
        while (i < c.terms.size()) {
            WgradLaunch W;
            memset(&W, 0, sizeof(W));
            const int p = c.terms[i].plane;
            int dmin = c.terms[i].d;
            while (i < c.terms.size() && c.terms[i].plane == p && W.nterms < 8 && c.terms[i].d - dmin <= 15) {
                W.d[W.nterms] = c.terms[i].d;
                W.woff[W.nterms] = (c.terms[i].tap * op.cin_tot + c.terms[i].coff) * op.cout;
                ++W.nterms; ++i;
            }
            W.plane = make_plane(h, call, op.planes[p]);
            W.dpre = dpre;
            W.m_lo = c.m_lo; W.m_hi = c.m_hi;
            W.N = op.cout; W.w_sk = op.cout; W.w_sn = 1;
            W.dW = grads + P.params[op.w_param].offset;
            W.scale = scale; W.batch = call.batch;
            groups.push_back(W);
        }
    }
    // tensor cores: all groups of the layer in ONE launch
    bool use_umma = h->opt.umma_enabled && h->opt.umma_pass[2] && !groups.empty() && groups.size() <= (size_t)kWgMaxGroups;
    UmmaWgradLaunch U;
    if (use_umma) {
        memset(&U, 0, sizeof(U));
        U.ngroups = (int)groups.size(); U.batch = call.batch; U.dW = groups[0].dW;
        U.w_sp = op.cout; U.w_sg = 1; U.scale = scale;
        for (size_t g = 0; g < groups.size(); ++g) {
            WgGroup& G = U.grp[g];
            G.P = groups[g].plane; G.G = groups[g].dpre; G.m_lo = groups[g].m_lo; G.m_hi = groups[g].m_hi;
            G.ntaps = groups[g].nterms;
            for (int t = 0; t < G.ntaps; ++t) { G.d[t] = groups[g].d[t]; G.woff[t] = groups[g].woff[t]; }
        }
        use_umma = umma_plan_wgrad(&U);
    }
    float* bias_grad = grads ? grads + P.params[op.b_param].offset : nullptr;
    auto colsum_launches = [&]() {                        // bias gradient by its own kernel (paths without a split pass)
        for (const auto& dp : class_dpre) {
            Op& o = add(b, OP_COLSUM, b.ws);
            o.colsum.V = dp; o.colsum.batch = call.batch; o.colsum.scale = scale; o.colsum.out = bias_grad;
        }
    };
    if (use_umma) {
        const size_t split_need = h->opt.bulk_wgrad ? umma_plan_wgrad_split(U, 1, nullptr, nullptr, nullptr) : 0;
        const bool bulk = split_need > 0;                 // 0: too many distinct views for one split pass -> converter-fed kernel
        // Bias column sums inside the split pass instead of their own launches (WUN_SPLIT_COLSUM: 1 = default, 0 = separate colsum
        // launches, 2 = fused only for the layers with few rows).  History: while the dgrad chain was the critical path the separate
        // launches were 0.05 ms faster per step (they fill SMs the big-shared-memory kernels leave thread slots on); since the epilogue
        // work of round 2 the wgrad stream is the critical path and the fused form wins (5.45 -> 5.39 ms, wgrad family 2.52 -> 2.24 ms).
        int max_rows_g = 0;
        for (const auto& dp : class_dpre) max_rows_g = std::max(max_rows_g, dp.r_hi - dp.r_lo);
        const bool fused_colsum = h->opt.split_colsum == 1 || (h->opt.split_colsum == 2 && max_rows_g <= 4096);
        if (bulk) {      // + the split pass and the fixed-order reduction of the partial tiles / column sums
            b.split_item = std::max(b.split_item, split_need);
            b.wg_partial = std::max(b.wg_partial, umma_wgrad_partial_bytes(U));
        }
        if (!bulk || !fused_colsum) colsum_launches();
        if (!bulk) {
            add(b, OP_WGRAD_UMMA, b.ws).wgu.U = U;
            return WUN_OK;
        }
        uint8_t* arena = ws_at(call, call.map.split[ahead ? b.wg_index & 1 : 0]);
        // split arrays, then the partial tiles, in this half; the class-gradient views among the jobs also produce the
        // bias gradient (their column sums)
        decltype(Op::wgu) W;     // shared by the split pass, the wgrad and its reduction
        if (!umma_wgrad_bulk_setup(&U, call.batch, arena, class_dpre.data(), (int)class_dpre.size(), fused_colsum ? bias_grad : nullptr,
                                   scale, &W.S, &W.J))
            return set_err(WUN_E_INVALID, "wgrad split pass: class gradient view not among the split jobs");
        W.U = U;
        const StreamRole ss = ahead ? ST_SPLIT : b.ws;   // else the same stream as the wgrad: the arena is reused layer after layer
        const int k = ahead ? b.wg_index++ : 0;
        if (ahead) {
            add(b, OP_MAKE, ST_SPLIT, EV_SPLIT_DONE, k + 1);
            add(b, OP_MAKE, ST_SPLIT, EV_WG_DONE, k + 1);
            if (k >= 2) add(b, OP_WAIT, ST_SPLIT, EV_WG_DONE, k - 2);     // its arena half is free again
        }
        add(b, OP_SPLIT, ss).wgu = W;
        if (ahead) {
            add(b, OP_RECORD, ST_SPLIT, EV_SPLIT_DONE, k);
            add(b, OP_WAIT, b.ws, EV_SPLIT_DONE, k);
        }
        add(b, OP_WGRAD_BULK, b.ws).wgu = W;
        add(b, OP_WGRAD_REDUCE, b.ws).wgu = W;
        if (ahead) add(b, OP_RECORD, b.ws, EV_WG_DONE, k);
        return WUN_OK;
    }
    colsum_launches();
    for (size_t g = 0; g < groups.size(); ++g) add(b, OP_WGRAD, b.ws, EV_NONE, (int)g).wg = groups[g];
    return WUN_OK;
}

// fork: everything enqueued on the main stream so far is visible to the side stream
static void fork_side(Build& b) {
    if (b.ws == ST_CALLER) return;
    add(b, OP_MAKE, ST_CALLER, EV_FORK, b.fork_used + 1);
    add(b, OP_RECORD, ST_CALLER, EV_FORK, b.fork_used);
    add(b, OP_WAIT, ST_SIDE, EV_FORK, b.fork_used);
    if (b.h->opt.split_ahead) {
        add(b, OP_MAKE, ST_SPLIT);
        add(b, OP_WAIT, ST_SPLIT, EV_FORK, b.fork_used);
    }
    ++b.fork_used;
}

// Every gradient at a flat offset >= `ready_from` has been enqueued (side-stream work in order, main-stream work up to the
// last fork): record the events of the buckets this completes.  Called right after a fork (side waits for main) or at the end.
static void mark_grads_ready(Build& b, int64_t ready_from, StreamRole on) {
    const WunHandle* h = b.h;
    while (b.bucket_next < (int)h->bucket_first.size() && h->bucket_first[b.bucket_next] >= ready_from) {
        add(b, OP_RECORD, on, EV_BUCKET, b.bucket_next);
        ++b.bucket_next;
    }
}

static int64_t op_first_offset(const Plan& P, const ConvOp& op, const UpsampleSpec* us) {
    int64_t o = std::min(P.params[op.w_param].offset, P.params[op.b_param].offset);
    if (us && us->interp_param >= 0) o = std::min<int64_t>(o, P.params[us->interp_param].offset);
    return o;
}

static void fill_output_launch(const WunHandle* h, const Call& call, OutputLaunch* O, const float* targets, float* outputs,
                               float* loss, int training) {
    const Plan& P = h->plan;
    memset(O, 0, sizeof(*O));
    O->params = call.params;
    for (int s = 0; s < P.nconv; ++s) {
        O->w_off[s] = P.params[P.out_w_param[s]].offset;
        O->b_off[s] = P.params[P.out_b_param[s]].offset;
    }
    O->mix = call.mix;
    O->feat = tensor_ptr(call, P.t_feat);
    O->targets = targets;
    O->outputs = outputs;
    O->dpre = (call.map.act[P.t_dpre_out] >= 0) ? const_cast<float*>(tensor_ptr(call, P.t_dpre_out)) : nullptr;
    O->loss = loss;
    O->loss_part = loss ? reinterpret_cast<float*>(ws_at(call, call.map.loss_part)) : nullptr;
    O->loss_count = loss ? reinterpret_cast<unsigned*>(ws_at(call, call.map.counters)) : nullptr;
    O->batch = call.batch; O->T_in = (int)P.T_in; O->Tf = (int)P.Tf; O->T_out = (int)P.T_out;
    O->C = P.cfg.num_channels; O->F = P.cfg.num_initial_filters;
    O->nconv = P.nconv; O->K = P.cfg.num_sources;
    O->ofs = P.cfg.output_filter_size; O->pad_left = P.out_pad_left;
    O->crop_feat = P.crop_feat; O->crop_out = P.crop_out;
    O->output_type = P.cfg.output_type; O->activation = P.cfg.output_activation; O->training = training;
    O->inv_count = 1.0f / (float)((double)call.batch * P.T_out * P.cfg.num_channels * P.cfg.num_sources);
}

static int build_forward(Build& b, const float* targets, float* outputs, float* loss, int training) {
    const WunHandle* h = b.h;
    const Call& call = b.call;
    const Plan& P = h->plan;
    const int L = P.cfg.num_layers;
    for (int i = 0; i < L; ++i) {
        const UpsampleSpec& us = P.ups[i];
        if (us.interp_param >= 0) {
            Op& o = add(b, OP_SIGMOID);
            o.sig.x = call.params + P.params[us.interp_param].offset;
            o.sig.y = const_cast<float*>(tensor_ptr(call, us.wsig_tensor)); o.sig.n = us.C;
        }
    }
    int rc;
    for (int i = 0; i < L; ++i)
        if ((rc = build_conv_forward(b, P.down[i], i)) != WUN_OK) return rc;
    if ((rc = build_conv_forward(b, P.bottleneck, L)) != WUN_OK) return rc;
    OutputLaunch O;
    fill_output_launch(h, call, &O, targets, outputs, loss, training);
    OutputFuse OF;
    memset(&OF, 0, sizeof(OF));
    b.out_fused = false;
    for (int i = 0; i < L; ++i) {
        if (i == L - 1 && h->opt.out_fuse_mode != 0 && P.cfg.output_filter_size == 1) {
            // the output layer rides in this conv's epilogue when the planner picks the persistent kernel for it
            OF.O = O;
            const bool bw = targets != nullptr && b.grads != nullptr;
            OF.gfeat = bw ? const_cast<float*>(tensor_ptr(call, P.grad_twin[P.t_feat])) : nullptr;
            OF.grads = (bw && h->opt.out_fuse_mode == 2) ? b.grads : nullptr;
            OF.grad_scale = b.scale;
            const ConvOp& op = P.up[i];
            bool geom = op.classes.size() >= 1 && op.classes.size() <= (size_t)kMaxClasses;
            OF.t_step = geom ? op.classes[0].out.row_step : 0;
            for (size_t q = 0; geom && q < op.classes.size(); ++q) {
                const ViewSpec& v = op.classes[q].out;
                if (v.tensor != P.t_feat || v.row_step != OF.t_step || v.kind != PLANE_DIRECT) geom = false;
                OF.t0[q] = v.row_offset;
            }
            // a pair-merged launch has ONE class whose second half is the next frame: classes (even, odd rows) = offsets (0, 1)
            if (geom && op.classes.size() == 2 && !(OF.t0[0] == 0 && OF.t0[1] == 1 && OF.t_step == 2)) geom = false;
            if (geom && (targets == nullptr || bw)) b.fuse = &OF;       // (loss without gradients: the separate kernel)
        }
        rc = build_conv_forward(b, P.up[i], L + 1 + i);
        b.fuse = nullptr;
        if (rc != WUN_OK) return rc;
    }
    if (b.out_fused) return WUN_OK;
    // the loss and interp-gradient sums count their CTAs here; each sum's last CTA sets its counter back to 0, this makes
    // sure they start from 0 whatever the workspace held before
    if (b.train) add(b, OP_COUNTERS).counters = reinterpret_cast<unsigned*>(ws_at(call, call.map.counters));
    add(b, OP_OUTPUT_FWD).out.O = O;
    return WUN_OK;
}

static int build_backward(Build& b, const float* targets, float* grads, float scale) {
    const WunHandle* h = b.h;
    const Call& call = b.call;
    const Plan& P = h->plan;
    const int L = P.cfg.num_layers;
    int rc;
    b.ws = h->opt.use_side ? ST_SIDE : ST_CALLER;
    b.fork_used = b.hoist ? 1 : 0;
    if (h->opt.use_side) add(b, OP_MAKE, ST_SIDE);
    OutputLaunch O;
    fill_output_launch(h, call, &O, targets, nullptr, nullptr, 1);
    // fused forward (build_forward): dL/dpre and the feature gradient already exist; only the output convs' weight gradient is left
    // (mode 1), and it goes to the wgrad stream right after the first fork below
    const bool out_wgrad_late = b.out_fused && h->opt.out_fuse_mode != 2;
    b.out_part = std::max(b.out_part, output_wgrad_partial_bytes(O));
    decltype(Op::out) out;         // the output layer's weight gradient (either form) and the gradient w.r.t. the features
    out.O = O; out.grads = grads; out.part = reinterpret_cast<float*>(ws_at(call, call.map.out_part)); out.scale = scale;
    out.gfeat = const_cast<float*>(tensor_ptr(call, P.grad_twin[P.t_feat]));
    if (!b.out_fused) {
        add(b, OP_OUTPUT_WGRAD).out = out;
        add(b, OP_OUTPUT_DGRAD).out = out;
    }
    int64_t ready_from = h->plan.param_numel;      // lowest flat offset whose gradient is complete once the next fork is passed
    if (P.nconv > 0) ready_from = std::min<int64_t>(P.params[P.out_w_param[0]].offset, P.params[P.out_b_param[0]].offset);
    for (int i = L - 1; i >= 0; --i) {
        const ConvOp& op = P.up[i];
        fork_side(b);
        if (i == L - 1 && out_wgrad_late) add(b, OP_OUTPUT_WGRAD, b.ws).out = out;
        mark_grads_ready(b, ready_from, b.ws);
        ready_from = std::min(ready_from, op_first_offset(P, op, &P.ups[i]));
        if ((rc = build_wgrad(b, op, grads, scale, L + 1 + i)) != WUN_OK) return rc;
        if ((rc = build_dgrad(b, op, h->bwd_up[i], L + 1 + i)) != WUN_OK) return rc;
        const UpsampleSpec& us = P.ups[i];
        UpsampleBwdLaunch U;
        memset(&U, 0, sizeof(U));
        U.due = tensor_ptr(call, P.t_gue);
        U.dmid = tensor_ptr(call, P.t_gmid);
        U.x = tensor_ptr(call, us.src_tensor);
        U.gx = const_cast<float*>(tensor_ptr(call, P.grad_twin[us.src_tensor]));
        U.blend = (us.wsig_tensor >= 0) ? tensor_ptr(call, us.wsig_tensor) : nullptr;
        U.dvar = (us.interp_param >= 0) ? grads + P.params[us.interp_param].offset : nullptr;
        U.part = U.dvar ? reinterpret_cast<float*>(ws_at(call, call.map.dvar_part)) : nullptr;
        U.count = U.dvar ? reinterpret_cast<unsigned*>(ws_at(call, call.map.counters)) + 1 : nullptr;
        U.batch = call.batch; U.N = us.N; U.nmid = us.nmid; U.C = us.C; U.mid_mode = us.mid_mode; U.scale = scale;
        Op& o = add(b, OP_UPSAMPLE_BWD);
        o.up = U; o.layer = L + 1 + i;
    }
    fork_side(b);
    mark_grads_ready(b, ready_from, b.ws);
    ready_from = std::min(ready_from, op_first_offset(P, P.bottleneck, nullptr));
    if ((rc = build_wgrad(b, P.bottleneck, grads, scale, L)) != WUN_OK) return rc;
    if ((rc = build_dgrad(b, P.bottleneck, h->bwd_bottleneck, L)) != WUN_OK) return rc;
    for (int i = L - 1; i >= 0; --i) {
        fork_side(b);
        mark_grads_ready(b, ready_from, b.ws);
        ready_from = std::min(ready_from, op_first_offset(P, P.down[i], nullptr));
        if ((rc = build_wgrad(b, P.down[i], grads, scale, i)) != WUN_OK) return rc;
        if ((rc = build_dgrad(b, P.down[i], h->bwd_down[i], i)) != WUN_OK) return rc;
    }
    if (b.ws != ST_CALLER) {       // join: the caller's stream continues only after all wgrads
        add(b, OP_RECORD, ST_SIDE, EV_JOIN);
        add(b, OP_WAIT, ST_CALLER, EV_JOIN);
        if (b.first_pending) { add(b, OP_WAIT, ST_CALLER, EV_FIRST_DONE); b.first_pending = false; }
    }
    mark_grads_ready(b, 0, ST_CALLER);    // whatever is left: final after the join
    return WUN_OK;
}

// A training step: forward + backward, the weight packs hoisted onto the side stream when there is one.
static int build_step(Build& b, const float* targets, float* outputs, float* loss, float* grads, float scale) {
    const WunHandle* h = b.h;
    b.hoist = h->opt.use_side && h->opt.umma_enabled;
    b.dgrad_fork = h->opt.dgrad_par && h->opt.use_side;
    b.grads = grads; b.scale = scale; b.train = true;
    if (b.hoist) {             // the packs go to the side stream behind the work already enqueued on the caller's stream
        add(b, OP_MAKE, ST_SIDE).early = true;
        add(b, OP_MAKE, ST_CALLER, EV_FORK, 1).early = true;
        add(b, OP_RECORD, ST_CALLER, EV_FORK).early = true;
        add(b, OP_WAIT, ST_SIDE, EV_FORK).early = true;
        b.packs_pending = true;
    }
    int rc = build_forward(b, targets, outputs, loss, 1);
    if (rc == WUN_OK) rc = build_backward(b, targets, grads, scale);
    if (rc != WUN_OK || !b.hoist) return rc;
    add(b, OP_RECORD, ST_SIDE, EV_PACKS).early = true;
    if (b.packs_pending) add(b, OP_WAIT, ST_CALLER, EV_PACKS);   // no tensor-core conv consumed the packs: still join the side stream
    return WUN_OK;
}

static cudaError_t make_events(std::vector<cudaEvent_t>& v, size_t n) {
    while (v.size() < n) {
        cudaEvent_t e;
        const cudaError_t r = cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
        if (r != cudaSuccess) return r;
        v.push_back(e);
    }
    return cudaSuccess;
}

static cudaError_t make(WunHandle* h, const Op& o) {
    if (o.pool != EV_NONE) return make_events(h->events[o.pool], o.index);
    cudaStream_t& s = h->streams[o.stream];
    if (s) return cudaSuccess;
    cudaError_t e = cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
    if (e == cudaSuccess && o.stream == ST_SIDE) e = make_events(h->events[EV_JOIN], 1);
    if (e == cudaSuccess && o.stream == ST_SIDE) e = make_events(h->events[EV_PACKS], 1);
    return e;
}

static int issue_op(WunHandle* h, cudaStream_t caller, const Op& o) {
    const cudaStream_t s = o.stream == ST_CALLER ? caller : h->streams[o.stream];
    cudaError_t e = cudaSuccess;
    switch (o.kind) {
        case OP_SIGMOID: launch_sigmoid(o.sig.x, o.sig.y, o.sig.n, s); break;
        case OP_FIRST_FWD: launch_first_fwd(o.first, h->plan.cfg.num_channels, h->plan.down[0].cout, s); break;
        case OP_CONV: launch_plane_conv_simt(o.conv, s); break;
        case OP_PACK: e = launch_umma_pack(o.pack, s); break;
        case OP_UMMA_CONV: e = launch_plane_conv_umma(o.umma.U, s, o.umma.fused ? &o.umma.fuse : nullptr); break;
        case OP_COUNTERS: e = cudaMemsetAsync(o.counters, 0, 2 * sizeof(unsigned), s); break;
        case OP_OUTPUT_FWD: launch_output_fwd(o.out.O, s); break;
        case OP_OUTPUT_WGRAD: launch_output_wgrad(o.out.O, o.out.grads, o.out.part, o.out.scale, s); break;
        case OP_OUTPUT_DGRAD: launch_output_dgrad(o.out.O, o.out.gfeat, s); break;
        case OP_UPSAMPLE_BWD: launch_upsample_bwd(o.up, s); break;
        case OP_FIRST_WGRAD: launch_first_wgrad(o.fw, h->plan.cfg.num_channels, h->plan.down[0].cout, s); break;
        case OP_COLSUM: launch_colsum(o.colsum.V, o.colsum.batch, o.colsum.scale, o.colsum.out, s); break;
        case OP_WGRAD: launch_plane_wgrad_simt(o.wg, s); break;
        case OP_WGRAD_UMMA: e = launch_wgrad_umma(o.wgu.U, s); break;
        case OP_SPLIT: e = launch_split_views(o.wgu.J, s); break;
        case OP_WGRAD_BULK: e = launch_wgrad_umma_bulk(o.wgu.U, o.wgu.S, s); break;
        case OP_WGRAD_REDUCE: e = launch_wgrad_reduce(o.wgu.U, o.wgu.J, s); break;
        case OP_RECORD: e = cudaEventRecord(h->events[o.pool][o.index], s); break;
        case OP_WAIT: e = cudaStreamWaitEvent(s, h->events[o.pool][o.index], 0); break;
        case OP_MAKE: e = make(h, o); break;
    }
    if (e != cudaSuccess) return set_err(WUN_E_CUDA, std::string(o.kind < OP_RECORD ? "launch: " : "stream / event call: ") + cudaGetErrorString(e));
    return WUN_OK;
}

// The records in order; with hoisted weight packs, the `early` ones (the packs and their events on the side stream) first.
static int issue(WunHandle* h, const Call& call, const std::vector<Op>& ops) {
    int rc = WUN_OK;
    for (int early = 1; early >= 0; --early)
        for (size_t i = 0; i < ops.size() && rc == WUN_OK; ++i)
            if (ops[i].early == (early == 1)) rc = issue_op(h, call.stream, ops[i]);
    return rc;
}

static int check_device() {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        cudaGetLastError();
        return set_err(WUN_E_NOGPU, "no CUDA device: the engine has no CPU fallback");
    }
    return WUN_OK;
}

// Checks a call's arguments and makes its context; the handle's launch-list storage is emptied for the call's records.
static int begin_call(WunHandle* h, Call* call, const float* params, const float* mix, int64_t batch, bool training, void* ws,
                      int64_t ws_bytes, void* stream) {
    if (!h) return set_err(WUN_E_INVALID, "null handle");
    if (batch < 1 || batch > (1 << 20)) return set_err(WUN_E_INVALID, "batch out of range");
    { int rc0 = check_device(); if (rc0 != WUN_OK) return rc0; }
    if (!params || !mix || !ws) return set_err(WUN_E_INVALID, "null device pointer");
    call->map = ws_map(h, batch, training);
    if (ws_bytes < call->map.end) return set_err(WUN_E_INVALID, "workspace too small");
    if (reinterpret_cast<uintptr_t>(ws) % 256 != 0) return set_err(WUN_E_INVALID, "workspace must be 256-byte aligned");
    call->params = params; call->mix = mix; call->ws = (float*)ws; call->stream = (cudaStream_t)stream; call->batch = (int)batch;
    h->ops.clear();
    return WUN_OK;
}

// A call that is only built, never issued (launch counts, descriptions, the create-time sizes): no buffers unless the caller
// sets fake ones, no stream.
static Call dry_call(const WunHandle* h, int64_t batch, bool training) {
    Call call;
    call.batch = (int)batch;
    call.map = ws_map(h, batch, training);
    return call;
}

// The launch list of a training step (`training` false: an inference forward) of a dry call, appended to `ops`.
static Build build_dry(const WunHandle* h, const Call& call, std::vector<Op>& ops, bool training) {
    Build b{h, call, ops};
    if (training) build_step(b, nullptr, nullptr, nullptr, nullptr, 1.f);
    else build_forward(b, nullptr, nullptr, nullptr, 0);
    return b;
}

static const ConvOp& layer_op(const WunHandle* h, int layer) {
    const int L = h->plan.cfg.num_layers;
    return (layer < L) ? h->plan.down[layer] : (layer == L ? h->plan.bottleneck : h->plan.up[layer - L - 1]);
}

// kernel records, counted as launches: the output and first-layer weight gradients are two kernels each (per-CTA sums + their
// fixed-order total), the counter memset counts as one
static int64_t kernel_launches(const std::vector<Op>& ops) {
    int64_t n = 0;
    for (const Op& o : ops)
        if (o.kind < OP_RECORD) n += (o.kind == OP_OUTPUT_WGRAD || o.kind == OP_FIRST_WGRAD) ? 2 : 1;
    return n;
}

// ------------------------------------------------------------------------------------------------
// launch descriptions (wun_debug_plan, wun_debug_launches)
// ------------------------------------------------------------------------------------------------
static long long addr(const void* p) { return (long long)reinterpret_cast<uintptr_t>(p); }

static void appendf(std::string& s, const char* fmt, ...) {
    char line[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(line, sizeof(line), fmt, ap);
    va_end(ap);
    s += line;
}

static int64_t copy_out(const std::string& s, char* buf, int64_t capacity) {
    if (buf && capacity > 0) {
        int64_t n = std::min<int64_t>(capacity - 1, (int64_t)s.size());
        memcpy(buf, s.data(), n);
        buf[n] = 0;
    }
    return (int64_t)s.size() + 1;
}

// wun_debug_plan: one line per tensor-core conv, one per group of a tensor-core weight gradient
static void audit_op(std::string& s, const Op& o) {
    if (o.kind == OP_UMMA_CONV) {
        const ConvLaunch& L = o.umma.L;
        const UmmaChoice& ch = o.umma.ch;
        long long tiles = 0, mmas = 0; int max_rows = 0, span = 0;
        for (int q = 0; q < L.ncls; ++q) {
            const int rows = L.cls[q].m_hi - L.cls[q].m_lo;
            const long long tq = (long long)((rows + ch.MT * 128 - 1) / (ch.MT * 128)) * ch.nsplit * L.batch;
            tiles += tq;
            max_rows = std::max(max_rows, rows);
            int t = L.cls[q].term_begin;
            long long ksteps = 0;                       // (16-channel chunk, tap) pairs of one tile of this class
            while (t < L.cls[q].term_end) {
                int t1 = t, dmin = L.terms[t].d, dmax = dmin;
                while (t1 < L.cls[q].term_end && L.terms[t1].plane == L.terms[t].plane) {
                    dmin = std::min(dmin, L.terms[t1].d); dmax = std::max(dmax, L.terms[t1].d); ++t1; }
                span = std::max(span, dmax - dmin);
                ksteps += (long long)((L.planes[L.terms[t].plane].C + 15) / 16) * (t1 - t);
                t = t1;
            }
            mmas += tq * ch.MT * ksteps * 3;
        }
        appendf(s, "conv layer=%d pass=%d kernel=wgmma N=%d NPAD=%d nsplit=%d MT=%d rows_alloc=%d span=%d "
                "TB=%d nbs=%d tiles=%lld mmas=%lld max_rows=%d smem=%zu pack_bytes=%zu pair=%d outfuse=%d\n",
                o.layer, o.pass, L.N, ch.NPAD, ch.nsplit, ch.MT, ch.rows_alloc, span, ch.TB, ch.nbs, tiles, mmas,
                max_rows, umma_choice_smem_bytes(ch), ch.pack_bytes, L.pairC, o.umma.fused ? 1 : 0);
    } else if (o.kind == OP_WGRAD_UMMA || o.kind == OP_WGRAD_BULK) {
        const UmmaWgradLaunch& U = o.wgu.U;
        for (int g = 0; g < U.ngroups; ++g) {
            const WgGroup& G = U.grp[g];
            appendf(s, "wgrad layer=%d group=%d Cp=%d Cg=%d swap=%d NT=%d mtiles=%d ntiles=%d ntaps=%d taps_per_cta=%d "
                    "tapsets=%d chunks_per_cta=%d n_ctas_x=%d chunks=%lld grid=%dx%dx%d nstages=%d smem=%zu issued_macs=%lld useful_macs=%lld\n",
                    o.layer, g, G.P.C, G.G.C, G.swap, G.NT, G.n_mtiles, G.n_ntiles, G.ntaps, G.taps_per_cta, G.n_tapsets,
                    G.chunks_per_cta, G.n_ctas_x, (long long)U.batch * G.chunks_per_batch, U.grid_x, U.grid_y, U.grid_z, U.nstages,
                    umma_wgrad_smem_bytes(U), umma_wgrad_issued_macs(G, U.batch),
                    (long long)U.batch * G.chunks_per_batch * 64 * G.ntaps * G.P.C * G.G.C);
        }
    }
}

static void describe_view(std::string& s, const char* tag, const PlaneView& P) {
    appendf(s, "%s base=%lld bstride=%lld rstride=%d r_lo=%d r_hi=%d C=%d kind=%d mid_mode=%d xrows=%d blend=%lld\n",
            tag, addr(P.base), P.bstride, P.rstride, P.r_lo, P.r_hi, P.C, P.kind, P.mid_mode, P.xrows, P.blend ? addr(P.blend) : -1LL);
}

// one plane-convolution launch; tests/test_launch_semantics.py interprets these descriptions in numpy: the pair-merged form of
// a launch must compute exactly what its two-class form does
static void describe_conv(std::string& s, const ConvLaunch& L, int layer, int pass) {
    appendf(s, "launch layer=%d pass=%d N=%d pairC=%d w_sk=%d w_sn=%d W=%lld bias=%lld epilogue=%d batch=%d nplanes=%d ncls=%d\n",
            layer, pass, L.N, L.pairC, L.w_sk, L.w_sn, addr(L.W), L.bias ? addr(L.bias) : -1LL, L.epilogue, L.batch, L.nplanes, L.ncls);
    for (int p = 0; p < L.nplanes; ++p) describe_view(s, ("plane i=" + std::to_string(p)).c_str(), L.planes[p]);
    int nterm = 0;
    for (int q = 0; q < L.ncls; ++q) {
        const OutView& O = L.cls[q];
        nterm = std::max(nterm, O.term_end);
        appendf(s, "cls i=%d base=%lld bstride=%lld rstride=%d m_lo=%d m_hi=%d saved=%lld acc_lo=%d acc_hi=%d term_begin=%d term_end=%d "
                "pairC=%d base2=%lld bstride2=%lld rstride2=%d saved2=%lld acc_lo2=%d acc_hi2=%d lo0=%d hi0=%d lo1=%d hi1=%d\n",
                q, addr(O.base), O.bstride, O.rstride, O.m_lo, O.m_hi, O.saved ? addr(O.saved) : -1LL, O.acc_lo, O.acc_hi, O.term_begin, O.term_end,
                O.pairC, O.pairC ? addr(O.base2) : -1LL, O.bstride2, O.rstride2, (O.pairC && O.saved2) ? addr(O.saved2) : -1LL, O.acc_lo2, O.acc_hi2,
                O.lo_h[0], O.hi_h[0], O.lo_h[1], O.hi_h[1]);
    }
    for (int t = 0; t < nterm; ++t)
        appendf(s, "term i=%d plane=%d d=%d woff=%d woff2=%d\n", t, L.terms[t].plane, L.terms[t].d, L.terms[t].woff, L.pairC ? L.terms[t].woff2 : -1);
}

// one (class, plane) group of a layer's weight gradient (dW[woff + c*cout + n], any form); dW / db = flat parameter offsets
static void describe_wgrad(std::string& s, const WunHandle* h, const WgGroup& G, int layer, int g, int batch) {
    const ConvOp& op = layer_op(h, layer);
    appendf(s, "wgrad layer=%d group=%d N=%d w_sk=%d w_sn=%d dW=%lld db=%lld m_lo=%d m_hi=%d nterms=%d batch=%d\n",
            layer, g, op.cout, op.cout, 1, (long long)h->plan.params[op.w_param].offset, (long long)h->plan.params[op.b_param].offset,
            G.m_lo, G.m_hi, G.ntaps, batch);
    describe_view(s, "wplane", G.P);
    describe_view(s, "wdpre", G.G);
    for (int t = 0; t < G.ntaps; ++t) appendf(s, "wterm i=%d d=%d woff=%d\n", t, G.d[t], G.woff[t]);
}

// wun_debug_launches: every launch of the step as text (addresses are raw integers relative to the call's fake bases - nothing
// is dereferenced)
static void describe_op(std::string& s, const WunHandle* h, const Call& call, const Op& o) {
    const Plan& P = h->plan;
    if (o.kind == OP_FIRST_FWD) {        // its weight gradient has the same geometry; gdec / godd = the gradient tensors it reads
        const FirstLayer& F = o.first;
        const ConvOp& op = P.down[0];
        appendf(s, "first C=%d N=%d k=%d pad_left=%d batch=%d x=%lld x_bstride=%lld T=%d dec=%lld dec_bstride=%lld Td=%d "
                "odd=%lld odd_bstride=%lld mo_lo=%d mo_hi=%d gdec=%lld godd=%lld dW=%lld db=%lld\n",
                P.cfg.num_channels, op.cout, F.k, F.pad_left, F.batch, addr(F.x), F.x_bstride, F.T, addr(F.dec), F.dec_bstride, F.Td,
                addr(F.odd), F.odd_bstride, F.mo_lo, F.mo_hi, addr(tensor_ptr(call, P.grad_twin[op.classes[0].out.tensor])),
                addr(tensor_ptr(call, P.grad_twin[op.classes[1].out.tensor])), (long long)P.params[op.w_param].offset,
                (long long)P.params[op.b_param].offset);
    } else if (o.kind == OP_CONV || o.kind == OP_UMMA_CONV) {
        describe_conv(s, o.kind == OP_CONV ? o.conv : o.umma.L, o.layer, o.pass);
    } else if (o.kind == OP_OUTPUT_FWD) {    // caller buffers: include/wun.h layouts
        const OutputLaunch& O = o.out.O;
        appendf(s, "output batch=%d T_in=%d Tf=%d T_out=%d C=%d F=%d nconv=%d K=%d ofs=%d pad_left=%d crop_feat=%d "
                "crop_out=%d output_type=%d activation=%d feat=%lld dpre=%lld gfeat=%lld",
                O.batch, O.T_in, O.Tf, O.T_out, O.C, O.F, O.nconv, O.K, O.ofs, O.pad_left, O.crop_feat, O.crop_out, O.output_type,
                O.activation, addr(O.feat), addr(O.dpre), addr(tensor_ptr(call, P.grad_twin[P.t_feat])));
        for (int k = 0; k < 8; ++k)
            appendf(s, " w_off%d=%lld b_off%d=%lld", k, k < O.nconv ? O.w_off[k] : -1LL, k, k < O.nconv ? O.b_off[k] : -1LL);
        s += "\n";
    } else if (o.kind == OP_UPSAMPLE_BWD) {  // dvar = the interp parameter's flat offset (gradient buffer) or -1
        const UpsampleBwdLaunch& U = o.up;
        const int i = o.layer - P.cfg.num_layers - 1;
        appendf(s, "upsample level=%d batch=%d N=%d nmid=%d C=%d mid_mode=%d due=%lld dmid=%lld x=%lld gx=%lld blend=%lld dvar=%lld\n",
                i, U.batch, U.N, U.nmid, U.C, U.mid_mode, addr(U.due), addr(U.dmid), addr(U.x), addr(U.gx), U.blend ? addr(U.blend) : -1LL,
                P.ups[i].interp_param >= 0 ? (long long)P.params[P.ups[i].interp_param].offset : -1LL);
    } else if (o.kind == OP_WGRAD) {         // one group per CUDA-core launch
        WgGroup G;
        G.P = o.wg.plane; G.G = o.wg.dpre; G.m_lo = o.wg.m_lo; G.m_hi = o.wg.m_hi; G.ntaps = o.wg.nterms;
        for (int t = 0; t < G.ntaps; ++t) { G.d[t] = o.wg.d[t]; G.woff[t] = o.wg.woff[t]; }
        describe_wgrad(s, h, G, o.layer, o.index, call.batch);
    } else if (o.kind == OP_WGRAD_UMMA || o.kind == OP_WGRAD_BULK) {    // all groups of the layer in one launch
        for (int g = 0; g < o.wgu.U.ngroups; ++g) describe_wgrad(s, h, o.wgu.U.grp[g], o.layer, g, call.batch);
    }
}

// ------------------------------------------------------------------------------------------------
// C ABI
// ------------------------------------------------------------------------------------------------
extern "C" {

const char* wun_last_error(void) { return g_err.c_str(); }
const char* wun_version(void) { return "wun-b200 0.2 (sm_90a)"; }

int wun_get_padding(const WunConfig* cfg, int64_t num_frames, int64_t* t_in, int64_t* t_out) {
    if (!cfg || !t_in || !t_out) return set_err(WUN_E_INVALID, "null argument");
    std::string msg;
    int rc = solve_padding(*cfg, num_frames, t_in, t_out, &msg);
    if (rc != WUN_OK) return set_err(rc, msg);
    return WUN_OK;
}

int wun_create_for_input(const WunConfig* cfg, int64_t input_frames, WunHandle** out) {
    if (!cfg || !out) return set_err(WUN_E_INVALID, "null argument");
    WunHandle* h = new WunHandle();
    std::string msg;
    int rc = build_plan(*cfg, input_frames, &h->plan, &msg);
    if (rc != WUN_OK) { delete h; return set_err(rc, msg); }
    plan_backward(h);
    h->opt = read_options();
    // the launch list of a batch-1 training step: which kernel each layer uses and how much scratch the launches need
    const Call call = dry_call(h, 1, true);
    const Build b = build_dry(h, call, h->ops, true);
    h->arena_sum = b.pack_sum; h->split_item_bytes = b.split_item; h->wg_partial_bytes = b.wg_partial; h->out_part_bytes = b.out_part;
    h->kernel_used.assign((size_t)(2 * h->plan.cfg.num_layers + 1) * 3, "simt");
    for (const Op& o : b.ops)      // a layer pass runs on the kernel of its last plane convolution / weight gradient
        if (o.kind == OP_CONV || o.kind == OP_WGRAD) h->kernel_used[o.layer * 3 + o.pass] = "simt";
        else if (o.kind == OP_UMMA_CONV || o.kind == OP_WGRAD_UMMA || o.kind == OP_WGRAD_BULK) h->kernel_used[o.layer * 3 + o.pass] = "umma";
    *out = h;
    return WUN_OK;
}

int wun_create(const WunConfig* cfg, int64_t num_frames, WunHandle** out) {
    if (!cfg || !out) return set_err(WUN_E_INVALID, "null argument");
    int64_t t_in = 0, t_out = 0;
    std::string msg;
    int rc = solve_padding(*cfg, num_frames, &t_in, &t_out, &msg);
    if (rc != WUN_OK) return set_err(rc, msg);
    return wun_create_for_input(cfg, t_in, out);
}

int wun_destroy(WunHandle* h) {
    if (h) {
        for (const auto& pool : h->events)
            for (auto e : pool) cudaEventDestroy(e);
        for (auto st : h->streams)
            if (st) cudaStreamDestroy(st);
        delete h;
    }
    return WUN_OK;
}

int64_t wun_input_frames(const WunHandle* h) { return h ? h->plan.T_in : -1; }
int64_t wun_output_frames(const WunHandle* h) { return h ? h->plan.T_out : -1; }
int64_t wun_param_count(const WunHandle* h) { return h ? (int64_t)h->plan.params.size() : -1; }
int64_t wun_param_numel(const WunHandle* h) { return h ? h->plan.param_numel : -1; }

int wun_param_table(const WunHandle* h, WunParamInfo* out, int64_t capacity) {
    if (!h || !out) return set_err(WUN_E_INVALID, "null argument");
    if (capacity < (int64_t)h->plan.params.size()) return set_err(WUN_E_INVALID, "param table capacity too small");
    for (size_t i = 0; i < h->plan.params.size(); ++i) out[i] = h->plan.params[i];
    return WUN_OK;
}

int64_t wun_workspace_bytes(const WunHandle* h, int64_t batch, int training) {
    if (!h || batch < 1) return -1;
    return ws_map(h, batch, training != 0).end + 256;
}

double wun_forward_flops(const WunHandle* h, int64_t batch) { return h ? h->plan.fwd_flops_per_item * batch : 0; }
double wun_forward_backward_flops(const WunHandle* h, int64_t batch) {
    return h ? (3.0 * h->plan.fwd_flops_per_item - h->plan.dgrad0_flops_per_item) * batch : 0;
}

static int64_t dry_launches(const WunHandle* h, bool training) {
    if (!h) return -1;
    std::vector<Op> ops;
    build_dry(h, dry_call(h, 1, training), ops, training);
    return kernel_launches(ops);
}

int64_t wun_launches_forward(const WunHandle* h) { return dry_launches(h, false); }
int64_t wun_launches_forward_backward(const WunHandle* h) { return dry_launches(h, true); }

int wun_forward(WunHandle* h, const float* params, const float* mix, int64_t batch, int training, float* outputs,
                void* workspace, int64_t workspace_bytes, void* stream) {
    Call call;
    int rc = begin_call(h, &call, params, mix, batch, false, workspace, workspace_bytes, stream);
    if (rc != WUN_OK) return rc;
    if (!outputs) return set_err(WUN_E_INVALID, "outputs is null");
    Build b{h, call, h->ops};
    rc = build_forward(b, nullptr, outputs, nullptr, training);
    if (rc == WUN_OK) rc = issue(h, call, b.ops);
    if (rc != WUN_OK) return rc;
    WUN_CUDA_OK(cudaGetLastError());
    return WUN_OK;
}

int wun_forward_backward(WunHandle* h, const float* params, const float* mix, const float* targets, int64_t batch,
                         float* outputs, float* loss, float* grads, float grad_scale, void* workspace,
                         int64_t workspace_bytes, void* stream) {
    Call call;
    int rc = begin_call(h, &call, params, mix, batch, true, workspace, workspace_bytes, stream);
    if (rc != WUN_OK) return rc;
    if (!targets || !loss || !grads) return set_err(WUN_E_INVALID, "targets/loss/grads must not be null");
    WUN_CUDA_OK(cudaMemsetAsync(loss, 0, sizeof(float), call.stream));
    WUN_CUDA_OK(cudaMemsetAsync(grads, 0, sizeof(float) * h->plan.param_numel, call.stream));
    Build b{h, call, h->ops};
    rc = build_step(b, targets, outputs, loss, grads, grad_scale);
    if (rc == WUN_OK) rc = issue(h, call, b.ops);
    if (rc != WUN_OK) return rc;
    WUN_CUDA_OK(cudaGetLastError());
    return WUN_OK;
}

int wun_adam_step(WunHandle* h, float* params, const float* grads, float* m, float* v, int64_t step, float lr,
                  float beta1, float beta2, float eps, void* stream) {
    if (!h || !params || !grads || !m || !v) return set_err(WUN_E_INVALID, "null argument");
    if (step < 1) return set_err(WUN_E_INVALID, "step must be >= 1");
    int rc = check_device();
    if (rc != WUN_OK) return rc;
    const double lr_t = (double)lr * sqrt(1.0 - pow((double)beta2, (double)step)) / (1.0 - pow((double)beta1, (double)step));
    launch_adam(params, grads, m, v, h->plan.param_numel, (float)lr_t, beta1, beta2, eps, nullptr, (cudaStream_t)stream);
    WUN_CUDA_OK(cudaGetLastError());
    return WUN_OK;
}

int wun_adam_step_device(WunHandle* h, float* params, const float* grads, float* m, float* v, float* state, float lr,
                         float beta1, float beta2, float eps, void* stream) {
    if (!h || !params || !grads || !m || !v || !state) return set_err(WUN_E_INVALID, "null argument");
    int rc = check_device();
    if (rc != WUN_OK) return rc;
    launch_adam(params, grads, m, v, h->plan.param_numel, lr, beta1, beta2, eps, state, (cudaStream_t)stream);
    WUN_CUDA_OK(cudaGetLastError());
    return WUN_OK;
}

int wun_set_grad_buckets(WunHandle* h, int n, const int64_t* first_offset) {
    if (!h || n < 0 || (n > 0 && !first_offset)) return set_err(WUN_E_INVALID, "bad argument");
    for (int k = 0; k < n; ++k) {
        if (first_offset[k] < 0 || first_offset[k] >= h->plan.param_numel || (k > 0 && first_offset[k] >= first_offset[k - 1]))
            return set_err(WUN_E_INVALID, "bucket offsets must be strictly descending (production order) inside the flat buffer");
    }
    if (n > 0 && first_offset[n - 1] != 0) return set_err(WUN_E_INVALID, "the last bucket must start at offset 0");
    if (n > 0) { int rc = check_device(); if (rc != WUN_OK) return rc; }
    WUN_CUDA_OK(make_events(h->events[EV_BUCKET], n));
    h->bucket_first.assign(first_offset, first_offset + n);
    return WUN_OK;
}

int wun_stream_wait_grad_bucket(WunHandle* h, int k, void* stream) {
    if (!h || k < 0 || k >= (int)h->bucket_first.size()) return set_err(WUN_E_INVALID, "no such gradient bucket");
    WUN_CUDA_OK(cudaStreamWaitEvent((cudaStream_t)stream, h->events[EV_BUCKET][k], 0));
    return WUN_OK;
}

int wun_gather_windows(WunHandle* h, const float* padded, int64_t n_padded, const int64_t* starts, int64_t n_windows,
                       float* mix_batch, void* stream) {
    if (!h || !padded || !starts || !mix_batch) return set_err(WUN_E_INVALID, "null argument");
    int rc = check_device();
    if (rc != WUN_OK) return rc;
    launch_gather_windows(padded, n_padded, (const long long*)starts, (int)n_windows, (int)h->plan.T_in,
                          h->plan.cfg.num_channels, mix_batch, (cudaStream_t)stream);
    WUN_CUDA_OK(cudaGetLastError());
    return WUN_OK;
}

int wun_scatter_windows(WunHandle* h, const float* outputs, const int64_t* starts, int64_t n_windows, float* preds,
                        int64_t n_frames, void* stream) {
    if (!h || !outputs || !starts || !preds) return set_err(WUN_E_INVALID, "null argument");
    int rc = check_device();
    if (rc != WUN_OK) return rc;
    launch_scatter_windows(outputs, (const long long*)starts, (int)n_windows, h->plan.cfg.num_sources,
                           (int)h->plan.T_out, h->plan.cfg.num_channels, preds, n_frames, (cudaStream_t)stream);
    WUN_CUDA_OK(cudaGetLastError());
    return WUN_OK;
}

int wun_feed_batch(WunHandle* h, const float* pool, int64_t total_frames, const int64_t* track_offset,
                   const int64_t* track_length, int64_t n_tracks, int64_t batch, int augmentation, uint64_t seed,
                   int64_t* step_state, float* mix_out, float* targets_out, int64_t* chosen, void* stream) {
    if (!h || !pool || !track_offset || !track_length || !step_state || !mix_out || !targets_out)
        return set_err(WUN_E_INVALID, "null argument");
    if (n_tracks < 1 || n_tracks > (1 << 30) || batch < 1 || batch > 65535 || total_frames < h->plan.T_in)
        return set_err(WUN_E_INVALID, "feeder: need >= 1 track, 1 <= batch <= 65535 and a pool of at least T_in frames");
    if (h->plan.cfg.num_sources < 1 || h->plan.cfg.num_sources > 8) return set_err(WUN_E_INVALID, "feeder: 1..8 sources");
    int rc = check_device();
    if (rc != WUN_OK) return rc;
    WUN_CUDA_OK(launch_feed_batch(pool, total_frames, (const long long*)track_offset, (const long long*)track_length,
                                  (int)n_tracks, (int)batch, h->plan.cfg.num_sources, h->plan.cfg.num_channels,
                                  (int)h->plan.T_in, (int)h->plan.T_out, augmentation, (unsigned long long)seed,
                                  (long long*)step_state, mix_out, targets_out, (long long*)chosen, (cudaStream_t)stream));
    return WUN_OK;
}

int64_t wun_describe(const WunHandle* h, char* buf, int64_t capacity) {
    if (!h) return -1;
    std::string s = h->plan.describe();
    s += "  kernels (fwd/dgrad/wgrad): ";
    for (size_t i = 0; i + 2 < h->kernel_used.size(); i += 3)
        s += h->kernel_used[i] + "/" + h->kernel_used[i + 1] + "/" + h->kernel_used[i + 2] + " ";
    s += "\n";
    return copy_out(s, buf, capacity);
}

int64_t wun_debug_plan(const WunHandle* h, int64_t batch, char* buf, int64_t capacity) {
    if (!h || batch < 1) return -1;
    std::vector<Op> ops;
    build_dry(h, dry_call(h, batch, true), ops, true);
    std::string s;
    for (const Op& o : ops) audit_op(s, o);
    return copy_out(s, buf, capacity);
}

int64_t wun_debug_launches(const WunHandle* h, int64_t batch, char* buf, int64_t capacity) {
    if (!h || batch < 1) return -1;
    // fake, far-apart bases (never dereferenced): every described address identifies its buffer
    Call call = dry_call(h, batch, true);
    call.ws = reinterpret_cast<float*>((uintptr_t)1 << 40); call.params = reinterpret_cast<const float*>((uintptr_t)1 << 41);
    call.mix = reinterpret_cast<const float*>((uintptr_t)1 << 42);
    std::vector<Op> ops;
    build_dry(h, call, ops, true);
    std::string s;
    for (const Op& o : ops) describe_op(s, h, call, o);
    s += "adam n=" + std::to_string((long long)h->plan.param_numel) + "\n";     // wun_adam_step(_device) over the flat buffer
    return copy_out(s, buf, capacity);
}

static double op_forward_flops(const ConvOp& op, int64_t batch) {
    double f = 0;
    for (const auto& c : op.classes) {
        double ks = 0;
        for (const auto& t : c.terms) ks += op.planes[t.plane].C;
        f += 2.0 * std::max(0, c.m_hi - c.m_lo) * ks * op.cout;
    }
    return f * batch;
}

int wun_debug_run_layer(WunHandle* h, int layer, int pass, int iters, const float* params, const float* mix, float* grads_scratch,
                        int64_t batch, void* workspace, int64_t workspace_bytes, void* stream, double* flops_per_launch) {
    if (!h || iters < 1 || pass < 0 || pass > 2) return set_err(WUN_E_INVALID, "bad argument");
    const int L = h->plan.cfg.num_layers;
    if (layer < 0 || layer > 2 * L) return set_err(WUN_E_INVALID, "layer out of range");
    if (pass == 2 && !grads_scratch) return set_err(WUN_E_INVALID, "wgrad pass needs a gradient scratch buffer");
    Call call;
    int rc = begin_call(h, &call, params, mix, batch, true, workspace, workspace_bytes, stream);
    if (rc != WUN_OK) return rc;
    const ConvOp& op = layer_op(h, layer);
    const OpBackward& ob = (layer < L) ? h->bwd_down[layer] : (layer == L ? h->bwd_bottleneck : h->bwd_up[layer - L - 1]);
    if (flops_per_launch) {
        // algorithmic (live-position) FLOPs: dgrad = the forward MACs of the planes that need a gradient, wgrad = all of them
        double f = op_forward_flops(op, batch);
        if (pass == 1) {
            double keep = 0, all = 0;
            for (const auto& c : op.classes)
                for (const auto& t : c.terms) {
                    const double w = (double)std::max(0, c.m_hi - c.m_lo) * op.planes[t.plane].C;
                    all += w;
                    if (op.plane_grad_tensor[t.plane] != -2) keep += w;
                }
            f = (all > 0) ? f * keep / all : 0;
        }
        *flops_per_launch = f;
    }
    // the layer pass as in a step, on the caller's stream (a dgrad's second launch on the helper stream once a step made it)
    Build b{h, call, h->ops};
    b.dgrad_fork = h->opt.dgrad_par && h->opt.use_side && h->streams[ST_SIDE] != nullptr;
    rc = (pass == 0) ? build_conv_forward(b, op, layer) : (pass == 1) ? build_dgrad(b, op, ob, layer) : build_wgrad(b, op, grads_scratch, 1.f, layer);
    if (rc == WUN_OK) rc = issue(h, call, b.ops);
    // forward: packed once, the tensor-core conv enqueued `iters` times; dgrad / wgrad: the whole pass again
    for (int i = 1; i < iters && rc == WUN_OK; ++i)
        for (size_t k = 0; k < b.ops.size() && rc == WUN_OK; ++k)
            if (pass != 0 || b.ops[k].kind == OP_UMMA_CONV) rc = issue_op(h, call.stream, b.ops[k]);
    if (rc != WUN_OK) return rc;
    WUN_CUDA_OK(cudaGetLastError());
    return WUN_OK;
}

int wun_debug_run_conv(WunHandle* h, int layer, int iters, const float* params, const float* mix, int64_t batch,
                       void* workspace, int64_t workspace_bytes, void* stream, double* flops_per_launch) {
    return wun_debug_run_layer(h, layer, 0, iters, params, mix, nullptr, batch, workspace, workspace_bytes, stream, flops_per_launch);
}

int wun_debug_tensor(const WunHandle* h, const char* name, int64_t batch, int training, int64_t* offset_floats,
                     int64_t* rows, int32_t* channels) {
    if (!h || !name || !offset_floats || !rows || !channels) return set_err(WUN_E_INVALID, "null argument");
    const WsMap m = ws_map(h, batch, training != 0);
    for (size_t i = 0; i < h->plan.tensors.size(); ++i)
        if (h->plan.tensors[i].name == name) {
            if (m.act[i] < 0) return set_err(WUN_E_INVALID, "tensor exists only in training workspaces");
            *offset_floats = m.act[i]; *rows = h->plan.tensors[i].rows; *channels = h->plan.tensors[i].C;
            return WUN_OK;
        }
    return set_err(WUN_E_INVALID, std::string("no workspace tensor named ") + name);
}

const char* wun_layer_kernel(const WunHandle* h, int layer, int pass) {
    if (!h) return "";
    const size_t slot = (size_t)layer * 3 + pass;
    if (layer < 0 || pass < 0 || pass > 2 || slot >= h->kernel_used.size()) return "";
    return h->kernel_used[slot].c_str();
}

}  // extern "C"
