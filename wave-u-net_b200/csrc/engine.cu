// engine.cu - C ABI (include/wun.h) of the Wave-U-Net engine (H100, sm_90a): turns the host plan into kernel launches.
//
// Forward  = get_output             /root/reference/Models/UnetAudioSeparator.py:85-144
// Backward = what tf.gradients builds for AdamOptimizer.minimize, /root/reference/Training.py:77
// (the reference has no backward source; the derivation is in DESIGN.md "Backward").
#include <cuda_runtime.h>
#include <math.h>
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

struct Layout {
    std::vector<int64_t> off;   // float offsets per tensor; -1 = not allocated
    int64_t total = 0;
};

}  // namespace

struct WunHandle {
    Plan plan;
    std::vector<OpBackward> bwd_down, bwd_up;
    OpBackward bwd_bottleneck;
    bool umma_enabled = true;            // tensor-core path on (WUN_DISABLE_UMMA=1 turns it off, for A/B tests)
    bool umma_pass[3] = {true, true, true};   // per pass (fwd, dgrad, wgrad): WUN_UMMA_FWD=0 / WUN_UMMA_DGRAD=0 / WUN_UMMA_WGRAD=0
    size_t arena_bytes = 0;              // scratch for packed bf16 weights (max over launches)
    std::vector<std::string> kernel_used;   // [layer*3 + pass] -> "simt" | "umma" (filled by dry runs)
    int cur_layer = 0, cur_pass = 0;
    int debug_iters = 0;                 // > 0: wun_debug_run_conv - pack once, enqueue the conv kernel this many times
    // weight-gradient kernels run on an internal side stream, concurrently with the dgrad chain on the caller's stream
    cudaStream_t side = nullptr;
    // A dgrad with two launches (the up blocks: skip pair and upsampled pair have different widths) runs the second one on this
    // helper stream, concurrently with the first: both read the same gradient planes and write different tensors, and in the deep
    // layers neither fills the GPU (WUN_DGRAD_PAR=0 disables)
    cudaStream_t side2 = nullptr;
    std::vector<cudaEvent_t> par_events;      // fork / join pairs, one pair per use inside a call (graph capture needs distinct events)
    int par_used = 0;
    bool dgrad_par = true;
    std::vector<cudaEvent_t> fork_events;
    cudaEvent_t join_event = nullptr;
    int fork_used = 0;
    bool use_side = true;                // WUN_SIDE_STREAM=0 disables
    bool first_fast = true;              // dedicated first-layer kernels (kernels_first.cu); WUN_FIRST_LAYER=0 = generic path
    bool bulk_wgrad = true;              // split pass + bulk-copy-fed tensor-core wgrad; WUN_BULK_WGRAD=0 = converter-fed kernel
    // output layer in the last up block's conv epilogue (kernels_umma.h OutputFuse).  WUN_OUT_FUSE: 0 = separate kernels, 1 (default) =
    // estimates + loss + dL/dpre + the gradient w.r.t. the features fused, the output convs' weight gradient as its own launch on
    // the wgrad stream (off the critical path), 2 = the weight gradient in the epilogue too (measured slower: it serialises
    // ~650 shuffle-reduction instructions per row tile on the four epilogue warps)
    int out_fuse_mode = 1;
    const OutputFuse* fuse_out = nullptr;   // set by run_forward around the last up block's forward conv
    bool out_fused = false;              // that conv carried the output layer: no output_fwd / output_dgrad / output_wgrad launches
    float* bw_grads = nullptr;           // wun_forward_backward: gradient buffer / scale, known to the forward pass for the fused epilogue
    float bw_scale = 1.f;
    int pair_min_ctas = 120;             // WUN_PAIR_MIN_CTAS
    bool pair_fwd = true;                // the same for the forward classes of the up blocks; WUN_PAIR_FWD=0 disables
    int pair_dgrad = 4;                  // pair-merged dgrad classes (launch.h OutView::pairC); WUN_PAIR_DGRAD=0 off, 1 all, 2 down blocks only,
                                         // 3 up blocks only, 4 (default) down blocks whose merged width still takes the fused-N MMAs (2C <= 64)
    size_t split_item_bytes = 0;         // per batch item: largest split arena any layer's wgrad needs (dry run)
    size_t wg_partial_bytes = 0;         // largest partial-tile scratch of a layer's wgrad (any batch; dry run)
    size_t out_part_bytes = 0;           // the output layer's per-CTA weight-gradient sums (any batch; dry run)
    cudaStream_t wstream = nullptr;      // stream the wgrad-side launches go to (side or main)
    // split passes run one layer AHEAD of the wgrad kernels, on their own stream, into a double-buffered arena: the split pass is
    // DRAM-bound, the wgrad kernel L2 / tensor bound, so they overlap well (WUN_SPLIT_AHEAD=0: same stream, one arena half)
    cudaStream_t split_stream = nullptr;
    std::vector<cudaEvent_t> split_done, wg_done;
    int wg_index = 0;
    bool split_ahead = true;
    cudaEvent_t first_done = nullptr;     // first-layer weight gradient on the split stream
    bool first_pending = false;
    // weight packs are hoisted off the critical path: phase 1 enqueues every pack kernel of the step on the side stream
    // (they only depend on the parameters), phase 2 enqueues everything else; phase 0 = inline (inference, debug hook)
    int phase = 0;
    size_t arena_cur = 0;                // bump pointer into the pack arena (same sequence in phase 1 and 2)
    size_t pack_floor = 0;               // launch_conv reserves at least this much: the pair-merge decision depends on the batch
                                         // (folded or not) but the arena is sized by a batch-1 dry run, so both forms' bytes count
    size_t arena_sum = 0;                // total pack bytes of one forward+backward (dry run)
    cudaEvent_t packs_event = nullptr;
    bool packs_pending = false;          // main stream has not yet waited for the hoisted packs
    // one event per FORWARD weight pack, so that forward conv i waits for pack i only instead of for all ~60 packs of the
    // step (the backward convs still wait for the single packs_event); WUN_PACK_EVENTS=0 disables
    bool pack_events_on = true;
    std::vector<cudaEvent_t> pack_events;
    int pack_idx = 0;                    // forward tensor-core conv counter of the current phase
    std::vector<std::string>* audit = nullptr;   // dry runs: one line per tensor-core launch (wun_debug_plan)
    std::vector<std::string>* export_launches = nullptr;   // dry runs: the full description of every plane-convolution launch (wun_debug_launches)
    // data-parallel overlap: gradient buckets in PRODUCTION order (output layer first, down0 last); bucket k = flat offsets
    // >= bucket_first[k] (and below bucket k-1's).  bucket_events[k] is recorded once every gradient of the bucket is final.
    std::vector<int64_t> bucket_first;
    std::vector<cudaEvent_t> bucket_events;
    int bucket_next = 0;
    // per-call state
    bool dry = false;
    int64_t launches = 0;
    cudaStream_t stream = nullptr;
    const float* params = nullptr;
    const float* mix = nullptr;
    float* ws = nullptr;
    Layout lay;
    int batch = 0;
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

static Layout make_layout(const Plan& P, int64_t B, bool training) {
    Layout l;
    l.off.assign(P.tensors.size(), -1);
    int64_t cur = 0;
    for (size_t i = 0; i < P.tensors.size(); ++i) {
        const TensorSpec& t = P.tensors[i];
        if (t.training_only && !training) continue;
        int64_t n = t.rows * t.C * (t.per_batch ? B : 1);
        l.off[i] = cur;
        cur += (n + 63) / 64 * 64;
    }
    l.total = cur + 64;
    return l;
}

// ------------------------------------------------------------------------------------------------
// materialisation of launch blocks
// ------------------------------------------------------------------------------------------------
static const float* tensor_ptr(const WunHandle* h, int tensor) {
    if (tensor == TENSOR_MIX) return h->mix;
    return h->ws + h->lay.off[tensor];
}

static void tensor_geom(const WunHandle* h, int tensor, int64_t* rows, int* C, bool* per_batch) {
    if (tensor == TENSOR_MIX) { *rows = h->plan.T_in; *C = h->plan.cfg.num_channels; *per_batch = true; return; }
    const TensorSpec& t = h->plan.tensors[tensor];
    *rows = t.rows; *C = t.C; *per_batch = t.per_batch;
}

static PlaneView make_plane(const WunHandle* h, const ViewSpec& v) {
    PlaneView p;
    memset(&p, 0, sizeof(p));
    int64_t rows; int C; bool pb;
    tensor_geom(h, v.tensor, &rows, &C, &pb);
    p.base = tensor_ptr(h, v.tensor) + (long long)v.row_offset * C;
    p.bstride = pb ? rows * C : 0;
    p.rstride = v.row_step * C;
    p.r_lo = v.r_lo; p.r_hi = v.r_hi; p.C = v.C;
    p.kind = v.kind; p.mid_mode = v.mid_mode; p.xrows = v.xrows;
    p.blend = (v.blend_tensor >= 0) ? tensor_ptr(h, v.blend_tensor) : nullptr;
    return p;
}

// the same geometry as `v`, but on another tensor (gradient twin / scratch) with explicit batch stride
static PlaneView make_plane_on(const WunHandle* h, const ViewSpec& v, int tensor, long long bstride, int r_lo, int r_hi) {
    PlaneView p;
    memset(&p, 0, sizeof(p));
    p.base = tensor_ptr(h, tensor) + (long long)v.row_offset * v.C;
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

// wun_debug_launches: one plane-convolution launch as text (addresses are raw integers relative to the fake bases the dry run
// installs: workspace 1 << 40, parameters 1 << 41, mix 1 << 42 - nothing is dereferenced).  tests/test_launch_semantics.py
// interprets these descriptions in numpy: the pair-merged form of a launch must compute exactly what its two-class form does.
static void export_launch(WunHandle* h, const ConvLaunch& L) {
    char line[768];
    auto addr = [](const void* p) { return (long long)reinterpret_cast<uintptr_t>(p); };
    snprintf(line, sizeof(line), "launch layer=%d pass=%d N=%d pairC=%d w_sk=%d w_sn=%d W=%lld bias=%lld epilogue=%d batch=%d nplanes=%d ncls=%d",
             h->cur_layer, h->cur_pass, L.N, L.pairC, L.w_sk, L.w_sn, addr(L.W), L.bias ? addr(L.bias) : -1LL, L.epilogue, L.batch, L.nplanes, L.ncls);
    h->export_launches->push_back(line);
    for (int p = 0; p < L.nplanes; ++p) {
        const PlaneView& P = L.planes[p];
        snprintf(line, sizeof(line), "plane i=%d base=%lld bstride=%lld rstride=%d r_lo=%d r_hi=%d C=%d kind=%d mid_mode=%d xrows=%d blend=%lld",
                 p, addr(P.base), P.bstride, P.rstride, P.r_lo, P.r_hi, P.C, P.kind, P.mid_mode, P.xrows, P.blend ? addr(P.blend) : -1LL);
        h->export_launches->push_back(line);
    }
    int nterm = 0;
    for (int q = 0; q < L.ncls; ++q) {
        const OutView& O = L.cls[q];
        nterm = std::max(nterm, O.term_end);
        snprintf(line, sizeof(line), "cls i=%d base=%lld bstride=%lld rstride=%d m_lo=%d m_hi=%d saved=%lld acc_lo=%d acc_hi=%d term_begin=%d term_end=%d "
                 "pairC=%d base2=%lld bstride2=%lld rstride2=%d saved2=%lld acc_lo2=%d acc_hi2=%d lo0=%d hi0=%d lo1=%d hi1=%d",
                 q, addr(O.base), O.bstride, O.rstride, O.m_lo, O.m_hi, O.saved ? addr(O.saved) : -1LL, O.acc_lo, O.acc_hi, O.term_begin, O.term_end,
                 O.pairC, O.pairC ? addr(O.base2) : -1LL, O.bstride2, O.rstride2, (O.pairC && O.saved2) ? addr(O.saved2) : -1LL, O.acc_lo2, O.acc_hi2,
                 O.lo_h[0], O.hi_h[0], O.lo_h[1], O.hi_h[1]);
        h->export_launches->push_back(line);
    }
    for (int t = 0; t < nterm; ++t) {
        snprintf(line, sizeof(line), "term i=%d plane=%d d=%d woff=%d woff2=%d", t, L.terms[t].plane, L.terms[t].d, L.terms[t].woff, L.pairC ? L.terms[t].woff2 : -1);
        h->export_launches->push_back(line);
    }
}

// Every plane convolution goes through here: tensor cores (wgmma) when the launch is eligible, CUDA cores otherwise.
static int launch_conv(WunHandle* h, const ConvLaunch& L) {
    if (h->dry && h->export_launches) export_launch(h, L);
    UmmaChoice ch;
    const bool use_umma = h->umma_enabled && h->umma_pass[h->cur_pass] && umma_plan_from_conv(L, &ch);
    const size_t slot = (size_t)h->cur_layer * 3 + h->cur_pass;
    if (h->dry && slot < h->kernel_used.size()) h->kernel_used[slot] = use_umma ? "umma" : "simt";
    if (use_umma) {
        if (h->fuse_out && h->debug_iters == 0 && umma_output_fusable(L, ch, h->fuse_out->O)) h->out_fused = true;
        if (h->phase != 1) h->launches += 2;    // weight pack + conv (counted once)
        if (h->dry) {
            h->arena_bytes = std::max(h->arena_bytes, std::max(ch.pack_bytes, h->pack_floor)); h->arena_sum += std::max(ch.pack_bytes, h->pack_floor);
            if (h->audit) {
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
                char line[512];
                snprintf(line, sizeof(line), "conv layer=%d pass=%d kernel=wgmma N=%d NPAD=%d nsplit=%d MT=%d rows_alloc=%d span=%d "
                         "TB=%d nbs=%d tiles=%lld mmas=%lld max_rows=%d smem=%zu pack_bytes=%zu pair=%d outfuse=%d",
                         h->cur_layer, h->cur_pass, L.N, ch.NPAD, ch.nsplit, ch.MT, ch.rows_alloc, span, ch.TB, ch.nbs, tiles, mmas,
                         max_rows, umma_choice_smem_bytes(ch), ch.pack_bytes, L.pairC,
                         (h->fuse_out && umma_output_fusable(L, ch, h->fuse_out->O)) ? 1 : 0);
                h->audit->push_back(line);
            }
            return WUN_OK;
        }
        uint8_t* arena = reinterpret_cast<uint8_t*>(h->ws + h->lay.total) + h->arena_cur;
        h->arena_cur += std::max(ch.pack_bytes, h->pack_floor);
        UmmaLaunch U; UmmaPackLaunch PL;
        cudaError_t e = umma_build(L, ch, arena, &U, &PL);
        if (e == cudaSuccess && h->phase != 2) e = launch_umma_pack(PL, (h->phase == 1) ? h->side : h->stream);
        const bool per_pack = h->pack_events_on && h->cur_pass == 0 && h->phase != 0;
        if (per_pack) {
            const int idx = h->pack_idx++;
            while ((int)h->pack_events.size() <= idx && e == cudaSuccess) {
                cudaEvent_t ev;
                e = cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
                if (e == cudaSuccess) h->pack_events.push_back(ev);
            }
            if (e == cudaSuccess && h->phase == 1) e = cudaEventRecord(h->pack_events[idx], h->side);
            if (e == cudaSuccess && h->phase == 2) e = cudaStreamWaitEvent(h->stream, h->pack_events[idx], 0);
        }
        if (e == cudaSuccess && h->phase != 1) {
            if (h->packs_pending && !per_pack) {   // first conv that needs ALL hoisted packs (with per-pack events: the first dgrad)
                e = cudaStreamWaitEvent(h->stream, h->packs_event, 0);
                h->packs_pending = false;
            }
            const int iters = (h->debug_iters > 0) ? h->debug_iters : 1;
            const OutputFuse* fuse = (h->fuse_out && h->debug_iters == 0 && umma_output_fusable(L, ch, h->fuse_out->O)) ? h->fuse_out : nullptr;
            if (fuse) h->out_fused = true;
            for (int i = 0; i < iters && e == cudaSuccess; ++i) e = launch_plane_conv_umma(U, h->stream, fuse);
        }
        if (e != cudaSuccess) return set_err(WUN_E_CUDA, std::string("tensor-core conv launch: ") + cudaGetErrorString(e));
        return WUN_OK;
    }
    if (h->phase == 1) return WUN_OK;
    ++h->launches;
    if (!h->dry) launch_plane_conv_simt(L, h->stream);
    return WUN_OK;
}

// The first down block in the form kernels_first.cu wants, if the op has exactly the shape plan.cpp builds for it: input =
// the caller's mix in two parity planes, class 0 = even full-rate rows -> dec0, class 1 = odd rows of the skip window -> odd0.
static bool first_layer_desc(const WunHandle* h, const ConvOp& op, FirstLayer* F) {
    if (!h->first_fast || op.planes.size() != 2 || op.classes.size() != 2) return false;
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
    F->x = h->mix; F->x_bstride = (long long)h->plan.T_in * C; F->T = (int)h->plan.T_in;
    F->k = op.k; F->pad_left = pad;
    F->dec = const_cast<float*>(tensor_ptr(h, c0.out.tensor)); F->dec_bstride = view_bstride(h, c0.out); F->Td = c0.m_hi;
    F->odd = const_cast<float*>(tensor_ptr(h, c1.out.tensor)); F->odd_bstride = view_bstride(h, c1.out);
    F->mo_lo = c1.m_lo; F->mo_hi = c1.m_hi;
    F->W = h->params + h->plan.params[op.w_param].offset;
    F->bias = h->params + h->plan.params[op.b_param].offset;
    F->batch = h->batch;
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
    return ctas >= h->pair_min_ctas;
}

static int conv_forward(WunHandle* h, const ConvOp& op, int layer_index) {
    h->cur_layer = layer_index; h->cur_pass = 0;
    if (layer_index == 0) {
        FirstLayer F;
        if (first_layer_desc(h, op, &F)) {
            if (h->phase == 1) return WUN_OK;
            ++h->launches;
            if (!h->dry) launch_first_fwd(F, h->plan.cfg.num_channels, op.cout, h->stream);
            return WUN_OK;
        }
    }
    ConvLaunch L;
    memset(&L, 0, sizeof(L));
    L.nplanes = (int)op.planes.size();
    for (int p = 0; p < L.nplanes; ++p) L.planes[p] = make_plane(h, op.planes[p]);
    L.ncls = (int)op.classes.size();
    int nt = 0, max_rows = 0;
    for (int q = 0; q < L.ncls; ++q) {
        const ClassSpec& c = op.classes[q];
        OutView& o = L.cls[q];
        PlaneView ov = make_plane(h, c.out);
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
    L.W = h->params + h->plan.params[op.w_param].offset;
    L.bias = h->params + h->plan.params[op.b_param].offset;
    L.epilogue = EPI_BIAS_LRELU; L.batch = h->batch; L.max_rows = max_rows;
    // the even / odd output rows of an up block (and of the bottleneck) read the same planes at the same shifts: one
    // pair-merged class of 2*cout columns (out tensor viewed as [B, rows/2, 2*cout]) - 6+6 taps instead of 2 x (5+5)
    ConvLaunch M;
    h->pack_floor = 0;
    if (h->pair_fwd && L.ncls == 2 && h->umma_enabled && h->umma_pass[0] && merge_pair(L, &M)) {
        UmmaChoice ch0, ch;
        const bool ok0 = umma_plan_from_conv(L, &ch0), ok1 = umma_plan_from_conv(M, &ch);
        if (ok0 && ok1) {
            h->pack_floor = std::max(ch0.pack_bytes, ch.pack_bytes);
            if (pair_worthwhile(h, M, ch)) L = M;
        }
    }
    const int rc = launch_conv(h, L);
    h->pack_floor = 0;
    return rc;
}

// dgrad: one class per forward input plane that needs a gradient; the forward classes' gradient
// tensors become the input planes.
static int conv_dgrad(WunHandle* h, const ConvOp& op, const OpBackward& ob, int layer_index) {
    if (ob.dgrad.empty()) return WUN_OK;
    h->cur_layer = layer_index; h->cur_pass = 1;
    const Plan& P = h->plan;
    ConvLaunch L;
    memset(&L, 0, sizeof(L));
    L.nplanes = (int)op.classes.size();
    for (int q = 0; q < L.nplanes; ++q) {
        const ClassSpec& c = op.classes[q];
        L.planes[q] = make_plane_on(h, c.out, P.grad_twin[c.out.tensor], view_bstride(h, c.out), c.m_lo, c.m_hi);
    }
    L.ncls = (int)ob.dgrad.size();
    int nt = 0, max_rows = 0;
    for (int k = 0; k < L.ncls; ++k) {
        const DgradClass& dc = ob.dgrad[k];
        const ViewSpec& v = op.planes[dc.plane];
        const int gt = op.plane_grad_tensor[dc.plane];
        long long bs = view_bstride(h, v);
        if (gt == P.t_gmid) bs = (long long)(v.r_hi - v.r_lo) * v.C;   // [B, nmid, C]
        PlaneView ov = make_plane_on(h, v, gt, bs, dc.r_lo, dc.r_hi);
        OutView& o = L.cls[k];
        o.base = const_cast<float*>(ov.base); o.bstride = ov.bstride; o.rstride = ov.rstride;
        o.m_lo = dc.r_lo; o.m_hi = dc.r_hi;
        o.saved = op.plane_slope[dc.plane] ? make_plane(h, v).base : nullptr;
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
    cudaEvent_t ev_fork = nullptr;          // recorded on the caller's stream before the first launch (see `par` below)
    if (h->dgrad_par && !h->dry && h->phase != 1 && h->use_side && h->side != nullptr && h->debug_iters == 0 && !h->packs_pending && L.ncls > 2) {
        while ((int)h->par_events.size() < h->par_used + 2) {
            cudaEvent_t e;
            WUN_CUDA_OK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
            h->par_events.push_back(e);
        }
        ev_fork = h->par_events[h->par_used];
        WUN_CUDA_OK(cudaEventRecord(ev_fork, h->stream));
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
        S.W = h->params + P.params[op.w_param].offset;
        S.bias = nullptr;
        // slope is per class (saved != null); classes without saved use EPI_PLAIN semantics via null check
        S.epilogue = EPI_SLOPE;
        S.batch = h->batch;
        if (S.max_rows <= 0) continue;
        // Pair merge: two classes of the same width (the even / odd input rows of a down block; the skip-even / skip-odd or
        // the copied / interpolated inputs of an up block) read the same gradient planes with the same row shifts.  As ONE
        // class of N = 2C columns every slab is staged once instead of twice and a tap costs one MMA instead of two (for
        // N <= 64 an MMA costs the same ~46 cycles whatever N is) - launch.h OutView::pairC.
        ConvLaunch M;
        // Measured (M4 batch 16, same-box A/B): down1 (2C = 48, fused-N MMAs) 368 -> 332 us; wider pairs lose the fused-N form and
        // got slower (down2 276 -> 317, down3 216 -> 250, down4 156 -> 183, up11 194 -> 215 us): their dgrad is bound by the
        // epilogue's slope / accumulate read-backs, not by slab fills or MMAs.
        const bool pair_on = h->pair_dgrad == 1 || (h->pair_dgrad == 2 && op.planes.size() == 2) || (h->pair_dgrad == 3 && op.planes.size() == 4) ||
                             (h->pair_dgrad == 4 && op.planes.size() == 2 && 2 * S.N <= 64);
        h->pack_floor = 0;
        if (h->pair_dgrad != 0 && S.ncls == 2 && h->umma_enabled && h->umma_pass[1] && merge_pair(S, &M)) {
            UmmaChoice ch0, ch;
            const bool ok0 = umma_plan_from_conv(S, &ch0), ok1 = umma_plan_from_conv(M, &ch);
            if (ok0 && ok1) {
                h->pack_floor = std::max(ch0.pack_bytes, ch.pack_bytes);
                if (pair_on && pair_worthwhile(h, M, ch)) S = M;
            }
        }
        // second (third ...) launch of this dgrad: on the helper stream, forked from the point the first launch was enqueued at
        const bool par = ev_fork != nullptr && n_launched > 0 && !h->dry && h->phase != 1 && h->use_side && h->side != nullptr &&
                         h->debug_iters == 0 && !h->packs_pending;
        cudaStream_t main_stream = h->stream;
        cudaEvent_t ev_join = nullptr;
        if (par) {
            if (!h->side2) WUN_CUDA_OK(cudaStreamCreateWithFlags(&h->side2, cudaStreamNonBlocking));
            while ((int)h->par_events.size() < h->par_used + 2) {
                cudaEvent_t e;
                WUN_CUDA_OK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
                h->par_events.push_back(e);
            }
            ev_join = h->par_events[h->par_used + 1];
            WUN_CUDA_OK(cudaStreamWaitEvent(h->side2, ev_fork, 0));
            h->stream = h->side2;
        }
        int rc = launch_conv(h, S);
        h->pack_floor = 0;
        if (par) {
            h->stream = main_stream;
            if (rc == WUN_OK) {
                WUN_CUDA_OK(cudaEventRecord(ev_join, h->side2));
                WUN_CUDA_OK(cudaStreamWaitEvent(main_stream, ev_join, 0));
            }
            h->par_used += 2;
        }
        if (rc != WUN_OK) return rc;
        ++n_launched;
    }
    return WUN_OK;
}

static int64_t split_arena_half_bytes(const WunHandle* h, int64_t batch) {
    return (int64_t)h->split_item_bytes * batch + 256 * (kSplitMaxJobs + 1) + (int64_t)h->wg_partial_bytes + 256;
}

static int64_t split_arena_bytes(const WunHandle* h, int64_t batch);
static float* out_part_ptr(const WunHandle* h);

static int conv_wgrad(WunHandle* h, const ConvOp& op, float* grads, float scale, int layer_index) {
    const Plan& P = h->plan;
    h->cur_layer = layer_index;
    if (layer_index == 0) {
        FirstWgrad FW;
        if (first_layer_desc(h, op, &FW.L)) {          // one launch: dW and db of both classes
            if (h->phase == 1) return WUN_OK;
            h->launches += 2;                             // per-CTA sums + their fixed-order total
            if (!h->dry) {
                FW.part = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(h->ws + h->lay.total) + h->arena_sum +
                                                   split_arena_bytes(h, h->batch));
                FW.L.dec = const_cast<float*>(tensor_ptr(h, P.grad_twin[op.classes[0].out.tensor]));
                FW.L.odd = const_cast<float*>(tensor_ptr(h, P.grad_twin[op.classes[1].out.tensor]));
                FW.dW = grads + P.params[op.w_param].offset;
                FW.db = grads + P.params[op.b_param].offset;
                FW.scale = scale; FW.rows_per_cta = 0;
                // the CUDA-core first-layer gradient is the tail of the step: on the split stream it runs next to the second
                // block's tensor-core wgrad instead of behind it (joined at the end of run_backward)
                static const bool tail_on = [] { const char* e = getenv("WUN_FIRST_TAIL"); return !(e && e[0] == '0'); }();
                const bool tail_par = tail_on && h->split_ahead && h->split_stream != nullptr && h->wstream != h->stream;
                launch_first_wgrad(FW, P.cfg.num_channels, op.cout, tail_par ? h->split_stream : h->wstream);
                if (tail_par) {
                    if (!h->first_done) WUN_CUDA_OK(cudaEventCreateWithFlags(&h->first_done, cudaEventDisableTiming));
                    WUN_CUDA_OK(cudaEventRecord(h->first_done, h->split_stream));
                    h->first_pending = true;
                }
            }
            return WUN_OK;
        }
    }
    // collect (class, plane) groups
    std::vector<WgradLaunch> groups;
    std::vector<PlaneView> class_dpre;
    for (const auto& c : op.classes) {
        if (c.m_hi <= c.m_lo) continue;
        PlaneView dpre = make_plane_on(h, c.out, P.grad_twin[c.out.tensor], view_bstride(h, c.out), c.m_lo, c.m_hi);
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
            W.plane = make_plane(h, op.planes[p]);
            W.dpre = dpre;
            W.m_lo = c.m_lo; W.m_hi = c.m_hi;
            W.N = op.cout; W.w_sk = op.cout; W.w_sn = 1;
            W.dW = grads + P.params[op.w_param].offset;
            W.scale = scale; W.batch = h->batch;
            groups.push_back(W);
        }
    }
    if (h->dry && h->export_launches) {      // wun_debug_launches: the (class, plane) groups of this layer's weight gradient
        char line[512];
        auto addr = [](const void* p) { return (long long)reinterpret_cast<uintptr_t>(p); };
        for (size_t g = 0; g < groups.size(); ++g) {
            const WgradLaunch& W = groups[g];
            snprintf(line, sizeof(line), "wgrad layer=%d group=%d N=%d w_sk=%d w_sn=%d dW=%lld db=%lld m_lo=%d m_hi=%d nterms=%d batch=%d",
                     layer_index, (int)g, W.N, W.w_sk, W.w_sn, (long long)P.params[op.w_param].offset, (long long)P.params[op.b_param].offset,
                     W.m_lo, W.m_hi, W.nterms, W.batch);
            h->export_launches->push_back(line);
            const PlaneView* V[2] = {&W.plane, &W.dpre};
            for (int k = 0; k < 2; ++k) {
                snprintf(line, sizeof(line), "%s base=%lld bstride=%lld rstride=%d r_lo=%d r_hi=%d C=%d kind=%d mid_mode=%d xrows=%d blend=%lld",
                         k == 0 ? "wplane" : "wdpre", addr(V[k]->base), V[k]->bstride, V[k]->rstride, V[k]->r_lo, V[k]->r_hi, V[k]->C, V[k]->kind,
                         V[k]->mid_mode, V[k]->xrows, V[k]->blend ? addr(V[k]->blend) : -1LL);
                h->export_launches->push_back(line);
            }
            for (int t = 0; t < W.nterms; ++t) {
                snprintf(line, sizeof(line), "wterm i=%d d=%d woff=%d", t, W.d[t], W.woff[t]);
                h->export_launches->push_back(line);
            }
        }
    }
    // tensor cores: all groups of the layer in ONE launch
    bool use_umma = h->umma_enabled && h->umma_pass[2] && !groups.empty() && groups.size() <= (size_t)kWgMaxGroups;
    UmmaWgradLaunch U;
    if (use_umma) {
        memset(&U, 0, sizeof(U));
        U.ngroups = (int)groups.size(); U.batch = h->batch; U.dW = groups[0].dW;
        U.w_sp = op.cout; U.w_sg = 1; U.scale = scale;
        for (size_t g = 0; g < groups.size(); ++g) {
            WgGroup& G = U.grp[g];
            G.P = groups[g].plane; G.G = groups[g].dpre; G.m_lo = groups[g].m_lo; G.m_hi = groups[g].m_hi;
            G.ntaps = groups[g].nterms;
            for (int t = 0; t < G.ntaps; ++t) { G.d[t] = groups[g].d[t]; G.woff[t] = groups[g].woff[t]; }
        }
        use_umma = umma_plan_wgrad(&U);
    }
    const size_t slot = (size_t)h->cur_layer * 3 + 2;
    if (h->dry && slot < h->kernel_used.size()) h->kernel_used[slot] = use_umma ? "umma" : "simt";
    if (h->dry && h->audit && use_umma) {
        for (int g = 0; g < U.ngroups; ++g) {
            const WgGroup& G = U.grp[g];
            char line[512];
            snprintf(line, sizeof(line), "wgrad layer=%d group=%d Cp=%d Cg=%d swap=%d NT=%d mtiles=%d ntiles=%d ntaps=%d taps_per_cta=%d "
                     "tapsets=%d chunks_per_cta=%d n_ctas_x=%d chunks=%lld grid=%dx%dx%d nstages=%d smem=%zu issued_macs=%lld useful_macs=%lld",
                     h->cur_layer, g, G.P.C, G.G.C, G.swap, G.NT, G.n_mtiles, G.n_ntiles, G.ntaps, G.taps_per_cta, G.n_tapsets,
                     G.chunks_per_cta, G.n_ctas_x, (long long)U.batch * G.chunks_per_batch, U.grid_x, U.grid_y, U.grid_z, U.nstages, umma_wgrad_smem_bytes(U),
                     umma_wgrad_issued_macs(G, U.batch), (long long)U.batch * G.chunks_per_batch * 64 * G.ntaps * G.P.C * G.G.C);
            h->audit->push_back(line);
        }
    }
    if (h->phase == 1) return WUN_OK;
    float* bias_grad = grads ? grads + P.params[op.b_param].offset : nullptr;
    auto colsum_launches = [&]() {                        // bias gradient by its own kernel (paths without a split pass)
        for (const auto& dp : class_dpre) {
            ++h->launches;
            if (!h->dry) launch_colsum(dp, h->batch, scale, bias_grad, h->wstream);
        }
    };
    if (use_umma) {
        ++h->launches;
        const size_t split_need = h->bulk_wgrad ? umma_plan_wgrad_split(U, 1, nullptr, nullptr, nullptr) : 0;
        const bool bulk = split_need > 0;                 // 0: too many distinct views for one split pass -> converter-fed kernel
        // Bias column sums inside the split pass instead of their own launches (WUN_SPLIT_COLSUM: 1 = default, 0 = separate colsum
        // launches, 2 = fused only for the layers with few rows).  History: while the dgrad chain was the critical path the separate
        // launches were 0.05 ms faster per step (they fill SMs the big-shared-memory kernels leave thread slots on); since the epilogue
        // work of round 2 the wgrad stream is the critical path and the fused form wins (5.45 -> 5.39 ms, wgrad family 2.52 -> 2.24 ms).
        static const int colsum_mode = [] { const char* e = getenv("WUN_SPLIT_COLSUM"); return e ? atoi(e) : 1; }();
        int max_rows_g = 0;
        for (const auto& dp : class_dpre) max_rows_g = std::max(max_rows_g, dp.r_hi - dp.r_lo);
        const bool fused_colsum = colsum_mode == 1 || (colsum_mode == 2 && max_rows_g <= 4096);
        if (bulk) {      // + the split pass and the fixed-order reduction of the partial tiles / column sums
            h->launches += 2;
            if (h->dry) {
                h->split_item_bytes = std::max(h->split_item_bytes, split_need);
                h->wg_partial_bytes = std::max(h->wg_partial_bytes, umma_wgrad_partial_bytes(U));
            }
        }
        if (!bulk || !fused_colsum) colsum_launches();
        if (!h->dry) {
            cudaError_t e;
            if (bulk) {
                const bool ahead = h->split_ahead && h->split_stream != nullptr && h->wstream != h->stream;
                uint8_t* arena = reinterpret_cast<uint8_t*>(h->ws + h->lay.total) + h->arena_sum;
                if (ahead && (h->wg_index & 1)) arena += split_arena_half_bytes(h, h->batch);
                arena += (256 - (reinterpret_cast<uintptr_t>(arena) & 255)) & 255;
                // split arrays, then the partial tiles, in this half; the class-gradient views among the jobs also produce the
                // bias gradient (their column sums)
                WgSplit S; SplitJobs J;
                if (!umma_wgrad_bulk_setup(&U, h->batch, arena, class_dpre.data(), (int)class_dpre.size(), fused_colsum ? bias_grad : nullptr,
                                           scale, &S, &J))
                    return set_err(WUN_E_INVALID, "wgrad split pass: class gradient view not among the split jobs");
                if (ahead) {
                    const int k = h->wg_index++;
                    while ((int)h->split_done.size() <= k) {
                        cudaEvent_t e1, e2;
                        WUN_CUDA_OK(cudaEventCreateWithFlags(&e1, cudaEventDisableTiming));
                        WUN_CUDA_OK(cudaEventCreateWithFlags(&e2, cudaEventDisableTiming));
                        h->split_done.push_back(e1); h->wg_done.push_back(e2);
                    }
                    if (k >= 2) WUN_CUDA_OK(cudaStreamWaitEvent(h->split_stream, h->wg_done[k - 2], 0));     // its arena half is free again
                    e = launch_split_views(J, h->split_stream);
                    if (e == cudaSuccess) e = cudaEventRecord(h->split_done[k], h->split_stream);
                    if (e == cudaSuccess) e = cudaStreamWaitEvent(h->wstream, h->split_done[k], 0);
                    if (e == cudaSuccess) e = launch_wgrad_umma_bulk(U, S, h->wstream);
                    if (e == cudaSuccess) e = launch_wgrad_reduce(U, J, h->wstream);
                    if (e == cudaSuccess) e = cudaEventRecord(h->wg_done[k], h->wstream);
                } else {
                    e = launch_split_views(J, h->wstream);      // same stream as the wgrad: the arena is reused layer after layer
                    if (e == cudaSuccess) e = launch_wgrad_umma_bulk(U, S, h->wstream);
                    if (e == cudaSuccess) e = launch_wgrad_reduce(U, J, h->wstream);
                }
            } else {
                e = launch_wgrad_umma(U, h->wstream);
            }
            if (e != cudaSuccess) return set_err(WUN_E_CUDA, std::string("tensor-core wgrad launch: ") + cudaGetErrorString(e));
        }
        return WUN_OK;
    }
    colsum_launches();
    for (const auto& W : groups) {
        ++h->launches;
        if (!h->dry) launch_plane_wgrad_simt(W, h->wstream);
    }
    return WUN_OK;
}

static int ensure_side(WunHandle* h) {
    if (!h->side) {
        WUN_CUDA_OK(cudaStreamCreateWithFlags(&h->side, cudaStreamNonBlocking));
        WUN_CUDA_OK(cudaEventCreateWithFlags(&h->join_event, cudaEventDisableTiming));
        WUN_CUDA_OK(cudaEventCreateWithFlags(&h->packs_event, cudaEventDisableTiming));
    }
    return WUN_OK;
}

// fork: everything enqueued on the main stream so far is visible to the side stream
static int fork_side(WunHandle* h) {
    if (h->dry || h->phase == 1 || h->wstream == h->stream) return WUN_OK;
    if (h->fork_used >= (int)h->fork_events.size()) {
        cudaEvent_t e;
        WUN_CUDA_OK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        h->fork_events.push_back(e);
    }
    cudaEvent_t ev = h->fork_events[h->fork_used++];
    WUN_CUDA_OK(cudaEventRecord(ev, h->stream));
    WUN_CUDA_OK(cudaStreamWaitEvent(h->side, ev, 0));
    if (h->split_ahead) {
        if (!h->split_stream) WUN_CUDA_OK(cudaStreamCreateWithFlags(&h->split_stream, cudaStreamNonBlocking));
        WUN_CUDA_OK(cudaStreamWaitEvent(h->split_stream, ev, 0));
    }
    return WUN_OK;
}

// Every gradient at a flat offset >= `ready_from` has been enqueued (side-stream work in order, main-stream work up to the
// last fork): record the events of the buckets this completes.  Called right after a fork (side waits for main) or at the end.
static int mark_grads_ready(WunHandle* h, int64_t ready_from, cudaStream_t on) {
    if (h->dry || h->phase == 1) return WUN_OK;
    while (h->bucket_next < (int)h->bucket_first.size() && h->bucket_first[h->bucket_next] >= ready_from) {
        WUN_CUDA_OK(cudaEventRecord(h->bucket_events[h->bucket_next], on));
        ++h->bucket_next;
    }
    return WUN_OK;
}

static int64_t op_first_offset(const Plan& P, const ConvOp& op, const UpsampleSpec* us) {
    int64_t o = std::min(P.params[op.w_param].offset, P.params[op.b_param].offset);
    if (us && us->interp_param >= 0) o = std::min<int64_t>(o, P.params[us->interp_param].offset);
    return o;
}

static void fill_output_launch(const WunHandle* h, OutputLaunch* O, const float* targets, float* outputs, float* loss,
                               int training) {
    const Plan& P = h->plan;
    memset(O, 0, sizeof(*O));
    O->params = h->params;
    for (int s = 0; s < P.nconv; ++s) {
        O->w_off[s] = P.params[P.out_w_param[s]].offset;
        O->b_off[s] = P.params[P.out_b_param[s]].offset;
    }
    O->mix = h->mix;
    O->feat = tensor_ptr(h, P.t_feat);
    O->targets = targets;
    O->outputs = outputs;
    O->dpre = (h->lay.off[P.t_dpre_out] >= 0) ? const_cast<float*>(tensor_ptr(h, P.t_dpre_out)) : nullptr;
    O->loss = loss;
    O->batch = h->batch; O->T_in = (int)P.T_in; O->Tf = (int)P.Tf; O->T_out = (int)P.T_out;
    O->C = P.cfg.num_channels; O->F = P.cfg.num_initial_filters;
    O->nconv = P.nconv; O->K = P.cfg.num_sources;
    O->ofs = P.cfg.output_filter_size; O->pad_left = P.out_pad_left;
    O->crop_feat = P.crop_feat; O->crop_out = P.crop_out;
    O->output_type = P.cfg.output_type; O->activation = P.cfg.output_activation; O->training = training;
    O->inv_count = 1.0f / (float)((double)h->batch * P.T_out * P.cfg.num_channels * P.cfg.num_sources);
}

static int run_forward(WunHandle* h, const float* targets, float* outputs, float* loss, int training) {
    const Plan& P = h->plan;
    const int L = P.cfg.num_layers;
    for (int i = 0; i < L; ++i) {
        const UpsampleSpec& us = P.ups[i];
        if (us.interp_param >= 0) {
            if (h->phase != 1) ++h->launches;
            if (!h->dry && h->phase != 1)
                launch_sigmoid(h->params + P.params[us.interp_param].offset,
                               const_cast<float*>(tensor_ptr(h, us.wsig_tensor)), us.C, h->stream);
        }
    }
    int rc;
    for (int i = 0; i < L; ++i)
        if ((rc = conv_forward(h, P.down[i], i)) != WUN_OK) return rc;
    if ((rc = conv_forward(h, P.bottleneck, L)) != WUN_OK) return rc;
    OutputLaunch O;
    fill_output_launch(h, &O, targets, outputs, loss, training);
    OutputFuse OF;
    memset(&OF, 0, sizeof(OF));
    h->out_fused = false;
    for (int i = 0; i < L; ++i) {
        if (i == L - 1 && h->out_fuse_mode != 0 && P.cfg.output_filter_size == 1) {
            // the output layer rides in this conv's epilogue when the planner picks the persistent kernel for it
            OF.O = O;
            const bool bw = targets != nullptr && h->bw_grads != nullptr;
            OF.gfeat = bw ? const_cast<float*>(tensor_ptr(h, P.grad_twin[P.t_feat])) : nullptr;
            OF.grads = (bw && h->out_fuse_mode == 2) ? h->bw_grads : nullptr;
            OF.grad_scale = h->bw_scale;
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
            if (geom && (targets == nullptr || bw)) h->fuse_out = &OF;       // (loss without gradients: the separate kernel)
        }
        rc = conv_forward(h, P.up[i], L + 1 + i);
        h->fuse_out = nullptr;
        if (rc != WUN_OK) return rc;
    }
    if (h->out_fused) return WUN_OK;
    if (h->phase != 1) ++h->launches;
    if (!h->dry && h->phase != 1) launch_output_fwd(O, h->stream);
    return WUN_OK;
}

static int run_backward(WunHandle* h, const float* targets, float* grads, float scale) {
    const Plan& P = h->plan;
    const int L = P.cfg.num_layers;
    int rc;
    h->wstream = h->stream;
    if (h->phase != 1) h->fork_used = (h->phase == 2) ? 1 : 0;
    if (!h->dry && h->use_side) {
        int rcs = ensure_side(h);
        if (rcs != WUN_OK) return rcs;
        h->wstream = h->side;
    }
    OutputLaunch O;
    fill_output_launch(h, &O, targets, nullptr, nullptr, 1);
    // fused forward (run_forward): dL/dpre and the feature gradient already exist; only the output convs' weight gradient is left
    // (mode 1), and it goes to the wgrad stream right after the first fork below
    const bool out_wgrad_late = h->out_fused && h->out_fuse_mode != 2;
    if (h->dry) h->out_part_bytes = std::max(h->out_part_bytes, output_wgrad_partial_bytes(O));
    if (h->phase != 1 && !h->out_fused) h->launches += 3;
    if (h->phase != 1 && out_wgrad_late) h->launches += 2;
    if (!h->dry && h->phase != 1 && !h->out_fused) {
        launch_output_wgrad(O, grads, out_part_ptr(h), scale, h->stream);
        launch_output_dgrad(O, const_cast<float*>(tensor_ptr(h, P.grad_twin[P.t_feat])), h->stream);
    }
    if (h->phase != 1) h->bucket_next = 0;
    int64_t ready_from = h->plan.param_numel;      // lowest flat offset whose gradient is complete once the next fork is passed
    if (P.nconv > 0) ready_from = std::min<int64_t>(P.params[P.out_w_param[0]].offset, P.params[P.out_b_param[0]].offset);
    for (int i = L - 1; i >= 0; --i) {
        const ConvOp& op = P.up[i];
        if ((rc = fork_side(h)) != WUN_OK) return rc;
        if (i == L - 1 && out_wgrad_late && !h->dry && h->phase != 1) launch_output_wgrad(O, grads, out_part_ptr(h), scale, h->wstream);
        if ((rc = mark_grads_ready(h, ready_from, h->wstream)) != WUN_OK) return rc;
        ready_from = std::min(ready_from, op_first_offset(P, op, &P.ups[i]));
        if ((rc = conv_wgrad(h, op, grads, scale, L + 1 + i)) != WUN_OK) return rc;
        if ((rc = conv_dgrad(h, op, h->bwd_up[i], L + 1 + i)) != WUN_OK) return rc;
        const UpsampleSpec& us = P.ups[i];
        UpsampleBwdLaunch U;
        memset(&U, 0, sizeof(U));
        U.due = tensor_ptr(h, P.t_gue);
        U.dmid = tensor_ptr(h, P.t_gmid);
        U.x = tensor_ptr(h, us.src_tensor);
        U.gx = const_cast<float*>(tensor_ptr(h, P.grad_twin[us.src_tensor]));
        U.blend = (us.wsig_tensor >= 0) ? tensor_ptr(h, us.wsig_tensor) : nullptr;
        U.dvar = (us.interp_param >= 0) ? grads + P.params[us.interp_param].offset : nullptr;
        U.batch = h->batch; U.N = us.N; U.nmid = us.nmid; U.C = us.C; U.mid_mode = us.mid_mode; U.scale = scale;
        if (h->phase != 1) ++h->launches;
        if (!h->dry && h->phase != 1) launch_upsample_bwd(U, h->stream);
    }
    if ((rc = fork_side(h)) != WUN_OK) return rc;
    if ((rc = mark_grads_ready(h, ready_from, h->wstream)) != WUN_OK) return rc;
    ready_from = std::min(ready_from, op_first_offset(P, P.bottleneck, nullptr));
    if ((rc = conv_wgrad(h, P.bottleneck, grads, scale, L)) != WUN_OK) return rc;
    if ((rc = conv_dgrad(h, P.bottleneck, h->bwd_bottleneck, L)) != WUN_OK) return rc;
    for (int i = L - 1; i >= 0; --i) {
        if ((rc = fork_side(h)) != WUN_OK) return rc;
        if ((rc = mark_grads_ready(h, ready_from, h->wstream)) != WUN_OK) return rc;
        ready_from = std::min(ready_from, op_first_offset(P, P.down[i], nullptr));
        if ((rc = conv_wgrad(h, P.down[i], grads, scale, i)) != WUN_OK) return rc;
        if ((rc = conv_dgrad(h, P.down[i], h->bwd_down[i], i)) != WUN_OK) return rc;
    }
    if (!h->dry && h->phase != 1 && h->wstream != h->stream) {       // join: the caller's stream continues only after all wgrads
        WUN_CUDA_OK(cudaEventRecord(h->join_event, h->side));
        WUN_CUDA_OK(cudaStreamWaitEvent(h->stream, h->join_event, 0));
        if (h->first_pending) { WUN_CUDA_OK(cudaStreamWaitEvent(h->stream, h->first_done, 0)); h->first_pending = false; }
    }
    if ((rc = mark_grads_ready(h, 0, h->stream)) != WUN_OK) return rc;    // whatever is left: final after the join
    return WUN_OK;
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

// bytes of the split arena behind the weight packs (bulk-fed wgrad only; per-item size from the dry run at create time)
static int64_t split_arena_bytes(const WunHandle* h, int64_t batch) {
    return (h && h->bulk_wgrad && h->split_item_bytes) ? 2 * split_arena_half_bytes(h, batch) : 0;     // two halves
}
// training scratch behind the activations, the weight packs and the split arena: the first layer's per-CTA gradient sums
static int64_t train_scratch_bytes(const WunHandle* h, int64_t batch) {
    return split_arena_bytes(h, batch) + (int64_t)first_wgrad_partial_bytes((int)batch) + (int64_t)h->out_part_bytes;
}
// the output layer's per-CTA weight-gradient sums, behind the first layer's
static float* out_part_ptr(const WunHandle* h) {
    return reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(h->ws + h->lay.total) + h->arena_sum + split_arena_bytes(h, h->batch) +
                                    first_wgrad_partial_bytes(h->batch));
}

static int begin_call(WunHandle* h, const float* params, const float* mix, int64_t batch, bool training, void* ws,
                      int64_t ws_bytes, void* stream, bool dry) {
    if (!h) return set_err(WUN_E_INVALID, "null handle");
    if (batch < 1 || batch > (1 << 20)) return set_err(WUN_E_INVALID, "batch out of range");
    h->lay = make_layout(h->plan, batch, training);
    h->dry = dry;
    h->launches = 0;
    h->batch = (int)batch;
    h->bw_grads = nullptr; h->bw_scale = 1.f; h->fuse_out = nullptr; h->out_fused = false; h->par_used = 0; h->wg_index = 0; h->first_pending = false;
    if (dry) return WUN_OK;
    { int rc0 = check_device(); if (rc0 != WUN_OK) return rc0; }
    if (!params || !mix || !ws) return set_err(WUN_E_INVALID, "null device pointer");
    if (ws_bytes < h->lay.total * (int64_t)sizeof(float) + (int64_t)h->arena_sum + (training ? train_scratch_bytes(h, batch) : 0))
        return set_err(WUN_E_INVALID, "workspace too small");
    if (reinterpret_cast<uintptr_t>(ws) % 256 != 0) return set_err(WUN_E_INVALID, "workspace must be 256-byte aligned");
    h->params = params; h->mix = mix; h->ws = (float*)ws; h->stream = (cudaStream_t)stream;
    return WUN_OK;
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
    const char* dis = getenv("WUN_DISABLE_UMMA");
    h->umma_enabled = !(dis && dis[0] == '1');
    { const char* names[3] = {"WUN_UMMA_FWD", "WUN_UMMA_DGRAD", "WUN_UMMA_WGRAD"};
      for (int i = 0; i < 3; ++i) { const char* v = getenv(names[i]); h->umma_pass[i] = !(v && v[0] == '0'); } }
    { const char* v = getenv("WUN_SIDE_STREAM"); h->use_side = !(v && v[0] == '0'); }
    // "=0" selects the generic path for A/B runs
    { const char* v = getenv("WUN_FIRST_LAYER"); h->first_fast = !(v && v[0] == '0'); }
    { const char* v = getenv("WUN_PACK_EVENTS"); h->pack_events_on = !(v && v[0] == '0'); }
    { const char* v = getenv("WUN_BULK_WGRAD"); h->bulk_wgrad = !(v && v[0] == '0'); }
    { const char* v = getenv("WUN_PAIR_DGRAD"); h->pair_dgrad = v ? atoi(v) : 4; }
    { const char* v = getenv("WUN_DGRAD_PAR"); h->dgrad_par = !(v && v[0] == '0'); }
    { const char* v = getenv("WUN_SPLIT_AHEAD"); h->split_ahead = !(v && v[0] == '0'); }
    { const char* v = getenv("WUN_PAIR_MIN_CTAS"); h->pair_min_ctas = v ? atoi(v) : 120; }
    { const char* v = getenv("WUN_OUT_FUSE"); h->out_fuse_mode = v ? atoi(v) : 1; }
    { const char* v = getenv("WUN_PAIR_FWD"); h->pair_fwd = !(v && v[0] == '0'); }
    h->kernel_used.assign((size_t)(2 * h->plan.cfg.num_layers + 1) * 3, "simt");
    // dry run: which kernel each layer uses and how much pack scratch the tensor-core launches need
    wun_launches_forward_backward(h);
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
        for (auto e : h->fork_events) cudaEventDestroy(e);
        if (h->join_event) cudaEventDestroy(h->join_event);
        if (h->packs_event) cudaEventDestroy(h->packs_event);
        for (auto e : h->pack_events) cudaEventDestroy(e);
        for (auto e : h->bucket_events) cudaEventDestroy(e);
        if (h->side) cudaStreamDestroy(h->side);
        if (h->side2) cudaStreamDestroy(h->side2);
        if (h->split_stream) cudaStreamDestroy(h->split_stream);
        for (auto e : h->split_done) cudaEventDestroy(e);
        for (auto e : h->wg_done) cudaEventDestroy(e);
        if (h->first_done) cudaEventDestroy(h->first_done);
        for (auto e : h->par_events) cudaEventDestroy(e);
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
    Layout l = make_layout(h->plan, batch, training != 0);
    return l.total * (int64_t)sizeof(float) + (int64_t)h->arena_sum + 256 + (training ? train_scratch_bytes(h, batch) : 0);
}

double wun_forward_flops(const WunHandle* h, int64_t batch) { return h ? h->plan.fwd_flops_per_item * batch : 0; }
double wun_forward_backward_flops(const WunHandle* h, int64_t batch) {
    return h ? (3.0 * h->plan.fwd_flops_per_item - h->plan.dgrad0_flops_per_item) * batch : 0;
}

int64_t wun_launches_forward(const WunHandle* hc) {
    WunHandle* h = const_cast<WunHandle*>(hc);
    if (begin_call(h, nullptr, nullptr, 1, false, nullptr, 0, nullptr, true) != WUN_OK) return -1;
    const size_t keep = h->arena_sum;
    h->phase = 0;
    run_forward(h, nullptr, nullptr, nullptr, 0);
    h->arena_sum = keep;
    return h->launches;
}

int64_t wun_launches_forward_backward(const WunHandle* hc) {
    WunHandle* h = const_cast<WunHandle*>(hc);
    if (begin_call(h, nullptr, nullptr, 1, true, nullptr, 0, nullptr, true) != WUN_OK) return -1;
    h->arena_sum = 0; h->phase = 0;
    run_forward(h, nullptr, nullptr, nullptr, 1);
    run_backward(h, nullptr, nullptr, 1.f);
    return h->launches;
}

int wun_forward(WunHandle* h, const float* params, const float* mix, int64_t batch, int training, float* outputs,
                void* workspace, int64_t workspace_bytes, void* stream) {
    int rc = begin_call(h, params, mix, batch, false, workspace, workspace_bytes, stream, false);
    if (rc != WUN_OK) return rc;
    if (!outputs) return set_err(WUN_E_INVALID, "outputs is null");
    h->phase = 0; h->arena_cur = 0;
    rc = run_forward(h, nullptr, outputs, nullptr, training);
    if (rc != WUN_OK) return rc;
    WUN_CUDA_OK(cudaGetLastError());
    return WUN_OK;
}

int wun_forward_backward(WunHandle* h, const float* params, const float* mix, const float* targets, int64_t batch,
                         float* outputs, float* loss, float* grads, float grad_scale, void* workspace,
                         int64_t workspace_bytes, void* stream) {
    int rc = begin_call(h, params, mix, batch, true, workspace, workspace_bytes, stream, false);
    if (rc != WUN_OK) return rc;
    if (!targets || !loss || !grads) return set_err(WUN_E_INVALID, "targets/loss/grads must not be null");
    WUN_CUDA_OK(cudaMemsetAsync(loss, 0, sizeof(float), h->stream));
    WUN_CUDA_OK(cudaMemsetAsync(grads, 0, sizeof(float) * h->plan.param_numel, h->stream));
    h->bw_grads = grads; h->bw_scale = grad_scale;
    if (h->use_side && h->umma_enabled) {
        // phase 1: every weight pack of the step on the side stream, behind the work already enqueued on `stream`
        rc = ensure_side(h);
        if (rc != WUN_OK) return rc;
        if (h->fork_events.empty()) { cudaEvent_t e; WUN_CUDA_OK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming)); h->fork_events.push_back(e); }
        WUN_CUDA_OK(cudaEventRecord(h->fork_events[0], h->stream));
        WUN_CUDA_OK(cudaStreamWaitEvent(h->side, h->fork_events[0], 0));
        h->phase = 1; h->arena_cur = 0; h->pack_idx = 0;
        rc = run_forward(h, targets, outputs, loss, 1);
        if (rc == WUN_OK) rc = run_backward(h, targets, grads, grad_scale);
        h->phase = 0;
        if (rc != WUN_OK) return rc;
        WUN_CUDA_OK(cudaEventRecord(h->packs_event, h->side));
        h->packs_pending = true;
        h->phase = 2;
    }
    h->arena_cur = 0; h->pack_idx = 0;
    rc = run_forward(h, targets, outputs, loss, 1);
    if (rc == WUN_OK) rc = run_backward(h, targets, grads, grad_scale);
    h->phase = 0;
    if (rc != WUN_OK) return rc;
    if (h->packs_pending) {                     // no tensor-core conv consumed the packs: still join the side stream
        WUN_CUDA_OK(cudaStreamWaitEvent(h->stream, h->packs_event, 0));
        h->packs_pending = false;
    }
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
    while ((int)h->bucket_events.size() < n) {
        cudaEvent_t e;
        WUN_CUDA_OK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        h->bucket_events.push_back(e);
    }
    h->bucket_first.assign(first_offset, first_offset + n);
    h->bucket_next = 0;
    return WUN_OK;
}

int wun_stream_wait_grad_bucket(WunHandle* h, int k, void* stream) {
    if (!h || k < 0 || k >= (int)h->bucket_first.size()) return set_err(WUN_E_INVALID, "no such gradient bucket");
    WUN_CUDA_OK(cudaStreamWaitEvent((cudaStream_t)stream, h->bucket_events[k], 0));
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
    if (buf && capacity > 0) {
        int64_t n = std::min<int64_t>(capacity - 1, (int64_t)s.size());
        memcpy(buf, s.data(), n);
        buf[n] = 0;
    }
    return (int64_t)s.size() + 1;
}

int64_t wun_debug_plan(const WunHandle* hc, int64_t batch, char* buf, int64_t capacity) {
    WunHandle* h = const_cast<WunHandle*>(hc);
    if (!h || batch < 1) return -1;
    std::vector<std::string> lines;
    const size_t keep_sum = h->arena_sum, keep_max = h->arena_bytes;
    const std::vector<std::string> keep_used = h->kernel_used;
    if (begin_call(h, nullptr, nullptr, batch, true, nullptr, 0, nullptr, true) != WUN_OK) return -1;
    h->audit = &lines; h->phase = 0;
    run_forward(h, nullptr, nullptr, nullptr, 1);
    run_backward(h, nullptr, nullptr, 1.f);
    h->audit = nullptr;
    h->arena_sum = keep_sum; h->arena_bytes = keep_max; h->kernel_used = keep_used;
    std::string s;
    for (const auto& l : lines) { s += l; s += "\n"; }
    if (buf && capacity > 0) {
        int64_t n = std::min<int64_t>(capacity - 1, (int64_t)s.size());
        memcpy(buf, s.data(), n);
        buf[n] = 0;
    }
    return (int64_t)s.size() + 1;
}

int64_t wun_debug_launches(const WunHandle* hc, int64_t batch, char* buf, int64_t capacity) {
    WunHandle* h = const_cast<WunHandle*>(hc);
    if (!h || batch < 1) return -1;
    std::vector<std::string> lines;
    const size_t keep_sum = h->arena_sum, keep_max = h->arena_bytes;
    const std::vector<std::string> keep_used = h->kernel_used;
    if (begin_call(h, nullptr, nullptr, batch, true, nullptr, 0, nullptr, true) != WUN_OK) return -1;
    h->export_launches = &lines; h->phase = 0;
    // fake, far-apart bases (never dereferenced in a dry run): every exported address identifies its buffer
    h->ws = reinterpret_cast<float*>((uintptr_t)1 << 40); h->params = reinterpret_cast<const float*>((uintptr_t)1 << 41);
    h->mix = reinterpret_cast<const float*>((uintptr_t)1 << 42);
    run_forward(h, nullptr, nullptr, nullptr, 1);
    run_backward(h, nullptr, nullptr, 1.f);
    h->export_launches = nullptr; h->ws = nullptr; h->params = nullptr; h->mix = nullptr;
    h->arena_sum = keep_sum; h->arena_bytes = keep_max; h->kernel_used = keep_used;
    std::string s;
    for (const auto& l : lines) { s += l; s += "\n"; }
    if (buf && capacity > 0) {
        int64_t n = std::min<int64_t>(capacity - 1, (int64_t)s.size());
        memcpy(buf, s.data(), n);
        buf[n] = 0;
    }
    return (int64_t)s.size() + 1;
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
    int rc = begin_call(h, params, mix, batch, true, workspace, workspace_bytes, stream, false);
    if (rc != WUN_OK) return rc;
    const ConvOp& op = (layer < L) ? h->plan.down[layer] : (layer == L ? h->plan.bottleneck : h->plan.up[layer - L - 1]);
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
    h->phase = 0; h->arena_cur = 0; h->wstream = h->stream;
    if (pass == 0) {
        h->debug_iters = iters;
        rc = conv_forward(h, op, layer);
        h->debug_iters = 0;
    } else {
        for (int i = 0; i < iters && rc == WUN_OK; ++i) {
            h->arena_cur = 0;
            rc = (pass == 1) ? conv_dgrad(h, op, ob, layer) : conv_wgrad(h, op, grads_scratch, 1.f, layer);
        }
    }
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
    Layout l = make_layout(h->plan, batch, training != 0);
    for (size_t i = 0; i < h->plan.tensors.size(); ++i)
        if (h->plan.tensors[i].name == name) {
            if (l.off[i] < 0) return set_err(WUN_E_INVALID, "tensor exists only in training workspaces");
            *offset_floats = l.off[i]; *rows = h->plan.tensors[i].rows; *channels = h->plan.tensors[i].C;
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
