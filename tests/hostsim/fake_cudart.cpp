// fake_cudart.cpp - a recording stand-in for the 19 CUDA runtime entry points libwun.so uses (TEST INFRASTRUCTURE, host only).
//
// tests/test_stream_schedule.py builds the engine a second time with `nvcc --cudart none` and links it against this library:
// the REAL non-dry host code of the engine (engine.cu: launch sequencing, the four internal streams, every event fork / join)
// then runs on a machine without a GPU.  Nothing executes on a device; every stream / event operation and every kernel launch is
// appended to a trace instead, and each launch is decoded - from the by-value parameter blocks of csrc/launch.h, kernels.h and
// kernels_umma.h - into the exact set of global-memory words it reads, writes or atomically accumulates into.  The Python side
// replays the trace through a vector-clock happens-before checker (a software racecheck of the step's launch DAG).
//
// Trace lines (text, one operation each):
//   C <stream>                                   stream created
//   N <event>                                    event created
//   E <event> <stream>                           cudaEventRecord
//   S <stream> <event>                           cudaStreamWaitEvent
//   L <stream> <kernel name> [G:gx:gy:gz:bx:by:bz:smem:opted_in_smem:cluster_x] <accesses...>   kernel launch / memset; accesses:
//        V:<R|W|A>:<byte address>:<batch>:<bstride>:<row lo>:<row hi>:<rstride>:<C>     fp32 view (strides in elements)
//        F:<R|W|A>:<byte address>:<bytes>                                                 flat range
#include <cuda_runtime.h>
#include <cxxabi.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "kernels.h"
#include "kernels_umma.h"
#include "launch.h"

using namespace wun;

namespace cpudev {                                   // cpu_kernels.cpp: reference execution of a launch on host memory
bool execute(const std::string& name, void** args);
void reset();
}

namespace {

int g_execute = 0;                                   // fakecuda_set_execute(1): carry every launch out on the caller's (host) buffers;
                                                     // (2): the same under the footprint poison test (registered buffers)

std::mutex g_mu;
std::vector<std::string> g_trace;
std::map<const void*, std::string> g_kernels;      // host stub address -> demangled kernel name
uintptr_t g_next_stream = 0x1000, g_next_event = 0x100000;
struct CallCfg { dim3 grid, block; size_t smem; void* stream; };
std::map<const void*, int> g_max_dyn_smem;          // cudaFuncSetAttribute(cudaFuncAttributeMaxDynamicSharedMemorySize)
std::vector<CallCfg> g_cfg_stack;

std::string demangle(const char* name) {
    int status = 0;
    char* d = abi::__cxa_demangle(name, nullptr, nullptr, &status);
    std::string s = (status == 0 && d) ? d : name;
    free(d);
    return s;
}

void emit(const std::string& line) {
    std::lock_guard<std::mutex> lk(g_mu);
    g_trace.push_back(line);
}

// ---- access formatting -------------------------------------------------------------------------------------------------
struct AccessRec { char mode; bool is_view; uintptr_t base; long long batch, bstride, rlo, rhi, rstride, C, bytes; };
struct Acc {
    std::string s;
    std::vector<AccessRec> recs;
    void view(char mode, const void* base, long long batch, long long bstride, long long rlo, long long rhi, long long rstride, long long C) {
        if (!base || rhi <= rlo || C <= 0 || batch <= 0) return;
        recs.push_back({mode, true, (uintptr_t)base, batch, bstride, rlo, rhi, rstride, C, 0});
        char b[200];
        snprintf(b, sizeof(b), " V:%c:%llu:%lld:%lld:%lld:%lld:%lld:%lld", mode, (unsigned long long)(uintptr_t)base, batch, bstride, rlo, rhi, rstride, C);
        s += b;
    }
    void flat(char mode, const void* p, long long bytes) {
        if (!p || bytes <= 0) return;
        recs.push_back({mode, false, (uintptr_t)p, 0, 0, 0, 0, 0, 0, bytes});
        char b[120];
        snprintf(b, sizeof(b), " F:%c:%llu:%lld", mode, (unsigned long long)(uintptr_t)p, bytes);
        s += b;
    }
    // plane rows [lo, hi) of V, clipped to its valid range; an interpolated (MID) row reads its successor too, and its blend vector
    void plane(const PlaneView& V, int batch, long long lo, long long hi) {
        lo = lo < V.r_lo ? V.r_lo : lo;
        hi = hi > V.r_hi ? V.r_hi : hi;
        if (hi <= lo) return;
        if (V.kind == PLANE_MID) {
            long long h2 = hi + 1;
            if (V.mid_mode != MID_VALID && h2 > V.xrows) h2 = V.xrows;
            if (h2 > hi) hi = h2;
            if (V.blend) flat('R', V.blend, 4LL * V.C);
        }
        view('R', V.base, batch, V.bstride, lo, hi, V.rstride, V.C);
    }
};

// what one output class of a plane convolution touches (kernels_simt.cu plane_conv_kernel = the reference semantics)
void out_half(Acc& a, int epilogue, int batch, float* base, long long bstride, int rstride, int lo, int hi, int ncol, const float* saved,
              int acc_lo, int acc_hi) {
    if (hi <= lo) return;
    a.view('W', base, batch, bstride, lo, hi, rstride, ncol);
    if (epilogue == EPI_SLOPE && saved) a.view('R', saved, batch, bstride, lo, hi, rstride, ncol);
    const int alo = acc_lo > lo ? acc_lo : lo, ahi = acc_hi < hi ? acc_hi : hi;
    if (ahi > alo) a.view('R', base, batch, bstride, alo, ahi, rstride, ncol);       // += : the destination is read first
}

void out_class(Acc& a, const OutView& O, int epilogue, int batch, int N, int pairC) {
    if (O.m_hi <= O.m_lo) return;
    if (pairC > 0) {
        out_half(a, epilogue, batch, O.base, O.bstride, O.rstride, O.lo_h[0], O.hi_h[0], pairC, O.saved, O.acc_lo, O.acc_hi);
        out_half(a, epilogue, batch, O.base2, O.bstride2, O.rstride2, O.lo_h[1], O.hi_h[1], pairC, O.saved2, O.acc_lo2, O.acc_hi2);
    } else {
        out_half(a, epilogue, batch, O.base, O.bstride, O.rstride, O.m_lo, O.m_hi, N, O.saved, O.acc_lo, O.acc_hi);
    }
}

void decode_umma_conv(Acc& a, const UmmaLaunch& L) {
    for (int q = 0; q < L.ncls; ++q) {
        const UmmaClass& c = L.cls[q];
        if (c.out.m_hi <= c.out.m_lo) continue;
        for (int g = 0; g < c.ngroups; ++g) {
            const UmmaGroup& G = c.groups[g];
            int dmin = L.d[G.term_begin], dmax = dmin;
            for (int t = G.term_begin; t < G.term_end; ++t) { dmin = L.d[t] < dmin ? L.d[t] : dmin; dmax = L.d[t] > dmax ? L.d[t] : dmax; }
            a.plane(L.planes[G.plane], L.batch, (long long)c.out.m_lo + dmin, (long long)c.out.m_hi + dmax);
        }
        for (int s = 0; s < L.nsplit && s < kUmmaMaxSplit; ++s) a.flat('R', c.wpack[s], 16);     // the packed weights of (class, split): first block
        out_class(a, c.out, L.epilogue, L.batch, L.N, L.pairC);
    }
    if (L.bias) a.flat('R', L.bias, 4LL * (L.pairC > 0 ? L.pairC : L.N));
}

// weight slice of one term: element (k, n) at W + woff + k * w_sk + n * w_sn, k < Ck, n < ncols (forward: w_sn = 1; dgrad: w_sk = 1)
void weight_slice(Acc& a, const float* W, long long woff, int Ck, int ncols, int w_sk, int w_sn) {
    if (w_sn == 1) a.view('R', W + woff, 1, 0, 0, Ck, w_sk, ncols);
    else if (w_sk == 1) a.view('R', W + woff, 1, 0, 0, ncols, w_sn, Ck);
    else
        for (int k = 0; k < Ck; ++k) a.view('R', W + woff + (long long)k * w_sk, 1, 0, 0, ncols, w_sn, 1);
}

void decode_conv(Acc& a, const ConvLaunch& L) {
    for (int q = 0; q < L.ncls; ++q) {
        const OutView& O = L.cls[q];
        if (O.m_hi <= O.m_lo) continue;
        for (int t = O.term_begin; t < O.term_end; ++t) {
            const Term& T = L.terms[t];
            a.plane(L.planes[T.plane], L.batch, (long long)O.m_lo + T.d, (long long)O.m_hi + T.d);
            const PlaneView& P = L.planes[T.plane];
            const int half = L.pairC > 0 ? L.pairC : L.N;
            if (T.woff >= 0 || L.pairC == 0) weight_slice(a, L.W, T.woff, P.C, half, L.w_sk, L.w_sn);
            if (L.pairC > 0 && T.woff2 >= 0) weight_slice(a, L.W, T.woff2, P.C, half, L.w_sk, L.w_sn);
        }
        out_class(a, O, L.epilogue, L.batch, L.N, L.pairC);
    }
    if (L.bias) a.flat('R', L.bias, 4LL * (L.pairC > 0 ? L.pairC : L.N));
}

// dW block of one tap: element (cp, cg) at dW + woff + cp * w_sp + cg * w_sg
void dw_block(Acc& a, float* dW, long long woff, int Cp, int Cg, int w_sp, int w_sg) {
    if (w_sg == 1) a.view('A', dW + woff, 1, 0, 0, Cp, w_sp, Cg);
    else if (w_sp == 1) a.view('A', dW + woff, 1, 0, 0, Cg, w_sg, Cp);
    else a.flat('A', dW + woff, 4LL * ((long long)(Cp - 1) * w_sp + (long long)(Cg - 1) * w_sg + 1));
}

// the partial tiles a bulk-fed wgrad launch stores (kernels_umma.cu: one 128 x 256-float slot per CTA of the launch)
long long wgrad_partial_bytes(const UmmaWgradLaunch& L) {
    long long slots = 0;
    for (int g = 0; g < L.ngroups; ++g) slots += (long long)L.grp[g].n_tapsets * L.grp[g].n_mtiles * L.grp[g].n_ntiles * L.grp[g].n_ctas_x;
    return slots * 128 * 256 * 4;
}
// the per-CTA column sums of split job j: [batch][chunk][2048-row block][16]
long long colsum_part_bytes(const SplitJobs& J, int j) {
    return 4LL * J.batch * J.job[j].nchunk * ((J.job[j].rows + 2047) / 2048) * 16;
}

void decode_wgrad_groups(Acc& a, const UmmaWgradLaunch& L, const WgSplit* S) {
    for (int g = 0; g < L.ngroups; ++g) {
        const WgGroup& G = L.grp[g];
        if (G.m_hi <= G.m_lo) continue;
        if (S) {            // bulk-fed: the operands are the split arrays [batch][chunk][4 sub-planes][rows][16 B]
            a.flat('R', S->P[g], (long long)L.batch * S->p_nchunk[g] * 4 * S->p_pstride[g]);
            a.flat('R', S->G[g], (long long)L.batch * S->g_nchunk[g] * 4 * S->g_pstride[g]);
        } else {
            int dmin = G.d[0], dmax = G.d[0];
            for (int t = 1; t < G.ntaps; ++t) { dmin = G.d[t] < dmin ? G.d[t] : dmin; dmax = G.d[t] > dmax ? G.d[t] : dmax; }
            a.plane(G.P, L.batch, (long long)G.m_lo + dmin, (long long)G.m_hi + dmax);
            a.plane(G.G, L.batch, G.m_lo, G.m_hi);
        }
        for (int t = 0; t < G.ntaps; ++t) dw_block(a, L.dW, G.woff[t], G.P.C, G.G.C, L.w_sp, L.w_sg);
    }
}

void decode_output(Acc& a, const OutputLaunch& O, bool reads_feat, bool writes_out) {
    const long long per_src = (long long)O.batch * O.T_out * O.C;
    a.flat('R', O.mix, 4LL * O.batch * O.T_in * O.C);
    if (reads_feat) a.flat('R', O.feat, 4LL * O.batch * O.Tf * O.F);
    const int Cin = O.C + O.F;
    for (int k = 0; k < O.nconv; ++k) {
        a.flat('R', O.params + O.w_off[k], 4LL * O.ofs * Cin * O.C);
        a.flat('R', O.params + O.b_off[k], 4LL * O.C);
    }
    if (writes_out) {
        if (O.outputs) a.flat('W', O.outputs, 4LL * O.K * per_src);
        if (O.targets) {
            a.flat('R', O.targets, 4LL * O.K * per_src);
            a.flat('W', O.dpre, 4LL * O.batch * O.T_out * O.nconv * O.C);
            if (O.loss) a.flat('A', O.loss, 4);
        }
    }
}

int template_int(const std::string& name, int index) {      // index-th integer template argument of "kernel<a, b>(...)"
    size_t p = name.find('<');
    if (p == std::string::npos) return -1;
    size_t e = name.find('>', p);
    std::string args = name.substr(p + 1, e - p - 1);
    size_t pos = 0;
    for (int i = 0; i < index; ++i) { pos = args.find(',', pos); if (pos == std::string::npos) return -1; ++pos; }
    return atoi(args.c_str() + pos);
}

bool has(const std::string& s, const char* sub) { return s.find(sub) != std::string::npos; }

// Decodes the global-memory footprint of one launch from its argument array.  Unknown kernels are reported as such: the
// checker fails on them, so a kernel added to the engine has to be described here before the schedule test passes again.
Acc decode(const std::string& name, void** args, bool* known) {
    Acc a;
    *known = true;
    if (has(name, "plane_conv_umma_persistent_out")) {
        const UmmaLaunch& L = *static_cast<const UmmaLaunch*>(args[0]);
        const OutputFuse& F = *static_cast<const OutputFuse*>(args[2]);
        decode_umma_conv(a, L);
        decode_output(a, F.O, false, true);                    // the features come from the accumulators, not from memory
        if (F.gfeat) a.flat('W', F.gfeat, 4LL * F.O.batch * F.O.Tf * F.O.F);
        if (F.grads)
            for (int k = 0; k < F.O.nconv; ++k) {
                a.flat('A', F.grads + F.O.w_off[k], 4LL * F.O.ofs * (F.O.C + F.O.F) * F.O.C);
                a.flat('A', F.grads + F.O.b_off[k], 4LL * F.O.C);
            }
    } else if (has(name, "plane_conv_umma_")) {                // plane_conv_umma_kernel<NPAD, DG>
        decode_umma_conv(a, *static_cast<const UmmaLaunch*>(args[0]));
    } else if (has(name, "wgrad_umma_bulk_kernel")) {
        const UmmaWgradLaunch& L = *static_cast<const UmmaWgradLaunch*>(args[0]);
        decode_wgrad_groups(a, L, static_cast<const WgSplit*>(args[1]));
        if (L.partial) a.flat('W', L.partial, wgrad_partial_bytes(L));
    } else if (has(name, "wgrad_reduce_kernel")) {
        const UmmaWgradLaunch& L = *static_cast<const UmmaWgradLaunch*>(args[0]);
        const SplitJobs& J = *static_cast<const SplitJobs*>(args[1]);
        if (L.partial) {
            a.flat('R', L.partial, wgrad_partial_bytes(L));
            for (int g = 0; g < L.ngroups; ++g)
                for (int t = 0; t < L.grp[g].ntaps; ++t) dw_block(a, L.dW, L.grp[g].woff[t], L.grp[g].P.C, L.grp[g].G.C, L.w_sp, L.w_sg);
        }
        for (int j = 0; j < J.njobs; ++j)
            if (J.job[j].colsum) {
                a.flat('R', J.job[j].colsum_part, colsum_part_bytes(J, j));
                a.flat('A', J.job[j].colsum, 4LL * J.job[j].V.C);
            }
    } else if (has(name, "wgrad_umma_kernel")) {
        decode_wgrad_groups(a, *static_cast<const UmmaWgradLaunch*>(args[0]), nullptr);
    } else if (has(name, "split_views_kernel")) {
        const SplitJobs& J = *static_cast<const SplitJobs*>(args[0]);
        for (int j = 0; j < J.njobs; ++j) {
            const SplitJob& S = J.job[j];
            a.plane(S.V, J.batch, S.row0, (long long)S.row0 + S.rows);
            a.flat('W', S.out, (long long)J.batch * S.nchunk * 4 * S.rows * 16);
            if (S.colsum) a.flat('A', S.colsum, 4LL * S.V.C);                  // (what the host reference of the launch adds)
            if (S.colsum && S.colsum_part) a.flat('W', S.colsum_part, colsum_part_bytes(J, j));
        }
    } else if (has(name, "umma_pack_kernel")) {
        const UmmaPackLaunch& P = *static_cast<const UmmaPackLaunch*>(args[0]);
        for (int j = 0; j < P.njobs; ++j) {
            const UmmaPackJob& J = P.jobs[j];
            a.flat('W', J.out, (long long)J.nblocks * 64 * P.NPAD);
            for (int g = 0; g < J.ngroups; ++g)
                for (int t = J.g_term_begin[g]; t < J.g_term_begin[g] + J.g_nterm[g]; ++t) {
                    const int half = P.pairC > 0 ? P.pairC : P.N;
                    if (P.woff[t] >= 0 || P.pairC == 0) weight_slice(a, P.W, P.woff[t], J.g_C[g], half, P.w_sk, P.w_sn);
                    if (P.pairC > 0 && P.woff2[t] >= 0) weight_slice(a, P.W, P.woff2[t], J.g_C[g], half, P.w_sk, P.w_sn);
                }
        }
    } else if (has(name, "first_wgrad_sum_kernel")) {
        const FirstWgrad& P = *static_cast<const FirstWgrad*>(args[0]);
        const int C = *static_cast<const int*>(args[1]), N = *static_cast<const int*>(args[2]);
        a.flat('R', P.part, 4LL * 2 * P.L.batch * P.grid_x * (P.L.k * C * N + N));
        a.flat('A', P.dW, 4LL * P.L.k * C * N);
        if (P.db) a.flat('A', P.db, 4LL * N);
    } else if (has(name, "first_fwd_kernel") || has(name, "first_wgrad_kernel")) {
        const bool wg = has(name, "first_wgrad_kernel");
        const FirstLayer& L = wg ? static_cast<const FirstWgrad*>(args[0])->L : *static_cast<const FirstLayer*>(args[0]);
        const int C = template_int(name, 0), N = template_int(name, 1);
        a.view('R', L.x, L.batch, L.x_bstride, 0, L.T, C, C);
        a.view(wg ? 'R' : 'W', L.dec, L.batch, L.dec_bstride, 0, L.Td, N, N);
        a.view(wg ? 'R' : 'W', L.odd, L.batch, L.odd_bstride, 0, L.mo_hi - L.mo_lo, N, N);
        if (wg) {
            const FirstWgrad& P = *static_cast<const FirstWgrad*>(args[0]);
            a.flat('A', P.dW, 4LL * L.k * C * N);                       // (what the host reference of the launch adds)
            if (P.db) a.flat('A', P.db, 4LL * N);
            a.flat('W', P.part, 4LL * 2 * L.batch * P.grid_x * (L.k * C * N + N));
        } else {
            a.flat('R', L.W, 4LL * L.k * C * N);
            a.flat('R', L.bias, 4LL * N);
        }
    } else if (has(name, "plane_conv_kernel")) {
        decode_conv(a, *static_cast<const ConvLaunch*>(args[0]));
    } else if (has(name, "plane_wgrad_kernel") || has(name, "plane_wgrad_smallc_kernel")) {
        const WgradLaunch& W = *static_cast<const WgradLaunch*>(args[0]);
        int dmin = W.d[0], dmax = W.d[0];
        for (int t = 1; t < W.nterms; ++t) { dmin = W.d[t] < dmin ? W.d[t] : dmin; dmax = W.d[t] > dmax ? W.d[t] : dmax; }
        a.plane(W.plane, W.batch, (long long)W.m_lo + dmin, (long long)W.m_hi + dmax);
        a.plane(W.dpre, W.batch, W.m_lo, W.m_hi);
        for (int t = 0; t < W.nterms; ++t) dw_block(a, W.dW, W.woff[t], W.plane.C, W.N, W.w_sk, W.w_sn);
    } else if (has(name, "colsum_kernel")) {
        const PlaneView& V = *static_cast<const PlaneView*>(args[0]);
        a.plane(V, *static_cast<const int*>(args[1]), V.r_lo, V.r_hi);
        a.flat('A', *static_cast<float* const*>(args[4]), 4LL * V.C);
    } else if (has(name, "output_fwd_kernel")) {
        const OutputLaunch& O = *static_cast<const OutputLaunch*>(args[0]);
        decode_output(a, O, true, true);
        if (O.targets && O.loss) {                                      // per-CTA loss sums + the CTA counter of their fixed-order total
            a.flat('W', O.loss_part, 4 * (((long long)O.batch * O.T_out + 127) / 128));
            a.flat('A', O.loss_count, 4);
        }
    } else if (has(name, "output_dgrad_kernel")) {
        const OutputLaunch& O = *static_cast<const OutputLaunch*>(args[0]);
        decode_output(a, O, true, false);
        a.flat('R', O.dpre, 4LL * O.batch * O.T_out * O.nconv * O.C);
        a.flat('W', *static_cast<float* const*>(args[1]), 4LL * O.batch * O.Tf * O.F);
    } else if (has(name, "output_wgrad_kernel")) {                  // per-CTA sums: [tap][row chunk][(C + F + 1) * nconv * C]
        const OutputLaunch& O = *static_cast<const OutputLaunch*>(args[0]);
        const float* part = *static_cast<float* const*>(args[1]);
        const long long per = *static_cast<const int*>(args[2]), nx = ((long long)O.batch * O.T_out + per - 1) / per;
        decode_output(a, O, true, false);
        a.flat('R', O.dpre, 4LL * O.batch * O.T_out * O.nconv * O.C);
        a.flat('W', part, 4LL * O.ofs * nx * (O.C + O.F + 1) * O.nconv * O.C);
    } else if (has(name, "output_wgrad_sum_kernel")) {
        const OutputLaunch& O = *static_cast<const OutputLaunch*>(args[0]);
        const float* part = *static_cast<float* const*>(args[1]);
        const long long nx = *static_cast<const int*>(args[2]);
        float* grads = *static_cast<float* const*>(args[3]);
        a.flat('R', part, 4LL * O.ofs * nx * (O.C + O.F + 1) * O.nconv * O.C);
        decode_output(a, O, true, false);                                  // (what the host reference of the launch reads)
        a.flat('R', O.dpre, 4LL * O.batch * O.T_out * O.nconv * O.C);
        for (int k = 0; k < O.nconv; ++k) {
            a.flat('A', grads + O.w_off[k], 4LL * O.ofs * (O.C + O.F) * O.C);
            a.flat('A', grads + O.b_off[k], 4LL * O.C);
        }
    } else if (has(name, "upsample_bwd_kernel")) {
        const UpsampleBwdLaunch& U = *static_cast<const UpsampleBwdLaunch*>(args[0]);
        a.flat('R', U.due, 4LL * U.batch * U.N * U.C);
        a.flat('R', U.dmid, 4LL * U.batch * U.nmid * U.C);
        a.flat('R', U.x, 4LL * U.batch * U.N * U.C);
        a.flat('W', U.gx, 4LL * U.batch * U.N * U.C);
        if (U.blend) a.flat('R', U.blend, 4LL * U.C);
        if (U.dvar) {
            a.flat('A', U.dvar, 4LL * U.C);
            // per-CTA sums [item * row chunks][C] + the CTA counter of their fixed-order total (rows_per_cta: set by the launcher)
            a.flat('W', U.part, 4LL * U.batch * ((U.N + U.rows_per_cta - 1) / U.rows_per_cta) * U.C);
            a.flat('A', U.count, 4);
        }
    } else if (has(name, "sigmoid_kernel")) {
        const int n = *static_cast<const int*>(args[2]);
        a.flat('R', *static_cast<const float* const*>(args[0]), 4LL * n);
        a.flat('W', *static_cast<float* const*>(args[1]), 4LL * n);
    } else if (has(name, "adam_advance_kernel")) {
        a.flat('R', *static_cast<float* const*>(args[0]), 12);
        a.flat('W', *static_cast<float* const*>(args[0]), 12);
    } else if (has(name, "adam_kernel")) {
        const long long n = *static_cast<const long long*>(args[4]);
        for (int i = 0; i < 4; ++i) a.flat('R', *static_cast<float* const*>(args[i]), 4 * n);
        a.flat('W', *static_cast<float* const*>(args[0]), 4 * n);
        a.flat('W', *static_cast<float* const*>(args[2]), 4 * n);
        a.flat('W', *static_cast<float* const*>(args[3]), 4 * n);
        if (*static_cast<const float* const*>(args[9])) a.flat('R', *static_cast<const float* const*>(args[9]), 12);
    } else if (has(name, "gather_windows_kernel")) {
        const long long n_padded = *static_cast<const long long*>(args[1]);
        const int nw = *static_cast<const int*>(args[3]), T_in = *static_cast<const int*>(args[4]), C = *static_cast<const int*>(args[5]);
        a.flat('R', *static_cast<const float* const*>(args[0]), 4 * n_padded * C);
        a.flat('R', *static_cast<const long long* const*>(args[2]), 8LL * nw);
        a.flat('W', *static_cast<float* const*>(args[6]), 4LL * nw * T_in * C);
    } else if (has(name, "scatter_windows_kernel")) {
        const int nw = *static_cast<const int*>(args[2]), K = *static_cast<const int*>(args[3]), T_out = *static_cast<const int*>(args[4]),
                  C = *static_cast<const int*>(args[5]);
        const long long n_frames = *static_cast<const long long*>(args[7]);
        a.flat('R', *static_cast<const float* const*>(args[0]), 4LL * K * nw * T_out * C);
        a.flat('R', *static_cast<const long long* const*>(args[1]), 8LL * nw);
        a.flat('W', *static_cast<float* const*>(args[6]), 4LL * K * n_frames * C);
    } else {
        *known = false;
    }
    return a;
}

// ---- footprint verification (fakecuda_set_execute(2)): "poison test" ----------------------------------------------------------
// Before a launch is carried out on the registered host buffers, every word OUTSIDE its decoded footprint is overwritten with a
// marked NaN; afterwards (a) a word outside the decoded WRITE footprint that no longer holds what it held = a write the decoder
// does not know about, (b) a NaN in a written word that was not NaN before = the routine read a word outside the decoded READ
// footprint (NaN propagates through every product, also with zero).  Then the untouched words are restored.  The reference
// routines reproduce the oracle, so their accesses are the ones the computation needs: the decoded footprints the racecheck
// relies on are checked to CONTAIN them.
struct HostBuf { uint8_t* p; size_t bytes; };
std::vector<HostBuf> g_bufs;
const uint32_t kPoison = 0x7fc0dead;

void mark_range(std::vector<std::vector<uint8_t>>& mask, uintptr_t a0, long long nbytes, uint8_t bit) {
    for (size_t i = 0; i < g_bufs.size(); ++i) {
        const uintptr_t b0 = (uintptr_t)g_bufs[i].p, b1 = b0 + g_bufs[i].bytes;
        uintptr_t lo = a0 < b0 ? b0 : a0, hi = (a0 + (uintptr_t)nbytes) > b1 ? b1 : (a0 + (uintptr_t)nbytes);
        if (a0 + (uintptr_t)nbytes <= b0 || a0 >= b1 || hi <= lo) continue;
        for (size_t w = (lo - b0) / 4; w < (hi - b0 + 3) / 4 && w < mask[i].size(); ++w) mask[i][w] |= bit;
    }
}

void mark(std::vector<std::vector<uint8_t>>& mask, const std::vector<AccessRec>& recs) {
    for (const AccessRec& r : recs) {
        const uint8_t bit = r.mode == 'R' ? 1 : 2;                  // W and A both write
        if (!r.is_view) { mark_range(mask, r.base, r.bytes, bit); continue; }
        for (long long b = 0; b < r.batch; ++b)
            for (long long row = r.rlo; row < r.rhi; ++row)
                mark_range(mask, r.base + 4 * (uintptr_t)(b * r.bstride + row * r.rstride), 4 * r.C, bit);
    }
}

std::string poison_checked_execute(const std::string& name, void** args, const Acc& acc) {
    std::vector<std::vector<uint8_t>> mask(g_bufs.size());
    std::vector<std::vector<uint32_t>> saved(g_bufs.size());
    for (size_t i = 0; i < g_bufs.size(); ++i) {
        mask[i].assign(g_bufs[i].bytes / 4, 0);
        saved[i].assign((uint32_t*)g_bufs[i].p, (uint32_t*)g_bufs[i].p + g_bufs[i].bytes / 4);
    }
    mark(mask, acc.recs);
    if (name.find("wgrad_umma_bulk_kernel") != std::string::npos) {      // the reference routine reads the groups' own views, not the
        Acc views;                                                           // split arrays the device kernel is fed from
        decode_wgrad_groups(views, *static_cast<const UmmaWgradLaunch*>(args[0]), nullptr);
        mark(mask, views.recs);
    }
    for (size_t i = 0; i < g_bufs.size(); ++i) {
        uint32_t* w = (uint32_t*)g_bufs[i].p;
        for (size_t k = 0; k < mask[i].size(); ++k) if (!mask[i][k]) w[k] = kPoison;
    }
    const bool ok = cpudev::execute(name, args);
    long long stray_writes = 0, stray_reads = 0;
    for (size_t i = 0; i < g_bufs.size(); ++i) {
        uint32_t* w = (uint32_t*)g_bufs[i].p;
        for (size_t k = 0; k < mask[i].size(); ++k) {
            if (!(mask[i][k] & 2)) {                                   // not in the decoded write footprint
                const uint32_t expect = mask[i][k] ? saved[i][k] : kPoison;
                if (w[k] != expect) ++stray_writes;
                w[k] = saved[i][k];
            } else {
                float now, before;
                memcpy(&now, &w[k], 4); memcpy(&before, &saved[i][k], 4);
                if (now != now && before == before) {                  // a NaN appeared
                    if (stray_reads < 3 && getenv("FAKECUDA_POISON_DEBUG"))
                        fprintf(stderr, "poison: %s: NaN at buffer %zu word %zu (address %llu)\n", name.c_str(), i, k,
                                (unsigned long long)((uintptr_t)g_bufs[i].p + 4 * k));
                    ++stray_reads;
                }
            }
        }
    }
    if (!ok) return "UNKNOWN:";
    if (stray_writes || stray_reads) {
        char b[160];
        snprintf(b, sizeof(b), "FOOTPRINT-MISS(%lld_words_written_outside,%lld_NaNs_from_reads_outside):", stray_writes, stray_reads);
        return b;
    }
    return "";
}

cudaError_t record_launch(const void* func, void** args, void* stream, dim3 grid, dim3 block, size_t smem, unsigned cluster_x) {
    std::string name;
    int attr = -1;
    {
        std::lock_guard<std::mutex> lk(g_mu);
        auto it = g_kernels.find(func);
        name = it == g_kernels.end() ? "?unregistered" : it->second;
        auto at = g_max_dyn_smem.find(func);
        if (at != g_max_dyn_smem.end()) attr = at->second;
    }
    bool known = false;
    Acc decoded = decode(name, args, &known);
    const std::string& acc = decoded.s;
    std::string flag;
    if (g_execute == 2 && known) flag = poison_checked_execute(name, args, decoded);
    else if (g_execute && known && !cpudev::execute(name, args)) known = false;
    for (char& c : name) if (c == ' ') c = '_';                // one token per field in the trace line
    char head[64], geo[160];
    snprintf(head, sizeof(head), "L %llu ", (unsigned long long)(uintptr_t)stream);
    // launch geometry: grid, block, dynamic shared memory asked for, the kernel's opted-in maximum (-1 = never set), cluster width
    snprintf(geo, sizeof(geo), " G:%u:%u:%u:%u:%u:%u:%zu:%d:%u", grid.x, grid.y, grid.z, block.x, block.y, block.z, smem, attr, cluster_x);
    emit(std::string(head) + (known ? "" : "UNKNOWN:") + flag + name + geo + acc);
    return cudaSuccess;
}

}  // namespace

// ---- the trace, for the Python side -----------------------------------------------------------------------------------------
extern "C" {

void fakecuda_reset() { std::lock_guard<std::mutex> lk(g_mu); g_trace.clear(); }
void fakecuda_set_execute(int on) { g_execute = on; cpudev::reset(); g_bufs.clear(); }
void fakecuda_register_buffer(void* p, long long bytes) { g_bufs.push_back({static_cast<uint8_t*>(p), (size_t)bytes}); }

long long fakecuda_trace(char* buf, long long capacity) {
    std::lock_guard<std::mutex> lk(g_mu);
    std::string s;
    for (const auto& l : g_trace) { s += l; s += "\n"; }
    if (buf && capacity > 0) {
        long long n = (long long)s.size() < capacity - 1 ? (long long)s.size() : capacity - 1;
        memcpy(buf, s.data(), n);
        buf[n] = 0;
    }
    return (long long)s.size() + 1;
}

// operations the caller of the library performs itself (the facade's own streams, events and the NCCL all-reduce)
void fakecuda_user_line(const char* line) { emit(line); }

// ---- registration (nvcc-generated module constructors) ---------------------------------------------------------------------
void** __cudaRegisterFatBinary(void* fatCubin) { static void* handle[1]; (void)fatCubin; return handle; }
void __cudaRegisterFatBinaryEnd(void** h) { (void)h; }
void __cudaUnregisterFatBinary(void** h) { (void)h; }
void __cudaRegisterFunction(void** h, const char* hostFun, char* deviceFun, const char* deviceName, int thread_limit, uint3* tid,
                            uint3* bid, dim3* bDim, dim3* gDim, int* wSize) {
    (void)h; (void)deviceFun; (void)thread_limit; (void)tid; (void)bid; (void)bDim; (void)gDim; (void)wSize;
    std::lock_guard<std::mutex> lk(g_mu);
    g_kernels[hostFun] = demangle(deviceName);
}
unsigned __cudaPushCallConfiguration(dim3 gridDim, dim3 blockDim, size_t sharedMem, struct CUstream_st* stream) {
    std::lock_guard<std::mutex> lk(g_mu);
    g_cfg_stack.push_back({gridDim, blockDim, sharedMem, stream});
    return 0;
}
cudaError_t __cudaPopCallConfiguration(dim3* gridDim, dim3* blockDim, size_t* sharedMem, void* stream) {
    std::lock_guard<std::mutex> lk(g_mu);
    if (g_cfg_stack.empty()) return cudaErrorInvalidConfiguration;
    CallCfg c = g_cfg_stack.back();
    g_cfg_stack.pop_back();
    *gridDim = c.grid; *blockDim = c.block; *sharedMem = c.smem; *static_cast<void**>(stream) = c.stream;
    return cudaSuccess;
}

// ---- runtime API -----------------------------------------------------------------------------------------------------------
cudaError_t cudaLaunchKernel(const void* func, dim3 gridDim, dim3 blockDim, void** args, size_t sharedMem, cudaStream_t stream) {
    return record_launch(func, args, stream, gridDim, blockDim, sharedMem, 1);
}
cudaError_t cudaLaunchKernelExC(const cudaLaunchConfig_t* config, const void* func, void** args) {
    unsigned cx = 1;
    for (unsigned i = 0; i < config->numAttrs; ++i)
        if (config->attrs[i].id == cudaLaunchAttributeClusterDimension) cx = config->attrs[i].val.clusterDim.x;
    return record_launch(func, args, config->stream, config->gridDim, config->blockDim, config->dynamicSmemBytes, cx);
}
cudaError_t cudaMemsetAsync(void* devPtr, int value, size_t count, cudaStream_t stream) {
    if (g_execute) memset(devPtr, value, count);
    char b[160];
    snprintf(b, sizeof(b), "L %llu memset F:W:%llu:%lld", (unsigned long long)(uintptr_t)stream, (unsigned long long)(uintptr_t)devPtr, (long long)count);
    emit(b);
    return cudaSuccess;
}
cudaError_t cudaStreamCreateWithFlags(cudaStream_t* s, unsigned flags) {
    (void)flags;
    uintptr_t id;
    { std::lock_guard<std::mutex> lk(g_mu); id = g_next_stream; g_next_stream += 0x10; }
    *s = reinterpret_cast<cudaStream_t>(id);
    char b[64];
    snprintf(b, sizeof(b), "C %llu", (unsigned long long)id);
    emit(b);
    return cudaSuccess;
}
cudaError_t cudaStreamDestroy(cudaStream_t s) { (void)s; return cudaSuccess; }
cudaError_t cudaEventCreateWithFlags(cudaEvent_t* e, unsigned flags) {
    (void)flags;
    uintptr_t id;
    { std::lock_guard<std::mutex> lk(g_mu); id = g_next_event; g_next_event += 0x10; }
    *e = reinterpret_cast<cudaEvent_t>(id);
    char b[64];
    snprintf(b, sizeof(b), "N %llu", (unsigned long long)id);
    emit(b);
    return cudaSuccess;
}
cudaError_t cudaEventDestroy(cudaEvent_t e) { (void)e; return cudaSuccess; }
cudaError_t cudaEventRecord(cudaEvent_t e, cudaStream_t s) {
    char b[96];
    snprintf(b, sizeof(b), "E %llu %llu", (unsigned long long)(uintptr_t)e, (unsigned long long)(uintptr_t)s);
    emit(b);
    return cudaSuccess;
}
cudaError_t cudaStreamWaitEvent(cudaStream_t s, cudaEvent_t e, unsigned flags) {
    (void)flags;
    char b[96];
    snprintf(b, sizeof(b), "S %llu %llu", (unsigned long long)(uintptr_t)s, (unsigned long long)(uintptr_t)e);
    emit(b);
    return cudaSuccess;
}
cudaError_t cudaFuncSetAttribute(const void* func, cudaFuncAttribute attr, int value) {
    if (attr == cudaFuncAttributeMaxDynamicSharedMemorySize) {
        if (value > 232448) return cudaErrorInvalidValue;          // 227 KB: the opt-in limit per CTA on sm_90
        std::lock_guard<std::mutex> lk(g_mu);
        g_max_dyn_smem[func] = value;
    }
    return cudaSuccess;
}
cudaError_t cudaGetDeviceCount(int* count) { *count = 1; return cudaSuccess; }
cudaError_t cudaGetLastError(void) { return cudaSuccess; }
const char* cudaGetErrorString(cudaError_t e) { (void)e; return "fake cudart: no error"; }

}  // extern "C"
