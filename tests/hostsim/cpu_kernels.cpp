// cpu_kernels.cpp - reference execution of the engine's launches on HOST memory (TEST INFRASTRUCTURE; never part of libwun.so).
//
// With fakecuda_set_execute(1) the recording runtime of fake_cudart.cpp does more than record: every launch is carried out
// immediately, in issue order (a valid execution order: tests/test_stream_schedule.py proves the schedule race-free), by the
// plain loops below on the buffers the caller passed - ordinary host arrays.  Each routine is a second, independent statement
// of what the corresponding CUDA kernel is specified to compute from its by-value parameter block (csrc/launch.h, kernels.h,
// kernels_umma.h), written from those contracts in double-precision accumulation: the tensor-core kernels' tiling, pipelines
// and bf16 hi/lo arithmetic do not appear - only WHAT they must produce.  tests/test_cpu_device.py runs whole training steps of
// the engine's real host code this way and compares loss, every gradient and the Adam update with the oracle: that checks the
// parameter blocks the host builds for the tensor-core kernels (plane / class / group / term tables, packed-weight jobs, pair-merged
// halves, split-pass jobs, fused output epilogue, scales, accumulate ranges) for configurations no GPU test has run.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <map>
#include <string>
#include <vector>

#include "kernels.h"
#include "kernels_umma.h"
#include "launch.h"

using namespace wun;

namespace cpudev {

static inline bool has(const std::string& s, const char* sub) { return s.find(sub) != std::string::npos; }

static double plane_at(const PlaneView& P, int b, long long r, int c) {      // kernels_simt.cu plane_load
    if (r < P.r_lo || r >= P.r_hi || c >= P.C) return 0.0;
    const float* p = P.base + (long long)b * P.bstride + r * P.rstride + c;
    double x = *p;
    if (P.kind == PLANE_MID) {
        double nx;
        if (P.mid_mode == MID_VALID || r + 1 < P.xrows) nx = p[P.rstride];
        else nx = (P.mid_mode == MID_CLAMP) ? x : 0.0;
        if (P.blend) { const double w = P.blend[c]; x = w * x + (1.0 - w) * nx; }
        else x = x + (nx - x) * 0.5;
    }
    return x;
}

static inline double lrelu(double v) { return v > 0.2 * v ? v : 0.2 * v; }

// ---- optional arithmetic model of the tensor-core kernels (FAKECUDA_MMA_MODEL) ----------------------------------------------------
//   0 (default): exact products, double accumulation - the contract.
//   3: every fp32 operand split into two bf16 (hi = rn(x), lo = rn(x - hi)), hi*hi + hi*lo + lo*hi accumulated in fp32 - the
//      scheme of kernels_umma.cu (DESIGN.md 4.1); 1: hi*hi only (a single bf16 pass), for comparison.
static int g_mma_model = 0;
static inline float bf16_rn(float x) {
    uint32_t u;
    memcpy(&u, &x, 4);
    if ((u & 0x7f800000u) == 0x7f800000u) return x;                  // inf / nan
    u += 0x7fffu + ((u >> 16) & 1u);                                 // round to nearest even
    u &= 0xffff0000u;
    float r;
    memcpy(&r, &u, 4);
    return r;
}
struct Acc {                       // one accumulator in the active arithmetic model
    double d = 0.0;
    float f = 0.f;
    inline void mac(double x, double w) {
        if (g_mma_model == 0) { d += x * w; return; }
        const float xf = (float)x, wf = (float)w;
        const float xh = bf16_rn(xf), wh = bf16_rn(wf);
        f += xh * wh;                                                // (bf16 x bf16 products are exact in fp32)
        if (g_mma_model == 3) {
            const float xl = bf16_rn(xf - xh), wl = bf16_rn(wf - wh);
            f += xh * wl;
            f += xl * wh;
        }
    }
    inline double value() const { return g_mma_model == 0 ? d : (double)f; }
};

// one finished accumulator value -> its place, through the epilogue of launch.h (bias + LeakyReLU | slope | plain; accumulate rows)
static void store_out(float* base, long long bstride, int rstride, const float* saved, int acc_lo, int acc_hi, int epilogue, const float* bias,
                      int b, int m, int col, int bias_col, double v) {
    const long long off = (long long)b * bstride + (long long)m * rstride + col;
    if (epilogue == EPI_BIAS_LRELU) { if (bias) v += bias[bias_col]; v = lrelu(v); }
    else if (epilogue == EPI_SLOPE && saved) v *= (saved[off] > 0.f) ? 1.0 : 0.2;
    if (m >= acc_lo && m < acc_hi) v += base[off];
    base[off] = (float)v;
}

// ---- packed weights: what umma_pack_kernel is specified to put into a (class, split) job ------------------------------------
struct PackedJob {
    int n0 = 0, NPAD = 0, N = 0, pairC = 0;
    std::map<int, std::vector<double>> W;      // term -> [C][NPAD]
    std::map<int, int> C;
};
static std::map<const uint8_t*, PackedJob> g_packs;

static void run_pack(const UmmaPackLaunch& P) {
    for (int j = 0; j < P.njobs; ++j) {
        const UmmaPackJob& J = P.jobs[j];
        PackedJob pj;
        pj.n0 = J.n0; pj.NPAD = P.NPAD; pj.N = P.N; pj.pairC = P.pairC;
        for (int g = 0; g < J.ngroups; ++g)
            for (int t = J.g_term_begin[g]; t < J.g_term_begin[g] + J.g_nterm[g]; ++t) {
                std::vector<double> w((size_t)J.g_C[g] * P.NPAD, 0.0);
                for (int k = 0; k < J.g_C[g]; ++k)
                    for (int n = 0; n < P.NPAD; ++n) {
                        const int nn = J.n0 + n;
                        if (nn >= P.N) continue;
                        const bool h2 = P.pairC > 0 && nn >= P.pairC;
                        const int wo = h2 ? P.woff2[t] : P.woff[t];
                        if (wo >= 0 || P.pairC == 0)
                            w[(size_t)k * P.NPAD + n] = P.W[(long long)wo + (long long)k * P.w_sk + (long long)(h2 ? nn - P.pairC : nn) * P.w_sn];
                    }
                pj.W[t] = std::move(w);
                pj.C[t] = J.g_C[g];
            }
        g_packs[J.out] = std::move(pj);
    }
}

// ---- tensor-core plane convolution + the fused output epilogue -------------------------------------------------------
static bool run_umma_conv(const UmmaLaunch& L, const OutputFuse* F) {
    const int ncol_out = F ? F->O.nconv * F->O.C : 0;
    double lsum = 0.0;
    for (int q = 0; q < L.ncls; ++q) {
        const UmmaClass& K = L.cls[q];
        const OutView& O = K.out;
        if (O.m_hi <= O.m_lo) continue;
        std::vector<const PackedJob*> jobs;
        for (int s = 0; s < L.nsplit; ++s) {
            auto it = g_packs.find(K.wpack[s]);
            if (it == g_packs.end()) return false;                    // a conv whose weights were never packed
            jobs.push_back(&it->second);
        }
        std::vector<Acc> acc(L.N);
        std::vector<double> act(L.N);
        for (int b = 0; b < L.batch; ++b)
            for (int m = O.m_lo; m < O.m_hi; ++m) {
                std::fill(acc.begin(), acc.end(), Acc());
                for (int g = 0; g < K.ngroups; ++g) {
                    const UmmaGroup& G = K.groups[g];
                    const PlaneView& P = L.planes[G.plane];
                    for (int t = G.term_begin; t < G.term_end; ++t)
                        for (int k = 0; k < P.C; ++k) {
                            const double x = plane_at(P, b, (long long)m + L.d[t], k);
                            if (x == 0.0) continue;
                            for (const PackedJob* pj : jobs) {
                                auto wt = pj->W.find(t);
                                if (wt == pj->W.end()) return false;
                                const double* w = wt->second.data() + (size_t)k * pj->NPAD;
                                const int nmax = (L.N - pj->n0) < pj->NPAD ? (L.N - pj->n0) : pj->NPAD;
                                for (int n = 0; n < nmax; ++n) acc[pj->n0 + n].mac(x, w[n]);
                            }
                        }
                }
                for (int nn = 0; nn < L.N; ++nn) {
                    const int h = (L.pairC > 0 && nn >= L.pairC) ? 1 : 0;
                    const int col = nn - h * L.pairC;
                    double v = acc[nn].value();
                    if (L.epilogue == EPI_BIAS_LRELU) act[nn] = lrelu(v + (L.bias ? L.bias[L.pairC > 0 ? col : nn] : 0.0));
                    if (L.pairC > 0) {
                        if (m < O.lo_h[h] || m >= O.hi_h[h]) continue;
                        if (h == 0) store_out(O.base, O.bstride, O.rstride, O.saved, O.acc_lo, O.acc_hi, L.epilogue, L.bias, b, m, col, col, v);
                        else store_out(O.base2, O.bstride2, O.rstride2, O.saved2, O.acc_lo2, O.acc_hi2, L.epilogue, L.bias, b, m, col, col, v);
                    } else {
                        store_out(O.base, O.bstride, O.rstride, O.saved, O.acc_lo, O.acc_hi, L.epilogue, L.bias, b, m, nn, nn, v);
                    }
                }
                if (!F) continue;
                // fused output layer (kernels_umma.h OutputFuse): one or (pair-merged) two output frames per feature row
                const OutputLaunch& U = F->O;
                const int Cin = U.C + U.F;
                const long long src_stride = (long long)U.batch * U.T_out * U.C;
                for (int hh = 0; hh < 2; ++hh) {
                    const bool ok_row = (L.pairC > 0) ? (m >= O.lo_h[hh] && m < O.hi_h[hh]) : (hh == 0);
                    const int tt = F->t0[q] + F->t_step * m + hh;
                    if (!ok_row || tt >= U.T_out) continue;
                    const int width = L.pairC > 0 ? L.pairC : L.N;                 // = U.F
                    const double* feat = act.data() + (hh ? L.pairC : 0);
                    std::vector<double> pre(ncol_out), est(ncol_out), g(ncol_out, 0.0);
                    for (int conv = 0; conv < U.nconv; ++conv)
                        for (int oc = 0; oc < U.C; ++oc) {
                            double s = U.params[U.b_off[conv] + oc];
                            for (int c = 0; c < Cin; ++c) {
                                const double x = c < U.C ? U.mix[((long long)b * U.T_in + U.crop_feat + tt) * U.C + c] : feat[c - U.C];
                                s += x * U.params[U.w_off[conv] + (long long)c * U.C + oc];
                            }
                            pre[conv * U.C + oc] = s;
                        }
                    (void)width;
                    for (int k = 0; k < ncol_out; ++k) {
                        double e = pre[k];
                        if (U.activation == 0) e = tanh(e);
                        else if (!U.training) e = e < -1.0 ? -1.0 : (e > 1.0 ? 1.0 : e);
                        est[k] = e;
                    }
                    const long long frame = ((long long)b * U.T_out + tt) * U.C;
                    double g_last[2] = {0.0, 0.0};
                    if (U.output_type == 1)
                        for (int oc = 0; oc < U.C; ++oc) {
                            double s = 0.0;
                            for (int conv = 0; conv < U.nconv; ++conv) s += est[conv * U.C + oc];
                            double last = U.mix[((long long)b * U.T_in + U.crop_out + tt) * U.C + oc] - s;
                            if (!U.training) last = last < -1.0 ? -1.0 : (last > 1.0 ? 1.0 : last);
                            if (U.outputs) U.outputs[(long long)U.nconv * src_stride + frame + oc] = (float)last;
                            if (U.targets) {
                                const double e = last - U.targets[(long long)U.nconv * src_stride + frame + oc];
                                lsum += e * e;
                                g_last[oc] = 2.0 * e * U.inv_count;
                            }
                        }
                    for (int conv = 0; conv < U.nconv; ++conv)
                        for (int oc = 0; oc < U.C; ++oc) {
                            const int k = conv * U.C + oc;
                            if (U.outputs) U.outputs[(long long)conv * src_stride + frame + oc] = (float)est[k];
                            if (U.targets) {
                                const double e = est[k] - U.targets[(long long)conv * src_stride + frame + oc];
                                lsum += e * e;
                                double gg = 2.0 * e * U.inv_count - g_last[oc];
                                if (U.activation == 0) gg *= (1.0 - est[k] * est[k]);
                                if (U.dpre) U.dpre[((long long)b * U.T_out + tt) * ncol_out + k] = (float)gg;
                                g[k] = gg;
                            }
                        }
                    if (F->gfeat) {          // gradient w.r.t. the features' pre-activation, stored with the feature view's geometry
                        float* fbase = hh ? O.base2 : O.base;
                        const long long bs = hh ? O.bstride2 : O.bstride;
                        const int rs = hh ? O.rstride2 : O.rstride;
                        float* gdst = F->gfeat + (fbase - U.feat);
                        for (int c = 0; c < U.F; ++c) {
                            double s = 0.0;
                            for (int conv = 0; conv < U.nconv; ++conv)
                                for (int oc = 0; oc < U.C; ++oc) s += g[conv * U.C + oc] * U.params[U.w_off[conv] + (long long)(U.C + c) * U.C + oc];
                            gdst[(long long)b * bs + (long long)m * rs + c] = (float)(s * (feat[c] > 0.0 ? 1.0 : 0.2));
                        }
                    }
                    if (F->grads)            // WUN_OUT_FUSE=2: the output convs' own weight / bias gradients in the epilogue as well
                        for (int conv = 0; conv < U.nconv; ++conv)
                            for (int oc = 0; oc < U.C; ++oc) {
                                const double gq = g[conv * U.C + oc] * F->grad_scale;
                                for (int c = 0; c < Cin; ++c) {
                                    const double x = c < U.C ? U.mix[((long long)b * U.T_in + U.crop_feat + tt) * U.C + c] : feat[c - U.C];
                                    F->grads[U.w_off[conv] + (long long)c * U.C + oc] += (float)(x * gq);
                                }
                                F->grads[U.b_off[conv] + oc] += (float)gq;
                            }
                }
            }
    }
    if (F && F->O.targets && F->O.loss) *F->O.loss += (float)(lsum * F->O.inv_count);
    return true;
}

// ---- generic plane convolution / weight gradient (kernels_simt.cu) -----------------------------------------------------------
static void run_conv(const ConvLaunch& L) {
    std::vector<double> acc(L.N);
    for (int q = 0; q < L.ncls; ++q) {
        const OutView& O = L.cls[q];
        for (int b = 0; b < L.batch; ++b)
            for (int m = O.m_lo; m < O.m_hi; ++m) {
                std::fill(acc.begin(), acc.end(), 0.0);
                for (int t = O.term_begin; t < O.term_end; ++t) {
                    const Term& T = L.terms[t];
                    const PlaneView& P = L.planes[T.plane];
                    for (int k = 0; k < P.C; ++k) {
                        const double x = plane_at(P, b, (long long)m + T.d, k);
                        if (x == 0.0) continue;
                        const float* w = L.W + (long long)T.woff + (long long)k * L.w_sk;
                        for (int n = 0; n < L.N; ++n) acc[n] += x * w[(long long)n * L.w_sn];
                    }
                }
                for (int n = 0; n < L.N; ++n)
                    store_out(O.base, O.bstride, O.rstride, O.saved, O.acc_lo, O.acc_hi, L.epilogue, L.bias, b, m, n, n, acc[n]);
            }
    }
}

static void wgrad_group(const PlaneView& P, const PlaneView& G, int m_lo, int m_hi, int nt, const int* d, const int* woff, float* dW,
                        int w_sp, int w_sg, double scale, int batch, bool tensor_core = false) {
    const int keep = g_mma_model;
    if (!tensor_core) g_mma_model = 0;                 // the CUDA-core kernels are exact fp32
    for (int t = 0; t < nt; ++t)
        for (int cp = 0; cp < P.C; ++cp)
            for (int cg = 0; cg < G.C; ++cg) {
                Acc s;
                for (int b = 0; b < batch; ++b)
                    for (int m = m_lo; m < m_hi; ++m) s.mac(plane_at(P, b, (long long)m + d[t], cp), plane_at(G, b, m, cg));
                dW[(long long)woff[t] + (long long)cp * w_sp + (long long)cg * w_sg] += (float)(s.value() * scale);
            }
    g_mma_model = keep;
}

static void run_output_fwd(const OutputLaunch& L) {
    const int Cin = L.C + L.F, ncol = L.nconv * L.C;
    const long long src_stride = (long long)L.batch * L.T_out * L.C;
    double lsum = 0.0;
    auto in = [&](int b, int row, int c) -> double {
        if (row < 0 || row >= L.Tf) return 0.0;
        if (c < L.C) return L.mix[((long long)b * L.T_in + L.crop_feat + row) * L.C + c];
        return L.feat[((long long)b * L.Tf + row) * L.F + (c - L.C)];
    };
    std::vector<double> pre(ncol), est(ncol);
    for (int b = 0; b < L.batch; ++b)
        for (int t = 0; t < L.T_out; ++t) {
            for (int conv = 0; conv < L.nconv; ++conv)
                for (int oc = 0; oc < L.C; ++oc) {
                    double s = L.params[L.b_off[conv] + oc];
                    for (int j = 0; j < L.ofs; ++j)
                        for (int c = 0; c < Cin; ++c) s += in(b, t + j - L.pad_left, c) * L.params[L.w_off[conv] + ((long long)j * Cin + c) * L.C + oc];
                    pre[conv * L.C + oc] = s;
                }
            for (int k = 0; k < ncol; ++k) {
                double e = pre[k];
                if (L.activation == 0) e = tanh(e);
                else if (!L.training) e = e < -1.0 ? -1.0 : (e > 1.0 ? 1.0 : e);
                est[k] = e;
            }
            const long long frame = ((long long)b * L.T_out + t) * L.C;
            double g_last[4] = {0, 0, 0, 0};
            if (L.output_type == 1)
                for (int oc = 0; oc < L.C; ++oc) {
                    double s = 0.0;
                    for (int conv = 0; conv < L.nconv; ++conv) s += est[conv * L.C + oc];
                    double last = L.mix[((long long)b * L.T_in + L.crop_out + t) * L.C + oc] - s;
                    if (!L.training) last = last < -1.0 ? -1.0 : (last > 1.0 ? 1.0 : last);
                    if (L.outputs) L.outputs[(long long)L.nconv * src_stride + frame + oc] = (float)last;
                    if (L.targets) {
                        const double e = last - L.targets[(long long)L.nconv * src_stride + frame + oc];
                        lsum += e * e;
                        g_last[oc] = 2.0 * e * L.inv_count;
                    }
                }
            for (int conv = 0; conv < L.nconv; ++conv)
                for (int oc = 0; oc < L.C; ++oc) {
                    const int k = conv * L.C + oc;
                    if (L.outputs) L.outputs[(long long)conv * src_stride + frame + oc] = (float)est[k];
                    if (L.targets) {
                        const double e = est[k] - L.targets[(long long)conv * src_stride + frame + oc];
                        lsum += e * e;
                        double g = 2.0 * e * L.inv_count - g_last[oc];
                        if (L.activation == 0) g *= (1.0 - est[k] * est[k]);
                        L.dpre[((long long)b * L.T_out + t) * ncol + k] = (float)g;
                    }
                }
        }
    if (L.targets && L.loss) *L.loss += (float)(lsum * L.inv_count);
}

static void run_output_dgrad(const OutputLaunch& L, float* gfeat) {
    const int Cin = L.C + L.F, ncol = L.nconv * L.C;
    for (int b = 0; b < L.batch; ++b)
        for (int r = 0; r < L.Tf; ++r)
            for (int c = 0; c < L.F; ++c) {
                double s = 0.0;
                for (int j = 0; j < L.ofs; ++j) {
                    const int t = r - j + L.pad_left;
                    if (t < 0 || t >= L.T_out) continue;
                    const float* dp = L.dpre + ((long long)b * L.T_out + t) * ncol;
                    for (int conv = 0; conv < L.nconv; ++conv)
                        for (int oc = 0; oc < L.C; ++oc) s += dp[conv * L.C + oc] * (double)L.params[L.w_off[conv] + ((long long)j * Cin + L.C + c) * L.C + oc];
                }
                const long long gid = ((long long)b * L.Tf + r) * L.F + c;
                gfeat[gid] = (float)(s * (L.feat[gid] > 0.f ? 1.0 : 0.2));
            }
}

static void run_output_wgrad(const OutputLaunch& L, float* grads, double scale) {
    const int Cin = L.C + L.F, ncol = L.nconv * L.C;
    auto in = [&](int b, int row, int c) -> double {
        if (row < 0 || row >= L.Tf) return 0.0;
        if (c < L.C) return L.mix[((long long)b * L.T_in + L.crop_feat + row) * L.C + c];
        return L.feat[((long long)b * L.Tf + row) * L.F + (c - L.C)];
    };
    for (int conv = 0; conv < L.nconv; ++conv)
        for (int oc = 0; oc < L.C; ++oc) {
            const int k = conv * L.C + oc;
            for (int j = 0; j < L.ofs; ++j)
                for (int c = 0; c < Cin; ++c) {
                    double s = 0.0;
                    for (int b = 0; b < L.batch; ++b)
                        for (int t = 0; t < L.T_out; ++t) s += in(b, t + j - L.pad_left, c) * L.dpre[((long long)b * L.T_out + t) * ncol + k];
                    grads[L.w_off[conv] + ((long long)j * Cin + c) * L.C + oc] += (float)(s * scale);
                }
            double sb = 0.0;
            for (int b = 0; b < L.batch; ++b)
                for (int t = 0; t < L.T_out; ++t) sb += L.dpre[((long long)b * L.T_out + t) * ncol + k];
            grads[L.b_off[conv] + oc] += (float)(sb * scale);
        }
}

static void run_upsample_bwd(const UpsampleBwdLaunch& L) {
    for (int c = 0; c < L.C; ++c) {
        const double w = L.blend ? L.blend[c] : 0.5;
        double dv = 0.0;
        for (int b = 0; b < L.batch; ++b) {
            const long long xb = (long long)b * L.N * L.C + c, mb = (long long)b * L.nmid * L.C + c;
            for (int s = 0; s < L.N; ++s) {
                double g = L.due[xb + (long long)s * L.C];
                const double dm = s < L.nmid ? L.dmid[mb + (long long)s * L.C] : 0.0;
                const double dmp = (s >= 1 && s - 1 < L.nmid) ? L.dmid[mb + (long long)(s - 1) * L.C] : 0.0;
                g += w * dm + (1.0 - w) * dmp;
                if (L.mid_mode == MID_CLAMP && s == L.N - 1) g += (1.0 - w) * dm;
                const double x = L.x[xb + (long long)s * L.C];
                L.gx[xb + (long long)s * L.C] = (float)(g * (x > 0.0 ? 1.0 : 0.2));
                if (L.dvar && s < L.nmid) {
                    const double nx = (s + 1 < L.N) ? L.x[xb + (long long)(s + 1) * L.C] : 0.0;
                    dv += dm * (x - nx);
                }
            }
        }
        if (L.dvar) L.dvar[c] += (float)(dv * w * (1.0 - w) * L.scale);
    }
}

static void run_first(const FirstLayer& L, int C, int N, const FirstWgrad* P) {
    // class 0: rows a = 2m, m in [0, Td) -> dec[b][m][n];  class 1: a = 2m + 1, m in [mo_lo, mo_hi) -> odd[b][m - mo_lo][n]
    std::vector<double> dW(P ? (size_t)L.k * C * N : 0, 0.0), db(P ? N : 0, 0.0);
    for (int q = 0; q < 2; ++q) {
        const int m_lo = q == 0 ? 0 : L.mo_lo, m_hi = q == 0 ? L.Td : L.mo_hi;
        for (int b = 0; b < L.batch; ++b) {
            const float* xb = L.x + (long long)b * L.x_bstride;
            float* yb = q == 0 ? L.dec + (long long)b * L.dec_bstride : L.odd + (long long)b * L.odd_bstride - (long long)L.mo_lo * N;
            for (int m = m_lo; m < m_hi; ++m) {
                const int a = 2 * m + q;
                for (int n = 0; n < N; ++n) {
                    if (!P) {
                        double s = L.bias[n];
                        for (int j = 0; j < L.k; ++j) {
                            const int t = a + j - L.pad_left;
                            if (t < 0 || t >= L.T) continue;
                            for (int c = 0; c < C; ++c) s += (double)xb[(long long)t * C + c] * L.W[((long long)j * C + c) * N + n];
                        }
                        yb[(long long)m * N + n] = (float)lrelu(s);
                    } else {
                        const double g = yb[(long long)m * N + n];
                        db[n] += g;
                        for (int j = 0; j < L.k; ++j) {
                            const int t = a + j - L.pad_left;
                            if (t < 0 || t >= L.T) continue;
                            for (int c = 0; c < C; ++c) dW[((size_t)j * C + c) * N + n] += (double)xb[(long long)t * C + c] * g;
                        }
                    }
                }
            }
        }
    }
    if (P) {
        for (size_t i = 0; i < dW.size(); ++i) P->dW[i] += (float)(dW[i] * P->scale);
        if (P->db) for (int n = 0; n < N; ++n) P->db[n] += (float)(db[n] * P->scale);
    }
}

static int template_int(const std::string& name, int index) {
    size_t p = name.find('<');
    if (p == std::string::npos) return -1;
    size_t e = name.find('>', p);
    std::string args = name.substr(p + 1, e - p - 1);
    size_t pos = 0;
    for (int i = 0; i < index; ++i) { pos = args.find(',', pos); if (pos == std::string::npos) return -1; ++pos; }
    return atoi(args.c_str() + pos);
}

// -> false when the kernel is unknown (or its packed weights are missing): the caller reports it
bool execute(const std::string& name, void** args) {
    if (has(name, "plane_conv_umma_persistent_out"))
        return run_umma_conv(*static_cast<const UmmaLaunch*>(args[0]), static_cast<const OutputFuse*>(args[2]));
    if (has(name, "plane_conv_umma_")) return run_umma_conv(*static_cast<const UmmaLaunch*>(args[0]), nullptr);
    if (has(name, "umma_pack_kernel")) { run_pack(*static_cast<const UmmaPackLaunch*>(args[0])); return true; }
    if (has(name, "wgrad_umma_bulk_kernel") || has(name, "wgrad_umma_kernel")) {
        const UmmaWgradLaunch& L = *static_cast<const UmmaWgradLaunch*>(args[0]);
        for (int g = 0; g < L.ngroups; ++g) {
            const WgGroup& G = L.grp[g];
            wgrad_group(G.P, G.G, G.m_lo, G.m_hi, G.ntaps, G.d, G.woff, L.dW, L.w_sp, L.w_sg, L.scale, L.batch, true);
        }
        return true;
    }
    // the partial tiles / per-CTA column sums are an internal format of the device kernels: the wgrad and split references above
    // and below produce the final dW and bias sums themselves, so what the reduction adds on the device is already there
    if (has(name, "wgrad_reduce_kernel") || has(name, "first_wgrad_sum_kernel")) return true;
    if (has(name, "split_views_kernel")) {              // the split arrays themselves are an internal operand format of the device
        const SplitJobs& J = *static_cast<const SplitJobs*>(args[0]);      // kernels; what the rest of the step sees: the bias sums
        for (int j = 0; j < J.njobs; ++j) {
            const SplitJob& S = J.job[j];
            if (!S.colsum) continue;
            for (int c = 0; c < S.V.C; ++c) {
                double s = 0.0;
                for (int b = 0; b < J.batch; ++b)
                    for (int r = S.row0; r < S.row0 + S.rows; ++r) s += plane_at(S.V, b, r, c);
                S.colsum[c] += (float)(s * J.colsum_scale);
            }
        }
        return true;
    }
    if (has(name, "first_fwd_kernel")) { run_first(*static_cast<const FirstLayer*>(args[0]), template_int(name, 0), template_int(name, 1), nullptr); return true; }
    if (has(name, "first_wgrad_kernel")) {
        const FirstWgrad& P = *static_cast<const FirstWgrad*>(args[0]);
        run_first(P.L, template_int(name, 0), template_int(name, 1), &P);
        return true;
    }
    if (has(name, "plane_conv_kernel")) { run_conv(*static_cast<const ConvLaunch*>(args[0])); return true; }
    if (has(name, "plane_wgrad_kernel") || has(name, "plane_wgrad_smallc_kernel")) {
        const WgradLaunch& W = *static_cast<const WgradLaunch*>(args[0]);
        wgrad_group(W.plane, W.dpre, W.m_lo, W.m_hi, W.nterms, W.d, W.woff, W.dW, W.w_sk, W.w_sn, W.scale, W.batch);
        return true;
    }
    if (has(name, "colsum_kernel")) {
        const PlaneView& V = *static_cast<const PlaneView*>(args[0]);
        const int batch = *static_cast<const int*>(args[1]);
        const double scale = *static_cast<const float*>(args[3]);
        float* out = *static_cast<float* const*>(args[4]);
        for (int c = 0; c < V.C; ++c) {
            double s = 0.0;
            for (int b = 0; b < batch; ++b)
                for (int r = V.r_lo; r < V.r_hi; ++r) s += V.base[(long long)b * V.bstride + (long long)r * V.rstride + c];
            out[c] += (float)(s * scale);
        }
        return true;
    }
    if (has(name, "output_fwd_kernel")) { run_output_fwd(*static_cast<const OutputLaunch*>(args[0])); return true; }
    if (has(name, "output_dgrad_kernel")) { run_output_dgrad(*static_cast<const OutputLaunch*>(args[0]), *static_cast<float* const*>(args[1])); return true; }
    // output_wgrad_kernel leaves per-CTA sums; the reference of the whole gradient runs at the launch that adds them up
    if (has(name, "output_wgrad_kernel")) return true;
    if (has(name, "output_wgrad_sum_kernel")) {
        run_output_wgrad(*static_cast<const OutputLaunch*>(args[0]), *static_cast<float* const*>(args[3]), *static_cast<const float*>(args[4]));
        return true;
    }
    if (has(name, "upsample_bwd_kernel")) { run_upsample_bwd(*static_cast<const UpsampleBwdLaunch*>(args[0])); return true; }
    if (has(name, "sigmoid_kernel")) {
        const float* x = *static_cast<const float* const*>(args[0]);
        float* y = *static_cast<float* const*>(args[1]);
        const int n = *static_cast<const int*>(args[2]);
        for (int i = 0; i < n; ++i) y[i] = (float)(1.0 / (1.0 + exp(-(double)x[i])));
        return true;
    }
    if (has(name, "adam_advance_kernel")) {
        float* st = *static_cast<float* const*>(args[0]);
        st[0] *= *static_cast<const float*>(args[1]);
        st[1] *= *static_cast<const float*>(args[2]);
        st[2] += 1.f;
        return true;
    }
    if (has(name, "adam_kernel")) {
        float* p = *static_cast<float* const*>(args[0]);
        const float* g = *static_cast<const float* const*>(args[1]);
        float* m = *static_cast<float* const*>(args[2]);
        float* v = *static_cast<float* const*>(args[3]);
        const long long n = *static_cast<const long long*>(args[4]);
        double lr_t = *static_cast<const float*>(args[5]);
        const double b1 = *static_cast<const float*>(args[6]), b2 = *static_cast<const float*>(args[7]), eps = *static_cast<const float*>(args[8]);
        const float* st = *static_cast<const float* const*>(args[9]);
        if (st) lr_t = lr_t * sqrt(1.0 - st[1]) / (1.0 - st[0]);
        for (long long i = 0; i < n; ++i) {
            const double mk = b1 * m[i] + (1.0 - b1) * g[i], vk = b2 * v[i] + (1.0 - b2) * (double)g[i] * g[i];
            m[i] = (float)mk; v[i] = (float)vk;
            p[i] = (float)(p[i] - lr_t * mk / (sqrt(vk) + eps));
        }
        return true;
    }
    if (has(name, "gather_windows_kernel")) {              // Evaluate.py:131-132
        const float* padded = *static_cast<const float* const*>(args[0]);
        const long long n_padded = *static_cast<const long long*>(args[1]);
        const long long* starts = *static_cast<const long long* const*>(args[2]);
        const int nw = *static_cast<const int*>(args[3]), T_in = *static_cast<const int*>(args[4]), C = *static_cast<const int*>(args[5]);
        float* out = *static_cast<float* const*>(args[6]);
        for (int w = 0; w < nw; ++w)
            for (long long off = 0; off < (long long)T_in * C; ++off) {
                const long long src = starts[w] * C + off;
                out[(long long)w * T_in * C + off] = src < n_padded * C ? padded[src] : 0.f;
            }
        return true;
    }
    if (has(name, "scatter_windows_kernel")) {             // Evaluate.py:138-139: plain overwrite, the shifted last window wins
        const float* outs = *static_cast<const float* const*>(args[0]);
        const long long* starts = *static_cast<const long long* const*>(args[1]);
        const int nw = *static_cast<const int*>(args[2]), K = *static_cast<const int*>(args[3]), T_out = *static_cast<const int*>(args[4]),
                  C = *static_cast<const int*>(args[5]);
        float* preds = *static_cast<float* const*>(args[6]);
        const long long n_frames = *static_cast<const long long*>(args[7]);
        for (int k = 0; k < K; ++k)
            for (int w = 0; w < nw; ++w)
                for (int t = 0; t < T_out; ++t) {
                    const long long frame = starts[w] + t;
                    if (frame >= n_frames) continue;
                    for (int c = 0; c < C; ++c) preds[((long long)k * n_frames + frame) * C + c] = outs[(((long long)k * nw + w) * T_out + t) * C + c];
                }
        return true;
    }
    return false;
}

void reset() {
    g_packs.clear();
    const char* e = getenv("FAKECUDA_MMA_MODEL");
    g_mma_model = e ? atoi(e) : 0;
}

}  // namespace cpudev
