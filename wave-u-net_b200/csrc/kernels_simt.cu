// kernels_simt.cu - CUDA-core (fp32 FFMA) kernels of the Wave-U-Net engine.
//
// These are the exact-fp32 kernels: they run every layer shape the reference allows (any filter size,
// any channel count, 'same' or 'valid' padding) and are the path for the memory-bound / irregular
// layers (down0 with C_in = 1|2, the 1x1 output layer, tiny test nets).  The tensor-core (wgmma)
// kernels in kernels_umma.cu take over the regular, compute-bound layers.
//
// Reference semantics implemented here (file:line into /root/reference):
//   conv + bias + LeakyReLU(0.2) + decimation/crop as live-position planes  UnetAudioSeparator.py:97-102,123
//   linear / learned upsampling as MID planes                               UnetAudioSeparator.py:109-118, InterpolationLayer.py:19-39
//   output layer (independent / difference, tanh / clip)                   OutputLayer.py:5-23, Utils.py:82-92
//   MSE loss and its gradient                                               Training.py:50-63
//   Adam (TF formulation)                                                   Training.py:77
//   predict_track gather/scatter                                            Evaluate.py:125-139
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.h"
#include "launch.h"

namespace wun {

// ------------------------------------------------------------------------------------------------
// plane element load (zero outside the valid rows; MID planes blend two rows)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float plane_load(const PlaneView& P, int b, int r, int c) {
    if (r < P.r_lo || r >= P.r_hi || c >= P.C) return 0.f;
    const float* p = P.base + (long long)b * P.bstride + (long long)r * P.rstride + c;
    float x = __ldg(p);
    if (P.kind == PLANE_MID) {
        float nx;
        if (P.mid_mode == MID_VALID) nx = __ldg(p + P.rstride);
        else if (r + 1 < P.xrows) nx = __ldg(p + P.rstride);
        else nx = (P.mid_mode == MID_CLAMP) ? x : 0.f;
        if (P.blend) {
            float w = __ldg(P.blend + c);
            x = w * x + (1.f - w) * nx;          // InterpolationLayer.py:20-23
        } else {
            x = x + (nx - x) * 0.5f;             // resize_bilinear lerp, UnetAudioSeparator.py:115-117
        }
    }
    return x;
}

// ------------------------------------------------------------------------------------------------
// plane convolution: out_cls[b, m, n] = epi( sum_terms plane[b, m+d, :] . W_term[:, n] )
//   grid  = (ceil(max_rows/BM), ceil(N/BN), batch*ncls),  128 threads, 8x8 register tile / thread
// ------------------------------------------------------------------------------------------------
template <int BN, int CK>
__global__ void __launch_bounds__(128) plane_conv_kernel(const __grid_constant__ ConvLaunch L) {
    constexpr int NTH = BN / 8;
    constexpr int MTH = 128 / NTH;
    constexpr int BM = MTH * 8;
    constexpr int SPAN = 36;
    constexpr int SR = BM + SPAN;               // == 4 (mod 32): conflict-free transposed stores
    __shared__ float slab[CK][SR];
    __shared__ __align__(16) float wsm[8][CK][BN];

    const int tid = threadIdx.x;
    const int cls = blockIdx.z % L.ncls;
    const int b = blockIdx.z / L.ncls;
    const OutView& O = L.cls[cls];
    const int m0 = O.m_lo + blockIdx.x * BM;
    if (m0 >= O.m_hi) return;
    const int n0 = blockIdx.y * BN;
    const int n_t = tid % NTH, m_t = tid / NTH;

    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

    int t = O.term_begin;
    while (t < O.term_end) {
        const int p = L.terms[t].plane;
        int dmin = L.terms[t].d, dmax = dmin, t1 = t + 1;
        while (t1 < O.term_end && t1 - t < 8 && L.terms[t1].plane == p) {
            int d = L.terms[t1].d;
            int lo = d < dmin ? d : dmin, hi = d > dmax ? d : dmax;
            if (hi - lo > SPAN) break;
            dmin = lo; dmax = hi; ++t1;
        }
        const int nt = t1 - t;
        const PlaneView& P = L.planes[p];
        const int nrows = BM + (dmax - dmin);
        for (int c0 = 0; c0 < P.C; c0 += CK) {
            for (int idx = tid; idx < nrows * CK; idx += 128) {
                int c = idx % CK, rr = idx / CK;
                slab[c][rr] = plane_load(P, b, m0 + dmin + rr, c0 + c);
            }
            for (int idx = tid; idx < nt * CK * BN; idx += 128) {
                int n = idx % BN, c = (idx / BN) % CK, tt = idx / (BN * CK);
                int k = c0 + c, nn = n0 + n;
                float w = 0.f;
                if (k < P.C && nn < L.N)
                    w = __ldg(L.W + (long long)L.terms[t + tt].woff + (long long)k * L.w_sk + (long long)nn * L.w_sn);
                wsm[tt][c][n] = w;
            }
            __syncthreads();
            for (int tt = 0; tt < nt; ++tt) {
                const int doff = L.terms[t + tt].d - dmin + m_t * 8;
#pragma unroll
                for (int c = 0; c < CK; ++c) {
                    float a[8], bb[8];
#pragma unroll
                    for (int i = 0; i < 8; ++i) a[i] = slab[c][doff + i];
                    const float4 b0 = *reinterpret_cast<const float4*>(&wsm[tt][c][n_t * 8]);
                    const float4 b1 = *reinterpret_cast<const float4*>(&wsm[tt][c][n_t * 8 + 4]);
                    bb[0] = b0.x; bb[1] = b0.y; bb[2] = b0.z; bb[3] = b0.w;
                    bb[4] = b1.x; bb[5] = b1.y; bb[6] = b1.z; bb[7] = b1.w;
#pragma unroll
                    for (int i = 0; i < 8; ++i)
#pragma unroll
                        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
                }
            }
            __syncthreads();
        }
        t = t1;
    }

    // epilogue
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int m = m0 + m_t * 8 + i;
        if (m >= O.m_hi) break;
        const long long roff = (long long)b * O.bstride + (long long)m * O.rstride;
        const bool accum = (m >= O.acc_lo && m < O.acc_hi);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int n = n0 + n_t * 8 + j;
            if (n >= L.N) break;
            float v = acc[i][j];
            if (L.epilogue == EPI_BIAS_LRELU) {
                if (L.bias) v += __ldg(L.bias + n);
                v = fmaxf(0.2f * v, v);                       // Utils.py:79-80
            } else if (L.epilogue == EPI_SLOPE && O.saved) {
                const float s = __ldg(O.saved + roff + n);
                v *= (s > 0.f) ? 1.f : 0.2f;                  // MaximumGrad: slope 0.2 at 0
            }
            float* dst = O.base + roff + n;
            if (accum) v += *dst;
            *dst = v;
        }
    }
}

void launch_plane_conv_simt(const ConvLaunch& L, cudaStream_t stream) {
    // pick the column tile that wastes the least work
    auto waste = [&](int bn) { return ((L.N + bn - 1) / bn) * bn; };
    int bn = 64;
    if (waste(32) < waste(64)) bn = 32;
    if (L.N <= 16) bn = 16;
    const int nth = bn / 8, bm = (128 / nth) * 8;
    dim3 grid((L.max_rows + bm - 1) / bm, (L.N + bn - 1) / bn, L.batch * L.ncls);
    if (grid.x == 0 || grid.y == 0 || grid.z == 0) return;
    int maxc = 0;
    for (int p = 0; p < L.nplanes; ++p) maxc = (L.planes[p].C > maxc) ? L.planes[p].C : maxc;
    if (maxc <= 2) {            // first layer (mono / stereo input): 2-channel chunks instead of 8
        if (bn == 64) plane_conv_kernel<64, 2><<<grid, 128, 0, stream>>>(L);
        else if (bn == 32) plane_conv_kernel<32, 2><<<grid, 128, 0, stream>>>(L);
        else plane_conv_kernel<16, 2><<<grid, 128, 0, stream>>>(L);
    } else {
        if (bn == 64) plane_conv_kernel<64, 8><<<grid, 128, 0, stream>>>(L);
        else if (bn == 32) plane_conv_kernel<32, 8><<<grid, 128, 0, stream>>>(L);
        else plane_conv_kernel<16, 8><<<grid, 128, 0, stream>>>(L);
    }
}

// ------------------------------------------------------------------------------------------------
// wgrad: dW[woff_t + c*sk + n*sn] += scale * sum_{b,m} plane[b, m+d_t, c] * dpre[b, m, n]
//   grid = (row chunks * batch, ceil(C/16), ceil(N/64)), 128 threads.
//   thread (m_t, n_t): tap = m_t/2, channels (m_t%2)*8..+8, columns n_t*8..+8
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) plane_wgrad_kernel(const __grid_constant__ WgradLaunch L) {
    constexpr int RK = 32, CI = 16, CO = 64, XR = RK + 16;
    __shared__ __align__(16) float Xs[XR][CI];
    __shared__ __align__(16) float Ys[RK][CO];
    const int tid = threadIdx.x;
    const int rows = L.m_hi - L.m_lo;
    const int chunks = (rows + L.rows_per_cta - 1) / L.rows_per_cta;
    const int b = blockIdx.x / chunks;
    const int mc0 = L.m_lo + (blockIdx.x % chunks) * L.rows_per_cta;
    const int mc1 = min(mc0 + L.rows_per_cta, L.m_hi);
    const int ci0 = blockIdx.y * CI, co0 = blockIdx.z * CO;
    const int n_t = tid % 8, m_t = tid / 8;
    const int tap = m_t >> 1, csub = (m_t & 1) * 8;
    int dmin = L.d[0], dmax = L.d[0];
    for (int i = 1; i < L.nterms; ++i) { dmin = min(dmin, L.d[i]); dmax = max(dmax, L.d[i]); }
    const int span = dmax - dmin;
    const bool active = tap < L.nterms;
    const int doff = active ? (L.d[tap] - dmin) : 0;

    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

    for (int mb = mc0; mb < mc1; mb += RK) {
        const int nr = min(RK, mc1 - mb);
        for (int idx = tid; idx < (RK + span) * CI; idx += 128) {
            int c = idx % CI, rr = idx / CI;
            float v = 0.f;
            if (rr < nr + span) v = plane_load(L.plane, b, mb + dmin + rr, ci0 + c);
            Xs[rr][c] = v;
        }
        for (int idx = tid; idx < RK * CO; idx += 128) {
            int n = idx % CO, rr = idx / CO;
            float v = 0.f;
            if (rr < nr) v = plane_load(L.dpre, b, mb + rr, co0 + n);
            Ys[rr][n] = v;
        }
        __syncthreads();
        if (active) {
#pragma unroll 4
            for (int r = 0; r < RK; ++r) {
                const float4 a0 = *reinterpret_cast<const float4*>(&Xs[r + doff][csub]);
                const float4 a1 = *reinterpret_cast<const float4*>(&Xs[r + doff][csub + 4]);
                const float4 b0 = *reinterpret_cast<const float4*>(&Ys[r][n_t * 8]);
                const float4 b1 = *reinterpret_cast<const float4*>(&Ys[r][n_t * 8 + 4]);
                const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
                const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
                for (int i = 0; i < 8; ++i)
#pragma unroll
                    for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
            }
        }
        __syncthreads();
    }
    if (!active) return;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int c = ci0 + csub + i;
        if (c >= L.plane.C) break;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int n = co0 + n_t * 8 + j;
            if (n >= L.N) break;
            atomicAdd(L.dW + (long long)L.woff[tap] + (long long)c * L.w_sk + (long long)n * L.w_sn,
                      acc[i][j] * L.scale);
        }
    }
}

// ------------------------------------------------------------------------------------------------
// wgrad for planes with very few channels (the first layer: C_in = 1 or 2).  Thread = (tap, channel, 4 output
// columns); the row chunk is staged in shared memory.  grid = (row chunks * batch), 256 threads.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) plane_wgrad_smallc_kernel(const __grid_constant__ WgradLaunch L) {
    constexpr int RK = 128, XR = RK + 16;
    __shared__ float Xs[XR][4];
    __shared__ __align__(16) float Gs[RK * 64];
    const int tid = threadIdx.x;
    const int C = L.plane.C, N = L.N, NQ = (N + 3) / 4, NP = NQ * 4;
    const int rows = L.m_hi - L.m_lo;
    const int chunks = (rows + L.rows_per_cta - 1) / L.rows_per_cta;
    const int b = blockIdx.x / chunks;
    const int mc0 = L.m_lo + (blockIdx.x % chunks) * L.rows_per_cta;
    const int mc1 = min(mc0 + L.rows_per_cta, L.m_hi);
    int dmin = L.d[0], dmax = L.d[0];
    for (int i = 1; i < L.nterms; ++i) { dmin = min(dmin, L.d[i]); dmax = max(dmax, L.d[i]); }
    const int span = dmax - dmin;
    const int OG = L.nterms * C * NQ;                // output groups (tap, c, column quad)
    // when there are few output groups, several thread groups split the rows of a chunk between them
    const int parts = (OG <= 128) ? 256 / OG : 1;
    const int og = (OG <= 128) ? tid % OG : tid;
    const int part = (OG <= 128) ? tid / OG : 0;
    const bool active = (OG <= 128) ? (part < parts) : true;
    float acc[2][4];
#pragma unroll
    for (int u = 0; u < 2; ++u)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[u][j] = 0.f;
    for (int mb = mc0; mb < mc1; mb += RK) {
        const int nr = min(RK, mc1 - mb);
        for (int idx = tid; idx < (RK + span) * 4; idx += 256) {
            const int c = idx & 3, rr = idx >> 2;
            Xs[rr][c] = (rr < nr + span && c < C) ? plane_load(L.plane, b, mb + dmin + rr, c) : 0.f;
        }
        for (int idx = tid; idx < RK * NP; idx += 256) {
            const int n = idx % NP, rr = idx / NP;
            Gs[idx] = (rr < nr && n < N) ? plane_load(L.dpre, b, mb + rr, n) : 0.f;
        }
        __syncthreads();
        if (active) {
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                const int o = og + u * 256;
                if (o < OG && (u == 0 || OG > 128)) {
                    const int nq = o % NQ, tc = o / NQ;
                    const int c = tc % C, doff = L.d[tc / C] - dmin;
                    for (int r = part; r < RK; r += parts) {
                        const float x = Xs[r + doff][c];
                        const float4 g = *reinterpret_cast<const float4*>(&Gs[r * NP + nq * 4]);
                        acc[u][0] = fmaf(x, g.x, acc[u][0]); acc[u][1] = fmaf(x, g.y, acc[u][1]);
                        acc[u][2] = fmaf(x, g.z, acc[u][2]); acc[u][3] = fmaf(x, g.w, acc[u][3]);
                    }
                }
            }
        }
        __syncthreads();
    }
    if (!active) return;
#pragma unroll
    for (int u = 0; u < 2; ++u) {
        const int o = og + u * 256;
        if (o >= OG || (u == 1 && OG <= 128)) continue;
        const int nq = o % NQ, tc = o / NQ;
        const int c = tc % C, t = tc / C;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int n = nq * 4 + j;
            if (n < N) atomicAdd(L.dW + (long long)L.woff[t] + (long long)c * L.w_sk + (long long)n * L.w_sn, acc[u][j] * L.scale);
        }
    }
}

void launch_plane_wgrad_simt(WgradLaunch L, cudaStream_t stream) {
    const int rows = L.m_hi - L.m_lo;
    if (rows <= 0 || L.nterms <= 0) return;
    if (L.plane.C <= 4 && L.N <= 64 && L.nterms * L.plane.C * ((L.N + 3) / 4) <= 512) {
        long long per = ((long long)rows * L.batch + 132 * 6 - 1) / (132 * 6);
        per = ((per + 127) / 128) * 128;
        if (per > rows) per = ((rows + 127) / 128) * 128;
        L.rows_per_cta = (int)per;
        const int chunks = (rows + L.rows_per_cta - 1) / L.rows_per_cta;
        plane_wgrad_smallc_kernel<<<chunks * L.batch, 256, 0, stream>>>(L);
        return;
    }
    const int tiles = ((L.plane.C + 15) / 16) * ((L.N + 63) / 64);
    // aim at ~8 CTAs per SM over the whole launch, at least 32 rows per CTA
    long long target = 132LL * 8;
    long long per = ((long long)rows * L.batch * tiles + target - 1) / target;
    per = ((per + 31) / 32) * 32;
    if (per < 32) per = 32;
    if (per > rows) per = ((rows + 31) / 32) * 32;
    L.rows_per_cta = (int)per;
    const int chunks = (rows + L.rows_per_cta - 1) / L.rows_per_cta;
    dim3 grid(chunks * L.batch, (L.plane.C + 15) / 16, (L.N + 63) / 64);
    plane_wgrad_kernel<<<grid, 128, 0, stream>>>(L);
}

// ------------------------------------------------------------------------------------------------
// column sum (bias gradient): out[n] += scale * sum_{b, m in [r_lo,r_hi)} view[b, m, n]
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) colsum_kernel(PlaneView V, int batch, int rows_per_cta, float scale,
                                                      float* __restrict__ out) {
    __shared__ float red[8][33];
    const int lane = threadIdx.x % 32, rl = threadIdx.x / 32;
    const int rows = V.r_hi - V.r_lo;
    const int chunks = (rows + rows_per_cta - 1) / rows_per_cta;
    const int b = blockIdx.x / chunks;
    const int r0 = V.r_lo + (blockIdx.x % chunks) * rows_per_cta;
    const int r1 = min(r0 + rows_per_cta, V.r_hi);
    const int n = blockIdx.y * 32 + lane;
    float s = 0.f;
    if (n < V.C) {
        const float* p = V.base + (long long)b * V.bstride + n;
        for (int r = r0 + rl; r < r1; r += 8) s += __ldg(p + (long long)r * V.rstride);
    }
    red[rl][lane] = s;
    __syncthreads();
    if (rl == 0 && n < V.C) {
        float tot = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) tot += red[i][lane];
        atomicAdd(out + n, tot * scale);
    }
}

void launch_colsum(const PlaneView& V, int batch, float scale, float* out, cudaStream_t stream) {
    const int rows = V.r_hi - V.r_lo;
    if (rows <= 0) return;
    long long per = ((long long)rows * batch + 132 * 4 - 1) / (132 * 4);
    if (per < 64) per = 64;
    if (per > rows) per = rows;
    const int chunks = (rows + (int)per - 1) / (int)per;
    dim3 grid(chunks * batch, (V.C + 31) / 32);
    colsum_kernel<<<grid, 256, 0, stream>>>(V, batch, (int)per, scale, out);
}

// ------------------------------------------------------------------------------------------------
// output layer forward (+ loss + dpre).  One thread per output frame (b, t).
// ------------------------------------------------------------------------------------------------
constexpr int kMaxOutCols = WUN_MAX_OUT_COLS;   // nconv * C

__device__ __forceinline__ float out_in_load(const OutputLaunch& L, int b, int row, int c) {
    // input of the output conv = [crop(mix) || features]  (UnetAudioSeparator.py:127); `row` is in
    // feature-row coordinates, zero outside [0, Tf) ('same' padding).
    if (row < 0 || row >= L.Tf) return 0.f;
    if (c < L.C) return __ldg(L.mix + ((long long)b * L.T_in + L.crop_feat + row) * L.C + c);
    return __ldg(L.feat + ((long long)b * L.Tf + row) * L.F + (c - L.C));
}

__global__ void __launch_bounds__(128) output_fwd_kernel(const __grid_constant__ OutputLaunch L) {
    extern __shared__ float wsm[];   // [nconv][ofs][Cin][C] then bias [nconv][C]
    const int Cin = L.C + L.F;
    const int wn = L.nconv * L.ofs * Cin * L.C;
    for (int i = threadIdx.x; i < wn + L.nconv * L.C; i += blockDim.x) {
        float v;
        if (i < wn) {
            int conv = i / (L.ofs * Cin * L.C), rem = i % (L.ofs * Cin * L.C);
            v = __ldg(L.params + L.w_off[conv] + rem);
        } else {
            int conv = (i - wn) / L.C, c = (i - wn) % L.C;
            v = __ldg(L.params + L.b_off[conv] + c);
        }
        wsm[i] = v;
    }
    __syncthreads();
    const float* bsm = wsm + wn;
    const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)L.batch * L.T_out;
    float lsum = 0.f;
    if (gid < total) {
        const int b = (int)(gid / L.T_out), t = (int)(gid % L.T_out);
        float pre[kMaxOutCols];
        const int ncol = L.nconv * L.C;
        for (int q = 0; q < ncol; ++q) pre[q] = bsm[q];
        for (int j = 0; j < L.ofs; ++j) {
            const int row = t + j - L.pad_left;
            for (int c = 0; c < Cin; ++c) {
                const float x = out_in_load(L, b, row, c);
                for (int conv = 0; conv < L.nconv; ++conv)
                    for (int oc = 0; oc < L.C; ++oc)
                        pre[conv * L.C + oc] = fmaf(x, wsm[((conv * L.ofs + j) * Cin + c) * L.C + oc],
                                                    pre[conv * L.C + oc]);
            }
        }
        // activation (UnetAudioSeparator.py:131-136)
        float est[kMaxOutCols];
        for (int q = 0; q < ncol; ++q) {
            float v = pre[q];
            if (L.activation == 0) v = tanhf(v);
            else if (!L.training) v = fminf(fmaxf(v, -1.f), 1.f);     // AudioClip, Utils.py:89-92
            est[q] = v;
        }
        const long long frame = ((long long)b * L.T_out + t) * L.C;
        const long long src_stride = (long long)L.batch * L.T_out * L.C;
        float g_last[4] = {0.f, 0.f, 0.f, 0.f};
        const bool diff = (L.output_type == 1);
        if (diff) {   // OutputLayer.py:17-22
            for (int oc = 0; oc < L.C; ++oc) {
                float s = 0.f;
                for (int conv = 0; conv < L.nconv; ++conv) s += est[conv * L.C + oc];
                float last = __ldg(L.mix + ((long long)b * L.T_in + L.crop_out + t) * L.C + oc) - s;
                if (!L.training) last = fminf(fmaxf(last, -1.f), 1.f);
                if (L.outputs) L.outputs[(long long)L.nconv * src_stride + frame + oc] = last;
                if (L.targets) {
                    float e = last - __ldg(L.targets + (long long)L.nconv * src_stride + frame + oc);
                    lsum += e * e;
                    g_last[oc] = 2.f * e * L.inv_count;
                }
            }
        }
        for (int conv = 0; conv < L.nconv; ++conv)
            for (int oc = 0; oc < L.C; ++oc) {
                const int q = conv * L.C + oc;
                if (L.outputs) L.outputs[(long long)conv * src_stride + frame + oc] = est[q];
                if (L.targets) {
                    float e = est[q] - __ldg(L.targets + (long long)conv * src_stride + frame + oc);
                    lsum += e * e;
                    float g = 2.f * e * L.inv_count - g_last[oc];       // Training.py:62-63 / OutputLayer.py:20
                    if (L.activation == 0) g *= (1.f - est[q] * est[q]);  // tanh'
                    L.dpre[((long long)b * L.T_out + t) * ncol + q] = g;
                }
            }
    }
    if (L.targets && L.loss) {
        // every CTA stores its sum; the CTA that finishes last adds all of them in a fixed order (thread t: sums t, t + 128, ...,
        // then a fixed tree) with one += into *loss - the same bits on every run, unlike float atomics from the CTAs
        __shared__ float red[128];
        __shared__ bool last;
        for (int o = 16; o > 0; o >>= 1) lsum += __shfl_xor_sync(0xffffffffu, lsum, o);
        if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = lsum;
        __syncthreads();
        if (threadIdx.x == 0) {
            L.loss_part[blockIdx.x] = (red[0] + red[1] + red[2] + red[3]) * L.inv_count;
            __threadfence();
            last = atomicAdd(L.loss_count, 1u) == gridDim.x - 1;
        }
        __syncthreads();
        if (last) {
            float s = 0.f;
            for (unsigned i0 = threadIdx.x; i0 < gridDim.x; i0 += 512) {           // 4 loads in flight, added in order
                float v[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) v[u] = (i0 + 128 * u < gridDim.x) ? __ldcg(L.loss_part + i0 + 128 * u) : 0.f;
#pragma unroll
                for (int u = 0; u < 4; ++u) s += v[u];
            }
            red[threadIdx.x] = s;
            for (int h = 64; h > 0; h >>= 1) {
                __syncthreads();
                if (threadIdx.x < h) red[threadIdx.x] += red[threadIdx.x + h];
            }
            if (threadIdx.x == 0) {
                *L.loss += red[0];
                *L.loss_count = 0u;                  // ready for the next launch
            }
        }
    }
}

size_t output_loss_partial_bytes(int batch, int T_out) {
    return (size_t)(((long long)batch * T_out + 127) / 128) * sizeof(float) + 256;
}

void launch_output_fwd(const OutputLaunch& L, cudaStream_t stream) {
    const long long total = (long long)L.batch * L.T_out;
    const int Cin = L.C + L.F;
    const size_t smem = (size_t)(L.nconv * L.ofs * Cin * L.C + L.nconv * L.C) * sizeof(float);
    output_fwd_kernel<<<(unsigned)((total + 127) / 128), 128, smem, stream>>>(L);
}

// dFeat[b,t,c] = slope(feat[b,t,c]) * sum_{conv,j,oc} dpre[b, t-j+pad, conv*C+oc] * W[conv][j][C+c][oc]
__global__ void __launch_bounds__(256) output_dgrad_kernel(const __grid_constant__ OutputLaunch L,
                                                            float* __restrict__ gfeat) {
    extern __shared__ float wsm[];   // [nconv][ofs][F][C]
    const int Cin = L.C + L.F;
    const int wn = L.nconv * L.ofs * L.F * L.C;
    for (int i = threadIdx.x; i < wn; i += blockDim.x) {
        int oc = i % L.C, c = (i / L.C) % L.F, j = (i / (L.C * L.F)) % L.ofs, conv = i / (L.C * L.F * L.ofs);
        wsm[i] = __ldg(L.params + L.w_off[conv] + ((long long)j * Cin + L.C + c) * L.C + oc);
    }
    __syncthreads();
    const long long total = (long long)L.batch * L.Tf * L.F;
    const int ncol = L.nconv * L.C;
    for (long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x; gid < total;
         gid += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(gid % L.F);
        const long long fr = gid / L.F;
        const int r = (int)(fr % L.Tf), b = (int)(fr / L.Tf);
        float s = 0.f;
        for (int j = 0; j < L.ofs; ++j) {
            const int t = r - j + L.pad_left;
            if (t < 0 || t >= L.T_out) continue;
            const float* dp = L.dpre + ((long long)b * L.T_out + t) * ncol;
            for (int conv = 0; conv < L.nconv; ++conv)
                for (int oc = 0; oc < L.C; ++oc)
                    s = fmaf(__ldg(dp + conv * L.C + oc), wsm[((conv * L.ofs + j) * L.F + c) * L.C + oc], s);
        }
        const float a = __ldg(L.feat + gid);
        gfeat[gid] = s * ((a > 0.f) ? 1.f : 0.2f);
    }
}

void launch_output_dgrad(const OutputLaunch& L, float* gfeat, cudaStream_t stream) {
    const long long total = (long long)L.batch * L.Tf * L.F;
    const size_t smem = (size_t)(L.nconv * L.ofs * L.F * L.C) * sizeof(float);
    int blocks = (int)((total + 255) / 256);
    if (blocks > 132 * 16) blocks = 132 * 16;
    output_dgrad_kernel<<<blocks, 256, smem, stream>>>(L, gfeat);
}

constexpr int kOutWgradCtas = 132 * 4;     // row chunks of the output-layer weight gradient (~4 CTAs per SM)

// dW[conv][j][c][oc] += scale * sum_{b,t} in[b, t+j-pad, c] * dpre[b,t,conv*C+oc];  db likewise.
//   block = 8 row lanes x 32 channel lanes; grid.x = row chunks, grid.y = tap j.  Every CTA stores its sums at
//   part[(tap * gridDim.x + chunk) * (Cin + 1) * ncol ...]; output_wgrad_sum_kernel adds them in chunk order (the same bits on
//   every run, unlike float atomics from the CTAs)
__global__ void __launch_bounds__(256) output_wgrad_kernel(const __grid_constant__ OutputLaunch L, float* __restrict__ part,
                                                            int rows_per_cta) {
    __shared__ float red[8][32];
    const int lane = threadIdx.x % 32, rl = threadIdx.x / 32;
    const int Cin = L.C + L.F;
    const int ncol = L.nconv * L.C;
    const int j = blockIdx.y;
    const long long total = (long long)L.batch * L.T_out;
    const long long g0 = (long long)blockIdx.x * rows_per_cta;
    const long long g1 = min(g0 + rows_per_cta, total);
    for (int cbase = 0; cbase < Cin + 1; cbase += 32) {       // channel index Cin = the bias "channel"
        const int c = cbase + lane;
        float acc[kMaxOutCols];
        for (int q = 0; q < ncol; ++q) acc[q] = 0.f;
        if (c <= Cin && (c < Cin || j == 0)) {
            for (long long g = g0 + rl; g < g1; g += 8) {
                const int b = (int)(g / L.T_out), t = (int)(g % L.T_out);
                const float x = (c < Cin) ? out_in_load(L, b, t + j - L.pad_left, c) : 1.f;
                const float* dp = L.dpre + g * ncol;
                for (int q = 0; q < ncol; ++q) acc[q] = fmaf(x, __ldg(dp + q), acc[q]);
            }
        }
        for (int q = 0; q < ncol; ++q) {
            red[rl][lane] = acc[q];
            __syncthreads();
            if (rl == 0 && c <= Cin && (c < Cin || j == 0)) {
                float tot = 0.f;
                for (int i = 0; i < 8; ++i) tot += red[i][lane];
                part[((size_t)j * gridDim.x + blockIdx.x) * (Cin + 1) * ncol + (size_t)c * ncol + q] = tot;
            }
            __syncthreads();
        }
    }
}

// grads of the output convs = scale * the sums of output_wgrad_kernel's CTAs, added in chunk order
__global__ void __launch_bounds__(256) output_wgrad_sum_kernel(const __grid_constant__ OutputLaunch L, const float* __restrict__ part,
                                                                int nx, float* __restrict__ grads, float scale) {
    const int Cin = L.C + L.F, ncol = L.nconv * L.C, per_tap = (Cin + 1) * ncol;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < L.ofs * per_tap; i += gridDim.x * blockDim.x) {
        const int j = i / per_tap, c = (i % per_tap) / ncol, q = i % ncol;
        if (c == Cin && j != 0) continue;                       // the bias "channel" exists for tap 0 only
        float s = 0.f;
        for (int x = 0; x < nx; ++x) s += part[((size_t)j * nx + x) * per_tap + (size_t)c * ncol + q];
        const int conv = q / L.C, oc = q % L.C;
        if (c < Cin) grads[L.w_off[conv] + ((long long)j * Cin + c) * L.C + oc] += s * scale;
        else grads[L.b_off[conv] + oc] += s * scale;
    }
}

size_t output_wgrad_partial_bytes(const OutputLaunch& L) {
    return (size_t)(kOutWgradCtas + 1) * L.ofs * (L.C + L.F + 1) * L.nconv * L.C * sizeof(float) + 256;
}

void launch_output_wgrad(const OutputLaunch& L, float* grads, float* part, float scale, cudaStream_t stream) {
    const long long total = (long long)L.batch * L.T_out;
    long long per = (total + kOutWgradCtas - 1) / kOutWgradCtas;
    if (per < 64) per = 64;
    const int nx = (int)((total + per - 1) / per);
    output_wgrad_kernel<<<dim3(nx, L.ofs), 256, 0, stream>>>(L, part, (int)per);
    const int len = L.ofs * (L.C + L.F + 1) * L.nconv * L.C;
    output_wgrad_sum_kernel<<<(len + 255) / 256, 256, 0, stream>>>(L, part, nx, grads, scale);
}

// ------------------------------------------------------------------------------------------------
// upsampling backward: dX[s] = dUe[s] + a*dMid[s] + (1-a)*dMid[s-1] (+ boundary), times the LeakyReLU
// slope of the producer's saved output; learned: dvar[c] += w(1-w) * sum dMid*(x[s]-x[s+1]).
//   block (32 channels, 8 rows); grid (ceil(C/32), row chunks * batch)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) upsample_bwd_kernel(const __grid_constant__ UpsampleBwdLaunch L) {
    __shared__ float red[8][32];
    const int c = blockIdx.x * 32 + threadIdx.x;
    const int chunks = (L.N + L.rows_per_cta - 1) / L.rows_per_cta;
    const int b = blockIdx.y / chunks;
    const int s0 = (blockIdx.y % chunks) * L.rows_per_cta;
    const int s1 = min(s0 + L.rows_per_cta, L.N);
    float dv = 0.f;
    if (c < L.C) {
        const float w = L.blend ? __ldg(L.blend + c) : 0.5f;
        const long long xb = (long long)b * L.N * L.C + c;
        const long long mb = (long long)b * L.nmid * L.C + c;
        for (int s = s0 + threadIdx.y; s < s1; s += 8) {
            float g = __ldg(L.due + xb + (long long)s * L.C);
            const float dm = (s < L.nmid) ? __ldg(L.dmid + mb + (long long)s * L.C) : 0.f;
            const float dmp = (s >= 1 && s - 1 < L.nmid) ? __ldg(L.dmid + mb + (long long)(s - 1) * L.C) : 0.f;
            g += w * dm + (1.f - w) * dmp;
            if (L.mid_mode == MID_CLAMP && s == L.N - 1) g += (1.f - w) * dm;   // next row clamped onto itself
            const float x = __ldg(L.x + xb + (long long)s * L.C);
            L.gx[xb + (long long)s * L.C] = g * ((x > 0.f) ? 1.f : 0.2f);
            if (L.dvar && s < L.nmid) {
                float nx = 0.f;
                if (s + 1 < L.N) nx = __ldg(L.x + xb + (long long)(s + 1) * L.C);
                dv += dm * (x - nx);
            }
        }
    }
    if (L.dvar) {
        // every CTA stores its sums at slot (item, row chunk) = blockIdx.y; the CTA that finishes last adds the slots of every
        // channel in a fixed order (thread row ty: slots ty, ty + 8, ..., then the 8 rows in order), applies w(1-w) * scale once
        // and does one += into dvar - the same bits on every run, unlike float atomics from the CTAs
        __shared__ bool last;
        red[threadIdx.y][threadIdx.x] = dv;
        __syncthreads();
        if (threadIdx.y == 0) {
            if (c < L.C) {
                float tot = 0.f;
                for (int i = 0; i < 8; ++i) tot += red[i][threadIdx.x];
                L.part[(long long)blockIdx.y * L.C + c] = tot;
            }
            __threadfence();                     // the slot is visible before this CTA is counted
        }
        __syncthreads();
        if (threadIdx.x == 0 && threadIdx.y == 0) last = atomicAdd(L.count, 1u) == gridDim.x * gridDim.y - 1;
        __syncthreads();
        if (!last) return;
        for (int cb = 0; cb < L.C; cb += 32) {
            const int cc = cb + threadIdx.x;
            float s = 0.f;
            if (cc < L.C)
                for (unsigned y0 = threadIdx.y; y0 < gridDim.y; y0 += 64) {      // 8 loads in flight, added in slot order
                    float v[8];
#pragma unroll
                    for (int u = 0; u < 8; ++u) {
                        const unsigned y = y0 + 8 * u;
                        v[u] = (y < gridDim.y) ? __ldcg(L.part + (long long)y * L.C + cc) : 0.f;
                    }
#pragma unroll
                    for (int u = 0; u < 8; ++u) s += v[u];
                }
            __syncthreads();
            red[threadIdx.y][threadIdx.x] = s;
            __syncthreads();
            if (threadIdx.y == 0 && cc < L.C) {
                float tot = 0.f;
                for (int i = 0; i < 8; ++i) tot += red[i][threadIdx.x];
                const float w = __ldg(L.blend + cc);
                L.dvar[cc] += tot * w * (1.f - w) * L.scale;
            }
        }
        if (threadIdx.x == 0 && threadIdx.y == 0) *L.count = 0u;     // ready for the next launch
    }
}

static int upsample_rows_per_cta(int N, int batch) {
    long long per = ((long long)N * batch + 132 * 4 - 1) / (132 * 4);
    if (per < 32) per = 32;
    if (per > N) per = N;
    return (int)per;
}

size_t upsample_dvar_partial_bytes(int batch, int C) {
    // rows_per_cta >= N * batch / 528 or >= 32 > N * batch / 528 or = N: at most 528 + batch CTAs along y
    return (size_t)(132 * 4 + batch) * C * sizeof(float) + 256;
}

void launch_upsample_bwd(UpsampleBwdLaunch L, cudaStream_t stream) {
    L.rows_per_cta = upsample_rows_per_cta(L.N, L.batch);
    const int chunks = (L.N + L.rows_per_cta - 1) / L.rows_per_cta;
    dim3 grid((L.C + 31) / 32, chunks * L.batch), block(32, 8);
    upsample_bwd_kernel<<<grid, block, 0, stream>>>(L);
}

// ------------------------------------------------------------------------------------------------
// small elementwise kernels
// ------------------------------------------------------------------------------------------------
__global__ void sigmoid_kernel(const float* __restrict__ x, float* __restrict__ y, int n) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) y[i] = 1.f / (1.f + expf(-x[i]));
}
void launch_sigmoid(const float* x, float* y, int n, cudaStream_t stream) {
    sigmoid_kernel<<<(n + 127) / 128, 128, 0, stream>>>(x, y, n);
}

// tf.train.AdamOptimizer: p -= lr_t * m / (sqrt(v) + eps) (Training.py:77).  lr_t comes either folded on the host
// (state == nullptr) or from the device-resident accumulators state = {beta1_power, beta2_power, step} that TF keeps as
// the variables beta1_power / beta2_power: lr_t = lr * sqrt(1 - beta2_power) / (1 - beta1_power).  The second form is
// what a CUDA-graph replay needs - nothing step-dependent is baked into the launch; adam_advance_kernel moves the
// accumulators after the update, like TF's _finish().
__global__ void __launch_bounds__(256) adam_kernel(float* __restrict__ p, const float* __restrict__ g,
                                                    float* __restrict__ m, float* __restrict__ v, long long n,
                                                    float lr_t, float b1, float b2, float eps,
                                                    const float* __restrict__ state) {
    if (state) lr_t = lr_t * sqrtf(1.f - state[1]) / (1.f - state[0]);
    const long long stride = (long long)gridDim.x * blockDim.x * 4;
    for (long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 4; i < n; i += stride) {
        if (i + 3 < n) {
            float4 pp = *reinterpret_cast<float4*>(p + i);
            const float4 gg = *reinterpret_cast<const float4*>(g + i);
            float4 mm = *reinterpret_cast<float4*>(m + i);
            float4 vv = *reinterpret_cast<float4*>(v + i);
#define WUN_ADAM1(f)                                          \
    mm.f = b1 * mm.f + (1.f - b1) * gg.f;                     \
    vv.f = b2 * vv.f + (1.f - b2) * gg.f * gg.f;              \
    pp.f -= lr_t * mm.f / (sqrtf(vv.f) + eps);
            WUN_ADAM1(x) WUN_ADAM1(y) WUN_ADAM1(z) WUN_ADAM1(w)
#undef WUN_ADAM1
            *reinterpret_cast<float4*>(p + i) = pp;
            *reinterpret_cast<float4*>(m + i) = mm;
            *reinterpret_cast<float4*>(v + i) = vv;
        } else {
            for (long long k = i; k < n; ++k) {
                float mk = b1 * m[k] + (1.f - b1) * g[k];
                float vk = b2 * v[k] + (1.f - b2) * g[k] * g[k];
                m[k] = mk; v[k] = vk;
                p[k] -= lr_t * mk / (sqrtf(vk) + eps);
            }
        }
    }
}
__global__ void adam_advance_kernel(float* state, float b1, float b2) {
    state[0] *= b1;
    state[1] *= b2;
    state[2] += 1.f;
}
void launch_adam(float* p, const float* g, float* m, float* v, long long n, float lr_t, float b1, float b2,
                 float eps, float* state, cudaStream_t stream) {
    long long blocks = (n / 4 + 255) / 256;
    if (blocks > 132 * 8) blocks = 132 * 8;
    if (blocks < 1) blocks = 1;
    adam_kernel<<<(unsigned)blocks, 256, 0, stream>>>(p, g, m, v, n, lr_t, b1, b2, eps, state);
    if (state) adam_advance_kernel<<<1, 1, 0, stream>>>(state, b1, b2);
}

// Evaluate.py:131-132 (gather) and :138-139 (scatter, plain overwrite; later windows win because
// windows are processed in order and only the LAST one can overlap its predecessor)
__global__ void gather_windows_kernel(const float* __restrict__ padded, long long n_padded,
                                      const long long* __restrict__ starts, int n_windows, int T_in, int C,
                                      float* __restrict__ out) {
    const long long per = (long long)T_in * C;
    const long long total = per * n_windows;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int w = (int)(i / per);
        const long long off = i % per;
        const long long src = starts[w] * C + off;
        out[i] = (src < n_padded * C) ? __ldg(padded + src) : 0.f;
    }
}
void launch_gather_windows(const float* padded, long long n_padded, const long long* starts, int n_windows,
                           int T_in, int C, float* out, cudaStream_t stream) {
    long long total = (long long)T_in * C * n_windows;
    long long blocks = (total + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    if (blocks < 1) return;
    gather_windows_kernel<<<(unsigned)blocks, 256, 0, stream>>>(padded, n_padded, starts, n_windows, T_in, C, out);
}

__global__ void scatter_windows_kernel(const float* __restrict__ outs, const long long* __restrict__ starts,
                                       int n_windows, int n_sources, int T_out, int C, float* __restrict__ preds,
                                       long long n_frames) {
    // a frame covered by window w and by the (shifted) last window takes the last window's value
    const long long per = (long long)T_out * C;
    const long long total = per * n_windows * n_sources;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const long long off = i % per;
        const int w = (int)((i / per) % n_windows);
        const int s = (int)(i / (per * n_windows));
        const long long frame = starts[w] + off / C;
        if (frame >= n_frames) continue;
        if (w != n_windows - 1 && frame >= starts[n_windows - 1]) continue;   // overwritten by the last window
        preds[(long long)s * n_frames * C + frame * C + off % C] = __ldg(outs + i);
    }
}
void launch_scatter_windows(const float* outs, const long long* starts, int n_windows, int n_sources, int T_out,
                            int C, float* preds, long long n_frames, cudaStream_t stream) {
    long long total = (long long)T_out * C * n_windows * n_sources;
    long long blocks = (total + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    if (blocks < 1) return;
    scatter_windows_kernel<<<(unsigned)blocks, 256, 0, stream>>>(outs, starts, n_windows, n_sources, T_out, C,
                                                                preds, n_frames);
}

}  // namespace wun
