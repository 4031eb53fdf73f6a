// kernels_first.cu - dedicated CUDA-core kernels for the first down block (C_in = 1 | 2 waveform channels;
// UnetAudioSeparator.py:97-100 with i = 0): forward and weight (+ bias) gradient.  Memory-shaped work (AI 13 FLOP/B) that
// stays off the tensor cores and is cheaper in these kernels than in the generic plane kernels; WUN_FIRST_LAYER=0
// selects the generic plane kernels.
//   first_fwd_kernel   thread = 2 output rows x all N filters in registers; x staged de-interleaved by parity so that the
//                      stride-2 row reads are conflict-free; weights read as warp-broadcast float4 from shared memory
//   first_wgrad_kernel 16 thread groups take the rows of a chunk round-robin; thread = 6 (tap, channel) x 8 filter
//                      register tile (5 shared-memory loads per 48 FMAs); groups reduce through shared memory, one atomic per
//                      weight per CTA; the bias gradient (column sum of g) rides along
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.h"

namespace wun {

// ------------------------------------------------------------------------------------------------
// forward: block = 128 threads = 256 consecutive class rows of one batch item
// ------------------------------------------------------------------------------------------------
template <int C, int N>
__global__ void __launch_bounds__(128) first_fwd_kernel(const __grid_constant__ FirstLayer L) {
    constexpr int ROWS = 256, KMAX = 16;
    __shared__ __align__(16) float Ws[KMAX * C * N];
    __shared__ float bs[N];
    // x de-interleaved by parity of (t - t0): Xp[par][i][c] = x[t0 + 2i + par][c]
    __shared__ __align__(8) float Xp[2][ROWS + KMAX / 2 + 2][C];
    const int q = blockIdx.z, b = blockIdx.y, tid = threadIdx.x;
    const int m_lo = q == 0 ? 0 : L.mo_lo, m_hi = q == 0 ? L.Td : L.mo_hi;
    const int m0 = m_lo + blockIdx.x * ROWS;
    if (m0 >= m_hi) return;
    for (int i = tid; i < L.k * C * N; i += 128) Ws[i] = __ldg(L.W + i);
    if (tid < N) bs[tid] = __ldg(L.bias + tid);
    const int t0 = 2 * m0 + q - L.pad_left;         // x row of (row m0, tap 0)
    const int nt = 2 * ROWS + L.k;                  // x rows the tile can touch
    const float* xb = L.x + (long long)b * L.x_bstride;
    for (int i = tid; i < nt * C; i += 128) {
        const int tt = i / C, c = i - tt * C, t = t0 + tt;
        Xp[tt & 1][tt >> 1][c] = (t >= 0 && t < L.T) ? __ldg(xb + (long long)t * C + c) : 0.f;
    }
    __syncthreads();
    float acc[2][N];
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int n = 0; n < N; ++n) acc[r][n] = 0.f;
    for (int j = 0; j < L.k; ++j) {
        // row (m0 + i) reads x row t0 + 2i + j  ->  parity j & 1, index i + (j >> 1)
        float xv[2][C];
#pragma unroll
        for (int r = 0; r < 2; ++r)
#pragma unroll
            for (int c = 0; c < C; ++c) xv[r][c] = Xp[j & 1][tid + r * 128 + (j >> 1)][c];
#pragma unroll
        for (int c = 0; c < C; ++c) {
            const float4* w4 = reinterpret_cast<const float4*>(&Ws[(j * C + c) * N]);
#pragma unroll
            for (int n4 = 0; n4 < N / 4; ++n4) {
                const float4 w = w4[n4];
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    acc[r][4 * n4 + 0] = fmaf(xv[r][c], w.x, acc[r][4 * n4 + 0]);
                    acc[r][4 * n4 + 1] = fmaf(xv[r][c], w.y, acc[r][4 * n4 + 1]);
                    acc[r][4 * n4 + 2] = fmaf(xv[r][c], w.z, acc[r][4 * n4 + 2]);
                    acc[r][4 * n4 + 3] = fmaf(xv[r][c], w.w, acc[r][4 * n4 + 3]);
                }
            }
        }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int m = m0 + tid + r * 128;
        if (m >= m_hi) continue;
        float* o = (q == 0) ? L.dec + (long long)b * L.dec_bstride + (long long)m * N
                            : L.odd + (long long)b * L.odd_bstride + (long long)(m - L.mo_lo) * N;
#pragma unroll
        for (int n4 = 0; n4 < N / 4; ++n4) {
            float4 v;
            float y;
            y = acc[r][4 * n4 + 0] + bs[4 * n4 + 0]; v.x = fmaxf(0.2f * y, y);
            y = acc[r][4 * n4 + 1] + bs[4 * n4 + 1]; v.y = fmaxf(0.2f * y, y);
            y = acc[r][4 * n4 + 2] + bs[4 * n4 + 2]; v.z = fmaxf(0.2f * y, y);
            y = acc[r][4 * n4 + 3] + bs[4 * n4 + 3]; v.w = fmaxf(0.2f * y, y);
            reinterpret_cast<float4*>(o)[n4] = v;
        }
    }
}

// ------------------------------------------------------------------------------------------------
// weight (+ bias) gradient:  dW[j][c][n] += scale * sum x[a + j - pad][c] * g[a][n],   db[n] += scale * sum g[a][n]
// g = dPre of the two classes, stored like dec / odd.  block = 256 threads = 16 groups x 16 threads.
// ------------------------------------------------------------------------------------------------

template <int C, int N>
__global__ void __launch_bounds__(256) first_wgrad_kernel(const __grid_constant__ FirstWgrad P) {
    constexpr int RK = 128, KMAX = 16, XT = 6, NTL = 8;
    constexpr int NNT = N / NTL;                               // filter tiles
    const FirstLayer& L = P.L;
    const int XC = L.k * C;                                    // (tap, channel) pairs = consecutive floats of the window
    const int NXT = (XC + XT - 1) / XT;                        // x tiles; NXT * NNT <= 16 threads per group
    __shared__ __align__(16) float Gs[RK * N];
    __shared__ __align__(8) float Xs[(2 * RK + KMAX) * C + 8];
    __shared__ float red[KMAX * C * N + N];
    const int q = blockIdx.z, b = blockIdx.y, tid = threadIdx.x;
    const int m_lo = q == 0 ? 0 : L.mo_lo, m_hi = q == 0 ? L.Td : L.mo_hi;
    const int mc0 = m_lo + blockIdx.x * P.rows_per_cta;
    if (mc0 >= m_hi) return;
    const int mc1 = min(mc0 + P.rows_per_cta, m_hi);
    const int grp = tid >> 4, tx = tid & 15;
    const int xt = tx / NNT, ntile = tx - xt * NNT;
    const bool active = tx < NXT * NNT;
    for (int i = tid; i < XC * N + N; i += 256) red[i] = 0.f;
    float acc[XT][NTL], accb[NTL];
#pragma unroll
    for (int u = 0; u < XT; ++u)
#pragma unroll
        for (int v = 0; v < NTL; ++v) acc[u][v] = 0.f;
#pragma unroll
    for (int v = 0; v < NTL; ++v) accb[v] = 0.f;
    const float* xb = L.x + (long long)b * L.x_bstride;
    const float* gb = (q == 0) ? L.dec + (long long)b * L.dec_bstride : L.odd + (long long)b * L.odd_bstride - (long long)L.mo_lo * N;
    for (int mb = mc0; mb < mc1; mb += RK) {
        const int nr = min(RK, mc1 - mb);
        __syncthreads();
        // g rows mb .. mb+nr-1 (contiguous in memory)
        for (int i = tid; i < RK * N / 4; i += 256) {
            const int rr = (4 * i) / N;
            reinterpret_cast<float4*>(Gs)[i] = (rr < nr) ? __ldg(reinterpret_cast<const float4*>(gb + (long long)mb * N) + i) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
        // x rows t0 .. : row (mb + ri) tap j reads x row t0 + 2*ri + j
        const int t0 = 2 * mb + q - L.pad_left;
        for (int i = tid; i < (2 * RK + L.k) * C; i += 256) {
            const int tt = i / C, c = i - tt * C, t = t0 + tt;
            Xs[i] = (t >= 0 && t < L.T) ? __ldg(xb + (long long)t * C + c) : 0.f;
        }
        __syncthreads();
        if (active) {
            for (int ri = grp; ri < RK; ri += 16) {            // rows past nr hold g = 0
                float xv[XT], gv[NTL];
                const float* xp = &Xs[2 * ri * C + XT * xt];
#pragma unroll
                for (int u = 0; u < XT; ++u) xv[u] = xp[u];     // (2*ri*C + 6*xt) is even: 8-byte aligned pairs
                const float4* gp = reinterpret_cast<const float4*>(&Gs[ri * N + NTL * ntile]);
                const float4 g0 = gp[0], g1 = gp[1];
                gv[0] = g0.x; gv[1] = g0.y; gv[2] = g0.z; gv[3] = g0.w; gv[4] = g1.x; gv[5] = g1.y; gv[6] = g1.z; gv[7] = g1.w;
#pragma unroll
                for (int u = 0; u < XT; ++u)
#pragma unroll
                    for (int v = 0; v < NTL; ++v) acc[u][v] = fmaf(xv[u], gv[v], acc[u][v]);
                if (xt == 0) {
#pragma unroll
                    for (int v = 0; v < NTL; ++v) accb[v] += gv[v];
                }
            }
        }
    }
    // the 16 groups add their sums in group order (the threads of one group own distinct entries): the same bits on every run
    for (int g = 0; g < 16; ++g) {
        __syncthreads();
        if (active && grp == g) {
#pragma unroll
            for (int u = 0; u < XT; ++u) {
                const int jc = XT * xt + u;                     // = j*C + c
                if (jc < XC) {
#pragma unroll
                    for (int v = 0; v < NTL; ++v) red[jc * N + NTL * ntile + v] += acc[u][v];
                }
            }
            if (xt == 0) {
#pragma unroll
                for (int v = 0; v < NTL; ++v) red[XC * N + NTL * ntile + v] += accb[v];
            }
        }
    }
    __syncthreads();
    float* part = P.part + ((size_t)(q * gridDim.y + b) * gridDim.x + blockIdx.x) * (XC * N + N);
    for (int i = tid; i < XC * N + N; i += 256) part[i] = red[i];
}

// dW / db = scale * the CTAs' sums of first_wgrad_kernel, added in (class, item, row block) order
__global__ void __launch_bounds__(256) first_wgrad_sum_kernel(const __grid_constant__ FirstWgrad P, int C, int N) {
    const FirstLayer& L = P.L;
    const int len = L.k * C * N + N;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < len; i += gridDim.x * blockDim.x) {
        float s = 0.f;
        for (int q = 0; q < 2; ++q) {
            const int m_lo = q == 0 ? 0 : L.mo_lo, m_hi = q == 0 ? L.Td : L.mo_hi;
            for (int b = 0; b < L.batch; ++b)
                for (int x = 0; x < P.grid_x && m_lo + x * P.rows_per_cta < m_hi; ++x)     // (CTAs without rows wrote nothing)
                    s += P.part[((size_t)(q * L.batch + b) * P.grid_x + x) * len + i];
        }
        if (i < len - N) P.dW[i] += s * P.scale;
        else if (P.db) P.db[i - (len - N)] += s * P.scale;
    }
}

constexpr int kFirstCtas = 132 * 4;      // ~4 CTAs per SM

size_t first_wgrad_partial_bytes(int batch) {
    // launch_first_wgrad: rows_per_cta >= rows * batch / kFirstCtas, so <= kFirstCtas / batch + 1 row blocks per (item, class)
    return (size_t)2 * (kFirstCtas + batch) * (16 * 2 * 24 + 24) * sizeof(float) + 256;
}


bool first_layer_supported(int C, int N, int k) {
    // the wgrad kernel gives every (6-value x tile, 8-filter tile) pair one thread of a 16-thread group
    return (C == 1 || C == 2) && (N == 16 || N == 24) && k >= 1 && k <= 16 && ((k * C + 5) / 6) * (N / 8) <= 16;
}

void launch_first_fwd(const FirstLayer& L, int C, int N, cudaStream_t stream) {
    const int rows = max(L.Td, L.mo_hi - L.mo_lo);
    if (rows <= 0 || L.batch <= 0) return;
    dim3 grid((rows + 255) / 256, L.batch, 2);
    if (C == 2 && N == 24) first_fwd_kernel<2, 24><<<grid, 128, 0, stream>>>(L);
    else if (C == 1 && N == 24) first_fwd_kernel<1, 24><<<grid, 128, 0, stream>>>(L);
    else if (C == 2 && N == 16) first_fwd_kernel<2, 16><<<grid, 128, 0, stream>>>(L);
    else if (C == 1 && N == 16) first_fwd_kernel<1, 16><<<grid, 128, 0, stream>>>(L);
}

void launch_first_wgrad(FirstWgrad P, int C, int N, cudaStream_t stream) {
    const long long rows = max(P.L.Td, P.L.mo_hi - P.L.mo_lo);
    if (rows <= 0 || P.L.batch <= 0) return;
    long long per = (rows * P.L.batch + kFirstCtas - 1) / kFirstCtas;
    per = (per + 127) / 128 * 128;
    if (per > rows) per = (rows + 127) / 128 * 128;
    P.rows_per_cta = (int)per;
    P.grid_x = (int)((rows + per - 1) / per);
    dim3 grid((unsigned)P.grid_x, P.L.batch, 2);
    if (C == 2 && N == 24) first_wgrad_kernel<2, 24><<<grid, 256, 0, stream>>>(P);
    else if (C == 1 && N == 24) first_wgrad_kernel<1, 24><<<grid, 256, 0, stream>>>(P);
    else if (C == 2 && N == 16) first_wgrad_kernel<2, 16><<<grid, 256, 0, stream>>>(P);
    else if (C == 1 && N == 16) first_wgrad_kernel<1, 16><<<grid, 256, 0, stream>>>(P);
    first_wgrad_sum_kernel<<<(P.L.k * C * N + N + 255) / 256, 256, 0, stream>>>(P, C, N);
}

}  // namespace wun
