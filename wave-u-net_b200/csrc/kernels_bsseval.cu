// BSS Eval v4 ("images" decomposition, filters solved once over the whole track, applied frame by frame) in fp64:
// museval 0.2.0 evaluate(references, estimates, win, hop, mode="v4"), which the reference calls through
// museval.eval_mus_track (Evaluate.py:71).  DESIGN.md §4.5 describes the stages; oracle/bsseval_oracle.py restates them
// in numpy.
//
// BSS Eval v3 (mode="v3": the same decomposition with the filters solved again for every frame, from that frame's samples
// only) runs the same stages over batches of frames (wun_bss_eval_v3, DESIGN.md §4.12).
//
// museval's bss_eval switches (wun_bss_eval_ex, DESIGN.md §4.13): the permutation search scores every (reference,
// estimate) pair and keeps, per frame, the pairing with the largest mean SIR; the "sources" decomposition changes SDR and
// drops ISR.  wun_bss_eval and wun_bss_eval_v3 are that driver with flags 0 and WUN_BSS_FRAMEWISE_FILTERS.
//
// Every sum runs in a fixed order (per-CTA partial slots, then an ordered second pass; no float atomics), so a call
// returns the same bits on every run.  fp32 inputs are widened to fp64 when staged: each product of two of them is exact.
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "../../include/wun.h"

namespace {

constexpr int kL = 512;              // museval filters_len
constexpr int kR = 8;                // outputs (lags or samples) per thread, kept in registers
constexpr int kXcThreads = kL / kR;  // one CTA covers all L lags of a signal pair
constexpr int kXcChunk = 1024;       // samples staged per step
constexpr int kMaxSegs = 256;        // sample segments of the correlation (partial slots per lag)
constexpr int kPanel = 64;           // LDL^T panel width
constexpr int kFrThreads = 128;
constexpr int kFrTile = kFrThreads * kR;  // output samples per framewise CTA

__host__ __device__ constexpr int skew(int i) { return i + (i >> 4); }  // one pad double per 16: stride-8 reads hit distinct banks

// The frames one launch covers.  v4 (list == nullptr): a single slot, the whole track.  v3: slot s of the pass is frame
// list[1 + s0 + s] while s0 + s < list[0] (list holds the frames that are not silent, in order) and idle beyond, so that
// silent frames cost no work although the host, which never synchronises, does not know how many there are.  Batched
// kernels hold `per` systems per slot.
struct Pass {
    const int* list;
    int64_t s0;
    int per;
};

__device__ __forceinline__ int64_t pass_frame(const Pass& p, int64_t slot) {
    if (!p.list) return 0;
    return p.s0 + slot < p.list[0] ? p.list[1 + p.s0 + slot] : -1;
}

// ---- stage 1: lag correlations corr(x, y, tau) = sum_m x[m] y[m + tau], tau in [0, L) ----------------------------------------
// Task t = a * 2nref + s pairs reference signal a = (k, c) with signal s: references 0..nref-1, then estimates.  G needs
// every ordered reference pair (corr(a, b, -tau) = corr(b, a, tau)), D every (reference, estimate) pair.  CTA (seg, t) sums
// its segment of samples; thread i owns lags 8i .. 8i+7 and slides a window of y through registers.
// v3 (blockIdx.z: the pass's slot): the frame's slice [t*hop, t*hop + win) stands for the whole track, so a product that
// reaches outside the frame is never formed - museval zero-extends each slice.
__global__ void __launch_bounds__(kXcThreads) bss_xcorr_kernel(const float* __restrict__ ref, const float* __restrict__ est,
                                                                int nsrc, int nchan, int64_t N, int64_t seg_len,
                                                                double* __restrict__ slots, Pass pass, int64_t win,
                                                                int64_t hop) {
    const int64_t t = pass_frame(pass, blockIdx.z);
    if (t < 0) return;
    __shared__ double xs[kXcChunk];
    __shared__ double ys[skew(kXcChunk + kL)];
    const int nref = nsrc * nchan, task = blockIdx.y, tid = threadIdx.x;
    const int a = task / (2 * nref), s = task % (2 * nref), b = s % nref;
    const int64_t f0 = pass.list ? t * hop : 0, len = pass.list ? win : N;
    const float* xp = ref + ((int64_t)(a / nchan) * N + f0) * nchan + a % nchan;
    const float* yp = (s < nref ? ref : est) + ((int64_t)(b / nchan) * N + f0) * nchan + b % nchan;
    const int64_t lo = (int64_t)blockIdx.x * seg_len, hi = min(len, lo + seg_len);
    double acc[kR];
#pragma unroll
    for (int i = 0; i < kR; ++i) acc[i] = 0.0;
    for (int64_t m0 = lo; m0 < hi; m0 += kXcChunk) {
        __syncthreads();
        for (int i = tid; i < kXcChunk; i += kXcThreads) {
            const int64_t m = m0 + i;
            xs[i] = m < hi ? (double)xp[m * nchan] : 0.0;
        }
        for (int i = tid; i < kXcChunk + kL; i += kXcThreads) {
            const int64_t m = m0 + i;
            ys[skew(i)] = m < len ? (double)yp[m * nchan] : 0.0;
        }
        __syncthreads();
        double w[2 * kR];
#pragma unroll
        for (int k = 0; k < kR; ++k) w[k] = ys[skew(kR * tid + k)];
        for (int mb = 0; mb < kXcChunk; mb += kR) {
#pragma unroll
            for (int k = 0; k < kR; ++k) w[kR + k] = ys[skew(mb + kR * tid + kR + k)];
#pragma unroll
            for (int st = 0; st < kR; ++st) {
                const double xm = xs[mb + st];
#pragma unroll
                for (int i = 0; i < kR; ++i) acc[i] = fma(xm, w[st + i], acc[i]);
            }
#pragma unroll
            for (int k = 0; k < kR; ++k) w[k] = w[kR + k];
        }
    }
    double* out = slots + (((int64_t)blockIdx.z * gridDim.x + blockIdx.x) * gridDim.y + task) * kL + kR * tid;
#pragma unroll
    for (int i = 0; i < kR; ++i) out[i] = acc[i];
}

// lags[t][tau] = sum over segments in order (blockIdx.y: the pass's slot)
__global__ void bss_lag_reduce_kernel(const double* __restrict__ slots, int64_t nseg, int64_t nvals, double* __restrict__ lags,
                                      Pass pass) {
    const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= nvals || pass_frame(pass, blockIdx.y) < 0) return;
    slots += (int64_t)blockIdx.y * nseg * nvals;
    lags += (int64_t)blockIdx.y * nvals;
    double s = 0.0;
    for (int64_t g = 0; g < nseg; ++g) s += slots[g * nvals + v];
    lags[v] = s;
}

// ---- stage 2: assembly --------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double lag(const double* lags, int nref, int a, int s, int tau) {
    return lags[((int64_t)a * 2 * nref + s) * kL + tau];
}

// <S_p r_a, S_q r_b> = corr(a, b, p - q)
__device__ __forceinline__ double gram(const double* lags, int nref, int a, int p, int b, int q) {
    return p >= q ? lag(lags, nref, a, b, p - q) : lag(lags, nref, b, a, q - p);
}

// Lower triangle of G + eps I (z = 0, order nref*L) and of the diagonal blocks G[j,j] + eps I (z = 1 + j, order nchan*L).
// The epsilon is museval's: numpy's float64 eps, added to the whole diagonal.  blockIdx.z = slot * (1 + nsrc) + z.
__global__ void bss_assemble_gram_kernel(const double* __restrict__ lags, int nsrc, int nchan, double* __restrict__ G,
                                         double* __restrict__ Gjj, Pass pass) {
    const int nref = nsrc * nchan, slot = blockIdx.z / (1 + nsrc), z = blockIdx.z % (1 + nsrc);
    const int n = (z == 0 ? nref : nchan) * kL, a0 = z == 0 ? 0 : (z - 1) * nchan;
    const int i = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n || j > i || pass_frame(pass, slot) < 0) return;
    const int64_t nbig = (int64_t)nref * kL, nsmall = (int64_t)nchan * kL;
    lags += (int64_t)slot * 2 * nref * nref * kL;
    G += slot * nbig * nbig;
    Gjj += slot * nsrc * nsmall * nsmall;
    double* A = z == 0 ? G : Gjj + (int64_t)(z - 1) * n * n;
    double v = gram(lags, nref, a0 + i / kL, i % kL, a0 + j / kL, j % kL);
    if (i == j) v += 2.220446049250313e-16;
    A[(int64_t)i * n + j] = v;
}

// Right-hand sides, one contiguous column per (estimate j, estimate channel e):
//   C  [j][e][(k, c, l)]      = D_j[(k, c, l), e] = <S_l r_{k,c}, est_{j,e}>
//   Cj [jt][j'][e][(c, l)]    = D_j[(jt, c, l), e]   (reference jt's rows: the single-source system against G[jt,jt])
// Without pairs (npair 1) only jt == j is kept, at j' = 0; with pairs (npair = nsrc) every jt, at j' = j.
__global__ void bss_assemble_rhs_kernel(const double* __restrict__ lags, int nsrc, int nchan, int npair,
                                        double* __restrict__ C, double* __restrict__ Cj, Pass pass) {
    const int nref = nsrc * nchan, col = blockIdx.y, j = col / nchan, e = col % nchan;
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= nref * kL || pass_frame(pass, blockIdx.z) < 0) return;
    lags += (int64_t)blockIdx.z * 2 * nref * nref * kL;
    C += (int64_t)blockIdx.z * nref * nref * kL;
    Cj += (int64_t)blockIdx.z * nref * nchan * npair * kL;
    const int a = r / kL, l = r % kL, jt = a / nchan;
    const double v = lag(lags, nref, a, nref + j * nchan + e, l);
    C[(int64_t)col * nref * kL + r] = v;
    if (npair > 1 || jt == j)
        Cj[(((int64_t)jt * npair + (npair > 1 ? j : 0)) * nchan + e) * nchan * kL + (a % nchan) * kL + l] = v;
}

// ---- stage 3: blocked LDL^T without pivoting, in place on the lower triangle ------------------------------------------------
// After panel k0: L (unit diagonal implied) below the diagonal, D on it; the panel's columns of L are mirrored into the upper
// triangle (A[p][i] = L[i][p], i beyond the panel's diagonal block) so that back substitution reads them coalesced.
// Batch z: A + z * n * n.  n is a multiple of 64.
__global__ void __launch_bounds__(256) bss_ldl_diag_kernel(double* __restrict__ A0, int n, int k0, Pass pass) {
    if (pass_frame(pass, blockIdx.x / pass.per) < 0) return;
    __shared__ double S[kPanel][kPanel + 1];
    double* A = A0 + (int64_t)blockIdx.x * n * n;
    const int tid = threadIdx.x;
    for (int idx = tid; idx < kPanel * kPanel; idx += 256) {
        const int r = idx / kPanel, c = idx % kPanel;
        S[r][c] = c <= r ? A[(int64_t)(k0 + r) * n + k0 + c] : 0.0;
    }
    __syncthreads();
    for (int j = 0; j < kPanel; ++j) {
        const double d = S[j][j];
        for (int idx = tid; idx < kPanel * kPanel; idx += 256) {
            const int r = idx / kPanel, c = idx % kPanel;
            if (c > j && c <= r) S[r][c] -= S[r][j] * S[c][j] / d;
        }
        __syncthreads();
        if (tid > j && tid < kPanel) S[tid][j] /= d;
        __syncthreads();
    }
    for (int idx = tid; idx < kPanel * kPanel; idx += 256) {
        const int r = idx / kPanel, c = idx % kPanel;
        if (c <= r) A[(int64_t)(k0 + r) * n + k0 + c] = S[r][c];
    }
}

// Rows below the diagonal block: l_i = (L11^{-1} a_i) / d, one row per thread.
__global__ void __launch_bounds__(128) bss_ldl_panel_kernel(double* __restrict__ A0, int n, int k0, Pass pass) {
    if (pass_frame(pass, blockIdx.y / pass.per) < 0) return;
    extern __shared__ double sm[];
    double* Ld = sm;                          // [64][65]: L11 below, d on the diagonal
    double* R = sm + kPanel * (kPanel + 1);   // [64][129]: the CTA's rows, transposed
    double* A = A0 + (int64_t)blockIdx.y * n * n;
    const int tid = threadIdx.x, k1 = k0 + kPanel, row0 = k1 + blockIdx.x * 128;
    for (int idx = tid; idx < kPanel * kPanel; idx += 128) {
        const int r = idx / kPanel, c = idx % kPanel;
        Ld[r * (kPanel + 1) + c] = c <= r ? A[(int64_t)(k0 + r) * n + k0 + c] : 0.0;
    }
    for (int idx = tid; idx < 128 * kPanel; idx += 128) {
        const int rl = idx / kPanel, c = idx % kPanel, i = row0 + rl;
        R[c * 129 + rl] = i < n ? A[(int64_t)i * n + k0 + c] : 0.0;
    }
    __syncthreads();
    for (int c = 0; c < kPanel; ++c) {
        double s = R[c * 129 + tid];
        for (int p = 0; p < c; ++p) s -= Ld[c * (kPanel + 1) + p] * R[p * 129 + tid];
        R[c * 129 + tid] = s;
    }
    for (int c = 0; c < kPanel; ++c) R[c * 129 + tid] /= Ld[c * (kPanel + 1) + c];
    __syncthreads();
    for (int idx = tid; idx < 128 * kPanel; idx += 128) {
        const int rl = idx / kPanel, c = idx % kPanel, i = row0 + rl;
        if (i < n) A[(int64_t)i * n + k0 + c] = R[c * 129 + rl];
    }
    for (int idx = tid; idx < 128 * kPanel; idx += 128) {
        const int c = idx / 128, rl = idx % 128, i = row0 + rl;
        if (i < n) A[(int64_t)(k0 + c) * n + i] = R[c * 129 + rl];
    }
}

// Trailing update A22 -= L21 D L21^T on 64x64 lower tiles; 4x4 outputs per thread.
__global__ void __launch_bounds__(256) bss_ldl_update_kernel(double* __restrict__ A0, int n, int k0) {
    const int ti = blockIdx.y, tj = blockIdx.x;
    if (tj > ti) return;
    constexpr int kK = kPanel / 2;   // the panel's columns in two halves (static shared memory)
    __shared__ double Li[kK][kPanel + 4];
    __shared__ double Lj[kK][kPanel + 4];
    double* A = A0 + (int64_t)blockIdx.z * n * n;
    const int tid = threadIdx.x, k1 = k0 + kPanel, i0 = k1 + ti * kPanel, j0 = k1 + tj * kPanel;
    const int ty = tid / 16, tx = tid % 16;
    double acc[4][4] = {};
    for (int kh = 0; kh < kPanel; kh += kK) {
        __syncthreads();
        for (int idx = tid; idx < kPanel * kK; idx += 256) {
            const int r = idx / kK, k = idx % kK, kk = k0 + kh + k;
            Li[k][r] = A[(int64_t)(i0 + r) * n + kk];
            Lj[k][r] = A[(int64_t)(j0 + r) * n + kk] * A[(int64_t)kk * n + kk];
        }
        __syncthreads();
        for (int k = 0; k < kK; ++k) {
            double x[4], y[4];
#pragma unroll
            for (int r = 0; r < 4; ++r) { x[r] = Li[k][ty * 4 + r]; y[r] = Lj[k][tx * 4 + r]; }
#pragma unroll
            for (int r = 0; r < 4; ++r)
#pragma unroll
                for (int c = 0; c < 4; ++c) acc[r][c] = fma(x[r], y[c], acc[r][c]);
        }
    }
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const int i = i0 + ty * 4 + r, j = j0 + tx * 4 + c;
            if (j <= i) A[(int64_t)i * n + j] -= acc[r][c];
        }
}

// D = A B + C on the FP64 tensor cores, one 8x8x4 step: a = A[g][q], b = B[q][g], c/d = C[g][2q + i] (g = lane / 4, q = lane % 4).
__device__ __forceinline__ void dmma_8x8x4(double (&d)[2], double a, double b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};\n"
                 : "+d"(d[0]), "+d"(d[1])
                 : "d"(a), "d"(b));
}

// The same trailing update as bss_ldl_update_kernel (v3's batches of frames, blockIdx.z = system), with the products on the
// FP64 tensor cores: each warp owns a 16x32 part of the 64x64 tile as 2x4 accumulators of mma.m8n8k4, and the panel's
// columns run in k order, four per MMA.  Row pitch 36 doubles (4 mod 16): a fragment load's 8 rows x 4 columns hit
// distinct banks.
__global__ void __launch_bounds__(256) bss_ldl_update_dmma_kernel(double* __restrict__ A0, int n, int k0, Pass pass) {
    const int ti = blockIdx.y, tj = blockIdx.x;
    if (tj > ti || pass_frame(pass, blockIdx.z / pass.per) < 0) return;
    constexpr int kK = kPanel / 2, kPitch = kK + 4;
    __shared__ double Li[kPanel][kPitch];
    __shared__ double Lj[kPanel][kPitch];
    double* A = A0 + (int64_t)blockIdx.z * n * n;
    const int tid = threadIdx.x, lane = tid % 32, warp = tid / 32, g = lane / 4, q = lane % 4;
    const int k1 = k0 + kPanel, i0 = k1 + ti * kPanel, j0 = k1 + tj * kPanel;
    const int wr = (warp / 2) * 16, wc = (warp % 2) * 32;
    double acc[2][4][2] = {};
    for (int kh = 0; kh < kPanel; kh += kK) {
        __syncthreads();
        for (int idx = tid; idx < kPanel * kK; idx += 256) {
            const int r = idx / kK, k = idx % kK, kk = k0 + kh + k;
            Li[r][k] = A[(int64_t)(i0 + r) * n + kk];
            Lj[r][k] = A[(int64_t)(j0 + r) * n + kk] * A[(int64_t)kk * n + kk];
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < kK; k += 4) {
            double a[2], b[4];
#pragma unroll
            for (int r = 0; r < 2; ++r) a[r] = Li[wr + 8 * r + g][k + q];
#pragma unroll
            for (int c = 0; c < 4; ++c) b[c] = Lj[wc + 8 * c + g][k + q];
#pragma unroll
            for (int r = 0; r < 2; ++r)
#pragma unroll
                for (int c = 0; c < 4; ++c) dmma_8x8x4(acc[r][c], a[r], b[c]);
        }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c)
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int i = i0 + wr + 8 * r + g, j = j0 + wc + 8 * c + 2 * q + h;
                if (j <= i) A[(int64_t)i * n + j] -= acc[r][c][h];
            }
}

__device__ __forceinline__ double warp_sum(double s) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    return s;
}

// L D L^T x = b for one right-hand side column per CTA (grid: columns x batch), solved in place.  Left-looking: each
// panel's rows first subtract the finished part as warp dot products (coalesced along a row of L, or along the mirrored
// row of L^T), then the 64x64 unit-triangular block is solved column by column.
__global__ void __launch_bounds__(256) bss_ldl_solve_kernel(const double* __restrict__ A0, int n, double* __restrict__ B0,
                                                            Pass pass) {
    if (pass_frame(pass, blockIdx.y / pass.per) < 0) return;
    extern __shared__ double y[];
    const double* A = A0 + (int64_t)blockIdx.y * n * n;
    double* b = B0 + ((int64_t)blockIdx.y * gridDim.x + blockIdx.x) * n;
    const int tid = threadIdx.x, lane = tid % 32, warp = tid / 32;
    for (int i = tid; i < n; i += 256) y[i] = b[i];
    __syncthreads();
    for (int k0 = 0; k0 < n; k0 += kPanel) {
        for (int r = warp; r < kPanel; r += 8) {
            const double* row = A + (int64_t)(k0 + r) * n;
            double s = 0.0;
            for (int p = lane; p < k0; p += 32) s = fma(row[p], y[p], s);
            s = warp_sum(s);
            if (lane == 0) y[k0 + r] -= s;
        }
        __syncthreads();
        for (int j = 0; j < kPanel; ++j) {
            if (tid > j && tid < kPanel) y[k0 + tid] -= A[(int64_t)(k0 + tid) * n + k0 + j] * y[k0 + j];
            __syncthreads();
        }
    }
    for (int i = tid; i < n; i += 256) y[i] /= A[(int64_t)i * n + i];
    __syncthreads();
    for (int k0 = n - kPanel; k0 >= 0; k0 -= kPanel) {
        for (int r = warp; r < kPanel; r += 8) {
            const double* row = A + (int64_t)(k0 + r) * n;   // upper mirror: row[i] = L[i][k0 + r]
            double s = 0.0;
            for (int i = k0 + kPanel + lane; i < n; i += 32) s = fma(row[i], y[i], s);
            s = warp_sum(s);
            if (lane == 0) y[k0 + r] -= s;
        }
        __syncthreads();
        for (int j = kPanel - 1; j > 0; --j) {
            if (tid < j) y[k0 + tid] -= A[(int64_t)(k0 + j) * n + k0 + tid] * y[k0 + j];
            __syncthreads();
        }
    }
    for (int i = tid; i < n; i += 256) b[i] = y[i];
}

// ---- stage 4: framewise decomposition ---------------------------------------------------------------------------------------
// CTA (tile, estimate j, frame t): output samples w = tile*1024 + 8*tid + i of P_all = sum_{k,c} C_j * frame slice of r_{k,c}
// and, for each scored reference jt, P_j = sum_c Cj_{jt,j} * slice of r_{jt,c}, over the frame's W = win + L - 1 samples
// (slices zero-extended, no context from neighbouring frames).  Only the energies leave the CTA, as one ordered partial per
// (pair, tile).  Samples past W come out as zero (every tap reads beyond the slice there) and add nothing.
// Without pairs (npair 1) the one reference scored is jt = j.  With pairs (npair = nsrc) P_all is computed once and kept in
// registers while each other reference's P_j is filtered from its own slices, staged again.
// FRAMEWISE (v3): blockIdx.x / ntile is the pass's slot, which holds the frame's own filters; idle slots exit.
constexpr int kEnergies = 8;   // the images version writes the first seven, the sources version all eight

// xs[u] = slice[w0 - (L-1) + u] of signal xp (channel stride NCH), zero outside [0, win)
template <int NCH>
__device__ __forceinline__ void stage_slice(double* xs, const float* __restrict__ xp, int64_t f0, int64_t w0, int64_t win) {
    __syncthreads();
    for (int u = threadIdx.x; u < kFrTile + kL; u += kFrThreads) {
        const int64_t v = w0 - (kL - 1) + u;
        xs[skew(u)] = (v >= 0 && v < win) ? (double)xp[(f0 + v) * NCH] : 0.0;
    }
}

// P[w] += sum_u h[u] xs[w - w0 + u] for this thread's 8 samples: into pa with the taps h (ALL), into pj with hj (own).
template <int NCH, bool ALL>
__device__ __forceinline__ void filter_slice(const double* xs, const double (*h)[kL], const double (*hj)[kL], bool own,
                                             double (&pa)[NCH][kR], double (&pj)[NCH][kR]) {
    const int tid = threadIdx.x;
    double w[2 * kR];
#pragma unroll
    for (int k = 0; k < kR; ++k) w[k] = xs[skew(kR * tid + k)];
    for (int ub = 0; ub < kL; ub += kR) {
#pragma unroll
        for (int k = 0; k < kR; ++k) w[kR + k] = xs[skew(ub + kR * tid + kR + k)];
#pragma unroll
        for (int st = 0; st < kR; ++st) {
            if (ALL) {
#pragma unroll
                for (int e = 0; e < NCH; ++e) {
                    const double he = h[e][ub + st];
#pragma unroll
                    for (int i = 0; i < kR; ++i) pa[e][i] = fma(he, w[st + i], pa[e][i]);
                }
            }
            if (own) {
#pragma unroll
                for (int e = 0; e < NCH; ++e) {
                    const double he = hj[e][ub + st];
#pragma unroll
                    for (int i = 0; i < kR; ++i) pj[e][i] = fma(he, w[st + i], pj[e][i]);
                }
            }
        }
#pragma unroll
        for (int k = 0; k < kR; ++k) w[k] = w[kR + k];
    }
}

// The pair's energies (reference jt, estimate j) over the CTA, added in thread order into out[0 .. ne):
// E0 |P_j|^2, E1 |est - r_jt|^2, E2 |r_jt|^2, E3 |P_j - r_jt|^2, E4 |P_all - P_j|^2, E5 |P_all|^2, E6 |est - P_all|^2,
// E7 |est - P_j|^2.  The next use of `red` follows the barrier in stage_slice (or the kernel's end).
template <int NCH>
__device__ __forceinline__ void pair_energies(const float* __restrict__ ref, const float* __restrict__ est, int64_t N, int jt,
                                              int j, int64_t f0, int64_t w0, int64_t win, const double (&pa)[NCH][kR],
                                              const double (&pj)[NCH][kR], double (*red)[kFrThreads], int ne,
                                              double* __restrict__ out) {
    const int tid = threadIdx.x;
    double en[kEnergies] = {};
#pragma unroll
    for (int i = 0; i < kR; ++i) {
        const int64_t v = w0 + kR * tid + i;
#pragma unroll
        for (int e = 0; e < NCH; ++e) {
            const int64_t off = (f0 + v) * NCH + e;
            const double s = v < win ? (double)est[(int64_t)j * N * NCH + off] : 0.0;
            const double r = v < win ? (double)ref[(int64_t)jt * N * NCH + off] : 0.0;
            const double p = pj[e][i], q = pa[e][i];
            en[0] += p * p;
            en[1] += (s - r) * (s - r);
            en[2] += r * r;
            en[3] += (p - r) * (p - r);
            en[4] += (q - p) * (q - p);
            en[5] += q * q;
            en[6] += (s - q) * (s - q);
            en[7] += (s - p) * (s - p);
        }
    }
#pragma unroll
    for (int k = 0; k < kEnergies; ++k) red[k][tid] = en[k];
    __syncthreads();
    if (tid < ne) {
        double s = 0.0;
        for (int i = 0; i < kFrThreads; ++i) s += red[tid][i];
        out[tid] = s;
    }
}

template <int NCH, bool FRAMEWISE>
__global__ void __launch_bounds__(kFrThreads) bss_frame_energy_kernel(const float* __restrict__ ref, const float* __restrict__ est,
                                                                       const double* __restrict__ C, const double* __restrict__ Cj,
                                                                       int nsrc, int64_t N, int64_t win, int64_t hop, int ntile,
                                                                       int npair, int ne, double* __restrict__ energies,
                                                                       Pass pass) {
    const int64_t t = FRAMEWISE ? pass_frame(pass, blockIdx.x / ntile) : blockIdx.x / ntile;
    if (FRAMEWISE && t < 0) return;
    const int64_t slot = FRAMEWISE ? blockIdx.x / ntile : 0;   // the frame's own filters
    __shared__ double xs[skew(kFrTile + kL)];
    __shared__ double h[NCH][kL], hj[NCH][kL];
    __shared__ double red[kEnergies][kFrThreads];
    const int nref = nsrc * NCH, tid = threadIdx.x, j = blockIdx.y;
    const int tile = blockIdx.x % ntile;
    const int64_t f0 = t * hop, w0 = (int64_t)tile * kFrTile;
    const int jsel = npair > 1 ? j : 0;
    const double* cj = Cj + slot * nsrc * npair * NCH * NCH * kL;   // + (jt * npair + jsel) * NCH * NCH * kL: [e][c][l] of (jt, j)
    double* out = energies + (((int64_t)t * nsrc + j) * npair * ntile + tile) * ne;   // + (npair > 1 ? jt : 0) * ntile * ne
    double pa[NCH][kR], pj[NCH][kR];
#pragma unroll
    for (int e = 0; e < NCH; ++e)
#pragma unroll
        for (int i = 0; i < kR; ++i) pa[e][i] = pj[e][i] = 0.0;
    // P_all from every reference, and the P_j of reference j from the same staged slices
    for (int a = 0; a < nref; ++a) {
        const bool own = a / NCH == j;
        stage_slice<NCH>(xs, ref + (int64_t)(a / NCH) * N * NCH + a % NCH, f0, w0, win);
        // taps reversed so that P[w] = sum_u h[u] xs[w - w0 + u]
        for (int u = tid; u < NCH * kL; u += kFrThreads) {
            const int e = u / kL, l = u % kL;
            h[e][kL - 1 - l] = C[((slot * nref + j * NCH + e) * nref + a) * kL + l];
            if (own) hj[e][kL - 1 - l] = cj[((j * npair + jsel) * NCH * NCH + e * NCH + a % NCH) * kL + l];
        }
        __syncthreads();
        filter_slice<NCH, true>(xs, h, hj, own, pa, pj);
    }
    pair_energies<NCH>(ref, est, N, j, j, f0, w0, win, pa, pj, red, ne, out + (npair > 1 ? j : 0) * ntile * ne);
    for (int jt = 0; npair > 1 && jt < nsrc; ++jt) {
        if (jt == j) continue;
#pragma unroll
        for (int e = 0; e < NCH; ++e)
#pragma unroll
            for (int i = 0; i < kR; ++i) pj[e][i] = 0.0;
        for (int c = 0; c < NCH; ++c) {
            stage_slice<NCH>(xs, ref + (int64_t)jt * N * NCH + c, f0, w0, win);
            for (int u = tid; u < NCH * kL; u += kFrThreads) {
                const int e = u / kL, l = u % kL;
                hj[e][kL - 1 - l] = cj[((jt * npair + j) * NCH * NCH + e * NCH + c) * kL + l];
            }
            __syncthreads();
            filter_slice<NCH, false>(xs, h, hj, true, pa, pj);
        }
        pair_energies<NCH>(ref, est, N, jt, j, f0, w0, win, pa, pj, red, ne, out + jt * ntile * ne);
    }
}

__device__ __forceinline__ double safe_db(double num, double den) {
    return den == 0.0 ? __longlong_as_double(0x7ff0000000000000LL) : 10.0 * log10(num / den);
}

// museval's _any_source_silent over references and estimates: frame t is NaN for every target if some reference or some
// estimate has sum_c x[n][c] == 0 on every sample of it.  Called by every thread of the CTA.
__device__ bool frame_silent(const float* __restrict__ ref, const float* __restrict__ est, int nsrc, int nchan, int64_t N,
                             int64_t win, int64_t f0) {
    bool silent = false;
    for (int k = 0; k < 2 * nsrc; ++k) {
        const float* x = (k < nsrc ? ref : est) + (int64_t)(k % nsrc) * N * nchan;
        int nonzero = 0;
        for (int64_t v = threadIdx.x; v < win && !nonzero; v += blockDim.x) {
            double s = 0.0;
            for (int c = 0; c < nchan; ++c) s += (double)x[(f0 + v) * nchan + c];
            nonzero = s != 0.0;
        }
        silent |= !__syncthreads_or(nonzero);
    }
    return silent;
}

// One CTA per frame: the silence rule, then the four metrics of every scored pair from its tiles' energies (in order).
// Without pairs (npair 1): pair (j, j) into metrics [4][nsrc][nwin]; with pairs: every (jt, j) into [4][nsrc][nsrc][nwin].
__global__ void __launch_bounds__(256) bss_frame_metrics_kernel(const float* __restrict__ ref, const float* __restrict__ est,
                                                                int nsrc, int nchan, int64_t N, int64_t win, int64_t hop,
                                                                int64_t nwin, int ntile, int npair, bool sources,
                                                                const double* __restrict__ energies,
                                                                double* __restrict__ metrics) {
    const int64_t t = blockIdx.x, f0 = t * hop;
    const bool silent = frame_silent(ref, est, nsrc, nchan, N, win, f0);
    const int p = threadIdx.x, ne = sources ? 8 : 7;
    if (p >= nsrc * npair) return;
    const int j = p / npair, js = p % npair, jt = npair > 1 ? js : j;   // estimate j scored against reference jt
    double E[kEnergies] = {};
    for (int tile = 0; tile < ntile; ++tile)
#pragma unroll
        for (int k = 0; k < kEnergies; ++k)
            if (k < ne) E[k] += energies[((((int64_t)t * nsrc + j) * npair + js) * ntile + tile) * ne + k];
    const double nan = __longlong_as_double(0x7ff8000000000000LL);
    double sdr, isr;
    if (sources) {   // sources decomposition: s_filt = P_j
        sdr = silent ? nan : safe_db(E[0], E[7]);   // |s_filt|^2 / |e_interf + e_artif|^2
        isr = nan;
    } else {         // images decomposition: s_true = r_j, e_spat = P_j - r_j, e_interf = P_all - P_j, e_artif = est - P_all
        sdr = silent ? nan : safe_db(E[2], E[1]);   // |s_true|^2 / |e_spat + e_interf + e_artif|^2
        isr = silent ? nan : safe_db(E[2], E[3]);
    }
    const double sir = silent ? nan : safe_db(E[0], E[4]);
    const double sar = silent ? nan : safe_db(E[5], E[6]);
    const int64_t o = ((int64_t)jt * npair + (npair > 1 ? j : 0)) * nwin + t, m = (int64_t)nsrc * npair * nwin;
    metrics[o] = sdr;
    metrics[m + o] = isr;
    metrics[2 * m + o] = sir;
    metrics[3 * m + o] = sar;
}

// ---- permutation: choose, per frame, which reference each estimate is scored against ----------------------------------------
// Candidate idx of itertools.permutations(range(nsrc)): lexicographic order, so idx's factorial-base digits pick the
// remaining values in order.
__device__ void nth_permutation(int idx, int nsrc, int* perm) {
    int left[WUN_MAX_SOURCES];
    int f = 1;
    for (int k = 0; k < nsrc; ++k) left[k] = k;
    for (int k = 2; k < nsrc; ++k) f *= k;   // (nsrc - 1)!
    for (int pos = 0; pos < nsrc; ++pos) {
        const int d = idx / f;
        idx %= f;
        perm[pos] = left[d];
        for (int k = d; k < nsrc - 1 - pos; ++k) left[k] = left[k + 1];
        if (pos < nsrc - 1) f /= nsrc - 1 - pos;
    }
}

// numpy's argmax order: (a, ia) is taken over (b, ib) if it is the first NaN, or, with no NaN, the larger value or the
// earlier candidate of equal ones.  ib < 0: nothing yet.  A total order, so any reduction tree picks the same candidate.
__device__ __forceinline__ bool argmax_before(double a, int ia, double b, int ib) {
    if (ia < 0) return false;
    if (ib < 0) return true;
    const bool an = isnan(a), bn = isnan(b);
    if (an != bn) return an;
    if (!an && a != b) return a > b;
    return ia < ib;
}

// One CTA per frame: every candidate perm (estimate j paired with reference perm[j]) scored by its mean pair SIR, summed
// over j in order and divided by nsrc; the first maximum wins.  Then perm[j][t] and metrics[.][j][t] = pair[.][perm[j]][j][t].
__global__ void __launch_bounds__(256) bss_perm_select_kernel(const double* __restrict__ pair, int nsrc, int64_t nwin,
                                                              double* __restrict__ metrics, int64_t* __restrict__ perm) {
    __shared__ double bv[256];
    __shared__ int bi[256];
    const int64_t t = blockIdx.x;
    const int tid = threadIdx.x;
    const double* sir = pair + 2 * (int64_t)nsrc * nsrc * nwin;   // [jtrue][jest][nwin]
    int ncand = 1;
    for (int k = 2; k <= nsrc; ++k) ncand *= k;
    double best = 0.0;
    int besti = -1;
    for (int i = tid; i < ncand; i += blockDim.x) {
        int p[WUN_MAX_SOURCES];
        nth_permutation(i, nsrc, p);
        double s = sir[(int64_t)p[0] * nsrc * nwin + t];
        for (int j = 1; j < nsrc; ++j) s += sir[((int64_t)p[j] * nsrc + j) * nwin + t];
        const double mean = s / nsrc;
        if (argmax_before(mean, i, best, besti)) { best = mean; besti = i; }
    }
    bv[tid] = best;
    bi[tid] = besti;
    __syncthreads();
    for (int s = blockDim.x / 2; s > 0; s >>= 1) {
        if (tid < s && argmax_before(bv[tid + s], bi[tid + s], bv[tid], bi[tid])) { bv[tid] = bv[tid + s]; bi[tid] = bi[tid + s]; }
        __syncthreads();
    }
    if (tid < nsrc) {
        int p[WUN_MAX_SOURCES];
        nth_permutation(bi[0], nsrc, p);
        const int j = tid, jt = p[j];
        perm[j * nwin + t] = jt;
        const int64_t m = (int64_t)nsrc * nwin, mp = (int64_t)nsrc * nsrc * nwin;
        for (int k = 0; k < 4; ++k) metrics[k * m + j * nwin + t] = pair[k * mp + ((int64_t)jt * nsrc + j) * nwin + t];
    }
}

// ---- v3: the frames to solve ------------------------------------------------------------------------------------------------
// One CTA per frame: silent[t] = the silence rule of bss_frame_metrics_kernel, which later turns the frame into NaN.
__global__ void __launch_bounds__(256) bss_frame_silent_kernel(const float* __restrict__ ref, const float* __restrict__ est,
                                                               int nsrc, int nchan, int64_t N, int64_t win, int64_t hop,
                                                               int* __restrict__ silent) {
    const bool s = frame_silent(ref, est, nsrc, nchan, N, win, (int64_t)blockIdx.x * hop);
    if (threadIdx.x == 0) silent[blockIdx.x] = s;
}

// list[0] = the number of frames that are not silent, list[1..] those frames in order.  One thread: nwin is small.
__global__ void bss_frame_list_kernel(const int* __restrict__ silent, int64_t nwin, int* __restrict__ list) {
    int count = 0;
    for (int64_t t = 0; t < nwin; ++t)
        if (!silent[t]) list[1 + count++] = (int)t;
    list[0] = count;
}

// filters[t] = (C, Cj) of frame t: the pass's slots copied to their frames (blockIdx.x: slot), or NaN for the silent
// frames (silent != nullptr, blockIdx.x: frame), whose filters are never computed.
__global__ void bss_frame_filters_kernel(const double* __restrict__ C, const double* __restrict__ Cj, int64_t csz, int64_t cjsz,
                                         const int* __restrict__ silent, Pass pass, double* __restrict__ filters) {
    const int64_t i = (int64_t)blockIdx.y * blockDim.x + threadIdx.x, b = blockIdx.x;
    if (i >= csz + cjsz) return;
    if (silent) {
        if (silent[b]) filters[b * (csz + cjsz) + i] = __longlong_as_double(0x7ff8000000000000LL);
        return;
    }
    const int64_t t = pass_frame(pass, b);
    if (t >= 0) filters[t * (csz + cjsz) + i] = i < csz ? C[b * csz + i] : Cj[b * cjsz + i - csz];
}

// ---- host side --------------------------------------------------------------------------------------------------------------
constexpr int kFlags = WUN_BSS_FRAMEWISE_FILTERS | WUN_BSS_PERMUTATION | WUN_BSS_SOURCES;

struct Layout {
    int64_t nref, ntask, n, m, nseg, seg_len, nwin, ntile;
    int npair, ne;       // references scored per estimate (nsrc with WUN_BSS_PERMUTATION, else 1); energies per pair
    bool permute;
    int64_t slots, lags, G, Gjj, C, Cj, E, PM, total;   // byte offsets into the workspace (v4)
};

bool make_layout(int64_t nsrc, int64_t nchan, int64_t N, int64_t win, int64_t hop, int flags, Layout* o) {
    if (nsrc < 1 || nsrc > WUN_MAX_SOURCES || (nchan != 1 && nchan != 2) || N < 1 || win < 1 || hop < 1) return false;
    if (win > (int64_t)1 << 40 || hop > (int64_t)1 << 40 || N > (int64_t)1 << 40 || (flags & ~kFlags)) return false;
    Layout& L = *o;
    L.nref = nsrc * nchan;
    L.ntask = 2 * L.nref * L.nref;
    L.n = L.nref * kL;
    L.m = nchan * kL;
    const int64_t nchunks = (N + kXcChunk - 1) / kXcChunk, per_seg = (nchunks + kMaxSegs - 1) / kMaxSegs;
    L.nseg = (nchunks + per_seg - 1) / per_seg;
    L.seg_len = per_seg * kXcChunk;
    L.nwin = N >= win ? (N - win) / hop + 1 : 0;   // floor((N - win + hop) / hop), at least 0
    L.ntile = (win + kL - 1 + kFrTile - 1) / kFrTile;
    if (L.nwin * L.ntile >= ((int64_t)1 << 31)) return false;
    L.permute = flags & WUN_BSS_PERMUTATION;
    L.npair = L.permute ? (int)nsrc : 1;
    L.ne = flags & WUN_BSS_SOURCES ? 8 : 7;
    int64_t off = 0;
    auto take = [&](int64_t doubles) { const int64_t at = off; off += (doubles * 8 + 255) / 256 * 256; return at; };
    L.slots = take(L.nseg * L.ntask * kL);
    L.lags = take(L.ntask * kL);
    L.G = take(L.n * L.n);
    L.Gjj = take(nsrc * L.m * L.m);
    L.C = take(L.nref * L.n);
    L.Cj = take(L.nref * L.m * L.npair);
    L.E = take(L.nwin * nsrc * L.npair * L.ntile * L.ne);
    L.PM = take(L.permute ? 4 * nsrc * nsrc * L.nwin : 0);
    L.total = off;
    return true;
}

// Blocked LDL^T of `batch` matrices of order n, then solve for ncol right-hand-side columns each.  v4 (pass.list == nullptr)
// keeps its CUDA-core trailing update; v3's batches of frames take the tensor-core one.
cudaError_t ldl_solve(double* A, int n, int batch, double* B, int ncol, Pass pass, cudaStream_t st) {
    const int panel_smem = (kPanel * (kPanel + 1) + kPanel * 129) * 8;
    cudaError_t e = cudaFuncSetAttribute(bss_ldl_panel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, panel_smem);
    if (e == cudaSuccess)
        e = cudaFuncSetAttribute(bss_ldl_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, n * 8);
    if (e != cudaSuccess) return e;
    for (int k0 = 0; k0 < n; k0 += kPanel) {
        bss_ldl_diag_kernel<<<batch, 256, 0, st>>>(A, n, k0, pass);
        const int rest = n - k0 - kPanel;
        if (rest > 0) {
            bss_ldl_panel_kernel<<<dim3((rest + 127) / 128, batch), 128, panel_smem, st>>>(A, n, k0, pass);
            const int nt = rest / kPanel;
            if (pass.list)
                bss_ldl_update_dmma_kernel<<<dim3(nt, nt, batch), 256, 0, st>>>(A, n, k0, pass);
            else
                bss_ldl_update_kernel<<<dim3(nt, nt, batch), 256, 0, st>>>(A, n, k0);
        }
    }
    bss_ldl_solve_kernel<<<dim3(ncol, batch), 256, n * 8, st>>>(A, n, B, pass);
    return cudaGetLastError();
}

void launch_energies(bool framewise, dim3 grid, cudaStream_t st, const float* ref, const float* est, const double* C,
                     const double* Cj, int ns, int nc, int64_t N, int64_t win, int64_t hop, const Layout& S, double* E,
                     Pass pass) {
    const int ntile = (int)S.ntile;
    if (nc == 1 && !framewise)
        bss_frame_energy_kernel<1, false><<<grid, kFrThreads, 0, st>>>(ref, est, C, Cj, ns, N, win, hop, ntile, S.npair, S.ne, E, pass);
    else if (nc == 1)
        bss_frame_energy_kernel<1, true><<<grid, kFrThreads, 0, st>>>(ref, est, C, Cj, ns, N, win, hop, ntile, S.npair, S.ne, E, pass);
    else if (!framewise)
        bss_frame_energy_kernel<2, false><<<grid, kFrThreads, 0, st>>>(ref, est, C, Cj, ns, N, win, hop, ntile, S.npair, S.ne, E, pass);
    else
        bss_frame_energy_kernel<2, true><<<grid, kFrThreads, 0, st>>>(ref, est, C, Cj, ns, N, win, hop, ntile, S.npair, S.ne, E, pass);
}

// v4: the filters once over the whole track, then the energies of every frame.
cudaError_t energies_v4(const float* ref, const float* est, int ns, int nc, int64_t N, int64_t win, int64_t hop,
                        const Layout& L, char* ws, double* filters, cudaStream_t st) {
    double *slots = (double*)(ws + L.slots), *lags = (double*)(ws + L.lags), *G = (double*)(ws + L.G),
           *Gjj = (double*)(ws + L.Gjj), *C = (double*)(ws + L.C), *Cj = (double*)(ws + L.Cj), *E = (double*)(ws + L.E);
    const int nref = (int)L.nref;
    const Pass whole{nullptr, 0, 1};
    bss_xcorr_kernel<<<dim3((unsigned)L.nseg, (unsigned)L.ntask), kXcThreads, 0, st>>>(ref, est, ns, nc, N, L.seg_len, slots,
                                                                                        whole, win, hop);
    const int64_t nvals = L.ntask * kL;
    bss_lag_reduce_kernel<<<(unsigned)((nvals + 255) / 256), 256, 0, st>>>(slots, L.nseg, nvals, lags, whole);
    bss_assemble_gram_kernel<<<dim3((unsigned)(L.n + 255) / 256, (unsigned)L.n, 1 + ns), 256, 0, st>>>(lags, ns, nc, G, Gjj,
                                                                                                       whole);
    bss_assemble_rhs_kernel<<<dim3((unsigned)(L.n + 255) / 256, nref), 256, 0, st>>>(lags, ns, nc, L.npair, C, Cj, whole);
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = ldl_solve(G, (int)L.n, 1, C, nref, whole, st);
    if (e == cudaSuccess) e = ldl_solve(Gjj, (int)L.m, ns, Cj, nc * L.npair, whole, st);
    if (e == cudaSuccess && L.nwin > 0) {
        launch_energies(false, dim3((unsigned)(L.nwin * L.ntile), ns), st, ref, est, C, Cj, ns, nc, N, win, hop, L, E, whole);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess && filters) {
        e = cudaMemcpyAsync(filters, C, L.nref * L.n * 8, cudaMemcpyDeviceToDevice, st);
        if (e == cudaSuccess)
            e = cudaMemcpyAsync(filters + L.nref * L.n, Cj, L.nref * L.m * L.npair * 8, cudaMemcpyDeviceToDevice, st);
    }
    return e;
}

constexpr int kV3Segs = 16;            // sample segments of a frame's correlations (partial slots per lag)
constexpr int64_t kV3MaxPass = 2048;   // frames per pass at most: keeps the assembly grid's z = slots * (1 + nsrc) in range

// v3's workspace: the silence flags, the frame list, the energies and pair metrics of the whole call, then the per-frame
// arrays of one pass of P frames.  Every per-frame array is a multiple of 4 KiB, so the total is fixed + P * per_frame.
struct LayoutV3 {
    Layout s;                          // shapes as v4 (nref, ntask, n, m, nwin, ntile, npair, ne); its offsets are not used
    int64_t nseg, seg_len, P;
    int64_t silent, list, E, PM, slots, lags, G, Gjj, C, Cj;   // byte offsets into the workspace
    int64_t fixed, per_frame, total;
};

bool make_layout_v3(int64_t nsrc, int64_t nchan, int64_t N, int64_t win, int64_t hop, int flags, int64_t frames_per_pass,
                    LayoutV3* o) {
    if (frames_per_pass < 1 || !make_layout(nsrc, nchan, N, win, hop, flags, &o->s)) return false;
    const Layout& S = o->s;
    const int64_t nchunks = (win + kXcChunk - 1) / kXcChunk, per_seg = (nchunks + kV3Segs - 1) / kV3Segs;
    o->nseg = (nchunks + per_seg - 1) / per_seg;
    o->seg_len = per_seg * kXcChunk;
    o->P = std::min(std::min(frames_per_pass, S.nwin), kV3MaxPass);
    int64_t off = 0;
    auto take = [&](int64_t bytes) { const int64_t at = off; off += (bytes + 255) / 256 * 256; return at; };
    o->silent = take(S.nwin * 4);
    o->list = take((1 + S.nwin) * 4);
    o->E = take(S.nwin * nsrc * S.npair * S.ntile * S.ne * 8);
    o->PM = take(S.permute ? 4 * nsrc * nsrc * S.nwin * 8 : 0);
    o->fixed = off;
    const int64_t d_slots = o->nseg * S.ntask * kL, d_lags = S.ntask * kL, d_G = S.n * S.n, d_Gjj = nsrc * S.m * S.m,
                  d_C = S.nref * S.n, d_Cj = S.nref * S.m * S.npair;
    o->per_frame = 8 * (d_slots + d_lags + d_G + d_Gjj + d_C + d_Cj);
    o->slots = take(o->P * d_slots * 8);
    o->lags = take(o->P * d_lags * 8);
    o->G = take(o->P * d_G * 8);
    o->Gjj = take(o->P * d_Gjj * 8);
    o->C = take(o->P * d_C * 8);
    o->Cj = take(o->P * d_Cj * 8);
    o->total = off;
    return true;
}

// v3: the frames that are not silent, in passes of L.P; each pass solves its frames' filters and adds their energies.
cudaError_t energies_v3(const float* ref, const float* est, int ns, int nc, int64_t N, int64_t win, int64_t hop,
                        const LayoutV3& L, char* ws, double* filters, cudaStream_t st) {
    const Layout& S = L.s;
    int *silent = (int*)(ws + L.silent), *list = (int*)(ws + L.list);
    double *slots = (double*)(ws + L.slots), *lags = (double*)(ws + L.lags), *G = (double*)(ws + L.G),
           *Gjj = (double*)(ws + L.Gjj), *C = (double*)(ws + L.C), *Cj = (double*)(ws + L.Cj), *E = (double*)(ws + L.E);
    const int nref = (int)S.nref;
    const int64_t csz = S.nref * S.n, cjsz = S.nref * S.m * S.npair, nvals = S.ntask * kL;
    const unsigned fblocks = (unsigned)((csz + cjsz + 255) / 256);

    bss_frame_silent_kernel<<<(unsigned)S.nwin, 256, 0, st>>>(ref, est, ns, nc, N, win, hop, silent);
    bss_frame_list_kernel<<<1, 1, 0, st>>>(silent, S.nwin, list);
    if (filters)
        bss_frame_filters_kernel<<<dim3((unsigned)S.nwin, fblocks), 256, 0, st>>>(nullptr, nullptr, csz, cjsz, silent,
                                                                                  Pass{nullptr, 0, 1}, filters);
    cudaError_t e = cudaGetLastError();
    for (int64_t s0 = 0; s0 < S.nwin && e == cudaSuccess; s0 += L.P) {
        const unsigned np = (unsigned)std::min(L.P, S.nwin - s0);
        const Pass pass{list, s0, 1}, per_source{list, s0, ns};
        bss_xcorr_kernel<<<dim3((unsigned)L.nseg, (unsigned)S.ntask, np), kXcThreads, 0, st>>>(ref, est, ns, nc, N, L.seg_len,
                                                                                               slots, pass, win, hop);
        bss_lag_reduce_kernel<<<dim3((unsigned)((nvals + 255) / 256), np), 256, 0, st>>>(slots, L.nseg, nvals, lags, pass);
        bss_assemble_gram_kernel<<<dim3((unsigned)(S.n + 255) / 256, (unsigned)S.n, np * (1 + ns)), 256, 0, st>>>(
            lags, ns, nc, G, Gjj, pass);
        bss_assemble_rhs_kernel<<<dim3((unsigned)(S.n + 255) / 256, nref, np), 256, 0, st>>>(lags, ns, nc, S.npair, C, Cj,
                                                                                             pass);
        e = cudaGetLastError();
        if (e == cudaSuccess) e = ldl_solve(G, (int)S.n, (int)np, C, nref, pass, st);
        if (e == cudaSuccess) e = ldl_solve(Gjj, (int)S.m, (int)np * ns, Cj, nc * S.npair, per_source, st);
        if (e != cudaSuccess) break;
        launch_energies(true, dim3((unsigned)(np * S.ntile), ns), st, ref, est, C, Cj, ns, nc, N, win, hop, S, E, pass);
        if (filters)
            bss_frame_filters_kernel<<<dim3(np, fblocks), 256, 0, st>>>(C, Cj, csz, cjsz, nullptr, pass, filters);
        e = cudaGetLastError();
    }
    return e;
}

}  // namespace

extern "C" int64_t wun_bss_eval_ex_workspace_bytes(int64_t nsrc, int64_t nchan, int64_t nsampl, int64_t win, int64_t hop,
                                                   int flags, int64_t frames_per_pass) {
    LayoutV3 L;
    if (flags & WUN_BSS_FRAMEWISE_FILTERS)
        return make_layout_v3(nsrc, nchan, nsampl, win, hop, flags, frames_per_pass, &L) ? L.total : WUN_E_INVALID;
    return make_layout(nsrc, nchan, nsampl, win, hop, flags, &L.s) ? L.s.total : WUN_E_INVALID;
}

extern "C" int wun_bss_eval_ex(const float* references, const float* estimates, int64_t nsrc, int64_t nchan, int64_t nsampl,
                               int64_t win, int64_t hop, int flags, double* metrics, int64_t* perm, double* pair_metrics,
                               double* filters, void* workspace, int64_t workspace_bytes, void* stream) {
    const bool framewise = flags & WUN_BSS_FRAMEWISE_FILTERS, permute = flags & WUN_BSS_PERMUTATION;
    LayoutV3 L;
    const Layout& S = L.s;
    if (framewise ? !make_layout_v3(nsrc, nchan, nsampl, win, hop, flags, 1, &L)
                  : !make_layout(nsrc, nchan, nsampl, win, hop, flags, &L.s))
        return WUN_E_INVALID;
    if (!references || !estimates || !workspace || (!metrics && S.nwin > 0)) return WUN_E_INVALID;
    if (permute ? (!perm && S.nwin > 0) : (perm || pair_metrics)) return WUN_E_INVALID;
    const int64_t need = framewise ? L.total : S.total;   // v3: one frame per pass at least
    if (workspace_bytes < need || reinterpret_cast<uintptr_t>(workspace) % 256 != 0) return WUN_E_INVALID;
    if (framewise && S.nwin > 1)
        make_layout_v3(nsrc, nchan, nsampl, win, hop, flags, (workspace_bytes - L.fixed) / L.per_frame, &L);
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        return WUN_E_NOGPU;
    }
    if (framewise && S.nwin == 0) return WUN_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    char* ws = static_cast<char*>(workspace);
    const int ns = (int)nsrc, nc = (int)nchan;
    cudaError_t e = framewise ? energies_v3(references, estimates, ns, nc, nsampl, win, hop, L, ws, filters, st)
                              : energies_v4(references, estimates, ns, nc, nsampl, win, hop, S, ws, filters, st);
    if (e == cudaSuccess && S.nwin > 0) {
        const double* E = (const double*)(ws + (framewise ? L.E : S.E));
        double* pm = !permute ? metrics : pair_metrics ? pair_metrics : (double*)(ws + (framewise ? L.PM : S.PM));
        bss_frame_metrics_kernel<<<(unsigned)S.nwin, 256, 0, st>>>(references, estimates, ns, nc, nsampl, win, hop, S.nwin,
                                                                   (int)S.ntile, S.npair, flags & WUN_BSS_SOURCES, E, pm);
        if (permute) bss_perm_select_kernel<<<(unsigned)S.nwin, 256, 0, st>>>(pm, ns, S.nwin, metrics, perm);
        e = cudaGetLastError();
    }
    return e == cudaSuccess ? WUN_OK : WUN_E_CUDA;
}

extern "C" int64_t wun_bss_eval_workspace_bytes(int64_t nsrc, int64_t nchan, int64_t nsampl, int64_t win, int64_t hop) {
    return wun_bss_eval_ex_workspace_bytes(nsrc, nchan, nsampl, win, hop, 0, 1);
}

extern "C" int wun_bss_eval(const float* references, const float* estimates, int64_t nsrc, int64_t nchan, int64_t nsampl,
                            int64_t win, int64_t hop, double* metrics, double* filters, void* workspace,
                            int64_t workspace_bytes, void* stream) {
    return wun_bss_eval_ex(references, estimates, nsrc, nchan, nsampl, win, hop, 0, metrics, nullptr, nullptr, filters,
                           workspace, workspace_bytes, stream);
}

extern "C" int64_t wun_bss_eval_v3_workspace_bytes(int64_t nsrc, int64_t nchan, int64_t nsampl, int64_t win, int64_t hop,
                                                   int64_t frames_per_pass) {
    return wun_bss_eval_ex_workspace_bytes(nsrc, nchan, nsampl, win, hop, WUN_BSS_FRAMEWISE_FILTERS, frames_per_pass);
}

extern "C" int wun_bss_eval_v3(const float* references, const float* estimates, int64_t nsrc, int64_t nchan, int64_t nsampl,
                               int64_t win, int64_t hop, double* metrics, double* filters, void* workspace,
                               int64_t workspace_bytes, void* stream) {
    return wun_bss_eval_ex(references, estimates, nsrc, nchan, nsampl, win, hop, WUN_BSS_FRAMEWISE_FILTERS, metrics, nullptr,
                           nullptr, filters, workspace, workspace_bytes, stream);
}
