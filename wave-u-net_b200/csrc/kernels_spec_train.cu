// kernels_spec_train.cu - the training step of the spectrogram U-Net baselines (the reference's
// Models/UnetSpectrogramSeparator.py get_output with training=True, and the loss / gradients of Training.py:47-77),
// FP32 on CUDA cores like the inference kernels of kernels_spec.cu.
//
//   spec_train_conv_kernel     one 5x5 stride-2 gather over NHWC tensors at a channel pitch, in either geometry: a stride-2
//                              conv (output o reads input 2o + k - 1) or a transposed conv (output o gathers input (o + 1 - k) / 2).
//                              Serves the forward of the down / up / mask layers (+ bias, pre-BN output) and both input
//                              gradients: the down conv's dgrad is a transposed-conv gather, the transposed conv's a stride-2 conv.
//                              Optional dropout masks on the input (forward) or on the output (dgrad), and accumulation into
//                              the output (the skip gradient's second part)
//   spec_chan_sum_kernel       per-channel fp64 sums over the rows of an [N][C] tensor, per CTA into partials:
//                              (z, z^2) for the batch statistics, (dy, dy * xhat) for the batch-norm backward, dz for a bias
//   spec_chan_local_kernel     the partials summed in a fixed order per channel: a conv bias gradient, or the call's own sums
//   spec_chan_finish_kernel    the ranks' gathered sums added in rank order, then: batch mean / rstd and the moving-average
//                              update, or beta's gradient and the backward's two means
//   spec_bn_apply_kernel       (z - mean) * rstd + beta, LeakyReLU(0.2) / ReLU, into the concatenation buffer
//   spec_bn_backward_kernel    dz = rstd * (dy - mean(dy) - xhat * mean(dy * xhat)), dy = g * activation slope; in place over z
//   spec_dropout_kernel        keep masks of tf.layers.dropout(rate 0.5) from a counter-based hash (spec_dropout_keep) of
//                              the element's index in the whole batch
//   spec_mask_apply_kernel     sigmoid of the mask conv, kept for the backward, times X (complex) or |X|, bin 512 = 0.5
//   spec_mask_backward_kernel  d loss / d mask-logit: U7 through the adjoint of the inverse STFT (a windowed forward real DFT of
//                              the frame-gathered audio gradient), U7a through the L1 magnitude loss; then sigmoid'
//   spec_wgrad_kernel          weight gradient of either conv kind, split over positions into per-CTA partials
//   spec_wgrad_finish_kernel   the partials summed in a fixed order
//
// No float atomics: every sum has an order fixed by the shapes alone, so two runs give the same bits.  DESIGN.md §4.9.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "kernels.h"

namespace wun {

namespace {

constexpr int kN = 1024;
constexpr int kHop = 768;
constexpr int kBins = kN / 2 + 1;
constexpr int kFftThreads = 256;
constexpr int kRedRows = 8;                     // rows per CTA step of spec_chan_sum_kernel (32 channels x 8 rows)
constexpr float kDecayComplement = (float)(1.0 - 0.999);   // TF converts 1 - decay in double, then to float32

unsigned blocks_for(long long threads, int per_block) { return (unsigned)((threads + per_block - 1) / per_block); }

template <bool UP, int P>
__global__ void __launch_bounds__(128) spec_train_conv_kernel(const SpecTrainConv A) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int co = (int)(t % A.Co);
    const long long tile = t / A.Co;
    const int groups = (A.Wo + P - 1) / P;
    const int g = (int)(tile % groups);
    const long long r = tile / groups;
    const int ho = (int)(r % A.Ho);
    const int b = (int)(r / A.Ho);
    if (b >= A.batch) return;
    const int wo0 = g * P;
    float acc[P];
#pragma unroll
    for (int p = 0; p < P; ++p) acc[p] = 0.f;
    for (int kh = 0; kh < 5; ++kh) {
        int hi;
        if (UP) {
            const int a = ho + 1 - kh;
            if (a < 0 || (a & 1)) continue;
            hi = a >> 1;
        } else {
            hi = 2 * ho + kh - 1;
        }
        if (hi < 0 || hi >= A.Hi) continue;
        const long long row = ((long long)b * A.Hi + hi) * A.Wi;
        for (int kw = 0; kw < 5; ++kw) {
            long long xo[P];
            bool any = false;
#pragma unroll
            for (int p = 0; p < P; ++p) {
                int wi;
                bool ok = wo0 + p < A.Wo;
                if (UP) {
                    const int e = wo0 + p + 1 - kw;
                    ok = ok && e >= 0 && !(e & 1);
                    wi = e >> 1;
                } else {
                    wi = 2 * (wo0 + p) + kw - 1;
                }
                ok = ok && wi >= 0 && wi < A.Wi;
                xo[p] = ok ? (row + wi) * A.x_pitch : -1;
                any |= ok;
            }
            if (!any) continue;
            const float* wp = A.W + (long long)(kh * 5 + kw) * A.w_tap + (long long)co * A.w_co;
            for (int ci = 0; ci < A.Ci; ++ci) {
                const float w = __ldg(wp + (long long)ci * A.w_ci);
#pragma unroll
                for (int p = 0; p < P; ++p) {
                    if (xo[p] < 0) continue;
                    float v = __ldg(A.x + xo[p] + ci);
                    if (A.x_drop) v = A.x_drop[xo[p] + ci] ? 2.f * v : 0.f;
                    acc[p] = fmaf(v, w, acc[p]);
                }
            }
        }
    }
    const float bias = A.bias ? __ldg(A.bias + co) : 0.f;
#pragma unroll
    for (int p = 0; p < P; ++p) {
        if (wo0 + p >= A.Wo) break;
        const long long o = (((long long)b * A.Ho + ho) * A.Wo + wo0 + p) * A.y_pitch + A.y_off + co;
        float v = A.bias ? acc[p] + bias : acc[p];
        if (A.y_drop) v = A.y_drop[o] ? 2.f * v : 0.f;
        A.y[o] = A.accumulate ? A.y[o] + v : v;
    }
}

// Block (32 channels, 8 rows); CTA (blockIdx.x, blockIdx.y) reduces channels [32 x, 32 x + 32) over the rows
// r = blockIdx.y * 8 + ty + k * 8 * gridDim.y, then its 8 row lanes in order, into part[blockIdx.y][c].
__global__ void __launch_bounds__(256) spec_chan_sum_kernel(const SpecChanSum S) {
    __shared__ double s1[kRedRows][32], s2[kRedRows][32];
    const int c = blockIdx.x * 32 + threadIdx.x;
    double a1 = 0.0, a2 = 0.0;
    if (c < S.C) {
        const float2 st = S.mode == 1 ? S.stat[c] : make_float2(0.f, 0.f);
        for (long long r = (long long)blockIdx.y * kRedRows + threadIdx.y; r < S.N; r += (long long)gridDim.y * kRedRows) {
            const float z = S.z[r * S.C + c];
            if (S.mode == 0) {
                a1 += (double)z;
                a2 += (double)z * (double)z;
            } else if (S.mode == 1) {
                const float act = S.a[r * S.pitch + c];
                const float dy = S.g[r * S.pitch + c] * (act > 0.f ? 1.f : S.neg_slope);
                const float xhat = (z - st.x) * st.y;
                a1 += (double)dy;
                a2 += (double)dy * (double)xhat;
            } else {
                a1 += (double)z;
            }
        }
    }
    s1[threadIdx.y][threadIdx.x] = a1;
    s2[threadIdx.y][threadIdx.x] = a2;
    __syncthreads();
    if (threadIdx.y == 0 && c < S.C) {
        double t1 = 0.0, t2 = 0.0;
        for (int k = 0; k < kRedRows; ++k) {
            t1 += s1[k][threadIdx.x];
            t2 += s2[k][threadIdx.x];
        }
        S.part[(long long)blockIdx.y * S.C + c] = make_double2(t1, t2);
    }
}

// The partials summed in a fixed order per channel: a conv bias gradient (mode 2), or this call's (sum 1, sum 2) into local[c].
__global__ void spec_chan_local_kernel(const SpecChanSum S, int P) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= S.C) return;
    double t1 = 0.0, t2 = 0.0;
    for (int p = 0; p < P; ++p) {
        const double2 v = S.part[(long long)p * S.C + c];
        t1 += v.x;
        t2 += v.y;
    }
    if (S.mode == 2) S.out[c] = (float)t1;
    else S.local[c] = make_double2(t1, t2);
}

// The ranks' sums gathered[r][c] added in rank order from 0.0 over n = S.n rows (the whole batch's); one rank gives the
// single-device arithmetic bit for bit, as 0.0 + t = t.
__global__ void spec_chan_finish_kernel(const SpecChanSum S, int world) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= S.C) return;
    double t1 = 0.0, t2 = 0.0;
    for (int r = 0; r < world; ++r) {
        const double2 v = S.gathered[(long long)r * S.C + c];
        t1 += v.x;
        t2 += v.y;
    }
    const double n = S.n;
    if (S.mode == 0) {
        const double mean = t1 / n;
        const double var = fmax(t2 / n - mean * mean, 0.0);                     // biased: normalises the batch
        S.stat[c] = make_float2((float)mean, (float)(1.0 / sqrt(var + 1e-3)));
        // UPDATE_OPS: moving -= (moving - batch value) * (1 - decay); the variance Bessel-corrected
        const float bm = (float)mean, bv = (float)(var * n / fmax(n - 1.0, 1.0));
        S.moving_mean[c] = __fsub_rn(S.moving_mean[c], __fmul_rn(__fsub_rn(S.moving_mean[c], bm), kDecayComplement));
        S.moving_var[c] = __fsub_rn(S.moving_var[c], __fmul_rn(__fsub_rn(S.moving_var[c], bv), kDecayComplement));
    } else {
        // d beta = this call's own sum dy: the gradient all-reduce after a data-parallel step adds the ranks'
        S.out[c] = (float)S.local[c].x;
        S.coef[c] = make_float2((float)(t1 / n), (float)(t2 / n));
    }
}

__global__ void __launch_bounds__(256) spec_bn_apply_kernel(const float* __restrict__ z, long long N, int C,
                                                            const float2* __restrict__ stat, const float* __restrict__ beta,
                                                            float neg_slope, float* __restrict__ y, int y_pitch) {
    const long long total = N * C;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const float2 st = stat[c];
        const float v = (z[i] - st.x) * st.y + __ldg(beta + c);
        y[(i / C) * y_pitch + c] = fmaxf(neg_slope * v, v);                     // LeakyReLU(0.2) or ReLU (slope 0)
    }
}

__global__ void __launch_bounds__(256) spec_bn_backward_kernel(float* __restrict__ z, long long N, int C,
                                                               const float* __restrict__ g, const float* __restrict__ a,
                                                               int pitch, float neg_slope, const float2* __restrict__ stat,
                                                               const float2* __restrict__ coef) {
    const long long total = N * C;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int c = (int)(i % C);
        const long long o = (i / C) * pitch + c;
        const float dy = g[o] * (a[o] > 0.f ? 1.f : neg_slope);
        const float2 st = stat[c], k = coef[c];
        const float xhat = (z[i] - st.x) * st.y;
        z[i] = st.y * (dy - k.x - xhat * k.y);
    }
}

__global__ void __launch_bounds__(256) spec_dropout_kernel(uint8_t* __restrict__ keep, long long n, long long first,
                                                           unsigned long long seed, const long long* __restrict__ step_state,
                                                           int source, int level) {
    const uint64_t step = (uint64_t)step_state[0];
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        keep[i] = (uint8_t)spec_dropout_keep(seed, step, source, level, (uint64_t)(first + i));
}

// One thread per (example, frame, bin < 512); the thread of bin 0 also writes bin 512 with the constant mask 0.5.
__global__ void __launch_bounds__(128) spec_mask_apply_kernel(float* __restrict__ mask, long long frames,
                                                              const float* __restrict__ X, float* __restrict__ out,
                                                              int magnitude) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= frames * (kBins - 1)) return;
    const long long fr = t / (kBins - 1);
    const int k = (int)(t % (kBins - 1));
    const float m = 1.f / (1.f + expf(-mask[t]));
    mask[t] = m;
    const long long bin = fr * kBins + k;
    const float2* Xc = reinterpret_cast<const float2*>(X);
    const float2 x = Xc[bin];
    if (magnitude) {
        out[bin] = m * hypotf(x.x, x.y);
        if (k == 0) {
            const float2 xl = Xc[bin + kBins - 1];
            out[bin + kBins - 1] = 0.5f * hypotf(xl.x, xl.y);
        }
    } else {
        float2* Y = reinterpret_cast<float2*>(out);
        Y[bin] = make_float2(m * x.x, m * x.y);
        if (k == 0) {
            const float2 xl = Xc[bin + kBins - 1];
            Y[bin + kBins - 1] = make_float2(0.5f * xl.x, 0.5f * xl.y);
        }
    }
}

// One CTA per (frame, example).  U7: the audio gradient 2 (audio - target) * scale of the frame's 1024 samples (the
// overlap-add's adjoint gathers every frame sample from its output sample) times the inverse window, then per bin k < 512
// G_k = c_k / 1024 * sum_j g_j e^{-2 pi i k j / 1024} with c_0 = 1, c_k = 2 otherwise (the irfft weights; bin 512 has the
// constant mask), and d mask = Re(conj(G) X).  U7a: d mask = sign(mask |X| - target |X|) |X| * scale, sign(0) = 0.
__global__ void __launch_bounds__(kFftThreads) spec_mask_backward_kernel(const SpecMaskBwd M) {
    __shared__ float c[kN], s[kN], g[kN];
    const int f = blockIdx.x, b = blockIdx.y;
    const long long fr = (long long)b * M.n_frames + f;
    const float2* Xc = reinterpret_cast<const float2*>(M.X) + fr * kBins;
    const float* mask = M.mask + fr * (kBins - 1);
    float* dlogit = M.dlogit + fr * (kBins - 1);
    if (M.raw_audio) {
        for (int m = threadIdx.x; m < kN; m += blockDim.x) {
            float sv, cv;
            sincospif((float)m / 512.f, &sv, &cv);
            c[m] = cv;
            s[m] = sv;
        }
        __syncthreads();
        const long long t0 = (long long)b * M.T + (long long)f * kHop;
        for (int j = threadIdx.x; j < kN; j += blockDim.x) {
            const int q = j % kHop;
            const float h0 = 0.5f - 0.5f * c[q], h1 = q + kHop < kN ? 0.5f - 0.5f * c[q + kHop] : 0.f;
            const float w = (0.5f - 0.5f * c[j]) / (h0 * h0 + h1 * h1);
            g[j] = 2.f * (M.audio[t0 + j] - M.target[t0 + j]) * M.scale * w;
        }
        __syncthreads();
    }
    for (int k = threadIdx.x; k < kBins - 1; k += blockDim.x) {
        const float2 x = Xc[k];
        float dm;
        if (M.raw_audio) {
            float re = 0.f, im = 0.f;
            for (int j = 0; j < kN; ++j) {
                const int m = (k * j) & (kN - 1);
                re = fmaf(g[j], c[m], re);
                im = fmaf(-g[j], s[m], im);
            }
            const float ck = (k == 0 ? 1.f : 2.f) / kN;
            dm = ck * re * x.x + ck * im * x.y;
        } else {
            const float mag = hypotf(x.x, x.y);
            const float d = mask[k] * mag - M.tmag[fr * kBins + k];
            dm = (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f)) * mag * M.scale;
        }
        const float m = mask[k];
        dlogit[k] = dm * m * (1.f - m);
    }
}

// Thread: one weight (tap, c_hi, c_lo), c_lo fastest, summed over the positions of split blockIdx.y in order.
__global__ void __launch_bounds__(128) spec_wgrad_kernel(const SpecWgrad G, int P) {
    const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long n_out = 25LL * G.Chi * G.Clo;
    if (o >= n_out) return;
    const int c_lo = (int)(o % G.Clo);
    const int c_hi = (int)((o / G.Clo) % G.Chi);
    const int tap = (int)(o / ((long long)G.Clo * G.Chi));
    const int kh = tap / 5, kw = tap % 5;
    const long long positions = (long long)G.batch * G.Hl * G.Wl;
    const long long per = (positions + P - 1) / P;
    const long long p0 = (long long)blockIdx.y * per, p1 = min(positions, p0 + per);
    const int Hh = 2 * G.Hl, Wh = 2 * G.Wl;
    float acc = 0.f;
    for (long long p = p0; p < p1; ++p) {
        const int w = (int)(p % G.Wl);
        const long long q = p / G.Wl;
        const int h = (int)(q % G.Hl);
        const int b = (int)(q / G.Hl);
        const int hr = 2 * h + kh - 1, wc = 2 * w + kw - 1;
        if (hr < 0 || hr >= Hh || wc < 0 || wc >= Wh) continue;
        const long long lo_i = p * G.lo_pitch + c_lo;
        const long long hi_i = (((long long)b * Hh + hr) * Wh + wc) * G.hi_pitch + c_hi;
        float lo = __ldg(G.lo + lo_i);
        if (G.lo_drop) lo = G.lo_drop[lo_i] ? 2.f * lo : 0.f;
        acc = fmaf(lo, __ldg(G.hi + hi_i), acc);
    }
    const long long dst = tap * G.w_tap + (long long)c_lo * G.w_lo + (long long)c_hi * G.w_hi;
    if (P == 1) G.dW[dst] = acc;
    else G.part[(long long)blockIdx.y * n_out + o] = acc;
}

__global__ void __launch_bounds__(256) spec_wgrad_finish_kernel(const SpecWgrad G, int P) {
    const long long o = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long n_out = 25LL * G.Chi * G.Clo;
    if (o >= n_out) return;
    float acc = 0.f;
    for (int p = 0; p < P; ++p) acc += G.part[(long long)p * n_out + o];
    const int c_lo = (int)(o % G.Clo);
    const int c_hi = (int)((o / G.Clo) % G.Chi);
    const long long tap = o / ((long long)G.Clo * G.Chi);
    G.dW[tap * G.w_tap + (long long)c_lo * G.w_lo + (long long)c_hi * G.w_hi] = acc;
}

__global__ void spec_step_advance_kernel(long long* step_state) { step_state[0] += 1; }

unsigned grid_stride_blocks(long long n) {
    long long blocks = (n + 255) / 256;
    if (blocks > 132 * 16) blocks = 132 * 16;
    return (unsigned)(blocks < 1 ? 1 : blocks);
}

}  // namespace

// Same tiling rule as the inference kernels: four output columns per thread while that still fills the GPU.
void launch_spec_train_conv(const SpecTrainConv& A, int up, cudaStream_t stream) {
    const bool wide = (long long)A.batch * A.Ho * ((A.Wo + 3) / 4) * A.Co >= 132LL * 2 * 128;
    const long long threads = (long long)A.batch * A.Ho * (wide ? (A.Wo + 3) / 4 : A.Wo) * A.Co;
    const unsigned blocks = blocks_for(threads, 128);
    if (up) {
        if (wide) spec_train_conv_kernel<true, 4><<<blocks, 128, 0, stream>>>(A);
        else spec_train_conv_kernel<true, 1><<<blocks, 128, 0, stream>>>(A);
    } else {
        if (wide) spec_train_conv_kernel<false, 4><<<blocks, 128, 0, stream>>>(A);
        else spec_train_conv_kernel<false, 1><<<blocks, 128, 0, stream>>>(A);
    }
}

int spec_chan_partials(long long N) {
    const long long p = (N + 32 * kRedRows - 1) / (32 * kRedRows);
    return (int)(p < 1 ? 1 : (p > 256 ? 256 : p));
}

void launch_spec_chan_sum(const SpecChanSum& S, cudaStream_t stream) {
    const int P = spec_chan_partials(S.N);
    spec_chan_sum_kernel<<<dim3((unsigned)((S.C + 31) / 32), (unsigned)P), dim3(32, kRedRows), 0, stream>>>(S);
    spec_chan_local_kernel<<<blocks_for(S.C, 128), 128, 0, stream>>>(S, P);
}

void launch_spec_chan_finish(const SpecChanSum& S, int world, cudaStream_t stream) {
    spec_chan_finish_kernel<<<blocks_for(S.C, 128), 128, 0, stream>>>(S, world);
}

void launch_spec_bn_apply(const float* z, long long N, int C, const float2* stat, const float* beta, float neg_slope,
                          float* y, int y_pitch, cudaStream_t stream) {
    spec_bn_apply_kernel<<<grid_stride_blocks(N * C), 256, 0, stream>>>(z, N, C, stat, beta, neg_slope, y, y_pitch);
}

void launch_spec_bn_backward(float* z, long long N, int C, const float* g, const float* a, int pitch, float neg_slope,
                             const float2* stat, const float2* coef, cudaStream_t stream) {
    spec_bn_backward_kernel<<<grid_stride_blocks(N * C), 256, 0, stream>>>(z, N, C, g, a, pitch, neg_slope, stat, coef);
}

void launch_spec_dropout(uint8_t* keep, long long n, long long first, unsigned long long seed, const long long* step_state,
                         int source, int level, cudaStream_t stream) {
    spec_dropout_kernel<<<grid_stride_blocks(n), 256, 0, stream>>>(keep, n, first, seed, step_state, source, level);
}

void launch_spec_mask_apply(float* mask, long long frames, const float* X, float* out, int magnitude, cudaStream_t stream) {
    spec_mask_apply_kernel<<<blocks_for(frames * (kBins - 1), 128), 128, 0, stream>>>(mask, frames, X, out, magnitude);
}

void launch_spec_mask_backward(const SpecMaskBwd& M, int batch, cudaStream_t stream) {
    spec_mask_backward_kernel<<<dim3((unsigned)M.n_frames, (unsigned)batch), kFftThreads, 0, stream>>>(M);
}

int spec_wgrad_partials(const SpecWgrad& G) {
    const long long n_out = 25LL * G.Chi * G.Clo;
    const long long positions = (long long)G.batch * G.Hl * G.Wl;
    long long p = (132LL * 1024 + n_out - 1) / n_out;                           // about one wave of 1024 threads per SM
    const long long cap = (positions + 31) / 32;                                 // at least 32 positions per split
    if (p > cap) p = cap;
    return (int)(p < 1 ? 1 : p);
}

void launch_spec_wgrad(const SpecWgrad& G, cudaStream_t stream) {
    const int P = spec_wgrad_partials(G);
    const long long n_out = 25LL * G.Chi * G.Clo;
    spec_wgrad_kernel<<<dim3(blocks_for(n_out, 128), (unsigned)P), 128, 0, stream>>>(G, P);
    if (P > 1) spec_wgrad_finish_kernel<<<blocks_for(n_out, 256), 256, 0, stream>>>(G, P);
}

void launch_spec_step_advance(long long* step_state, cudaStream_t stream) {
    spec_step_advance_kernel<<<1, 1, 0, stream>>>(step_state);
}

}  // namespace wun
