// kernels_spec.cu - the inference graph of the spectrogram U-Net baselines (the reference's
// Models/UnetSpectrogramSeparator.py, get_output with training=False), FP32 on CUDA cores.
//
//   spec_stft_kernel      tf.contrib.signal.stft(frame 1024, hop 768, fft 1024, periodic Hann), one CTA per frame: a direct
//                         DFT of the 513 bins with the twiddles in shared memory.  Writes the complex spectrum, log1p(|X|)
//                         without the last bin (the network input, NHWC [B][n][512][1]) and / or |X| (the L1 loss targets)
//   spec_down_kernel      conv2d 5x5 stride 2 'same' (1 before, 2 after) + bias + inference batch norm + LeakyReLU(0.2)
//   spec_up_kernel        conv2d_transpose 5x5 stride 2 'same' + bias + inference batch norm + ReLU, written straight into
//                         its half of the concatenation buffer
//   spec_mask_kernel      conv2d_transpose to one channel + sigmoid, the constant 0.5 for bin 512, and the product with the
//                         mixture: mask * X (complex, for the audio output) or mask * |X| (the magnitude output)
//   spec_istft_kernel     irfft(1024) of one frame times inverse_stft_window_fn(768, hann)
//   spec_ola_kernel       overlap-add with hop 768: every output sample gathers from its <= 2 frames in a fixed order
//
// Every output element is summed by one thread in an order fixed by the shapes alone (tap row, tap column, input channel),
// so a window's estimate has the same bits whatever batch it is placed in.  DESIGN.md §4.8.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "kernels.h"

namespace wun {

namespace {

constexpr int kN = 1024;          // frame length = fft length
constexpr int kHop = 768;
constexpr int kBins = kN / 2 + 1;
constexpr int kThreads = 256;

// cos / sin of 2*pi*m/1024 for m < 1024
__device__ __forceinline__ void load_twiddles(float* c, float* s) {
    for (int m = threadIdx.x; m < kN; m += blockDim.x) {
        float sv, cv;
        sincospif((float)m / 512.f, &sv, &cv);
        c[m] = cv;
        s[m] = sv;
    }
}

// periodic Hann window, 0.5 - 0.5 * cos(2*pi*j/1024) (window_ops.hann_window(periodic=True))
__device__ __forceinline__ float hann(const float* c, int j) { return 0.5f - 0.5f * c[j & (kN - 1)]; }

__global__ void __launch_bounds__(kThreads) spec_stft_kernel(const SpecStft P) {
    __shared__ float x[kN], c[kN], s[kN];
    const int f = blockIdx.x, sig = blockIdx.y;
    load_twiddles(c, s);
    __syncthreads();
    const float* src = P.signal + (long long)sig * P.T + (long long)f * kHop;
    for (int j = threadIdx.x; j < kN; j += blockDim.x) x[j] = __ldg(src + j) * hann(c, j);
    __syncthreads();
    const long long fr = (long long)sig * P.n_frames + f;
    for (int k = threadIdx.x; k < kBins; k += blockDim.x) {
        float re = 0.f, im = 0.f;
        for (int j = 0; j < kN; ++j) {
            const int m = (k * j) & (kN - 1);
            re = fmaf(x[j], c[m], re);
            im = fmaf(-x[j], s[m], im);
        }
        const float mag = hypotf(re, im);
        if (P.spec) reinterpret_cast<float2*>(P.spec)[fr * kBins + k] = make_float2(re, im);
        if (P.logmag && k < kBins - 1) P.logmag[fr * (kBins - 1) + k] = log1pf(mag);
        if (P.mag) P.mag[fr * kBins + k] = mag;
    }
}

__device__ __forceinline__ float batch_norm(float v, const SpecConv& A, int co) {
    return (v - __ldg(A.mean + co)) * rsqrtf(__ldg(A.var + co) + 1e-3f) + __ldg(A.beta + co);
}

// One thread: output channel co at P consecutive output columns of one output row.
template <int P>
__global__ void __launch_bounds__(128) spec_down_kernel(const SpecConv A) {
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
        const int hi = 2 * ho + kh - 1;
        if (hi < 0 || hi >= A.Hi) continue;
        const float* xrow = A.x + ((long long)b * A.Hi + hi) * A.Wi * A.x_pitch;
        for (int kw = 0; kw < 5; ++kw) {
            const float* xp[P];
#pragma unroll
            for (int p = 0; p < P; ++p) {
                const int wi = 2 * (wo0 + p) + kw - 1;
                xp[p] = (wo0 + p < A.Wo && wi >= 0 && wi < A.Wi) ? xrow + (long long)wi * A.x_pitch : nullptr;
            }
            const float* wp = A.W + (long long)(kh * 5 + kw) * A.Ci * A.Co + co;      // [5][5][Ci][Co]
            for (int ci = 0; ci < A.Ci; ++ci) {
                const float w = __ldg(wp + (long long)ci * A.Co);
#pragma unroll
                for (int p = 0; p < P; ++p)
                    if (xp[p]) acc[p] = fmaf(__ldg(xp[p] + ci), w, acc[p]);
            }
        }
    }
    const float bias = __ldg(A.bias + co);
#pragma unroll
    for (int p = 0; p < P; ++p) {
        if (wo0 + p >= A.Wo) break;
        const float v = batch_norm(acc[p] + bias, A, co);
        A.y[(((long long)b * A.Ho + ho) * A.Wo + wo0 + p) * A.y_pitch + A.y_off + co] = fmaxf(0.2f * v, v);
    }
}

// Transposed conv: input row i, tap k feed output row o = 2i + k - 1; outputs at or beyond 2N are dropped.
template <int P>
__global__ void __launch_bounds__(128) spec_up_kernel(const SpecConv A) {
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
        const int a = ho + 1 - kh;
        if (a < 0 || (a & 1) || (a >> 1) >= A.Hi) continue;
        const float* xrow = A.x + ((long long)b * A.Hi + (a >> 1)) * A.Wi * A.x_pitch;
        for (int kw = 0; kw < 5; ++kw) {
            const float* xp[P];
            bool any = false;
#pragma unroll
            for (int p = 0; p < P; ++p) {
                const int e = wo0 + p + 1 - kw;
                const bool ok = wo0 + p < A.Wo && e >= 0 && !(e & 1) && (e >> 1) < A.Wi;
                xp[p] = ok ? xrow + (long long)(e >> 1) * A.x_pitch : nullptr;
                any |= ok;
            }
            if (!any) continue;
            const float* wp = A.W + ((long long)(kh * 5 + kw) * A.Co + co) * A.Ci;      // [5][5][Co][Ci]
            for (int ci = 0; ci < A.Ci; ++ci) {
                const float w = __ldg(wp + ci);
#pragma unroll
                for (int p = 0; p < P; ++p)
                    if (xp[p]) acc[p] = fmaf(__ldg(xp[p] + ci), w, acc[p]);
            }
        }
    }
    const float bias = __ldg(A.bias + co);
#pragma unroll
    for (int p = 0; p < P; ++p) {
        if (wo0 + p >= A.Wo) break;
        const float v = batch_norm(acc[p] + bias, A, co);
        A.y[(((long long)b * A.Ho + ho) * A.Wo + wo0 + p) * A.y_pitch + A.y_off + co] = fmaxf(v, 0.f);
    }
}

// One thread per (example, frame, bin < 512); the thread of bin 0 also writes bin 512 with the constant mask 0.5.
__global__ void __launch_bounds__(128) spec_mask_kernel(const SpecConv A, const float* __restrict__ X, float* __restrict__ out,
                                                        int magnitude) {
    const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const int wo = (int)(t % A.Wo);
    const long long r = t / A.Wo;
    const int ho = (int)(r % A.Ho);
    const int b = (int)(r / A.Ho);
    if (b >= A.batch) return;
    float acc = 0.f;
    for (int kh = 0; kh < 5; ++kh) {
        const int a = ho + 1 - kh;
        if (a < 0 || (a & 1) || (a >> 1) >= A.Hi) continue;
        const float* xrow = A.x + ((long long)b * A.Hi + (a >> 1)) * A.Wi * A.x_pitch;
        for (int kw = 0; kw < 5; ++kw) {
            const int e = wo + 1 - kw;
            if (e < 0 || (e & 1) || (e >> 1) >= A.Wi) continue;
            const float* xp = xrow + (long long)(e >> 1) * A.x_pitch;
            const float* wp = A.W + (long long)(kh * 5 + kw) * A.Ci;                     // [5][5][1][Ci]
            for (int ci = 0; ci < A.Ci; ++ci) acc = fmaf(__ldg(xp + ci), __ldg(wp + ci), acc);
        }
    }
    const float mask = 1.f / (1.f + expf(-(acc + __ldg(A.bias))));
    const long long bin = ((long long)b * A.Ho + ho) * kBins + wo;
    const float2* Xc = reinterpret_cast<const float2*>(X);
    const float2 x = Xc[bin];
    if (magnitude) {
        out[bin] = mask * hypotf(x.x, x.y);
        if (wo == 0) {
            const float2 xl = Xc[bin + kBins - 1];
            out[bin + kBins - 1] = 0.5f * hypotf(xl.x, xl.y);
        }
    } else {
        float2* Y = reinterpret_cast<float2*>(out);
        Y[bin] = make_float2(mask * x.x, mask * x.y);
        if (wo == 0) {
            const float2 xl = Xc[bin + kBins - 1];
            Y[bin + kBins - 1] = make_float2(0.5f * xl.x, 0.5f * xl.y);
        }
    }
}

// x[j] = (Re Y0 + (-1)^j Re Y512 + 2 sum_{k=1}^{511} Re(Yk e^{2 pi i kj/1024})) / 1024 (irfft: the imaginary parts of bins 0
// and 512 do not enter), times the inverse window hann[j] / (hann[j mod 768]^2 + hann[j mod 768 + 768]^2).
__global__ void __launch_bounds__(kThreads) spec_istft_kernel(const float* __restrict__ Y, int n_frames,
                                                              float* __restrict__ frames) {
    __shared__ float c[kN], s[kN], re[kBins], im[kBins];
    const long long fr = (long long)blockIdx.y * n_frames + blockIdx.x;
    load_twiddles(c, s);
    const float2* y = reinterpret_cast<const float2*>(Y) + fr * kBins;
    for (int k = threadIdx.x; k < kBins; k += blockDim.x) {
        const float2 v = y[k];
        re[k] = v.x;
        im[k] = v.y;
    }
    __syncthreads();
    for (int j = threadIdx.x; j < kN; j += blockDim.x) {
        float acc = 0.f;
        for (int k = 1; k < kBins - 1; ++k) {
            const int m = (k * j) & (kN - 1);
            acc = fmaf(re[k], c[m], acc);
            acc = fmaf(-im[k], s[m], acc);
        }
        const float v = (re[0] + ((j & 1) ? -re[kBins - 1] : re[kBins - 1]) + 2.f * acc) * (1.f / kN);
        const int q = j % kHop;
        const float w0 = hann(c, q), w1 = q + kHop < kN ? hann(c, q + kHop) : 0.f;
        frames[fr * kN + j] = v * (hann(c, j) / (w0 * w0 + w1 * w1));
    }
}

__global__ void __launch_bounds__(kThreads) spec_ola_kernel(const float* __restrict__ frames, int n_frames, long long T,
                                                            int batch, float* __restrict__ out) {
    const long long total = (long long)batch * T;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int b = (int)(i / T);
        const long long t = i % T;
        int hi = (int)(t / kHop);
        if (hi > n_frames - 1) hi = n_frames - 1;
        const float* fb = frames + (long long)b * n_frames * kN;
        float v = 0.f;
        if (hi >= 1 && t - (long long)(hi - 1) * kHop < kN) v = fb[(long long)(hi - 1) * kN + (t - (long long)(hi - 1) * kHop)];
        v += fb[(long long)hi * kN + (t - (long long)hi * kHop)];
        out[i] = v;
    }
}

unsigned blocks_for(long long threads, int per_block) { return (unsigned)((threads + per_block - 1) / per_block); }

}  // namespace

void launch_spec_stft(const SpecStft& P, int signals, cudaStream_t stream) {
    spec_stft_kernel<<<dim3((unsigned)P.n_frames, (unsigned)signals), kThreads, 0, stream>>>(P);
}

// Four output columns per thread while that still leaves two CTAs of 128 threads per SM; one column otherwise (the deep
// layers, which have few output positions and many channels).
static bool wide_tiles(const SpecConv& A) {
    return (long long)A.batch * A.Ho * ((A.Wo + 3) / 4) * A.Co >= 132LL * 2 * 128;
}

void launch_spec_down(const SpecConv& A, cudaStream_t stream) {
    if (wide_tiles(A))
        spec_down_kernel<4><<<blocks_for((long long)A.batch * A.Ho * ((A.Wo + 3) / 4) * A.Co, 128), 128, 0, stream>>>(A);
    else
        spec_down_kernel<1><<<blocks_for((long long)A.batch * A.Ho * A.Wo * A.Co, 128), 128, 0, stream>>>(A);
}

void launch_spec_up(const SpecConv& A, cudaStream_t stream) {
    if (wide_tiles(A))
        spec_up_kernel<4><<<blocks_for((long long)A.batch * A.Ho * ((A.Wo + 3) / 4) * A.Co, 128), 128, 0, stream>>>(A);
    else
        spec_up_kernel<1><<<blocks_for((long long)A.batch * A.Ho * A.Wo * A.Co, 128), 128, 0, stream>>>(A);
}

void launch_spec_mask(const SpecConv& A, const float* X, float* out, int magnitude, cudaStream_t stream) {
    spec_mask_kernel<<<blocks_for((long long)A.batch * A.Ho * A.Wo, 128), 128, 0, stream>>>(A, X, out, magnitude);
}

void launch_spec_istft(const float* Y, int n_frames, int batch, float* frames, float* out, long long T, cudaStream_t stream) {
    spec_istft_kernel<<<dim3((unsigned)n_frames, (unsigned)batch), kThreads, 0, stream>>>(Y, n_frames, frames);
    long long blocks = ((long long)batch * T + kThreads - 1) / kThreads;
    if (blocks > 132 * 16) blocks = 132 * 16;
    spec_ola_kernel<<<(unsigned)blocks, kThreads, 0, stream>>>(frames, n_frames, T, batch, out);
}

}  // namespace wun
