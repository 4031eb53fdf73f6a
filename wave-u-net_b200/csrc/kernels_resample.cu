// Band-limited resampling as librosa 0.6.2 resample(y, sr_in, sr_out) computes it with res_type='kaiser_best': the inner loop
// of resampy 0.2's resample_f, bit for bit, then librosa's fix_length zero padding.  The reference resamples every track to
// expected_sr before separating it and the estimates back afterwards (Evaluate.py:64,104, Utils.resample).  DESIGN.md §4.6
// describes the algorithm; oracle/resample_oracle.py restates it in numpy.
//
// One thread per output frame, all channels in that thread, so the filter weight is formed once per tap.  Every product and
// sum is written with an explicit _rn intrinsic: resampy evaluates weight = win + eta * delta and y += weight * x in fp64
// without contraction, rounding y back to fp32 after each addition, and a DFMA would change the bits.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/wun.h"

namespace {

constexpr int kThreads = 256;
constexpr long long kMantMask = (1LL << 52) - 1;

// resampy's time_register after t steps: the sequential fp64 sum 0 + inc + inc + ... (t terms), without the scan.  Inside one
// binade [2^e, 2^(e+1)) every addition of inc that starts from a value produced by an addition inside the same binade adds
// the same number d of ulps: round-to-nearest of inc / ulp is fixed, and where it is a tie, ties-to-even makes every such
// value even in ulps, so the tie always resolves the same way.  Only the step entering the binade and the step after it can
// differ.  So: take real steps until two consecutive ones stayed inside one binade, then jump over every further step that
// stays inside it, and repeat in the next binade; about 3 real steps per binade (25 binades for 3 minutes at 44.1 kHz).
__device__ double time_register(int64_t t, double inc) {
    double x = 0.0;
    int64_t s = 0;
    int inside = 0;                        // consecutive real steps that began and ended in x's binade
    while (s < t) {
        const double nx = __dadd_rn(x, inc);
        const long long b0 = __double_as_longlong(x), b1 = __double_as_longlong(nx);
        inside = (b0 >> 52) == (b1 >> 52) ? inside + 1 : 0;
        x = nx;
        ++s;
        if (inside >= 2 && s < t) {
            const long long d = b1 - b0;                         // ulps per step from here on, while inside the binade
            const long long room = (b1 | kMantMask) - b1;        // ulps left below the next power of two
            const int64_t k = d > 0 ? min((int64_t)(room / d), t - s) : t - s;
            x = __longlong_as_double(b1 + k * d);
            s += k;
            inside = 0;
        }
    }
    return x;
}

// One wing of resampy's filter response: taps i < min(limit, (nwin - offset) // index_step), input frame first + dir * i.
// Frames at or past n_in read as zero (adding a zero product leaves y's bits alone); resampy never reaches them for inputs
// shorter than hours, where the sequential time register has drifted by less than a frame.
template <int C>
__device__ __forceinline__ void wing(float (&acc)[C], const float* __restrict__ x, int64_t n_in, int64_t first, int dir,
                                     int64_t limit, double frac, double precision, int index_step,
                                     const double* __restrict__ win, const double* __restrict__ delta, int nwin) {
    const double index_frac = __dmul_rn(frac, precision);
    const int offset = (int)index_frac;                                  // int(): truncation, index_frac >= 0
    const double eta = __dsub_rn(index_frac, (double)offset);
    const int64_t m = min(limit, (int64_t)((nwin - offset) / index_step));
    for (int64_t i = 0; i < m; ++i) {
        const int64_t f = first + dir * i;
        if (f >= n_in) continue;
        const int idx = offset + (int)i * index_step;
        const double w = __dadd_rn(__ldg(win + idx), __dmul_rn(eta, __ldg(delta + idx)));
        const float* xr = x + f * C;
#pragma unroll
        for (int c = 0; c < C; ++c)
            acc[c] = __double2float_rn(__dadd_rn((double)acc[c], __dmul_rn(w, (double)__ldg(xr + c))));
    }
}

// y[t] for t < n_valid = floor(n_in * ratio) as resample_f computes it; y[t] = 0 for n_valid <= t < n_out (fix_length).
template <int C>
__global__ void __launch_bounds__(kThreads) resample_kernel(const float* __restrict__ x, int64_t n_in, double inc, double scale,
                                                            double precision, int index_step,
                                                            const double* __restrict__ win,
                                                            const double* __restrict__ delta, int nwin, int64_t n_valid,
                                                            int64_t n_out, float* __restrict__ y) {
    const int64_t t = (int64_t)blockIdx.x * kThreads + threadIdx.x;
    if (t >= n_out) return;
    float acc[C];
#pragma unroll
    for (int c = 0; c < C; ++c) acc[c] = 0.0f;
    if (t < n_valid) {
        const double tr = time_register(t, inc);
        const int64_t n = (int64_t)tr;                                   // int(time_register): truncation
        const double frac = __dmul_rn(scale, __dsub_rn(tr, (double)n));
        wing<C>(acc, x, n_in, n, -1, n + 1, frac, precision, index_step, win, delta, nwin);
        wing<C>(acc, x, n_in, n + 1, 1, n_in - n - 1, __dsub_rn(scale, frac), precision, index_step, win, delta, nwin);
    }
#pragma unroll
    for (int c = 0; c < C; ++c) y[t * C + c] = acc[c];
}

}  // namespace

extern "C" int64_t wun_resample_frames(int64_t n_in, int64_t sr_in, int64_t sr_out) {
    if (n_in < 0 || sr_in <= 0 || sr_out <= 0) return WUN_E_INVALID;
    const double ratio = (double)sr_out / (double)sr_in;
    double v = (double)n_in * ratio, c = (double)(int64_t)v;
    return (int64_t)(c < v ? c + 1.0 : c);                               // np.ceil(n_in * ratio)
}

extern "C" int wun_resample(const float* x, int64_t n_in, int64_t nchan, int64_t sr_in, int64_t sr_out, const double* win,
                            const double* delta, int64_t nwin, int64_t precision, float* y, int64_t n_out, void* stream) {
    if (nchan != 1 && nchan != 2) return WUN_E_INVALID;
    if (n_in < 1 || sr_in <= 0 || sr_out <= 0 || n_out != wun_resample_frames(n_in, sr_in, sr_out)) return WUN_E_INVALID;
    if (!x || !y || !win || !delta || nwin < 1 || nwin > INT32_MAX || precision < 1) return WUN_E_INVALID;
    const double ratio = (double)sr_out / (double)sr_in;
    const double scale = ratio < 1.0 ? ratio : 1.0;
    const double inc = 1.0 / ratio;
    const int64_t index_step = (int64_t)(scale * (double)precision);
    const int64_t n_valid = (int64_t)((double)n_in * ratio);             // resampy's output length: int(n_in * ratio)
    if (n_valid < 1 || index_step < 1) return WUN_E_INVALID;              // resampy raises ValueError for n_valid < 1
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        return WUN_E_NOGPU;
    }
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const unsigned blocks = (unsigned)((n_out + kThreads - 1) / kThreads);
    if (nchan == 1)
        resample_kernel<1><<<blocks, kThreads, 0, st>>>(x, n_in, inc, scale, (double)precision, (int)index_step, win, delta,
                                                        (int)nwin, n_valid, n_out, y);
    else
        resample_kernel<2><<<blocks, kThreads, 0, st>>>(x, n_in, inc, scale, (double)precision, (int)index_step, win, delta,
                                                        (int)nwin, n_valid, n_out, y);
    return cudaGetLastError() == cudaSuccess ? WUN_OK : WUN_E_CUDA;
}
