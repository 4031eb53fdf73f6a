// kernels_eval.cu - the data path of the reference's validation and test loss (Test.test, Test.py:57-79) on the device.
//
//   snippet_batch_kernel  one evaluation batch cut out of a partition pool: the recorded mix at every snippet start and the
//                         centre T_out frames of every source (Datasets.py:21-25 take_all_snippets, :207 crop_sample; no
//                         augmentation).  The batch index comes from a device counter that the call advances, so one captured
//                         CUDA graph of batch -> forward -> loss replays once per batch of the partition.
//   eval_loss_partials    per-CTA fp64 sums of (target - estimate)^2 for every source, into caller-owned slots
//   eval_loss_finish      one CTA: the slots reduced in a fixed order, curr = sum_k mean_k / K, and the running mean
//                         total += (1 / n) * (curr - total) of Test.py:76 applied to a device {total, n}
//
// The grid of the loss is a compile-time constant, independent of the device, and every reduction is a fixed tree: the same
// inputs give the same bits on every call and on every GPU, so ranks that each evaluate a whole partition agree exactly.
// fp64 arithmetic is written with _rn intrinsics so that no FMA contraction occurs.  DESIGN.md §4.7.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/wun.h"
#include "kernels.h"

namespace {

constexpr int kThreads = 256;
constexpr int kLossCtas = WUN_EVAL_LOSS_CTAS;

struct SnippetLaunch {
    const float* pool;                 // [K + 1][total_frames][C]
    long long total_frames;
    const long long* positions;        // [n_batches * batch] absolute pool frame of every snippet
    long long n_batches;
    int batch, K, C, T_in, T_out;
    const long long* batch_state;      // device int64[1]
    float* mix_out;                    // [B][T_in][C]
    float* targets_out;                // [K][B][T_out][C]
};

__global__ void __launch_bounds__(kThreads) snippet_batch_kernel(const SnippetLaunch S) {
    const int b = blockIdx.y;
    const long long batch_idx = S.batch_state[0] % S.n_batches;
    const long long f0 = __ldg(S.positions + batch_idx * S.batch + b);
    const long long per_src = S.total_frames * S.C;
    const long long n_in = (long long)S.T_in * S.C;
    const long long crop = (long long)((S.T_in - S.T_out) / 2) * S.C;
    const long long n_out = (long long)S.T_out * S.C;
    const float* mix_src = S.pool + (long long)S.K * per_src + f0 * S.C;
    float* mix_dst = S.mix_out + (long long)b * n_in;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_in; i += (long long)gridDim.x * blockDim.x)
        mix_dst[i] = __ldg(mix_src + i);
    for (int k = 0; k < S.K; ++k) {
        const float* src = S.pool + (long long)k * per_src + f0 * S.C + crop;
        float* dst = S.targets_out + ((long long)k * S.batch + b) * n_out;
        for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_out; i += (long long)gridDim.x * blockDim.x)
            dst[i] = __ldg(src + i);
    }
}

__global__ void snippet_advance_kernel(long long* batch_state) { batch_state[0] += 1; }

// Sum over the block in a fixed tree: warp shuffles, then warp 0 over the warp sums.  Valid in thread 0.
__device__ __forceinline__ double block_sum(double v, double* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_down_sync(0xffffffffu, v, o));
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) red[warp] = v;
    __syncthreads();
    if (warp == 0) {
        v = lane < kThreads / 32 ? red[lane] : 0.0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_down_sync(0xffffffffu, v, o));
    }
    __syncthreads();
    return v;
}

// slots[k][cta] = sum over this CTA's elements of source k of (target - estimate)^2, or |target - estimate| with kL1 (the
// spectrogram U-Net's magnitude loss, Test.py:63-67), each thread in a fixed grid stride.
template <bool kL1>
__global__ void __launch_bounds__(kThreads) eval_loss_partials(const float* __restrict__ outputs,
                                                               const float* __restrict__ targets, long long n,
                                                               double* __restrict__ slots) {
    __shared__ double red[kThreads / 32];
    const int k = blockIdx.y;
    const float* o = outputs + (long long)k * n;
    const float* t = targets + (long long)k * n;
    double acc = 0.0;
    for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n; i += (long long)kLossCtas * kThreads) {
        const double d = __dsub_rn((double)__ldg(t + i), (double)__ldg(o + i));
        acc = __dadd_rn(acc, kL1 ? fabs(d) : __dmul_rn(d, d));
    }
    acc = block_sum(acc, red);
    if (threadIdx.x == 0) slots[(long long)k * kLossCtas + blockIdx.x] = acc;
}

__global__ void __launch_bounds__(kThreads) eval_loss_finish(const double* __restrict__ slots, int K, long long n,
                                                             double* __restrict__ state, double* __restrict__ batch_loss) {
    __shared__ double red[kThreads / 32];
    double curr = 0.0;
    for (int k = 0; k < K; ++k) {
        double v = 0.0;
        for (int s = threadIdx.x; s < kLossCtas; s += kThreads) v = __dadd_rn(v, slots[(long long)k * kLossCtas + s]);
        v = block_sum(v, red);
        if (threadIdx.x == 0) curr = __dadd_rn(curr, __ddiv_rn(v, (double)n));        // reduce_mean, summed over sources
    }
    if (threadIdx.x == 0) {
        curr = __ddiv_rn(curr, (double)K);                                              // / num_sources (Test.py:71)
        const double total = state[0], count = __dadd_rn(state[1], 1.0);
        state[0] = __dadd_rn(total, __dmul_rn(__ddiv_rn(1.0, count), __dsub_rn(curr, total)));     // Test.py:76
        state[1] = count;
        if (batch_loss) batch_loss[0] = curr;
    }
}

bool have_gpu() {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        return false;
    }
    return true;
}

}  // namespace

extern "C" int wun_snippet_batch(const float* pool, int64_t total_frames, int64_t num_sources, int64_t nchan,
                                 int64_t input_frames, int64_t output_frames, const int64_t* positions, int64_t n_positions,
                                 int64_t batch, int64_t* batch_state, float* mix_out, float* targets_out, void* stream) {
    if (num_sources < 1 || num_sources > WUN_MAX_SOURCES || (nchan != 1 && nchan != 2)) return WUN_E_INVALID;
    if (input_frames < 1 || output_frames < 1 || output_frames > input_frames || input_frames > INT32_MAX) return WUN_E_INVALID;
    if (batch < 1 || batch > 65535 || n_positions < batch || n_positions % batch != 0 || total_frames < input_frames)
        return WUN_E_INVALID;
    if (!pool || !positions || !batch_state || !mix_out || !targets_out) return WUN_E_INVALID;
    if (!have_gpu()) return WUN_E_NOGPU;
    SnippetLaunch S;
    S.pool = pool; S.total_frames = total_frames; S.positions = reinterpret_cast<const long long*>(positions);
    S.n_batches = n_positions / batch; S.batch = (int)batch; S.K = (int)num_sources; S.C = (int)nchan;
    S.T_in = (int)input_frames; S.T_out = (int)output_frames;
    S.batch_state = reinterpret_cast<const long long*>(batch_state); S.mix_out = mix_out; S.targets_out = targets_out;
    const long long n_in = input_frames * nchan;
    int bx = (int)((n_in + kThreads - 1) / kThreads);
    const int cap = (int)((132 * 8 + batch - 1) / batch);                  // ~8 CTAs per SM over the whole batch
    if (bx > cap) bx = cap;
    if (bx < 1) bx = 1;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    snippet_batch_kernel<<<dim3(bx, (unsigned)batch), kThreads, 0, st>>>(S);
    snippet_advance_kernel<<<1, 1, 0, st>>>(reinterpret_cast<long long*>(batch_state));
    return cudaGetLastError() == cudaSuccess ? WUN_OK : WUN_E_CUDA;
}

extern "C" int wun_eval_batch_loss(const float* outputs, const float* targets, int64_t num_sources, int64_t n,
                                   double* state, double* batch_loss, void* workspace, int64_t workspace_bytes, void* stream) {
    if (num_sources < 1 || num_sources > WUN_MAX_SOURCES || n < 1) return WUN_E_INVALID;
    if (!outputs || !targets || !state || !workspace) return WUN_E_INVALID;
    if (workspace_bytes < num_sources * kLossCtas * (int64_t)sizeof(double) || (reinterpret_cast<uintptr_t>(workspace) & 7))
        return WUN_E_INVALID;
    if (!have_gpu()) return WUN_E_NOGPU;
    wun::launch_eval_loss(outputs, targets, (int)num_sources, n, state, batch_loss, static_cast<double*>(workspace), false,
                          static_cast<cudaStream_t>(stream));
    return cudaGetLastError() == cudaSuccess ? WUN_OK : WUN_E_CUDA;
}

void wun::launch_eval_loss(const float* outputs, const float* targets, int K, long long n, double* state, double* batch_loss,
                           double* slots, bool l1, cudaStream_t stream) {
    if (l1)
        eval_loss_partials<true><<<dim3(kLossCtas, (unsigned)K), kThreads, 0, stream>>>(outputs, targets, n, slots);
    else
        eval_loss_partials<false><<<dim3(kLossCtas, (unsigned)K), kThreads, 0, stream>>>(outputs, targets, n, slots);
    eval_loss_finish<<<1, kThreads, 0, stream>>>(slots, K, n, state, batch_loss);
}
