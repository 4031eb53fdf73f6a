// kernels_feed.cu - training-batch construction on the device (SURVEY 8(f) row N4).
//
// What the reference's tf.data pipeline does per training example (Datasets.py:16-19,196-207; Utils.py:26-42), with the
// tracks resident in HBM instead of TFRecords:
//   take_random_snippets  start ~ U{0 .. length - T_in - 1}, T_in frames of every source (and of the mix)   Datasets.py:16-19
//   random_amplify        source_k *= U(0.7, 1.0) (one gain per source per snippet); mix = sum_k source_k    Utils.py:26-36
//   crop_sample           sources keep their centre T_out frames (crop (T_in - T_out)//2 each side)           Utils.py:38-42
//   shuffle + batch       here: the track of every example is drawn uniformly at random
// Pure HBM-bound byte movement: per example K*T_in*C floats read, (T_in + K*T_out)*C written, coalesced; no tensor cores.
//
// Randomness is a counter-based hash of (seed, step, example, slot) - the step counter lives on the device and is advanced
// by the kernel launch itself, so the feeder can sit inside the CUDA graph of a training step.  oracle/feeder_oracle.py
// restates the same arithmetic in numpy; the products / sums below are written with explicit round-to-nearest intrinsics so
// that no FMA contraction can make the device differ from that restatement (bit-exact parity test).
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.h"

namespace wun {

// slot 0: track, 1: start position, 2 + k: gain of source k
__host__ __device__ __forceinline__ uint64_t feed_rand(uint64_t seed, uint64_t step, uint32_t example, uint32_t slot) {
    const uint64_t key = (step << 32) ^ ((uint64_t)example << 8) ^ (uint64_t)slot;
    return feed_mix64(seed ^ feed_mix64(key + 0x9E3779B97F4A7C15ull));
}

struct FeedLaunch {
    const float* pool;                 // [K + 1][total_frames][C]: sources in source_names order, then the mix
    long long total_frames;
    const long long* track_offset;     // [n_tracks] first frame of each track inside the pool
    const long long* track_length;     // [n_tracks] frames (padding included, as write_records stores them)
    int n_tracks, batch, K, C, T_in, T_out, augmentation;
    unsigned long long seed;
    const long long* step_state;       // device int64[1]
    float* mix_out;                    // [B][T_in][C]
    float* targets_out;                // [K][B][T_out][C]
    long long* chosen;                 // optional [B][2] (track, start) for tests / logging
};

__global__ void __launch_bounds__(256) feed_batch_kernel(const FeedLaunch F) {
    const int b = blockIdx.y;
    const uint64_t step = (uint64_t)F.step_state[0];
    const int track = (int)(feed_rand(F.seed, step, b, 0) % (uint64_t)F.n_tracks);
    const long long len = F.track_length[track];
    const long long span = len - F.T_in;                                   // tf.random_uniform(maxval) is exclusive
    const long long pos = (span > 0) ? (long long)(feed_rand(F.seed, step, b, 1) % (uint64_t)span) : 0;
    const long long f0 = F.track_offset[track] + pos;                      // first pool frame of the snippet
    if (F.chosen && blockIdx.x == 0 && threadIdx.x == 0) { F.chosen[2 * b] = track; F.chosen[2 * b + 1] = pos; }
    float gain[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        gain[k] = 1.f;
        if (k < F.K && F.augmentation) {
            const float u = (float)(feed_rand(F.seed, step, b, 2 + k) >> 40) * (1.0f / 16777216.0f);
            gain[k] = __fadd_rn(__fmul_rn(u, 0.3f), 0.7f);                 // rand * (1.0 - 0.7) + 0.7
        }
    }
    const int crop = (F.T_in - F.T_out) / 2;
    const long long per_src = F.total_frames * F.C;
    const long long n_in = (long long)F.T_in * F.C;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_in; i += (long long)gridDim.x * blockDim.x) {
        const long long t = i / F.C;
        const long long src = f0 * F.C + i;
        float mix;
        if (F.augmentation) {
            mix = 0.f;
            for (int k = 0; k < F.K; ++k) {
                const float v = __fmul_rn(gain[k], __ldg(F.pool + (long long)k * per_src + src));
                mix = (k == 0) ? v : __fadd_rn(mix, v);                    // tf.add_n over the sources, in order
                const long long to = t - crop;
                if (to >= 0 && to < F.T_out)
                    F.targets_out[(((long long)k * F.batch + b) * F.T_out + to) * F.C + (i - t * F.C)] = v;
            }
        } else {
            mix = __ldg(F.pool + (long long)F.K * per_src + src);          // the recorded mixture
            const long long to = t - crop;
            if (to >= 0 && to < F.T_out)
                for (int k = 0; k < F.K; ++k)
                    F.targets_out[(((long long)k * F.batch + b) * F.T_out + to) * F.C + (i - t * F.C)] =
                        __ldg(F.pool + (long long)k * per_src + src);
        }
        F.mix_out[(long long)b * n_in + i] = mix;
    }
}

__global__ void feed_advance_kernel(long long* step_state) { step_state[0] += 1; }

cudaError_t launch_feed_batch(const float* pool, long long total_frames, const long long* track_offset,
                              const long long* track_length, int n_tracks, int batch, int K, int C, int T_in, int T_out,
                              int augmentation, unsigned long long seed, long long* step_state, float* mix_out,
                              float* targets_out, long long* chosen, cudaStream_t stream) {
    if (K < 1 || K > 8 || batch < 1 || n_tracks < 1) return cudaErrorInvalidValue;
    FeedLaunch F;
    F.pool = pool; F.total_frames = total_frames; F.track_offset = track_offset; F.track_length = track_length;
    F.n_tracks = n_tracks; F.batch = batch; F.K = K; F.C = C; F.T_in = T_in; F.T_out = T_out; F.augmentation = augmentation;
    F.seed = seed; F.step_state = step_state; F.mix_out = mix_out; F.targets_out = targets_out; F.chosen = chosen;
    const long long n_in = (long long)T_in * C;
    int bx = (int)((n_in + 255) / 256);
    const int cap = (132 * 8 + batch - 1) / batch;                         // ~8 CTAs per SM over the whole batch
    if (bx > cap) bx = cap;
    if (bx < 1) bx = 1;
    feed_batch_kernel<<<dim3(bx, batch), 256, 0, stream>>>(F);
    feed_advance_kernel<<<1, 1, 0, stream>>>(step_state);
    return cudaGetLastError();
}

}  // namespace wun
