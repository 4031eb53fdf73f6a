// FLAC encoding on the GPU: the separated estimates written as 16- or 24-bit FLAC (DESIGN.md §4.11).  The frame code is in
// flac_encode.h, shared with the host build the CPU tests run; here it runs with a CUDA block as the team:
//
//   flac_quantise_kernel  float32 samples -> int32 at the stream's depth (float input only)
//   flac_analyse_kernel   one block per (frame, signal): the cheapest subframe and its exact bit count
//   flac_layout_kernel    one block: each frame's channel assignment and byte size, then the exclusive scan of the sizes into
//                         the caller's frame offsets
//   flac_pack_kernel      one block per frame: header, subframes and CRC-16 into the zeroed output
//
// The host (wun.write_flac, wun/flac.py) adds the `fLaC` marker, STREAMINFO (with the MD5) and a VORBIS_COMMENT block.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/wun.h"
#include "flac_encode.h"

namespace {

namespace F = wun::flac;

constexpr int kLayoutThreads = 1024;

struct Block {
    __device__ int tid() const { return threadIdx.x; }
    __device__ int n() const { return blockDim.x; }
    __device__ void sync() const { __syncthreads(); }
    __device__ void add(uint64_t* p, uint64_t v) const {
        atomicAdd(reinterpret_cast<unsigned long long*>(p), (unsigned long long)v);
    }
    __device__ void or_flag(int32_t* p, int32_t v) const {
        if (v) atomicOr(p, v);
    }
    __device__ void or_word(uint32_t* w, uint32_t v) const { atomicOr(w, v); }
    __device__ uint32_t load_word(const uint32_t* w) const { return __ldcg(w); }
};

struct Workspace {                                           // carved out of the caller's workspace, 256-byte aligned pieces
    int32_t* quantised;                                      // n * C (float input)
    F::SubChoice* sub;                                       // frames * signals
    F::FrameChoice* frames;                                  // frames
    int32_t* error;                                          // 1
    int64_t bytes;
};

int64_t align256(int64_t v) { return (v + 255) & ~(int64_t)255; }

Workspace carve(void* base, int64_t n, int C, int block_size) {
    const int64_t frames = (n + block_size - 1) / block_size;
    char* p = static_cast<char*>(base);
    Workspace w;
    int64_t off = 0;
    w.quantised = reinterpret_cast<int32_t*>(p + off);
    off += align256(n * C * 4);
    w.sub = reinterpret_cast<F::SubChoice*>(p + off);
    off += align256(frames * F::signals_of(C) * (int64_t)sizeof(F::SubChoice));
    w.frames = reinterpret_cast<F::FrameChoice*>(p + off);
    off += align256(frames * (int64_t)sizeof(F::FrameChoice));
    w.error = reinterpret_cast<int32_t*>(p + off);
    off += 256;
    w.bytes = off;
    return w;
}

__global__ void flac_quantise_kernel(const float* __restrict__ x, int64_t count, int bps, int32_t* __restrict__ out) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x)
        out[i] = F::quantise(x[i], bps);
}

__global__ void __launch_bounds__(F::kThreads) flac_analyse_kernel(const int32_t* __restrict__ x, int64_t n, int C, int bps,
                                                                   int rate, int block_size, F::SubChoice* __restrict__ sub) {
    extern __shared__ __align__(16) unsigned char smem[];
    F::Scratch& s = *reinterpret_cast<F::Scratch*>(smem);
    const int64_t frame = blockIdx.x;
    const int sig = blockIdx.y;
    const int64_t first = frame * block_size;
    const int bs = (int)(n - first < block_size ? n - first : block_size);
    F::analyse_signal(Block(), s, x + first * C, C, sig, bs, bps, rate, sub + frame * F::signals_of(C) + sig);
}

__global__ void __launch_bounds__(kLayoutThreads) flac_layout_kernel(const F::SubChoice* __restrict__ sub, int64_t frames,
                                                                     int64_t n, int C, int bps, int rate, int block_size,
                                                                     F::FrameChoice* __restrict__ fc,
                                                                     int64_t* __restrict__ offsets,
                                                                     int32_t* __restrict__ error) {
    __shared__ int64_t part[kLayoutThreads];
    __shared__ int bad;
    if (threadIdx.x == 0) bad = 0;
    __syncthreads();
    const int S = F::signals_of(C);
    const int64_t per = (frames + kLayoutThreads - 1) / kLayoutThreads;
    const int64_t a = threadIdx.x * per, b = a + per < frames ? a + per : frames;
    int64_t sum = 0;
    for (int64_t j = a; j < b; ++j) {
        const int bs = (int)(n - j * block_size < block_size ? n - j * block_size : block_size);
        for (int c = 0; c < S; ++c)
            if (sub[j * S + c].range_error) atomicOr(&bad, 1);
        fc[j] = F::decide_frame(sub + j * S, C, bs, bps, rate, j);
        sum += fc[j].bytes;
    }
    part[threadIdx.x] = sum;
    __syncthreads();
    if (threadIdx.x == 0) {
        int64_t acc = 0;
        for (int i = 0; i < kLayoutThreads; ++i) {
            const int64_t v = part[i];
            part[i] = acc;
            acc += v;
        }
    }
    __syncthreads();
    int64_t acc = part[threadIdx.x];
    for (int64_t j = a; j < b; ++j) {
        offsets[j] = acc;
        acc += fc[j].bytes;
    }
    if (b == frames && a < b) offsets[frames] = bad ? -1 : acc;
    if (threadIdx.x == 0) {
        *error = bad;
        if (frames == 0) offsets[0] = 0;
    }
}

__global__ void __launch_bounds__(F::kThreads) flac_pack_kernel(const int32_t* __restrict__ x, int64_t n, int C, int bps,
                                                                int rate, int block_size, const F::SubChoice* __restrict__ sub,
                                                                const F::FrameChoice* __restrict__ fc,
                                                                const int64_t* __restrict__ offsets,
                                                                const int32_t* __restrict__ error, uint32_t* words) {
    if (*error) return;
    extern __shared__ __align__(16) unsigned char smem[];
    F::Scratch& s = *reinterpret_cast<F::Scratch*>(smem);
    const int64_t frame = blockIdx.x;
    const int64_t first = frame * block_size;
    const int bs = (int)(n - first < block_size ? n - first : block_size);
    F::pack_frame(Block(), s, x + first * C, C, bs, bps, rate, frame, sub + frame * F::signals_of(C), fc[frame], words,
                  offsets[frame]);
}

bool stream_ok(int64_t n, int32_t C, int32_t bps, int32_t rate, int32_t block_size) {
    int extra;
    return n >= 0 && C >= 1 && C <= 8 && bps >= 4 && bps <= 24 && rate > 0 && rate < (1 << 20) &&
           F::rate_code(rate, &extra) >= 0 && block_size >= 16 && block_size <= F::kMaxBlock &&
           (n + block_size - 1) / block_size < (int64_t)1 << 31;
}

int have_gpu() {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        return 0;
    }
    return 1;
}

}  // namespace

extern "C" int64_t wun_flac_encode_workspace_bytes(int64_t n, int32_t channels, int32_t block_size) {
    if (!stream_ok(n, channels, 16, 44100, block_size)) return -1;
    return carve(nullptr, n, channels, block_size).bytes;
}

extern "C" int64_t wun_flac_encode_capacity(int64_t n, int32_t channels, int32_t bps, int32_t block_size) {
    if (!stream_ok(n, channels, bps, 44100, block_size)) return -1;
    const int64_t full = n / block_size, rest = n % block_size;
    int64_t bytes = full * F::frame_bound(block_size, channels, bps) + (rest ? F::frame_bound((int)rest, channels, bps) : 0);
    return (bytes + 3) & ~(int64_t)3;
}

extern "C" int wun_flac_encode_frames(const void* samples, int32_t sample_type, int64_t n, int32_t channels, int32_t bps,
                                      int32_t rate, int32_t block_size, void* workspace, int64_t workspace_bytes, uint8_t* out,
                                      int64_t out_capacity, int64_t* frame_offsets, void* stream) {
    if (!stream_ok(n, channels, bps, rate, block_size) || (sample_type != WUN_FLAC_INT32 && sample_type != WUN_FLAC_FLOAT32))
        return WUN_E_INVALID;
    if (!frame_offsets || (n > 0 && (!samples || !workspace || !out))) return WUN_E_INVALID;
    if (reinterpret_cast<uintptr_t>(out) % 4 || reinterpret_cast<uintptr_t>(workspace) % 256) return WUN_E_INVALID;
    const Workspace ws = carve(workspace, n, channels, block_size);
    if (workspace_bytes < ws.bytes || out_capacity < wun_flac_encode_capacity(n, channels, bps, block_size))
        return WUN_E_INVALID;
    if (!have_gpu()) return WUN_E_NOGPU;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (n == 0) return cudaMemsetAsync(frame_offsets, 0, sizeof(int64_t), st) == cudaSuccess ? WUN_OK : WUN_E_CUDA;
    const int64_t frames = (n + block_size - 1) / block_size;
    const int32_t* x = static_cast<const int32_t*>(samples);
    if (sample_type == WUN_FLAC_FLOAT32) {
        const int64_t count = n * channels;
        const int64_t blocks = (count + 255) / 256 < 4096 ? (count + 255) / 256 : 4096;
        flac_quantise_kernel<<<(unsigned)blocks, 256, 0, st>>>(static_cast<const float*>(samples), count, bps, ws.quantised);
        x = ws.quantised;
    }
    const int smem = (int)sizeof(F::Scratch);
    if (cudaFuncSetAttribute(flac_analyse_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess ||
        cudaFuncSetAttribute(flac_pack_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess)
        return WUN_E_CUDA;
    if (cudaMemsetAsync(out, 0, (size_t)wun_flac_encode_capacity(n, channels, bps, block_size), st) != cudaSuccess)
        return WUN_E_CUDA;
    flac_analyse_kernel<<<dim3((unsigned)frames, (unsigned)F::signals_of(channels)), F::kThreads, smem, st>>>(
        x, n, channels, bps, rate, block_size, ws.sub);
    flac_layout_kernel<<<1, kLayoutThreads, 0, st>>>(ws.sub, frames, n, channels, bps, rate, block_size, ws.frames,
                                                     frame_offsets, ws.error);
    flac_pack_kernel<<<(unsigned)frames, F::kThreads, smem, st>>>(x, n, channels, bps, rate, block_size, ws.sub, ws.frames,
                                                                  frame_offsets, ws.error, reinterpret_cast<uint32_t*>(out));
    return cudaGetLastError() == cudaSuccess ? WUN_OK : WUN_E_CUDA;
}
