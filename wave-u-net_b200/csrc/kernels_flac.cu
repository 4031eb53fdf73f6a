// FLAC decoding on the GPU: the reference reads compressed audio through librosa 0.6 / audioread / ffmpeg (Utils.load); this is
// the FLAC part of that, lossless and self-checking (DESIGN.md §4.10).  The host parses the metadata and chains the frames
// (wun/flac.py); the device does the per-byte work:
//
//   flac_find_kernel    one thread per byte offset of the frame area: a sync code, a legal header agreeing with STREAMINFO and
//                       a matching CRC-8 make a candidate, which the same thread then parses to its end and CRC-16.
//   flac_decode_kernel  one thread per frame of the chain the host kept: decode every subframe straight into the frame's rows
//                       of the int32 [n][C] output, then undo the stereo decorrelation in place.
//
// A false candidate is parsed but never decoded, so it writes nothing but its own record.  The frame decoder itself is in
// flac_frame.h, shared with the host build the CPU tests run.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/wun.h"
#include "flac_frame.h"

namespace {

constexpr int kFindThreads = 256;
constexpr int kDecodeThreads = 64;

__global__ void __launch_bounds__(kFindThreads) flac_find_kernel(const uint8_t* __restrict__ buf, int64_t n,
                                                                 wun::flac::StreamInfo si, WunFlacFrame* __restrict__ frames,
                                                                 int64_t capacity, unsigned long long* __restrict__ count) {
    const int64_t off = (int64_t)blockIdx.x * kFindThreads + threadIdx.x;
    if (off + 1 >= n || buf[off] != 0xFF || (buf[off + 1] & 0xFE) != 0xF8) return;
    wun::flac::Header h;
    if (!wun::flac::parse_header(buf, n, off, si, &h)) return;
    const int64_t end = wun::flac::decode_frame(buf, n, off, si, h, nullptr);
    const unsigned long long slot = atomicAdd(count, 1ull);
    if ((int64_t)slot >= capacity) return;
    WunFlacFrame f;
    f.offset = off;
    f.number = h.number;
    f.end = end;
    f.block_size = h.block_size;
    f.variable = h.variable;
    frames[slot] = f;
}

__global__ void __launch_bounds__(kDecodeThreads) flac_decode_kernel(const uint8_t* __restrict__ buf, int64_t n,
                                                                     wun::flac::StreamInfo si,
                                                                     const int64_t* __restrict__ offsets,
                                                                     const int64_t* __restrict__ first_samples,
                                                                     int64_t nframes, int32_t* __restrict__ out,
                                                                     int64_t total, int32_t* __restrict__ status) {
    const int64_t j = (int64_t)blockIdx.x * kDecodeThreads + threadIdx.x;
    if (j >= nframes) return;
    wun::flac::Header h;
    const int64_t first = first_samples[j];
    if (!wun::flac::parse_header(buf, n, offsets[j], si, &h)) {
        status[j] = wun::flac::kBadHeader;
        return;
    }
    if (first < 0 || first + h.block_size > total) {
        status[j] = wun::flac::kBadPosition;
        return;
    }
    const int64_t end = wun::flac::decode_frame(buf, n, offsets[j], si, h, out + first * si.channels);
    status[j] = end < 0 ? (int32_t)end : 0;
}

bool stream_info_ok(int32_t bps, int32_t channels, int32_t rate, int32_t max_block) {
    return bps >= 4 && bps <= 24 && channels >= 1 && channels <= 8 && rate > 0 && max_block >= 0 && max_block <= 65535;
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

extern "C" int wun_flac_find_frames(const uint8_t* buf, int64_t nbytes, int32_t bps, int32_t channels, int32_t rate,
                                    int32_t max_block, WunFlacFrame* frames, int64_t capacity, uint64_t* count, void* stream) {
    if (!buf || nbytes < 1 || !count || capacity < 0 || (capacity > 0 && !frames)) return WUN_E_INVALID;
    if (!stream_info_ok(bps, channels, rate, max_block)) return WUN_E_INVALID;
    if (!have_gpu()) return WUN_E_NOGPU;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (cudaMemsetAsync(count, 0, sizeof(uint64_t), st) != cudaSuccess) return WUN_E_CUDA;
    const wun::flac::StreamInfo si{bps, channels, rate, max_block};
    const int64_t blocks = (nbytes + kFindThreads - 1) / kFindThreads;
    flac_find_kernel<<<(unsigned)blocks, kFindThreads, 0, st>>>(buf, nbytes, si, frames, capacity,
                                                                reinterpret_cast<unsigned long long*>(count));
    return cudaGetLastError() == cudaSuccess ? WUN_OK : WUN_E_CUDA;
}

extern "C" int wun_flac_decode_frames(const uint8_t* buf, int64_t nbytes, int32_t bps, int32_t channels, int32_t rate,
                                      int32_t max_block, const int64_t* offsets, const int64_t* first_samples,
                                      int64_t nframes, int32_t* out, int64_t total_samples, int32_t* status, void* stream) {
    if (!buf || nbytes < 1 || nframes < 0 || total_samples < 0) return WUN_E_INVALID;
    if (nframes > 0 && (!offsets || !first_samples || !out || !status)) return WUN_E_INVALID;
    if (!stream_info_ok(bps, channels, rate, max_block)) return WUN_E_INVALID;
    if (!have_gpu()) return WUN_E_NOGPU;
    if (nframes == 0) return WUN_OK;
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const wun::flac::StreamInfo si{bps, channels, rate, max_block};
    const int64_t blocks = (nframes + kDecodeThreads - 1) / kDecodeThreads;
    flac_decode_kernel<<<(unsigned)blocks, kDecodeThreads, 0, st>>>(buf, nbytes, si, offsets, first_samples, nframes, out,
                                                                    total_samples, status);
    return cudaGetLastError() == cudaSuccess ? WUN_OK : WUN_E_CUDA;
}
