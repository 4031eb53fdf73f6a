// Host build of the GPU FLAC encoder's frame code (wave-u-net_b200/csrc/flac_encode.h) for the CPU tests, compiled with
// AddressSanitizer and UBSan: the passes kernels_flac_encode.cu runs, with one serial team doing each block's work.
//
//   flac_encode_host <samples.bin> <n> <channels> <bps> <rate> <block_size> <area.bin> <offsets.bin>
//       samples.bin: int32 [n][channels]; writes the frame area and the n_frames + 1 int64 frame offsets (the last -1 when a
//       sample lies outside the depth, as the device's are)
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <vector>

#include "flac_encode.h"

namespace F = wun::flac;

int main(int argc, char** argv) {
    if (argc != 9) return 2;
    const int64_t n = atoll(argv[2]);
    const int C = atoi(argv[3]), bps = atoi(argv[4]), rate = atoi(argv[5]), block = atoi(argv[6]);
    // exact-size heap buffers, so that AddressSanitizer reports any access one element past them
    int32_t* x = (int32_t*)malloc((size_t)(n * C > 0 ? n * C : 1) * 4);
    FILE* f = fopen(argv[1], "rb");
    if (!f || fread(x, 4, (size_t)(n * C), f) != (size_t)(n * C)) return 2;
    fclose(f);
    const int64_t frames = (n + block - 1) / block, S = F::signals_of(C);
    F::Scratch* s = new F::Scratch;
    std::vector<F::SubChoice> sub((size_t)(frames * S));
    std::vector<F::FrameChoice> fc((size_t)frames);
    std::vector<int64_t> offsets((size_t)frames + 1, 0);
    const F::Serial tm;
    bool bad = false;
    for (int64_t j = 0; j < frames; ++j) {
        const int bs = (int)(n - j * block < block ? n - j * block : block);
        for (int sig = 0; sig < S; ++sig) {
            F::analyse_signal(tm, *s, x + j * block * C, C, sig, bs, bps, rate, &sub[(size_t)(j * S + sig)]);
            bad |= sub[(size_t)(j * S + sig)].range_error != 0;
        }
        fc[(size_t)j] = F::decide_frame(&sub[(size_t)(j * S)], C, bs, bps, rate, j);
        offsets[(size_t)j + 1] = offsets[(size_t)j] + fc[(size_t)j].bytes;
    }
    const int64_t total = offsets[(size_t)frames];
    int64_t words = (total + 3) / 4;
    uint32_t* area = (uint32_t*)calloc((size_t)(words > 0 ? words : 1), 4);
    if (!bad)
        for (int64_t j = 0; j < frames; ++j) {
            const int bs = (int)(n - j * block < block ? n - j * block : block);
            F::pack_frame(tm, *s, x + j * block * C, C, bs, bps, rate, j, &sub[(size_t)(j * S)], fc[(size_t)j], area,
                          offsets[(size_t)j]);
        }
    if (bad) offsets[(size_t)frames] = -1;
    FILE* o = fopen(argv[7], "wb");
    fwrite(area, 1, (size_t)(bad ? 0 : total), o);
    fclose(o);
    o = fopen(argv[8], "wb");
    fwrite(offsets.data(), 8, offsets.size(), o);
    fclose(o);
    free(area);
    free(x);
    delete s;
    return 0;
}
