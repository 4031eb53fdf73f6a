// Host build of the GPU FLAC decoder's frame code (wave-u-net_b200/csrc/flac_frame.h) for the CPU tests, compiled with
// AddressSanitizer: the same passes kernels_flac.cu runs, one loop iteration per device thread.
//
//   flac_host find   <area> <bps> <channels> <rate> <max_block> <frames.bin>
//       every byte offset of the frame area through parse_header + decode_frame(out = nullptr); writes one record of five
//       int64 (offset, number, end, block_size, variable) per candidate, in offset order
//   flac_host decode <area> <bps> <channels> <rate> <max_block> <chain.bin> <total> <out.bin>
//       chain.bin: int64 pairs (offset, first sample); writes int32 [total][channels] and exits 3 naming the first frame
//       that fails, as the device's status array would
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <string>
#include <vector>

#include "flac_frame.h"

static std::vector<uint8_t> slurp(const char* path) {
    std::vector<uint8_t> v;
    FILE* f = fopen(path, "rb");
    if (!f) exit(2);
    int c;
    while ((c = fgetc(f)) != EOF) v.push_back((uint8_t)c);
    fclose(f);
    return v;
}

int main(int argc, char** argv) {
    if (argc < 8) return 2;
    const std::vector<uint8_t> area = slurp(argv[2]);
    // an exact-size heap copy, so that AddressSanitizer reports any read one byte past the frame area
    uint8_t* buf = (uint8_t*)malloc(area.size() ? area.size() : 1);
    for (size_t i = 0; i < area.size(); ++i) buf[i] = area[i];
    const int64_t n = (int64_t)area.size();
    const wun::flac::StreamInfo si{atoi(argv[3]), atoi(argv[4]), atoi(argv[5]), atoi(argv[6])};
    const std::string mode = argv[1];
    if (mode == "find") {
        FILE* o = fopen(argv[7], "wb");
        for (int64_t off = 0; off + 1 < n; ++off) {
            if (buf[off] != 0xFF || (buf[off + 1] & 0xFE) != 0xF8) continue;
            wun::flac::Header h;
            if (!wun::flac::parse_header(buf, n, off, si, &h)) continue;
            const int64_t rec[5] = {off, h.number, wun::flac::decode_frame(buf, n, off, si, h, nullptr), h.block_size,
                                    h.variable};
            fwrite(rec, sizeof(rec), 1, o);
        }
        fclose(o);
    } else if (mode == "decode" && argc >= 10) {
        const std::vector<uint8_t> chain = slurp(argv[7]);
        const int64_t total = atoll(argv[8]);
        const int64_t nframes = (int64_t)(chain.size() / 16);
        const int64_t* c = (const int64_t*)chain.data();
        int32_t* out = (int32_t*)malloc((size_t)(total * si.channels * 4 + 4));
        for (int64_t j = 0; j < nframes; ++j) {
            wun::flac::Header h;
            const int64_t off = c[2 * j], first = c[2 * j + 1];
            int64_t st = wun::flac::kBadHeader;
            if (wun::flac::parse_header(buf, n, off, si, &h))
                st = (first < 0 || first + h.block_size > total) ? wun::flac::kBadPosition
                                                                 : wun::flac::decode_frame(buf, n, off, si, h, out + first * si.channels);
            if (st < 0) {
                fprintf(stderr, "frame %lld: status %lld\n", (long long)j, (long long)st);
                return 3;
            }
        }
        FILE* o = fopen(argv[9], "wb");
        fwrite(out, 4, (size_t)(total * si.channels), o);
        fclose(o);
        free(out);
    } else {
        return 2;
    }
    free(buf);
    return 0;
}
