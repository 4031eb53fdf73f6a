// flac_frame.h - the FLAC frame decoder, shared by the CUDA kernels (kernels_flac.cu) and a host build the CPU tests run under
// AddressSanitizer (tests/flac_host.cpp).  Everything here is plain C++ on integers: no CUDA intrinsics, so both builds run
// the same code.
//
// A frame is a header (sync code, block size, rate, channel assignment, sample size, UTF-8 frame or sample number, CRC-8),
// one subframe per channel (CONSTANT, VERBATIM, FIXED order 0-4 or LPC order 1-32, each with optional wasted bits) and a
// CRC-16.  DESIGN.md §4.10 describes the format and the decode; oracle/flac_oracle.py restates it in Python.
//
// Every bit read is checked against the end of the buffer and every count against the block size: a malformed or false
// candidate returns a negative status and never reads or writes outside [buf, buf + nbytes) and the frame's rows of `out`.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define FLAC_HD __host__ __device__ __forceinline__
#else
#define FLAC_HD inline
#endif

namespace wun {
namespace flac {

// statuses a frame decode returns (non-negative: the byte offset just past the frame's CRC-16)
enum Status : int {
    kTruncated = -1,     // a read ran past the end of the buffer
    kBadHeader = -2,     // sync code, reserved value, mismatch with STREAMINFO or CRC-8
    kBadSubframe = -3,   // reserved subframe type, padding bit set, order above the block size, bad LPC precision or shift
    kBadResidual = -4,   // reserved coding method, or partitions that do not divide the block size
    kBadCrc16 = -5,      // the frame's CRC-16 does not match
    kBadPosition = -6,   // the frame's samples do not fit the output (decode pass only)
};

struct StreamInfo {
    int bps;             // bits per sample, 4..24
    int channels;        // 1..8
    int rate;            // Hz
    int max_block;       // STREAMINFO maximum block size (0: unknown)
};

struct Header {
    int64_t number;      // frame number (fixed block size) or first sample number (variable block size)
    int block_size;
    int assignment;      // 0-7 independent (assignment + 1 channels), 8 left/side, 9 right/side, 10 mid/side
    int variable;        // blocking strategy bit
    int bytes;           // header length including the CRC-8
};

FLAC_HD uint8_t crc8(const uint8_t* p, int64_t n) {
    unsigned c = 0;
    for (int64_t i = 0; i < n; ++i) {
        c ^= p[i];
        for (int b = 0; b < 8; ++b) c = (c & 0x80) ? ((c << 1) ^ 0x07) & 0xff : (c << 1) & 0xff;
    }
    return (uint8_t)c;
}

FLAC_HD uint16_t crc16(const uint8_t* p, int64_t n) {
    unsigned c = 0;
    for (int64_t i = 0; i < n; ++i) {
        c ^= (unsigned)p[i] << 8;
        for (int b = 0; b < 8; ++b) c = (c & 0x8000) ? ((c << 1) ^ 0x8005) & 0xffff : (c << 1) & 0xffff;
    }
    return (uint16_t)c;
}

// MSB-first bit reader over [p, p + n).  A read past the end sets `bad`, leaves the position at the end and returns 0, so
// every loop driven by a corrupt count stops consuming input at once and is bounded by the block size.
struct Bits {
    const uint8_t* p;
    int64_t nbits;
    int64_t pos;
    bool bad;

    FLAC_HD uint32_t read(int k) {                               // 0 <= k <= 32
        if (k == 0) return 0;
        if (pos + k > nbits) {
            bad = true;
            pos = nbits;
            return 0;
        }
        const int64_t byte = pos >> 3;
        const int sh = (int)(pos & 7);
        const int need = (sh + k + 7) >> 3;                      // <= 5 bytes
        uint64_t w = 0;
        for (int i = 0; i < need; ++i) w = (w << 8) | p[byte + i];
        w <<= 8 * (8 - need) + sh;                               // left-align the first wanted bit
        pos += k;
        return (uint32_t)(w >> (64 - k));
    }
    FLAC_HD int32_t read_signed(int k) {
        if (k == 0) return 0;
        const uint32_t v = read(k);
        return (int32_t)(v << (32 - k)) >> (32 - k);
    }
    FLAC_HD uint32_t unary() {                                   // zeros before the next one bit
        uint32_t q = 0;
        while (true) {
            if (pos >= nbits) {
                bad = true;
                return 0;
            }
            const int sh = (int)(pos & 7);
            unsigned b = (unsigned)(uint8_t)(p[pos >> 3] << sh);
            if (b) {
                int z = 0;
                while (!(b & 0x80)) {
                    b <<= 1;
                    ++z;
                }
                pos += z + 1;
                return q + (uint32_t)z;
            }
            q += (uint32_t)(8 - sh);
            pos += 8 - sh;
        }
    }
};

// header codes 1-7 of the sample size and 1-11 of the sample rate
FLAC_HD int sample_size(int code) {
    switch (code) {
        case 1: return 8;
        case 2: return 12;
        case 4: return 16;
        case 5: return 20;
        case 6: return 24;
        case 7: return 32;
        default: return 0;
    }
}

FLAC_HD int table_rate(int code) {
    switch (code) {
        case 1: return 88200;
        case 2: return 176400;
        case 3: return 192000;
        case 4: return 8000;
        case 5: return 16000;
        case 6: return 22050;
        case 7: return 24000;
        case 8: return 32000;
        case 9: return 44100;
        case 10: return 48000;
        default: return 96000;
    }
}

// The frame header at buf[off], read only inside [buf, buf + n).  Returns true when every field is legal, agrees with
// STREAMINFO and the CRC-8 matches.
FLAC_HD bool parse_header(const uint8_t* buf, int64_t n, int64_t off, const StreamInfo& si, Header* h) {
    if (off < 0 || off + 6 > n) return false;                   // the shortest header is 6 bytes
    const uint8_t* p = buf + off;
    if (p[0] != 0xFF || (p[1] & 0xFE) != 0xF8) return false;    // 14-bit sync + reserved 0
    const int variable = p[1] & 1;
    const int bs_code = p[2] >> 4, rate_code = p[2] & 15;
    const int assignment = p[3] >> 4, size_code = (p[3] >> 1) & 7;
    if (bs_code == 0 || rate_code == 15 || assignment > 10 || size_code == 3 || (p[3] & 1)) return false;
    const int channels = assignment < 8 ? assignment + 1 : 2;
    if (channels != si.channels) return false;
    if (size_code != 0 && sample_size(size_code) != si.bps) return false;
    int64_t i = 4;
    // UTF-8-style coded number: up to 6 bytes (31 bits) for a frame number, 7 (36 bits) for a sample number
    const unsigned x = p[i++];
    int more;
    int64_t v;
    if (!(x & 0x80)) { v = x; more = 0; }
    else if ((x & 0xE0) == 0xC0) { v = x & 0x1F; more = 1; }
    else if ((x & 0xF0) == 0xE0) { v = x & 0x0F; more = 2; }
    else if ((x & 0xF8) == 0xF0) { v = x & 0x07; more = 3; }
    else if ((x & 0xFC) == 0xF8) { v = x & 0x03; more = 4; }
    else if ((x & 0xFE) == 0xFC) { v = x & 0x01; more = 5; }
    else if (x == 0xFE && variable) { v = 0; more = 6; }
    else return false;
    if (off + i + more + 1 > n) return false;
    for (int k = 0; k < more; ++k) {
        const unsigned y = p[i++];
        if ((y & 0xC0) != 0x80) return false;
        v = (v << 6) | (y & 0x3F);
    }
    int bs;
    if (bs_code == 1) bs = 192;
    else if (bs_code <= 5) bs = 576 << (bs_code - 2);
    else if (bs_code >= 8) bs = 256 << (bs_code - 8);
    else {
        const int extra = bs_code == 6 ? 1 : 2;
        if (off + i + extra + 1 > n) return false;
        bs = extra == 1 ? p[i] : (p[i] << 8) | p[i + 1];
        bs += 1;
        i += extra;
    }
    if (bs > 65535 || (si.max_block > 0 && bs > si.max_block)) return false;
    int rate = si.rate;
    if (rate_code >= 1 && rate_code <= 11) rate = table_rate(rate_code);
    else if (rate_code >= 12) {
        const int extra = rate_code == 12 ? 1 : 2;
        if (off + i + extra + 1 > n) return false;
        rate = extra == 1 ? p[i] * 1000 : ((p[i] << 8) | p[i + 1]) * (rate_code == 14 ? 10 : 1);
        i += extra;
    }
    if (rate != si.rate) return false;
    if (off + i + 1 > n || crc8(p, i) != p[i]) return false;
    h->number = v;
    h->block_size = bs;
    h->assignment = assignment;
    h->variable = variable;
    h->bytes = (int)(i + 1);
    return true;
}

FLAC_HD void put(int32_t* out, int64_t stride, int64_t i, int64_t v) {
    out[i * stride] = (int32_t)(uint32_t)(uint64_t)v;          // two's-complement wrap: a corrupt residual is no UB
}

// One subframe of `bs` samples at `sbps` bits into out[i * stride] (out == nullptr: parse only).  Returns 0 or a status.
FLAC_HD int decode_subframe(Bits& b, int bs, int sbps, int32_t* out, int64_t stride) {
    if (b.read(1) != 0) return b.bad ? kTruncated : kBadSubframe;
    const int type = (int)b.read(6);
    int wasted = 0;
    if (b.read(1)) {
        wasted = (int)b.unary() + 1;
        if (b.bad) return kTruncated;
        if (wasted >= sbps) return kBadSubframe;
        sbps -= wasted;
    }
    if (b.bad) return kTruncated;
    int order;
    bool lpc = false;
    if (type == 0) {                                             // CONSTANT
        const int32_t v = b.read_signed(sbps);
        if (b.bad) return kTruncated;
        if (out)
            for (int i = 0; i < bs; ++i) put(out, stride, i, (int64_t)v * ((int64_t)1 << wasted));
        return 0;
    } else if (type == 1) {                                      // VERBATIM
        for (int i = 0; i < bs; ++i) {
            const int32_t v = b.read_signed(sbps);
            if (b.bad) return kTruncated;
            if (out) put(out, stride, i, (int64_t)v * ((int64_t)1 << wasted));
        }
        return 0;
    } else if (type >= 8 && type <= 12) {
        order = type - 8;
    } else if (type >= 32) {
        order = type - 31;
        lpc = true;
    } else {
        return kBadSubframe;
    }
    if (order > bs) return kBadSubframe;
    for (int i = 0; i < order; ++i) {
        const int32_t v = b.read_signed(sbps);
        if (out) put(out, stride, i, v);
    }
    int precision = 0, shift = 0;
    int32_t coef[32];
    if (lpc) {
        precision = (int)b.read(4) + 1;
        shift = b.read_signed(5);
        if (b.bad) return kTruncated;
        if (precision == 16 || shift < 0) return kBadSubframe;
        for (int j = 0; j < order; ++j) coef[j] = b.read_signed(precision);
    }
    if (b.bad) return kTruncated;
    // residual: coding method 0 (4-bit Rice parameters, escape 15) or 1 (5-bit, escape 31)
    const int method = (int)b.read(2);
    const int porder = (int)b.read(4);
    if (b.bad) return kTruncated;
    if (method > 1 || (bs & ((1 << porder) - 1)) || (bs >> porder) < order) return kBadResidual;
    const int pbits = method ? 5 : 4, escape = method ? 31 : 15;
    int64_t i = order;
    for (int part = 0; part < (1 << porder); ++part) {
        const int64_t cnt = (bs >> porder) - (part == 0 ? order : 0);
        const int k = (int)b.read(pbits);
        if (k == escape) {
            const int nb = (int)b.read(5);
            for (int64_t j = 0; j < cnt; ++j, ++i) {
                const int32_t r = b.read_signed(nb);
                if (out) put(out, stride, i, r);
            }
        } else {
            for (int64_t j = 0; j < cnt; ++j, ++i) {
                const uint32_t q = b.unary();
                const uint32_t u = (q << k) | b.read(k);
                if (b.bad) return kTruncated;
                if (out) put(out, stride, i, (int32_t)((u >> 1) ^ (0u - (u & 1))));
            }
        }
        if (b.bad) return kTruncated;
    }
    if (!out) return 0;
    // prediction in place: out holds warm-up samples then residuals
    for (int64_t t = order; t < bs; ++t) {
        int64_t pred = 0;
        const int32_t* x = out + t * stride;
        if (lpc) {
            for (int j = 0; j < order; ++j) pred += (int64_t)coef[j] * x[-(j + 1) * stride];
            pred >>= shift;
        } else if (order == 1) {
            pred = x[-stride];
        } else if (order == 2) {
            pred = 2 * (int64_t)x[-stride] - x[-2 * stride];
        } else if (order == 3) {
            pred = 3 * (int64_t)x[-stride] - 3 * (int64_t)x[-2 * stride] + x[-3 * stride];
        } else if (order == 4) {
            pred = 4 * (int64_t)x[-stride] - 6 * (int64_t)x[-2 * stride] + 4 * (int64_t)x[-3 * stride] - x[-4 * stride];
        }
        put(out, stride, t, (int64_t)x[0] + pred);
    }
    if (wasted)
        for (int t = 0; t < bs; ++t) put(out, stride, t, (int64_t)out[t * stride] * ((int64_t)1 << wasted));
    return 0;
}

// The whole frame at buf[off] whose header `h` parse_header gave.  out == nullptr: parse and check only; otherwise `out`
// points at the frame's first row of an int32 [n][channels] array.  Returns the offset past the CRC-16, or a status.
FLAC_HD int64_t decode_frame(const uint8_t* buf, int64_t n, int64_t off, const StreamInfo& si, const Header& h,
                             int32_t* out) {
    Bits b{buf, n * 8, (off + h.bytes) * 8, false};
    const int C = si.channels;
    for (int c = 0; c < C; ++c) {
        const bool side = (h.assignment == 8 && c == 1) || (h.assignment == 9 && c == 0) || (h.assignment == 10 && c == 1);
        const int st = decode_subframe(b, h.block_size, si.bps + (side ? 1 : 0), out ? out + c : nullptr, C);
        if (st) return st;
    }
    const int64_t end = (b.pos + 7) >> 3;                        // zero padding to the byte boundary
    if (end + 2 > n) return kTruncated;
    if (crc16(buf + off, end - off) != (uint16_t)((buf[end] << 8) | buf[end + 1])) return kBadCrc16;
    if (out && h.assignment >= 8) {
        for (int t = 0; t < h.block_size; ++t) {
            int32_t* r = out + (int64_t)t * C;
            const int64_t a = r[0], s = r[1];
            if (h.assignment == 8) {                             // left, side = left - right
                put(r, 1, 1, a - s);
            } else if (h.assignment == 9) {                      // side, right
                put(r, 1, 0, a + s);
            } else {                                             // mid, side
                const int64_t m = a * 2 + (s & 1);
                put(r, 1, 0, (m + s) >> 1);
                put(r, 1, 1, (m - s) >> 1);
            }
        }
    }
    return end + 2;
}

}  // namespace flac
}  // namespace wun
