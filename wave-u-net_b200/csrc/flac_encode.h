// flac_encode.h - the FLAC frame encoder, shared by the CUDA kernels (kernels_flac_encode.cu) and a host build the CPU tests
// run under AddressSanitizer and UBSan (tests/flacenc/flac_encode_host.cpp).  Like flac_frame.h it is plain C++ on integers
// and doubles; the only difference between the builds is the `Team` the cooperative functions take:
//
//   a CUDA block    tid() = threadIdx.x, n() = blockDim.x (a power of two <= kThreads), sync() = __syncthreads(), word ORs
//                   and shared counters atomic;
//   Serial (below)  one lane doing every lane's work in order, sync() a no-op.
//
// Every cooperative step is a loop `for (i = tid; i < count; i += n)` whose iterations are independent, followed by sync(),
// or a step only lane 0 runs; no lane keeps state in registers across a sync().  So the serial build runs the same
// arithmetic, and the output never depends on how the lanes are scheduled: integer sums are exact, double sums are reduced
// in a fixed tree, and bits land through disjoint ORs into a zeroed buffer.
//
// Per frame (DESIGN.md §4.11):
//   analyse_signal  one signal of one frame (a channel, or for stereo also side = L - R and mid = (L + R) >> 1): wasted bits,
//                   CONSTANT, VERBATIM, FIXED 0-4 and LPC 1..max order (Tukey(0.5) window, autocorrelation, Levinson-Durbin,
//                   15-bit quantised coefficients), each residual computed exactly in 64 bits and priced exactly with the
//                   best Rice parameter per partition over every legal partition order and both coding methods; a predictor
//                   whose residual leaves int32 is rejected.  Writes the cheapest choice and its exact bit count.
//   decide_frame    the channel assignment (stereo: independent, left/side, right/side, mid/side by exact bits) and the frame's
//                   byte size (header, subframes, zero padding, CRC-16).
//   pack_frame      header (sync, codes, UTF-8 frame number, CRC-8), subframes with per-chunk bit offsets from a scan, CRC-16.
#pragma once
#include <math.h>
#include <stdint.h>

#include "flac_frame.h"

namespace wun {
namespace flac {

constexpr int kThreads = 256;          // lanes of a device team (power of two)
constexpr int kMaxBlock = 4608;        // streamable subset at <= 48 kHz
constexpr int kMaxLpc = 32;
constexpr int kMaxPorder = 8;          // streamable subset
constexpr int kMaxParts = 1 << kMaxPorder;
constexpr int kRiceParams = 31;        // Rice parameters 0..30 (method 1; method 0 stops at 14)
constexpr int kPrecision = 15;         // quantised LPC coefficient precision
constexpr int kMaxHeader = 16;         // frame header bytes including the CRC-8

enum SubType : int32_t { kConstant = 0, kVerbatim = 1, kFixed = 2, kLpc = 3 };

// The encoder's choice for one signal of one frame.
struct SubChoice {
    int64_t bits;                      // exact subframe size
    int32_t type, order, wasted, shift;
    int32_t method, porder;            // residual coding method (0: 4-bit parameters, 1: 5-bit) and partition order
    int32_t value;                     // CONSTANT's sample
    int32_t range_error;               // a sample outside the stream's bits per sample (input signals only)
    int32_t coef[kMaxLpc];
    uint8_t rice[kMaxParts];           // Rice parameter per partition
};

struct FrameChoice {
    int64_t bytes;                     // whole frame including the CRC-16
    int32_t assignment;                // FLAC channel assignment 0-10
    int32_t header_bytes;
};

// float -> integer at `bps` bits: clamp(rint(x * 2^(bps-1)), -2^(bps-1), 2^(bps-1) - 1), ties to even, NaN -> 0.  The
// product is exact in float32, so this inverts the read rule x = s / 2^(bps-1).
FLAC_HD int32_t quantise(float x, int bps) {
    if (x != x) return 0;
    const float hi = (float)((1 << (bps - 1)) - 1), lo = -(float)(1 << (bps - 1));
    float v = rintf(x * (float)(1 << (bps - 1)));
    v = v < lo ? lo : (v > hi ? hi : v);
    return (int32_t)v;
}

FLAC_HD int signals_of(int C) { return C == 2 ? 4 : C; }     // stereo: L, R, side, mid
FLAC_HD int signal_bps(int s, int C, int bps) { return C == 2 && s == 2 ? bps + 1 : bps; }
FLAC_HD int max_lpc_order(int rate) { return rate <= 48000 ? 12 : 32; }

// sample t of signal s from interleaved int32 [n][C] samples (frame-relative pointer)
FLAC_HD int32_t signal_sample(const int32_t* x, int C, int s, int t) {
    if (C != 2 || s < 2) return x[(int64_t)t * C + s];
    const int64_t l = x[(int64_t)t * 2], r = x[(int64_t)t * 2 + 1];
    return (int32_t)(s == 2 ? l - r : (l + r) >> 1);
}

// the frame's channel -> signal for a channel assignment
FLAC_HD int channel_signal(int assignment, int c) {
    if (assignment < 8) return c;
    if (assignment == 8) return c == 0 ? 0 : 2;
    if (assignment == 9) return c == 0 ? 2 : 1;
    return c == 0 ? 3 : 2;
}

// header codes: 0 when the value has no code of its own
FLAC_HD int size_code(int bps) {
    switch (bps) {
        case 8: return 1;
        case 12: return 2;
        case 16: return 4;
        case 20: return 5;
        case 24: return 6;
        default: return 0;
    }
}

// rate code and the bytes it appends; -1 when a frame header cannot express the rate
FLAC_HD int rate_code(int rate, int* extra) {
    *extra = 0;
    for (int c = 1; c <= 11; ++c)
        if (table_rate(c) == rate) return c;
    if (rate % 1000 == 0 && rate / 1000 <= 255) { *extra = 1; return 12; }
    if (rate <= 65535) { *extra = 2; return 13; }
    if (rate % 10 == 0 && rate / 10 <= 65535) { *extra = 2; return 14; }
    return -1;
}

FLAC_HD int block_code(int bs, int* extra) {
    *extra = 0;
    if (bs == 192) return 1;
    for (int k = 0; k < 4; ++k)
        if (bs == 576 << k) return 2 + k;
    for (int k = 0; k < 8; ++k)
        if (bs == 256 << k) return 8 + k;
    if (bs <= 256) { *extra = 1; return 6; }
    *extra = 2;
    return 7;
}

// The frame header of frame `number` into h[0..kMaxHeader); returns its length including the CRC-8.
FLAC_HD int write_header(uint8_t* h, int64_t number, int bs, int rate, int assignment, int bps) {
    int bs_extra, rate_extra;
    const int bc = block_code(bs, &bs_extra), rc = rate_code(rate, &rate_extra);
    int i = 0;
    h[i++] = 0xFF;
    h[i++] = 0xF8;                                          // fixed blocking
    h[i++] = (uint8_t)(bc << 4 | rc);
    h[i++] = (uint8_t)(assignment << 4 | size_code(bps) << 1);
    const uint64_t v = (uint64_t)number;                    // UTF-8-style coding, up to 31 bits
    if (v < 0x80) {
        h[i++] = (uint8_t)v;
    } else {
        int more = v < 0x800 ? 1 : v < 0x10000 ? 2 : v < 0x200000 ? 3 : v < 0x4000000 ? 4 : 5;
        h[i++] = (uint8_t)((0xFF80u >> more) & 0xFF) | (uint8_t)(v >> (6 * more));
        for (int k = more - 1; k >= 0; --k) h[i++] = (uint8_t)(0x80 | ((v >> (6 * k)) & 0x3F));
    }
    if (bs_extra == 1) h[i++] = (uint8_t)(bs - 1);
    if (bs_extra == 2) { h[i++] = (uint8_t)((bs - 1) >> 8); h[i++] = (uint8_t)(bs - 1); }
    const int rv = rc == 12 ? rate / 1000 : rc == 14 ? rate / 10 : rate;
    if (rate_extra == 1) h[i++] = (uint8_t)rv;
    if (rate_extra == 2) { h[i++] = (uint8_t)(rv >> 8); h[i++] = (uint8_t)rv; }
    h[i] = crc8(h, i);
    return i + 1;
}

// Largest frame the encoder can write: VERBATIM subframes at the stream's depth always compete, so no frame exceeds this.
FLAC_HD int64_t frame_bound(int bs, int C, int bps) {
    return kMaxHeader + ((int64_t)C * (8 + (int64_t)bs * bps) + 7) / 8 + 2;
}

FLAC_HD uint32_t zigzag(int64_t r) { return (uint32_t)(r < 0 ? ((uint64_t)(-r) << 1) - 1 : (uint64_t)r << 1); }

// residual of sample t (>= order) of x for a FIXED (type kFixed) or LPC predictor, exact in 64 bits
FLAC_HD int64_t residual(const int32_t* x, int t, int type, int order, const int32_t* coef, int shift) {
    int64_t pred = 0;
    if (type == kLpc) {
        for (int j = 0; j < order; ++j) pred += (int64_t)coef[j] * x[t - 1 - j];
        pred >>= shift;
    } else if (order == 1) {
        pred = x[t - 1];
    } else if (order == 2) {
        pred = 2 * (int64_t)x[t - 1] - x[t - 2];
    } else if (order == 3) {
        pred = 3 * (int64_t)x[t - 1] - 3 * (int64_t)x[t - 2] + x[t - 3];
    } else if (order == 4) {
        pred = 4 * (int64_t)x[t - 1] - 6 * (int64_t)x[t - 2] + 4 * (int64_t)x[t - 3] - x[t - 4];
    }
    return (int64_t)x[t] - pred;
}

// largest partition order <= 8 that divides the block and leaves the first partition room for the warm-up samples
FLAC_HD int max_porder(int bs, int order) {
    int p = 0;
    while (p < kMaxPorder && (bs & ((2 << p) - 1)) == 0 && (bs >> (p + 1)) >= order) ++p;
    return p;
}

// Scratch memory of one team (a CUDA block's shared memory; one heap object in the serial build).
struct Scratch {
    int32_t x[kMaxBlock];                                  // the signal, wasted bits removed
    union {
        double xw[kMaxBlock];                              // windowed signal (LPC analysis)
        uint64_t sums[kRiceParams][kMaxParts];             // sum of (u >> k) per partition (Rice pricing)
        int64_t chunk_bits[kThreads + 1];                  // residual chunk sizes (packing)
    } u;
    double red[kThreads];
    double autoc[kMaxLpc + 1];
    double lpc[kMaxLpc][kMaxLpc];                          // lpc[m - 1][j]: order-m predictor
    uint64_t cost[2][kMaxPorder + 1];                      // residual bits per method and partition order
    uint8_t rice[2][2 * kMaxParts];                        // best parameter per method, level p at offset 2^p - 1
    SubChoice cand, best;
    int32_t or_bits, differs, overflow, range_error, lpc_orders;
    uint8_t header[kMaxHeader];
    int64_t sub_start, residual_start;
};

struct Serial {
    int tid() const { return 0; }
    int n() const { return 1; }
    void sync() const {}
    void add(uint64_t* p, uint64_t v) const { *p += v; }
    void or_flag(int32_t* p, int32_t v) const { *p |= v; }
    void or_word(uint32_t* w, uint32_t v) const { *w |= v; }
    uint32_t load_word(const uint32_t* w) const { return *w; }
};

// sum over lanes of one double per lane, reduced in a fixed tree (the same bits on every run)
template <class Team>
FLAC_HD double team_sum(const Team& tm, Scratch& s, double v) {
    s.red[tm.tid()] = v;
    tm.sync();
    for (int h = tm.n() / 2; h > 0; h >>= 1) {
        if (tm.tid() < h) s.red[tm.tid()] += s.red[tm.tid() + h];
        tm.sync();
    }
    const double r = s.red[0];
    tm.sync();
    return r;
}

// Price candidate s.cand (FIXED or LPC, order and coefficients set) on signal s.x[0..bs): exact residual bits with the best
// Rice parameters over every legal partition order and both methods.  Sets s.cand.bits (INT64_MAX when the residual leaves
// int32), method, porder and rice[].
template <class Team>
FLAC_HD void price_candidate(const Team& tm, Scratch& s, int bs, int sbps, int head_bits) {
    SubChoice& c = s.cand;
    const int P = max_porder(bs, c.order);
    const int parts = 1 << P, psize = bs >> P;
    if (tm.tid() == 0) {
        s.overflow = 0;
        for (int m = 0; m < 2; ++m)
            for (int p = 0; p <= kMaxPorder; ++p) s.cost[m][p] = 0;
    }
    tm.sync();
    for (int j = tm.tid(); j < parts; j += tm.n()) {
        uint64_t acc[kRiceParams];
        for (int k = 0; k < kRiceParams; ++k) acc[k] = 0;
        int bad = 0;
        for (int t = j == 0 ? c.order : j * psize; t < (j + 1) * psize; ++t) {
            const int64_t r = residual(s.x, t, c.type, c.order, c.coef, c.shift);
            if (r < INT32_MIN || r > INT32_MAX) bad = 1;
            const uint32_t u = zigzag(r);
            for (int k = 0; k < kRiceParams; ++k) acc[k] += u >> k;
        }
        for (int k = 0; k < kRiceParams; ++k) s.u.sums[k][j] = acc[k];
        if (bad) tm.or_flag(&s.overflow, 1);
    }
    tm.sync();
    if (s.overflow) {
        if (tm.tid() == 0) c.bits = INT64_MAX;
        tm.sync();
        return;
    }
    for (int p = P; p >= 0; --p) {
        const int step = 1 << (P - p);                       // finest partitions per partition of this level
        for (int j = tm.tid(); j < (1 << p); j += tm.n()) {
            const int64_t cnt = (int64_t)(bs >> p) - (j == 0 ? c.order : 0);
            for (int m = 0; m < 2; ++m) {
                const int kmax = m ? 30 : 14;
                uint64_t best = UINT64_MAX;
                int bk = 0;
                for (int k = 0; k <= kmax; ++k) {
                    const uint64_t cost = (uint64_t)cnt * (uint64_t)(k + 1) + s.u.sums[k][j * step];
                    if (cost < best) { best = cost; bk = k; }
                }
                s.rice[m][(1 << p) - 1 + j] = (uint8_t)bk;
                tm.add(&s.cost[m][p], best + (m ? 5 : 4));
            }
        }
        tm.sync();
        if (p > 0) {                                         // merge pairs into the next coarser level, in place
            const int pairs = 1 << (p - 1);
            for (int i = tm.tid(); i < pairs * kRiceParams; i += tm.n()) {
                const int k = i / pairs, j = i % pairs;
                s.u.sums[k][2 * j * step] += s.u.sums[k][(2 * j + 1) * step];
            }
            tm.sync();
        }
    }
    if (tm.tid() == 0) {
        uint64_t best = UINT64_MAX;
        for (int p = 0; p <= P; ++p)
            for (int m = 0; m < 2; ++m)
                if (s.cost[m][p] < best) { best = s.cost[m][p]; c.method = m; c.porder = p; }
        for (int j = 0; j < (1 << c.porder); ++j) c.rice[j] = s.rice[c.method][(1 << c.porder) - 1 + j];
        int64_t bits = head_bits + (int64_t)c.order * sbps + 6 + (int64_t)best;
        if (c.type == kLpc) bits += 4 + 5 + (int64_t)c.order * kPrecision;
        c.bits = bits;
    }
    tm.sync();
}

// keep s.cand when it is strictly cheaper than s.best (lane 0; candidates are tried in a fixed order)
template <class Team>
FLAC_HD void keep_if_better(const Team& tm, Scratch& s) {
    if (tm.tid() == 0 && s.cand.bits < s.best.bits) s.best = s.cand;
    tm.sync();
}

// Quantise the order-m predictor s.lpc[m - 1] to kPrecision bits into s.cand (libFLAC's rule: shift from the largest
// coefficient, rounding with error feedback).  Returns false when the coefficients need a negative shift.
FLAC_HD bool quantise_lpc(Scratch& s, int m) {
    const double* a = s.lpc[m - 1];
    double cmax = 0;
    for (int j = 0; j < m; ++j) cmax = fabs(a[j]) > cmax ? fabs(a[j]) : cmax;
    if (!(cmax > 0)) return false;
    int e;
    frexp(cmax, &e);                                        // cmax = f * 2^e, 0.5 <= f < 1
    int shift = (kPrecision - 1) - e;
    if (shift > 15) shift = 15;
    if (shift < 0) return false;
    const int32_t qmax = (1 << (kPrecision - 1)) - 1, qmin = -(1 << (kPrecision - 1));
    double err = 0;
    for (int j = 0; j < m; ++j) {
        err += a[j] * (double)(1 << shift);
        double q = floor(err + 0.5);
        q = q > qmax ? qmax : (q < qmin ? qmin : q);
        s.cand.coef[j] = (int32_t)q;
        err -= q;
    }
    s.cand.shift = shift;
    return true;
}

// The cheapest subframe for signal `sig` of the frame at x (interleaved int32, `bs` rows of C channels).  Writes *out.
template <class Team>
FLAC_HD void analyse_signal(const Team& tm, Scratch& s, const int32_t* x, int C, int sig, int bs, int bps, int rate,
                            SubChoice* out) {
    const int sbps0 = signal_bps(sig, C, bps);
    if (tm.tid() == 0) { s.or_bits = 0; s.differs = 0; s.range_error = 0; }
    tm.sync();
    int32_t orv = 0, diff = 0, range = 0;
    const int32_t lo = -(1 << (bps - 1)), hi = (1 << (bps - 1)) - 1;
    const int32_t first = signal_sample(x, C, sig, 0);
    for (int t = tm.tid(); t < bs; t += tm.n()) {
        const int32_t v = signal_sample(x, C, sig, t);
        s.x[t] = v;
        orv |= v;
        diff |= v != first;
        if (sig < C && (v < lo || v > hi)) range = 1;
    }
    tm.or_flag(&s.or_bits, orv);
    tm.or_flag(&s.differs, diff);
    tm.or_flag(&s.range_error, range);
    tm.sync();
    if (!s.differs || s.range_error) {                       // CONSTANT (a range error makes the frame unusable anyway)
        if (tm.tid() == 0) {
            SubChoice& b = s.best;
            b.type = kConstant;
            b.value = first;
            b.bits = 8 + sbps0;
            b.order = b.wasted = b.shift = b.method = b.porder = 0;
            b.range_error = s.range_error;
            *out = b;
        }
        tm.sync();
        return;
    }
    int wasted = 0;
    while (!((s.or_bits >> wasted) & 1)) ++wasted;
    const int sbps = sbps0 - wasted;
    const int head = 8 + wasted;
    if (wasted)
        for (int t = tm.tid(); t < bs; t += tm.n()) s.x[t] >>= wasted;
    if (tm.tid() == 0) {
        SubChoice& b = s.best;
        b.type = kVerbatim;
        b.bits = head + (int64_t)bs * sbps;
        b.order = b.shift = b.method = b.porder = 0;
        s.cand = b;
    }
    tm.sync();
    for (int order = 0; order <= 4 && order <= bs; ++order) {
        if (tm.tid() == 0) { s.cand.type = kFixed; s.cand.order = order; s.cand.shift = 0; }
        tm.sync();
        price_candidate(tm, s, bs, sbps, head);
        keep_if_better(tm, s);
    }
    const int max_order = bs - 1 < max_lpc_order(rate) ? bs - 1 : max_lpc_order(rate);
    if (max_order >= 1) {
        // Tukey(0.5) window and autocorrelation
        const int edge = bs / 4;
        for (int t = tm.tid(); t < bs; t += tm.n()) {
            double w = 1.0;
            if (edge > 0 && t < edge) w = 0.5 - 0.5 * cos(3.141592653589793 * t / edge);
            else if (edge > 0 && t >= bs - edge) w = 0.5 - 0.5 * cos(3.141592653589793 * (bs - 1 - t) / edge);
            s.u.xw[t] = w * s.x[t];
        }
        tm.sync();
        for (int lag = 0; lag <= max_order; ++lag) {
            double acc = 0;
            for (int t = lag + tm.tid(); t < bs; t += tm.n()) acc += s.u.xw[t] * s.u.xw[t - lag];
            const double r = team_sum(tm, s, acc);
            if (tm.tid() == 0) s.autoc[lag] = r;
        }
        tm.sync();
        if (tm.tid() == 0) {                                 // Levinson-Durbin: predictors of every order up to max_order
            const double* R = s.autoc;
            double a[kMaxLpc], err = R[0];
            int orders = 0;
            for (int m = 1; m <= max_order && err > 0; ++m) {
                double k = R[m];
                for (int j = 0; j < m - 1; ++j) k -= a[j] * R[m - 1 - j];
                k /= err;
                double na[kMaxLpc];
                for (int j = 0; j < m - 1; ++j) na[j] = a[j] - k * a[m - 2 - j];
                na[m - 1] = k;
                for (int j = 0; j < m; ++j) a[j] = s.lpc[m - 1][j] = na[j];
                err *= 1 - k * k;
                orders = m;
            }
            s.lpc_orders = orders;
        }
        tm.sync();
        for (int m = 1; m <= s.lpc_orders; ++m) {
            if (tm.tid() == 0) {
                s.cand.type = kLpc;
                s.cand.order = m;
                s.differs = quantise_lpc(s, m);              // reused as the "usable" flag
            }
            tm.sync();
            const int usable = s.differs;
            tm.sync();
            if (!usable) continue;
            price_candidate(tm, s, bs, sbps, head);
            keep_if_better(tm, s);
        }
    }
    if (tm.tid() == 0) {
        s.best.wasted = wasted;
        s.best.range_error = 0;
        *out = s.best;
    }
    tm.sync();
}

// Channel assignment and byte size of frame `number` from its signals' choices (sub[signal]).
FLAC_HD FrameChoice decide_frame(const SubChoice* sub, int C, int bs, int bps, int rate, int64_t number) {
    FrameChoice f;
    int64_t bits;
    if (C == 2) {
        const int64_t modes[4] = {sub[0].bits + sub[1].bits, sub[0].bits + sub[2].bits, sub[2].bits + sub[1].bits,
                                  sub[3].bits + sub[2].bits};
        int m = 0;
        for (int i = 1; i < 4; ++i)
            if (modes[i] < modes[m]) m = i;
        f.assignment = m == 0 ? 1 : 7 + m;
        bits = modes[m];
    } else {
        f.assignment = C - 1;
        bits = 0;
        for (int c = 0; c < C; ++c) bits += sub[c].bits;
    }
    uint8_t h[kMaxHeader];
    f.header_bytes = write_header(h, number, bs, rate, f.assignment, bps);
    f.bytes = f.header_bytes + (bits + 7) / 8 + 2;
    return f;
}

// MSB-first bit writer into a zeroed buffer of 32-bit words (byte order as in memory), one team lane at absolute bit `pos`.
// Whole words go out through Team::or_word, so lanes writing neighbouring bit ranges never lose each other's bits.
template <class Team>
struct BitSink {
    const Team& tm;
    uint32_t* words;
    int64_t pos;
    uint32_t cur;                                            // pending bits of word pos >> 5, big-endian within the word

    FLAC_HD static uint32_t bswap(uint32_t v) {
        return (v >> 24) | ((v >> 8) & 0xFF00u) | ((v << 8) & 0xFF0000u) | (v << 24);
    }
    FLAC_HD void flush() {
        if (cur) tm.or_word(words + (pos >> 5), bswap(cur));
        cur = 0;
    }
    FLAC_HD void put(uint32_t v, int k) {                    // the low k bits of v, 0 <= k <= 32
        while (k > 0) {
            const int off = (int)(pos & 31), take = k < 32 - off ? k : 32 - off;
            const uint32_t bits = (uint32_t)(((uint64_t)v >> (k - take)) & ((1ull << take) - 1));
            cur |= (uint32_t)((uint64_t)bits << (32 - off - take));
            k -= take;
            if (off + take == 32) flush();
            pos += take;
        }
    }
    FLAC_HD void put_signed(int64_t v, int k) { put((uint32_t)(uint64_t)v & (uint32_t)((1ull << k) - 1), k); }
    FLAC_HD void skip(int64_t k) {                           // k zero bits
        if (k <= 0) return;
        if ((pos & 31) + k >= 32) flush();
        pos += k;
    }
};

// residual bits of sample t given its partition's Rice parameter
FLAC_HD int64_t rice_bits(uint32_t u, int k) { return (int64_t)(u >> k) + 1 + k; }

// Write the frame whose samples start at x (interleaved int32 rows), choices sub[signal] and frame choice f at byte `offset`
// of the zeroed word buffer.  All lanes of the team take part.
template <class Team>
FLAC_HD void pack_frame(const Team& tm, Scratch& s, const int32_t* x, int C, int bs, int bps, int rate, int64_t number,
                        const SubChoice* sub, const FrameChoice& f, uint32_t* words, int64_t offset) {
    if (tm.tid() == 0) {
        const int hb = write_header(s.header, number, bs, rate, f.assignment, bps);
        BitSink<Team> w{tm, words, offset * 8, 0};
        for (int i = 0; i < hb; ++i) w.put(s.header[i], 8);
        w.flush();
        s.sub_start = offset * 8 + hb * 8;
    }
    tm.sync();
    for (int c = 0; c < C; ++c) {
        const int sig = channel_signal(f.assignment, c);
        const SubChoice& ch = sub[sig];
        const int sbps = signal_bps(sig, C, bps) - ch.wasted;       // CONSTANT subframes have no wasted bits
        for (int t = tm.tid(); t < bs; t += tm.n()) s.x[t] = signal_sample(x, C, sig, t) >> ch.wasted;
        tm.sync();
        if (tm.tid() == 0) {                                 // subframe header, warm-up, LPC parameters, residual preamble
            BitSink<Team> w{tm, words, s.sub_start, 0};
            const int type = ch.type == kConstant ? 0 : ch.type == kVerbatim ? 1 : ch.type == kFixed ? 8 + ch.order : 31 + ch.order;
            w.put((uint32_t)type << 1 | (ch.wasted ? 1 : 0), 8);
            if (ch.wasted) {
                w.skip(ch.wasted - 1);
                w.put(1, 1);
            }
            if (ch.type == kConstant) {
                w.put_signed(ch.value, sbps);
            } else if (ch.type == kVerbatim) {
                for (int t = 0; t < bs; ++t) w.put_signed(s.x[t], sbps);
            } else {
                for (int t = 0; t < ch.order; ++t) w.put_signed(s.x[t], sbps);
                if (ch.type == kLpc) {
                    w.put(kPrecision - 1, 4);
                    w.put_signed(ch.shift, 5);
                    for (int j = 0; j < ch.order; ++j) w.put_signed(ch.coef[j], kPrecision);
                }
                w.put((uint32_t)ch.method, 2);
                w.put((uint32_t)ch.porder, 4);
                w.put(ch.rice[0], ch.method ? 5 : 4);
            }
            w.flush();
            s.residual_start = w.pos;
        }
        tm.sync();
        if (ch.type == kFixed || ch.type == kLpc) {
            // contiguous chunks of residual samples, one per lane; a chunk carries the parameter of each partition it starts
            const int n = tm.n(), len = (bs + n - 1) / n, psize = bs >> ch.porder, pbits = ch.method ? 5 : 4;
            for (int i = tm.tid(); i < n; i += n) {
                int64_t bits = 0;
                const int a = i * len > ch.order ? i * len : ch.order, b = (i + 1) * len < bs ? (i + 1) * len : bs;
                for (int t = a; t < b; ++t) {
                    if (t % psize == 0 && t > 0) bits += pbits;
                    bits += rice_bits(zigzag(residual(s.x, t, ch.type, ch.order, ch.coef, ch.shift)), ch.rice[t / psize]);
                }
                s.u.chunk_bits[i] = bits;
            }
            tm.sync();
            if (tm.tid() == 0) {                             // exclusive scan of the chunk sizes
                int64_t acc = s.residual_start;
                for (int i = 0; i < n; ++i) {
                    const int64_t b = s.u.chunk_bits[i];
                    s.u.chunk_bits[i] = acc;
                    acc += b;
                }
                s.u.chunk_bits[n] = acc;
            }
            tm.sync();
            for (int i = tm.tid(); i < n; i += n) {
                const int a = i * len > ch.order ? i * len : ch.order, b = (i + 1) * len < bs ? (i + 1) * len : bs;
                BitSink<Team> w{tm, words, s.u.chunk_bits[i], 0};
                for (int t = a; t < b; ++t) {
                    if (t % psize == 0 && t > 0) w.put(ch.rice[t / psize], pbits);
                    const uint32_t u = zigzag(residual(s.x, t, ch.type, ch.order, ch.coef, ch.shift));
                    const int k = ch.rice[t / psize];
                    w.skip((int64_t)(u >> k));
                    w.put(1, 1);
                    w.put(u & (uint32_t)((1ull << k) - 1), k);
                }
                w.flush();
            }
            tm.sync();
            if (tm.tid() == 0) s.sub_start = s.u.chunk_bits[n];
        } else if (tm.tid() == 0) {
            s.sub_start = s.residual_start;
        }
        tm.sync();
    }
    // zero padding to the byte boundary is already there; the CRC-16 covers the frame up to it
    if (tm.tid() == 0) {
        const int64_t end = (s.sub_start + 7) >> 3;
        unsigned crc = 0;
        for (int64_t i = offset; i < end; ++i) {
            const uint32_t word = tm.load_word(words + (i >> 2));
            crc ^= ((word >> (8 * (i & 3))) & 0xFF) << 8;
            for (int b = 0; b < 8; ++b) crc = (crc & 0x8000) ? ((crc << 1) ^ 0x8005) & 0xffff : (crc << 1) & 0xffff;
        }
        BitSink<Team> w{tm, words, end * 8, 0};
        w.put(crc, 16);
        w.flush();
    }
    tm.sync();
}

}  // namespace flac
}  // namespace wun
