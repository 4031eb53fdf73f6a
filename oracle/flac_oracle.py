"""FLAC restated in plain Python / numpy: a decoder that follows the format frame by frame, and a writer that can emit every
feature the GPU decoder handles (csrc/flac_frame.h, DESIGN.md §4.10), including those FFmpeg's encoder never writes: escaped
partitions, variable block size, explicit rate / block-size header bytes, wasted bits, CONSTANT and VERBATIM subframes and
5-bit Rice parameters.

decode(data)              -> (info dict, int64 samples [n, C] at full depth); raises ValueError on any malformed stream.
write(samples, rate, bps, ...) -> bytes of a FLAC stream holding `samples` (int [n, C]), with the STREAMINFO MD5.
signal(seed, n, C, bps)   a seeded music-like test signal: tones, a glide and noise, clipped to bps.

The writer is vectorised per frame (residuals, Rice codes and bit packing in numpy, CRC-16 across all frames at once), so a
3-minute stereo stream takes seconds.  The decoder is a straightforward bit-string walk meant for short fixtures.
"""
import hashlib

import numpy as np

RATES = {88200: 1, 176400: 2, 192000: 3, 8000: 4, 16000: 5, 22050: 6, 24000: 7, 32000: 8, 44100: 9, 48000: 10, 96000: 11}
SIZES = {8: 1, 12: 2, 16: 4, 20: 5, 24: 6}
FIXED = [[], [1], [2, -1], [3, -3, 1], [4, -6, 4, -1]]
MODES = {"independent": None, "left_side": 8, "right_side": 9, "mid_side": 10}


def _crc8(data):
    c = 0
    for b in data:
        c ^= b
        for _ in range(8):
            c = ((c << 1) ^ 0x07) & 0xFF if c & 0x80 else (c << 1) & 0xFF
    return c


def _crc16_table():
    t = np.zeros(256, np.uint32)
    for i in range(256):
        c = i << 8
        for _ in range(8):
            c = ((c << 1) ^ 0x8005) & 0xFFFF if c & 0x8000 else (c << 1) & 0xFFFF
        t[i] = c
    return t


CRC16 = _crc16_table()


def crc16(data):
    c = 0
    for b in data:
        c = ((c << 8) & 0xFFFF) ^ int(CRC16[(c >> 8) ^ b])
    return c


def crc16_many(frames):
    """CRC-16 of every bytes object in `frames` at once: zero-init CRCs ignore leading zero bytes, so the frames are
    right-aligned in one matrix and run through the table column by column."""
    L = max(len(f) for f in frames)
    m = np.zeros((len(frames), L), np.uint32)
    for i, f in enumerate(frames):
        m[i, L - len(f):] = np.frombuffer(f, np.uint8)
    c = np.zeros(len(frames), np.uint32)
    for j in range(L):
        c = ((c << 8) & 0xFFFF) ^ CRC16[(c >> 8) ^ m[:, j]]
    return [int(v) for v in c]


def md5(samples, bps):
    nb = (bps + 7) // 8
    a = np.ascontiguousarray(np.asarray(samples, np.int64).astype("<i4").view(np.uint8).reshape(-1, 4)[:, :nb])
    return hashlib.md5(a.tobytes()).digest()


# --------------------------------------------------------------------------------------------------------------- decoder
class _Bits:
    def __init__(self, s, pos):
        self.s = s                 # the stream as a string of '0' / '1'
        self.pos = pos * 8

    def u(self, k):
        if k == 0:
            return 0
        if self.pos + k > len(self.s):
            raise ValueError("truncated")
        v = int(self.s[self.pos:self.pos + k], 2)
        self.pos += k
        return v

    def s_(self, k):
        v = self.u(k)
        return v - (1 << k) if k and v >> (k - 1) else v

    def unary(self):
        j = self.s.find("1", self.pos)
        if j < 0:
            raise ValueError("truncated")
        q = j - self.pos
        self.pos = j + 1
        return q


def _utf8(data, i, variable):
    x = data[i]
    for more, mask in ((0, 0x80), (1, 0xE0), (2, 0xF0), (3, 0xF8), (4, 0xFC), (5, 0xFE)):
        if (x & mask) == ((mask << 1) & 0xFF):
            break
    else:
        if x == 0xFE and variable:
            more, mask = 6, 0xFF
        else:
            raise ValueError("bad coded number")
    v = x & ((1 << (6 - more)) - 1 if more else 0x7F)
    for k in range(more):
        y = data[i + 1 + k]
        if y & 0xC0 != 0x80:
            raise ValueError("bad coded number")
        v = (v << 6) | (y & 0x3F)
    return v, i + 1 + more


def parse_metadata(data):
    pos = 0
    if data[:3] == b"ID3":
        size = 0
        for b in data[6:10]:
            size = (size << 7) | b
        pos = 10 + size + (10 if data[5] & 0x10 else 0)
    if data[pos:pos + 4] != b"fLaC":
        raise ValueError("no fLaC marker")
    pos += 4
    info, last = None, False
    while not last:
        last, kind, length = data[pos] >> 7, data[pos] & 0x7F, int.from_bytes(data[pos + 1:pos + 4], "big")
        body = data[pos + 4:pos + 4 + length]
        if kind == 0:
            v = int.from_bytes(body[10:18], "big")
            info = dict(min_block=int.from_bytes(body[0:2], "big"), max_block=int.from_bytes(body[2:4], "big"),
                        rate=v >> 44, channels=((v >> 41) & 7) + 1, bps=((v >> 36) & 31) + 1,
                        total_samples=v & ((1 << 36) - 1), md5=bytes(body[18:34]))
        pos += 4 + length
    if info is None:
        raise ValueError("no STREAMINFO")
    info["frames_start"] = pos
    return info


def _subframe(b, bs, sbps):
    if b.u(1):
        raise ValueError("subframe padding bit set")
    t = b.u(6)
    wasted = 0
    if b.u(1):
        wasted = b.unary() + 1
        sbps -= wasted
    if t == 0:
        x = np.full(bs, b.s_(sbps), np.int64)
    elif t == 1:
        x = np.array([b.s_(sbps) for _ in range(bs)], np.int64)
    elif 8 <= t <= 12 or t >= 32:
        order = t - 8 if t <= 12 else t - 31
        if order > bs:
            raise ValueError("predictor order above the block size")
        x = np.zeros(bs, np.int64)
        for i in range(order):
            x[i] = b.s_(sbps)
        if t >= 32:
            prec = b.u(4) + 1
            shift = b.s_(5)
            if prec == 16 or shift < 0:
                raise ValueError("bad LPC precision / shift")
            coefs = [b.s_(prec) for _ in range(order)]
        else:
            coefs, shift = FIXED[order], 0
        method, porder = b.u(2), b.u(4)
        if method > 1 or bs % (1 << porder) or (bs >> porder) < order:
            raise ValueError("bad residual")
        pbits, esc = (5, 31) if method else (4, 15)
        res = []
        for p in range(1 << porder):
            cnt = (bs >> porder) - (order if p == 0 else 0)
            k = b.u(pbits)
            if k == esc:
                nb = b.u(5)
                res += [b.s_(nb) for _ in range(cnt)]
            else:
                for _ in range(cnt):
                    u = (b.unary() << k) | b.u(k)
                    res.append((u >> 1) ^ -(u & 1))
        for i, r in enumerate(res):
            n = order + i
            acc = 0
            for j, c in enumerate(coefs):
                acc += c * int(x[n - 1 - j])
            x[n] = r + (acc >> shift)
    else:
        raise ValueError("reserved subframe type %d" % t)
    return x << wasted


def bit_string(data):
    return "".join("{:08b}".format(b) for b in data)


def decode_frame(data, off, info, bits=None):
    """(samples [bs, C], first sample number, variable, end offset) of the frame at data[off]; `bits` is bit_string(data)."""
    if data[off] != 0xFF or data[off + 1] & 0xFE != 0xF8:
        raise ValueError("no sync code")
    variable = data[off + 1] & 1
    bs_code, rate_code = data[off + 2] >> 4, data[off + 2] & 15
    assignment, size_code = data[off + 3] >> 4, (data[off + 3] >> 1) & 7
    if bs_code == 0 or rate_code == 15 or assignment > 10 or size_code in (3, 7) or data[off + 3] & 1:
        raise ValueError("reserved header value")
    number, i = _utf8(data, off + 4, variable)
    if bs_code == 1:
        bs = 192
    elif bs_code <= 5:
        bs = 576 << (bs_code - 2)
    elif bs_code >= 8:
        bs = 256 << (bs_code - 8)
    else:
        nb = 1 if bs_code == 6 else 2
        bs = int.from_bytes(data[i:i + nb], "big") + 1
        i += nb
    rate = info["rate"]
    if 1 <= rate_code <= 11:
        rate = {v: k for k, v in RATES.items()}[rate_code]
    elif rate_code >= 12:
        nb = 1 if rate_code == 12 else 2
        rate = int.from_bytes(data[i:i + nb], "big") * {12: 1000, 13: 1, 14: 10}[rate_code]
        i += nb
    bps = info["bps"] if size_code == 0 else {v: k for k, v in SIZES.items()}[size_code]
    if rate != info["rate"] or bps != info["bps"]:
        raise ValueError("header disagrees with STREAMINFO")
    if _crc8(data[off:i]) != data[i]:
        raise ValueError("CRC-8 mismatch")
    C = assignment + 1 if assignment < 8 else 2
    if C != info["channels"]:
        raise ValueError("channel count disagrees with STREAMINFO")
    b = _Bits(bits if bits is not None else bit_string(data), i + 1)
    chans = []
    for c in range(C):
        side = (assignment in (8, 10) and c == 1) or (assignment == 9 and c == 0)
        chans.append(_subframe(b, bs, bps + side))
    end = (b.pos + 7) // 8
    if end + 2 > len(data):
        raise ValueError("truncated")
    if crc16(data[off:end]) != int.from_bytes(data[end:end + 2], "big"):
        raise ValueError("CRC-16 mismatch")
    if assignment == 8:
        chans[1] = chans[0] - chans[1]
    elif assignment == 9:
        chans[0] = chans[0] + chans[1]
    elif assignment == 10:
        m = chans[0] * 2 + (chans[1] & 1)
        chans = [(m + chans[1]) >> 1, (m - chans[1]) >> 1]
    return np.stack(chans, 1), number, variable, end + 2


def decode(data, check_md5=True):
    """(info, int64 samples [n, C]) of a whole stream: the frames parsed one after the other from the end of the metadata."""
    info = parse_metadata(data)
    pos, out, sample, nominal = info["frames_start"], [], 0, None
    bits = bit_string(data)
    while pos < len(data):
        x, number, variable, end = decode_frame(data, pos, info, bits)
        if not variable:
            nominal = nominal or len(x)
            number *= nominal
        if number != sample:
            raise ValueError("frame at byte %d starts at sample %d, expected %d" % (pos, number, sample))
        out.append(x)
        sample += len(x)
        pos = end
    x = np.concatenate(out) if out else np.zeros((0, info["channels"]), np.int64)
    if info["total_samples"] and info["total_samples"] != len(x):
        raise ValueError("sample count disagrees with STREAMINFO")
    if check_md5 and info["md5"] != bytes(16) and md5(x, info["bps"]) != info["md5"]:
        raise ValueError("MD5 mismatch")
    return info, x


# ---------------------------------------------------------------------------------------------------------------- writer
class _Fields:
    """(value, width) fields of one frame, packed MSB first; a value never has more than 32 significant bits, a width may
    be larger (unary codes: a one bit after width - 1 zeros)."""

    def __init__(self):
        self.v, self.w = [], []

    def add(self, v, w):
        self.v.append(np.atleast_1d(np.asarray(v, np.int64)).astype(np.uint64) & np.uint64(0xFFFFFFFF))
        self.w.append(np.broadcast_to(np.asarray(w, np.int64), self.v[-1].shape))

    def pack(self):
        v = np.concatenate(self.v)
        w = np.concatenate(self.w).astype(np.int64)
        end = np.cumsum(w)
        total = int(end[-1]) if len(end) else 0
        bits = np.zeros((total + 7) // 8 * 8, np.uint8)
        for j in range(32):
            sel = ((v >> np.uint64(j)) & np.uint64(1)).astype(bool) & (w > j)
            bits[end[sel] - 1 - j] = 1
        return np.packbits(bits).tobytes()


def _utf8_bytes(v):
    if v < 0x80:
        return bytes([v])
    n = 1
    while v >= 1 << (5 * n + 6 if n < 6 else 36):
        n += 1
    out = []
    for _ in range(n):
        out.append(0x80 | (v & 0x3F))
        v >>= 6
    lead = (0xFF << (7 - n)) & 0xFF
    return bytes([lead | v] + out[::-1])


def _residual(f, res, order, bs, partition_order, rice_bits, escape, rng):
    f.add(1 if rice_bits == 5 else 0, 2)
    f.add(partition_order, 4)
    psize = bs >> partition_order
    esc_code, kmax = (31, 30) if rice_bits == 5 else (15, 14)
    start = 0
    for p in range(1 << partition_order):
        cnt = psize - (order if p == 0 else 0)
        r = res[start:start + cnt]
        start += cnt
        use_escape = escape == "all" or (escape == "some" and rng.random() < 0.3)
        if use_escape:
            nb = 0
            if cnt:
                m = int(max(r.max(), -r.min() - 1, 0))
                nb = m.bit_length() + 1 if (r != 0).any() else 0
            f.add(esc_code, rice_bits)
            f.add(nb, 5)
            if nb:
                f.add(r, nb)
            continue
        u = np.where(r >= 0, r * 2, -r * 2 - 1).astype(np.int64)
        mean = float(u.mean()) if cnt else 0.0
        k = min(kmax, max(0, int(np.floor(np.log2(mean))) if mean >= 1 else 0))
        f.add(k, rice_bits)
        if cnt:                  # one field per sample: (u >> k) zeros, a one, then the k low bits
            f.add((1 << k) | (u & ((1 << k) - 1)), (u >> k) + 1 + k)


def _lpc_coefs(x, order, precision):
    """Quantised Levinson-Durbin predictor of a block (quality only matters for the size of the stream)."""
    xf = x.astype(np.float64)
    r = np.array([xf[:len(xf) - k] @ xf[k:] for k in range(order + 1)])
    if r[0] == 0:
        return np.zeros(order, np.int64), 0
    r[0] *= 1 + 1e-9
    a = np.zeros(order)
    err = r[0]
    for i in range(order):
        k = (r[i + 1] - a[:i] @ r[i:0:-1]) / err
        a[:i] = a[:i] - k * a[:i][::-1]
        a[i] = k
        err *= 1 - k * k
    cmax = float(np.abs(a).max())
    if cmax == 0:
        return np.zeros(order, np.int64), 0
    shift = int(precision - 1 - np.ceil(np.log2(cmax + 1e-12)))
    shift = max(0, min(15, shift))
    q = np.clip(np.round(a * (1 << shift)), -(1 << (precision - 1)), (1 << (precision - 1)) - 1).astype(np.int64)
    return q, shift


def _predict(x, coefs, shift, order):
    """x[n] - ((sum_j coefs[j] x[n-1-j]) >> shift) for n >= order."""
    acc = np.zeros(len(x) - order, np.int64)
    for j, c in enumerate(coefs):
        acc += int(c) * x[order - 1 - j:len(x) - 1 - j]
    return x[order:] - (acc >> shift)


def _subframe_fields(f, x, sbps, predictor, partition_order, rice_bits, escape, wasted, rng):
    w = 0
    if wasted and (x != 0).any():
        nz = np.bitwise_or.reduce(np.abs(x))
        while not (nz >> w) & 1 and w < sbps - 1:
            w += 1
    x = x >> w
    sbps -= w
    bs = len(x)
    if (x == x[0]).all() and predictor != "verbatim":
        f.add(0, 1)
        f.add(0, 6)
        _wasted(f, w)
        f.add(x[0], sbps)
        return
    kind = predictor[0] if isinstance(predictor, tuple) else predictor
    if kind == "verbatim":
        f.add(0, 1)
        f.add(1, 6)
        _wasted(f, w)
        f.add(x, sbps)
        return
    po = partition_order
    if kind == "fixed":
        order = min(predictor[1], bs)
        coefs, shift = FIXED[order], 0
        f.add(0, 1)
        f.add(8 + order, 6)
        _wasted(f, w)
    else:
        order, precision = min(predictor[1], bs, 32), predictor[2]
        coefs, shift = _lpc_coefs(x, order, precision)
        f.add(0, 1)
        f.add(31 + order, 6)
        _wasted(f, w)
    while po and (bs % (1 << po) or (bs >> po) < order):
        po -= 1
    f.add(x[:order], sbps)
    if kind != "fixed":
        f.add(precision - 1, 4)
        f.add(shift, 5)
        f.add(coefs, precision)
    _residual(f, _predict(x, coefs, shift, order), order, bs, po, rice_bits, escape, rng)


def _wasted(f, w):
    if w:
        f.add(1, 1)
        f.add(1, w)            # unary w - 1: w - 1 zeros then a one
    else:
        f.add(0, 1)


def write(samples, rate, bps, block_size=4096, variable=False, channel_mode="independent", predictor=("lpc", 8, 12),
          partition_order=4, rice_bits=4, escape=None, wasted=True, explicit=False, from_streaminfo=False,
          total_samples=True, with_md5=True, blocks=("vorbis", "padding"), id3=False, seed=0):
    """A FLAC stream of `samples` (int [n, C], values within bps bits).

    block_size       int (fixed blocking; the last frame holds the rest) or a list of sizes (cycled)
    variable         the variable-blocksize strategy: headers carry sample numbers
    channel_mode     independent / left_side / right_side / mid_side (stereo only)
    predictor        ("lpc", order, precision) / ("fixed", order) / "verbatim"; a block of one repeated value is CONSTANT
    partition_order  the highest Rice partition order (lowered where the block size does not allow it)
    rice_bits        4 (coding method 0) or 5 (method 1)
    escape           None / "some" / "all": partitions written as raw bits
    wasted           shift out common trailing zero bits of each subframe
    explicit         rate and block size as explicit header bytes (codes 12-14, 6-7) instead of table codes
    from_streaminfo  rate and sample size codes 0 (take them from STREAMINFO)
    total_samples    False writes 0 (unknown); with_md5 False writes an all-zero MD5
    blocks           metadata after STREAMINFO: vorbis, padding, seektable, picture, unknown
    id3              a leading ID3v2 tag
    """
    x = np.asarray(samples, np.int64)
    n, C = x.shape
    rng = np.random.default_rng(seed)
    sizes = [block_size] if np.isscalar(block_size) else list(block_size)
    mode = MODES[channel_mode]
    if mode is not None and C != 2:
        raise ValueError("stereo decorrelation needs two channels")
    heads, bodies, starts = [], [], []
    pos, k = 0, 0
    while pos < n:
        bs = min(int(sizes[k % len(sizes)]), n - pos)
        starts.append(pos)
        blk = x[pos:pos + bs]
        h = bytearray([0xFF, 0xF8 | (1 if variable else 0)])
        std = {192: 1, 576: 2, 1152: 3, 2304: 4, 4608: 5, 256: 8, 512: 9, 1024: 10, 2048: 11, 4096: 12, 8192: 13,
               16384: 14, 32768: 15}
        if bs in std and not explicit:
            bs_code, bs_extra = std[bs], b""
        elif bs <= 256:
            bs_code, bs_extra = 6, bytes([bs - 1])
        else:
            bs_code, bs_extra = 7, (bs - 1).to_bytes(2, "big")
        if from_streaminfo:
            rate_code, rate_extra = 0, b""
        elif rate in RATES and not explicit:
            rate_code, rate_extra = RATES[rate], b""
        elif rate % 1000 == 0 and rate // 1000 < 256:
            rate_code, rate_extra = 12, bytes([rate // 1000])
        elif rate < 65536:
            rate_code, rate_extra = 13, rate.to_bytes(2, "big")
        elif rate % 10 == 0 and rate // 10 < 65536:
            rate_code, rate_extra = 14, (rate // 10).to_bytes(2, "big")
        else:
            rate_code, rate_extra = 0, b""
        h.append(bs_code << 4 | rate_code)
        size_code = 0 if from_streaminfo else SIZES.get(bps, 0)
        assignment = C - 1 if mode is None else mode
        h.append(assignment << 4 | size_code << 1)
        h += _utf8_bytes(pos if variable else k) + bs_extra + rate_extra
        h.append(_crc8(h))
        f = _Fields()
        if mode is None:
            chans = [(blk[:, c], bps) for c in range(C)]
        else:
            L, R = blk[:, 0], blk[:, 1]
            chans = {8: [(L, bps), (L - R, bps + 1)], 9: [(L - R, bps + 1), (R, bps)],
                     10: [((L + R) >> 1, bps), (L - R, bps + 1)]}[mode]
        for ch, sb in chans:
            _subframe_fields(f, ch, sb, predictor, partition_order, rice_bits, escape, wasted, rng)
        heads.append(bytes(h))
        bodies.append(f.pack())
        pos += bs
        k += 1
    frames = [h + b for h, b in zip(heads, bodies)]
    crcs = crc16_many(frames) if frames else []
    frames = [fr + c.to_bytes(2, "big") for fr, c in zip(frames, crcs)]
    lens = [len(fr) for fr in frames]
    bsizes = [int(b) for b in np.diff(starts + [n])]
    minb = min(bsizes[:-1] or bsizes or [16])
    maxb = max(bsizes or [16])
    if not variable:
        minb = maxb
    si = (max(16, minb) if len(bsizes) > 1 else max(16, maxb)).to_bytes(2, "big") + max(16, maxb).to_bytes(2, "big")
    si += (min(lens) if lens else 0).to_bytes(3, "big") + (max(lens) if lens else 0).to_bytes(3, "big")
    v = (rate << 44) | ((C - 1) << 41) | ((bps - 1) << 36) | (n if total_samples else 0)
    si += v.to_bytes(8, "big") + (md5(x, bps) if with_md5 else bytes(16))
    meta = [(0, si)]
    for kind in blocks:
        if kind == "vorbis":
            vendor = b"flac_oracle"
            body = len(vendor).to_bytes(4, "little") + vendor + (1).to_bytes(4, "little")
            c = b"TITLE=test"
            meta.append((4, body + len(c).to_bytes(4, "little") + c))
        elif kind == "padding":
            meta.append((1, bytes(64)))
        elif kind == "seektable":
            meta.append((3, (0).to_bytes(8, "big") + (0).to_bytes(8, "big") + (sizes[0] & 0xFFFF).to_bytes(2, "big")))
        elif kind == "picture":
            img = b"\x89PNG\r\n\x1a\n" + bytes(40)
            mime, desc = b"image/png", b"cover"
            body = (3).to_bytes(4, "big") + len(mime).to_bytes(4, "big") + mime + len(desc).to_bytes(4, "big") + desc
            body += bytes(16) + len(img).to_bytes(4, "big") + img
            meta.append((6, body))
        elif kind == "unknown":
            meta.append((99, b"\xff\xf8\x69\x08" * 5))      # content that looks like a frame sync, inside metadata
    out = bytearray(b"fLaC")
    for i, (kind, body) in enumerate(meta):
        out.append((0x80 if i == len(meta) - 1 else 0) | kind)
        out += len(body).to_bytes(3, "big") + body
    if id3:
        out = id3_tag() + out
    return bytes(out) + b"".join(frames)


def id3_tag(payload=b"TIT2\x00\x00\x00\x05\x00\x00test"):
    size = len(payload)
    syncsafe = bytes([(size >> 21) & 0x7F, (size >> 14) & 0x7F, (size >> 7) & 0x7F, size & 0x7F])
    return b"ID3\x04\x00\x00" + syncsafe + payload


def signal(seed, n, C, bps, silence=None):
    """Seeded test audio: per channel a few tones, a glide and noise at about -6 dBFS, as int64 within bps bits.  `silence`
    (start, stop) zeroes a stretch (digital silence)."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / 44100.0
    out = np.zeros((n, C))
    for c in range(C):
        for _ in range(3):
            out[:, c] += rng.uniform(0.05, 0.2) * np.sin(2 * np.pi * rng.uniform(50, 3000) * t + rng.uniform(0, 6.3))
        out[:, c] += 0.1 * np.sin(2 * np.pi * (200 + 400 * t) * t)
        out[:, c] += rng.normal(0, 0.02, n)
    full = (1 << (bps - 1)) - 1
    x = np.clip(np.round(out * full), -full - 1, full).astype(np.int64)
    if silence is not None:
        x[silence[0]:silence[1]] = 0
    return x
