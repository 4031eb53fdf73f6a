"""The host half of FLAC decoding: the stream's metadata and the chain of frames (DESIGN.md §4.10).

parse_stream(data)   -> StreamInfo: an optional ID3v2 tag, the `fLaC` marker and the metadata blocks.  STREAMINFO is required;
                        SEEKTABLE, VORBIS_COMMENT, PICTURE, PADDING and unknown blocks are skipped.
chain_frames(...)    keeps, out of the device's frame candidates, the frames that follow one another from the first byte of
                        the frame area to its end, each starting at the sample its header names.  False sync candidates drop
                        out; a broken chain raises ValueError naming the byte offset and the frame.
md5_of(samples, bps) the STREAMINFO MD5: every sample as (bps + 7) // 8 little-endian bytes, channels interleaved.

The host half of FLAC encoding (DESIGN.md §4.11):
quantise(x, bps)     the rule the device applies to float input, restated in numpy for the tests.
assemble(...)        `fLaC`, STREAMINFO (block and frame size bounds from the real frames, total samples, MD5) and a
                        VORBIS_COMMENT block in front of the frame area wun.write_flac copied from the device.

Pure host code; wun.read_flac and wun.write_flac run the kernels between them.  All O(metadata + frames).
"""
import collections
import hashlib

import numpy as np

StreamInfo = collections.namedtuple("StreamInfo", "min_block max_block rate channels bps total_samples md5 frames_start")

STATUS = {-1: "truncated", -2: "bad header", -3: "bad subframe", -4: "bad residual", -5: "CRC-16 mismatch",
          -6: "samples outside the stream"}


def _id3v2_length(data):
    """Bytes of a leading ID3v2 tag (header, syncsafe size, optional footer), 0 when there is none."""
    if len(data) < 10 or data[:3] != b"ID3":
        return 0
    size = 0
    for b in data[6:10]:
        if b & 0x80:
            raise ValueError("FLAC: malformed ID3v2 tag size")
        size = (size << 7) | b
    return 10 + size + (10 if data[5] & 0x10 else 0)


def parse_stream(data):
    """StreamInfo of a FLAC stream in `data` (bytes).  Raises ValueError for anything that is not a FLAC stream this decoder
    supports: 4-24 bits per sample, 1-8 channels."""
    pos = _id3v2_length(data)
    if data[pos:pos + 4] != b"fLaC":
        raise ValueError("not a FLAC stream: no fLaC marker at byte %d" % pos)
    pos += 4
    info = None
    last = False
    while not last:
        if pos + 4 > len(data):
            raise ValueError("FLAC: metadata block header at byte %d runs past the end of the stream" % pos)
        last, kind, length = data[pos] >> 7, data[pos] & 0x7F, int.from_bytes(data[pos + 1:pos + 4], "big")
        body = data[pos + 4:pos + 4 + length]
        if len(body) < length:
            raise ValueError("FLAC: metadata block at byte %d runs past the end of the stream" % pos)
        if kind == 0:
            if info is not None or length < 34:
                raise ValueError("FLAC: bad STREAMINFO block at byte %d" % pos)
            v = int.from_bytes(body[10:18], "big")
            info = dict(min_block=int.from_bytes(body[0:2], "big"), max_block=int.from_bytes(body[2:4], "big"),
                        rate=v >> 44, channels=((v >> 41) & 7) + 1, bps=((v >> 36) & 31) + 1,
                        total_samples=v & ((1 << 36) - 1), md5=bytes(body[18:34]))
        elif kind == 127:
            raise ValueError("FLAC: invalid metadata block type 127 at byte %d" % pos)
        pos += 4 + length
    if info is None:
        raise ValueError("FLAC: no STREAMINFO block")
    if not 4 <= info["bps"] <= 24:
        raise ValueError("FLAC: %d bits per sample is not supported (4 to 24)" % info["bps"])
    if info["rate"] == 0:
        raise ValueError("FLAC: STREAMINFO gives a sample rate of 0")
    return StreamInfo(frames_start=pos, **info)


def chain_frames(frames, nbytes, info):
    """(offsets, first_samples, n_samples) of the frames that chain through the frame area, from the candidate records
    `frames` (numpy structured array with WunFlacFrame's fields, any order).  Frame offsets are relative to the frame area;
    errors name them as byte offsets in the whole stream."""
    order = np.argsort(frames["offset"], kind="stable")
    frames = frames[order]
    index = {int(o): i for i, o in enumerate(frames["offset"])}
    offsets, firsts = [], []
    pos, sample, nominal = 0, 0, None
    while pos < nbytes:
        where = "FLAC frame %d at byte offset %d" % (len(offsets), info.frames_start + pos)
        i = index.get(pos)
        if i is None:
            raise ValueError("%s: no valid frame header" % where)
        f = frames[i]
        if f["end"] < 0:
            raise ValueError("%s: %s" % (where, STATUS.get(int(f["end"]), "invalid")))
        if f["variable"]:
            first = int(f["number"])
        else:
            nominal = int(f["block_size"]) if nominal is None else nominal
            first = int(f["number"]) * nominal
        if first != sample:
            raise ValueError("%s: starts at sample %d, the previous frames end at sample %d" % (where, first, sample))
        offsets.append(pos)
        firsts.append(first)
        sample += int(f["block_size"])
        pos = int(f["end"])
    if info.total_samples and sample != info.total_samples:
        raise ValueError("FLAC: the frames hold %d samples, STREAMINFO says %d" % (sample, info.total_samples))
    return np.asarray(offsets, np.int64), np.asarray(firsts, np.int64), sample


def packed_bytes(samples, bps):
    """The bytes STREAMINFO's MD5 covers: int32 samples [n, C] as (bps + 7) // 8 little-endian bytes each (numpy or torch;
    torch tensors are packed where they live and copied to the host once)."""
    nb = (bps + 7) // 8
    if isinstance(samples, np.ndarray):
        return np.ascontiguousarray(samples.astype("<i4").view(np.uint8).reshape(-1, 4)[:, :nb]).tobytes()
    import torch
    b = samples.contiguous().view(torch.uint8).reshape(-1, 4)[:, :nb].contiguous()
    return b.cpu().numpy().tobytes()


def md5_of(samples, bps):
    return hashlib.md5(packed_bytes(samples, bps)).digest()


def to_float(samples, bps):
    """librosa 0.6's load() of a FLAC file through ffmpeg's s16le output (tests/golden/flac pin it against FFmpeg): full-depth
    samples left-aligned to 16 bits, or arithmetically shifted down to 16 bits, then divided by 32768.  float32 [n, C]."""
    x = np.asarray(samples, np.int32)
    x = x << (16 - bps) if bps <= 16 else x >> (bps - 16)
    return x.astype(np.float32) / np.float32(32768)


VENDOR = b"wave-u-net_b200 GPU FLAC encoder"


def quantise(x, bps):
    """float samples -> int32 at `bps` bits: clamp(rint(x * 2^(bps-1)), -2^(bps-1), 2^(bps-1) - 1), ties to even, NaN -> 0
    (include/wun.h WUN_FLAC_FLOAT32).  x * 2^(bps-1) is exact in float32, so s / 2^(bps-1) read back gives s again."""
    x = np.asarray(x, np.float32)
    with np.errstate(over="ignore", invalid="ignore"):                # +-inf clip like the device's saturation
        v = np.rint(x * np.float32(1 << (bps - 1)))
    v = np.clip(np.where(np.isnan(v), 0, v), -(1 << (bps - 1)), (1 << (bps - 1)) - 1)
    return v.astype(np.int32)


def header_rate_ok(rate):
    """Whether a frame header can state `rate` (a table code, kHz in 8 bits, Hz or tens of Hz in 16 bits)."""
    return rate in (8000, 16000, 22050, 24000, 32000, 44100, 48000, 88200, 96000, 176400, 192000) or \
        (rate % 1000 == 0 and rate // 1000 <= 255) or 0 < rate <= 65535 or (rate % 10 == 0 and rate // 10 <= 65535)


def _block(kind, body, last):
    return bytes([(0x80 if last else 0) | kind]) + len(body).to_bytes(3, "big") + body


def assemble(area, offsets, block_size, rate, channels, bps, total_samples, md5):
    """The whole stream: `fLaC`, STREAMINFO, VORBIS_COMMENT (vendor string, no fields), then the frame area `area` (bytes)
    whose frames start at offsets[:-1] (numpy int64, offsets[-1] == len(area))."""
    sizes = np.diff(np.asarray(offsets, np.int64))
    min_frame, max_frame = (int(sizes.min()), int(sizes.max())) if sizes.size else (0, 0)
    info = (block_size.to_bytes(2, "big") * 2 + min_frame.to_bytes(3, "big") + max_frame.to_bytes(3, "big") +
            ((rate << 44) | ((channels - 1) << 41) | ((bps - 1) << 36) | total_samples).to_bytes(8, "big") + md5)
    comment = len(VENDOR).to_bytes(4, "little") + VENDOR + (0).to_bytes(4, "little")
    return b"fLaC" + _block(0, info, False) + _block(4, comment, True) + bytes(area)
