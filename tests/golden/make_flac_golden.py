"""Writes tests/golden/flac/: FLAC fixtures encoded by FFmpeg's flac encoder, each with FFmpeg's own decode converted to
signed 16 bits by libswresample, which is what the reference's loader reads (librosa 0.6 -> audioread -> `ffmpeg -f s16le`).

    python tests/golden/make_flac_golden.py <directory holding libavcodec / libavformat / libavutil / libswresample>

FFmpeg is used through its shared libraries with ctypes.  Only options (av_opt_*) and the long-stable leading fields of
AVPacket, AVFrame, AVFormatContext and AVStream are touched.  Each fixture <name>.flac comes with <name>.npz:
  input     int32 [n, C] the seeded samples that were encoded (FFmpeg's decode at full depth equals them: checked here)
  s16       int16 [n, C] that decode through libswresample to s16 (no dither, as the ffmpeg tool does by default)
FFmpeg's encoder writes only 16- and 24-bit streams; the 8-bit and 12-bit fixtures and the one with an ID3v2 tag and a
PICTURE block are written by oracle/flac_oracle.py and decoded by FFmpeg the same way.
"""
import ctypes
import glob
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import flac_oracle as F  # noqa: E402

OUT = os.path.join(HERE, "flac")
REFERENCE_WAV = os.environ.get("WUN_REFERENCE_WAV")     # optional: a 16-bit WAV to take a short excerpt from
VP, I, I64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64


def load(libdir):
    pending, libs = sorted(glob.glob(os.path.join(libdir, "*.so*"))), {}
    while pending:                                       # load in dependency order
        left = []
        for p in pending:
            try:
                libs[os.path.basename(p)] = ctypes.CDLL(p, mode=ctypes.RTLD_GLOBAL)
            except OSError:
                left.append(p)
        if len(left) == len(pending):
            raise OSError("cannot load %s" % left)
        pending = left

    def pick(stem):
        return next(v for k, v in libs.items() if k.startswith(stem))
    av = dict(u=pick("libavutil"), c=pick("libavcodec"), f=pick("libavformat"), s=pick("libswresample"))
    for name, lib, res, args in [
            ("av_opt_set", "u", I, [VP, ctypes.c_char_p, ctypes.c_char_p, I]),
            ("av_opt_set_int", "u", I, [VP, ctypes.c_char_p, I64, I]),
            ("av_frame_alloc", "u", VP, []), ("av_frame_unref", "u", None, [VP]),
            ("av_get_sample_fmt_name", "u", ctypes.c_char_p, [I]),
            ("avcodec_find_encoder_by_name", "c", VP, [ctypes.c_char_p]),
            ("avcodec_find_decoder_by_name", "c", VP, [ctypes.c_char_p]),
            ("avcodec_alloc_context3", "c", VP, [VP]), ("avcodec_open2", "c", I, [VP, VP, VP]),
            ("avcodec_parameters_alloc", "c", VP, []),
            ("avcodec_parameters_from_context", "c", I, [VP, VP]), ("avcodec_parameters_to_context", "c", I, [VP, VP]),
            ("avcodec_send_packet", "c", I, [VP, VP]), ("avcodec_receive_frame", "c", I, [VP, VP]),
            ("avcodec_send_frame", "c", I, [VP, VP]), ("avcodec_receive_packet", "c", I, [VP, VP]),
            ("av_packet_alloc", "c", VP, []), ("av_new_packet", "c", I, [VP, I]), ("av_packet_unref", "c", None, [VP]),
            ("av_packet_get_side_data", "c", VP, [VP, I, ctypes.POINTER(ctypes.c_size_t)]),
            ("avcodec_descriptor_get_by_name", "c", VP, [ctypes.c_char_p]),
            ("avformat_open_input", "f", I, [ctypes.POINTER(VP), ctypes.c_char_p, VP, VP]),
            ("avformat_find_stream_info", "f", I, [VP, VP]), ("av_read_frame", "f", I, [VP, VP]),
            ("swr_alloc", "s", VP, []), ("swr_init", "s", I, [VP]),
            ("swr_convert", "s", I, [VP, ctypes.POINTER(VP), I, ctypes.POINTER(VP), I])]:
        fn = getattr(av[lib], name)
        fn.restype, fn.argtypes = res, args
    return av


def _ok(rc, what):
    if rc < 0:
        raise RuntimeError("%s failed (%d)" % (what, rc))
    return rc


# leading fields stable across FFmpeg releases
def _pkt_data(p):
    return ctypes.c_void_p.from_address(p + 24).value, ctypes.c_int.from_address(p + 32).value


def _frame_fields(fr):
    return ctypes.c_int.from_address(fr + 112).value, ctypes.c_int.from_address(fr + 116).value   # nb_samples, format


def _frame_plane(fr, c):
    ext = ctypes.c_void_p.from_address(fr + 96).value                                              # extended_data
    return ctypes.c_void_p.from_address(ext + 8 * c).value


LAYOUT = {1: "mono", 2: "stereo", 6: "6c"}


def encode(av, x, rate, bps, options):
    """FLAC bytes of int samples x [n, C] by FFmpeg's encoder: PCM packets through the pcm decoder give correctly described
    frames; their parameters configure the flac encoder; its packets are the frames and its last STREAMINFO heads them."""
    n, C = x.shape
    u, c = av["u"], av["c"]
    wide = bps > 16
    pcm = c.avcodec_alloc_context3(c.avcodec_find_decoder_by_name(b"pcm_s32le" if wide else b"pcm_s16le"))
    u.av_opt_set(pcm, b"ch_layout", LAYOUT[C].encode(), 0)
    u.av_opt_set_int(pcm, b"ar", rate, 0)
    _ok(c.avcodec_open2(pcm, c.avcodec_find_decoder_by_name(b"pcm_s32le" if wide else b"pcm_s16le"), None), "pcm open")
    par = c.avcodec_parameters_alloc()
    _ok(c.avcodec_parameters_from_context(par, pcm), "parameters")
    flac_id = ctypes.c_int.from_address(c.avcodec_descriptor_get_by_name(b"flac")).value
    ctypes.c_int.from_address(par + 4).value = flac_id                                             # codec_id
    codec = c.avcodec_find_encoder_by_name(b"flac")
    enc = c.avcodec_alloc_context3(codec)
    _ok(c.avcodec_parameters_to_context(enc, par), "parameters to encoder")
    u.av_opt_set(enc, b"time_base", ("1/%d" % rate).encode(), 0)
    u.av_opt_set_int(enc, b"bits_per_raw_sample", bps, 0)
    for k, v in options.items():
        _ok(u.av_opt_set(enc, k.encode(), str(v).encode(), 1), "option %s" % k)
    _ok(c.avcodec_open2(enc, codec, None), "flac encoder open")
    fs = ctypes.c_int64()
    u.av_opt_get_int.argtypes = [VP, ctypes.c_char_p, I, ctypes.POINTER(ctypes.c_int64)]
    _ok(u.av_opt_get_int(enc, b"frame_size", 0, ctypes.byref(fs)), "frame_size")
    fs = fs.value
    raw = (x.astype(np.int32) << (32 - bps)) if wide else x.astype(np.int16)
    pkt, frame, out = c.av_packet_alloc(), u.av_frame_alloc(), c.av_packet_alloc()
    frames, streaminfo = [], None

    def drain():
        nonlocal streaminfo
        while c.avcodec_receive_packet(enc, out) >= 0:
            data, size = _pkt_data(out)
            frames.append(ctypes.string_at(data, size))
            sz = ctypes.c_size_t()
            sd = c.av_packet_get_side_data(out, 1, ctypes.byref(sz))                              # NEW_EXTRADATA
            if sd:
                streaminfo = ctypes.string_at(sd, sz.value)
            c.av_packet_unref(out)
    for s in range(0, n, fs):
        chunk = np.ascontiguousarray(raw[s:s + fs]).tobytes()
        _ok(c.av_new_packet(pkt, len(chunk)), "packet")
        ctypes.memmove(_pkt_data(pkt)[0], chunk, len(chunk))
        _ok(c.avcodec_send_packet(pcm, pkt), "pcm send")
        c.av_packet_unref(pkt)
        while c.avcodec_receive_frame(pcm, frame) >= 0:
            _ok(c.avcodec_send_frame(enc, frame), "encode")
            u.av_frame_unref(frame)
            drain()
    _ok(c.avcodec_send_frame(enc, None), "flush")
    drain()
    if streaminfo is None:
        raise RuntimeError("the encoder gave no final STREAMINFO")
    head = b"fLaC" + bytes([0x80, 0, 0, 34]) + streaminfo[-34:]
    return head + b"".join(frames)


def decode(av, path, bps, C):
    """(full-depth int32 [n, C], s16 [n, C]) of FFmpeg's flac decoder on `path`, the s16 through libswresample."""
    u, c, f, s = av["u"], av["c"], av["f"], av["s"]
    fmt = VP()
    _ok(f.avformat_open_input(ctypes.byref(fmt), path.encode(), None, None), "open")
    _ok(f.avformat_find_stream_info(fmt, None), "stream info")
    st = ctypes.c_void_p.from_address(ctypes.c_void_p.from_address(fmt.value + 48).value).value    # streams[0]
    par = ctypes.c_void_p.from_address(st + 16).value                                              # codecpar
    codec = c.avcodec_find_decoder_by_name(b"flac")
    dec = c.avcodec_alloc_context3(codec)
    _ok(c.avcodec_parameters_to_context(dec, par), "parameters")
    _ok(c.avcodec_open2(dec, codec, None), "decoder open")
    pkt, frame = c.av_packet_alloc(), u.av_frame_alloc()
    full, s16, swr = [], [], None
    while True:
        eof = f.av_read_frame(fmt, pkt) < 0
        if not eof and ctypes.c_int.from_address(pkt + 36).value != 0:        # stream_index: a PICTURE is stream 1
            c.av_packet_unref(pkt)
            continue
        _ok(c.avcodec_send_packet(dec, None if eof else pkt), "send")
        if not eof:
            c.av_packet_unref(pkt)
        while c.avcodec_receive_frame(dec, frame) >= 0:
            ns, sf = _frame_fields(frame)
            name = u.av_get_sample_fmt_name(sf).decode()
            width = 2 if name.startswith("s16") else 4
            dt = np.int16 if width == 2 else np.int32
            if name.endswith("p"):
                a = np.stack([np.frombuffer(ctypes.string_at(_frame_plane(frame, ch), ns * width), dt)
                              for ch in range(C)], 1)
            else:
                a = np.frombuffer(ctypes.string_at(_frame_plane(frame, 0), ns * width * C), dt).reshape(ns, C)
            full.append(a.astype(np.int32) >> ((16 if width == 2 else 32) - bps))
            if swr is None:
                swr = s.swr_alloc()
                for k in ("in_chlayout", "out_chlayout"):
                    _ok(u.av_opt_set(swr, k.encode(), LAYOUT[C].encode(), 0), k)
                for k in ("in_sample_rate", "out_sample_rate"):
                    _ok(u.av_opt_set_int(swr, k.encode(), 44100, 0), k)
                _ok(u.av_opt_set(swr, b"in_sample_fmt", name.encode(), 0), "in fmt")
                _ok(u.av_opt_set(swr, b"out_sample_fmt", b"s16", 0), "out fmt")
                _ok(s.swr_init(swr), "swr_init")
            o = np.zeros((ns, C), np.int16)
            outp = (VP * 1)(o.ctypes.data)
            inp = (VP * C)(*[_frame_plane(frame, ch) for ch in range(C)]) if name.endswith("p") else \
                (VP * 1)(_frame_plane(frame, 0))
            got = _ok(s.swr_convert(swr, outp, ns, inp, ns), "swr_convert")
            s16.append(o[:got])
            u.av_frame_unref(frame)
        if eof:
            break
    return np.concatenate(full), np.concatenate(s16)


def cases():
    """(name, samples, rate, bps, ffmpeg encoder options or None for the oracle writer, writer options)"""
    sig = F.signal
    yield "lvl0_fixed_16_stereo", sig(1, 5000, 2, 16), 44100, 16, dict(compression_level=0, lpc_type="fixed"), None
    yield "lvl5_levinson_16_stereo", sig(2, 9000, 2, 16), 44100, 16, dict(compression_level=5, lpc_type="levinson"), None
    yield "lvl12_cholesky_24_stereo", sig(3, 9000, 2, 24), 48000, 24, dict(compression_level=12, lpc_type="cholesky"), None
    for mode in ("indep", "left_side", "right_side", "mid_side"):
        yield "chmode_%s" % mode, sig(4, 3000, 2, 16), 22050, 16, dict(compression_level=5, ch_mode=mode, frame_size=1152), None
    yield "mono_8000_576", sig(5, 4000, 1, 16), 8000, 16, dict(compression_level=8, frame_size=576), None
    yield "six_channels_24_96k", sig(6, 2500, 6, 24), 96000, 24, dict(compression_level=5, frame_size=1024), None
    silence = sig(7, 12000, 2, 16, silence=(2000, 9000))
    yield "silence_16_stereo", silence, 44100, 16, dict(compression_level=5, frame_size=2048), None
    yield "oracle_8bit_stereo", sig(8, 4000, 2, 8), 32000, 8, None, dict(channel_mode="mid_side", block_size=1152)
    yield "oracle_12bit_mono_fixed", sig(9, 3000, 1, 12), 11025, 12, None, dict(predictor=("fixed", 3), block_size=512,
                                                                               explicit=True)
    yield "oracle_id3_picture", sig(10, 3000, 2, 16), 44100, 16, None, dict(id3=True, blocks=("seektable", "vorbis",
                                                                                             "picture", "padding"))
    if REFERENCE_WAV:
        import scipy.io.wavfile
        rate, pcm = scipy.io.wavfile.read(REFERENCE_WAV)
        start = len(pcm) // 2
        yield "reference_excerpt", pcm[start:start + 8192].reshape(8192, -1).astype(np.int64), rate, 16, \
            dict(compression_level=8), None


def main(libdir):
    av = load(libdir)
    os.makedirs(OUT, exist_ok=True)
    for name, x, rate, bps, opts, wopts in cases():
        data = encode(av, x, rate, bps, opts) if opts is not None else F.write(x, rate, bps, **wopts)
        path = os.path.join(OUT, name + ".flac")
        with open(path, "wb") as f:
            f.write(data)
        full, s16 = decode(av, path, bps, x.shape[1])
        assert np.array_equal(full, x), name                 # FFmpeg decodes what it was given
        np.savez_compressed(os.path.join(OUT, name + ".npz"), input=x.astype(np.int32), s16=s16)
        print("%-28s %7d bytes  %d samples x %d" % (name, len(data), x.shape[0], x.shape[1]))


if __name__ == "__main__":
    main(sys.argv[1])
