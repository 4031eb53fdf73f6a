"""The GPU FLAC encoder's frame code (csrc/flac_encode.h) built for the host with AddressSanitizer and UBSan
(tests/flacenc), encode() on top of it with the same host assembly as wun.write_flac, and audit(), which parses every frame
and subframe header of a stream for the streamable-subset checks.  Built on first use under tests/flacenc/_build
(git-ignored), or the temp directory when the tree is read-only."""
import os
import shutil
import subprocess
import tempfile

import numpy as np

from oracle import flac_oracle as F

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "flacenc", "flac_encode_host.cpp")
CSRC = os.path.join(os.path.dirname(HERE), "wave-u-net_b200", "csrc")
HEADERS = [os.path.join(CSRC, "flac_encode.h"), os.path.join(CSRC, "flac_frame.h")]


class HostEncodeError(RuntimeError):
    """The host program failed: non-zero exit, or a sanitizer report."""


def build():
    """Path of the sanitizer build of the host encoder, or None without g++."""
    if not shutil.which("g++"):
        return None
    out_dir = os.path.join(HERE, "flacenc", "_build")
    try:
        os.makedirs(out_dir, exist_ok=True)
        open(os.path.join(out_dir, ".writable"), "w").close()
    except OSError:
        out_dir = os.path.join(tempfile.gettempdir(), "wun_flacenc_build")
        os.makedirs(out_dir, exist_ok=True)
    exe = os.path.join(out_dir, "flac_encode_host")
    if not os.path.exists(exe) or any(os.path.getmtime(p) > os.path.getmtime(exe) for p in [SRC] + HEADERS):
        tmp = "%s.%d.tmp" % (exe, os.getpid())
        subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                               "-fno-omit-frame-pointer", "-I", CSRC, "-o", tmp, SRC])
        os.replace(tmp, exe)
    return exe


def frames(x, rate, bps, block_size=4096):
    """(frame area bytes, int64 frame offsets) of int32 samples [n, C] through the host build."""
    import wun.flac  # noqa: F401  (the package path the tests set up)
    exe = build()
    x = np.ascontiguousarray(x, np.int32)
    n, C = x.shape
    with tempfile.TemporaryDirectory() as tmp:
        ps, pa, po = (os.path.join(tmp, k) for k in ("samples", "area", "offsets"))
        x.tofile(ps)
        env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0:exitcode=97")
        r = subprocess.run([exe, ps, str(n), str(C), str(bps), str(rate), str(block_size), pa, po], stdout=subprocess.PIPE,
                           stderr=subprocess.PIPE, env=env)
        if b"Sanitizer" in r.stderr or b"runtime error" in r.stderr or r.returncode:
            raise HostEncodeError("host encoder failed (%d):\n%s" % (r.returncode, r.stderr.decode(errors="replace")[-3000:]))
        with open(pa, "rb") as f:
            area = f.read()
        return area, np.fromfile(po, np.int64)


def encode(x, rate, bps, block_size=4096):
    """The whole stream, assembled on the host as wun.write_flac assembles it."""
    from wun import flac as W
    area, offsets = frames(x, rate, bps, block_size)
    if offsets[-1] < 0:
        raise ValueError("samples lie outside %d bits" % bps)
    x = np.asarray(x, np.int32)
    return W.assemble(area, offsets, block_size, rate, x.shape[1], bps, x.shape[0], W.md5_of(x, bps))


def _subframe_header(b, bs, sbps):
    """Parse one subframe (skipping its samples); returns a dict of its header fields."""
    assert b.u(1) == 0
    t = b.u(6)
    wasted = b.unary() + 1 if b.u(1) else 0
    sbps -= wasted
    d = dict(type=t, wasted=wasted)
    if t == 0:
        b.s_(sbps)
        return d
    if t == 1:
        b.pos += bs * sbps
        return d
    order = t - 8 if t <= 12 else t - 31
    d["order"] = order
    b.pos += order * sbps
    if t >= 32:
        d["precision"], d["shift"] = b.u(4) + 1, b.s_(5)
        b.pos += order * d["precision"]
    d["method"], d["porder"] = b.u(2), b.u(4)
    pbits = 5 if d["method"] else 4
    ks = []
    for p in range(1 << d["porder"]):
        k = b.u(pbits)
        ks.append(k)
        for _ in range((bs >> d["porder"]) - (order if p == 0 else 0)):
            b.unary()
            b.pos += k
    d["rice"] = ks
    return d


def audit(data):
    """(info, [frame dicts]) of a stream: each frame's offset, size, header codes and subframe headers."""
    info = F.parse_metadata(data)
    bits = F.bit_string(data)
    pos, out = info["frames_start"], []
    while pos < len(data):
        _, number, variable, end = F.decode_frame(data, pos, info, bits)
        hdr = dict(offset=pos, bytes=end - pos, number=number, variable=variable, bs_code=data[pos + 2] >> 4,
                   rate_code=data[pos + 2] & 15, assignment=data[pos + 3] >> 4, size_code=(data[pos + 3] >> 1) & 7)
        lead = data[pos + 4]                             # the coded number, then the optional block size and rate bytes
        i = pos + 5 + (0 if lead < 0x80 else bin(lead)[2:].index("0") - 1)
        i += {6: 1, 7: 2}.get(hdr["bs_code"], 0) + {12: 1, 13: 2, 14: 2}.get(hdr["rate_code"], 0)
        b = F._Bits(bits, i + 1)
        bs = len(F.decode_frame(data, pos, info, bits)[0])
        hdr["block_size"] = bs
        subs = []
        for c in range(info["channels"]):
            side = (hdr["assignment"] in (8, 10) and c == 1) or (hdr["assignment"] == 9 and c == 0)
            subs.append(_subframe_header(b, bs, info["bps"] + side))
        assert (b.pos + 7) // 8 + 2 == end
        hdr["subframes"] = subs
        out.append(hdr)
        pos = end
    return info, out


def check_subset(data, block_size=4096):
    """Assert the streamable-subset rules on every frame; returns the audit."""
    info, frames_ = audit(data)
    max_lpc = 12 if info["rate"] <= 48000 else 32
    for j, f in enumerate(frames_):
        assert not f["variable"] and f["number"] == j
        assert f["block_size"] == block_size or (j == len(frames_) - 1 and f["block_size"] < block_size)
        assert 1 <= f["rate_code"] <= 14
        if info["bps"] in (8, 12, 16, 20, 24):
            assert f["size_code"] != 0
        for s in f["subframes"]:
            if s["type"] >= 32:
                assert s["order"] <= max_lpc and s["precision"] <= 15 and 0 <= s["shift"] <= 15
            if "porder" in s:
                assert s["porder"] <= 8
                assert all(k < (31 if s["method"] else 15) for k in s["rice"])
                assert s["method"] == 1 or all(k <= 14 for k in s["rice"])
    sizes = [f["bytes"] for f in frames_]
    assert data[4] & 0x7F == 0                           # STREAMINFO first: its frame-size bounds are the real frames'
    bounds = int.from_bytes(data[12:15], "big"), int.from_bytes(data[15:18], "big")
    assert bounds == ((min(sizes), max(sizes)) if sizes else (0, 0))
    assert info["min_block"] == info["max_block"] == block_size
    return info, frames_
