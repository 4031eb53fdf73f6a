"""The GPU FLAC decoder's frame code (csrc/flac_frame.h) built for the host with AddressSanitizer (tests/flachost), and
read_flac() on top of it: the same find -> chain -> decode sequence as wun.read_flac, with the device passes replaced by the
host program.  Built on first use under tests/flachost/_build (git-ignored), or the temp directory when the tree is
read-only."""
import os
import shutil
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "flachost", "flac_host.cpp")
HEADER = os.path.join(os.path.dirname(HERE), "wave-u-net_b200", "csrc", "flac_frame.h")
FRAME = np.dtype([("offset", np.int64), ("number", np.int64), ("end", np.int64), ("block_size", np.int64),
                  ("variable", np.int64)])


class HostDecodeError(RuntimeError):
    """The host program failed: non-zero exit, or an AddressSanitizer report."""


def build():
    """Path of the ASan build of the host decoder, or None without g++."""
    if not shutil.which("g++"):
        return None
    out_dir = os.path.join(HERE, "flachost", "_build")
    try:
        os.makedirs(out_dir, exist_ok=True)
        probe = os.path.join(out_dir, ".writable")
        open(probe, "w").close()
    except OSError:
        out_dir = os.path.join(tempfile.gettempdir(), "wun_flachost_build")
        os.makedirs(out_dir, exist_ok=True)
    exe = os.path.join(out_dir, "flac_host")
    if not os.path.exists(exe) or any(os.path.getmtime(p) > os.path.getmtime(exe) for p in (SRC, HEADER)):
        subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                               "-fno-omit-frame-pointer", "-I", os.path.dirname(HEADER), "-o", exe + ".tmp", SRC])
        os.replace(exe + ".tmp", exe)
    return exe


def _run(args):
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0:abort_on_error=0:exitcode=97")
    r = subprocess.run(args, stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=env)
    if b"Sanitizer" in r.stderr or b"runtime error" in r.stderr or r.returncode == 97:
        raise HostDecodeError("sanitizer report:\n" + r.stderr.decode(errors="replace")[-3000:])
    return r


def read_flac(data):
    """(info, int32 [n, C]) of a FLAC stream through the host build; ValueError as wun.read_flac raises it."""
    import wun.flac as W
    exe = build()
    info = W.parse_stream(data)
    area = data[info.frames_start:]
    si = [str(info.bps), str(info.channels), str(info.rate), str(info.max_block)]
    with tempfile.TemporaryDirectory() as tmp:
        p_area, p_frames = os.path.join(tmp, "area"), os.path.join(tmp, "frames")
        with open(p_area, "wb") as f:
            f.write(area)
        r = _run([exe, "find", p_area] + si + [p_frames])
        if r.returncode:
            raise HostDecodeError("find failed (%d): %s" % (r.returncode, r.stderr.decode(errors="replace")))
        frames = np.fromfile(p_frames, FRAME)
        offsets, firsts, n = W.chain_frames(frames, len(area), info)
        p_chain, p_out = os.path.join(tmp, "chain"), os.path.join(tmp, "out")
        np.stack([offsets, firsts], 1).astype(np.int64).tofile(p_chain)
        r = _run([exe, "decode", p_area] + si + [p_chain, str(n), p_out])
        if r.returncode == 3:
            raise ValueError("FLAC: " + r.stderr.decode(errors="replace").strip())
        if r.returncode:
            raise HostDecodeError("decode failed (%d): %s" % (r.returncode, r.stderr.decode(errors="replace")))
        out = np.fromfile(p_out, np.int32).reshape(n, info.channels)
    if info.md5 != bytes(16) and W.md5_of(out, info.bps) != info.md5:
        raise ValueError("FLAC: the decoded samples do not match the stream's MD5")
    return info, out
