"""FLAC decoding without a GPU: the oracle (oracle/flac_oracle.py) against FFmpeg-encoded fixtures and FFmpeg's own s16
conversion (tests/golden/flac), the oracle writer against the oracle decoder, and the GPU decoder's frame code
(csrc/flac_frame.h) built for the host under AddressSanitizer (tests/flac_host.py) against both, on well-formed, truncated
and corrupted streams."""
import glob
import os

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import flac_host
import Predict
from oracle import flac_oracle as F
from wun import flac as W

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "flac")
FIXTURES = sorted(os.path.splitext(os.path.basename(p))[0] for p in glob.glob(os.path.join(GOLDEN, "*.flac")))

# one writer stream per feature of the decoder (csrc/flac_frame.h)
FEATURES = {
    "lpc_independent": dict(),
    "lpc32_prec15": dict(predictor=("lpc", 32, 15)),
    "fixed_orders": dict(predictor=("fixed", 4), channel_mode="left_side"),
    "fixed_order0": dict(predictor=("fixed", 0), channel_mode="right_side"),
    "mid_side": dict(channel_mode="mid_side"),
    "verbatim": dict(predictor="verbatim"),
    "rice5_escape_some": dict(rice_bits=5, escape="some"),
    "escape_all": dict(escape="all", partition_order=0),
    "partition_order_15": dict(block_size=65535 - 32767, partition_order=15, predictor=("fixed", 1)),
    "variable_explicit": dict(variable=True, block_size=[100, 4096, 37, 1000, 16], explicit=True),
    "from_streaminfo": dict(from_streaminfo=True, block_size=1000),
    "no_total_no_md5": dict(total_samples=False, with_md5=False),
    "metadata_id3": dict(id3=True, blocks=("seektable", "picture", "unknown", "vorbis", "padding")),
}


def fixture(name):
    with open(os.path.join(GOLDEN, name + ".flac"), "rb") as f:
        data = f.read()
    with np.load(os.path.join(GOLDEN, name + ".npz")) as z:
        return data, z["input"], z["s16"]


def feature_stream(name, bps=16, C=2, n=9000, seed=3):
    x = F.signal(seed, n, C, bps, silence=(2000, 4100))
    x[5000:5600] &= ~7                                   # wasted bits
    x[6000:6300] = 5                                     # a constant block
    return x, F.write(x, 44100 if "explicit" not in name else 37800, bps, seed=seed, **FEATURES[name])


def test_fixtures_present():
    assert len(FIXTURES) >= 13 and sum(os.path.getsize(p) for p in glob.glob(os.path.join(GOLDEN, "*"))) < 1_100_000


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_decodes_fixture(name):
    data, want, s16 = fixture(name)
    info, got = F.decode(data)
    assert np.array_equal(got, want)
    assert info["md5"] == F.md5(want, info["bps"]) and info["md5"] != bytes(16)
    # §1: the reference's loader sees FFmpeg's s16 output divided by 32768
    assert np.array_equal(W.to_float(got, info["bps"]) * 32768, s16.astype(np.float32))


@pytest.mark.parametrize("name", FIXTURES)
def test_host_decoder_matches_fixture(name):
    data, want, _ = fixture(name)
    info, got = flac_host.read_flac(data)
    assert np.array_equal(got, want)


@pytest.mark.parametrize("name", sorted(FEATURES))
@pytest.mark.parametrize("bps", [8, 16, 24])
def test_host_decoder_matches_oracle_on_features(name, bps):
    x, data = feature_stream(name, bps)
    assert np.array_equal(F.decode(data)[1], x)
    assert np.array_equal(flac_host.read_flac(data)[1], x)


@pytest.mark.parametrize("bps,C", [(4, 1), (12, 3), (20, 8), (24, 6)])
def test_host_decoder_odd_depths_and_channels(bps, C):
    x = F.signal(bps + C, 3000, C, bps)
    data = F.write(x, 48000, bps, block_size=1024)
    assert np.array_equal(flac_host.read_flac(data)[1], x)


@settings(max_examples=40, deadline=None)
@given(bps=st.integers(4, 24), mode=st.sampled_from(sorted(F.MODES)), block=st.integers(1, 5000),
       porder=st.integers(0, 8), rice=st.sampled_from([4, 5]), escape=st.sampled_from([None, "some", "all"]),
       pred=st.sampled_from([("lpc", 1, 5), ("lpc", 12, 14), ("fixed", 2), ("fixed", 4), "verbatim"]),
       variable=st.booleans(), n=st.integers(1, 6000), seed=st.integers(0, 2 ** 16))
def test_writer_decoder_round_trip(bps, mode, block, porder, rice, escape, pred, variable, n, seed):
    C = 2 if mode != "independent" else 1 + seed % 3
    x = F.signal(seed, n, C, bps)
    data = F.write(x, 44100, bps, block_size=block, variable=variable, channel_mode=mode, predictor=pred,
                   partition_order=porder, rice_bits=rice, escape=escape, seed=seed)
    assert np.array_equal(F.decode(data)[1], x)


def broken_streams():
    x, data = feature_stream("lpc_independent", 16, n=20000)
    start = W.parse_stream(data).frames_start
    rng = np.random.default_rng(5)
    out = [("truncated_%d" % k, data[:k]) for k in (len(data) - 1, len(data) - 2, start + 40, (start + len(data)) // 2)]
    for k in rng.integers(start, len(data), 12):
        b = bytearray(data)
        b[k] ^= 1 << int(rng.integers(0, 8))
        out.append(("flip_%d" % k, bytes(b)))
    return out


@pytest.mark.parametrize("name,data", broken_streams(), ids=lambda v: v if isinstance(v, str) else "")
def test_host_decoder_rejects_broken_streams(name, data):
    """Every truncation or bit flip raises ValueError naming the frame (the MD5 catches a flip the CRCs miss), and the
    AddressSanitizer build reports no out-of-range access."""
    with pytest.raises(ValueError, match=r"FLAC frame \d+ at byte offset \d+|MD5|samples"):
        flac_host.read_flac(data)
    with pytest.raises(ValueError):
        F.decode(data)


def test_stream_refusals():
    x = F.signal(1, 100, 1, 16)
    data = bytearray(F.write(x, 44100, 16))
    with pytest.raises(ValueError, match="fLaC"):
        W.parse_stream(b"RIFF" + bytes(40))
    data32 = bytearray(data)
    data32[8 + 12] |= 0x01                               # STREAMINFO bits per sample - 1: 5 bits across these two bytes
    data32[8 + 13] |= 0xF0
    with pytest.raises(ValueError, match="32 bits per sample is not supported"):
        W.parse_stream(bytes(data32))
    with pytest.raises(ValueError, match="STREAMINFO"):
        W.parse_stream(b"fLaC" + bytes([0x81, 0, 0, 4]) + bytes(4))


def test_to_float_rule():
    x = np.array([[-128, 127]], np.int32)
    assert np.array_equal(W.to_float(x, 8), np.array([[-32768, 32512]], np.float32) / 32768)
    x = np.array([[-(1 << 23), (1 << 23) - 1, -1, 255]], np.int32)
    assert np.array_equal(W.to_float(x, 24) * 32768, np.array([[-32768, 32767, -1, 0]], np.float32))


def test_reference_stems_in_both_formats_are_refused(tmp_path):
    for name in ("vocals.wav", "vocals.flac", "accompaniment.wav"):
        (tmp_path / name).write_bytes(b"")
    with pytest.raises(ValueError, match="vocals"):
        Predict.load_references(str(tmp_path), 44100)
    with pytest.raises(ValueError, match=".wav and .flac"):
        Predict.read_audio(str(tmp_path / "song.mp3"))
