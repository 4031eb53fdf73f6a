"""FLAC encoding without a GPU: the GPU encoder's frame code (csrc/flac_encode.h) built for the host under AddressSanitizer
and UBSan (tests/flac_encode_host.py), its streams decoded back by the oracle (oracle/flac_oracle.py) and audited for the
streamable subset; the float quantisation rule; and Predict's output options."""
import glob
import os

import numpy as np
import pytest
from hypothesis import given, settings, strategies as st

import flac_encode_host as H
import Predict
from oracle import flac_oracle as F
from wun import flac as W

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "flac")
FIXTURES = sorted(os.path.splitext(os.path.basename(p))[0] for p in glob.glob(os.path.join(GOLDEN, "*.flac")))


def fixture(name):
    with open(os.path.join(GOLDEN, name + ".flac"), "rb") as f:
        data = f.read()
    with np.load(os.path.join(GOLDEN, name + ".npz")) as z:
        return data, z["input"]


def round_trip(x, rate, bps, block_size=4096):
    """Encode on the host build, decode with the oracle (MD5 checked), audit the subset; returns the stream."""
    x = np.asarray(x, np.int32)
    data = H.encode(x, rate, bps, block_size)
    info, got = F.decode(data)
    assert (info["rate"], info["bps"], info["channels"], info["total_samples"]) == (rate, bps, x.shape[1], x.shape[0])
    assert info["md5"] == F.md5(x, bps)
    assert np.array_equal(got, x)
    H.check_subset(data, block_size)
    return data


def alternating(n, C, bps):
    """Full-scale +-2^(bps-1) square waves, opposite in neighbouring channels: the side channel needs bps + 1 bits."""
    lo, hi = -(1 << (bps - 1)), (1 << (bps - 1)) - 1
    col = np.where(np.arange(n) % 2 == 0, hi, lo)
    return np.stack([col if c % 2 == 0 else -col - 1 for c in range(C)], 1).astype(np.int32)


@pytest.mark.parametrize("name", FIXTURES)
def test_fixture_inputs_round_trip(name):
    data, x = fixture(name)
    info = W.parse_stream(data)
    round_trip(x, info.rate, info.bps)


@pytest.mark.parametrize("bps", [8, 12, 16, 24])
@pytest.mark.parametrize("C", [1, 2, 6])
def test_depths_and_channels(bps, C):
    round_trip(F.signal(bps * 10 + C, 9000, C, bps), 44100 if C != 6 else 96000, bps)


@pytest.mark.parametrize("bps", [8, 16, 24])
def test_constant_silence_and_full_scale(bps):
    x = F.signal(bps, 20000, 2, bps, silence=(4096, 9000)).astype(np.int32)
    x[12000:14000] = 7                                   # a constant stretch that is not silence
    x[15000:19000] = alternating(4000, 2, bps)           # full scale, opposite signs
    data = round_trip(x, 48000, bps)
    subs = [s for f in H.audit(data)[1] for s in f["subframes"]]
    assert any(s["type"] == 0 for s in subs)             # the silent frame is CONSTANT
    round_trip(alternating(9000, 2, bps), 44100, bps)
    round_trip(alternating(5000, 1, bps), 44100, bps)


def test_wasted_bits():
    x = F.signal(3, 9000, 2, 16).astype(np.int32) & ~15
    data = round_trip(x, 44100, 16)
    assert all(s["wasted"] == 4 for f in H.audit(data)[1] for s in f["subframes"] if s["type"] != 0)


@pytest.mark.parametrize("n", [1, 2, 100, 4095, 4096, 8192, 8193])
def test_lengths(n):
    round_trip(F.signal(n, n, 2, 16), 44100, 16)


def test_empty_stream():
    data = H.encode(np.zeros((0, 2), np.int32), 44100, 16)
    info, got = F.decode(data)
    assert got.shape == (0, 2) and info["total_samples"] == 0


@pytest.mark.parametrize("rate", [8000, 37800, 44100, 96000, 192000, 255000, 352800])
def test_rates(rate):
    round_trip(F.signal(rate % 97, 5000, 2, 24), rate, 24)


def test_sample_outside_depth_raises():
    x = F.signal(1, 5000, 2, 16).astype(np.int32)
    x[4500, 1] = 40000
    with pytest.raises(ValueError, match="outside 16 bits"):
        H.encode(x, 44100, 16)


@pytest.mark.parametrize("name", ["lvl0_fixed_16_stereo", "lvl5_levinson_16_stereo", "chmode_indep", "mono_8000_576",
                                  "six_channels_24_96k", "silence_16_stereo", "reference_excerpt"])
def test_host_build_compresses_like_ffmpeg(name):
    """FFmpeg fixtures with predictors of order <= 12: our frame area is at most 5 % larger than FFmpeg's."""
    data, x = fixture(name)
    info = W.parse_stream(data)
    area, _ = H.frames(x, info.rate, info.bps)
    assert len(area) <= 1.05 * (len(data) - info.frames_start)


@settings(max_examples=30, deadline=None)
@given(bps=st.integers(4, 24), C=st.integers(1, 8), n=st.integers(1, 10000), block=st.sampled_from([16, 192, 1000, 4096, 4608]),
       seed=st.integers(0, 2 ** 16), kind=st.sampled_from(["signal", "noise", "steps"]))
def test_random_round_trip(bps, C, n, block, seed, kind):
    rng = np.random.default_rng(seed)
    if kind == "signal":
        x = F.signal(seed, n, C, bps)
    elif kind == "noise":
        x = rng.integers(-(1 << (bps - 1)), 1 << (bps - 1), (n, C))
    else:
        x = np.repeat(rng.integers(-(1 << (bps - 1)), 1 << (bps - 1), (n // 50 + 1, C)), 50, 0)[:n]
    round_trip(x, 44100, bps, block)


def test_quantise_rule():
    half = np.float32(0.5) / 32768
    x = np.array([0.5 / 32768, 1.5 / 32768, 2.5 / 32768, -0.5 / 32768, -1.5 / 32768], np.float32)
    assert np.array_equal(W.quantise(x, 16), [0, 2, 2, 0, -2])                  # ties to even
    x = np.array([1.0, -1.0, 2.0, -3.0, np.inf, -np.inf, np.nan, 1 - half], np.float32)
    assert np.array_equal(W.quantise(x, 16), [32767, -32768, 32767, -32768, 32767, -32768, 0, 32767])
    assert np.array_equal(W.quantise(np.array([1.0, -1.0], np.float32), 24), [(1 << 23) - 1, -(1 << 23)])
    # every 16-bit integer, read as s / 32768 (the WAV and FLAC read rule), quantises back to itself
    s = np.arange(-32768, 32768, dtype=np.int32)
    assert np.array_equal(W.quantise(s.astype(np.float32) / np.float32(32768), 16), s)
    s24 = np.arange(-(1 << 23), 1 << 23, 997, dtype=np.int32)
    assert np.array_equal(W.quantise(s24.astype(np.float32) / np.float32(1 << 23), 24), s24)


def test_predict_output_options():
    assert Predict.output_options() == ("wav", None)
    assert Predict.output_options("wav") == ("wav", None)
    assert Predict.output_options("flac") == ("flac", 16)
    assert Predict.output_options("FLAC", 24) == ("flac", 24)
    with pytest.raises(ValueError, match="only meaningful with output_format=flac"):
        Predict.output_options(None, 16)
    with pytest.raises(ValueError, match="only meaningful"):
        Predict.output_options("wav", 24)
    for depth in (8, 20, 32, "16", True):
        with pytest.raises(ValueError, match="16 or 24"):
            Predict.output_options("flac", depth)
    with pytest.raises(ValueError, match="output_format=mp3"):
        Predict.output_options("mp3")


def test_predict_command_line_options():
    import Config
    _, extras = Config.parse_command_line(["with", "cfg.full_44KHz", "input_path=a.wav", "output_format=flac", "bit_depth=24"])
    assert Predict.output_options(extras.get("output_format"), extras.get("bit_depth")) == ("flac", 24)
    _, extras = Config.parse_command_line(["input_path=a.wav", "bit_depth=24"])
    with pytest.raises(ValueError):
        Predict.output_options(extras.get("output_format"), extras.get("bit_depth"))
