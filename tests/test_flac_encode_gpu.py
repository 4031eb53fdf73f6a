"""wun.write_flac (csrc/kernels_flac_encode.cu): round trips through wun.read_flac and the oracle, the streamable subset,
byte-identical repeat encodes, the frame area against FFmpeg's on the fixtures, and Predict writing FLAC estimates."""
import glob
import json
import os

import numpy as np
import pytest
import scipy.io.wavfile
import torch

import Config
import Evaluate
import Predict
import Training
import flac_encode_host as H
import wun
from Models.UnetAudioSeparator import UnetAudioSeparator
from oracle import flac_oracle as F
from oracle import wave_unet_oracle as O
from wun import flac as W

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "flac")
FIXTURES = sorted(os.path.splitext(os.path.basename(p))[0] for p in glob.glob(os.path.join(GOLDEN, "*.flac")))
# FFmpeg-encoded fixtures whose predictors have order <= 12 (tests/golden/make_flac_golden.py: levels 0, 5 and 8)
FFMPEG_LPC12 = ["chmode_indep", "chmode_left_side", "chmode_mid_side", "chmode_right_side", "lvl0_fixed_16_stereo",
                "lvl5_levinson_16_stereo", "mono_8000_576", "reference_excerpt", "silence_16_stereo", "six_channels_24_96k"]


def fixture(name):
    with open(os.path.join(GOLDEN, name + ".flac"), "rb") as f:
        data = f.read()
    with np.load(os.path.join(GOLDEN, name + ".npz")) as z:
        return data, z["input"].astype(np.int32)


def alternating(n, C, bps):
    lo, hi = -(1 << (bps - 1)), (1 << (bps - 1)) - 1
    col = np.where(np.arange(n) % 2 == 0, hi, lo)
    return np.stack([col if c % 2 == 0 else -col - 1 for c in range(C)], 1).astype(np.int32)


def cases():
    for name in FIXTURES:
        data, x = fixture(name)
        info = W.parse_stream(data)
        yield name, x, info.rate, info.bps
    for bps in (8, 12, 16, 24):
        for C in (1, 2, 6):
            yield "signal_%d_%d" % (bps, C), F.signal(bps * 10 + C, 9000, C, bps).astype(np.int32), 44100, bps
    for bps in (8, 16, 24):
        x = F.signal(bps, 20000, 2, bps, silence=(4096, 9000)).astype(np.int32)
        x[12000:14000] = 7
        x[15000:19000] = alternating(4000, 2, bps)
        yield "constant_silence_full_scale_%d" % bps, x, 48000, bps
        yield "alternating_%d" % bps, alternating(9000, 2, bps), 44100, bps
    for n in (1, 100, 4096, 8192, 8193):
        yield "length_%d" % n, F.signal(n, n, 2, 16).astype(np.int32), 44100, 16


CASES = list(cases())


@pytest.mark.parametrize("name,x,rate,bps", CASES, ids=[c[0] for c in CASES])
def test_round_trip_subset_determinism(name, x, rate, bps):
    xd = torch.from_numpy(x).cuda()
    data = wun.write_flac(xd, rate, bps)
    assert wun.write_flac(xd, rate, bps) == data                          # byte-identical on a second run
    got_rate, got_bps, got = wun.read_flac(data)                          # MD5 checked
    assert (got_rate, got_bps) == (rate, bps) and torch.equal(got, xd)
    info, y = F.decode(data)
    assert np.array_equal(y, x) and info["md5"] == F.md5(x, bps)
    H.check_subset(data)


def test_float_input_is_quantised_as_the_rule_says():
    rng = np.random.default_rng(3)
    x = (rng.standard_normal((30000, 2)) * 0.3).astype(np.float32)
    x[:10] = [[1.5, -1.5], [np.nan, 0.0], [0.5 / 32768, 1.5 / 32768], [-1.0, 1.0], [2.5 / 32768, -2.5 / 32768],
              [1.0, -1.0], [0, 0], [3e38, -3e38], [1e-9, -1e-9], [np.inf, -np.inf]]
    for bps in (16, 24):
        data = wun.write_flac(torch.from_numpy(x).cuda(), 44100, bps)
        assert data == wun.write_flac(torch.from_numpy(W.quantise(x, bps)).cuda(), 44100, bps)
        assert np.array_equal(wun.read_flac(data)[2].cpu().numpy(), W.quantise(x, bps))


def test_mono_vector_and_refusals(tmp_path):
    x = F.signal(2, 5000, 1, 16).astype(np.int32)
    path = str(tmp_path / "m.flac")
    data = wun.write_flac(torch.from_numpy(x[:, 0]).cuda(), 44100, 16, path)
    with open(path, "rb") as f:
        assert f.read() == data
    assert torch.equal(wun.read_flac(path)[2].cpu(), torch.from_numpy(x))
    bad = x.copy()
    bad[4000] = 1 << 15
    with pytest.raises(ValueError, match="outside 16 bits"):
        wun.write_flac(torch.from_numpy(bad).cuda(), 44100, 16)
    with pytest.raises(ValueError, match="cannot be written"):
        wun.write_flac(torch.from_numpy(x).cuda(), 700001, 16)
    with pytest.raises(ValueError, match="bps"):
        wun.write_flac(torch.from_numpy(x).cuda(), 44100, 32)
    assert wun.read_flac(wun.write_flac(torch.zeros((0, 2), dtype=torch.int32, device="cuda"), 44100, 16))[2].shape == (0, 2)


@pytest.mark.parametrize("bps", [16, 24])
def test_three_minutes_stereo(bps):
    x = F.signal(bps, 180 * 44100, 2, bps).astype(np.int32)
    xd = torch.from_numpy(x).cuda()
    data = wun.write_flac(xd, 44100, bps)
    assert wun.write_flac(xd, 44100, bps) == data
    rate, got_bps, got = wun.read_flac(data)                              # MD5 checked
    assert (rate, got_bps) == (44100, bps) and torch.equal(got, xd)
    # the oracle and the subset audit are pure Python: they read the first 20 s, re-encoded alone
    part = wun.write_flac(xd[:20 * 44100], 44100, bps)
    assert np.array_equal(F.decode(part)[1], x[:20 * 44100])
    H.check_subset(part)


@pytest.mark.parametrize("name", FFMPEG_LPC12)
def test_frame_area_within_five_percent_of_ffmpeg(name):
    data, x = fixture(name)
    info = W.parse_stream(data)
    ours = wun.write_flac(torch.from_numpy(x).cuda(), info.rate, info.bps)
    ours_area = len(ours) - W.parse_stream(ours).frames_start
    ffmpeg_area = len(data) - info.frames_start
    print("%s: frame area %d bytes, FFmpeg %d (%.3f)" % (name, ours_area, ffmpeg_area, ours_area / ffmpeg_area))
    assert ours_area <= 1.05 * ffmpeg_area


def small_model(seed):
    cfg = Config.build_config(["baseline_stereo"], dict(num_layers=3, num_frames=64), experiment_id=0)
    mc = cfg["model_config"]
    t_in, _ = O.get_padding(mc, 64)
    sep = UnetAudioSeparator(mc)
    sep.load_variables(O.init_params(mc, seed=seed), input_frames=t_in)
    return cfg, mc, sep


@pytest.mark.parametrize("bit_depth", [16, 24])
def test_predict_writes_flac_estimates(tmp_path, bit_depth):
    cfg, mc, sep = small_model(seed=6)
    model = Training.save_checkpoint(str(tmp_path / "model.npz"), sep)
    rng = np.random.default_rng(12)
    stems = {n: np.clip(np.round(rng.standard_normal((2 * 44100 + 77, 2)) * 6000), -32768, 32767).astype(np.int16)
             for n in mc["source_names"]}
    mix = np.clip(sum(s.astype(np.int64) for s in stems.values()), -32768, 32767).astype(np.int16)
    scipy.io.wavfile.write(str(tmp_path / "song.wav"), 44100, mix)
    os.makedirs(tmp_path / "stems")
    for name, audio in stems.items():
        scipy.io.wavfile.write(str(tmp_path / "stems" / (name + ".wav")), 44100, audio)
    Predict.main(cfg, model, str(tmp_path / "song.wav"), output_path=str(tmp_path / "wav"))
    Predict.main(cfg, model, str(tmp_path / "song.wav"), output_path=str(tmp_path / "flac"),
                 references_path=str(tmp_path / "stems"), results_dir=str(tmp_path / "results"), output_format="flac",
                 bit_depth=bit_depth)
    assert not glob.glob(str(tmp_path / "flac_*.wav"))
    scale = float(1 << (bit_depth - 1))
    read_back = {}
    for name in mc["source_names"]:
        _, want = scipy.io.wavfile.read(str(tmp_path / ("wav_%s.wav" % name)))
        rate, bps, got = wun.read_flac(str(tmp_path / ("flac_%s.flac" % name)))
        assert (rate, bps) == (44100, bit_depth)
        got = got.cpu().numpy().astype(np.float64) / scale
        v = np.rint(want.astype(np.float64) * scale)
        inside = (v >= -scale) & (v <= scale - 1)                     # not clipped at +-1
        assert np.all(np.abs(got - want)[inside] <= 2.0 ** -bit_depth), name
        assert np.array_equal(got[~inside], np.clip(np.sign(want[~inside]), -1, (scale - 1) / scale)), name
        assert np.array_equal(got, W.quantise(want, bit_depth) / scale), name
        read_back[name] = got.astype(np.float32)
    refs = Predict.load_references(str(tmp_path / "stems"), 44100)
    direct = {name: (W.quantise(scipy.io.wavfile.read(str(tmp_path / ("wav_%s.wav" % name)))[1], bit_depth) / scale)
              .astype(np.float32) for name in mc["source_names"]}
    a = Evaluate.eval_track(refs, read_back, 44100, output_dir=str(tmp_path / "a"), track_name="song")
    b = Evaluate.eval_track(refs, direct, 44100, output_dir=str(tmp_path / "b"), track_name="song")
    assert json.dumps(a, sort_keys=True) == json.dumps(b, sort_keys=True)
    with open(tmp_path / "a" / "song.json") as fa, open(tmp_path / "b" / "song.json") as fb:
        assert fa.read() == fb.read()
    assert os.path.exists(tmp_path / "results" / "song.json")
