"""wun.read_flac (csrc/kernels_flac.cu) bit for bit against the oracle fixtures and 3-minute writer streams, its refusal of
a truncated stream, and Predict / BSS Eval scoring from FLAC files giving what the same samples give from WAV."""
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
import wun
from Models.UnetAudioSeparator import UnetAudioSeparator
from oracle import flac_oracle as F
from oracle import wave_unet_oracle as O

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "flac")
FIXTURES = sorted(os.path.splitext(os.path.basename(p))[0] for p in glob.glob(os.path.join(GOLDEN, "*.flac")))


def same_bits(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("name", FIXTURES)
def test_fixture_bit_for_bit(name):
    path = os.path.join(GOLDEN, name + ".flac")
    with open(path, "rb") as f:
        info, want = F.decode(f.read())
    rate, bps, got = wun.read_flac(path)
    assert got.is_cuda and got.dtype == torch.int32
    assert (rate, bps) == (info["rate"], info["bps"])
    assert np.array_equal(got.cpu().numpy(), want)


@pytest.mark.parametrize("bps", [16, 24])
def test_three_minutes_stereo(bps):
    x = F.signal(bps, 180 * 44100, 2, bps)
    data = F.write(x, 44100, bps, block_size=4096, predictor=("lpc", 12, 14), channel_mode="mid_side", seed=bps)
    rate, got_bps, got = wun.read_flac(data)
    assert (rate, got_bps) == (44100, bps)
    assert np.array_equal(got.cpu().numpy(), x)


def test_every_writer_feature():
    for kw in [dict(variable=True, block_size=[100, 4096, 37, 1000, 16], explicit=True), dict(rice_bits=5, escape="some"),
               dict(predictor="verbatim", channel_mode="left_side"), dict(predictor=("fixed", 3), channel_mode="right_side"),
               dict(predictor=("lpc", 32, 15), id3=True, blocks=("picture", "unknown", "seektable")),
               dict(total_samples=False, with_md5=False, from_streaminfo=True)]:
        for bps, C in [(8, 2), (12, 2), (24, 2)] + ([(20, 1), (16, 8)] if "channel_mode" not in kw else []):
            x = F.signal(bps * 7 + C, 20000, C, bps, silence=(3000, 9000))
            x[10000:10500] &= ~3
            got = wun.read_flac(F.write(x, 44100 if "explicit" not in kw else 37800, bps, **kw))[2]
            assert np.array_equal(got.cpu().numpy(), x), (kw, bps, C)


def test_truncated_stream_raises():
    x = F.signal(4, 30000, 2, 16)
    data = F.write(x, 44100, 16)
    with pytest.raises(ValueError, match=r"FLAC frame \d+ at byte offset \d+"):
        wun.read_flac(data[:-100])
    b = bytearray(data)
    b[-500] ^= 0x10
    with pytest.raises(ValueError, match=r"FLAC frame \d+ at byte offset \d+|MD5"):
        wun.read_flac(bytes(b))


def small_model(seed):
    cfg = Config.build_config(["baseline_stereo"], dict(num_layers=3, num_frames=64), experiment_id=0)
    mc = cfg["model_config"]
    t_in, _ = O.get_padding(mc, 64)
    sep = UnetAudioSeparator(mc)
    sep.load_variables(O.init_params(mc, seed=seed), input_frames=t_in)
    return cfg, mc, sep


def test_predict_from_flac_equals_wav(tmp_path):
    cfg, mc, sep = small_model(seed=6)
    model = Training.save_checkpoint(str(tmp_path / "model.npz"), sep)
    rng = np.random.default_rng(12)
    stems = {n: np.clip(np.round(rng.standard_normal((2 * 44100 + 77, 2)) * 3000), -32768, 32767).astype(np.int16)
             for n in mc["source_names"]}
    mix = np.clip(sum(s.astype(np.int64) for s in stems.values()), -32768, 32767).astype(np.int16)
    scipy.io.wavfile.write(str(tmp_path / "song.wav"), 44100, mix)
    with open(tmp_path / "song.flac", "wb") as f:
        f.write(F.write(mix, 44100, 16))
    for fmt in ("wav", "flac"):
        os.makedirs(tmp_path / ("stems_" + fmt))
        for name, audio in stems.items():
            path = str(tmp_path / ("stems_" + fmt) / ("%s.%s" % (name, fmt)))
            if fmt == "wav":
                scipy.io.wavfile.write(path, 44100, audio)
            else:
                with open(path, "wb") as f:
                    f.write(F.write(audio, 44100, 16, channel_mode="mid_side"))
        Predict.main(cfg, model, str(tmp_path / ("song." + fmt)), output_path=str(tmp_path / ("out_" + fmt)),
                     references_path=str(tmp_path / ("stems_" + fmt)), results_dir=str(tmp_path / ("results_" + fmt)))
    for name in mc["source_names"]:
        rw, ew = scipy.io.wavfile.read(str(tmp_path / ("out_wav_%s.wav" % name)))
        rf, ef = scipy.io.wavfile.read(str(tmp_path / ("out_flac_%s.wav" % name)))
        assert rw == rf == 44100 and same_bits(ew, ef), name
    with open(tmp_path / "results_wav" / "song.json") as f:
        want = json.load(f)
    with open(tmp_path / "results_flac" / "song.json") as f:
        assert json.load(f) == want
