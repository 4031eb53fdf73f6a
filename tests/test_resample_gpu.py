"""kaiser_best resampling on the GPU (wun.resample, csrc/kernels_resample.cu) bit for bit against the numpy oracle
(oracle/resample_oracle.py), and the reference's predict() built on it (Evaluate.predict, Predict.py on WAV files)."""
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
from oracle import resample_oracle as R
from oracle import wave_unet_oracle as O

pytestmark = pytest.mark.gpu

RATIOS = [(44100, 22050), (22050, 44100), (48000, 22050), (22050, 48000), (44100, 8192), (16000, 22050)]


def oracle(x, sr_in, sr_out):
    win, delta = wun.resample_tables(sr_in, sr_out)
    return R.resample(x, sr_in, sr_out, win, delta, wun.KAISER_BEST_PRECISION)


def gpu(x, sr_in, sr_out):
    return wun.resample(torch.from_numpy(np.ascontiguousarray(x)).cuda(), sr_in, sr_out).cpu().numpy()


def same_bits(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def noise(rng, n, nchan):
    return (rng.standard_normal((n, nchan)) * 0.2).astype(np.float32)


@pytest.mark.parametrize("sr_in,sr_out", RATIOS)
@pytest.mark.parametrize("nchan", [1, 2])
def test_bit_for_bit_against_oracle(sr_in, sr_out, nchan):
    rng = np.random.default_rng(sr_in * 3 + sr_out + nchan)
    ratio = float(sr_out) / sr_in
    lengths = [n for n in list(range(1, 41)) + [97, 255, 256, 1000, 2047, 4000] if int(n * ratio) >= 1]
    for n in lengths:
        x = noise(rng, n, nchan)
        got = gpu(x, sr_in, sr_out)
        assert same_bits(got, oracle(x, sr_in, sr_out)), n
        assert same_bits(gpu(x, sr_in, sr_out), got), n


@pytest.mark.parametrize("sr_in,sr_out", [(44100, 22050), (22050, 44100), (48000, 22050)])
def test_thirty_seconds_bit_for_bit(sr_in, sr_out):
    rng = np.random.default_rng(7)
    x = noise(rng, 30 * sr_in, 2)
    got = gpu(x, sr_in, sr_out)
    assert same_bits(got, oracle(x, sr_in, sr_out))
    assert same_bits(gpu(x, sr_in, sr_out), got)


def test_time_register_exact_over_long_runs():
    """More than 2^23 output frames at 48000 -> 44100, where t * inc differs from the sequential sum almost everywhere: the
    kernel's closed form must still give the oracle's bits, here at the last frames, at every power of two of the time
    register and at random frames."""
    sr_in, sr_out = 48000, 44100
    n_in = 9_200_000
    ratio = float(sr_out) / sr_in
    n_valid = int(n_in * ratio)
    assert n_valid > 2 ** 23
    tr = R.time_register(n_valid, ratio)
    assert np.count_nonzero(np.arange(n_valid) * (1.0 / ratio) != tr) > n_valid // 2
    rng = np.random.default_rng(8)
    x = noise(rng, n_in, 1)
    got = gpu(x, sr_in, sr_out)
    crossings = np.searchsorted(tr, 2.0 ** np.arange(0, 24))
    frames = np.unique(np.concatenate([np.arange(n_valid - 5000, n_valid), rng.integers(0, n_valid, 20000),
                                       (crossings[:, None] + np.arange(-3, 4)).ravel().clip(0, n_valid - 1)]))
    win, delta = wun.resample_tables(sr_in, sr_out)
    want = R.resample_f(x, ratio, win, delta, wun.KAISER_BEST_PRECISION, frames=frames)
    assert same_bits(got[frames], want)
    assert np.all(got[n_valid:] == 0)


def test_equal_rates_and_invalid_inputs():
    x = torch.zeros((100, 2), device="cuda")
    assert wun.resample(x, 22050, 22050) is x
    with pytest.raises(ValueError):
        wun.resample(x[:1].contiguous(), 44100, 22050)
    y = torch.empty((50, 2), device="cuda")
    w = torch.zeros(32769, dtype=torch.float64, device="cuda")
    lib = wun.lib
    assert lib.wun_resample(x.data_ptr(), 100, 3, 44100, 22050, w.data_ptr(), w.data_ptr(), 32769, 512, y.data_ptr(), 50, None) == wun.WUN_E_INVALID
    assert lib.wun_resample(x.data_ptr(), 100, 2, 44100, 22050, w.data_ptr(), w.data_ptr(), 32769, 512, y.data_ptr(), 51, None) == wun.WUN_E_INVALID
    assert lib.wun_resample(x.data_ptr(), 100, 2, 0, 22050, w.data_ptr(), w.data_ptr(), 32769, 512, y.data_ptr(), 50, None) == wun.WUN_E_INVALID
    assert lib.wun_resample(x.data_ptr(), 1, 2, 44100, 22050, w.data_ptr(), w.data_ptr(), 32769, 512, y.data_ptr(), 1, None) == wun.WUN_E_INVALID


def small_model(named, seed):
    cfg = Config.build_config(named, dict(num_layers=3, num_frames=64), experiment_id=0)
    mc = cfg["model_config"]
    t_in, _ = O.get_padding(mc, 64)
    sep = UnetAudioSeparator(mc)
    sep.load_variables(O.init_params(mc, seed=seed), input_frames=t_in)
    return cfg, mc, sep


def composed(mc, sep, audio, rate):
    """The reference's predict() from its parts: oracle resample, predict_track, oracle resample back, cut, tile."""
    sr = mc["expected_sr"]
    mix = Evaluate._model_channels(mc, audio)
    preds = Evaluate.predict_track(mc, sep, oracle(mix, rate, sr))
    out = {}
    for name, est in preds.items():
        est = oracle(np.ascontiguousarray(est), sr, rate)[:audio.shape[0]]
        out[name] = np.tile(est, [1, audio.shape[1]]) if mc["mono_downmix"] and audio.shape[1] > 1 else est
    return out


@pytest.mark.parametrize("named", [["baseline_stereo"], []])
def test_predict_matches_composition(named, tmp_path):
    cfg, mc, sep = small_model(named, seed=4)
    assert mc["expected_sr"] == 22050
    rng = np.random.default_rng(9)
    refs = {n: noise(rng, 3 * 44100 + 37, 2) for n in mc["source_names"]}
    mix = sum(refs.values()).astype(np.float32)
    got = Evaluate.predict(mc, sep, mix, 44100, references=refs, results_dir=str(tmp_path), track_name="song")
    want = composed(mc, sep, mix, 44100)
    assert list(got) == list(mc["source_names"])
    for name in got:
        assert got[name].shape == mix.shape and same_bits(got[name], want[name]), name
    with open(tmp_path / "song.json") as f:
        scores = json.load(f)
    assert scores == Evaluate.eval_track(refs, got, 44100)
    assert len(scores["targets"][0]["frames"]) == 3


def test_predict_at_expected_rate_is_predict_track():
    cfg, mc, sep = small_model(["baseline_stereo"], seed=5)
    mix = noise(np.random.default_rng(10), 22050 + 555, 2)
    got = Evaluate.predict(mc, sep, mix, 22050)
    want = Evaluate.predict_track(mc, sep, mix)
    for name in want:
        assert same_bits(got[name], np.ascontiguousarray(want[name])), name


def test_predict_cli_on_wav(tmp_path):
    cfg, mc, sep = small_model(["baseline_stereo"], seed=6)
    model = Training.save_checkpoint(str(tmp_path / "model.npz"), sep)
    rng = np.random.default_rng(11)
    stems = {n: noise(rng, 2 * 44100 + 99, 2) for n in mc["source_names"]}
    pcm = np.clip(np.round(sum(stems.values()) * 32768), -32768, 32767).astype(np.int16)
    scipy.io.wavfile.write(str(tmp_path / "song.wav"), 44100, pcm)
    os.makedirs(tmp_path / "stems")
    for name, audio in stems.items():
        scipy.io.wavfile.write(str(tmp_path / "stems" / ("%s.wav" % name)), 44100, audio)
    preds = Predict.main(cfg, model, str(tmp_path / "song.wav"), output_path=str(tmp_path / "out"),
                         references_path=str(tmp_path / "stems"), results_dir=str(tmp_path / "results"))
    want = Evaluate.predict(mc, Evaluate.load_separator(mc, model), pcm.astype(np.float32) / 32768, 44100)
    for name in mc["source_names"]:
        rate, est = scipy.io.wavfile.read(str(tmp_path / ("out_%s.wav" % name)))
        assert rate == 44100 and same_bits(est, want[name]) and same_bits(preds[name], want[name]), name
    with open(tmp_path / "results" / "song.json") as f:
        scores = json.load(f)
    assert scores == Evaluate.eval_track(stems, want, 44100)
