"""The spectrogram U-Net baselines (U7 / U7a) on the GPU (csrc/kernels_spec.cu, csrc/spec.cu): the engine against the
fixtures of the reference's own UnetSpectrogramSeparator and against the float64 oracle at the presets' full size, bit
reproducibility across runs and batch placement, windowed separation, Test.test with both losses, and Predict on a WAV.

Tolerance.  Every kernel accumulates in float32 in a fixed order: the convolutions sum up to 25 * 512 = 12 800 products,
the DFTs 1 024.  With unit round-off u = 6e-8 a sum of m terms is off by at most ~m*u relative to the sum of magnitudes
and typically ~sqrt(m)*u (~7e-6 for m = 12 800); eleven layers in a row, batch norm with variances down to 0.5 and the
mask's product with the mixture carry a few such errors into the output.  The checks allow 2e-4 of the largest output
magnitude (audio or spectrogram), ~30x the typical single-layer error and far below any wiring mistake (a wrong tap,
channel half or window changes outputs by O(1) of their scale).  The largest observed errors are printed (-s)."""
import os

import numpy as np
import pytest
import scipy.io.wavfile
import torch

import Config
import Datasets
import Evaluate
import Predict
import TFCheckpoint
import Test
import wun
from Models.UnetSpectrogramSeparator import UnetSpectrogramSeparator
from dataset_fixtures import write_musdb
from oracle import spectrogram_oracle as S

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "spectrogram")
CASES = ["spec_l2", "spec_l3", "spec_l6"]
PRESET_FRAMES = 768 * 127 + 1024
TOL = 2e-4


def mc(named="unet_spectrogram", **kw):
    return Config.build_config([named], kw, experiment_id=0)["model_config"]


def separator(cfg, params, T):
    sep = UnetSpectrogramSeparator(cfg)
    sep.load_variables(params, device=torch.device("cuda"), num_frames=T)
    return sep


def rel_err(got, want):
    return float(np.abs(np.asarray(got, np.float64) - want).max() / np.abs(want).max())


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def signal(rng, B, T):
    t = np.arange(T) / 8192.0
    x = [0.3 * np.sin(2 * np.pi * rng.uniform(80, 900) * t) + rng.uniform(-0.4, 0.4, T) for _ in range(B)]
    return np.stack(x)[:, :, None].astype(np.float32)


@pytest.mark.parametrize("name", CASES)
def test_engine_matches_reference_fixtures(name):
    import json
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    cfg = json.loads(str(z["cfg_json"]))
    params = {k[len("param/"):]: z[k].astype(np.float32) for k in z.files if k.startswith("param/")}
    sep = separator(cfg, params, int(z["T"]))
    mix = torch.from_numpy(z["mix_pcm16"].astype(np.float32) / np.float32(32768)).cuda()
    for spectrogram, key in ((False, "audio"), (True, "mag")):
        out = sep.get_output(mix, False, spectrogram, reuse=True)
        for s in [s for s in cfg["source_names"] if "%s/%s" % (key, s) in z.files]:
            want = z["%s/%s" % (key, s)]
            got = out[s].cpu().numpy()
            assert got.shape == want.shape
            e = rel_err(got, want)
            print("fixture %s %s %s: max error %.2e of max |output|" % (name, key, s, e))
            assert e < TOL, (name, key, s, e)


@pytest.mark.parametrize("preset", ["unet_spectrogram", "unet_spectrogram_l1"])
def test_presets_at_full_size_match_oracle_and_repeat_bits(preset):
    cfg = mc(preset)
    params = S.random_params(cfg["num_layers"], cfg["num_initial_filters"], seed=11 if preset == "unet_spectrogram" else 12)
    sep = separator(cfg, params, PRESET_FRAMES)
    mix_np = signal(np.random.default_rng(3), 4, PRESET_FRAMES)
    mix = torch.from_numpy(mix_np).cuda()
    eng = sep.engine(num_frames=PRESET_FRAMES)
    for spectrogram, key in ((False, "audio"), (True, "mag")):
        want = S.forward(params, mix_np, cfg["num_layers"], cfg["source_names"], return_spectrogram=spectrogram)
        out = eng.forward(sep.params, mix, False, return_spectrogram=spectrogram).cpu().numpy()
        again = eng.forward(sep.params, mix, False, return_spectrogram=spectrogram).cpu().numpy()
        one = eng.forward(sep.params, mix[2:3].contiguous(), False, return_spectrogram=spectrogram).cpu().numpy()
        assert np.array_equal(bits(out), bits(again)), "two runs differ"
        assert np.array_equal(bits(out[:, 2:3]), bits(one)), "batch 1 and batch 4 differ for the same window"
        for k, s in enumerate(cfg["source_names"]):
            e = rel_err(out[k], want[s])
            print("%s %s %s: max error %.2e of max |output| %.3g" % (preset, key, s, e, np.abs(want[s]).max()))
            assert e < TOL, (preset, key, s, e)


def small(seed, L=2, F=4, n=4, **kw):
    T = 1024 + 768 * (n - 1)
    cfg = mc(num_layers=L, num_initial_filters=F, num_frames=T, **kw)
    params = S.random_params(L, F, seed)
    return cfg, params, T


def test_separate_on_device_matches_windowed_oracle():
    cfg, params, T = small(21)
    sep = separator(cfg, params, T)
    n_mix = 3 * T + 1000                                     # not a whole number of windows: the last one is shifted back
    mix = signal(np.random.default_rng(4), 1, n_mix)[0]
    got = Evaluate._separate_on_device(cfg, sep, torch.from_numpy(mix), batch_windows=16).cpu().numpy()
    got1 = Evaluate._separate_on_device(cfg, sep, torch.from_numpy(mix), batch_windows=1).cpu().numpy()
    assert np.array_equal(bits(got), bits(got1))
    want = np.zeros((2, n_mix, 1))
    for start in Evaluate.window_starts(n_mix, T):
        o = S.forward(params, mix[None, start:start + T], cfg["num_layers"], cfg["source_names"])
        for k, s in enumerate(cfg["source_names"]):
            want[k, start:start + T] = o[s][0]
    e = rel_err(got, want)
    print("windowed separation: max error %.2e" % e)
    assert got.shape == (2, n_mix, 1) and e < TOL


@pytest.mark.parametrize("named", ["unet_spectrogram", "unet_spectrogram_l1"])
def test_test_loss_matches_oracle_running_mean(tmp_path, named):
    cfg, params, T = small(31, n=4, batch_size=2)
    cfg = dict(cfg, raw_audio_loss=(named == "unet_spectrogram"))
    train = {"a_tr": (8192, 12000, 1, "float32"), "b_tr": (16384, 30000, 2, "float32"), "c_tr": (8192, 9000, 1, "pcm16")}
    test = {"t_one": (8192, 14000, 2, "float32"), "t_two": (8192, 11000, 1, "float32")}
    musdb = write_musdb(str(tmp_path / "musdb"), train=train, test=test)
    ds = Datasets.load_musdb(cfg, T, T, musdb, None, valid_tracks=2)
    sep = separator(cfg, params, T)
    B = 2
    got = Test.test(cfg, "test", "0", None, dataset=ds, separator=sep)
    again = Test.test(cfg, "test", "0", None, dataset=ds, separator=sep)
    assert bits(np.float64(got)).tobytes() == bits(np.float64(again)).tobytes()
    p = ds.partitions["test"]
    pos = Datasets.snippet_positions(p.offsets, p.lengths, T, T, B)
    assert len(pos) // B >= 3                                 # the captured graph is replayed more than once
    pool = p.pool.cpu().numpy()
    total = 0.0
    for n, b0 in enumerate(range(0, len(pos), B), start=1):
        s = pos[b0:b0 + B]
        mix = np.stack([pool[-1, f:f + T] for f in s])
        tg = [np.stack([pool[k, f:f + T] for f in s]) for k in range(2)]
        if cfg["raw_audio_loss"]:
            est = S.forward(params, mix, cfg["num_layers"], cfg["source_names"])
            curr = sum(np.mean((tg[k] - est[name]) ** 2) for k, name in enumerate(cfg["source_names"])) / 2
        else:
            est = S.forward(params, mix, cfg["num_layers"], cfg["source_names"], return_spectrogram=True)
            curr = S.magnitude_l1(tg, [est[name] for name in cfg["source_names"]])
        total = total + (1.0 / n) * (curr - total)
    print("%s test loss %.9g (oracle %.9g)" % (named, got, total))
    assert abs(got - total) <= 1e-4 * abs(total)


def test_predict_main_on_stereo_wav(tmp_path):
    cfg, params, T = small(41, L=3, F=3, n=8)
    prefix = TFCheckpoint.write_checkpoint(str(tmp_path / "u7-10"), TFCheckpoint.separator_tensors(params, global_step=10))
    rng = np.random.default_rng(5)
    audio = rng.uniform(-0.5, 0.5, size=(2 * 44100 + 77, 2)).astype(np.float32)
    scipy.io.wavfile.write(str(tmp_path / "song.wav"), 44100, audio)
    preds = Predict.main({"model_config": cfg}, prefix, str(tmp_path / "song.wav"), output_path=str(tmp_path / "out"))
    for name in cfg["source_names"]:
        rate, est = scipy.io.wavfile.read(str(tmp_path / ("out_%s.wav" % name)))
        assert rate == 44100 and est.dtype == np.float32 and est.shape == audio.shape, (name, rate, est.dtype, est.shape)
        assert np.array_equal(bits(est), bits(preds[name])) and np.isfinite(est).all()
        assert np.array_equal(est[:, 0], est[:, 1])           # a mono model's estimate tiled to the input's channels
