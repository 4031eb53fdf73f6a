"""Generate tests/golden/spectrogram_train/*.npz by executing the UNMODIFIED reference spectrogram U-Net in training mode.

Run where the reference checkout is (it is not needed anywhere else):

    python tests/golden/make_spectrogram_train_golden.py

What runs from the reference, verbatim: Models/UnetSpectrogramSeparator.py (ctor, get_output with training=True and
return_spectrogram = not raw_audio_loss, as Training.py:47 calls it) and Utils.LeakyReLU.  `tensorflow` is replaced by
tests/golden/tf_shim.py, tf_shim_spectrogram.py and tf_shim_spectrogram_train.py (eager torch-CPU, float64).  The loss is
Training.py:50-63 restated below; torch autograd differentiates the graph the reference code built.

Fixture content (per case): cfg (json), the mix [B, T, 1] and both targets [2, B, T, 1] as 16-bit PCM (value = pcm / 32768
in float32, exactly), params on a grid (kernels 2^-5, the rest 2^-8, stored as float16, which holds them exactly), the
dropout keep masks per (source, level) as packed bits with their shapes (the engine's hash at a recorded seed and dropout
step, so that the engine can run the same step), the loss and the moving statistics after the
step's UPDATE_OPS in float64, and every trainable variable's gradient rounded to float32 (so that each file stays under
200 kB).
"""
import importlib.util
import json
import os
import sys
import zlib

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
REF = "/root/reference"
sys.path.insert(0, HERE)

import tf_shim  # noqa: E402
import tf_shim_spectrogram  # noqa: E402
import tf_shim_spectrogram_train  # noqa: E402

tf_shim_spectrogram_train.install()
sys.path.insert(0, REF)
import Models.UnetSpectrogramSeparator as RefSpecSep  # noqa: E402  (the reference, unmodified)

sys.path.insert(0, REPO)
from oracle.spectrogram_train_oracle import keep_masks  # noqa: E402  (ours: the engine's dropout hash)

_spec = importlib.util.spec_from_file_location("b200_Config", os.path.join(REPO, "wave-u-net_b200", "Config.py"))
Config = importlib.util.module_from_spec(_spec)   # ours: only used to build the model_config dict
_spec.loader.exec_module(Config)

TRAIN = tf_shim_spectrogram_train.TRAIN
DROPOUT_SEED, DROPOUT_STEP = 1337, 5        # the keep masks are the engine's for this seed and dropout step

CASES = {
    # name: (named preset, overrides, batch, STFT frames)
    "train_l2_u7": ("unet_spectrogram", dict(num_layers=2, num_initial_filters=4), 2, 8),
    "train_l3_u7a": ("unet_spectrogram_l1", dict(num_layers=3, num_initial_filters=3), 1, 8),
    "train_l5_u7": ("unet_spectrogram", dict(num_layers=5, num_initial_filters=1), 1, 32),     # dropped and undropped levels
}


def pcm(T, batch, a, b):
    """Two sawtooths of coprime periods as 16-bit samples (many harmonics, compress well)."""
    j = np.arange(T)
    saw = [(j % (a + 12 * i)) * (48 + 8 * i) + (j % b) * 19 - 1300 for i in range(batch)]
    return np.stack(saw).astype(np.int16)[:, :, None]


def separator_loss(cfg, outs, targets):
    """Training.py:50-63: MSE on audio, or for the spectrogram U-Net without raw_audio_loss the mean absolute difference
    of the targets' STFT magnitudes (frame 1024, hop 768, periodic Hann) and the estimated magnitudes; over num_sources."""
    loss = 0
    for k, key in enumerate(cfg["source_names"]):
        real = targets[k]
        if cfg["network"] == "unet_spectrogram" and not cfg["raw_audio_loss"]:
            frames = real[:, :, 0].unfold(-1, 1024, 768)
            window = 0.5 - 0.5 * torch.cos(2 * np.pi * torch.arange(1024, dtype=torch.float64) / 1024)
            real_mag = torch.fft.rfft(frames * window, n=1024).abs()
            loss = loss + torch.mean(torch.abs(real_mag - outs[key].t))
        else:
            loss = loss + torch.mean((real - outs[key].t) ** 2)
    return loss / float(cfg["num_sources"])


def run_case(name, named, overrides, batch, n_frames):
    cfg = Config.build_config([named], overrides, experiment_id=0)["model_config"]
    sep = RefSpecSep.UnetSpectrogramSeparator(cfg)
    T = 1024 + 768 * (n_frames - 1)
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    mix_pcm = pcm(T, batch, 37, 53)
    tg_pcm = np.stack([pcm(T, batch, 29, 41), pcm(T, batch, 43, 31)])
    mix = tf_shim.T(torch.tensor(mix_pcm.astype(np.float32) / np.float32(32768), dtype=torch.float64))
    targets = [torch.tensor(t.astype(np.float32) / np.float32(32768), dtype=torch.float64) for t in tg_pcm]
    tf_shim.STATE.reset(seed=1337)
    sep.get_output(mix, False, False, reuse=False)                      # creates the variables
    for vname, v in tf_shim.STATE.vars.items():
        shape = tuple(v.shape)
        if vname.endswith("/kernel"):
            val = v.detach().numpy()
        elif vname.endswith("/moving_variance"):
            val = rng.uniform(0.5, 2.0, size=shape)
        else:
            val = rng.uniform(-0.1, 0.1, size=shape)
        grid = 32 if vname.endswith("/kernel") else 256
        with torch.no_grad():
            v.copy_(torch.tensor(np.round(val * grid) / grid))
    params = {n: v.detach().numpy().copy() for n, v in tf_shim.STATE.vars.items()}
    L, Fi = cfg["num_layers"], cfg["num_initial_filters"]
    rec = {"cfg_json": np.array(json.dumps(cfg)), "mix_pcm16": mix_pcm, "target_pcm16": tg_pcm, "T": np.int64(T),
           "dropout_seed": np.uint64(DROPOUT_SEED), "dropout_step": np.int64(DROPOUT_STEP)}
    TRAIN.reset()
    for k in range(2):                                                  # the order get_output calls dropout in
        for i in range(min(3, L - 1)):
            d = L - 2 - i
            shape = (batch, n_frames >> (d + 1), 512 >> (d + 1), 2 * Fi * 2 ** d)
            keep = keep_masks(DROPOUT_SEED, DROPOUT_STEP, k, d, shape)
            TRAIN.masks.append(keep)
            rec["keep/%d/%d" % (k, d)] = np.packbits(keep.reshape(-1))
            rec["keep_shape/%d/%d" % (k, d)] = np.array(shape, np.int64)
    tf_shim.STATE.counters = {}
    outs = sep.get_output(mix, True, not cfg["raw_audio_loss"], reuse=True)
    assert not TRAIN.masks
    loss = separator_loss(cfg, outs, targets)
    loss.backward()
    rec["loss"] = np.float64(loss.item())
    for vname, v in tf_shim.STATE.vars.items():
        rec["param/" + vname] = params[vname].astype(np.float16)       # exact: the values are on the grid
        if not vname.endswith(("/moving_mean", "/moving_variance")):
            rec["grad/" + vname] = v.grad.numpy().astype(np.float32)
    for vname, val in TRAIN.moving.items():
        rec["moving/" + vname] = val
    os.makedirs(os.path.join(HERE, "spectrogram_train"), exist_ok=True)
    path = os.path.join(HERE, "spectrogram_train", name + ".npz")
    np.savez_compressed(path, **rec)
    print("spectrogram_train/%-14s T=%d loss=%.9g  %d bytes" % (name, T, loss.item(), os.path.getsize(path)))


if __name__ == "__main__":
    for case, args in CASES.items():
        run_case(case, *args)
