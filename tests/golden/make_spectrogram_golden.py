"""Generate tests/golden/spectrogram/*.npz by executing the UNMODIFIED reference spectrogram U-Net.

Run where the reference checkout is (it is not needed anywhere else):

    python tests/golden/make_spectrogram_golden.py

What runs from the reference, verbatim: Models/UnetSpectrogramSeparator.py (ctor, get_output in test mode, both output
kinds) and Utils.LeakyReLU.  `tensorflow` is replaced by tests/golden/tf_shim.py plus tf_shim_spectrogram.py (eager
torch-CPU, float64).

Fixture content (per case): cfg (json), the mix [B, T, 1] as 16-bit PCM (mix = mix_pcm16 / 32768 in float32, exactly),
param_names in TF creation order, params (kernels on a grid of 2^-5, the rest of 2^-8, stored as float16, which holds them exactly), and the
outputs computed in float64 and stored rounded to float32: magnitudes [B, n, 513] and audio [B, T, 1] of both sources for
the two- and three-layer cases, and only the second source's magnitudes for the six-layer case, so that the file stays
small.  The audio path after the mask is the same at every depth, the first U-Net's wiring is the second's, and the
second one is where the name counters continue across sources.
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

tf_shim_spectrogram.install()
sys.path.insert(0, REF)
import Models.UnetSpectrogramSeparator as RefSpecSep  # noqa: E402  (the reference, unmodified)

_spec = importlib.util.spec_from_file_location("b200_Config", os.path.join(REPO, "wave-u-net_b200", "Config.py"))
Config = importlib.util.module_from_spec(_spec)   # ours: only used to build the model_config dict
_spec.loader.exec_module(Config)

CASES = {
    # name: (named preset, overrides, batch, STFT frames, every output (else the second source's magnitudes only))
    "spec_l2": ("unet_spectrogram", dict(num_layers=2, num_initial_filters=4), 2, 8, True),
    "spec_l3": ("unet_spectrogram_l1", dict(num_layers=3, num_initial_filters=3), 1, 8, True),
    "spec_l6": ("unet_spectrogram", dict(num_layers=6, num_initial_filters=1), 1, 64, False),       # vocals magnitudes
}


def run_case(name, named, overrides, batch, n_frames, full):
    """get_output in test mode after the variables were created and then given non-zero biases, betas and moving means
    and moving variances in [0.5, 2] (float32 values)."""
    cfg = Config.build_config([named], overrides, experiment_id=0)["model_config"]
    sep = RefSpecSep.UnetSpectrogramSeparator(cfg)
    T = 1024 + 768 * (n_frames - 1)
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    # two sawtooths of coprime periods as 16-bit samples: many harmonics, no bin where they line up with the frames, and a
    # repeating pattern that compresses well
    j = np.arange(T)
    saw = [(j % (37 + 12 * b)) * (64 + 8 * b) + (j % 53) * 23 - 1700 for b in range(batch)]
    pcm = np.stack(saw).astype(np.int16)[:, :, None]
    mix = pcm.astype(np.float32) / np.float32(32768)
    x = tf_shim.T(torch.tensor(mix, dtype=torch.float64))
    tf_shim.STATE.reset(seed=1337)
    sep.get_output(x, False, False, reuse=False)
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
    rec = {"cfg_json": np.array(json.dumps(cfg)), "mix_pcm16": pcm, "T": np.int64(T),
           "param_names": np.array(list(tf_shim.STATE.vars.keys()))}
    for spectrogram in ((False, True) if full else (True,)):
        tf_shim.STATE.counters = {}
        with torch.no_grad():
            outs = sep.get_output(x, False, spectrogram, reuse=True)
        for s in (cfg["source_names"] if full else cfg["source_names"][1:]):
            rec["%s/%s" % ("mag" if spectrogram else "audio", s)] = outs[s].t.detach().numpy().astype(np.float32)
    for vname, v in tf_shim.STATE.vars.items():
        rec["param/" + vname] = v.detach().numpy().astype(np.float16)         # exact: the values are on the grid
    os.makedirs(os.path.join(HERE, "spectrogram"), exist_ok=True)
    path = os.path.join(HERE, "spectrogram", name + ".npz")
    np.savez_compressed(path, **rec)
    print("spectrogram/%-12s T=%d params=%d  %d bytes" % (name, T, len(tf_shim.STATE.vars), os.path.getsize(path)))


if __name__ == "__main__":
    for case, args in CASES.items():
        run_case(case, *args)
