"""Tiny MUSDB18-WAV-layout and CCMixter-XML datasets for the dataset tests, written with scipy.io.wavfile.

Stems mix 16-bit PCM and float32 files, 44.1 and 22.05 kHz, mono and stereo; one test track is shorter than T_in of the
small models the tests use (T_in = 151, T_out = 41 for num_layers=2, num_frames=40 with context)."""
import os

import numpy as np
import scipy.io.wavfile

STEMS = ("mixture", "bass", "drums", "other", "vocals")

# name: (rate, frames, channels, sample format)
TRAIN = {
    "d_track": (44100, 1700, 2, "pcm16"),
    "a_track": (44100, 1234, 2, "float32"),
    "c_track": (22050, 700, 1, "pcm16"),
    "b_track": (44100, 1500, 1, "float32"),
    "e_track": (22050, 820, 2, "float32"),
}
TEST = {
    "t_long": (44100, 45000, 2, "pcm16"),       # over one second: BSS Eval scores one frame
    "t_short": (44100, 60, 2, "pcm16"),
    "t_mid": (22050, 500, 2, "float32"),        # MUSDB18 tracks are stereo; mono stems are in TRAIN
}


def _write(path, audio, fmt, rate):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    if fmt == "pcm16":
        data = np.clip(np.round(audio * 32767), -32768, 32767).astype(np.int16)
    else:
        data = audio.astype(np.float32)
    scipy.io.wavfile.write(path, rate, data[:, 0] if data.shape[1] == 1 else data)


def write_track(root, name, rate, frames, channels, fmt, seed):
    rng = np.random.default_rng(seed)
    stems = {s: rng.uniform(-0.45, 0.45, size=(frames, channels)).astype(np.float32) for s in STEMS[1:]}
    mix = stems["bass"] + stems["drums"] + stems["other"] + stems["vocals"]
    stems["mixture"] = np.clip(mix * np.float32(0.6), -1, 1).astype(np.float32)
    for s in STEMS:
        _write(os.path.join(root, name, s + ".wav"), stems[s], fmt, rate)


def write_musdb(root, train=TRAIN, test=TEST):
    for seed, (name, spec) in enumerate(sorted(train.items())):
        write_track(os.path.join(root, "train"), name, *spec, seed=seed)
    for seed, (name, spec) in enumerate(sorted(test.items())):
        write_track(os.path.join(root, "test"), name, *spec, seed=100 + seed)
    return root


def write_ccmixter(root, tracks=(("cc_one", 44100, 1300, 2, "pcm16"), ("cc_two", 22050, 650, 1, "float32"))):
    """An XML of the reference's CCMixter schema plus its files; returns the XML path."""
    db = os.path.join(root, "ccmixter")
    parts = ["<root>", "<databaseFolderPath>%s</databaseFolderPath>" % db, "<tracks>"]
    for seed, (name, rate, frames, channels, fmt) in enumerate(tracks):
        rng = np.random.default_rng(200 + seed)
        voice = rng.uniform(-0.4, 0.4, size=(frames, channels)).astype(np.float32)
        inst = rng.uniform(-0.4, 0.4, size=(frames, channels)).astype(np.float32)
        files = {"Voice": ("source-02.wav", voice), "Instrumental": ("source-01.wav", inst), "Mix": ("mix.wav", voice + inst)}
        parts.append("<track><trackName>%s</trackName><instruments>" % name)
        for inst_name, (fname, audio) in files.items():
            _write(os.path.join(db, name, fname), audio, fmt, rate)
            parts.append("<instrument><instrumentName>%s</instrumentName><relativeFilepath>%s</relativeFilepath></instrument>"
                         % (inst_name, os.path.join(name, fname)))
        parts.append("</instruments></track>")
    parts += ["</tracks>", "</root>"]
    path = os.path.join(root, "CCMixter.xml")
    with open(path, "w") as f:
        f.write("\n".join(parts))
    return path
