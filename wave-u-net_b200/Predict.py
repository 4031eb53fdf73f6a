"""Prediction entry point (stand-in for /root/reference/Predict.py:1-17):

    python Predict.py with cfg.full_44KHz model_path=checkpoints/123/123-2000 input_path=mix.npy [output_path=out]

model_path:  a TF-V2 checkpoint prefix (written by Training.py here or by the reference's Saver) or a round-1 .npz.
input_path: a .npy float array [n_frames, n_channels] already at model_config["expected_sr"] (decoding / resampling
audio files needs librosa + ffmpeg, which the reference uses at Evaluate.py:172 and which are out of scope here).
Writes <output_path or input_path>_<source>.npy per source (reference writes _<source>.wav, Evaluate.py:193).

With references_path=<refs.npz> (one [n_frames, n_channels] array per source name, at the mixture's rate) and
results_dir=<dir>, the predictions are also scored with BSS Eval v4 on the GPU (Evaluate.eval_track, the reference's
museval.eval_mus_track at Evaluate.py:71) and written to <results_dir>/<input file name>.json, which
Evaluate.compute_mean_metrics reads.  Mono-model estimates are tiled to the references' channel count (Evaluate.py:66-67).
"""
import os
import sys

import numpy as np

import Config
import Evaluate


def main(cfg, model_path, input_path, output_path=None, references_path=None, results_dir=None):
    model_config = cfg["model_config"]
    mix = np.load(input_path)
    preds = Evaluate.produce_source_estimates(model_config, model_path, mix)
    base = output_path if output_path is not None else input_path
    for name, audio in preds.items():
        np.save("%s_%s.npy" % (base, name), audio)
    if references_path is not None and results_dir is not None:
        with np.load(references_path) as z:
            refs = {name: z[name] for name in z.files}
        nchan = next(iter(refs.values())).shape[1]
        est = {name: np.tile(audio, [1, nchan]) if audio.shape[1] == 1 and nchan > 1 else audio
               for name, audio in preds.items()}
        track = os.path.splitext(os.path.basename(input_path))[0]
        Evaluate.eval_track(refs, est, model_config["expected_sr"], output_dir=results_dir, track_name=track)
    return preds


# the reference's defaults (Predict.py:9-13); its default input is an mp3 - decoding audio files is out of scope here, so
# input_path has to be given
DEFAULT_MODEL_PATH = os.path.join("checkpoints", "full_44KHz", "full_44KHz-236118")


if __name__ == "__main__":
    cfg, extras = Config.parse_command_line(sys.argv[1:])
    if "input_path" not in extras:
        raise SystemExit("Predict.py: input_path=<mix.npy> is required (a float array [n_frames, n_channels] at expected_sr; the "
                         "reference's default, an mp3 of audio_examples/, needs librosa + ffmpeg)\n" + __doc__)
    main(cfg, extras.get("model_path", DEFAULT_MODEL_PATH), extras["input_path"], extras.get("output_path"),
         extras.get("references_path"), extras.get("results_dir"))
