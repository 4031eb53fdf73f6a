"""Prediction entry point (stand-in for /root/reference/Predict.py:1-17):

    python Predict.py with cfg.full_44KHz model_path=checkpoints/123/123-2000 input_path=song.wav [output_path=out]
                      [output_format=flac [bit_depth=16|24]] [references_path=refs results_dir=dir [bss_mode=v4|v3]]

model_path:  a TF-V2 checkpoint prefix (written by Training.py here or by the reference's Saver) or a round-1 .npz.
input_path:
  *.wav  16-bit PCM (scaled by 1/32768, as librosa 0.6 loads it) or 32-bit float, mono or multichannel, at any rate.  The
         track is separated at its own rate through Evaluate.predict - resampled to expected_sr and back on the GPU with
         librosa's kaiser_best, as the reference's predict() does (Evaluate.py:60-71) - and every estimate is written to
         <output_path or input_path>_<source>.wav as 32-bit float WAV at the input's rate (librosa.output.write_wav,
         Evaluate.py:193).
  *.flac FLAC, 4 to 24 bits per sample, 1 to 8 channels, decoded on the GPU (wun.read_flac) and converted as the
         reference's ffmpeg path loads it: each sample shifted to 16 bits (left for fewer bits, arithmetically right for
         more) and divided by 32768.  Then as for WAV.
  *.npy  a float array [n_frames, n_channels] already at model_config["expected_sr"]; estimates are written to
         <output_path or input_path>_<source>.npy.
Other audio formats (mp3 and friends, Evaluate.py:172) are out of scope.

output_format=wav (the default) writes the WAV / FLAC input's estimates as above.  output_format=flac writes them as
<output_path or input_path>_<source>.flac instead, encoded on the GPU (wun.write_flac) at bit_depth bits (16, the default,
or 24): each float sample x becomes clamp(rint(x * 2^(bit_depth-1))), so an estimate read back and divided by
2^(bit_depth-1) is within 2^-bit_depth of the float one, except where it clipped at +-1.  bit_depth without
output_format=flac is an error, as is output_format=flac with a .npy input.

With references_path= and results_dir=<dir>, the predictions are also scored with BSS Eval v4 on the GPU
(Evaluate.eval_track, the reference's museval.eval_mus_track at Evaluate.py:71) at the input's rate and written to
<results_dir>/<input file name>.json, which Evaluate.compute_mean_metrics reads.  bss_mode=v3 scores with museval's
mode="v3" instead (distortion filters solved for every frame, as SiSEC 2016 / DSD100-era results were computed); the JSON
layout is the same.  bss_mode without both references_path and results_dir is an error, as is any value but v4 or v3.  references_path is a directory of
<source>.wav or <source>.flac stems at the input's rate, or a .npz with one [n_frames, n_channels] array per source name.  Mono-model
estimates are tiled to the references' channel count (Evaluate.py:66-67).
"""
import glob
import os
import sys

import numpy as np
import scipy.io.wavfile

import Config
import Evaluate


def read_wav(path):
    """(rate, float32 [n_frames, n_channels]) of a WAV file, as the reference's Utils.load(path, sr=None, mono=False) gives
    it: 16-bit PCM divided by 32768 (librosa 0.6's buf_to_float), 32-bit float unchanged.  Other sample formats raise."""
    rate, data = scipy.io.wavfile.read(path)
    if data.dtype == np.int16:
        audio = data.astype(np.float32) / np.float32(32768)
    elif data.dtype == np.float32:
        audio = data
    else:
        raise ValueError("%s: %s WAV samples are not supported (16-bit PCM or 32-bit float only)" % (path, data.dtype))
    return int(rate), np.ascontiguousarray(audio.reshape(audio.shape[0], -1))


def read_flac(path):
    """(rate, float32 [n_frames, n_channels]) of a FLAC file, as the reference's Utils.load gives it through librosa 0.6,
    audioread and `ffmpeg -f s16le`: decoded on the GPU, STREAMINFO MD5 checked, then wun.flac.to_float."""
    import wun
    from wun import flac
    rate, bps, samples = wun.read_flac(path)
    return int(rate), flac.to_float(samples.cpu().numpy(), bps)


def read_audio(path):
    """read_wav for .wav, read_flac for .flac; anything else raises ValueError."""
    ext = os.path.splitext(path)[1].lower()
    if ext == ".wav":
        return read_wav(path)
    if ext == ".flac":
        return read_flac(path)
    raise ValueError("%s: only .wav and .flac audio can be read" % path)


def write_wav(path, audio, rate):
    """32-bit float WAV of `audio` [n_frames, n_channels] at `rate`, as librosa.output.write_wav writes float32 audio."""
    audio = np.asarray(audio, np.float32)
    scipy.io.wavfile.write(path, int(rate), audio[:, 0] if audio.shape[1] == 1 else audio)


def load_references(references_path, rate):
    """name -> [n_frames, n_channels] from a directory of <source>.wav / <source>.flac stems at `rate`, or from a .npz.
    One source given in both formats raises ValueError."""
    if os.path.isdir(references_path):
        refs = {}
        paths = sorted(glob.glob(os.path.join(references_path, "*.wav")) + glob.glob(os.path.join(references_path, "*.flac")))
        names = [os.path.splitext(os.path.basename(p))[0] for p in paths]
        twice = sorted(set(n for n in names if names.count(n) > 1))
        if twice:
            raise ValueError("%s: sources %s are given both as .wav and as .flac" % (references_path, twice))
        for name, path in zip(names, paths):
            sr, audio = read_audio(path)
            if sr != rate:
                raise ValueError("%s is at %d Hz, the mixture at %d Hz" % (path, sr, rate))
            refs[name] = audio
        return refs
    with np.load(references_path) as z:
        return {name: z[name] for name in z.files}


def write_flac(path, audio, rate, bit_depth):
    """`audio` [n_frames, n_channels] as a FLAC file of bit_depth bits, quantised and encoded on the GPU."""
    import torch
    import wun
    wun.write_flac(torch.from_numpy(np.ascontiguousarray(audio, np.float32)).cuda(), rate, bit_depth, path)


OUTPUT_FORMATS = ("wav", "flac")
BIT_DEPTHS = (16, 24)


def output_options(output_format=None, bit_depth=None):
    """(format, bit depth or None) from the command line's output_format= and bit_depth=; ValueError for anything else."""
    fmt = "wav" if output_format is None else str(output_format).lower()
    if fmt not in OUTPUT_FORMATS:
        raise ValueError("output_format=%s: must be one of %s" % (output_format, ", ".join(OUTPUT_FORMATS)))
    if fmt != "flac":
        if bit_depth is not None:
            raise ValueError("bit_depth= is only meaningful with output_format=flac")
        return fmt, None
    depth = 16 if bit_depth is None else bit_depth
    if isinstance(depth, bool) or not isinstance(depth, int) or depth not in BIT_DEPTHS:
        raise ValueError("bit_depth=%s: must be 16 or 24" % (bit_depth,))
    return fmt, depth


def scoring_options(references_path=None, results_dir=None, bss_mode=None):
    """(score?, BSS Eval mode) from the command line's references_path=, results_dir= and bss_mode=; ValueError for a
    mode other than v4 / v3, or for bss_mode without both references_path and results_dir."""
    score = references_path is not None and results_dir is not None
    if bss_mode is None:
        return score, "v4"
    if not score:
        raise ValueError("bss_mode= is only meaningful with references_path= and results_dir=")
    mode = str(bss_mode).lower()
    if mode not in Evaluate.BSS_MODES:
        raise ValueError("bss_mode=%s: must be one of %s" % (bss_mode, ", ".join(Evaluate.BSS_MODES)))
    return score, mode


def main(cfg, model_path, input_path, output_path=None, references_path=None, results_dir=None, output_format="wav",
         bit_depth=None, bss_mode=None):
    output_format, bit_depth = output_options(output_format, bit_depth)
    score, mode = scoring_options(references_path, results_dir, bss_mode)
    model_config = cfg["model_config"]
    base = output_path if output_path is not None else input_path
    track = os.path.splitext(os.path.basename(input_path))[0]
    if input_path.lower().endswith((".wav", ".flac")):
        rate, mix = read_audio(input_path)
        refs = load_references(references_path, rate) if score else None
        preds = Evaluate.predict(model_config, Evaluate.load_separator(model_config, model_path), mix, rate,
                                 references=refs, results_dir=results_dir, track_name=track, mode=mode)
        for name, audio in preds.items():
            if output_format == "flac":
                write_flac("%s_%s.flac" % (base, name), audio, rate, bit_depth)
            else:
                write_wav("%s_%s.wav" % (base, name), audio, rate)
        return preds
    if output_format != "wav":
        raise ValueError("output_format=%s: .npy input writes .npy estimates" % output_format)
    mix = np.load(input_path)
    preds = Evaluate.produce_source_estimates(model_config, model_path, mix)
    for name, audio in preds.items():
        np.save("%s_%s.npy" % (base, name), audio)
    if score:
        refs = load_references(references_path, model_config["expected_sr"])
        nchan = next(iter(refs.values())).shape[1]
        est = {name: np.tile(audio, [1, nchan]) if audio.shape[1] == 1 and nchan > 1 else audio
               for name, audio in preds.items()}
        Evaluate.eval_track(refs, est, model_config["expected_sr"], output_dir=results_dir, track_name=track, mode=mode)
    return preds


# the reference's defaults (Predict.py:9-13); its default input is an mp3, which is not read here, so input_path has to be
# given
DEFAULT_MODEL_PATH = os.path.join("checkpoints", "full_44KHz", "full_44KHz-236118")


if __name__ == "__main__":
    cfg, extras = Config.parse_command_line(sys.argv[1:])
    if "input_path" not in extras:
        raise SystemExit("Predict.py: input_path=<song.wav, song.flac or mix.npy> is required (the reference's default, an "
                         "mp3 of audio_examples/, is not a format read here); output_format=flac [bit_depth=16|24] writes "
                         "FLAC estimates; references_path= results_dir= [bss_mode=v4|v3] scores them\n" + __doc__)
    try:
        output_options(extras.get("output_format"), extras.get("bit_depth"))
        scoring_options(extras.get("references_path"), extras.get("results_dir"), extras.get("bss_mode"))
    except ValueError as ex:
        raise SystemExit("Predict.py: %s\n%s" % (ex, __doc__))
    main(cfg, extras.get("model_path", DEFAULT_MODEL_PATH), extras["input_path"], extras.get("output_path"),
         extras.get("references_path"), extras.get("results_dir"), extras.get("output_format", "wav"),
         extras.get("bit_depth"), extras.get("bss_mode"))
