"""Windowed inference with the H100 engine: drop-in for the tiling half of the reference's Evaluate.py.

predict_track() keeps the semantics of /root/reference/Evaluate.py:82-145 exactly -
  mono-mix or channel duplication (:98-102), zero-extension of short inputs (:107-111), (T_in-T_out)//2 context
  padding on both sides (:121-122), hop = T_out, the LAST window shifted back to end at the final frame (:127-128),
  plain overwrite of overlapping frames (:138-139), removal of the extension (:142-143)
- but the windows, which the reference feeds one by one through sess.run (:134), are gathered ON THE DEVICE, pushed
through the network as batches, and scattered back on the device; with torch.distributed initialised the window list
is split over the ranks (no collective on the data path, results all-gathered at the end).

predict_track works on arrays already at model_config["expected_sr"]; predict() is the reference's predict() (Evaluate.py:
60-71) on an array at any rate, resampling on the GPU with librosa's kaiser_best (wun.resample) on the way in and out.
Scoring is here: evaluate() / eval_track() replace museval.evaluate / museval.eval_mus_track (Evaluate.py:71) with BSS
Eval v4 on the GPU (wun.bss_eval), or with museval's mode="v3" (filters solved per frame) when asked for, and
compute_mean_metrics is the reference's (Evaluate.py:195-232).  bss_eval and bss_eval_sources / bss_eval_images (and their
_framewise forms) are museval.metrics' functions of those names, with the permutation search and the "sources" decomposition,
on the GPU as well; the MUSDB path above does not use them, since museval never permutes named targets.
produce_musdb_source_estimates runs them over the MUSDB18 WAV layout.  Audio decoding beyond WAV (Predict.py) and the musdb
package are out of scope (SURVEY section 2).
"""
import glob
import json
import os
from collections import OrderedDict

import numpy as np

from wun import parallel


def window_starts(n_frames, t_out):
    """Start frame of every window (Evaluate.py:125-128)."""
    starts = []
    for pos in range(0, n_frames, t_out):
        if pos + t_out > n_frames:
            pos = n_frames - t_out
        starts.append(pos)
    return starts


def predict_track(model_config, separator, mix_audio, batch_windows=16, device="cuda"):
    """mix_audio: float array [n_frames, n_channels] at expected_sr.  `separator`: a
    Models.UnetAudioSeparator.UnetAudioSeparator or Models.UnetSpectrogramSeparator.UnetSpectrogramSeparator holding
    variables.  Returns OrderedDict name -> [n_frames, C]."""
    import torch
    assert len(mix_audio.shape) == 2
    mix_audio = _model_channels(model_config, mix_audio)
    preds = _separate_on_device(model_config, separator, torch.from_numpy(np.ascontiguousarray(mix_audio)), batch_windows,
                                device)
    result = preds.cpu().numpy()
    return OrderedDict((name, result[k]) for k, name in enumerate(model_config["source_names"]))


def _model_channels(model_config, mix_audio):
    """The mono downmix, or the tiling of a mono input to stereo, that predict_track applies (Evaluate.py:98-102)."""
    mix_audio = np.asarray(mix_audio, dtype=np.float32)
    if model_config["mono_downmix"]:
        return np.mean(mix_audio, axis=1, keepdims=True)
    if mix_audio.shape[1] == 1:
        return np.tile(mix_audio, [1, 2])
    return mix_audio


def _separate_on_device(model_config, separator, mix, batch_windows=16, device="cuda"):
    """predict_track's device half: `mix` a float32 tensor [n_frames, C] at expected_sr with the model's channel count
    (host or device).  Returns the estimates as a float32 CUDA tensor [K, n_frames, C] in source_names order."""
    import torch
    in_shape, out_shape = separator.get_padding(np.array([1, model_config["num_frames"], 0]))
    t_in, t_out = int(in_shape[1]), int(out_shape[1])
    n_mix, C = int(mix.shape[0]), int(mix.shape[1])
    n_frames = max(n_mix, t_in)          # zero-extension of short inputs, cut off again at the end (Evaluate.py:107-111,142-143)
    pad = (t_in - t_out) // 2                                   # context on both sides (Evaluate.py:121-122), zero-filled ON the device

    eng = separator.engine(input_frames=t_in)
    names = list(model_config["source_names"])
    K = len(names)
    starts_all = window_starts(n_frames, t_out)
    rank, ws = parallel.world()
    lo, hi = parallel.shard_range(len(starts_all), rank, ws)

    padded_d = torch.zeros((n_frames + 2 * pad, C), dtype=torch.float32, device=device)
    padded_d[pad:pad + n_mix].copy_(mix)        # (a host-side np.pad of a 3-minute track costs as much as a third of the
    # whole separation)
    preds_local = torch.empty((K, hi - lo, t_out, C), dtype=torch.float32, device=device)
    st_all = torch.tensor(starts_all, dtype=torch.int64, device=device)          # one upload; the batches take slices of it
    for b0 in range(lo, hi, batch_windows):
        b1 = min(b0 + batch_windows, hi)
        st = st_all[b0:b1]
        batch = torch.empty((b1 - b0, t_in, C), dtype=torch.float32, device=device)
        eng.gather_windows(padded_d, st, batch)
        separator._ensure_params(eng, padded_d.device, create=False)
        out = eng.forward(separator.params, batch, training=False)          # [K, nb, T_out, C]
        preds_local[:, b0 - lo:b1 - lo] = out
    preds_all = parallel.gather_window_predictions(preds_local, len(starts_all))
    # scatter (overwrite; the shifted last window wins where it overlaps its predecessor)
    preds = torch.zeros((K, n_frames, C), dtype=torch.float32, device=device)
    eng.scatter_windows(preds_all.contiguous(), st_all, preds)
    return preds[:, :n_mix]


def predict(model_config, separator, audio, rate, references=None, results_dir=None, track_name=None, mode="v4"):
    """The reference's predict() (Evaluate.py:60-71) on an array: `audio` float [n_frames, n_channels] at `rate` Hz.
    The mixture is downmixed or tiled to the model's channels, resampled to expected_sr with wun.resample (librosa's
    kaiser_best, Evaluate.py:104), separated, and every estimate is resampled back to `rate`, cut to n_frames and, for a
    mono model and a multichannel input, tiled to the input's channels (:64-67).  The track stays on the device from the
    upload to the download.  Returns OrderedDict name -> float32 [n_frames, n_channels].

    With `references` (name -> [n_frames, n_channels] at `rate`) the estimates are scored by eval_track at `rate` (the
    reference's museval.eval_mus_track, :71) with BSS Eval `mode` ("v4" or "v3"), written to <results_dir>/<track_name>.json
    when results_dir is given, and the per-target median SDR / ISR / SIR / SAR is printed."""
    import torch
    import wun
    assert len(audio.shape) == 2
    n_frames, mix_channels = int(audio.shape[0]), int(audio.shape[1])
    sr = int(model_config["expected_sr"])
    mix = torch.from_numpy(np.ascontiguousarray(_model_channels(model_config, audio))).cuda()
    preds = _separate_on_device(model_config, separator, wun.resample(mix, rate, sr))
    back = torch.stack([wun.resample(preds[k].contiguous(), sr, rate)[:n_frames] for k in range(preds.shape[0])])
    result = back.cpu().numpy()
    if model_config["mono_downmix"] and mix_channels > 1:
        result = np.tile(result, [1, 1, mix_channels])
    pred_audio = OrderedDict((name, result[k]) for k, name in enumerate(model_config["source_names"]))
    if references is not None:
        scores = eval_track(references, pred_audio, rate, output_dir=results_dir, track_name=track_name, mode=mode)
        for target in scores["targets"]:
            print("%s ==> %s" % (target["name"], "  ".join(
                "%s: %.3f" % (m, np.nanmedian([f["metrics"][m] for f in target["frames"]]))
                for m in ("SDR", "ISR", "SIR", "SAR"))))
    return pred_audio


def load_separator(model_config, load_model):
    """A separator holding the variables of `load_model` (a TF-V2 checkpoint prefix - written by Training.train or by the
    reference - or a round-1 .npz; reference restore: Evaluate.py:55-57); None leaves them uninitialised.  The class
    follows model_config["network"] as in the reference (Evaluate.py:27-32): a UnetAudioSeparator for "unet", a
    UnetSpectrogramSeparator (inference only) for "unet_spectrogram"."""
    if model_config["network"] == "unet":
        from Models.UnetAudioSeparator import UnetAudioSeparator as Separator
    elif model_config["network"] == "unet_spectrogram":
        from Models.UnetSpectrogramSeparator import UnetSpectrogramSeparator as Separator
    else:
        raise NotImplementedError
    separator = Separator(model_config)
    in_shape, _ = separator.get_padding(np.array([1, model_config["num_frames"], 0]))
    if load_model is not None:
        import TFCheckpoint
        TFCheckpoint.restore_separator(load_model, separator, int(in_shape[1]), with_optimizer=False)
    return separator


def produce_musdb_source_estimates(model_config, load_model, musdb_path, output_path, subsets=None, mode="v4"):
    """The reference's produce_musdb_source_estimates (Evaluate.py:147-159) over the MUSDB18 WAV layout: every track of
    `subsets` (both, as mus.run(subsets=None) does) is separated at its own rate with predict(), scored against its stems,
    and written as musdb and museval would: float32 WAV estimates in <output_path>/<subset>/<track>/<source>.wav and the BSS
    Eval JSON (BSS Eval `mode`, "v4" or "v3") in <output_path>/<subset>/<track>.json (Datasets.estimate_path /
    museval_json_dir).  The reference
    accompaniment is bass + drums + other, unclipped.  With torch.distributed every rank separates its share of the windows
    and rank 0 writes."""
    import Datasets
    from Predict import read_wav, write_wav
    print("Evaluating trained model saved at " + str(load_model) + " on MUSDB and saving source estimate audio to "
          + str(output_path))
    rank, _ = parallel.world()
    separator = load_separator(model_config, load_model)
    for subset in (subsets or Datasets.MUSDB_SUBSETS):
        for track in Datasets.musdb_tracks(musdb_path, subset):
            rate, mix = read_wav(track["mix"])
            if mix.shape[1] == 1 and not model_config["mono_downmix"]:
                raise ValueError("%s is mono: a stereo model's estimates cannot be scored against it (MUSDB18 is stereo)"
                                 % track["mix"])
            refs = OrderedDict((s, read_wav(track[s])[1]) for s in Datasets.MUSDB_STEMS)
            acc = refs[Datasets.ACCOMPANIMENT_STEMS[0]]
            for s in Datasets.ACCOMPANIMENT_STEMS[1:]:
                acc = acc + refs[s]
            refs["accompaniment"] = acc
            results_dir = Datasets.museval_json_dir(output_path, subset) if rank == 0 else None
            preds = predict(model_config, separator, mix, rate, references=refs, results_dir=results_dir,
                            track_name=track["name"], mode=mode)
            if rank == 0:
                for name, audio in preds.items():
                    path = Datasets.estimate_path(output_path, subset, track["name"], name)
                    os.makedirs(os.path.dirname(path), exist_ok=True)
                    write_wav(path, audio, rate)


def produce_source_estimates(model_config, load_model, mix_audio, separator=None):
    """Predict.py's work-horse for arrays already at expected_sr (reference Evaluate.py:161-193 minus file I/O): builds
    the separator with load_separator and separates `mix_audio`."""
    if separator is None:
        separator = load_separator(model_config, load_model)
    return predict_track(model_config, separator, mix_audio)


def _device_bss_eval(references, estimates, win, hop, mode="v4"):
    """[nsrc, N, nchan] float arrays -> numpy float64 [4 (SDR, ISR, SIR, SAR), nsrc, nwin] from wun.bss_eval."""
    import torch
    import wun
    ref = torch.from_numpy(np.ascontiguousarray(references, dtype=np.float32)).cuda()
    est = torch.from_numpy(np.ascontiguousarray(estimates, dtype=np.float32)).cuda()
    return torch.stack(wun.bss_eval(ref, est, win, hop, mode=mode)).cpu().numpy()


def _pad_or_truncate(estimates, n):
    if estimates.shape[1] >= n:
        return estimates[:, :n]
    return np.pad(estimates, ((0, 0), (0, n - estimates.shape[1]), (0, 0)))


BSS_MODES = ("v4", "v3")


def check_mode(mode):
    if mode not in BSS_MODES:
        raise ValueError("mode=%r: must be one of %s" % (mode, ", ".join(BSS_MODES)))


def evaluate(references, estimates, win=44100, hop=44100, mode="v4"):
    """museval.evaluate(references, estimates, win, hop, mode=mode, padding=True): arrays [nsrc, n_samples, nchan];
    estimates are cut or zero-extended to the references' length.  mode "v4" solves the distortion filters once over the
    track, "v3" again for every frame.  Returns SDR, ISR, SIR, SAR, each [nsrc, nwin]."""
    check_mode(mode)
    references = np.asarray(references)
    estimates = _pad_or_truncate(np.asarray(estimates), references.shape[1])
    args = (references, estimates, int(win), int(hop))         # v4 keeps the four-argument call
    sdr, isr, sir, sar = _device_bss_eval(*args) if mode == "v4" else _device_bss_eval(*args, mode=mode)
    return sdr, isr, sir, sar


def eval_track(references, estimates, rate, output_dir=None, track_name=None, mode="v4"):
    """museval.eval_mus_track with arrays: `references` and `estimates` map source names to [n_samples, nchan] arrays;
    the references' order plays the role of track.targets, and only names present in both are scored.  When vocals and
    accompaniment are both present, accompaniment leaves the list and the pair is scored as its own 2-source problem,
    reported last; the remaining targets (vocals included) are scored together if there are at least two of them, and
    all but vocals are reported from that problem.  Frames are one second at `rate` (win = hop), scored with BSS Eval
    `mode` (evaluate).  Returns
    {"targets": [...]} in museval's JSON layout (NaN for silent frames) and writes it to <output_dir>/<track_name>.json
    when output_dir is given."""
    check_mode(mode)
    win = hop = int(rate)
    names = [n for n in references if n in estimates]
    has_acc = "vocals" in names and "accompaniment" in names
    scenarios = []                  # (scored together, reported)
    rest = [n for n in names if not (has_acc and n == "accompaniment")]
    if len(rest) >= 2:
        scenarios.append((rest, [n for n in rest if not (has_acc and n == "vocals")]))
    if has_acc:
        scenarios.append((["vocals", "accompaniment"], ["vocals", "accompaniment"]))
    targets = []
    for group, report in scenarios:
        ref = np.stack([np.asarray(references[n]) for n in group])
        est = np.stack([_pad_or_truncate(np.asarray(estimates[n])[None], ref.shape[1])[0] for n in group])
        sdr, isr, sir, sar = evaluate(ref, est, win, hop, mode=mode)
        for k, name in enumerate(group):
            if name not in report:
                continue
            frames = [{"time": float(t * hop) / rate, "duration": float(win) / rate,
                       "metrics": {"SDR": float(sdr[k, t]), "SIR": float(sir[k, t]), "SAR": float(sar[k, t]),
                                   "ISR": float(isr[k, t])}}
                      for t in range(sdr.shape[1])]
            targets.append({"name": name, "frames": frames})
    scores = {"targets": targets}
    if output_dir is not None:
        os.makedirs(output_dir, exist_ok=True)
        with open(os.path.join(output_dir, "%s.json" % (track_name or "track")), "w") as f:
            json.dump(scores, f, indent=2, allow_nan=True)
    return scores


def _device_bss_eval_ex(references, estimates, win, hop, compute_permutation, framewise_filters, sources_version):
    """[nsrc, N, nchan] float arrays -> (numpy float64 [4 (SDR, ISR, SIR, SAR), nsrc, nwin], int64 popt [nsrc, nwin]) from
    wun.bss_eval; popt is the identity without compute_permutation."""
    import torch
    import wun
    ref = torch.from_numpy(np.ascontiguousarray(references, dtype=np.float32)).cuda()
    est = torch.from_numpy(np.ascontiguousarray(estimates, dtype=np.float32)).cuda()
    out = wun.bss_eval(ref, est, win, hop, mode="v3" if framewise_filters else "v4", permutation=compute_permutation,
                       sources_version=sources_version)
    metrics = torch.stack(out[:4]).cpu().numpy()
    if compute_permutation:
        return metrics, out[4].cpu().numpy()
    return metrics, np.tile(np.arange(metrics.shape[1], dtype=np.int64)[:, None], (1, metrics.shape[2]))


def _sources(x, what):
    """[nsrc, nsampl] gets a channel axis: [nsrc, nsampl, 1]."""
    x = np.asarray(x)
    if x.ndim == 2:
        x = x[:, :, None]
    if x.ndim != 3:
        raise ValueError("%s: expected [nsrc, nsampl] or [nsrc, nsampl, nchan], got shape %s" % (what, x.shape))
    return x


def bss_eval(reference_sources, estimated_sources, window=2 * 44100, hop=1.5 * 44100, compute_permutation=False,
             filters_len=512, framewise_filters=False, bsseval_sources_version=False):
    """museval.metrics.bss_eval on the GPU: arrays [nsrc, nsampl(, nchan)] of equal shape.  framewise_filters solves the
    512-tap filters for every frame (mode="v3") instead of once over the signal (mode="v4"); compute_permutation scores every
    (reference, estimate) pair and keeps, per frame, the permutation with the largest mean SIR; bsseval_sources_version
    scores the "sources" decomposition (ISR is NaN).  Returns SDR, ISR, SIR, SAR, each [nsrc, nwin] with row j estimate j,
    and popt [nsrc, nwin], the reference each estimate is scored against (the identity without compute_permutation)."""
    if filters_len != 512:
        raise ValueError("filters_len=%r: the GPU solves museval's 512-tap filters only" % (filters_len,))
    ref, est = _sources(reference_sources, "reference_sources"), _sources(estimated_sources, "estimated_sources")
    if ref.shape != est.shape:
        raise ValueError("estimated_sources %s must have the shape of reference_sources %s" % (est.shape, ref.shape))
    metrics, popt = _device_bss_eval_ex(ref, est, int(window), int(hop), bool(compute_permutation), bool(framewise_filters),
                                        bool(bsseval_sources_version))
    sdr, isr, sir, sar = metrics
    return sdr, isr, sir, sar, popt


def bss_eval_sources(reference_sources, estimated_sources, compute_permutation=True):
    """museval.metrics.bss_eval_sources: the whole signal as one frame, filters over it, "sources" decomposition.
    Returns SDR, SIR, SAR, perm, each [nsrc, 1]."""
    n = np.shape(reference_sources)[1]
    sdr, _, sir, sar, perm = bss_eval(reference_sources, estimated_sources, n, n, compute_permutation,
                                      framewise_filters=True, bsseval_sources_version=True)
    return sdr, sir, sar, perm


def bss_eval_sources_framewise(reference_sources, estimated_sources, window=30 * 44100, hop=15 * 44100,
                               compute_permutation=False):
    """museval.metrics.bss_eval_sources_framewise: filters per frame, "sources" decomposition.  Returns SDR, SIR, SAR,
    perm, each [nsrc, nwin]."""
    sdr, _, sir, sar, perm = bss_eval(reference_sources, estimated_sources, window, hop, compute_permutation,
                                      framewise_filters=True, bsseval_sources_version=True)
    return sdr, sir, sar, perm


def bss_eval_images(reference_sources, estimated_sources, compute_permutation=True):
    """museval.metrics.bss_eval_images: the whole signal as one frame, filters over it, images decomposition.  Returns
    SDR, ISR, SIR, SAR, perm, each [nsrc, 1]."""
    n = np.shape(reference_sources)[1]
    return bss_eval(reference_sources, estimated_sources, n, n, compute_permutation, framewise_filters=True,
                    bsseval_sources_version=False)


def bss_eval_images_framewise(reference_sources, estimated_sources, window=30 * 44100, hop=15 * 44100,
                              compute_permutation=False):
    """museval.metrics.bss_eval_images_framewise: filters per frame, images decomposition.  Returns SDR, ISR, SIR, SAR,
    perm, each [nsrc, nwin]."""
    return bss_eval(reference_sources, estimated_sources, window, hop, compute_permutation, framewise_filters=True,
                    bsseval_sources_version=False)


def compute_mean_metrics(json_folder, compute_averages=True, metric="SDR"):
    """The reference's compute_mean_metrics (Evaluate.py:195-232): per target, (median, MAD, mean, SD) of `metric` over
    every frame of every <track>.json in json_folder, ignoring NaN; with compute_averages=False the frame values."""
    files = glob.glob(os.path.join(json_folder, "*.json"))
    inst_list = None
    print("Found " + str(len(files)) + " JSON files to evaluate...")
    for path in files:
        if "test.json" in path:
            print("Found test JSON, skipping...")
            continue
        with open(path, "r") as f:
            js = json.load(f)
        if inst_list is None:
            inst_list = [list() for _ in range(len(js["targets"]))]
        for i in range(len(js["targets"])):
            inst_list[i].extend([float(f["metrics"][metric]) for f in js["targets"][i]["frames"]])
    inst_list = [np.array(perf) for perf in inst_list]
    if compute_averages:
        return [(np.nanmedian(perf), np.nanmedian(np.abs(perf - np.nanmedian(perf))), np.nanmean(perf), np.nanstd(perf))
                for perf in inst_list]
    return inst_list
