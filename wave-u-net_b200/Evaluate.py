"""Windowed inference with the H100 engine: drop-in for the tiling half of the reference's Evaluate.py.

predict_track() keeps the semantics of /root/reference/Evaluate.py:82-145 exactly -
  mono-mix or channel duplication (:98-102), zero-extension of short inputs (:107-111), (T_in-T_out)//2 context
  padding on both sides (:121-122), hop = T_out, the LAST window shifted back to end at the final frame (:127-128),
  plain overwrite of overlapping frames (:138-139), removal of the extension (:142-143)
- but the windows, which the reference feeds one by one through sess.run (:134), are gathered ON THE DEVICE, pushed
through the network as batches, and scattered back on the device; with torch.distributed initialised the window list
is split over the ranks (no collective on the data path, results all-gathered at the end).

Audio file I/O, resampling and museval scoring of the reference (librosa / musdb / museval, Evaluate.py:16-80,147-231)
are out of scope (SURVEY section 2): predict_track works on arrays already at model_config["expected_sr"].
"""
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
    Models.UnetAudioSeparator.UnetAudioSeparator holding variables.  Returns OrderedDict name -> [n_frames, C]."""
    import torch
    assert len(mix_audio.shape) == 2
    mix_audio = np.asarray(mix_audio, dtype=np.float32)
    if model_config["mono_downmix"]:
        mix_audio = np.mean(mix_audio, axis=1, keepdims=True)
    elif mix_audio.shape[1] == 1:
        mix_audio = np.tile(mix_audio, [1, 2])

    in_shape, out_shape = separator.get_padding(np.array([1, model_config["num_frames"], 0]))
    t_in, t_out = int(in_shape[1]), int(out_shape[1])
    extra_pad = 0
    if mix_audio.shape[0] < t_in:
        extra_pad = t_in - mix_audio.shape[0]
        mix_audio = np.pad(mix_audio, [(0, extra_pad), (0, 0)], mode="constant", constant_values=0.0)
    n_frames, C = mix_audio.shape
    pad = (t_in - t_out) // 2                                   # context on both sides (Evaluate.py:121-122), zero-filled ON the device

    eng = separator.engine(input_frames=t_in)
    names = list(model_config["source_names"])
    K = len(names)
    starts_all = window_starts(n_frames, t_out)
    rank, ws = parallel.world()
    lo, hi = parallel.shard_range(len(starts_all), rank, ws)

    padded_d = torch.zeros((n_frames + 2 * pad, C), dtype=torch.float32, device=device)
    padded_d[pad:pad + n_frames].copy_(torch.from_numpy(np.ascontiguousarray(mix_audio)))      # (a host-side np.pad of a 3-minute
    # track costs as much as a third of the whole separation)
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
    result = preds.cpu().numpy()
    if extra_pad > 0:
        result = result[:, :-extra_pad, :]
    return OrderedDict((name, result[k]) for k, name in enumerate(names))


def produce_source_estimates(model_config, load_model, mix_audio, separator=None):
    """Predict.py's work-horse (reference Evaluate.py:161-193 minus file I/O): builds the separator, loads variables
    from `load_model` (a TF-V2 checkpoint prefix - written by Training.train or by the reference - or a round-1 .npz;
    reference restore: Evaluate.py:55-57) and separates `mix_audio`."""
    from Models.UnetAudioSeparator import UnetAudioSeparator
    if separator is None:
        separator = UnetAudioSeparator(model_config)
        in_shape, _ = separator.get_padding(np.array([1, model_config["num_frames"], 0]))
        if load_model is not None:
            import TFCheckpoint
            TFCheckpoint.restore_separator(load_model, separator, int(in_shape[1]), with_optimizer=False)
    return predict_track(model_config, separator, mix_audio)
