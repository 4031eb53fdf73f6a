"""numpy restatement of the reference's data preparation and test loss, for the dataset tests (CPU only).

stage_track      write_records (Datasets.py:43-93) for one track: read (16-bit PCM / 32768, float32 as is), the voice
                 accompaniment clip(bass + drums + other, -1, 1) (Datasets.py:259-262), librosa's mono mean, kaiser_best
                 resampling (resample_oracle), tiling of a mono stem for a stereo model, zero padding at both ends
take_all_snippets / batch_and_drop_remainder   a literal transcription of Datasets.py:21-25 and :213
test_loss        Test.py:57-79's running mean for any given forward function
"""
import numpy as np
import scipy.io.wavfile

from oracle import resample_oracle


def read(path):
    rate, data = scipy.io.wavfile.read(path)
    audio = data.astype(np.float32) / np.float32(32768) if data.dtype == np.int16 else data.astype(np.float32)
    return int(rate), audio.reshape(audio.shape[0], -1)


def stage_track(paths, source_names, mono_downmix, expected_sr, t_in, t_out, tables):
    """{key: float32 [padded frames, C]} for key in source_names + ["mix"]; `paths` maps mix / sources (or bass, drums,
    other for a summed accompaniment) to WAV files; tables(sr_in, sr_out) -> (win, delta, precision)."""
    raw = {}
    rate = None
    for key, path in paths.items():
        rate, raw[key] = read(path)
    if "accompaniment" in source_names and "accompaniment" not in raw:
        raw["accompaniment"] = np.clip(raw["bass"] + raw["drums"] + raw["other"], -1.0, 1.0)
    pad = (t_in - t_out) // 2
    out = {}
    for key in list(source_names) + ["mix"]:
        audio = raw[key]
        if mono_downmix:
            audio = np.mean(audio, axis=1, keepdims=True)
        if rate != expected_sr:
            win, delta, precision = tables(rate, expected_sr)
            audio = resample_oracle.resample(audio, rate, expected_sr, win, delta, precision)
        if not mono_downmix and audio.shape[1] == 1:
            audio = np.tile(audio, [1, 2])
        out[key] = np.pad(audio, [(pad, pad), (0, 0)], mode="constant", constant_values=0.0)
    return out


def take_all_snippets(length, t_in, t_out):
    """tf.range(0, length - T_in, delta=T_out): start frames of a padded track."""
    return list(range(0, length - t_in, t_out))


def batch_and_drop_remainder(items, batch):
    return [items[i:i + batch] for i in range(0, len(items) - batch + 1, batch)]


def partition_batches(tracks, source_names, t_in, t_out, batch):
    """Every full batch of a partition: tracks (staged dicts) in order, their snippets in order; each batch is (mix
    [B, T_in, C], {source: [B, T_out, C]}) with the targets centre-cropped (Utils.crop_sample)."""
    crop = (t_in - t_out) // 2
    snippets = [(t, s) for t in tracks for s in take_all_snippets(t["mix"].shape[0], t_in, t_out)]
    out = []
    for group in batch_and_drop_remainder(snippets, batch):
        mix = np.stack([t["mix"][s:s + t_in] for t, s in group])
        targets = {k: np.stack([t[k][s + crop:s + crop + t_out] for t, s in group]) for k in source_names}
        out.append((mix, targets))
    return out


def test_loss(batches, forward, source_names):
    """Test.py:57-79: per batch curr = sum_k mean((target_k - estimate_k)^2) / K (float64 here), then total += (1 / n) *
    (curr - total).  `forward(mix)` -> {source: [B, T_out, C]}."""
    total = 0.0
    for n, (mix, targets) in enumerate(batches, start=1):
        est = forward(mix)
        curr = sum(float(np.mean((targets[k].astype(np.float64) - np.asarray(est[k], np.float64)) ** 2))
                   for k in source_names) / float(len(source_names))
        total = total + (1.0 / float(n)) * (curr - total)
    return total
